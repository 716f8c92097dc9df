// Shared helpers for the turboprune_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/turboprune_b200.h"

namespace tp {

void set_last_cuda_error(cudaError_t e, const char* where);

#define TP_CUDA_CHECK(expr)                                             \
  do {                                                                  \
    cudaError_t _e = (expr);                                            \
    if (_e != cudaSuccess) {                                            \
      ::tp::set_last_cuda_error(_e, #expr);                             \
      return TP_ERR_CUDA;                                               \
    }                                                                   \
  } while (0)

#define TP_LAUNCH_CHECK() TP_CUDA_CHECK(cudaGetLastError())

int sm_count();                       // cached
// Make the device that owns `p` current on the calling thread (binds its primary context).
// Needed because entry points are also called from torch's autograd thread, where no CUDA
// context may be current yet and the driver API (cuTensorMapEncode*) would fail.
int bind_device_of(const void* p);
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Programmatic dependent launch (PDL) for the kernels of the train step.  A step is ~540 dependent launches; without PDL
// every one of them pays grid drain + launch + ramp-up in full.  With it the next grid's CTAs are scheduled while the
// previous grid is still finishing (as soon as every CTA of the previous grid has STARTED and executed
// `griddepcontrol.launch_dependents`), and block in `griddepcontrol.wait` until that grid has completed and its memory
// is visible.  Rules kept here: (1) a kernel launched through launch() executes pdl_wait() before its first global
// access (pdl_enter() at the top, or after a prologue that touches only parameters / shared memory);
// (2) the trigger comes first, so grids queue up behind each other only as deep as the SMs have room for.
// Off by default; TP_PDL=1 turns it on.
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_enter() { pdl_trigger(); pdl_wait(); }

template <typename... KA, typename... A>
inline cudaError_t launch(void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KA>(args)...);
}
#endif

// A bump allocator over the caller's workspace.
struct Arena {
  char* base; size_t cap; size_t off;
  Arena(void* p, size_t bytes) : base((char*)p), cap(bytes), off(0) {}
  void* take(size_t bytes, size_t align = 256) {
    size_t o = align_up(off, align);
    if (o + bytes > cap) return nullptr;
    off = o + bytes;
    return base + o;
  }
};

// Segment table shared by the pruning / optimizer kernels: a list of fp32 tensors
// processed by ONE launch (no torch.cat — SURVEY K11).
struct Seg {
  const float* w;       // weights (or noise draw)
  const float* g;       // grads (nullable)
  const float* m;       // mask in
  float*       mo;      // mask out / second output (nullable)
  float*       buf;     // momentum buffer (optimizer only)
  long long    n;       // elements
  long long    start;   // global element offset of this segment
  long long    tile0;   // first tile index of this segment
};

constexpr int kTileElems = 4096;   // elements per CTA work item in the segment sweeps

// Upload a segment table (host arrays of device pointers) into workspace memory.
// Returns the number of tiles through *tiles_out.
int upload_segs(Arena& ar, const void* const* w, const void* const* g, const void* const* m,
                void* const* mo, void* const* buf, const int64_t* numel, int n_seg,
                Seg** dev_out, long long* tiles_out, long long* total_out, cudaStream_t st);

__device__ __forceinline__ int find_seg(const Seg* __restrict__ segs, int n_seg, long long tile) {
  int lo = 0, hi = n_seg - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (segs[mid].tile0 <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ int find_seg_by_elem(const Seg* __restrict__ segs, int n_seg, long long e) {
  int lo = 0, hi = n_seg - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (segs[mid].start <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// streaming 16-byte accesses (read-once data: keep it out of L1)
__device__ __forceinline__ float4 ld_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(float4* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

}  // namespace tp
