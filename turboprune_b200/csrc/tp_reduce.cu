// Gradient exchange over NVLink / NVSwitch peer memory (sm_90a).
//
// Replaces the c10d Reducer's per-bucket  grad/W -> ncclAllReduce(SUM) -> copy-back
// (harness_definitions/base_harness.py:81 of the reference; SURVEY K7) with ONE kernel per
// bucket that reads the peers' bucket copies directly through their mapped (symmetric)
// addresses, sums them in fixed rank order 0..W-1 (so every rank gets bit-identical results),
// scales by 1/W, multiplies by the pruning mask and writes the local result.  No NCCL call on
// the data path.
//
//   algo 0 — one-shot pull : every rank reads all W copies of the whole bucket
//                            (latency-optimal; (W-1)*S inbound bytes per GPU)
//   algo 1 — two-shot      : rank r reduces shard r from all W copies and PUSHES the result into
//                            shard r of every peer's buffer (in place: only rank r ever reads
//                            shard r), then everyone copies its now fully reduced buffer out
//                            (bandwidth-optimal: 2*S*(W-1)/W bytes per GPU over NVLink)
//
//   NVLS (tp_p2p_allreduce_nvls) — the two-shot schedule with both halves done INSIDE the NVSwitch: rank r issues
//                            multimem.ld_reduce on the multicast address of shard r (the switch fetches the W
//                            replicas and returns their sum), scales / masks it and multimem.st's it back (the
//                            switch writes all W replicas).  S/W bytes in and S/W bytes out per GPU instead of
//                            S*(W-1)/W each way; the summation order is the switch's (see the header).
//
// Cross-GPU synchronisation: per-CTA flag barriers on signal pads living in the symmetric
// allocation.  slot[b*W + src] in rank dst's pad is set 0->1 by CTA b of rank src
// (atom.cas.release.sys) and consumed 1->0 by CTA b of rank dst (atom.cas.acquire.sys), so a
// pad is reusable without epochs.  CTA b touches the same element ranges on every rank, hence
// no grid-wide barrier is needed.  All spins are bounded.
#include "tp_common.cuh"

namespace tp {

constexpr int kMaxWorld = 16;
constexpr int kRedThreads = 512;
constexpr int kPadSlots = 1024;          // uint32 slots per signal pad (4 KiB)

struct ReduceParams {
  float* bufs[kMaxWorld];
  uint32_t* pads[kMaxWorld];
  int rank, world;
  long long numel;
  const float* mask;
  float scale;
  float* out;
  long long spin_limit;        // clock64 ticks
  int* status;
};

__device__ __forceinline__ uint32_t cas_release_sys(uint32_t* addr, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.global.release.sys.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(addr), "r"(cmp), "r"(val) : "memory");
  return old;
}
__device__ __forceinline__ uint32_t cas_acquire_sys(uint32_t* addr, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(addr), "r"(cmp), "r"(val) : "memory");
  return old;
}
__device__ __forceinline__ float4 ld_sys(const float4* p) {
  float4 r;
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ float ld_sys1(const float* p) {
  float r;
  asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(r) : "l"(p) : "memory");
  return r;
}

// Every CTA b of every rank meets here.  Returns false on timeout.
__device__ __forceinline__ bool peer_barrier(const ReduceParams& p, int* s_fail) {
  __syncthreads();                       // this CTA's prior reads/writes are done
  const int t = threadIdx.x;
  if (t < p.world) {
    __threadfence_system();
    const long long t0 = clock64();
    uint32_t* theirs = p.pads[t] + (size_t)blockIdx.x * p.world + p.rank;
    while (cas_release_sys(theirs, 0u, 1u) != 0u) {
      if (clock64() - t0 > p.spin_limit) { *s_fail = 1; break; }
    }
    uint32_t* mine = p.pads[p.rank] + (size_t)blockIdx.x * p.world + t;
    while (cas_acquire_sys(mine, 1u, 0u) != 1u) {
      if (clock64() - t0 > p.spin_limit) { *s_fail = 1; break; }
    }
  }
  __syncthreads();
  return *s_fail == 0;
}

// Sum `W` replicas of up to U float4 elements per thread (indices i0 + u*stride < end) in fixed
// rank order, with all U loads of a replica in flight together (NVLink latency ~2 us).
template <int U>
__device__ __forceinline__ void reduce_group(const ReduceParams& p, long long i0, long long stride, long long end,
                                             float4 (&acc)[U], bool (&ok)[U]) {
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const long long i = i0 + u * stride;
    ok[u] = i < end;
    acc[u] = ok[u] ? ld_sys((const float4*)p.bufs[0] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll 1
  for (int j = 1; j < p.world; ++j) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * stride;
      v[u] = ok[u] ? ld_sys((const float4*)p.bufs[j] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) { acc[u].x += v[u].x; acc[u].y += v[u].y; acc[u].z += v[u].z; acc[u].w += v[u].w; }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    acc[u].x *= p.scale; acc[u].y *= p.scale; acc[u].z *= p.scale; acc[u].w *= p.scale;
    if (p.mask && ok[u]) {
      const float4 m = ((const float4*)p.mask)[i0 + u * stride];
      acc[u].x *= m.x; acc[u].y *= m.y; acc[u].z *= m.z; acc[u].w *= m.w;
    }
  }
}

template <int ALGO>
__global__ void __launch_bounds__(kRedThreads) k_p2p_allreduce(const __grid_constant__ ReduceParams p) {
  __shared__ int s_fail;
  if (threadIdx.x == 0) s_fail = 0;
  __syncthreads();
  if (!peer_barrier(p, &s_fail)) { if (threadIdx.x == 0 && p.status) atomicExch(p.status, 1); return; }

  const int W = p.world;
  const long long n4 = p.numel >> 2;                 // float4 body; tail handled by CTA 0
  const long long gsz = (long long)gridDim.x * blockDim.x;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;

  if (ALGO == 0) {
    constexpr int U = 4;
    for (long long i = gid; i < n4; i += U * gsz) {
      float4 acc[U]; bool ok[U];
      reduce_group<U>(p, i, gsz, n4, acc, ok);
#pragma unroll
      for (int u = 0; u < U; ++u) if (ok[u]) ((float4*)p.out)[i + u * gsz] = acc[u];
    }
    if (blockIdx.x == 0) {
      for (long long i = (n4 << 2) + threadIdx.x; i < p.numel; i += blockDim.x) {
        float acc = ld_sys1(p.bufs[0] + i);
        for (int j = 1; j < W; ++j) acc += ld_sys1(p.bufs[j] + i);
        acc *= p.scale;
        if (p.mask) acc *= p.mask[i];
        p.out[i] = acc;
      }
    }
  } else {
    // shard boundaries in float4 units; the scalar tail belongs to the last rank
    const long long per = (n4 + W - 1) / W;
    const long long s0 = min(n4, per * p.rank), s1 = min(n4, s0 + per);
    constexpr int U = 4;
    for (long long i = s0 + gid; i < s1; i += U * gsz) {
      float4 acc[U]; bool ok[U];
      reduce_group<U>(p, i, gsz, s1, acc, ok);
#pragma unroll 1
      for (int j = 0; j < W; ++j) {                     // push to every replica
#pragma unroll
        for (int u = 0; u < U; ++u) if (ok[u]) ((float4*)p.bufs[j])[i + u * gsz] = acc[u];
      }
    }
    if (p.rank == W - 1 && blockIdx.x == 0) {
      for (long long i = (n4 << 2) + threadIdx.x; i < p.numel; i += blockDim.x) {
        float acc = ld_sys1(p.bufs[0] + i);
        for (int j = 1; j < W; ++j) acc += ld_sys1(p.bufs[j] + i);
        acc *= p.scale;
        if (p.mask) acc *= p.mask[i];
        for (int j = 0; j < W; ++j) p.bufs[j][i] = acc;
      }
    }
    if (!peer_barrier(p, &s_fail)) { if (threadIdx.x == 0 && p.status) atomicExch(p.status, 1); return; }
    // my buffer now holds the full result: CTA b copies exactly the ranges the CTAs b wrote
    if (p.out != p.bufs[p.rank]) {
      for (int j = 0; j < W; ++j) {
        const long long r0 = min(n4, per * j), r1 = min(n4, r0 + per);
        for (long long i = r0 + gid; i < r1; i += gsz) ((float4*)p.out)[i] = ld_sys((const float4*)p.bufs[p.rank] + i);
      }
      if (blockIdx.x == 0)
        for (long long i = (n4 << 2) + threadIdx.x; i < p.numel; i += blockDim.x) p.out[i] = ld_sys1(p.bufs[p.rank] + i);
    }
  }
  // one-shot: nobody may refill its bucket buffer until every peer has finished reading it.  (Two-shot needs no third
  // barrier: every read of a peer's buffer happens before the second one.)
  if (ALGO == 0) { if (!peer_barrier(p, &s_fail)) { if (threadIdx.x == 0 && p.status) atomicExch(p.status, 1); } }
}

// ---- NVLS: in-switch reduction and broadcast through the multicast mapping of the symmetric bucket ------------
__device__ __forceinline__ float4 mm_ld_reduce_add(const float4* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void mm_st(float4* mc, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__global__ void __launch_bounds__(kRedThreads) k_p2p_allreduce_nvls(const __grid_constant__ ReduceParams p, float* mc) {
  __shared__ int s_fail;
  if (threadIdx.x == 0) s_fail = 0;
  __syncthreads();
  if (!peer_barrier(p, &s_fail)) { if (threadIdx.x == 0 && p.status) atomicExch(p.status, 1); return; }
  const int W = p.world;
  const long long n4 = p.numel >> 2;
  const long long gsz = (long long)gridDim.x * blockDim.x;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = (n4 + W - 1) / W;
  const long long s0 = min(n4, per * p.rank), s1 = min(n4, s0 + per);
  constexpr int U = 4;
  for (long long i = s0 + gid; i < s1; i += U * gsz) {
    float4 acc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long j = i + u * gsz;
      acc[u] = j < s1 ? mm_ld_reduce_add((const float4*)mc + j) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long j = i + u * gsz;
      if (j >= s1) continue;
      acc[u].x *= p.scale; acc[u].y *= p.scale; acc[u].z *= p.scale; acc[u].w *= p.scale;
      if (p.mask) {
        const float4 m = ((const float4*)p.mask)[j];
        acc[u].x *= m.x; acc[u].y *= m.y; acc[u].z *= m.z; acc[u].w *= m.w;
      }
      mm_st((float4*)mc + j, acc[u]);
    }
  }
  if (p.rank == W - 1 && blockIdx.x == 0) {          // scalar tail (numel % 4): plain peer loads / stores
    for (long long i = (n4 << 2) + threadIdx.x; i < p.numel; i += blockDim.x) {
      float acc = ld_sys1(p.bufs[0] + i);
      for (int j = 1; j < W; ++j) acc += ld_sys1(p.bufs[j] + i);
      acc *= p.scale;
      if (p.mask) acc *= p.mask[i];
      for (int j = 0; j < W; ++j) p.bufs[j][i] = acc;
    }
  }
  if (!peer_barrier(p, &s_fail)) { if (threadIdx.x == 0 && p.status) atomicExch(p.status, 1); return; }
  if (p.out != p.bufs[p.rank]) {
    for (int j = 0; j < W; ++j) {
      const long long r0 = min(n4, per * j), r1 = min(n4, r0 + per);
      for (long long i = r0 + gid; i < r1; i += gsz) ((float4*)p.out)[i] = ld_sys((const float4*)p.bufs[p.rank] + i);
    }
    if (blockIdx.x == 0)
      for (long long i = (n4 << 2) + threadIdx.x; i < p.numel; i += blockDim.x) p.out[i] = ld_sys1(p.bufs[p.rank] + i);
  }
}

// mask / scale only (world == 1 keeps the same call site): out = scale * mask * in
__global__ void __launch_bounds__(256) k_scale_mask(const float* __restrict__ in, const float* __restrict__ mask,
                                                    float scale, float* __restrict__ out, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += step) { float v = in[i] * scale; if (mask) v *= mask[i]; out[i] = v; }
}

}  // namespace tp

using namespace tp;

extern "C" {

static int fill_reduce_params(ReduceParams& p, void* const* peer_bufs, void* const* signal_pads, int rank, int world,
                              int64_t numel, const void* mask, float scale, void* out, int timeout_ms, int* status_dev) {
  if (!peer_bufs || !signal_pads || world < 2 || world > kMaxWorld || rank < 0 || rank >= world || numel < 0 || !out) return TP_ERR_INVALID;
  if ((((uintptr_t)out) & 15) || (mask && (((uintptr_t)mask) & 15))) return TP_ERR_INVALID;
  for (int j = 0; j < world; ++j) {
    if (!peer_bufs[j] || !signal_pads[j] || (((uintptr_t)peer_bufs[j]) & 15)) return TP_ERR_INVALID;
    p.bufs[j] = (float*)peer_bufs[j]; p.pads[j] = (uint32_t*)signal_pads[j];
  }
  p.rank = rank; p.world = world; p.numel = numel; p.mask = (const float*)mask; p.scale = scale; p.out = (float*)out;
  p.spin_limit = (long long)(timeout_ms > 0 ? timeout_ms : 10000) * 2000000ll;   // ~2 GHz ticks
  p.status = status_dev;
  return TP_OK;
}

// CTA count: bounded by the pad (slots / world) and by what saturates NVLink; must be equal on all ranks
static int reduce_blocks(int world, int64_t numel) {
  int blocks = kPadSlots / world;
  if (blocks > sm_count()) blocks = sm_count();
  const long long work = (numel / 4 + kRedThreads - 1) / kRedThreads;
  if (work < blocks) blocks = (int)(work > 0 ? work : 1);
  return blocks;
}

int tp_p2p_allreduce_mask(void* const* peer_bufs, void* const* signal_pads, int rank, int world,
                          int64_t numel, const void* mask, float scale, void* out,
                          int algo, int timeout_ms, int* status_dev, void* stream) {
  if (!peer_bufs || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || numel < 0 || !out) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  if (numel == 0) return TP_OK;
  if (world == 1) {
    long long g = (numel + 255) / 256; long long gm = (long long)sm_count() * 8;
    k_scale_mask<<<(unsigned)(g < gm ? g : gm), 256, 0, st>>>((const float*)peer_bufs[0], (const float*)mask, scale, (float*)out, numel);
    TP_LAUNCH_CHECK();
    return TP_OK;
  }
  ReduceParams p = {};
  int rc = fill_reduce_params(p, peer_bufs, signal_pads, rank, world, numel, mask, scale, out, timeout_ms, status_dev);
  if (rc) return rc;
  const int blocks = reduce_blocks(world, numel);
  if (algo == 0) k_p2p_allreduce<0><<<blocks, kRedThreads, 0, st>>>(p);
  else if (algo == 1) k_p2p_allreduce<1><<<blocks, kRedThreads, 0, st>>>(p);
  else return TP_ERR_INVALID;
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_p2p_allreduce_nvls(void* const* peer_bufs, void* const* signal_pads, void* multicast_buf, int rank, int world,
                          int64_t numel, const void* mask, float scale, void* out,
                          int timeout_ms, int* status_dev, void* stream) {
  if (!multicast_buf || (((uintptr_t)multicast_buf) & 15)) return TP_ERR_INVALID;
  if (numel == 0) return TP_OK;
  ReduceParams p = {};
  int rc = fill_reduce_params(p, peer_bufs, signal_pads, rank, world, numel, mask, scale, out, timeout_ms, status_dev);
  if (rc) return rc;
  k_p2p_allreduce_nvls<<<reduce_blocks(world, numel), kRedThreads, 0, (cudaStream_t)stream>>>(p, (float*)multicast_buf);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // extern "C"
