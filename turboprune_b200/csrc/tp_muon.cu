// Muon (torch.optim.Muon) for every hidden masked layer in a fixed number of launches: prepare (momentum, bf16 cast,
// transpose, padding, per-tile sums of squares), normalize, 3 * ns_steps Newton-Schulz GEMMs over one tile list that
// covers all layers, apply.  See include/turboprune_b200.h for the workspace's panel layout.
#include "tp_common.cuh"
#include "tp_ptx.cuh"
#include <cuda.h>

namespace tp {
using namespace ptx;

int make_tiled_map_bf16(CUtensorMap* m, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_rows);

constexpr int kMuonT = 64;                          // X tile edge = K block = one 128-B swizzle row of bf16
constexpr int kMuonPitch = kMuonT + 2;              // smem tile pitch (bf16) of the elementwise kernels

__device__ __forceinline__ int find_layer(const tp_muon_layer* __restrict__ L, int n, long long tile) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (L[mid].tile0 <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Element e (0..4095) of a 64 x 64 X tile -> (row ii, column jj): the walk that reads the fp32 [a][b] source coalesced
// (X = U^T: consecutive threads take consecutive X rows, i.e. consecutive source columns).
__device__ __forceinline__ void tile_elem(int e, bool trans, int& ii, int& jj) {
  if (trans) { ii = e & 63; jj = e >> 6; } else { ii = e >> 6; jj = e & 63; }
}

// Sum over the 256 threads in a fixed order (xor tree in each warp, warps in order): every CTA that folds the same
// values gets the same bits.
__device__ __forceinline__ float block_sum_fixed(float v, float* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
  __syncthreads();
  return t;
}

// Per layer: n = bf16(sqrt(sum of the partials folded in a fixed order)), then .clamp(min=eps) in fp32 and bf16 again.
// Run by the CTA that finishes the layer's tiles last (one fold per layer, whichever CTA it is).
__device__ __forceinline__ float layer_norm(const float* partial, long long tile0, int nt, float eps, float* s_red) {
  float v = 0.f;
  for (int k = threadIdx.x; k < nt; k += blockDim.x) v += __ldcg(partial + tile0 + k);
  const float ss = block_sum_fixed(v, s_red);
  float nf = __bfloat162float(__float2bfloat16_rn(__fsqrt_rn(ss)));               // ortho_grad.norm(): bf16
  if (!isnan(nf)) nf = __bfloat162float(__float2bfloat16_rn(fmaxf(nf, eps)));     // .clamp(min=eps)
  return nf;
}

__global__ void __launch_bounds__(256) k_muon_prepare(const tp_muon_layer* __restrict__ L, int n_layers,
                                                      __nv_bfloat16* __restrict__ ws, float* __restrict__ partial,
                                                      unsigned int* __restrict__ done, float* __restrict__ norms, float eps,
                                                      float w1, float omw1, float w2, float omw2, int nesterov) {
  pdl_enter();
  __shared__ unsigned short s[kMuonT * kMuonPitch];
  __shared__ float s_red[8];
  __shared__ bool s_last;
  const long long tile = blockIdx.x;
  const int li = find_layer(L, n_layers, tile);
  const tp_muon_layer ly = L[li];
  const int tpr = ly.np / kMuonT, local = (int)(tile - ly.tile0);
  const int ti = local / tpr, tj = local - ti * tpr;
  const bool trans = ly.trans != 0;
  const int m = trans ? ly.b : ly.a, n = trans ? ly.a : ly.b;
  const float* g = (const float*)ly.g;
  float* buf = (float*)ly.buf;
  const bool small1 = fabsf(w1) < 0.5f, small2 = fabsf(w2) < 0.5f;
  float sq = 0.f;
  for (int e = threadIdx.x; e < kMuonT * kMuonT; e += blockDim.x) {
    int ii, jj; tile_elem(e, trans, ii, jj);
    const int i = ti * kMuonT + ii, j = tj * kMuonT + jj;
    __nv_bfloat16 h = __float2bfloat16_rn(0.f);
    if (i < m && j < n) {
      const long long src = trans ? (long long)j * ly.b + i : (long long)i * ly.b + j;
      const float gv = g[src];
      const float bn = adamw_lerp(buf[src], gv, w1, omw1, small1);      // buf.lerp_(grad, 1 - momentum)
      buf[src] = bn;
      const float u = nesterov ? adamw_lerp(gv, bn, w2, omw2, small2) : bn;   // grad.lerp(buf, momentum)
      h = __float2bfloat16_rn(u);
      const float f = __bfloat162float(h);
      sq = fmaf(f, f, sq);
    }
    s[ii * kMuonPitch + jj] = __bfloat16_as_ushort(h);
  }
  __syncthreads();
  // the tile is 64 contiguous rows of 128 B in panel tj
  uint4* dst = reinterpret_cast<uint4*>(ws + (size_t)(ly.x0 + (long long)tj * ly.mp + ti * kMuonT) * kMuonT);
  for (int q = threadIdx.x; q < kMuonT * 8; q += blockDim.x) {
    const unsigned short* r = s + (q >> 3) * kMuonPitch + (q & 7) * 8;
    dst[q] = make_uint4(r[0] | ((unsigned)r[1] << 16), r[2] | ((unsigned)r[3] << 16), r[4] | ((unsigned)r[5] << 16),
                        r[6] | ((unsigned)r[7] << 16));
  }
  const float t = block_sum_fixed(sq, s_red);
  // the layer's last CTA to finish folds its partials (integer atomic on the count only: the fold order is fixed)
  const int nt = (ly.mp / kMuonT) * tpr;
  if (threadIdx.x == 0) {
    partial[tile] = t;
    __threadfence();
    s_last = atomicAdd(done + li, 1u) == (unsigned)(nt - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    const float nf = layer_norm(partial, ly.tile0, nt, eps, s_red);
    if (threadIdx.x == 0) { norms[li] = nf; done[li] = 0u; }       // the count restarts for the next step
  }
}

__global__ void __launch_bounds__(256) k_muon_normalize(const tp_muon_layer* __restrict__ L, int n_layers,
                                                        __nv_bfloat16* __restrict__ ws, const float* __restrict__ norms) {
  pdl_enter();
  const long long tile = blockIdx.x;
  const int li = find_layer(L, n_layers, tile);
  const tp_muon_layer ly = L[li];
  const int tpr = ly.np / kMuonT, local = (int)(tile - ly.tile0);
  const int ti = local / tpr, tj = local - ti * tpr;
  const float nf = norms[li];
  uint4* x = reinterpret_cast<uint4*>(ws + (size_t)(ly.x0 + (long long)tj * ly.mp + ti * kMuonT) * kMuonT);
  for (int q = threadIdx.x; q < kMuonT * 8; q += blockDim.x) {
    uint4 p = x[q];
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&p);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __bfloat1622float2(h[k]);
      h[k] = __floats2bfloat162_rn(__fdiv_rn(f.x, nf), __fdiv_rn(f.y, nf));    // div_: bf16(float(x) / float(n))
    }
    x[q] = p;
  }
}

__global__ void __launch_bounds__(256) k_muon_apply(const tp_muon_layer* __restrict__ L, int n_layers,
                                                    const __nv_bfloat16* __restrict__ ws, int which,
                                                    const double* __restrict__ lr_wd) {
  pdl_enter();
  __shared__ unsigned short s[kMuonT * kMuonPitch];
  const long long tile = blockIdx.x;
  const int li = find_layer(L, n_layers, tile);
  const tp_muon_layer ly = L[li];
  const int tpr = ly.np / kMuonT, local = (int)(tile - ly.tile0);
  const int ti = local / tpr, tj = local - ti * tpr;
  const bool trans = ly.trans != 0;
  const int m = trans ? ly.b : ly.a, n = trans ? ly.a : ly.b;
  const unsigned short* x = reinterpret_cast<const unsigned short*>(ws) +
                            (size_t)((which ? ly.x1 : ly.x0) + (long long)tj * ly.mp + ti * kMuonT) * kMuonT;
  for (int q = threadIdx.x; q < kMuonT * kMuonT / 2; q += blockDim.x) {
    const unsigned int v = reinterpret_cast<const unsigned int*>(x)[q];
    const int r = (2 * q) >> 6, c = (2 * q) & 63;
    s[r * kMuonPitch + c] = (unsigned short)(v & 0xFFFFu);
    s[r * kMuonPitch + c + 1] = (unsigned short)(v >> 16);
  }
  __syncthreads();
  // 1 - lr * wd and -(lr * ratio) as Python forms them: correctly rounded double ops (no contraction), then fp32
  const double lr = lr_wd[0];
  const float decay = __double2float_rn(__dsub_rn(1.0, __dmul_rn(lr, lr_wd[1])));
  const float alpha = __double2float_rn(-__dmul_rn(lr, ly.ratio));
  float* w = (float*)ly.w;
  for (int e = threadIdx.x; e < kMuonT * kMuonT; e += blockDim.x) {
    int ii, jj; tile_elem(e, trans, ii, jj);
    const int i = ti * kMuonT + ii, j = tj * kMuonT + jj;
    if (i < m && j < n) {
      const long long dst = trans ? (long long)j * ly.b + i : (long long)i * ly.b + j;
      const float o = __bfloat162float(__ushort_as_bfloat16(s[ii * kMuonPitch + jj]));
      w[dst] = fmaf(alpha, o, __fmul_rn(w[dst], decay));      // param.mul_(1 - lr wd); param.add_(O, alpha=-lr ratio)
    }
  }
}

// ---- Newton-Schulz GEMM ------------------------------------------------------------------------------------------
struct MuonTile { int a0, b0, sa, sb, nk, c0, o0, m0; };

constexpr int kNsStages = 4;
constexpr int kNsBox = kMuonT * kMuonT * 2;                     // 8 KB: one 64 x 64 bf16 box
constexpr int kNsStg = kMuonT + 8;                             // staging tile pitch (bf16): 144-B rows, 16-B aligned
constexpr int kNsThreads = 128 + 32;                           // consumer warpgroup + producer warp
constexpr size_t kNsSmem = 1024 + (size_t)kNsStages * 2 * kNsBox + (size_t)kMuonT * kNsStg * 2 + 2 * kNsStages * 8;

// out = bf16(alpha * (A B^T) + beta * C) per 64 x 64 tile.  TB = 0: B is K-major (64 rows of N, 64 K each), TB = 1:
// B is MN-major (64 rows of K, 64 N each) — the X operand of the UPDATE product.
template <int TB>
__global__ void __launch_bounds__(kNsThreads) k_muon_ns_gemm(const __grid_constant__ CUtensorMap tm,
                                                             const MuonTile* __restrict__ tiles, int n_tiles,
                                                             float alpha, float beta, __nv_bfloat16* __restrict__ ws) {
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __nv_bfloat16* stg = reinterpret_cast<__nv_bfloat16*>(smem + kNsStages * 2 * kNsBox);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg + kMuonT * kNsStg);
  uint64_t* empty_bar = full_bar + kNsStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tm);
    for (int i = 0; i < kNsStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 1); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 4) {                              // TMA producer: one lane
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const MuonTile tl = tiles[t];
        for (int k = 0; k < tl.nk; ++k) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], 2 * kNsBox);
          uint8_t* sA = smem + stage * 2 * kNsBox;
          tma_load_2d(sA, &tm, &full_bar[stage], 0, tl.a0 + k * tl.sa);
          tma_load_2d(sA + kNsBox, &tm, &full_bar[stage], 0, tl.b0 + k * tl.sb);
          if (++stage == kNsStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  const int tid = threadIdx.x;
  int stage = 0; uint32_t phase = 0;
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const MuonTile tl = tiles[t];
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int k = 0; k < tl.nk; ++k) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem + stage * 2 * kNsBox), b_addr = a_addr + kNsBox;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kMuonT / 16; ++kk) {
        const uint64_t adesc = make_smem_desc(a_addr, 16, 1024) + (uint64_t)(2 * kk);      // +32 B along K
        const uint32_t on = (k > 0 || kk > 0) ? 1u : 0u;
        if constexpr (TB == 0) {
          wgmma_m64n64<0, 0>(acc, adesc, make_smem_desc(b_addr, 16, 1024) + (uint64_t)(2 * kk), on);
        } else {
          // 16 K rows = two 8-row swizzle atoms = 2048 B; one 64-element N block
          wgmma_m64n64<0, 1>(acc, adesc, make_smem_desc(b_addr + 2048u * kk, kNsBox, 1024), on);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kNsStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);

    // fragments -> bf16(alpha * acc + beta * C) -> staging tile [64][kNsStg]
    const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h, c = 8 * j + 2 * (lane & 3);
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (tl.c0 >= 0) {
          const float2 cv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ws + (size_t)(tl.c0 + r) * kMuonT + c));
          v0 = fmaf(alpha, v0, __fmul_rn(beta, cv.x));
          v1 = fmaf(alpha, v1, __fmul_rn(beta, cv.y));
        } else {
          v0 = __fmul_rn(alpha, v0); v1 = __fmul_rn(alpha, v1);
        }
        *reinterpret_cast<__nv_bfloat162*>(stg + r * kNsStg + c) = __floats2bfloat162_rn(v0, v1);
      }
    bar_sync(1, 128);
    const bool diag = tl.m0 == tl.o0;
    for (int q = tid; q < kMuonT * 8; q += 128) {
      const int r = q >> 3, c8 = (q & 7) * 8;
      uint4 v;
      if (!diag) {
        v = *reinterpret_cast<const uint4*>(stg + r * kNsStg + c8);
      } else {                                  // out[r][c] = tile[min(r, c)][max(r, c)]: exactly symmetric
        unsigned short e[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int c = c8 + k;
          e[k] = __bfloat16_as_ushort(stg[min(r, c) * kNsStg + max(r, c)]);
        }
        v = make_uint4(e[0] | ((unsigned)e[1] << 16), e[2] | ((unsigned)e[3] << 16), e[4] | ((unsigned)e[5] << 16),
                       e[6] | ((unsigned)e[7] << 16));
      }
      *reinterpret_cast<uint4*>(ws + (size_t)(tl.o0 + r) * kMuonT + c8) = v;
      if (tl.m0 >= 0 && !diag) {                // the mirror tile: row r of it is column r of this one
        unsigned short e[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) e[k] = __bfloat16_as_ushort(stg[(c8 + k) * kNsStg + r]);
        *reinterpret_cast<uint4*>(ws + (size_t)(tl.m0 + r) * kMuonT + c8) =
            make_uint4(e[0] | ((unsigned)e[1] << 16), e[2] | ((unsigned)e[3] << 16), e[4] | ((unsigned)e[5] << 16),
                       e[6] | ((unsigned)e[7] << 16));
      }
    }
    bar_sync(1, 128);                           // the staging tile is free for the next tile
  }
}

template <int TB>
static int ns_gemm_launch(const CUtensorMap& tm, const MuonTile* tiles, int n_tiles, float alpha, float beta,
                          __nv_bfloat16* ws, cudaStream_t st) {
  static int per_sm[2] = {0, 0};
  if (!per_sm[TB]) {
    TP_CUDA_CHECK(cudaFuncSetAttribute(k_muon_ns_gemm<TB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kNsSmem));
    int nb = 0;
    TP_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_muon_ns_gemm<TB>, kNsThreads, kNsSmem));
    per_sm[TB] = nb > 0 ? nb : 1;
  }
  const long long gmax = (long long)sm_count() * per_sm[TB];
  const unsigned grid = (unsigned)(n_tiles < gmax ? n_tiles : gmax);
  launch(k_muon_ns_gemm<TB>, grid, kNsThreads, kNsSmem, st, tm, tiles, n_tiles, alpha, beta, ws);
  return TP_OK;
}

}  // namespace tp

using namespace tp;

extern "C" {

// table_ws: the layer table, then one uint32 completion count per layer
static size_t count_offset(int n_layers) { return align_up((size_t)n_layers * sizeof(tp_muon_layer), 256); }

size_t tp_muon_workspace_bytes(int n_layers) {
  return n_layers > 0 ? count_offset(n_layers) + (size_t)n_layers * sizeof(unsigned int) + 256 : 0;
}

int tp_muon_prepare(const tp_muon_layer* layers, int n_layers, int64_t n_tiles, int table_cached, void* xws,
                    void* partial, void* norms, double momentum, int nesterov, double eps, void* table_ws,
                    size_t table_bytes, void* stream) {
  if (n_layers <= 0 || n_tiles <= 0 || n_tiles > 0x7fffffffll || !xws || !partial || !norms || !table_ws) return TP_ERR_INVALID;
  if (table_bytes < tp_muon_workspace_bytes(n_layers)) return TP_ERR_WORKSPACE;
  unsigned int* done = (unsigned int*)((char*)table_ws + count_offset(n_layers));
  cudaStream_t st = (cudaStream_t)stream;
  if (!table_cached) {
    if (!layers) return TP_ERR_INVALID;
    long long t = 0;
    for (int i = 0; i < n_layers; ++i) {
      const tp_muon_layer& l = layers[i];
      if (!l.w || !l.g || !l.buf || l.a <= 0 || l.b <= 0 || l.mp % kMuonT || l.np % kMuonT) return TP_ERR_INVALID;
      const int m = l.trans ? l.b : l.a, n = l.trans ? l.a : l.b;
      if (m > n || l.mp < m || l.np < n || l.tile0 != t) return TP_ERR_INVALID;
      t += (long long)(l.mp / kMuonT) * (l.np / kMuonT);
    }
    if (t != n_tiles) return TP_ERR_INVALID;
    // pageable source: copied before the call returns (not capturable: cache the table first)
    TP_CUDA_CHECK(cudaMemcpyAsync(table_ws, layers, (size_t)n_layers * sizeof(tp_muon_layer), cudaMemcpyHostToDevice, st));
    TP_CUDA_CHECK(cudaMemsetAsync(done, 0, (size_t)n_layers * sizeof(unsigned int), st));
  }
  // the scalars as Python forms them: 1 - momentum in double, then fp32
  const float w1 = (float)(1.0 - momentum), w2 = (float)momentum;
  launch(k_muon_prepare, (unsigned)n_tiles, 256, 0, st, (const tp_muon_layer*)table_ws, n_layers, (__nv_bfloat16*)xws,
         (float*)partial, done, (float*)norms, (float)eps, w1, 1.f - w1, w2, 1.f - w2, nesterov ? 1 : 0);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_muon_normalize(int n_layers, int64_t n_tiles, void* xws, const void* norms, const void* table_ws, void* stream) {
  if (n_layers <= 0 || n_tiles <= 0 || n_tiles > 0x7fffffffll || !xws || !norms || !table_ws) return TP_ERR_INVALID;
  launch(k_muon_normalize, (unsigned)n_tiles, 256, 0, (cudaStream_t)stream, (const tp_muon_layer*)table_ws, n_layers,
         (__nv_bfloat16*)xws, (const float*)norms);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_muon_ns_gemm(int mode, void* xws, int64_t ws_rows, const void* tiles, int n_tiles, float alpha, float beta,
                    void* stream) {
  if (!xws || !tiles || n_tiles <= 0 || ws_rows <= 0 || ws_rows > 0x7fffffffll || mode < 0 || mode > 2) return TP_ERR_INVALID;
  if (mode == 0 && beta != 0.f) return TP_ERR_INVALID;
  if (bind_device_of(xws)) return TP_ERR_CUDA;
  CUtensorMap tm;
  int rc = make_tiled_map_bf16(&tm, xws, kMuonT, (uint64_t)ws_rows, kMuonT, kMuonT);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = mode == 2 ? ns_gemm_launch<1>(tm, (const MuonTile*)tiles, n_tiles, alpha, beta, (__nv_bfloat16*)xws, st)
                 : ns_gemm_launch<0>(tm, (const MuonTile*)tiles, n_tiles, alpha, beta, (__nv_bfloat16*)xws, st);
  if (rc) return rc;
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_muon_apply(int n_layers, int64_t n_tiles, const void* xws, int which, const void* lr_wd, const void* table_ws,
                  void* stream) {
  if (n_layers <= 0 || n_tiles <= 0 || n_tiles > 0x7fffffffll || !xws || !lr_wd || !table_ws || (which != 0 && which != 1))
    return TP_ERR_INVALID;
  launch(k_muon_apply, (unsigned)n_tiles, 256, 0, (cudaStream_t)stream, (const tp_muon_layer*)table_ws, n_layers,
         (const __nv_bfloat16*)xws, which, (const double*)lr_wd);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // extern "C"
