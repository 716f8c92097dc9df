// Fused BatchNorm (+ residual add) (+ ReLU) for NHWC bf16 activations, training and eval, sm_90a.
//
// SURVEY.md §8(f) row 1: the unmasked torchvision BatchNorm2d / ReLU / `out += identity` ops that sit
// between every pair of masked convolutions (created at utils/custom_models.py:184 of the reference,
// executed inside base_harness.py:124,127), in place of ATen's channels_last batch_norm_* kernels:
//
//   forward  : k_bn_stats (1 read)  -> k_bn_finalize_stats (tiny, fixed order => deterministic)
//              -> k_bn_apply: z = relu(y*scale + shift (+ residual))            (1-2 reads, 1 write)
//   backward : k_bn_bwd_reduce: g = dz*(z>0); sum g, sum g*xhat                 (2-3 reads)
//              -> k_bn_finalize_bwd -> k_bn_bwd_apply: dy = w*invstd*(g - mean(g) - xhat*mean(g*xhat))
//                 (+ dres = g)                                                  (2-3 reads, 1-2 writes)
//              With a residual the reduce pass already writes g (= dres), and the apply pass reads g and y
//              only: 3r+1w + 2r+1w instead of 3r + 3r+2w — one pass less over the widest activations.
//
// Layout: activations are [M pixels][C channels] bf16, C % 8 == 0; a thread owns one 16-byte vector
// (8 channels) and walks over pixels, so per-channel constants live in registers.
// Statistics are accumulated as shifted sums (shift = first pixel of the channel) in fp32 to avoid
// cancellation in E[x^2] - E[x]^2; running_var uses the unbiased estimate like torch.
#include "tp_common.cuh"

namespace tp {

constexpr int kBnThreads = 256;

struct BnGeom { int tx, ty, ctiles; int grid_x; };

static BnGeom bn_geom(long long M, int C) {
  BnGeom g;
  const int cv = C / 8;
  int tx = 1;
  while (tx < cv && tx < kBnThreads) tx <<= 1;
  g.tx = tx; g.ty = kBnThreads / tx;
  g.ctiles = (cv + tx - 1) / tx;
  long long rows = (M + g.ty - 1) / g.ty;
  long long want = (long long)sm_count() * 4 / g.ctiles;
  if (want < 1) want = 1;
  long long gx = (rows + 3) / 4;            // >= 4 pixel rows per thread
  if (gx > want) gx = want;
  if (gx < 1) gx = 1;
  g.grid_x = (int)gx;
  return g;
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}
__device__ __forceinline__ uint4 ldg16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- forward statistics --------------------------------------------------------------------------
// partial[blockIdx.x][0][c] = sum (x - shift_c), partial[blockIdx.x][1][c] = sum (x - shift_c)^2
__global__ void __launch_bounds__(kBnThreads) k_bn_stats(const __nv_bfloat16* __restrict__ y, long long M, int C,
                                                         float* __restrict__ partial) {
  pdl_enter();
  __shared__ float s_acc[kBnThreads][17];
  const int tx = threadIdx.x, ty = threadIdx.y, TX = blockDim.x, TY = blockDim.y;
  const int cvec = blockIdx.y * TX + tx;              // channel-vector index
  const bool act = cvec * 8 < C;
  float a1[8], a2[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { a1[i] = 0.f; a2[i] = 0.f; sh[i] = 0.f; }
  if (act) {
    unpack8(*reinterpret_cast<const uint4*>(y + (size_t)cvec * 8), sh);      // pixel 0 as the shift
    const long long stride = (long long)gridDim.x * TY;
    long long p = (long long)blockIdx.x * TY + ty;
    for (; p + 3 * stride < M; p += 4 * stride) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ldg16(y + (size_t)(p + u * stride) * C + (size_t)cvec * 8);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float f[8]; unpack8(v[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) { float d = f[i] - sh[i]; a1[i] += d; a2[i] = fmaf(d, d, a2[i]); }
      }
    }
    for (; p < M; p += stride) {
      float f[8]; unpack8(ldg16(y + (size_t)p * C + (size_t)cvec * 8), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) { float d = f[i] - sh[i]; a1[i] += d; a2[i] = fmaf(d, d, a2[i]); }
    }
  }
  const int tid = ty * TX + tx;
#pragma unroll
  for (int i = 0; i < 8; ++i) { s_acc[tid][i] = a1[i]; s_acc[tid][8 + i] = a2[i]; }
  __syncthreads();
  if (ty == 0 && act) {
    float r[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) r[i] = 0.f;
    for (int j = 0; j < TY; ++j)
#pragma unroll
      for (int i = 0; i < 16; ++i) r[i] += s_acc[j * TX + tx][i];
    float* dst = partial + (size_t)blockIdx.x * 2 * C;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[cvec * 8 + i] = r[i]; dst[C + cvec * 8 + i] = r[8 + i]; }
  }
}

// Fold the per-CTA partials of one channel in a fixed order: 8 part-lanes each sum a strided subset
// (coalesced across the 32 channel-lanes), then the 8 lane sums are added in lane order.
constexpr int kFinC = 32, kFinP = 32;
__device__ __forceinline__ void fold_partials(const float* __restrict__ partial, int nparts, int C, int c,
                                              float& s1, float& s2, float (*sm)[kFinP][kFinC]) {
  const int tx = threadIdx.x, ty = threadIdx.y;
  float a1 = 0.f, a2 = 0.f;
  if (c < C) {
    int j = ty;
    for (; j + 3 * kFinP < nparts; j += 4 * kFinP) {
      float v1[4], v2[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { v1[u] = partial[(size_t)(j + u * kFinP) * 2 * C + c]; v2[u] = partial[(size_t)(j + u * kFinP) * 2 * C + C + c]; }
#pragma unroll
      for (int u = 0; u < 4; ++u) { a1 += v1[u]; a2 += v2[u]; }
    }
    for (; j < nparts; j += kFinP) { a1 += partial[(size_t)j * 2 * C + c]; a2 += partial[(size_t)j * 2 * C + C + c]; }
  }
  sm[0][ty][tx] = a1; sm[1][ty][tx] = a2;
  __syncthreads();
  s1 = 0.f; s2 = 0.f;
#pragma unroll
  for (int k = 0; k < kFinP; ++k) { s1 += sm[0][k][tx]; s2 += sm[1][k][tx]; }
}

// one thread per channel: fold the partials in fixed order; emit mean / invstd / scale / shift and
// update the running statistics (torch semantics: momentum, unbiased running_var).
__global__ void __launch_bounds__(kFinC * kFinP) k_bn_finalize_stats(const float* __restrict__ partial, int nparts, const __nv_bfloat16* __restrict__ y,
                                    long long M, int C, const float* __restrict__ weight, const float* __restrict__ bias,
                                    float* running_mean, float* running_var, long long* nbt, float momentum, float eps,
                                    float* __restrict__ save_mean, float* __restrict__ save_invstd,
                                    float* __restrict__ scale, float* __restrict__ shift) {
  pdl_enter();
  __shared__ float sm[2][kFinP][kFinC];
  const int c = blockIdx.x * kFinC + threadIdx.x;
  float s1, s2;
  fold_partials(partial, nparts, C, c, s1, s2, sm);
  if (threadIdx.y != 0) return;
  if (c == 0 && nbt) *nbt += 1;
  if (c >= C) return;
  float mean, var;
  if (y) {
    const float sh = __bfloat162float(y[c]);
    const float inv_m = 1.f / (float)M;
    const float dm = s1 * inv_m;
    mean = sh + dm;
    var = fmaf(-dm, dm, s2 * inv_m);
  } else {
    // un-shifted sums from the conv epilogue: E[x^2] - E[x]^2 combined in double (one thread per channel)
    const double dmean = (double)s1 / (double)M;
    mean = (float)dmean;
    var = (float)((double)s2 / (double)M - dmean * dmean);
  }
  var = fmaxf(var, 0.f);
  const float invstd = rsqrtf(var + eps);
  save_mean[c] = mean; save_invstd[c] = invstd;
  const float w = weight ? weight[c] : 1.f, b = bias ? bias[c] : 0.f;
  scale[c] = w * invstd; shift[c] = fmaf(-mean, w * invstd, b);
  if (running_mean) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
    const float unbiased = M > 1 ? var * ((float)M / (float)(M - 1)) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
  }
}

// First fold level for statistics produced by the conv epilogue: ext[rows][2][C] (one row per 32 output pixels) ->
// partial[g][2][C], 1024 rows per CTA in a fixed order; k_bn_finalize_stats then folds the (few) g rows.
__global__ void __launch_bounds__(kFinC * kFinP) k_bn_fold_ext(const float* __restrict__ ext, long long rows, int C,
                                                               float* __restrict__ partial) {
  pdl_enter();
  __shared__ float sm[2][kFinP][kFinC];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * kFinC + tx;
  const long long r0 = (long long)blockIdx.y * 1024, r1 = min(rows, r0 + 1024);
  float a1 = 0.f, a2 = 0.f;
  if (c < C) {
    long long j = r0 + ty;
    for (; j + 3 * kFinP < r1; j += 4 * kFinP) {
      float v1[4], v2[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { v1[u] = ext[(size_t)(j + u * kFinP) * 2 * C + c]; v2[u] = ext[(size_t)(j + u * kFinP) * 2 * C + C + c]; }
#pragma unroll
      for (int u = 0; u < 4; ++u) { a1 += v1[u]; a2 += v2[u]; }
    }
    for (; j < r1; j += kFinP) { a1 += ext[(size_t)j * 2 * C + c]; a2 += ext[(size_t)j * 2 * C + C + c]; }
  }
  sm[0][ty][tx] = a1; sm[1][ty][tx] = a2;
  __syncthreads();
  if (ty == 0 && c < C) {
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < kFinP; ++k) { s1 += sm[0][k][tx]; s2 += sm[1][k][tx]; }
    partial[(size_t)blockIdx.y * 2 * C + c] = s1;
    partial[(size_t)blockIdx.y * 2 * C + C + c] = s2;
  }
}

__global__ void k_bn_eval_coeffs(int C, const float* __restrict__ weight, const float* __restrict__ bias,
                                 const float* __restrict__ running_mean, const float* __restrict__ running_var, float eps,
                                 float* __restrict__ scale, float* __restrict__ shift) {
  pdl_enter();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float invstd = rsqrtf(running_var[c] + eps);
  const float w = weight ? weight[c] : 1.f, b = bias ? bias[c] : 0.f;
  scale[c] = w * invstd; shift[c] = fmaf(-running_mean[c], w * invstd, b);
}

// z = [relu]( y*scale + shift [+ residual] )
template <bool RELU, bool RES>
__global__ void __launch_bounds__(kBnThreads) k_bn_apply(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ res,
                                                         __nv_bfloat16* __restrict__ z, long long M, int C,
                                                         const float* __restrict__ scale, const float* __restrict__ shift) {
  pdl_enter();
  const int tx = threadIdx.x, ty = threadIdx.y, TX = blockDim.x, TY = blockDim.y;
  const int cvec = blockIdx.y * TX + tx;
  if (cvec * 8 >= C) return;
  float sc[8], sf[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sc[i] = scale[cvec * 8 + i]; sf[i] = shift[cvec * 8 + i]; }
  const long long stride = (long long)gridDim.x * TY;
  long long p = (long long)blockIdx.x * TY + ty;
  for (; p + 3 * stride < M; p += 4 * stride) {
    uint4 v[4], r[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const size_t off = (size_t)(p + u * stride) * C + (size_t)cvec * 8;
      v[u] = ldg16(y + off);
      if (RES) r[u] = ldg16(res + off);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float f[8], g[8]; unpack8(v[u], f);
      if (RES) unpack8(r[u], g);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float o = fmaf(f[i], sc[i], sf[i]);
        if (RES) o += g[i];
        if (RELU) o = fmaxf(o, 0.f);
        f[i] = o;
      }
      stg16(z + (size_t)(p + u * stride) * C + (size_t)cvec * 8, pack8(f));
    }
  }
  for (; p < M; p += stride) {
    const size_t off = (size_t)p * C + (size_t)cvec * 8;
    float f[8], g[8]; unpack8(ldg16(y + off), f);
    if (RES) unpack8(ldg16(res + off), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float o = fmaf(f[i], sc[i], sf[i]);
      if (RES) o += g[i];
      if (RELU) o = fmaxf(o, 0.f);
      f[i] = o;
    }
    stg16(z + off, pack8(f));
  }
}

// ---- backward ----------------------------------------------------------------------------------------
// partial[b][0][c] = sum g, partial[b][1][c] = sum g * xhat, with g = dz * (z > 0) when RELU
// RELU: 0 = no activation, 1 = gate from the saved output (z > 0), 2 = gate recomputed from y (same fp32
// expression as the forward apply: no need to read z at all — one activation pass less)
template <int RELU, bool WRITE_G>
__global__ void __launch_bounds__(kBnThreads) k_bn_bwd_reduce(const __nv_bfloat16* __restrict__ dz, const __nv_bfloat16* __restrict__ z,
                                                              const __nv_bfloat16* __restrict__ y, long long M, int C,
                                                              const float* __restrict__ mean, const float* __restrict__ invstd,
                                                              const float* __restrict__ weight, const float* __restrict__ bias,
                                                              float* __restrict__ partial, __nv_bfloat16* __restrict__ gout) {
  pdl_enter();
  __shared__ float s_acc[kBnThreads][17];
  const int tx = threadIdx.x, ty = threadIdx.y, TX = blockDim.x, TY = blockDim.y;
  const int cvec = blockIdx.y * TX + tx;
  const bool act = cvec * 8 < C;
  float a1[8], a2[8], mu[8], is[8], sc[8], sf[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { a1[i] = 0.f; a2[i] = 0.f; mu[i] = 0.f; is[i] = 0.f; sc[i] = 0.f; sf[i] = 0.f; }
  if (act) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mu[i] = mean[cvec * 8 + i]; is[i] = invstd[cvec * 8 + i];
      if (RELU == 2) {
        const float w = weight ? weight[cvec * 8 + i] : 1.f, b = bias ? bias[cvec * 8 + i] : 0.f;
        sc[i] = w * is[i]; sf[i] = fmaf(-mu[i], w * is[i], b);      // identical to k_bn_finalize_stats
      }
    }
    const long long stride = (long long)gridDim.x * TY;
    long long p = (long long)blockIdx.x * TY + ty;
    // 2 pixel rows in flight per thread (4-6 independent 16-byte loads); more rows cost registers, and with them occupancy
    constexpr int UR = 2;
    for (; p + (UR - 1) * stride < M; p += UR * stride) {
      uint4 vd[UR], vz[UR], vy[UR];
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        const size_t off = (size_t)(p + u * stride) * C + (size_t)cvec * 8;
        vd[u] = ldg16(dz + off); vy[u] = ldg16(y + off);
        if (RELU == 1) vz[u] = ldg16(z + off);
      }
#pragma unroll
      for (int u = 0; u < UR; ++u) {
        float d[8], yy[8], zz[8]; unpack8(vd[u], d); unpack8(vy[u], yy);
        if (RELU == 1) unpack8(vz[u], zz);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const bool open = RELU == 0 ? true : (RELU == 1 ? (zz[i] > 0.f) : (fmaf(yy[i], sc[i], sf[i]) > 0.f));
          const float g = open ? d[i] : 0.f;
          if (WRITE_G) d[i] = g;
          a1[i] += g; a2[i] = fmaf(g, (yy[i] - mu[i]) * is[i], a2[i]);
        }
        if (WRITE_G) stg16(gout + (size_t)(p + u * stride) * C + (size_t)cvec * 8, pack8(d));
      }
    }
    for (; p < M; p += stride) {
      const size_t off = (size_t)p * C + (size_t)cvec * 8;
      float d[8], yy[8], zz[8]; unpack8(ldg16(dz + off), d); unpack8(ldg16(y + off), yy);
      if (RELU == 1) unpack8(ldg16(z + off), zz);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const bool open = RELU == 0 ? true : (RELU == 1 ? (zz[i] > 0.f) : (fmaf(yy[i], sc[i], sf[i]) > 0.f));
        const float g = open ? d[i] : 0.f;
        if (WRITE_G) d[i] = g;
        a1[i] += g; a2[i] = fmaf(g, (yy[i] - mu[i]) * is[i], a2[i]);
      }
      if (WRITE_G) stg16(gout + off, pack8(d));
    }
  }
  const int tid = ty * TX + tx;
#pragma unroll
  for (int i = 0; i < 8; ++i) { s_acc[tid][i] = a1[i]; s_acc[tid][8 + i] = a2[i]; }
  __syncthreads();
  if (ty == 0 && act) {
    float r[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) r[i] = 0.f;
    for (int j = 0; j < TY; ++j)
#pragma unroll
      for (int i = 0; i < 16; ++i) r[i] += s_acc[j * TX + tx][i];
    float* dst = partial + (size_t)blockIdx.x * 2 * C;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[cvec * 8 + i] = r[i]; dst[C + cvec * 8 + i] = r[8 + i]; }
  }
}

// dweight = sum g*xhat, dbias = sum g; coefficients for the apply pass:
//   dy = k0 * g + k1 * y + k2   with  k0 = w*invstd,  k1 = -k0*invstd*mean(g*xhat),
//                                     k2 = -k0*mean(g) - k1*mu
__global__ void __launch_bounds__(kFinC * kFinP) k_bn_finalize_bwd(const float* __restrict__ partial, int nparts, long long M, int C,
                                  const float* __restrict__ weight, const float* __restrict__ bias,
                                  const float* __restrict__ mean, const float* __restrict__ invstd,
                                  float* __restrict__ dweight, float* __restrict__ dbias, float* __restrict__ coef) {
  pdl_enter();
  __shared__ float sm[2][kFinP][kFinC];
  const int c = blockIdx.x * kFinC + threadIdx.x;
  float s1, s2;
  fold_partials(partial, nparts, C, c, s1, s2, sm);
  if (threadIdx.y != 0 || c >= C) return;
  if (dweight) dweight[c] = s2;
  if (dbias) dbias[c] = s1;
  const float inv_m = 1.f / (float)M;
  const float w = weight ? weight[c] : 1.f;
  const float k0 = w * invstd[c];
  const float k1 = -k0 * invstd[c] * (s2 * inv_m);
  const float k2 = -k0 * (s1 * inv_m) - k1 * mean[c];
  coef[c] = k0; coef[C + c] = k1; coef[2 * C + c] = k2;
  coef[3 * C + c] = k0;                                        // forward scale  (w * invstd)
  coef[4 * C + c] = fmaf(-mean[c], k0, bias ? bias[c] : 0.f);  // forward shift
}

template <int RELU, bool RES>
__global__ void __launch_bounds__(kBnThreads) k_bn_bwd_apply(const __nv_bfloat16* __restrict__ dz, const __nv_bfloat16* __restrict__ z,
                                                             const __nv_bfloat16* __restrict__ y, long long M, int C,
                                                             const float* __restrict__ coef, __nv_bfloat16* __restrict__ dy,
                                                             __nv_bfloat16* __restrict__ dres) {
  pdl_enter();
  const int tx = threadIdx.x, ty = threadIdx.y, TX = blockDim.x, TY = blockDim.y;
  const int cvec = blockIdx.y * TX + tx;
  if (cvec * 8 >= C) return;
  float k0[8], k1[8], k2[8], sf[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    k0[i] = coef[cvec * 8 + i]; k1[i] = coef[C + cvec * 8 + i]; k2[i] = coef[2 * C + cvec * 8 + i];
    sf[i] = RELU == 2 ? coef[4 * C + cvec * 8 + i] : 0.f;         // forward scale == k0
  }
  const long long stride = (long long)gridDim.x * TY;
  long long p = (long long)blockIdx.x * TY + ty;
  constexpr int UR = 2;
  for (; p + (UR - 1) * stride < M; p += UR * stride) {
    uint4 vd[UR], vz[UR], vy[UR];
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const size_t off = (size_t)(p + u * stride) * C + (size_t)cvec * 8;
      vd[u] = ldg16(dz + off); vy[u] = ldg16(y + off);
      if (RELU == 1) vz[u] = ldg16(z + off);
    }
#pragma unroll
    for (int u = 0; u < UR; ++u) {
      const size_t off = (size_t)(p + u * stride) * C + (size_t)cvec * 8;
      float d[8], yy[8], zz[8], o[8]; unpack8(vd[u], d); unpack8(vy[u], yy);
      if (RELU == 1) unpack8(vz[u], zz);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const bool open = RELU == 0 ? true : (RELU == 1 ? (zz[i] > 0.f) : (fmaf(yy[i], k0[i], sf[i]) > 0.f));
        const float g = open ? d[i] : 0.f;
        d[i] = g;
        o[i] = fmaf(k0[i], g, fmaf(k1[i], yy[i], k2[i]));
      }
      stg16(dy + off, pack8(o));
      if (RES) stg16(dres + off, pack8(d));
    }
  }
  for (; p < M; p += stride) {
    const size_t off = (size_t)p * C + (size_t)cvec * 8;
    float d[8], yy[8], zz[8], o[8]; unpack8(ldg16(dz + off), d); unpack8(ldg16(y + off), yy);
    if (RELU == 1) unpack8(ldg16(z + off), zz);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const bool open = RELU == 0 ? true : (RELU == 1 ? (zz[i] > 0.f) : (fmaf(yy[i], k0[i], sf[i]) > 0.f));
      const float g = open ? d[i] : 0.f;
      d[i] = g;
      o[i] = fmaf(k0[i], g, fmaf(k1[i], yy[i], k2[i]));
    }
    stg16(dy + off, pack8(o));
    if (RES) stg16(dres + off, pack8(d));
  }
}

}  // namespace tp

using namespace tp;

extern "C" {

size_t tp_bn_workspace_bytes(int64_t M, int C) {
  if (M <= 0 || C <= 0) return 0;
  BnGeom g = bn_geom(M, C);
  return (size_t)g.grid_x * 2 * C * sizeof(float) + (size_t)5 * C * sizeof(float) + 1024;
}

int tp_bn_forward(const void* y, const void* residual, void* z, int64_t M, int C,
                  const void* weight, const void* bias, void* running_mean, void* running_var,
                  void* num_batches_tracked, float momentum, float eps, int training, int relu,
                  void* save_mean, void* save_invstd, void* ws, size_t ws_bytes, void* stream) {
  return tp_bn_forward_ext(y, residual, z, M, C, weight, bias, running_mean, running_var, num_batches_tracked, momentum,
                           eps, training, relu, save_mean, save_invstd, nullptr, 0, ws, ws_bytes, stream);
}

int tp_bn_forward_ext(const void* y, const void* residual, void* z, int64_t M, int C,
                      const void* weight, const void* bias, void* running_mean, void* running_var,
                      void* num_batches_tracked, float momentum, float eps, int training, int relu,
                      void* save_mean, void* save_invstd, const void* ext_stats, int64_t ext_rows,
                      void* ws, size_t ws_bytes, void* stream) {
  if (!y || !z || M <= 0 || C <= 0 || C % 8 != 0 || !ws) return TP_ERR_INVALID;
  if (ext_stats && (!training || ext_rows <= 0)) return TP_ERR_INVALID;
  if (training && (!save_mean || !save_invstd)) return TP_ERR_INVALID;
  if (!training && (!running_mean || !running_var)) return TP_ERR_INVALID;
  if (ws_bytes < tp_bn_workspace_bytes(M, C)) return TP_ERR_WORKSPACE;
  int rc = bind_device_of(y); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  BnGeom g = bn_geom(M, C);
  float* partial = (float*)ws;
  float* scale = partial + (size_t)g.grid_x * 2 * C;
  float* shift = scale + C;
  dim3 block(g.tx, g.ty), grid(g.grid_x, g.ctiles);
  if (training && ext_stats) {
    // statistics came out of the producing convolution's epilogue: two small folds, no pass over the activation
    const long long groups = (ext_rows + 1023) / 1024;
    if (groups > g.grid_x) return TP_ERR_WORKSPACE;
    const float* fold_src = (const float*)ext_stats;       // <= 1024 rows: the finalize kernel folds them directly
    long long fold_rows = ext_rows;
    if (groups > 1) {
      launch(k_bn_fold_ext, dim3((C + kFinC - 1) / kFinC, (unsigned)groups), dim3(kFinC, kFinP), 0, st, (const float*)ext_stats, ext_rows, C, partial);
      fold_src = partial; fold_rows = groups;
    }
    launch(k_bn_finalize_stats, (C + kFinC - 1) / kFinC, dim3(kFinC, kFinP), 0, st, fold_src, (int)fold_rows, nullptr, M, C,
                                                          (const float*)weight, (const float*)bias, (float*)running_mean,
                                                          (float*)running_var, (long long*)num_batches_tracked, momentum, eps,
                                                          (float*)save_mean, (float*)save_invstd, scale, shift);
  } else if (training) {
    launch(k_bn_stats, grid, block, 0, st, (const __nv_bfloat16*)y, M, C, partial);
    launch(k_bn_finalize_stats, (C + kFinC - 1) / kFinC, dim3(kFinC, kFinP), 0, st, partial, g.grid_x, (const __nv_bfloat16*)y, M, C,
                                                          (const float*)weight, (const float*)bias, (float*)running_mean,
                                                          (float*)running_var, (long long*)num_batches_tracked, momentum, eps,
                                                          (float*)save_mean, (float*)save_invstd, scale, shift);
  } else {
    launch(k_bn_eval_coeffs, (C + 255) / 256, 256, 0, st, C, (const float*)weight, (const float*)bias, (const float*)running_mean,
                                                       (const float*)running_var, eps, scale, shift);
  }
  const __nv_bfloat16* yy = (const __nv_bfloat16*)y; const __nv_bfloat16* rr = (const __nv_bfloat16*)residual;
  __nv_bfloat16* zz = (__nv_bfloat16*)z;
  if (relu && rr) launch(k_bn_apply<true, true>, grid, block, 0, st, yy, rr, zz, M, C, scale, shift);
  else if (relu) launch(k_bn_apply<true, false>, grid, block, 0, st, yy, rr, zz, M, C, scale, shift);
  else if (rr) launch(k_bn_apply<false, true>, grid, block, 0, st, yy, rr, zz, M, C, scale, shift);
  else launch(k_bn_apply<false, false>, grid, block, 0, st, yy, rr, zz, M, C, scale, shift);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_bn_backward(const void* dz, const void* z, const void* y, int64_t M, int C, const void* weight, const void* bias,
                   const void* save_mean, const void* save_invstd, int relu, void* dy, void* dres,
                   void* dweight, void* dbias, void* ws, size_t ws_bytes, void* stream) {
  if (!dz || !y || !dy || !save_mean || !save_invstd || M <= 0 || C <= 0 || C % 8 != 0 || !ws) return TP_ERR_INVALID;
  if (relu < 0 || relu > 2 || (relu == 1 && !z)) return TP_ERR_INVALID;
  if (ws_bytes < tp_bn_workspace_bytes(M, C)) return TP_ERR_WORKSPACE;
  int rc = bind_device_of(y); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  BnGeom g = bn_geom(M, C);
  float* partial = (float*)ws;
  float* coef = partial + (size_t)g.grid_x * 2 * C;
  dim3 block(g.tx, g.ty), grid(g.grid_x, g.ctiles);
  const __nv_bfloat16 *d = (const __nv_bfloat16*)dz, *zz = (const __nv_bfloat16*)z, *yy = (const __nv_bfloat16*)y;
  const float *mu = (const float*)save_mean, *is = (const float*)save_invstd, *wp = (const float*)weight, *bp = (const float*)bias;
  __nv_bfloat16* o = (__nv_bfloat16*)dy; __nv_bfloat16* r = (__nv_bfloat16*)dres;
  // with an activation AND a residual the gated gradient g is the residual's gradient: write it in the reduce pass
  const bool g_first = relu != 0 && r != nullptr;
  if (relu == 1 && g_first) launch(k_bn_bwd_reduce<1, true>, grid, block, 0, st, d, zz, yy, M, C, mu, is, wp, bp, partial, r);
  else if (relu == 2 && g_first) launch(k_bn_bwd_reduce<2, true>, grid, block, 0, st, d, zz, yy, M, C, mu, is, wp, bp, partial, r);
  else if (relu == 1) launch(k_bn_bwd_reduce<1, false>, grid, block, 0, st, d, zz, yy, M, C, mu, is, wp, bp, partial, nullptr);
  else if (relu == 2) launch(k_bn_bwd_reduce<2, false>, grid, block, 0, st, d, zz, yy, M, C, mu, is, wp, bp, partial, nullptr);
  else launch(k_bn_bwd_reduce<0, false>, grid, block, 0, st, d, zz, yy, M, C, mu, is, wp, bp, partial, nullptr);
  launch(k_bn_finalize_bwd, (C + kFinC - 1) / kFinC, dim3(kFinC, kFinP), 0, st, partial, g.grid_x, M, C, wp, bp, mu, is,
                                                                          (float*)dweight, (float*)dbias, coef);
  if (g_first) launch(k_bn_bwd_apply<0, false>, grid, block, 0, st, r, zz, yy, M, C, coef, o, nullptr);     // g is final: no gate, no second write
  else if (relu == 1 && r) launch(k_bn_bwd_apply<1, true>, grid, block, 0, st, d, zz, yy, M, C, coef, o, r);
  else if (relu == 1) launch(k_bn_bwd_apply<1, false>, grid, block, 0, st, d, zz, yy, M, C, coef, o, r);
  else if (relu == 2 && r) launch(k_bn_bwd_apply<2, true>, grid, block, 0, st, d, zz, yy, M, C, coef, o, r);
  else if (relu == 2) launch(k_bn_bwd_apply<2, false>, grid, block, 0, st, d, zz, yy, M, C, coef, o, r);
  else if (r) launch(k_bn_bwd_apply<0, true>, grid, block, 0, st, d, zz, yy, M, C, coef, o, r);
  else launch(k_bn_bwd_apply<0, false>, grid, block, 0, st, d, zz, yy, M, C, coef, o, r);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

// BatchNorm(+ReLU) backward whose reduction was already done by the dgrad that produced its incoming gradient
// (tp_conv_dgrad_bnrelu): g = dz * [z > 0] is given together with per-32-row partial sums (sum g, sum g * xhat); what is
// left is the fold of the partials, the coefficients and the apply pass dy = k0 g + k1 y + k2.
int tp_bn_backward_ext(const void* g, const void* y, int64_t M, int C, const void* weight, const void* bias,
                       const void* save_mean, const void* save_invstd, const void* partial_rows, int64_t n_rows,
                       void* dy, void* dweight, void* dbias, void* ws, size_t ws_bytes, void* stream) {
  if (!g || !y || !dy || !save_mean || !save_invstd || !partial_rows || n_rows <= 0 || M <= 0 || C <= 0 || C % 8 != 0 || !ws) return TP_ERR_INVALID;
  if (ws_bytes < tp_bn_workspace_bytes(M, C)) return TP_ERR_WORKSPACE;
  int rc = bind_device_of(y); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  BnGeom gm = bn_geom(M, C);
  float* partial = (float*)ws;
  float* coef = partial + (size_t)gm.grid_x * 2 * C;
  const float* fold_src = (const float*)partial_rows;
  long long fold_rows = n_rows;
  const long long groups = (n_rows + 1023) / 1024;
  if (groups > 1) {
    if (groups > gm.grid_x) return TP_ERR_WORKSPACE;
    launch(k_bn_fold_ext, dim3((C + kFinC - 1) / kFinC, (unsigned)groups), dim3(kFinC, kFinP), 0, st, (const float*)partial_rows, n_rows, C, partial);
    fold_src = partial; fold_rows = groups;
  }
  launch(k_bn_finalize_bwd, (C + kFinC - 1) / kFinC, dim3(kFinC, kFinP), 0, st, fold_src, (int)fold_rows, M, C, (const float*)weight, (const float*)bias,
                                                                          (const float*)save_mean, (const float*)save_invstd,
                                                                          (float*)dweight, (float*)dbias, coef);
  dim3 block(gm.tx, gm.ty), grid(gm.grid_x, gm.ctiles);
  launch(k_bn_bwd_apply<0, false>, grid, block, 0, st, (const __nv_bfloat16*)g, nullptr, (const __nv_bfloat16*)y, M, C, coef, (__nv_bfloat16*)dy, nullptr);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // extern "C"
