// Weight staging (mask*w -> bf16 tensor-core layouts), activation layout conversion and
// the fused SGD step.  All HBM-bound streaming kernels.
#include "tp_common.cuh"
#include <vector>

namespace tp {

// One CTA per (cout, r*s-chunk): read OIHW fp32 (w, mask), write
//   wf[co][r][s][ci]                    (K-major B operand of fprop, K = (r,s,ci))
//   wd[ci][R-1-r][S-1-s][co]            (K-major B operand of dgrad, K = (r',s',co))
// OIHW -> O(RS)I is a small transpose per output channel: stage the [Cin][RS] slab of one
// output channel through shared memory so both the read and the wf write are coalesced.
// One CTA stages a tile of kCoT output channels x a slice of input channels: the [co][ci][tap] slab goes through shared
// memory so that the OIHW read, the wf write (channels contiguous per tap) and the wd write (kCoT output channels =
// one 16-byte store per (ci, tap)) are all coalesced.  (Staging one output channel per CTA makes every wd element a
// separate 2-byte sector write.)
constexpr int kCoT = 8;
constexpr int kSlabFloats = 8192;            // 32 KB

// K-block occupancy (BASELINE.json north_star: skip all-zero tiles): one bit per (64 rows of the staged operand) x (64 K
// columns), set when the block holds a non-zero masked weight.  kmf: rows = output channels, column = tap*cin_p + ci (wf);
// kmd: rows = input channels, column = rot_tap*cout_p + co (wd).  Bits are OR-ed into a buffer the host zeroed, so the
// result does not depend on CTA order.
//
// T = float: the fp32 operands of the TF32 GEMMs, same layouts, mask * w stored exactly (no occupancy masks are asked for).
template <typename T> __device__ __forceinline__ T to_operand(float v);
template <> __device__ __forceinline__ __nv_bfloat16 to_operand<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ float to_operand<float>(float v) { return v; }

template <typename T>
__device__ __forceinline__ void stage_slab(const float* __restrict__ w, const float* __restrict__ mask, int co0, int cout,
                                           int c0, int c1, int cin, int rs, T* __restrict__ wf, int cin_p, int wf_ld,
                                           T* __restrict__ wd, int cout_p, bool zero_pad, float* s_slab,
                                           uint32_t* __restrict__ kmf, int kmf_words, uint32_t* __restrict__ kmd, int kmd_words) {
  const int t = threadIdx.x;
  const int cw = c1 - c0;                    // channels in this slice
  const int per_co = cw * rs;
  const int nco = min(kCoT, cout - co0);
  for (int i = t; i < nco * per_co; i += blockDim.x) {
    const int cl = i / per_co, j = i - cl * per_co;
    const long long gi = ((long long)(co0 + cl) * cin + c0) * rs + j;
    const float mk = mask[gi], prod = mk * w[gi];
    s_slab[i] = prod;                        // utils/mask_layers.py:25 — fp32 product, then bf16 (autocast)
    // The fprop occupancy mask doubles as the MASK's occupancy for wgrad tile skipping (dW = mask * ... is zero under an
    // all-zero mask block): a kept weight that happens to be exactly zero must keep its block alive.  Never taken in practice.
    if (kmf && prod == 0.f && mk != 0.f) {
      const int c = j / rs, tap = j - c * rs, kb = (tap * cin_p + c0 + c) >> 6;
      atomicOr(&kmf[(size_t)(co0 >> 6) * kmf_words + (kb >> 5)], 1u << (kb & 31));
    }
  }
  __syncthreads();
  // wf: per output channel and tap, channels contiguous
  for (int i = t; i < nco * per_co; i += blockDim.x) {
    const int cl = i / per_co, j = i - cl * per_co;
    const int tap = j / cw, c = j - tap * cw;
    wf[(long long)(co0 + cl) * wf_ld + tap * cin_p + c0 + c] = to_operand<T>(s_slab[cl * per_co + c * rs + tap]);
  }
  if (wd) {
    // wd[ci][rs-1-tap][co0 .. co0+8): one 16-byte store per (ci, tap); channels past cout are the zero padding
    for (int j = t; j < per_co; j += blockDim.x) {
      const int c = j / rs, tap = j - c * rs;
      float f[kCoT];
#pragma unroll
      for (int cl = 0; cl < kCoT; ++cl) f[cl] = cl < nco ? s_slab[cl * per_co + j] : 0.f;
      T* dst = wd + ((long long)(c0 + c) * rs + (rs - 1 - tap)) * cout_p + co0;
      if (co0 + kCoT <= cout_p) {
        if constexpr (sizeof(T) == 4) {
          reinterpret_cast<float4*>(dst)[0] = make_float4(f[0], f[1], f[2], f[3]);
          reinterpret_cast<float4*>(dst)[1] = make_float4(f[4], f[5], f[6], f[7]);
        } else {
          uint4 v;
          __nv_bfloat162* hv = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
          for (int q = 0; q < 4; ++q) hv[q] = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
          *reinterpret_cast<uint4*>(dst) = v;
        }
      } else {
        for (int cl = 0; cl < kCoT && co0 + cl < cout_p; ++cl) dst[cl] = to_operand<T>(f[cl]);
      }
    }
  }
  if (kmf || (kmd && wd)) {
    const int warp = t >> 5, lane = t & 31, nwarps = blockDim.x >> 5;
    if (kmf) {
      for (int tap = 0; tap < rs; ++tap) {
        const int col0 = tap * cin_p + c0, col1 = tap * cin_p + c1;            // wf columns of this slice for this tap
        for (int kb = (col0 >> 6) + warp; kb <= ((col1 - 1) >> 6); kb += nwarps) {
          const int a = max(col0, kb << 6), b = min(col1, (kb + 1) << 6), wdt = b - a;
          bool nz = false;
          for (int e = lane; e < nco * wdt; e += 32) {
            const int cl = e / wdt, c = a + (e - cl * wdt) - tap * cin_p - c0;
            nz |= s_slab[cl * per_co + c * rs + tap] != 0.f;
          }
          if (__any_sync(0xffffffffu, nz) && lane == 0) atomicOr(&kmf[(size_t)(co0 >> 6) * kmf_words + (kb >> 5)], 1u << (kb & 31));
        }
      }
    }
    if (kmd && wd) {
      // rows = input channels (64 per group), column block of this CTA's 8 output channels under rotated tap rt
      const int g0 = c0 >> 6, g1 = (c1 - 1) >> 6;
      for (int item = warp; item < rs * (g1 - g0 + 1); item += nwarps) {
        const int tap = item / (g1 - g0 + 1), g = g0 + item % (g1 - g0 + 1);
        const int a = max(c0, g << 6), b = min(c1, (g + 1) << 6), wdt = b - a;
        bool nz = false;
        for (int e = lane; e < nco * wdt; e += 32) {
          const int cl = e / wdt, c = a + (e - cl * wdt) - c0;
          nz |= s_slab[cl * per_co + c * rs + tap] != 0.f;
        }
        const int kb = ((rs - 1 - tap) * cout_p + co0) >> 6;
        if (__any_sync(0xffffffffu, nz) && lane == 0) atomicOr(&kmd[(size_t)g * kmd_words + (kb >> 5)], 1u << (kb & 31));
      }
    }
  }
  // zero the channel padding of wf (cin..cin_p) — done by the first channel slice
  if (zero_pad && c0 == 0 && cin_p > cin) {
    const int padw = cin_p - cin;
    for (int i = t; i < nco * padw * rs; i += blockDim.x) {
      const int cl = i / (padw * rs), j = i - cl * (padw * rs);
      const int tap = j / padw, c = j - tap * padw;
      wf[(long long)(co0 + cl) * wf_ld + tap * cin_p + cin + c] = to_operand<T>(0.f);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) k_stage_weights(const float* __restrict__ w, const float* __restrict__ mask,
                                                       int cout, int cin, int rs,
                                                       T* __restrict__ wf, int cin_p,
                                                       T* __restrict__ wd, int cout_p, int wf_ld,
                                                       uint32_t* __restrict__ kmf, int kmf_words,
                                                       uint32_t* __restrict__ kmd, int kmd_words) {
  pdl_enter();
  extern __shared__ float s_slab[];       // [kCoT][cin_chunk][rs] fp32, sized by the host
  // process channels in chunks of CC so the slab fits in smem
  const int CC = (cin + gridDim.y - 1) / gridDim.y;
  const int c0 = blockIdx.y * CC;
  const int c1 = min(cin, c0 + CC);
  if (c0 >= c1) return;
  stage_slab(w, mask, blockIdx.x * kCoT, cout, c0, c1, cin, rs, wf, cin_p, wf_ld, wd, cout_p, true, s_slab, kmf, kmf_words, kmd, kmd_words);
}

// All masked layers of a model in ONE launch instead of one launch per layer (54 for ResNet-50).
// The operand buffers are persistent and zero-initialised by the host, so channel padding is never rewritten.
struct StageItem {
  const float* w; const float* mask; __nv_bfloat16* wf; __nv_bfloat16* wd;
  int cout, cin, rs, cin_p, cout_p, ysplit, cc, wf_ld;
  long long cta0;                         // first CTA of this layer; CTAs = ceil(cout / kCoT) * ysplit
  uint32_t* kmf; uint32_t* kmd;           // K-block occupancy masks (nullable)
  int kmf_words, kmd_words;
};

// T = float: wf / wd of the items point to fp32 buffers
template <typename T>
__global__ void __launch_bounds__(256) k_stage_weights_batched(const StageItem* __restrict__ items, int n_items) {
  pdl_enter();
  extern __shared__ float s_slab[];
  int lo = 0, hi = n_items - 1;
  const long long b = blockIdx.x;
  while (lo < hi) {                       // last item with cta0 <= b
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].cta0 <= b) lo = mid; else hi = mid - 1;
  }
  const StageItem it = items[lo];
  const int local = (int)(b - it.cta0);
  const int ct = local / it.ysplit, y = local - ct * it.ysplit;
  const int c0 = y * it.cc, c1 = min(it.cin, c0 + it.cc);
  if (ct * kCoT >= it.cout || c0 >= c1) return;
  stage_slab(it.w, it.mask, ct * kCoT, it.cout, c0, c1, it.cin, it.rs, reinterpret_cast<T*>(it.wf), it.cin_p, it.wf_ld,
             reinterpret_cast<T*>(it.wd), it.cout_p, false, s_slab, it.kmf, it.kmf_words, it.kmd, it.kmd_words);
}

// Number of EMPTY blocks of an occupancy mask, stored behind its last row: the GEMM kernels read this one word per CTA
// and walk the K loop without any per-block test when it is zero (every iid unstructured mask: a 64x64 block survives
// any density above ~1e-3) — testing every block cost fprop / dgrad ~12 % at ResNet-50 sizes.
__device__ __forceinline__ void kmask_count_empty(uint32_t* km, int rows, int words, int kblocks) {
  __shared__ unsigned int s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  unsigned int n = 0;
  for (int i = threadIdx.x; i < rows * words; i += blockDim.x) {
    const int wi = i % words;
    const int valid = min(32, kblocks - wi * 32);
    const uint32_t vm = valid >= 32 ? 0xffffffffu : ((1u << valid) - 1u);
    n += __popc(~km[i] & vm);
  }
  if (n) atomicAdd(&s_n, n);
  __syncthreads();
  if (threadIdx.x == 0) km[(size_t)rows * words] = s_n;
  __syncthreads();
}

__global__ void __launch_bounds__(256) k_kmask_summary(const StageItem* __restrict__ items, int n_items) {
  pdl_enter();
  const StageItem it = items[blockIdx.x];
  if (it.kmf) kmask_count_empty(it.kmf, (it.cout + 63) / 64, it.kmf_words, (it.wf_ld + 63) / 64);
  if (it.kmd && it.wd) kmask_count_empty(it.kmd, (it.cin + 63) / 64, it.kmd_words, (it.rs * it.cout_p + 63) / 64);
}

__global__ void __launch_bounds__(256) k_kmask_summary1(uint32_t* kmf, int rows_f, int words_f, int kb_f,
                                                         uint32_t* kmd, int rows_d, int words_d, int kb_d) {
  pdl_enter();
  if (kmf) kmask_count_empty(kmf, rows_f, words_f, kb_f);
  if (kmd) kmask_count_empty(kmd, rows_d, words_d, kb_d);
}

__global__ void k_zero_bf16(__nv_bfloat16* p, long long n) {
  pdl_enter();
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = __float2bfloat16_rn(0.f);
}

// src[n][c][h][w] with arbitrary element strides (fp32 or bf16) -> dst NHWC bf16 [n][h][w][c_pad]
template <typename T>
__global__ void __launch_bounds__(256) k_to_nhwc(const T* __restrict__ src, long long sn, long long sc, long long sh, long long sw,
                                                 int n, int c, int h, int w, __nv_bfloat16* __restrict__ dst, int c_pad) {
  pdl_enter();
  long long total = (long long)n * h * w * c_pad;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    int ci = (int)(i % c_pad);
    long long pix = i / c_pad;
    int wi = (int)(pix % w);
    long long t2 = pix / w;
    int hi = (int)(t2 % h);
    int ni = (int)(t2 / h);
    float v = 0.f;
    if (ci < c) v = (float)src[ni * sn + ci * sc + hi * sh + wi * sw];
    dst[i] = __float2bfloat16_rn(v);
  }
}

// src[n][c][h][w] fp32 (any element strides) -> dst NHWC fp32 [n][h][w][c_pad], channels >= c zero (values unchanged)
__global__ void __launch_bounds__(256) k_to_nhwc_f32(const float* __restrict__ src, long long sn, long long sc, long long sh, long long sw,
                                                     int n, int c, int h, int w, float* __restrict__ dst, int c_pad) {
  pdl_enter();
  const long long total = (long long)n * h * w * c_pad;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    const int ci = (int)(i % c_pad);
    const long long pix = i / c_pad;
    const int wi = (int)(pix % w);
    const long long t2 = pix / w;
    const int hi = (int)(t2 % h), ni = (int)(t2 / h);
    dst[i] = ci < c ? src[ni * sn + ci * sc + hi * sh + wi * sw] : 0.f;
  }
}

// Three-way bf16 split of an fp32 operand for the fp32 weight gradient: dst NHWC bf16 [3n][h][w][c_pad] holds image
// blocks b = 0, 1, 2 of n images each; block `lo_block` holds lo = bf16(v - hi), the other two hi = bf16(v).  v - hi is
// exact in fp32, so hi + lo carries 16 significant bits of v.  Stacking x as (hi, lo, hi) and dy as (hi, hi, lo), ONE
// bf16 wgrad over 3n images sums x_hi dy_hi + x_lo dy_hi + x_hi dy_lo.
__global__ void __launch_bounds__(256) k_wgrad_split3(const float* __restrict__ src, long long sn, long long sc, long long sh, long long sw,
                                                      int n, int c, int h, int w, __nv_bfloat16* __restrict__ dst, int c_pad,
                                                      int lo_block) {
  pdl_enter();
  const long long total = (long long)n * h * w * c_pad;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    const int ci = (int)(i % c_pad);
    const long long pix = i / c_pad;
    const int wi = (int)(pix % w);
    const long long t2 = pix / w;
    const int hi_ = (int)(t2 % h), ni = (int)(t2 / h);
    const float v = ci < c ? src[ni * sn + ci * sc + hi_ * sh + wi * sw] : 0.f;
    const __nv_bfloat16 vh = __float2bfloat16_rn(v);
    const __nv_bfloat16 vl = __float2bfloat16_rn(v - __bfloat162float(vh));
#pragma unroll
    for (int b = 0; b < 3; ++b) dst[i + b * total] = b == lo_block ? vl : vh;
  }
}


// Explicit im2col for convolutions whose input has too few channels for a 128-B TMA row
// (the 3-channel stem conv): x NHWC bf16 [n][h][w][8] -> xcol [n*p*q][kp] bf16 with column
// (r*S + s)*8 + c.  One thread moves one 16-byte (pixel, tap) cell; columns >= r*s*8 are zero.
__global__ void __launch_bounds__(256) k_im2col_c8(const uint4* __restrict__ x, int n, int h, int w,
                                                   int R, int S, int stride_h, int stride_w, int pad_h, int pad_w,
                                                   int P, int Q, uint4* __restrict__ xcol, int kp8) {
  pdl_enter();
  const long long total = (long long)n * P * Q * kp8;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += step) {
    const int cell = (int)(i % kp8);
    const long long pix = i / kp8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (cell < R * S) {
      const int r = cell / S, s = cell - r * S;
      const int q = (int)(pix % Q); const long long t2 = pix / Q;
      const int pp = (int)(t2 % P); const int ni = (int)(t2 / P);
      const int hi = pp * stride_h - pad_h + r, wi = q * stride_w - pad_w + s;
      if (hi >= 0 && hi < h && wi >= 0 && wi < w) v = x[((long long)ni * h + hi) * w + wi];
    }
    xcol[i] = v;
  }
}

// Stem im2col straight from the framework's input tensor (fp32 or bf16, any strides, c <= 8 channels): fuses the
// layout/precision conversion (k_to_nhwc) into the expansion, so the 3-channel image is read once and the
// intermediate NHWC8 copy never exists.  Column (r*S + s)*8 + ch, channels >= c are zero.
template <typename T>
__global__ void __launch_bounds__(256) k_im2col_stem(const T* __restrict__ src, long long sn, long long sc, long long sh, long long sw,
                                                     int n, int c, int h, int w, int R, int S, int cg, int stride_h, int stride_w,
                                                     int pad_h, int pad_w, int P, int Q, uint4* __restrict__ xcol, int kp8) {
  pdl_enter();
  // one thread = one 16-byte cell (8 consecutive columns) of the matrix; column e = tap * cg + channel.  The
  // (row offset, column offset, channel) of every column is decoded once per CTA into shared memory, so the inner
  // loop has no divisions.  cg = channels per tap: the RGB stem uses cg = 3 (K = 152 for 147 real columns) instead
  // of padding every tap to 8 channels (K = 392) — the matrix written here and read by two GEMMs shrinks 2.6x.
  extern __shared__ uint32_t s_col[];                  // [kp8 * 8]: dh << 16 | dw << 8 | ch, or ~0u for padding columns
  const int kp = kp8 * 8;
  for (int e = threadIdx.x; e < kp; e += blockDim.x) {
    uint32_t v = 0xFFFFFFFFu;
    const int tap = e / cg, ch = e - tap * cg;
    if (tap < R * S && ch < c) { const int r = tap / S, s_ = tap - r * S; v = ((uint32_t)r << 16) | ((uint32_t)s_ << 8) | (uint32_t)ch; }
    s_col[e] = v;
  }
  __syncthreads();
  const long long total = (long long)n * P * Q * kp8;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long step = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += step) {
    const int cell = (int)(i % kp8);
    const long long pix = i / kp8;
    const int q = (int)(pix % Q); const long long t2 = pix / Q;
    const int pp = (int)(t2 % P); const int ni = (int)(t2 / P);
    const int h0 = pp * stride_h - pad_h, w0 = q * stride_w - pad_w;
    const T* base = src + ni * sn;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t cd = s_col[cell * 8 + j];
      const int hi = h0 + (int)(cd >> 16), wi = w0 + (int)((cd >> 8) & 0xFF);
      f[j] = 0.f;
      if (cd != 0xFFFFFFFFu && hi >= 0 && hi < h && wi >= 0 && wi < w) f[j] = (float)base[hi * sh + wi * sw + (long long)(cd & 0xFF) * sc];
    }
    uint4 v;
    __nv_bfloat162* hv = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) hv[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
    xcol[i] = v;
  }
}

// The same matrix, one output-row strip per CTA: the R input rows under a strip of QS output pixels are staged ONCE into
// shared memory as bf16 (coalesced reads, padding resolved there), then every 16-byte cell of the strip's rows is a gather
// of 8 halfwords from shared memory with loop-invariant offsets (thread = one cell column, walking the strip's pixels).
// The per-cell kernel above spends its time on 8 bounds-checked scalar global loads + 8 table lookups + 3 divisions per
// cell; this one has none of them in the inner loop.
// TO = float: the fp32 matrix of the TF32 stem GEMM (the patch is staged as fp32, a cell is two 16-byte stores).
template <typename T, typename TO = __nv_bfloat16>
__global__ void __launch_bounds__(256) k_im2col_stem_rows(const T* __restrict__ src, long long sn, long long sc, long long sh, long long sw,
                                                          int n, int c, int h, int w, int R, int S, int cg, int stride_h, int stride_w,
                                                          int pad_h, int pad_w, int P, int Q, int QS, uint4* __restrict__ xcol, int kp8) {
  pdl_enter();
  constexpr bool kF32 = sizeof(TO) == 4;
  extern __shared__ __align__(16) unsigned short s_patch[];      // [R][pw * c] bf16 bits, then one zero slot
  float* const s_patch_f = reinterpret_cast<float*>(s_patch);    // TO = float: the same as fp32 values
  const int pw = (QS - 1) * stride_w + S;                       // input columns under a strip
  const int pitch = pw * c;
  const int zero_slot = R * pitch;
  const int strips_q = (Q + QS - 1) / QS;
  const long long n_strips = (long long)n * P * strips_q;
  // this thread's cell column and its 8 patch offsets (loop invariant)
  const int cells_per_pass = blockDim.x / kp8 * kp8 > 0 ? blockDim.x / kp8 : 0;   // pixels handled per pass
  const int cell = threadIdx.x % kp8, plane = threadIdx.x / kp8;
  const bool worker = plane < cells_per_pass;
  int off[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int e = cell * 8 + j, tap = e / cg, ch = e - tap * cg;
    off[j] = zero_slot;
    if (tap < R * S && ch < c) { const int r = tap / S, s_ = tap - r * S; off[j] = r * pitch + s_ * c + ch; }
  }
  for (long long strip = blockIdx.x; strip < n_strips; strip += gridDim.x) {
    const int sq = (int)(strip % strips_q); long long t = strip / strips_q;
    const int pp = (int)(t % P); const int ni = (int)(t / P);
    const int q0 = sq * QS, nq = min(QS, Q - q0);
    const int h0 = pp * stride_h - pad_h, w0 = q0 * stride_w - pad_w;
    __syncthreads();                                             // previous strip's gathers are done
    const T* base = src + ni * sn;
    const float inv_c = 1.0f / (float)c;
    for (int r = 0; r < R; ++r) {
      const int hh = h0 + r;
      const bool row_in = hh >= 0 && hh < h;
      const T* rowp = base + hh * sh;
      for (int rem = threadIdx.x; rem < pitch; rem += blockDim.x) {
        const int wi = (int)(((float)rem + 0.5f) * inv_c), ch = rem - wi * c;      // rem / c without an integer division (rem < 2^16)
        const int ww = w0 + wi;
        float v = 0.f;
        if (row_in && ww >= 0 && ww < w) v = (float)rowp[ww * sw + (long long)ch * sc];
        if constexpr (kF32) s_patch_f[r * pitch + rem] = v;
        else s_patch[r * pitch + rem] = __bfloat16_as_ushort(__float2bfloat16_rn(v));
      }
    }
    if constexpr (kF32) { if (threadIdx.x == 0) s_patch_f[zero_slot] = 0.f; }
    else { if (threadIdx.x == 0) s_patch[zero_slot] = 0; }
    __syncthreads();
    if (worker) {
      const long long row0 = ((long long)ni * P + pp) * Q + q0;
      for (int ql = plane; ql < nq; ql += cells_per_pass) {
        const int qo = ql * stride_w * c;
        if constexpr (kF32) {
          float hf[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) hf[j] = s_patch_f[off[j] == zero_slot ? zero_slot : off[j] + qo];
          float4* const dst = reinterpret_cast<float4*>(xcol) + ((row0 + ql) * kp8 + cell) * 2;
          dst[0] = make_float4(hf[0], hf[1], hf[2], hf[3]);
          dst[1] = make_float4(hf[4], hf[5], hf[6], hf[7]);
        } else {
          unsigned short hv[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) hv[j] = s_patch[off[j] == zero_slot ? zero_slot : off[j] + qo];
          uint4 v;
          v.x = hv[0] | ((unsigned)hv[1] << 16); v.y = hv[2] | ((unsigned)hv[3] << 16);
          v.z = hv[4] | ((unsigned)hv[5] << 16); v.w = hv[6] | ((unsigned)hv[7] << 16);
          xcol[(row0 + ql) * kp8 + cell] = v;
        }
      }
    }
  }
}

// torch.optim.SGD (momentum, weight_decay, dampening 0, nesterov False) — one launch for all
// parameters.  20 B/elem: read w,g,buf; write w,buf.
__global__ void __launch_bounds__(256) k_sgd(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                             const float* __restrict__ lr_p, float mu, float wd, int first) {
  pdl_enter();
  const float lr = *lr_p;
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    float* wp = const_cast<float*>(sg.w) + base;
    const float* gp = sg.g + base;
    float* bp = sg.buf + base;
    bool vec = n_in == kTileElems && ((((uintptr_t)wp) | ((uintptr_t)gp) | ((uintptr_t)bp)) & 15) == 0;
    if (vec) {
#pragma unroll
      for (int it = 0; it < kTileElems / (256 * 4); ++it) {
        int q = it * 256 + t;
        float4 w = ((const float4*)wp)[q];
        float4 g = ld_stream((const float4*)gp + q);
        float4 b = first ? make_float4(0.f, 0.f, 0.f, 0.f) : ((const float4*)bp)[q];
        float4 d;
        d.x = fmaf(wd, w.x, g.x); d.y = fmaf(wd, w.y, g.y); d.z = fmaf(wd, w.z, g.z); d.w = fmaf(wd, w.w, g.w);
        // buf.mul_(mu).add_(d): two separately rounded ops in torch (no FMA contraction)
        if (!first) { b.x = __fadd_rn(__fmul_rn(mu, b.x), d.x); b.y = __fadd_rn(__fmul_rn(mu, b.y), d.y); b.z = __fadd_rn(__fmul_rn(mu, b.z), d.z); b.w = __fadd_rn(__fmul_rn(mu, b.w), d.w); }
        else b = d;
        w.x = fmaf(-lr, b.x, w.x); w.y = fmaf(-lr, b.y, w.y); w.z = fmaf(-lr, b.z, w.z); w.w = fmaf(-lr, b.w, w.w);
        ((float4*)bp)[q] = b;
        ((float4*)wp)[q] = w;
      }
    } else {
      for (int i = t; i < n_in; i += 256) {
        float w = wp[i], g = gp[i];
        float d = fmaf(wd, w, g);
        float b = first ? d : __fadd_rn(__fmul_rn(mu, bp[i]), d);
        bp[i] = b;
        wp[i] = fmaf(-lr, b, w);
      }
    }
  }
}

// torch.optim.AdamW, capturable foreach branch (torch/optim/adam.py, _multi_tensor_adam): one launch for all parameters.
// 28 B/elem: read w, g, m, v; write w, m, v.  The segment table is SGD's with these roles:
//   w = weight, g = gradient, buf = exp_avg (m), mo = exp_avg_sq (v), m = the parameter's fp32 step count (0-dim).
// Every op is the one ATen runs, in the same order and rounding (opmath fp32; the scalars are Python doubles rounded to
// fp32, as Scalar.to<float>() does):
//   _foreach_mul_(w, c)                      w * c                          c = fp32(1 - lr * wd), only when wd != 0
//   _foreach_lerp_(m, g, 1 - b1)             ATen's two-branch lerp; nvcc contracts `self + weight * (end - self)` into
//                                            one FMA (the torch build compiles with the default -fmad=true)
//   _foreach_mul_(v, b2)                     v * b2
//   _foreach_addcmul_(v, g, g, 1 - b2)       fma(1 - b2, g * g, v)          DeviceAddCmulCdiv.cuh: explicit std::fma
//   _foreach_pow(b, step)                    powf(b, t)                     Pow.cuh: ::pow(float, float)
//   s = 1 / ((pow(b1, t) - 1) / lr)          _foreach_div_(x, lr) is x * fp32(1.0 / lr), the reciprocal taken in
//                                            double from the Python float (a plain x / fp32(lr) differs in ~1/3 of
//                                            the (t, lr) pairs); then an IEEE reciprocal  (s: the negative step size)
//   b = sqrt(-(pow(b2, t) - 1))              IEEE square root
//   d = (sqrt(v) / b + eps) / s              IEEE ops, no contraction possible
//   _foreach_addcdiv_(w, m, d)               w + m / d                      alpha == 1: no FMA
// Settled on an H100 against torch 2.11 / CUDA 12.8 (tests/test_adamw.py compares every bit of w, m, v and step; powf
// matched ATen's for every t in 1..300 and 10001..10059).  The lerp is adamw_lerp (tp_common.cuh).

struct AdamWCoef { float c, w1, omw1, b2, w2, eps, s, b; bool decay, small; };

__device__ __forceinline__ void adamw_elem(float& w, float g, float& m, float& v, const AdamWCoef& k) {
  if (k.decay) w = __fmul_rn(w, k.c);
  m = adamw_lerp(m, g, k.w1, k.omw1, k.small);
  v = fmaf(k.w2, __fmul_rn(g, g), __fmul_rn(v, k.b2));
  const float d = __fdiv_rn(__fadd_rn(__fdiv_rn(__fsqrt_rn(v), k.b), k.eps), k.s);
  w = __fadd_rn(w, __fdiv_rn(m, d));
}

// step += 1 for every segment: a launch of its own so that the update kernel's CTAs all read the incremented count
__global__ void k_adamw_count(const Seg* __restrict__ segs, int n_seg) {
  pdl_enter();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_seg) {
    float* st = const_cast<float*>(segs[i].m);
    *st = __fadd_rn(*st, 1.f);
  }
}

__global__ void __launch_bounds__(256) k_adamw(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                               const float* __restrict__ inv_lr_p, const float* __restrict__ decay_p,
                                               float b1, float b2, float w1, float w2, float eps) {
  pdl_enter();
  AdamWCoef k;
  const float inv_lr = *inv_lr_p;
  k.decay = decay_p != nullptr;
  k.c = k.decay ? *decay_p : 1.f;
  k.w1 = w1; k.omw1 = __fsub_rn(1.f, w1); k.small = fabsf(w1) < 0.5f;
  k.b2 = b2; k.w2 = w2; k.eps = eps;
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const Seg sg = segs[si];
    const float step = *sg.m;
    k.s = __fdiv_rn(1.f, __fmul_rn(__fsub_rn(powf(b1, step), 1.f), inv_lr));
    k.b = __fsqrt_rn(-__fsub_rn(powf(b2, step), 1.f));
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    float* wp = const_cast<float*>(sg.w) + base;
    const float* gp = sg.g + base;
    float* mp = sg.buf + base;
    float* vp = sg.mo + base;
    const bool vec = n_in == kTileElems && ((((uintptr_t)wp) | ((uintptr_t)gp) | ((uintptr_t)mp) | ((uintptr_t)vp)) & 15) == 0;
    if (vec) {
#pragma unroll
      for (int it = 0; it < kTileElems / (256 * 4); ++it) {
        const int q = it * 256 + t;
        float4 w = ((const float4*)wp)[q], m = ((const float4*)mp)[q], v = ((const float4*)vp)[q];
        const float4 g = ld_stream((const float4*)gp + q);
        adamw_elem(w.x, g.x, m.x, v.x, k); adamw_elem(w.y, g.y, m.y, v.y, k);
        adamw_elem(w.z, g.z, m.z, v.z, k); adamw_elem(w.w, g.w, m.w, v.w, k);
        ((float4*)mp)[q] = m;
        ((float4*)vp)[q] = v;
        ((float4*)wp)[q] = w;
      }
    } else {
      for (int i = t; i < n_in; i += 256) {
        float w = wp[i], m = mp[i], v = vp[i];
        adamw_elem(w, gp[i], m, v, k);
        mp[i] = m; vp[i] = v; wp[i] = w;
      }
    }
  }
}

// Schedule-Free SGD (Defazio et al. 2024; the schedulefree package's SGDScheduleFree, foreach branch): one launch for all
// parameters.  20 B/elem: read y, g, z; write y, z (the four torch launches move 48 B/elem, 36 without weight decay).
// The segment table is SGD's with these roles: w = y (the parameter), g = gradient, buf = z.  Per element, the ops ATen
// runs, in the same order and rounding (opmath fp32; lr, ckp1 and alpha_y = lr * (momentum * (1 - ckp1) - 1) are Python
// doubles rounded to fp32, as Scalar.to<float>() does):
//   _foreach_add_(g, y, alpha=wd)        g' = fma(wd, y, g)             only when wd != 0 (as in k_sgd)
//   _foreach_lerp_(y, z, weight=ckp1)    ATen's two-branch lerp (adamw_lerp, tp_common.cuh)
//   _foreach_add_(y, g', alpha=alpha_y)  fma(alpha_y, g', y)            ATen's `a + alpha * b`, contracted by nvcc
//   _foreach_sub_(z, g', alpha=lr)       fma(-lr, g', z)                ATen's `a - alpha * b`, contracted the same way
// Settled on an H100 against torch 2.11 / CUDA 12.8: tests/test_schedulefree.py compares every bit of y and z with the
// torch sequence over ResNet-50's and DeiT-S's parameters, with and without weight decay, through the warm-up.
// The package also writes g' back into the gradient; nothing reads p.grad after the step (the gradient storage is zeroed
// before the next backward), so this kernel does not.  first != 0: z does not exist yet and starts as a copy of y
// (the package's clone(p)), made here instead of in a launch of its own.
struct SFCoef { float lr, ckp1, omc, ay, wd; bool decay, small; };

__device__ __forceinline__ void schedulefree_elem(float& y, float g, float& z, const SFCoef& k) {
  const float gd = k.decay ? fmaf(k.wd, y, g) : g;
  y = fmaf(k.ay, gd, adamw_lerp(y, z, k.ckp1, k.omc, k.small));
  z = fmaf(-k.lr, gd, z);
}

__global__ void __launch_bounds__(256) k_schedulefree(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                      const float* __restrict__ sc, float wd, int decay, int first) {
  pdl_enter();
  SFCoef k;
  k.lr = sc[0]; k.ckp1 = sc[1]; k.ay = sc[2]; k.wd = wd; k.decay = decay != 0;
  k.omc = __fsub_rn(1.f, k.ckp1); k.small = fabsf(k.ckp1) < 0.5f;
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const Seg sg = segs[find_seg(segs, n_seg, tile)];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    float* yp = const_cast<float*>(sg.w) + base;
    const float* gp = sg.g + base;
    float* zp = sg.buf + base;
    const bool vec = n_in == kTileElems && ((((uintptr_t)yp) | ((uintptr_t)gp) | ((uintptr_t)zp)) & 15) == 0;
    if (vec) {
#pragma unroll
      for (int it = 0; it < kTileElems / (256 * 4); ++it) {
        const int q = it * 256 + t;
        float4 y = ((const float4*)yp)[q];
        const float4 g = ld_stream((const float4*)gp + q);
        float4 z = first ? y : ((const float4*)zp)[q];
        schedulefree_elem(y.x, g.x, z.x, k); schedulefree_elem(y.y, g.y, z.y, k);
        schedulefree_elem(y.z, g.z, z.z, k); schedulefree_elem(y.w, g.w, z.w, k);
        ((float4*)zp)[q] = z;
        ((float4*)yp)[q] = y;
      }
    } else {
      for (int i = t; i < n_in; i += 256) {
        float y = yp[i], z = first ? yp[i] : zp[i];
        schedulefree_elem(y, gp[i], z, k);
        zp[i] = z; yp[i] = y;
      }
    }
  }
}

// y = lerp(y, z, w) for every segment (w = y, buf = z): torch's per-tensor Tensor.lerp_(z, w) with a Python-scalar weight,
// the schedule-free train() / eval() switch.  12 B/elem.
__global__ void __launch_bounds__(256) k_lerp_segs(const Seg* __restrict__ segs, int n_seg, long long tiles, float wt) {
  pdl_enter();
  const float omw = __fsub_rn(1.f, wt);
  const bool small = fabsf(wt) < 0.5f;
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const Seg sg = segs[find_seg(segs, n_seg, tile)];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    float* yp = const_cast<float*>(sg.w) + base;
    const float* zp = sg.buf + base;
    if (n_in == kTileElems && ((((uintptr_t)yp) | ((uintptr_t)zp)) & 15) == 0) {
#pragma unroll
      for (int it = 0; it < kTileElems / (256 * 4); ++it) {
        const int q = it * 256 + t;
        float4 y = ((const float4*)yp)[q];
        const float4 z = ld_stream((const float4*)zp + q);
        y.x = adamw_lerp(y.x, z.x, wt, omw, small); y.y = adamw_lerp(y.y, z.y, wt, omw, small);
        y.z = adamw_lerp(y.z, z.z, wt, omw, small); y.w = adamw_lerp(y.w, z.w, wt, omw, small);
        ((float4*)yp)[q] = y;
      }
    } else {
      for (int i = t; i < n_in; i += 256) yp[i] = adamw_lerp(yp[i], zp[i], wt, omw, small);
    }
  }
}

// The segment table of an optimizer launch: uploaded, or (table_cached) the one an earlier call with the same pointers
// left in `ws`, in which case only the tiles are counted and no host->device copy is issued (capturable).
static int seg_table(Arena& ar, int table_cached, void* const* w, const void* const* g, void* const* buf,
                     const int64_t* numel, int n_seg, Seg** d_segs, long long* tiles, cudaStream_t st) {
  *tiles = 0;
  if (!table_cached) return upload_segs(ar, (const void* const*)w, g, nullptr, nullptr, buf, numel, n_seg, d_segs, tiles, nullptr, st);
  *d_segs = (Seg*)ar.take(sizeof(Seg) * n_seg);
  if (!*d_segs) return TP_ERR_WORKSPACE;
  for (int i = 0; i < n_seg; ++i) {
    if (numel[i] < 0) return TP_ERR_INVALID;
    *tiles += (numel[i] + kTileElems - 1) / kTileElems;
  }
  return TP_OK;
}

}  // namespace tp

using namespace tp;

extern "C" {

size_t tp_kblock_mask_words(int64_t columns) {
  if (columns <= 0) return 0;
  return (size_t)(((columns + 63) / 64 + 31) / 32);
}

int tp_stage_weights(const void* w, const void* mask, int cout, int cin, int r, int s,
                     void* wf, int cin_p, int wf_ld, void* wd, int cout_p, int cin_p2,
                     void* kmask_f, void* kmask_d, void* stream) {
  if (!w || !mask || !wf || cout <= 0 || cin <= 0 || r <= 0 || s <= 0 || cin_p < cin) return TP_ERR_INVALID;
  if (wd && (cout_p < cout || cin_p2 < cin)) return TP_ERR_INVALID;
  if (wf_ld <= 0) wf_ld = r * s * cin_p;
  if (wf_ld < r * s * cin_p) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const int rs = r * s;
  // slab of at most 8192 floats (32 KB) per CTA: kCoT output channels x cc input channels x rs taps
  int max_c = kSlabFloats / (kCoT * rs); if (max_c < 1) return TP_ERR_UNSUPPORTED;
  int ysplit = (cin + max_c - 1) / max_c;
  int cc = (cin + ysplit - 1) / ysplit;
  size_t smem = (size_t)kCoT * cc * rs * sizeof(float);
  if (wd) {
    long long nz = (long long)cin_p2 * rs * cout_p;
    if (cout_p > cout || cin_p2 > cin) {
      launch(k_zero_bf16, (unsigned)min((nz + 255) / 256, (long long)sm_count() * 16), 256, 0, st, (__nv_bfloat16*)wd, nz);
    }
  }
  const int kmf_words = (int)tp_kblock_mask_words(wf_ld), kmd_words = (int)tp_kblock_mask_words((int64_t)rs * cout_p);
  if (kmask_f) TP_CUDA_CHECK(cudaMemsetAsync(kmask_f, 0, ((size_t)((cout + 63) / 64) * kmf_words + 1) * 4, st));
  if (kmask_d && wd) TP_CUDA_CHECK(cudaMemsetAsync(kmask_d, 0, ((size_t)((cin + 63) / 64) * kmd_words + 1) * 4, st));
  dim3 grid((cout + kCoT - 1) / kCoT, ysplit);
  launch(k_stage_weights<__nv_bfloat16>, grid, 256, smem, st, (const float*)w, (const float*)mask, cout, cin, rs,
                                           (__nv_bfloat16*)wf, cin_p, (__nv_bfloat16*)wd, cout_p, wf_ld,
                                           (uint32_t*)kmask_f, kmf_words, (uint32_t*)kmask_d, kmd_words);
  if (kmask_f || (kmask_d && wd))
    launch(k_kmask_summary1, 1, 256, 0, st, (uint32_t*)kmask_f, (cout + 63) / 64, kmf_words, (wf_ld + 63) / 64,
                                         wd ? (uint32_t*)kmask_d : nullptr, (cin + 63) / 64, kmd_words, (rs * cout_p + 63) / 64);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_stage_weights_f32(const void* w, const void* mask, int cout, int cin, int r, int s,
                         void* wf, int cin_p, int wf_ld, void* wd, int cout_p, void* stream) {
  if (!w || !mask || !wf || cout <= 0 || cin <= 0 || r <= 0 || s <= 0 || cin_p < cin) return TP_ERR_INVALID;
  if (wd && cout_p < cout) return TP_ERR_INVALID;
  if (wf_ld <= 0) wf_ld = r * s * cin_p;
  if (wf_ld < r * s * cin_p) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const int rs = r * s;
  int max_c = kSlabFloats / (kCoT * rs); if (max_c < 1) return TP_ERR_UNSUPPORTED;
  const int ysplit = (cin + max_c - 1) / max_c;
  const int cc = (cin + ysplit - 1) / ysplit;
  const size_t smem = (size_t)kCoT * cc * rs * sizeof(float);
  if (wd && cout_p > cout) TP_CUDA_CHECK(cudaMemsetAsync(wd, 0, (size_t)cin * rs * cout_p * sizeof(float), st));
  launch(k_stage_weights<float>, dim3((cout + kCoT - 1) / kCoT, ysplit), 256, smem, st, (const float*)w, (const float*)mask,
         cout, cin, rs, (float*)wf, cin_p, (float*)wd, cout_p, wf_ld, (uint32_t*)nullptr, 0, (uint32_t*)nullptr, 0);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

size_t tp_stage_batched_workspace_bytes(int n_items) {
  return n_items > 0 ? (size_t)n_items * sizeof(StageItem) + 512 : 0;
}

static int stage_batched_impl(const tp_stage_item* items, int n_items, int table_cached, void* kmask_all, size_t kmask_bytes,
                              void* ws, size_t ws_bytes, void* stream, bool f32);

int tp_stage_weights_batched(const tp_stage_item* items, int n_items, int table_cached, void* kmask_all, size_t kmask_bytes,
                             void* ws, size_t ws_bytes, void* stream) {
  return stage_batched_impl(items, n_items, table_cached, kmask_all, kmask_bytes, ws, ws_bytes, stream, false);
}

int tp_stage_weights_batched_f32(const tp_stage_item* items, int n_items, int table_cached, void* ws, size_t ws_bytes, void* stream) {
  for (int i = 0; items && i < n_items; ++i)
    if (items[i].kmask_f || items[i].kmask_d) return TP_ERR_INVALID;          // fp32 operands carry no occupancy masks
  return stage_batched_impl(items, n_items, table_cached, nullptr, 0, ws, ws_bytes, stream, true);
}

static int stage_batched_impl(const tp_stage_item* items, int n_items, int table_cached, void* kmask_all, size_t kmask_bytes,
                              void* ws, size_t ws_bytes, void* stream, bool f32) {
  if (!items || n_items <= 0 || !ws) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  StageItem* d_items = (StageItem*)ar.take(sizeof(StageItem) * n_items);
  if (!d_items) return TP_ERR_WORKSPACE;
  std::vector<StageItem> h(n_items);
  long long cta = 0; size_t smem = 0;
  for (int i = 0; i < n_items; ++i) {
    const tp_stage_item& q = items[i];
    if (!q.w || !q.mask || !q.wf || q.cout <= 0 || q.cin <= 0 || q.r <= 0 || q.s <= 0 || q.cin_p < q.cin) return TP_ERR_INVALID;
    if (q.wd && q.cout_p < q.cout) return TP_ERR_INVALID;
    const int rs = q.r * q.s;
    int max_c = kSlabFloats / (kCoT * rs); if (max_c < 1) return TP_ERR_UNSUPPORTED;      // slab of at most 32 KB per CTA
    const int ysplit = (q.cin + max_c - 1) / max_c;
    const int cc = (q.cin + ysplit - 1) / ysplit;
    StageItem& t = h[i];
    t.w = (const float*)q.w; t.mask = (const float*)q.mask; t.wf = (__nv_bfloat16*)q.wf; t.wd = (__nv_bfloat16*)q.wd;
    t.cout = q.cout; t.cin = q.cin; t.rs = rs; t.cin_p = q.cin_p; t.cout_p = q.cout_p; t.ysplit = ysplit; t.cc = cc;
    t.wf_ld = q.wf_ld > 0 ? q.wf_ld : rs * q.cin_p;
    if (t.wf_ld < rs * q.cin_p) return TP_ERR_INVALID;
    t.cta0 = cta;
    t.kmf = (uint32_t*)q.kmask_f; t.kmd = (uint32_t*)q.kmask_d;
    t.kmf_words = (int)tp_kblock_mask_words(t.wf_ld); t.kmd_words = (int)tp_kblock_mask_words((int64_t)rs * q.cout_p);
    cta += (long long)((q.cout + kCoT - 1) / kCoT) * ysplit;
    const size_t need = (size_t)kCoT * cc * rs * sizeof(float);
    if (need > smem) smem = need;
  }
  if (cta > 0x7fffffffll) return TP_ERR_UNSUPPORTED;
  if (!table_cached)   // pageable source: staged by the runtime before returning (not capturable: cache the table first)
    TP_CUDA_CHECK(cudaMemcpyAsync(d_items, h.data(), sizeof(StageItem) * n_items, cudaMemcpyHostToDevice, st));
  if (kmask_all && kmask_bytes) TP_CUDA_CHECK(cudaMemsetAsync(kmask_all, 0, kmask_bytes, st));   // all layers' occupancy masks: one memset node
  if (f32) launch(k_stage_weights_batched<float>, (unsigned)cta, 256, smem, st, d_items, n_items);
  else launch(k_stage_weights_batched<__nv_bfloat16>, (unsigned)cta, 256, smem, st, d_items, n_items);
  if (kmask_all && kmask_bytes) launch(k_kmask_summary, n_items, 256, 0, st, d_items, n_items);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_to_nhwc_bf16(const void* src, int src_dtype, int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                    int n, int c, int h, int w, void* dst, int c_pad, void* stream) {
  if (!src || !dst || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  long long total = (long long)n * h * w * c_pad;
  unsigned grid = (unsigned)min((total + 255) / 256, (long long)sm_count() * 32);
  if (src_dtype == 0) launch(k_to_nhwc<float>, grid, 256, 0, st, (const float*)src, sn, sc, sh, sw, n, c, h, w, (__nv_bfloat16*)dst, c_pad);
  else if (src_dtype == 1) launch(k_to_nhwc<__nv_bfloat16>, grid, 256, 0, st, (const __nv_bfloat16*)src, sn, sc, sh, sw, n, c, h, w, (__nv_bfloat16*)dst, c_pad);
  else return TP_ERR_INVALID;
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_to_nhwc_f32(const void* src, int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                   int n, int c, int h, int w, void* dst, int c_pad, void* stream) {
  if (!src || !dst || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)n * h * w * c_pad;
  const unsigned grid = (unsigned)min((total + 255) / 256, (long long)sm_count() * 32);
  launch(k_to_nhwc_f32, grid, 256, 0, st, (const float*)src, sn, sc, sh, sw, n, c, h, w, (float*)dst, c_pad);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_wgrad_split3(const void* src, int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                    int n, int c, int h, int w, void* dst, int c_pad, int lo_block, void* stream) {
  if (!src || !dst || n <= 0 || c <= 0 || h <= 0 || w <= 0 || c_pad < c || lo_block < 0 || lo_block > 2) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)n * h * w * c_pad;
  const unsigned grid = (unsigned)min((total + 255) / 256, (long long)sm_count() * 32);
  launch(k_wgrad_split3, grid, 256, 0, st, (const float*)src, sn, sc, sh, sw, n, c, h, w, (__nv_bfloat16*)dst, c_pad, lo_block);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_im2col_stem_f32(const void* src, int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                       int n, int c, int h, int w, int r, int s, int cg, int stride_h, int stride_w, int pad_h, int pad_w,
                       int p, int q, void* xcol, int kp, void* stream) {
  if (!src || !xcol || n <= 0 || c <= 0 || c > 8 || cg < c || cg > 8 || kp % 8 != 0 || kp < r * s * cg) return TP_ERR_INVALID;
  if (r > 255 || s > 255 || kp > 8192) return TP_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const int QS = q < 128 ? q : 128;
  const int pw = (QS - 1) * stride_w + s;
  const size_t patch = ((size_t)r * pw * c + 8) * sizeof(float);
  if (patch > 80 * 1024 || kp / 8 > 256) return TP_ERR_UNSUPPORTED;
  if (patch > 48 * 1024)
    TP_CUDA_CHECK(cudaFuncSetAttribute(k_im2col_stem_rows<float, float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)patch));
  const long long strips = (long long)n * p * ((q + QS - 1) / QS);
  const unsigned g2 = (unsigned)min(strips, (long long)sm_count() * 8);
  launch(k_im2col_stem_rows<float, float>, g2, 256, patch, st, (const float*)src, sn, sc, sh, sw, n, c, h, w, r, s, cg, stride_h,
         stride_w, pad_h, pad_w, p, q, QS, (uint4*)xcol, kp / 8);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_im2col_c8(const void* x, int n, int h, int w, int r, int s, int stride_h, int stride_w,
                 int pad_h, int pad_w, int p, int q, void* xcol, int kp, void* stream) {
  if (!x || !xcol || n <= 0 || kp % 8 != 0 || kp < r * s * 8) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)n * p * q * (kp / 8);
  unsigned grid = (unsigned)min((total + 255) / 256, (long long)sm_count() * 32);
  launch(k_im2col_c8, grid, 256, 0, st, (const uint4*)x, n, h, w, r, s, stride_h, stride_w, pad_h, pad_w, p, q, (uint4*)xcol, kp / 8);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_im2col_stem(const void* src, int src_dtype, int64_t sn, int64_t sc, int64_t sh, int64_t sw,
                   int n, int c, int h, int w, int r, int s, int cg, int stride_h, int stride_w, int pad_h, int pad_w,
                   int p, int q, void* xcol, int kp, void* stream) {
  if (!src || !xcol || n <= 0 || c <= 0 || c > 8 || cg < c || cg > 8 || kp % 8 != 0 || kp < r * s * cg) return TP_ERR_INVALID;
  if (r > 255 || s > 255 || kp > 8192) return TP_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  // strip kernel: one output-row strip of up to 128 pixels per CTA, if its input patch fits in 40 KB of shared memory
  {
    const int QS = q < 128 ? q : 128;
    const int pw = (QS - 1) * stride_w + s;
    const size_t patch = ((size_t)r * pw * c + 8) * sizeof(unsigned short);
    const char* e = getenv("TP_STEM_IM2COL");
    if (patch <= 40 * 1024 && kp / 8 <= 256 && !(e && e[0] == 'c')) {        // TP_STEM_IM2COL=cell: the per-cell kernel (tests compare both)
      const long long strips = (long long)n * p * ((q + QS - 1) / QS);
      const unsigned g2 = (unsigned)min(strips, (long long)sm_count() * 8);
      if (src_dtype == 0)
        launch(k_im2col_stem_rows<float>, g2, 256, patch, st, (const float*)src, sn, sc, sh, sw, n, c, h, w, r, s, cg, stride_h, stride_w, pad_h, pad_w, p, q, QS, (uint4*)xcol, kp / 8);
      else if (src_dtype == 1)
        launch(k_im2col_stem_rows<__nv_bfloat16>, g2, 256, patch, st, (const __nv_bfloat16*)src, sn, sc, sh, sw, n, c, h, w, r, s, cg, stride_h, stride_w, pad_h, pad_w, p, q, QS, (uint4*)xcol, kp / 8);
      else return TP_ERR_INVALID;
      TP_LAUNCH_CHECK();
      return TP_OK;
    }
  }
  const long long total = (long long)n * p * q * (kp / 8);
  unsigned grid = (unsigned)min((total + 255) / 256, (long long)sm_count() * 32);
  const size_t smem = (size_t)kp * sizeof(uint32_t);
  if (src_dtype == 0)
    launch(k_im2col_stem<float>, grid, 256, smem, st, (const float*)src, sn, sc, sh, sw, n, c, h, w, r, s, cg, stride_h, stride_w, pad_h, pad_w, p, q, (uint4*)xcol, kp / 8);
  else if (src_dtype == 1)
    launch(k_im2col_stem<__nv_bfloat16>, grid, 256, smem, st, (const __nv_bfloat16*)src, sn, sc, sh, sw, n, c, h, w, r, s, cg, stride_h, stride_w, pad_h, pad_w, p, q, (uint4*)xcol, kp / 8);
  else return TP_ERR_INVALID;
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_sgd_momentum(void* const* w, const void* const* g, void* const* buf, const int64_t* numel,
                    int n_seg, const float* lr_dev, float momentum, float weight_decay,
                    int first_step, int table_cached, void* ws, size_t ws_bytes, void* stream) {
  if (!numel || n_seg <= 0 || !lr_dev || !ws) return TP_ERR_INVALID;
  if (!table_cached && (!w || !g || !buf)) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  if (table_cached) {
    // the caller guarantees `ws` still holds the table uploaded by an earlier call with the same
    // pointers: no host->device copy, so the call can be captured into a CUDA graph
    d_segs = (Seg*)ar.take(sizeof(Seg) * n_seg);
    if (!d_segs) return TP_ERR_WORKSPACE;
    for (int i = 0; i < n_seg; ++i) tiles += (numel[i] + kTileElems - 1) / kTileElems;
  } else {
    int rc = upload_segs(ar, (const void* const*)w, g, nullptr, nullptr, buf, numel, n_seg, &d_segs, &tiles, nullptr, st);
    if (rc) return rc;
  }
  if (tiles == 0) return TP_OK;
  long long gmax = (long long)sm_count() * 8;
  launch(k_sgd, (unsigned)(tiles < gmax ? tiles : gmax), 256, 0, st, d_segs, n_seg, tiles, lr_dev, momentum, weight_decay, first_step);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_adamw(void* const* w, const void* const* g, void* const* exp_avg, void* const* exp_avg_sq, void* const* step,
             const int64_t* numel, int n_seg, const float* inv_lr_dev, const float* decay_dev,
             double beta1, double beta2, double eps, int table_cached, void* ws, size_t ws_bytes, void* stream) {
  if (!numel || n_seg <= 0 || !inv_lr_dev || !ws) return TP_ERR_INVALID;
  if (!table_cached && (!w || !g || !exp_avg || !exp_avg_sq || !step)) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  if (table_cached) {
    // as tp_sgd_momentum: `ws` still holds the table of an earlier call with the same pointers (capturable)
    d_segs = (Seg*)ar.take(sizeof(Seg) * n_seg);
    if (!d_segs) return TP_ERR_WORKSPACE;
    for (int i = 0; i < n_seg; ++i) tiles += (numel[i] + kTileElems - 1) / kTileElems;
  } else {
    int rc = upload_segs(ar, (const void* const*)w, g, (const void* const*)step, exp_avg_sq, exp_avg, numel, n_seg,
                         &d_segs, &tiles, nullptr, st);
    if (rc) return rc;
  }
  launch(k_adamw_count, (unsigned)((n_seg + 255) / 256), 256, 0, st, (const Seg*)d_segs, n_seg);
  if (tiles > 0) {
    // the scalars as Python forms them: 1 - beta in double, then fp32 (Scalar.to<float>())
    const long long gmax = (long long)sm_count() * 8;
    launch(k_adamw, (unsigned)(tiles < gmax ? tiles : gmax), 256, 0, st, (const Seg*)d_segs, n_seg, tiles, inv_lr_dev, decay_dev,
           (float)beta1, (float)beta2, (float)(1.0 - beta1), (float)(1.0 - beta2), (float)eps);
  }
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_schedulefree_sgd(void* const* y, const void* const* g, void* const* z, const int64_t* numel, int n_seg,
                        const float* scalars_dev, double weight_decay, int first_step, int table_cached,
                        void* ws, size_t ws_bytes, void* stream) {
  if (!numel || n_seg <= 0 || !scalars_dev || !ws) return TP_ERR_INVALID;
  if (!table_cached && (!y || !g || !z)) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  int rc = seg_table(ar, table_cached, y, g, z, numel, n_seg, &d_segs, &tiles, st);
  if (rc) return rc;
  if (tiles == 0) return TP_OK;
  const long long gmax = (long long)sm_count() * 8;
  launch(k_schedulefree, (unsigned)(tiles < gmax ? tiles : gmax), 256, 0, st, (const Seg*)d_segs, n_seg, tiles, scalars_dev,
         (float)weight_decay, weight_decay != 0.0 ? 1 : 0, first_step ? 1 : 0);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_schedulefree_swap(void* const* y, const void* const* z, const int64_t* numel, int n_seg, double weight,
                         int table_cached, void* ws, size_t ws_bytes, void* stream) {
  if (!numel || n_seg <= 0 || !ws) return TP_ERR_INVALID;
  if (!table_cached && (!y || !z)) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  int rc = seg_table(ar, table_cached, y, nullptr, (void* const*)z, numel, n_seg, &d_segs, &tiles, st);
  if (rc) return rc;
  if (tiles == 0) return TP_OK;
  const long long gmax = (long long)sm_count() * 8;
  launch(k_lerp_segs, (unsigned)(tiles < gmax ? tiles : gmax), 256, 0, st, (const Seg*)d_segs, n_seg, tiles, (float)weight);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // extern "C"
