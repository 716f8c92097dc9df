// Data path either side of the model (SURVEY.md §8(f) row 3), sm_90a, HBM-bound:
//
//   k_cifar_augment : the airbench-style GPU augmentation of the reference's CifarLoader.__iter__
//                     (utils/dataset.py:192-226): random translate = batch_crop of the reflect-padded images (:43-69),
//                     per-image left-right flip (:38-40) and cutout (:72-98), fused into ONE gather pass — the
//                     reference runs a masked-assignment loop over 2(2r+1) shifts, a where() and a masked_fill(), each a
//                     full pass.  With a source index it is also the batch gather (images[perm[slice]]), so an epoch
//                     never writes a whole augmented copy of the data set.  The random draws (shifts, flip mask, cutout corners) stay torch's: their RNG stream is
//                     part of the parity contract, exactly like set_er_mask.
//   k_resized_crop  : the ImageNet loader's per-batch crop: each output image is a box of a decoded uint8 image,
//                     resized with PIL's bilinear (antialiased triangle) filter, optionally mirrored and normalised,
//                     written channels_last fp32 — one launch builds the whole batch from a table of boxes.
//   k_synth_normal / k_synth_labels : the synthetic on-device generator standing in for FFCV / the CIFAR tensors
//                     (no data sets here): counter-based Philox4x32-10 -> Box-Muller, four values per counter, written
//                     with 16-byte stores straight into the batch buffer (N(0,1) images — FFCV hands over
//                     mean/std-normalised fp32, dataset.py:391 — and uniform int64 labels).
#include "tp_common.cuh"

namespace tp {

// out[n][c][y][x] = cut(s, y, x) ? 0 : src[s][c][y + r + sy[s]][xf + r + sx[s]],  xf = flip[s] ? W-1-x : x,
// s = idx ? idx[n] : n.  src is [N_src][C][H+2r][W+2r] (r = 0 and no shifts: plain flip / cutout); every array of draws is
// optional and, like the reference's whole-dataset draws, indexed by the SOURCE image.
__global__ void __launch_bounds__(256) k_cifar_augment(const float* __restrict__ src, float* __restrict__ out,
                                                       const long long* __restrict__ idx,
                                                       const long long* __restrict__ shifts, const unsigned char* __restrict__ flip,
                                                       const long long* __restrict__ cut_y, const long long* __restrict__ cut_x,
                                                       int cut_size, int N, int C, int H, int W, int r) {
  const int Hp = H + 2 * r, Wp = W + 2 * r;
  const long long total = (long long)N * C * H * W;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % W); long long t = i / W;
    const int y = (int)(t % H); t /= H;
    const int c = (int)(t % C); const int n = (int)(t / C);
    const long long s = idx ? idx[n] : (long long)n;
    float v = 0.f;
    bool cut = false;
    if (cut_y) {
      const long long dy = y - cut_y[s], dx = x - cut_x[s];
      cut = dy >= 0 && dy < cut_size && dx >= 0 && dx < cut_size;
    }
    if (!cut) {
      const int sy = shifts ? (int)shifts[2 * s] : 0, sx = shifts ? (int)shifts[2 * s + 1] : 0;
      const int xf = (flip && flip[s]) ? W - 1 - x : x;
      v = src[((s * C + c) * Hp + (y + r + sy)) * Wp + (xf + r + sx)];
    }
    out[i] = v;
  }
}

// ---- resized crop (the ImageNet loader's RandomResizedCrop / centre crop + flip + normalise) --------------------------
// Block (oy, b) writes output row oy of image b.  PIL's bilinear filter (= F.interpolate(antialias=True)): per output
// pixel, taps [xmin, xend) of the triangle of half-width support = max(in/out, 1), centred at scale*(i+0.5), clamped to
// the BOX and normalised by their sum.  Tap ranges are computed in double exactly as ATen computes them; the weights
// 1 - |t| step from t0 by 1/scale in fp32, so no tap table is stored and a huge box costs no extra shared memory.
// Pass 1 (vertical) filters the box's source columns [xb, xe) of all three channels into shared memory; pass 2
// (horizontal) filters those into output pixels.  A source pixel is read about twice in all (overlapping supports);
// a box wider than RC_SPAN columns is handled RC_SPAN columns' worth of output pixels at a time.
constexpr int RC_THREADS = 256;
constexpr int RC_SPAN = 2048;      // source columns per pass (3 x 2048 fp32 = 24 KB shared)

struct RcTaps {
  int lo, n;                       // taps [lo, lo + n) in box coordinates
  float t0, dt;                    // tap j sits at t = t0 + j * dt (filter argument)
};

__device__ __forceinline__ RcTaps rc_taps(int i, double scale, double support, double invscale, int in_size) {
  const double center = scale * (i + 0.5);
  long long lo = (long long)(center - support + 0.5);
  if (lo < 0) lo = 0;
  long long hi = (long long)(center + support + 0.5);
  if (hi > in_size) hi = in_size;
  RcTaps t;
  t.lo = (int)lo; t.n = (int)(hi - lo);
  t.t0 = (float)((lo - center + 0.5) * invscale); t.dt = (float)invscale;
  return t;
}

__device__ __forceinline__ float rc_weight(const RcTaps& t, int j) {
  return fmaxf(0.f, 1.f - fabsf(fmaf((float)j, t.dt, t.t0)));
}

struct RcNorm { float mean[3], std[3]; };

__global__ void __launch_bounds__(RC_THREADS) k_resized_crop(const tp_crop_entry* __restrict__ table, int S, RcNorm nrm,
                                                             float* __restrict__ out) {
  __shared__ float col[3][RC_SPAN];
  const int oy = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const tp_crop_entry e = table[b];
  float* orow = out + ((long long)b * S + oy) * S * 3;
  const double sy = (double)e.h / S, sx = (double)e.w / S;
  const double supy = sy >= 1.0 ? sy : 1.0, supx = sx >= 1.0 ? sx : 1.0;
  const bool bad = !e.src || e.h <= 0 || e.w <= 0 || e.top < 0 || e.left < 0 || e.top + e.h > e.H ||
                   e.left + e.w > e.W || 2.0 * supx + 2.0 > RC_SPAN;
  if (bad) {                       // contract violation: the row is NaN rather than a read outside the image
    for (int i = tid; i < 3 * S; i += RC_THREADS) orow[i] = __int_as_float(0x7fc00000);
    return;
  }
  const RcTaps ty = rc_taps(oy, sy, supy, sy >= 1.0 ? 1.0 / sy : 1.0, e.h);
  const long long plane = (long long)e.H * e.W;
  const unsigned char* src = (const unsigned char*)e.src + (long long)(e.top + ty.lo) * e.W + e.left;
  // output columns per chunk: their taps span at most scale*(q+1) + 1 source columns
  const int q = sx <= 1.0 ? S : min(S, max(1, (int)((RC_SPAN - 1) / sx) - 1));
  float tot_y = 0.f;
  for (int j = 0; j < ty.n; ++j) tot_y += rc_weight(ty, j);
  const float inv_tot_y = 1.f / tot_y;
  for (int ox0 = 0; ox0 < S; ox0 += q) {
    const int ox1 = min(S, ox0 + q);
    const RcTaps first = rc_taps(ox0, sx, supx, sx >= 1.0 ? 1.0 / sx : 1.0, e.w);
    const RcTaps last = rc_taps(ox1 - 1, sx, supx, sx >= 1.0 ? 1.0 / sx : 1.0, e.w);
    const int xb = first.lo, xe = last.lo + last.n;
    if (ox0 > 0) __syncthreads();  // the previous chunk's pass 2 is done reading col[]
    for (int x = xb + tid; x < xe; x += RC_THREADS) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      const unsigned char* p = src + x;
      for (int j = 0; j < ty.n; ++j, p += e.W) {
        const float w = rc_weight(ty, j);
        a0 = fmaf(w, (float)__ldg(p), a0);
        a1 = fmaf(w, (float)__ldg(p + plane), a1);
        a2 = fmaf(w, (float)__ldg(p + 2 * plane), a2);
      }
      col[0][x - xb] = a0 * inv_tot_y; col[1][x - xb] = a1 * inv_tot_y; col[2][x - xb] = a2 * inv_tot_y;
    }
    __syncthreads();
    for (int ox = ox0 + tid; ox < ox1; ox += RC_THREADS) {
      const RcTaps tx = rc_taps(ox, sx, supx, sx >= 1.0 ? 1.0 / sx : 1.0, e.w);
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, tot = 0.f;
      for (int j = 0; j < tx.n; ++j) {
        const float w = rc_weight(tx, j);
        const int c = tx.lo - xb + j;
        tot += w;
        a0 = fmaf(w, col[0][c], a0); a1 = fmaf(w, col[1][c], a1); a2 = fmaf(w, col[2][c], a2);
      }
      float* o = orow + 3 * (e.flip ? S - 1 - ox : ox);
      o[0] = (a0 / tot - nrm.mean[0]) / nrm.std[0];
      o[1] = (a1 / tot - nrm.mean[1]) / nrm.std[1];
      o[2] = (a2 / tot - nrm.mean[2]) / nrm.std[2];
    }
  }
}

// ---- Philox4x32-10 (Salmon et al., SC'11): counter (ctr, 0, 0, 0) with key (seed_lo, seed_hi) --------------------------
__device__ __forceinline__ void philox4x32_10(unsigned long long ctr, unsigned long long seed, unsigned int (&o)[4]) {
  unsigned int c0 = (unsigned int)ctr, c1 = (unsigned int)(ctr >> 32), c2 = 0u, c3 = 0u;
  unsigned int k0 = (unsigned int)seed, k1 = (unsigned int)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const unsigned int hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const unsigned int hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const unsigned int n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  o[0] = c0; o[1] = c1; o[2] = c2; o[3] = c3;
}

// mode 0: raw 32-bit words (tests pin the stream against the oracle bit for bit); mode 1: N(0,1) by Box-Muller
__global__ void __launch_bounds__(256) k_synth_normal(float* __restrict__ out, long long n, unsigned long long seed,
                                                      unsigned long long offset, int mode) {
  const long long n4 = (n + 3) >> 2;
  for (long long q = blockIdx.x * 256ll + threadIdx.x; q < n4; q += (long long)gridDim.x * 256) {
    unsigned int u[4];
    philox4x32_10(offset + (unsigned long long)q, seed, u);
    float f[4];
    if (mode == 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j) f[j] = __uint_as_float(u[j]);
    } else {
      // (0, 1] uniforms from the top 24 bits; two Box-Muller pairs
      const float inv = 1.0f / 16777216.0f;
#pragma unroll
      for (int j = 0; j < 4; j += 2) {
        const float u1 = ((float)(u[j] >> 8) + 1.0f) * inv, u2 = (float)(u[j + 1] >> 8) * inv;
        const float rad = sqrtf(-2.0f * logf(u1));
        float sn, cs; sincospif(2.0f * u2, &sn, &cs);
        f[j] = rad * cs; f[j + 1] = rad * sn;
      }
    }
    if (4 * q + 3 < n && (((uintptr_t)out) & 15) == 0) {
      st_stream((float4*)out + q, make_float4(f[0], f[1], f[2], f[3]));
    } else {
      for (int j = 0; j < 4; ++j) if (4 * q + j < n) out[4 * q + j] = f[j];
    }
  }
}

__global__ void __launch_bounds__(256) k_synth_labels(long long* __restrict__ out, long long n, int num_classes,
                                                      unsigned long long seed, unsigned long long offset) {
  const long long n4 = (n + 3) >> 2;
  for (long long q = blockIdx.x * 256ll + threadIdx.x; q < n4; q += (long long)gridDim.x * 256) {
    unsigned int u[4];
    philox4x32_10(offset + (unsigned long long)q, seed, u);
    for (int j = 0; j < 4; ++j)
      if (4 * q + j < n) out[4 * q + j] = (long long)(((unsigned long long)u[j] * (unsigned long long)num_classes) >> 32);
  }
}

}  // namespace tp

using namespace tp;

extern "C" {

int tp_cifar_augment(const void* src, void* out, const int64_t* idx, const int64_t* shifts, const uint8_t* flip,
                     const int64_t* cut_y, const int64_t* cut_x, int cut_size,
                     int n, int c, int h, int w, int r, void* stream) {
  if (!src || !out || n <= 0 || c <= 0 || h <= 0 || w <= 0 || r < 0) return TP_ERR_INVALID;
  if ((cut_y == nullptr) != (cut_x == nullptr) || (cut_y && cut_size <= 0)) return TP_ERR_INVALID;
  if (shifts && r == 0) return TP_ERR_INVALID;
  const long long total = (long long)n * c * h * w;
  const long long g = (total + 255) / 256, gm = (long long)sm_count() * 16;
  k_cifar_augment<<<(unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream>>>(
      (const float*)src, (float*)out, (const long long*)idx, (const long long*)shifts, (const unsigned char*)flip,
      (const long long*)cut_y, (const long long*)cut_x, cut_size, n, c, h, w, r);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_resized_crop(const tp_crop_entry* table, int n, int size, const float* mean255, const float* std255, void* out,
                    void* stream) {
  if (!table || !out || n <= 0 || n > 65535 || size <= 0 || size > RC_SPAN) return TP_ERR_INVALID;
  RcNorm nrm;
  for (int c = 0; c < 3; ++c) {
    nrm.mean[c] = mean255 ? mean255[c] : 0.f;
    nrm.std[c] = std255 ? std255[c] : 1.f;
  }
  k_resized_crop<<<dim3((unsigned)size, (unsigned)n), RC_THREADS, 0, (cudaStream_t)stream>>>(table, size, nrm, (float*)out);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_synth_normal(void* out, int64_t numel, uint64_t seed, uint64_t counter_offset, int raw_words, void* stream) {
  if (!out || numel < 0) return TP_ERR_INVALID;
  if (numel == 0) return TP_OK;
  const long long g = ((numel + 3) / 4 + 255) / 256, gm = (long long)sm_count() * 16;
  k_synth_normal<<<(unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream>>>((float*)out, numel, seed, counter_offset, raw_words ? 0 : 1);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_synth_labels(void* out, int64_t numel, int num_classes, uint64_t seed, uint64_t counter_offset, void* stream) {
  if (!out || numel < 0 || num_classes <= 0) return TP_ERR_INVALID;
  if (numel == 0) return TP_OK;
  const long long g = ((numel + 3) / 4 + 255) / 256, gm = (long long)sm_count() * 8;
  k_synth_labels<<<(unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream>>>((long long*)out, numel, num_classes, seed, counter_offset);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // extern "C"
