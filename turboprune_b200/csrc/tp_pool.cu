// Max pooling (forward with saved arg-max, backward) for NHWC bf16 activations, sm_90a.
// The torchvision stem's MaxPool2d(3, 2, 1) sits between the first masked conv block and layer1
// (SURVEY.md §8(f) row 1: unmasked neighbours of the masked convs); these kernels replace ATen's NHWC max pooling.
//   forward : one thread per (output pixel, 8 channels): 16-byte loads over the window, -inf padding,
//             NaN propagates (torch semantics), first maximum wins; writes y and a uint8 window index
//   backward: gather form (no atomics, deterministic): one thread per (input pixel, 8 channels) sums dy
//             of the <= ceil(k/s)^2 windows whose arg-max is this pixel
#include "tp_common.cuh"

namespace tp {

__device__ __forceinline__ void unpack8p(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}

__global__ void __launch_bounds__(256) k_maxpool_fwd(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                     unsigned char* __restrict__ idx, int n, int h, int w, int c,
                                                     int k, int stride, int pad, int p, int q) {
  pdl_enter();
  const int cv = c >> 3;
  const long long total = (long long)n * p * q * cv;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % cv); long long t = i / cv;
    const int qi = (int)(t % q); t /= q;
    const int pi = (int)(t % p); const int ni = (int)(t / p);
    // window clipped to the image; the first in-bounds tap seeds the arg-max (ATen: `if (val > max || isnan(val))`)
    const int h0 = pi * stride - pad, w0 = qi * stride - pad;
    const int r0 = h0 < 0 ? -h0 : 0, s0 = w0 < 0 ? -w0 : 0;
    const int r1 = (h0 + k > h) ? h - h0 : k, s1 = (w0 + k > w) ? w - w0 : k;
    float best[8]; unsigned char bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; bi[j] = (unsigned char)(r0 * k + s0); }
    const __nv_bfloat16* xb = x + ((long long)ni * h * w) * c + ci * 8;
    for (int r = r0; r < r1; ++r) {
      const __nv_bfloat16* xr = xb + ((long long)(h0 + r) * w + w0) * c;
      for (int s = s0; s < s1; ++s) {
        float f[8];
        unpack8p(*reinterpret_cast<const uint4*>(xr + (long long)s * c), f);
        const unsigned char id = (unsigned char)(r * k + s);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (f[j] > best[j] || f[j] != f[j]) { best[j] = f[j]; bi[j] = id; }
      }
    }
    uint4 o; __nv_bfloat162* ho = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ho[j] = __floats2bfloat162_rn(best[2 * j], best[2 * j + 1]);
    const long long ob = (((long long)ni * p + pi) * q + qi) * c + ci * 8;
    *reinterpret_cast<uint4*>(y + ob) = o;
    uint2 ib;
    ib.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | ((unsigned)bi[3] << 24);
    ib.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | ((unsigned)bi[7] << 24);
    *reinterpret_cast<uint2*>(idx + ob) = ib;
  }
}

__global__ void __launch_bounds__(256) k_maxpool_bwd(const __nv_bfloat16* __restrict__ dy, const unsigned char* __restrict__ idx,
                                                     __nv_bfloat16* __restrict__ dx, int n, int h, int w, int c,
                                                     int k, int stride, int pad, int p, int q) {
  pdl_enter();
  const int cv = c >> 3;
  const long long total = (long long)n * h * w * cv;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % cv); long long t = i / cv;
    const int wi = (int)(t % w); t /= w;
    const int hi = (int)(t % h); const int ni = (int)(t / h);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // output rows whose window covers input row hi: pi*stride - pad <= hi <= pi*stride - pad + k - 1
    int p0 = hi + pad - (k - 1); p0 = p0 <= 0 ? 0 : (p0 + stride - 1) / stride;
    int p1 = (hi + pad) / stride; if (p1 > p - 1) p1 = p - 1;
    int q0 = wi + pad - (k - 1); q0 = q0 <= 0 ? 0 : (q0 + stride - 1) / stride;
    int q1 = (wi + pad) / stride; if (q1 > q - 1) q1 = q - 1;
    for (int pi = p0; pi <= p1; ++pi) {
      const int r = hi + pad - pi * stride;
      for (int qi = q0; qi <= q1; ++qi) {
        const int s = wi + pad - qi * stride;
        const unsigned char me = (unsigned char)(r * k + s);
        const long long ob = (((long long)ni * p + pi) * q + qi) * c + ci * 8;
        const uint2 ib = *reinterpret_cast<const uint2*>(idx + ob);
        float g[8];
        unpack8p(*reinterpret_cast<const uint4*>(dy + ob), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const unsigned char b = (unsigned char)(((j < 4 ? ib.x : ib.y) >> (8 * (j & 3))) & 0xff);
          if (b == me) acc[j] += g[j];
        }
      }
    }
    uint4 o; __nv_bfloat162* ho = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ho[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
    *reinterpret_cast<uint4*>(dx + (((long long)ni * h + hi) * w + wi) * c + ci * 8) = o;
  }
}

// ---- MaxPool2d(3, 2, 1) — the torchvision ResNet stem — with the geometry known at compile time: every tap is a predicated
// 16-byte load issued before the first compare (the generic kernels walk runtime-bounded loops).  Same tap order, same
// arg-max rule, same rounding.
__global__ void __launch_bounds__(256) k_maxpool_fwd_321(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                         unsigned char* __restrict__ idx, int n, int h, int w, int c, int p, int q) {
  pdl_enter();
  const int cv = c >> 3;
  const long long total = (long long)n * p * q * cv;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % cv); long long t = i / cv;
    const int qi = (int)(t % q); t /= q;
    const int pi = (int)(t % p); const int ni = (int)(t / p);
    const int h0 = pi * 2 - 1, w0 = qi * 2 - 1;
    const __nv_bfloat16* xb = x + ((long long)ni * h * w) * c + ci * 8;
    uint4 v[9]; bool ok[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s_ = 0; s_ < 3; ++s_) {
        const int hh = h0 + r, ww = w0 + s_;
        ok[r * 3 + s_] = hh >= 0 && hh < h && ww >= 0 && ww < w;
        v[r * 3 + s_] = make_uint4(0u, 0u, 0u, 0u);
        if (ok[r * 3 + s_]) v[r * 3 + s_] = *reinterpret_cast<const uint4*>(xb + ((long long)hh * w + ww) * c);
      }
    const int r0 = h0 < 0 ? 1 : 0, s0 = w0 < 0 ? 1 : 0;          // first in-bounds tap seeds the arg-max
    float best[8]; unsigned char bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; bi[j] = (unsigned char)(r0 * 3 + s0); }
#pragma unroll
    for (int tp_ = 0; tp_ < 9; ++tp_) {
      if (!ok[tp_]) continue;
      float f[8]; unpack8p(v[tp_], f);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (f[j] > best[j] || f[j] != f[j]) { best[j] = f[j]; bi[j] = (unsigned char)tp_; }
    }
    uint4 o; __nv_bfloat162* ho = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ho[j] = __floats2bfloat162_rn(best[2 * j], best[2 * j + 1]);
    const long long ob = (((long long)ni * p + pi) * q + qi) * c + ci * 8;
    *reinterpret_cast<uint4*>(y + ob) = o;
    uint2 ib;
    ib.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | ((unsigned)bi[3] << 24);
    ib.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | ((unsigned)bi[7] << 24);
    *reinterpret_cast<uint2*>(idx + ob) = ib;
  }
}

__global__ void __launch_bounds__(256) k_maxpool_bwd_321(const __nv_bfloat16* __restrict__ dy, const unsigned char* __restrict__ idx,
                                                         __nv_bfloat16* __restrict__ dx, int n, int h, int w, int c, int p, int q) {
  pdl_enter();
  const int cv = c >> 3;
  const long long total = (long long)n * h * w * cv;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ci = (int)(i % cv); long long t = i / cv;
    const int wi = (int)(t % w); t /= w;
    const int hi = (int)(t % h); const int ni = (int)(t / h);
    // windows covering (hi, wi): pi in {(hi+1)/2 - 1 [only when hi+1-2*pi <= 2], (hi+1)/2}; at most 2 x 2, in (pi, qi) order
    const int pa = (hi + 1) >> 1, qa = (wi + 1) >> 1;
    int pis[2] = {pa - 1, pa}, qis[2] = {qa - 1, qa};
    uint4 g4[4]; uint2 i4[4]; bool ok[4]; unsigned char me[4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int pi = pis[a], qi = qis[b];
        const int r = hi + 1 - pi * 2, s_ = wi + 1 - qi * 2;
        const int e = a * 2 + b;
        ok[e] = pi >= 0 && pi < p && qi >= 0 && qi < q && r >= 0 && r < 3 && s_ >= 0 && s_ < 3;
        me[e] = (unsigned char)(r * 3 + s_);
        g4[e] = make_uint4(0u, 0u, 0u, 0u); i4[e] = make_uint2(0xffffffffu, 0xffffffffu);
        if (ok[e]) {
          const long long ob = (((long long)ni * p + pi) * q + qi) * c + ci * 8;
          i4[e] = *reinterpret_cast<const uint2*>(idx + ob);
          g4[e] = *reinterpret_cast<const uint4*>(dy + ob);
        }
      }
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (!ok[e]) continue;
      float g[8]; unpack8p(g4[e], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const unsigned char bsel = (unsigned char)(((j < 4 ? i4[e].x : i4[e].y) >> (8 * (j & 3))) & 0xff);
        if (bsel == me[e]) acc[j] += g[j];
      }
    }
    uint4 o; __nv_bfloat162* ho = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ho[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
    *reinterpret_cast<uint4*>(dx + (((long long)ni * h + hi) * w + wi) * c + ci * 8) = o;
  }
}

}  // namespace tp

using namespace tp;

extern "C" {

int tp_maxpool_forward(const void* x, void* y, void* idx, int n, int h, int w, int c, int k, int stride, int pad,
                       int p, int q, void* stream) {
  if (!x || !y || !idx || n <= 0 || c % 8 != 0 || k <= 0 || k * k > 255 || stride <= 0) return TP_ERR_INVALID;
  int rc = bind_device_of(x); if (rc) return rc;
  const long long total = (long long)n * p * q * (c / 8);
  long long g = (total + 255) / 256, gm = (long long)sm_count() * 16;
  if (k == 3 && stride == 2 && pad == 1)
    launch(k_maxpool_fwd_321, (unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, (__nv_bfloat16*)y,
        (unsigned char*)idx, n, h, w, c, p, q);
  else
    launch(k_maxpool_fwd, (unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, (__nv_bfloat16*)y,
        (unsigned char*)idx, n, h, w, c, k, stride, pad, p, q);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_maxpool_backward(const void* dy, const void* idx, void* dx, int n, int h, int w, int c, int k, int stride, int pad,
                        int p, int q, void* stream) {
  if (!dy || !dx || !idx || n <= 0 || c % 8 != 0 || k <= 0 || stride <= 0) return TP_ERR_INVALID;
  int rc = bind_device_of(dy); if (rc) return rc;
  const long long total = (long long)n * h * w * (c / 8);
  long long g = (total + 255) / 256, gm = (long long)sm_count() * 16;
  if (k == 3 && stride == 2 && pad == 1)
    launch(k_maxpool_bwd_321, (unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)dy, (const unsigned char*)idx,
        (__nv_bfloat16*)dx, n, h, w, c, p, q);
  else
    launch(k_maxpool_bwd, (unsigned)(g < gm ? g : gm), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)dy, (const unsigned char*)idx,
        (__nv_bfloat16*)dx, n, h, w, c, k, stride, pad, p, q);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // extern "C"
