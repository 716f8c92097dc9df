// Pruning score -> exact global k-th smallest -> mask, for sm_90a.
//
// Replaces utils/pruning_utils.py:73-87 / :186-203 / :263-283 of the reference
// (per-layer score temporaries, torch.cat, single-CTA 16-pass torch.kthvalue, per-layer
// torch.where) with ONE kernel of resident CTAs (k_topk_fused) whose phases are separated by grid-wide barriers:
//
//   P0 sample   : 2^20 strided samples (runs of 16 neighbours), kept in shared memory; 2048-bin histogram of key
//                 bits [30:20], shared-memory privatised
//   P1 refine   : every CTA locates the coarse bins of the two bracket ranks (sample quantile +- 5 sigma of its
//                 rank error) and histograms bits [19:9] of its own samples inside them
//   P2 sweep    : bracket [lo, hi) from the fine histograms, then ONE pass over (w, m[, g]) at HBM rate: counts keys
//                 < lo and == lo, writes the final mask for every key outside (lo, hi) and appends the few keys
//                 inside to a candidate list                                   (12 B/elem mag, 16 snip / synflow)
//   P3 digit    : all CTAs histogram the top radix digit of the candidates (data in L2)
//   P4 narrow   : every CTA picks the digit, the candidates that match it (a few dozen) go to a second list
//   P5 finish   : every CTA selects the exact key among those in shared memory (no further barrier), patches its
//                 share of the candidates' masks; CTA 0 publishes threshold and status.
//
// If the bracket misses (adversarial ties, overflow of a list) the status says so and the host
// runs an exact 3-pass 11/11/10-bit radix select over the full data + one apply pass — tp_topk_finish, which is
// also where the status is read back, so the fast path itself never blocks the stream.
// Both paths are bit-exact with torch.kthvalue + torch.where(score <= thr, 0, 1).
//
// Keys: scores are |.| of fp32 products, so their IEEE bit patterns order like unsigned
// integers; NaN patterns (> 0x7f800000) sort above +inf exactly like ATen's radix key
// (SortingRadixSelect.cuh:20-39).
#include "tp_common.cuh"
#include <vector>

namespace tp {

struct SelState {
  unsigned long long k;
  unsigned long long n_lt, n_eq, n_cand;
  unsigned int lo, hi;           // bracket: lo inclusive lower edge, hi exclusive upper edge
  unsigned int thr_key;
  int status;                    // 0 ok, 1 bracket missed -> fallback, 2 ok but threshold is NaN
  unsigned int prefix, prefix_mask;   // exact radix path
  unsigned int c_lo, c_hi;            // coarse sample bins of the two bracket ranks
  unsigned long long before_lo, before_hi;
  unsigned long long k_rem;
  unsigned long long n_cand2;         // second-level list (candidates matching the top digit)
  unsigned int barrier; unsigned int pad_;   // arrival counter of the grid barrier
  unsigned long long t_phase[8];      // %globaltimer (ns) when CTA 0 entered P0..P5 and left (tools/topk_bench.py prints the deltas)
};

constexpr int kSampleBits = 20;
constexpr int kSweepThreads = 256;
constexpr int kSmemCand = 2048;       // candidate staging per CTA (16 KB: the sample-key array, dead by then)

template <int KIND>
__device__ __forceinline__ unsigned int score_key(float w, float g, float m) {
  float s;
  if (KIND == TP_SCORE_MAG) s = m * w;                 // pruning_utils.py:75
  else if (KIND == TP_SCORE_SNIP) s = (g * w) * m;     // pruning_utils.py:190
  else s = (m * g) * w;                                // pruning_utils.py:267
  return __float_as_uint(fabsf(s));
}

template <int KIND>
__device__ __forceinline__ unsigned int seg_key(const Seg& sg, long long i) {
  float w = sg.w[i], m = sg.m[i];
  float g = (KIND == TP_SCORE_MAG) ? 0.f : sg.g[i];
  return score_key<KIND>(w, g, m);
}

// ---------------------------------------------------------------------------------------------
// Block-wide rank search in a histogram of blockDim.x * PER bins: smallest bin whose inclusive
// cumulative count reaches `rank` (1-indexed).  All threads call; result through shared memory.
template <int PER>
__device__ __forceinline__ void block_find_rank(const unsigned int* __restrict__ hist, unsigned long long rank,
                                                unsigned int* s_bin, unsigned long long* s_before,
                                                unsigned long long* s_warp /* [32] */) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nwarps = blockDim.x >> 5;
  unsigned int h[PER];
  unsigned long long loc = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) { h[i] = hist[t * PER + i]; loc += h[i]; }
  unsigned long long inc = loc;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    unsigned long long v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  __syncthreads();                       // s_warp may still be read from a previous call
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    unsigned long long v = lane < nwarps ? s_warp[lane] : 0ull, x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += u;
    }
    s_warp[lane] = x - v;                // exclusive prefix of the warp totals
  }
  __syncthreads();
  const unsigned long long before = s_warp[warp] + inc - loc;
  if (rank > before && rank <= before + loc) {
    unsigned long long c = before;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      if (c + h[i] >= rank) { *s_bin = (unsigned int)(t * PER + i); *s_before = c; break; }
      c += h[i];
    }
  }
  __syncthreads();
}

constexpr int kCoarseShift = 20, kFineShift = 9, kDigitBins = 2048;

__device__ __forceinline__ int resolve_shift0(unsigned int lo, unsigned int hi) {
  const unsigned int span = lo ^ (hi - 1u);
  const int top = span ? (31 - __clz(span)) : 0;
  return (top / 11) * 11;
}

// ---------------------------------------------------------------------------------------------
struct SweepCtx {
  unsigned int lo, hi;
  unsigned int n_lt, n_eq;
  uint2* s_cand; unsigned int* s_ncand;
  unsigned int* s_dig; int shift0;
  SelState* st; uint2* cand; unsigned int cap;
};

__device__ __forceinline__ float classify(SweepCtx& c, unsigned int key, long long gidx) {
  if (key < c.lo) { c.n_lt++; return 0.f; }
  if (key == c.lo) { c.n_eq++; return 0.f; }
  if (key >= c.hi) return 1.f;
  // inside the bracket: rare (~0.1-1 %) -> candidate list, and its top radix digit is counted right away
  atomicAdd(&c.s_dig[(key >> c.shift0) & (kDigitBins - 1)], 1u);
  unsigned int slot = atomicAdd(c.s_ncand, 1u);
  if (slot < kSmemCand) {
    c.s_cand[slot] = make_uint2(key, (unsigned int)gidx);
  } else {
    unsigned long long gs = atomicAdd(&c.st->n_cand, 1ull);
    if (gs < c.cap) c.cand[gs] = make_uint2(key, (unsigned int)gidx);
  }
  return 0.f;   // provisional; the last phase of the kernel patches it
}

constexpr int kRun = 16;               // neighbouring elements per sample run
constexpr int kLocalKeys = 4096;      // sample keys one CTA keeps in shared memory between P0 and P1 (one round of 256 runs)
constexpr int kCand2 = 4096;          // capacity of the second-level list
constexpr int kSmemSegs = 128;        // segment tables up to this size are searched in shared memory

struct TopkArgs {
  const Seg* segs; int n_seg;
  long long tiles, N, S, k, r_lo, r_hi;
  SelState* st;
  unsigned int* hist;                 // [0,2048) coarse, [2048,6144) two fine, [6144,8192) candidate digit
  uint2* cand; unsigned int cap;
  unsigned int* cand2;                // keys of the second-level list
  float* thr_out;
};

// Grid-wide barrier for a grid that is fully resident (<= occupancy x SMs CTAs, checked on the host): one monotonically
// increasing arrival counter (zeroed with the rest of the state before the launch), release on arrive, acquire on the spin.
// A plain launch + this barrier costs less than a cooperative launch + cooperative_groups' grid.sync() per phase.
struct GridBarrier {
  unsigned int* ctr; unsigned int target;
  __device__ __forceinline__ void sync() {
    __syncthreads();
    if (threadIdx.x == 0) {
      target += gridDim.x;
      __threadfence();
      atomicAdd(ctr, 1u);
      unsigned int v;
      do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < target);
    }
    __syncthreads();
  }
};

__device__ __forceinline__ void stamp(SelState* st, int i) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    st->t_phase[i] = t;
  }
}

template <int KIND, bool WRITE>
__global__ void __launch_bounds__(kSweepThreads) k_topk_fused(const TopkArgs a) {
  __shared__ __align__(16) unsigned int s_keys[kLocalKeys];          // P0/P1: this CTA's sample keys; P2: candidate staging; P5: the second-level list
  __shared__ unsigned int s_h[2 * kDigitBins];          // histograms (coarse, then the two fine ones, then the candidates' top digit, then select digits)
  __shared__ __align__(16) Seg s_seg[kSmemSegs];        // the segment table (evicted from L2 by whatever ran before: every binary-search
                                                        // step of every thread was a DRAM round trip when it was read from global)
  uint2* const s_cand = reinterpret_cast<uint2*>(s_keys);             // kSmemCand * 8 B <= sizeof(s_keys); the sample keys are dead by P2
  __shared__ unsigned int s_ncand, s_flush[2];
  __shared__ unsigned long long s_base;
  __shared__ unsigned int s_red[2][kSweepThreads / 32];
  __shared__ unsigned int s_bin[2];
  __shared__ unsigned long long s_before[2], s_warp[32];
  const int t = threadIdx.x;
  SelState* st = a.st;
  unsigned int* hist_c = a.hist;
  unsigned int* hist_f = a.hist + kDigitBins;
  unsigned int* hist_r = a.hist + 3 * kDigitBins;

  // ---------------- P0: strided sample in runs of kRun = 16 neighbouring elements (one 64-byte burst per operand serves
  // 16 samples), keys stay in shared memory; coarse histogram of key bits [30:20] ----------------
  stamp(st, 0);
  GridBarrier grid; grid.ctr = &st->barrier; grid.target = 0;
  const bool seg_smem = a.n_seg <= kSmemSegs;
  if (seg_smem)
    for (int i = t; i < a.n_seg * (int)(sizeof(Seg) / 16); i += kSweepThreads)
      reinterpret_cast<uint4*>(s_seg)[i] = reinterpret_cast<const uint4*>(a.segs)[i];
  const Seg* const segs = seg_smem ? s_seg : a.segs;
  for (int i = t; i < kDigitBins; i += kSweepThreads) s_h[i] = 0;
  __syncthreads();
  // samples are taken in runs of kRun = 16 neighbouring elements: one 64-byte DRAM burst per operand serves 16 samples.
  // (Runs of 4 — one 32-byte sector — turn sampling into a random-access rate problem rather than a bandwidth one; the
  // host widens the rank band for the clustering.)
  const long long G = (a.S + kRun - 1) / kRun;
  const long long first = blockIdx.x * (long long)kSweepThreads, gstride = (long long)gridDim.x * kSweepThreads;
  const int rounds = first < G ? (int)((G - first + gstride - 1) / gstride) : 0;   // uniform over the CTA; host keeps rounds * 256 * kRun <= kLocalKeys
  for (int r = 0; r < rounds; ++r) {
    const long long gi = first + t + r * gstride;
    unsigned int key[kRun];
#pragma unroll
    for (int u = 0; u < kRun; ++u) key[u] = 0xFFFFFFFFu;                             // "no sample" (runs past S)
    if (gi < G) {
      long long e = (long long)(((unsigned long long)gi * (unsigned long long)a.N) / (unsigned long long)G);
      const int si = find_seg_by_elem(segs, a.n_seg, e);
      const Seg& sg = segs[si];
      long long l0 = (e - sg.start) & ~(long long)(kRun - 1);
      if (l0 + kRun > sg.n) l0 = sg.n >= kRun ? ((sg.n - kRun) & ~3ll) : 0;
      const long long nvalid = min((long long)kRun, min(sg.n - l0, a.S - gi * kRun));
      if (nvalid == kRun && (((uintptr_t)(sg.w + l0) | (uintptr_t)(sg.m + l0) | (KIND == TP_SCORE_MAG ? 0 : (uintptr_t)(sg.g + l0))) & 15) == 0) {
        float4 wv[kRun / 4], mv[kRun / 4], gv[kRun / 4];
#pragma unroll
        for (int q = 0; q < kRun / 4; ++q) {                                          // all loads in flight before the first use
          wv[q] = ld_stream((const float4*)(sg.w + l0) + q);
          mv[q] = ld_stream((const float4*)(sg.m + l0) + q);
          gv[q] = (KIND == TP_SCORE_MAG) ? make_float4(0.f, 0.f, 0.f, 0.f) : ld_stream((const float4*)(sg.g + l0) + q);
        }
#pragma unroll
        for (int q = 0; q < kRun / 4; ++q) {
          key[4 * q + 0] = score_key<KIND>(wv[q].x, gv[q].x, mv[q].x); key[4 * q + 1] = score_key<KIND>(wv[q].y, gv[q].y, mv[q].y);
          key[4 * q + 2] = score_key<KIND>(wv[q].z, gv[q].z, mv[q].z); key[4 * q + 3] = score_key<KIND>(wv[q].w, gv[q].w, mv[q].w);
        }
      } else {
#pragma unroll
        for (int u = 0; u < kRun; ++u) if (u < nvalid) key[u] = seg_key<KIND>(sg, l0 + u);
      }
#pragma unroll
      for (int u = 0; u < kRun; ++u) if (key[u] != 0xFFFFFFFFu) atomicAdd(&s_h[key[u] >> kCoarseShift], 1u);
    }
#pragma unroll
    for (int q = 0; q < kRun / 4; ++q)
      *reinterpret_cast<uint4*>(&s_keys[((r * kSweepThreads + t) * kRun) + 4 * q]) = make_uint4(key[4 * q], key[4 * q + 1], key[4 * q + 2], key[4 * q + 3]);
  }
  __syncthreads();
  // (No L2 prefetch of this CTA's first sweep tiles here: the histogram atomics and the grid barrier would queue behind
  // the prefetch traffic.)
  for (int i = t; i < kDigitBins; i += kSweepThreads) if (s_h[i]) atomicAdd(&hist_c[i], s_h[i]);
  grid.sync();
  stamp(st, 1);

  // ---------------- P1: coarse bins of the two bracket ranks (every CTA, 8 KB of L2 reads), fine histograms of the
  // own samples that fall inside them ----------------
  if (t < 2) { s_bin[t] = 0; s_before[t] = 0; }
  for (int i = t; i < 2 * kDigitBins; i += kSweepThreads) s_h[i] = 0;
  __syncthreads();
  block_find_rank<kDigitBins / kSweepThreads>(hist_c, (unsigned long long)(a.r_lo < 1 ? 1 : a.r_lo), &s_bin[0], &s_before[0], s_warp);
  block_find_rank<kDigitBins / kSweepThreads>(hist_c, (unsigned long long)(a.r_hi > a.S ? a.S : a.r_hi), &s_bin[1], &s_before[1], s_warp);
  const unsigned int c_lo = s_bin[0], c_hi = s_bin[1];
  const unsigned long long before_lo = s_before[0], before_hi = s_before[1];
  if (blockIdx.x == 0 && t == 0) { st->c_lo = c_lo; st->c_hi = c_hi; st->before_lo = before_lo; st->before_hi = before_hi; }
  for (int i = t; i < rounds * kSweepThreads * kRun; i += kSweepThreads) {
    const unsigned int key = s_keys[i];
    if (key == 0xFFFFFFFFu) continue;
    const unsigned int c = key >> kCoarseShift, f = (key >> kFineShift) & (kDigitBins - 1);
    if (c == c_lo) atomicAdd(&s_h[f], 1u);
    if (c == c_hi) atomicAdd(&s_h[kDigitBins + f], 1u);
  }
  __syncthreads();
  for (int i = t; i < 2 * kDigitBins; i += kSweepThreads) if (s_h[i]) atomicAdd(&hist_f[i], s_h[i]);
  grid.sync();
  stamp(st, 2);

  // ---------------- P2: bracket [lo, hi) from the fine histograms — every CTA derives the same two keys — and the
  // sweep ----------------
  if (t < 2) { s_bin[t] = 0; s_before[t] = 0; }
  __syncthreads();
  block_find_rank<kDigitBins / kSweepThreads>(hist_f, (unsigned long long)(a.r_lo < 1 ? 1 : a.r_lo) - before_lo,
                                              &s_bin[0], &s_before[0], s_warp);
  block_find_rank<kDigitBins / kSweepThreads>(hist_f + kDigitBins, (unsigned long long)(a.r_hi > a.S ? a.S : a.r_hi) - before_hi,
                                              &s_bin[1], &s_before[1], s_warp);
  unsigned int lo = (c_lo << kCoarseShift) | (s_bin[0] << kFineShift);
  unsigned int hi = (((c_hi << 11) | s_bin[1]) + 1u) << kFineShift;
  if (a.r_lo < 1) lo = 0u;                              // no lower bound
  if (a.r_hi > a.S || hi > 0x80000000u || hi == 0u) hi = 0x80000000u;   // no upper bound (keys are <= 0x7fffffff)
  if (blockIdx.x == 0 && t == 0) { st->lo = lo; st->hi = hi; }
  SweepCtx c;
  c.lo = lo; c.hi = hi; c.n_lt = 0; c.n_eq = 0;
  c.s_cand = s_cand; c.s_ncand = &s_ncand; c.st = st; c.cand = a.cand; c.cap = a.cap;
  const int shift0 = resolve_shift0(lo, hi);
  c.s_dig = s_h; c.shift0 = shift0;                     // top radix digit of every candidate, counted while sweeping
  for (int i = t; i < kDigitBins; i += kSweepThreads) s_h[i] = 0;
  __syncthreads();
  constexpr int kVecIters = kTileElems / (kSweepThreads * 4);   // 4
  // Candidates collect in shared memory ACROSS tiles and go out once per CTA (a CTA sees a few hundred of them in total);
  // the staging is emptied early only when it is half full.  The first version reserved the global slots after every tile:
  // one global atomic round trip with the whole CTA waiting behind it, and three barriers, per 48 KB of data.
  auto flush_cands = [&]() {                               // uniform over the CTA; caller has synchronised
    const unsigned int nc = s_ncand < (unsigned)kSmemCand ? s_ncand : (unsigned)kSmemCand;   // slots past the staging went to global directly
    if (nc) {
      if (t == 0) s_base = atomicAdd(&st->n_cand, (unsigned long long)nc);
      __syncthreads();
      const unsigned long long b = s_base;
      for (unsigned int i = t; i < nc; i += kSweepThreads)
        if (b + i < a.cap) a.cand[b + i] = s_cand[i];
    }
    __syncthreads();
    if (t == 0) s_ncand = 0;
    __syncthreads();
  };
  if (t == 0) s_ncand = 0;
  __syncthreads();
  int sweep_it = 0;
  for (long long tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int si = find_seg(segs, a.n_seg, tile);
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    const float* wp = sg.w + base;
    const float* mp = sg.m + base;
    const float* gp = (KIND == TP_SCORE_MAG) ? nullptr : sg.g + base;
    float* op = WRITE ? sg.mo + base : nullptr;
    const long long g0 = sg.start + base;
    bool vec = n_in == kTileElems &&
               ((((uintptr_t)wp) | ((uintptr_t)mp) | ((uintptr_t)gp) | ((uintptr_t)op)) & 15) == 0;
    if (vec) {
      float4 wv[kVecIters], mv[kVecIters], gv[kVecIters];
#pragma unroll
      for (int it = 0; it < kVecIters; ++it) {
        int q = it * kSweepThreads + t;
        wv[it] = ld_stream((const float4*)wp + q);
        mv[it] = ld_stream((const float4*)mp + q);
        if (KIND != TP_SCORE_MAG) gv[it] = ld_stream((const float4*)gp + q);
        else gv[it] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int it = 0; it < kVecIters; ++it) {
        int q = it * kSweepThreads + t;
        long long gi = g0 + (long long)q * 4;
        float4 o;
        o.x = classify(c, score_key<KIND>(wv[it].x, gv[it].x, mv[it].x), gi + 0);
        o.y = classify(c, score_key<KIND>(wv[it].y, gv[it].y, mv[it].y), gi + 1);
        o.z = classify(c, score_key<KIND>(wv[it].z, gv[it].z, mv[it].z), gi + 2);
        o.w = classify(c, score_key<KIND>(wv[it].w, gv[it].w, mv[it].w), gi + 3);
        if (WRITE) st_stream((float4*)op + q, o);
      }
    } else {
      for (int i = t; i < n_in; i += kSweepThreads) {
        float g = (KIND == TP_SCORE_MAG) ? 0.f : gp[i];
        float o = classify(c, score_key<KIND>(wp[i], g, mp[i]), g0 + i);
        if (WRITE) op[i] = o;
      }
    }
    // the early-flush decision must be the same in every thread: thread 0 publishes its view BEFORE the barrier (slots of
    // alternating parity: a slot is rewritten two barriers after it was read), late atomics of this tile only make it conservative
    if (t == 0) s_flush[sweep_it & 1] = s_ncand >= (unsigned)(kSmemCand / 2) ? 1u : 0u;
    __syncthreads();
    if (s_flush[sweep_it & 1]) flush_cands();
    ++sweep_it;
  }
  flush_cands();
  {  // block-reduce the two counters, one atomic pair per CTA
    unsigned int x = c.n_lt, y = c.n_eq;
    for (int o = 16; o; o >>= 1) { x += __shfl_xor_sync(0xffffffffu, x, o); y += __shfl_xor_sync(0xffffffffu, y, o); }
    if ((t & 31) == 0) { s_red[0][t >> 5] = x; s_red[1][t >> 5] = y; }
    __syncthreads();
    if (t == 0) {
      unsigned long long A = 0, B = 0;
      for (int i = 0; i < kSweepThreads / 32; ++i) { A += s_red[0][i]; B += s_red[1][i]; }
      if (A) atomicAdd(&st->n_lt, A);
      if (B) atomicAdd(&st->n_eq, B);
    }
    for (int i = t; i < kDigitBins; i += kSweepThreads) if (s_h[i]) atomicAdd(&hist_r[i], s_h[i]);
  }
  grid.sync();
  stamp(st, 3);

  // ---------------- P3: does the bracket hold the k-th key?  (every CTA takes the same decision from the same counters)
  const unsigned long long k = (unsigned long long)a.k, A = st->n_lt, B = st->n_eq, C = st->n_cand;
  if (k <= A || C > a.cap || k > A + B + C) {           // below / above the bracket, or the list overflowed: exact fallback
    if (blockIdx.x == 0 && t == 0) st->status = 1;
    return;
  }
  const unsigned int n = (unsigned int)C;
  unsigned int thr;
  if (k <= A + B) {
    thr = lo;                                             // the k-th key is the lower bracket edge itself
  } else {
    unsigned long long krem = k - A - B;
    stamp(st, 4);

    // ---------------- P4: pick the top digit (its histogram was accumulated during the sweep) (every CTA); candidates that carry it form the second-level list
    if (t < 2) { s_bin[t] = 0; s_before[t] = 0; }
    __syncthreads();
    block_find_rank<kDigitBins / kSweepThreads>(hist_r, krem, &s_bin[0], &s_before[0], s_warp);
    unsigned int prefix = ((shift0 + 11 >= 32) ? 0u : (lo & (0xFFFFFFFFu << (shift0 + 11)))) | (s_bin[0] << shift0);
    krem -= s_before[0];
    if (shift0 > 0) {
      const unsigned int pmask = 0xFFFFFFFFu << shift0;
      for (unsigned int i = blockIdx.x * (unsigned)kSweepThreads + t; i < n; i += gridDim.x * (unsigned)kSweepThreads) {
        const unsigned int key = a.cand[i].x;
        if ((key & pmask) == prefix) {
          const unsigned long long slot = atomicAdd(&st->n_cand2, 1ull);
          if (slot < (unsigned long long)kCand2) a.cand2[slot] = key;
        }
      }
      grid.sync();
      stamp(st, 5);

      // ---------------- P5: finish the remaining digits over the second-level list in shared memory (every CTA, no barrier)
      const unsigned long long n2 = st->n_cand2;
      if (n2 > (unsigned long long)kCand2) {            // thousands of candidates share 11+ leading bits (heavy ties): exact fallback
        if (blockIdx.x == 0 && t == 0) st->status = 1;
        return;
      }
      for (unsigned int i = t; i < (unsigned int)n2; i += kSweepThreads) s_keys[i] = a.cand2[i];
      __syncthreads();
      for (int shift = shift0 - 11; shift >= 0; shift -= 11) {
        for (int i = t; i < kDigitBins; i += kSweepThreads) s_h[i] = 0;
        if (t < 2) { s_bin[t] = 0; s_before[t] = 0; }
        __syncthreads();
        const unsigned int pm = 0xFFFFFFFFu << (shift + 11);
        for (unsigned int i = t; i < (unsigned int)n2; i += kSweepThreads)
          if ((s_keys[i] & pm) == prefix) atomicAdd(&s_h[(s_keys[i] >> shift) & (kDigitBins - 1)], 1u);
        __syncthreads();
        block_find_rank<kDigitBins / kSweepThreads>(s_h, krem, &s_bin[0], &s_before[0], s_warp);
        prefix |= (s_bin[0] << shift);
        krem -= s_before[0];
        __syncthreads();
      }
    }
    thr = prefix;
  }
  // final mask value of every candidate (the sweep wrote a provisional 0); a NaN threshold keeps everything (host applies)
  if (WRITE && thr <= 0x7f800000u) {
    for (unsigned int i = blockIdx.x * (unsigned)kSweepThreads + t; i < n; i += gridDim.x * (unsigned)kSweepThreads) {
      const uint2 cd = a.cand[i];
      if (cd.x > thr) {
        const int si = find_seg_by_elem(segs, a.n_seg, (long long)cd.y);
        segs[si].mo[(long long)cd.y - segs[si].start] = 1.f;
      }
    }
  }
  if (blockIdx.x == 0 && t == 0) {
    st->thr_key = thr;
    *a.thr_out = __uint_as_float(thr);
    st->status = (thr > 0x7f800000u) ? 2 : 0;
  }
  stamp(st, 6);
}

// ---------------------------------------------------------------------------------------------
// Exact fallback: 11/11/10-bit radix passes over the full data.
template <int KIND>
__global__ void __launch_bounds__(kSweepThreads) k_hist_pass(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                             const SelState* __restrict__ st, int shift, int nbits,
                                                             unsigned int* __restrict__ hist) {
  __shared__ unsigned int s_hist[2048];
  const int t = threadIdx.x;
  for (int i = t; i < 2048; i += kSweepThreads) s_hist[i] = 0;
  __syncthreads();
  const unsigned int prefix = st->prefix, pmask = st->prefix_mask, dmask = (1u << nbits) - 1u;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const Seg& sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    for (int i = t; i < n_in; i += kSweepThreads) {
      unsigned int key = seg_key<KIND>(sg, base + i);
      if ((key & pmask) == prefix) atomicAdd(&s_hist[(key >> shift) & dmask], 1u);
    }
  }
  __syncthreads();
  for (int i = t; i < (1 << nbits); i += kSweepThreads)
    if (s_hist[i]) atomicAdd(&hist[i], s_hist[i]);
}

__global__ void k_pick_digit(const unsigned int* __restrict__ hist, int shift, int nbits, SelState* st) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  unsigned long long cum = 0, kr = st->k_rem;
  for (int d = 0; d < (1 << nbits); ++d) {
    unsigned long long h = hist[d];
    if (cum + h >= kr) {
      st->prefix |= ((unsigned int)d << shift);
      st->prefix_mask |= (((1u << nbits) - 1u) << shift);
      st->k_rem = kr - cum;
      break;
    }
    cum += h;
  }
}

__global__ void k_publish_thr(SelState* st, float* thr_out) {
  st->thr_key = st->prefix;
  st->status = (st->prefix > 0x7f800000u) ? 2 : 0;
  *thr_out = __uint_as_float(st->prefix);
}

// mask_out = score <= thr ? 0 : 1 in fp32 compare semantics (NaN threshold keeps everything).
template <int KIND>
__global__ void __launch_bounds__(kSweepThreads) k_apply(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                         const float* __restrict__ thr_p) {
  const float thr = *thr_p;
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    const float* wp = sg.w + base;
    const float* mp = sg.m + base;
    const float* gp = (KIND == TP_SCORE_MAG) ? nullptr : sg.g + base;
    float* op = sg.mo + base;
    bool vec = n_in == kTileElems &&
               ((((uintptr_t)wp) | ((uintptr_t)mp) | ((uintptr_t)gp) | ((uintptr_t)op)) & 15) == 0;
    if (vec) {
#pragma unroll
      for (int it = 0; it < kTileElems / (kSweepThreads * 4); ++it) {
        int q = it * kSweepThreads + t;
        float4 w = ld_stream((const float4*)wp + q), m = ld_stream((const float4*)mp + q);
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if (KIND != TP_SCORE_MAG) g = ld_stream((const float4*)gp + q);
        float4 o;
        o.x = (__uint_as_float(score_key<KIND>(w.x, g.x, m.x)) <= thr) ? 0.f : 1.f;
        o.y = (__uint_as_float(score_key<KIND>(w.y, g.y, m.y)) <= thr) ? 0.f : 1.f;
        o.z = (__uint_as_float(score_key<KIND>(w.z, g.z, m.z)) <= thr) ? 0.f : 1.f;
        o.w = (__uint_as_float(score_key<KIND>(w.w, g.w, m.w)) <= thr) ? 0.f : 1.f;
        st_stream((float4*)op + q, o);
      }
    } else {
      for (int i = t; i < n_in; i += kSweepThreads) {
        float g = (KIND == TP_SCORE_MAG) ? 0.f : gp[i];
        op[i] = (__uint_as_float(score_key<KIND>(wp[i], g, mp[i])) <= thr) ? 0.f : 1.f;
      }
    }
  }
}

__global__ void __launch_bounds__(kSweepThreads) k_count_zeros(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                               unsigned long long* __restrict__ out) {
  __shared__ unsigned int s_red[kSweepThreads / 32];
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    const float* mp = sg.m + base;
    unsigned int z = 0;
    if (n_in == kTileElems && (((uintptr_t)mp) & 15) == 0) {
#pragma unroll
      for (int it = 0; it < kTileElems / (kSweepThreads * 4); ++it) {
        float4 m = ld_stream((const float4*)mp + it * kSweepThreads + t);
        z += (m.x == 0.f) + (m.y == 0.f) + (m.z == 0.f) + (m.w == 0.f);
      }
    } else {
      for (int i = t; i < n_in; i += kSweepThreads) z += (mp[i] == 0.f);
    }
    for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    if ((t & 31) == 0) s_red[t >> 5] = z;
    __syncthreads();
    if (t == 0) {
      unsigned long long tot = 0;
      for (int i = 0; i < kSweepThreads / 32; ++i) tot += s_red[i];
      if (tot) { atomicAdd(&out[si], tot); atomicAdd(&out[n_seg], tot); }
    }
    __syncthreads();
  }
}

static unsigned int cand_cap(long long N) {
  long long c = N / 8;
  if (c < (1 << 16)) c = 1 << 16;
  if (c > (1 << 23)) c = 1 << 23;
  return (unsigned int)c;
}

static int sweep_grid(long long tiles) {
  long long g = (long long)sm_count() * 8;
  return (int)(tiles < g ? (tiles > 0 ? tiles : 1) : g);
}

// Workspace layout shared by enqueue / finish (both re-derive it from the same arguments).
struct TopkWs {
  Seg* segs; SelState* st; unsigned int* hist; unsigned int* cand2; uint2* cand; unsigned int cap;
};
static int carve_topk_ws(void* ws, size_t ws_bytes, int n_seg, long long N, TopkWs* out) {
  Arena ar(ws, ws_bytes);
  out->segs = (Seg*)ar.take(sizeof(Seg) * (size_t)n_seg);
  // state and histograms are adjacent: one memset clears both before every call
  out->st = (SelState*)ar.take(align_up(sizeof(SelState), 256) + sizeof(unsigned int) * 4 * kDigitBins);
  out->hist = out->st ? (unsigned int*)((char*)out->st + align_up(sizeof(SelState), 256)) : nullptr;
  out->cand2 = (unsigned int*)ar.take(sizeof(unsigned int) * kCand2);
  out->cap = cand_cap(N);
  out->cand = (uint2*)ar.take(sizeof(uint2) * (size_t)out->cap);
  return (out->segs && out->st && out->cand2 && out->cand) ? TP_OK : TP_ERR_WORKSPACE;
}

template <int KIND, bool WRITE>
static int fused_grid(int* grid_out) {
  static int cached = 0;
  if (!cached) {
    int occ = 0;
    TP_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_topk_fused<KIND, WRITE>, kSweepThreads, 0));
    if (occ < 1) return TP_ERR_UNSUPPORTED;
    if (occ > 4) occ = 4;
    cached = occ * sm_count();
  }
  *grid_out = cached;
  return TP_OK;
}

// The whole fast path: one memset + one cooperative kernel, no host synchronisation.
template <int KIND, bool WRITE>
static int enqueue_topk(const TopkWs& w, int n_seg, long long tiles, long long N, long long k, float* thr_out, cudaStream_t st) {
  int grid = 0;
  int rc = fused_grid<KIND, WRITE>(&grid); if (rc) return rc;
  TP_CUDA_CHECK(cudaMemsetAsync(w.st, 0, align_up(sizeof(SelState), 256) + sizeof(unsigned int) * 4 * kDigitBins, st));
  long long S = N < (1ll << kSampleBits) ? N : (1ll << kSampleBits);
  const long long smax = (long long)grid * kLocalKeys;             // what the CTAs can keep in shared memory (one round of runs each)
  if (S > smax) S = smax;
  // sample rank of the population's k-th element and the +-5 sigma band of its sampling error
  long long rs = (long long)(((unsigned __int128)(unsigned long long)k * (unsigned long long)S + (unsigned long long)N - 1) /
                             (unsigned long long)N);
  if (rs < 1) rs = 1;
  if (rs > S) rs = S;
  const double pq = (double)rs / (double)S;
  // The samples come in runs of kRun neighbours (same filter: correlated scale), so the band is 6 sigma of the iid
  // rank error instead of 5 (covers a design effect of ~1.5 at 5 sigma); + kRun per segment: runs are clamped at segment ends, so a few
  // samples may repeat (also when S == N).  A miss is not an error, only the slow exact path.
  const long long delta = (long long)(6.0 * sqrt((double)S * pq * (1.0 - pq)) + 8.0) + (long long)kRun * n_seg;
  TopkArgs a;
  a.segs = w.segs; a.n_seg = n_seg; a.tiles = tiles; a.N = N; a.S = S; a.k = k; a.r_lo = rs - delta; a.r_hi = rs + delta;
  a.st = w.st; a.hist = w.hist; a.cand = w.cand; a.cap = w.cap; a.cand2 = w.cand2; a.thr_out = thr_out;
  // grid <= occupancy x SMs: every CTA is resident, which is what the in-kernel barrier needs
  k_topk_fused<KIND, WRITE><<<grid, kSweepThreads, 0, st>>>(a);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

// Status read-back (the only host synchronisation of the path) and the slow paths it may call for.
template <int KIND>
static int finish_topk(const TopkWs& w, int n_seg, long long tiles, long long k, bool write, float* thr_out, int64_t* info,
                       cudaStream_t st) {
  SelState h = {};
  TP_CUDA_CHECK(cudaMemcpyAsync(&h, w.st, sizeof(h), cudaMemcpyDeviceToHost, st));
  TP_CUDA_CHECK(cudaStreamSynchronize(st));
  const long long n_cand = (long long)h.n_cand, n_lt = (long long)h.n_lt;
  const int grid = sweep_grid(tiles);
  int path = 0;
  if (h.status == 1) {
    // exact fallback: 3 radix passes over the full data
    path = 1;
    SelState f = {};
    f.k = (unsigned long long)k; f.k_rem = (unsigned long long)k;
    TP_CUDA_CHECK(cudaMemcpyAsync(w.st, &f, sizeof(f), cudaMemcpyHostToDevice, st));
    const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
    for (int p = 0; p < 3; ++p) {
      TP_CUDA_CHECK(cudaMemsetAsync(w.hist, 0, sizeof(unsigned int) * 2048, st));
      k_hist_pass<KIND><<<grid, kSweepThreads, 0, st>>>(w.segs, n_seg, tiles, w.st, shifts[p], bits[p], w.hist);
      k_pick_digit<<<1, 32, 0, st>>>(w.hist, shifts[p], bits[p], w.st);
    }
    k_publish_thr<<<1, 1, 0, st>>>(w.st, thr_out);
    if (write) k_apply<KIND><<<grid, kSweepThreads, 0, st>>>(w.segs, n_seg, tiles, thr_out);
    TP_LAUNCH_CHECK();
    TP_CUDA_CHECK(cudaMemcpyAsync(&h, w.st, sizeof(h), cudaMemcpyDeviceToHost, st));
    TP_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  if (h.status == 2 && write && path == 0) {
    // NaN threshold: `score <= nan` is false everywhere -> every mask entry becomes 1
    k_apply<KIND><<<grid, kSweepThreads, 0, st>>>(w.segs, n_seg, tiles, thr_out);
    TP_LAUNCH_CHECK();
  }
  if (info) { info[0] = path; info[1] = n_cand; info[2] = n_lt; info[3] = (h.status == 2); }
  return TP_OK;
}

// ---------------------------------------------------------------------------------------------
// RigL drop-and-regrow (Evci et al. 2020), exact per segment (= layer):
//   DROP: among mask != 0, the k smallest |w|;   GROW: among new mask == 0 after the drop, the k largest |g|.
// Key: the fp32 bit pattern of |x| (sign cleared) as an unsigned integer; GROW uses its complement, so that both are
// "k smallest keys".  Ties at the k-th key go to the lower flat index first.  For each of DROP and GROW:
//   3 x (k_rigl_hist, k_rigl_pick) : 11/11/10-bit radix select on one 2048-bin histogram per segment -> threshold key T
//                                    and r = how many of the eligible keys == T are taken
//   k_rigl_ties                    : per tile, the eligible keys == T
//   k_rigl_tie_scan                : per segment, the exclusive prefix of those counts over its tiles
//   k_rigl_write                   : selected = key < T, or key == T with index-order rank < r (block prefix in the tile);
//                                    DROP writes new = (mask != 0) && !selected, GROW sets new = 1 where selected
// Every thread owns kRiglPer neighbouring elements of a tile, so the block prefix follows the flat index.  Integer
// atomics only: masks and counts are deterministic.  A k larger than the active count drops all of them; the grow
// always takes as many as the drop took, so every segment keeps its active count.
constexpr int kRiglPer = kTileElems / kSweepThreads;      // 16

struct RiglSel {
  unsigned long long k;          // requested count; after the first pick, min(k, eligible)
  unsigned long long k_rem;      // ties at the threshold still to take
  unsigned int prefix, pmask;    // selected digits so far; after three passes prefix is the threshold key T
  int none;                      // nothing to select in this segment (k == 0 or no eligible position)
  int pad_;
};

// Load this thread's kRiglPer elements of a tile: their keys, and a bit per eligible position.
template <int PHASE>
__device__ __forceinline__ unsigned int rigl_load(const Seg& sg, long long base, int n_in, unsigned int (&key)[kRiglPer]) {
  const int j0 = threadIdx.x * kRiglPer;
  int cnt = n_in - j0;
  cnt = cnt < 0 ? 0 : (cnt > kRiglPer ? kRiglPer : cnt);
  const float* a = (PHASE == 0 ? sg.m : sg.mo) + base + j0;     // eligibility operand
  const float* b = (PHASE == 0 ? sg.w : sg.g) + base + j0;      // key operand
  float va[kRiglPer], vb[kRiglPer];
  if (cnt == kRiglPer && ((((uintptr_t)a) | ((uintptr_t)b)) & 15) == 0) {
#pragma unroll
    for (int q = 0; q < kRiglPer / 4; ++q) {
      const float4 x = ((const float4*)a)[q], y = ((const float4*)b)[q];
      va[4 * q] = x.x; va[4 * q + 1] = x.y; va[4 * q + 2] = x.z; va[4 * q + 3] = x.w;
      vb[4 * q] = y.x; vb[4 * q + 1] = y.y; vb[4 * q + 2] = y.z; vb[4 * q + 3] = y.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < kRiglPer; ++j) { va[j] = j < cnt ? a[j] : 0.f; vb[j] = j < cnt ? b[j] : 0.f; }
  }
  unsigned int elig = 0;
#pragma unroll
  for (int j = 0; j < kRiglPer; ++j) {
    const unsigned int mag = __float_as_uint(vb[j]) & 0x7fffffffu;
    key[j] = PHASE == 0 ? mag : ~mag;
    const bool e = j < cnt && (PHASE == 0 ? va[j] != 0.f : va[j] == 0.f);
    elig |= (unsigned int)e << j;
  }
  return elig;
}

__device__ __forceinline__ unsigned int block_sum_u32(unsigned int v, unsigned int* s_red /* [kSweepThreads / 32] */) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned int tot = 0;
#pragma unroll
  for (int i = 0; i < kSweepThreads / 32; ++i) tot += s_red[i];
  return tot;
}

// Exclusive prefix of v over the block in thread order; *total gets the sum.
__device__ __forceinline__ unsigned int block_excl_scan_u32(unsigned int v, unsigned int* s_red /* [kSweepThreads / 32] */,
                                                            unsigned int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  __syncthreads();
  if (lane == 31) s_red[warp] = inc;
  __syncthreads();
  unsigned int before = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < kSweepThreads / 32; ++i) { before += i < warp ? s_red[i] : 0u; tot += s_red[i]; }
  *total = tot;
  return before + inc - v;
}

// One digit pass: per-segment histograms of the eligible keys that match the prefix.  Each CTA walks a contiguous
// range of tiles and flushes its shared histogram when the segment changes.
template <int PHASE>
__global__ void __launch_bounds__(kSweepThreads) k_rigl_hist(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                             const RiglSel* __restrict__ sel, int shift, int nbits,
                                                             unsigned int* __restrict__ hist) {
  __shared__ unsigned int s_hist[2048];
  const int t = threadIdx.x;
  const unsigned int dmask = (1u << nbits) - 1u;
  for (int i = t; i < 2048; i += kSweepThreads) s_hist[i] = 0;
  __syncthreads();
  const long long t0 = tiles * blockIdx.x / gridDim.x, t1 = tiles * (blockIdx.x + 1) / gridDim.x;
  int cur = -1;
  bool dirty = false;
  for (long long tile = t0; tile < t1; ++tile) {
    const int si = find_seg(segs, n_seg, tile);
    if (si != cur) {
      if (dirty) {
        __syncthreads();
        for (int i = t; i < 2048; i += kSweepThreads)
          if (s_hist[i]) { atomicAdd(&hist[(size_t)cur * 2048 + i], s_hist[i]); s_hist[i] = 0; }
        __syncthreads();
      }
      cur = si; dirty = false;
    }
    const RiglSel s = sel[si];
    if (s.none) continue;
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    unsigned int key[kRiglPer];
    const unsigned int elig = rigl_load<PHASE>(sg, base, rem < kTileElems ? (int)rem : kTileElems, key);
#pragma unroll
    for (int j = 0; j < kRiglPer; ++j)
      if (((elig >> j) & 1u) && (key[j] & s.pmask) == s.prefix) atomicAdd(&s_hist[(key[j] >> shift) & dmask], 1u);
    dirty = true;
  }
  if (dirty) {
    __syncthreads();
    for (int i = t; i < 2048; i += kSweepThreads)
      if (s_hist[i]) atomicAdd(&hist[(size_t)cur * 2048 + i], s_hist[i]);
  }
}

// One CTA per segment: pick the digit holding the k_rem-th key, then clear the histogram for the next pass.  The first
// pass clamps k to the eligible count and, for GROW, to what the DROP took (`cap`, NULL for DROP).
__global__ void __launch_bounds__(kSweepThreads) k_rigl_pick(unsigned int* __restrict__ hist, RiglSel* __restrict__ sel,
                                                             const RiglSel* __restrict__ cap, int shift, int nbits, int first) {
  __shared__ unsigned int s_bin, s_red[kSweepThreads / 32];
  __shared__ unsigned long long s_before, s_warp[32];
  const int t = threadIdx.x;
  RiglSel* s = sel + blockIdx.x;
  unsigned int* h = hist + (size_t)blockIdx.x * 2048;
  if (s->none) return;
  unsigned long long kr = s->k_rem;
  if (first) {
    unsigned int loc = 0;
#pragma unroll
    for (int i = 0; i < 2048 / kSweepThreads; ++i) loc += h[t * (2048 / kSweepThreads) + i];
    const unsigned long long eligible = block_sum_u32(loc, s_red);
    kr = s->k < eligible ? s->k : eligible;
    if (cap && cap[blockIdx.x].k < kr) kr = cap[blockIdx.x].k;
    if (kr == 0) {
      for (int i = t; i < 2048; i += kSweepThreads) h[i] = 0;
      if (t == 0) { s->k = 0; s->none = 1; }
      return;
    }
  }
  block_find_rank<2048 / kSweepThreads>(h, kr, &s_bin, &s_before, s_warp);
  for (int i = t; i < 2048; i += kSweepThreads) h[i] = 0;
  if (t == 0) {
    if (first) s->k = kr;
    s->prefix |= s_bin << shift;
    s->pmask |= ((1u << nbits) - 1u) << shift;
    s->k_rem = kr - s_before;
  }
}

template <int PHASE>
__global__ void __launch_bounds__(kSweepThreads) k_rigl_ties(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                             const RiglSel* __restrict__ sel, unsigned int* __restrict__ tie_cnt) {
  __shared__ unsigned int s_red[kSweepThreads / 32];
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const RiglSel s = sel[si];
    unsigned int c = 0;
    if (!s.none) {
      const Seg sg = segs[si];
      const long long base = (tile - sg.tile0) * kTileElems;
      const long long rem = sg.n - base;
      unsigned int key[kRiglPer];
      const unsigned int elig = rigl_load<PHASE>(sg, base, rem < kTileElems ? (int)rem : kTileElems, key);
#pragma unroll
      for (int j = 0; j < kRiglPer; ++j) c += ((elig >> j) & 1u) && key[j] == s.prefix;
    }
    const unsigned int tot = block_sum_u32(c, s_red);
    if (threadIdx.x == 0) tie_cnt[tile] = tot;
  }
}

// One CTA per segment: tie_off[tile] = ties of the segment in the tiles before this one.
__global__ void __launch_bounds__(kSweepThreads) k_rigl_tie_scan(const Seg* __restrict__ segs, const RiglSel* __restrict__ sel,
                                                                 const unsigned int* __restrict__ tie_cnt,
                                                                 unsigned int* __restrict__ tie_off) {
  __shared__ unsigned int s_red[kSweepThreads / 32];
  if (sel[blockIdx.x].none) return;
  const Seg sg = segs[blockIdx.x];
  const long long nt = (sg.n + kTileElems - 1) / kTileElems;
  unsigned int carry = 0;
  for (long long c0 = 0; c0 < nt; c0 += kSweepThreads) {
    const long long i = c0 + threadIdx.x;
    const unsigned int v = i < nt ? tie_cnt[sg.tile0 + i] : 0u;
    unsigned int tot;
    const unsigned int ex = block_excl_scan_u32(v, s_red, &tot);
    if (i < nt) tie_off[sg.tile0 + i] = carry + ex;
    carry += tot;
  }
}

template <int PHASE>
__global__ void __launch_bounds__(kSweepThreads) k_rigl_write(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                              const RiglSel* __restrict__ sel,
                                                              const unsigned int* __restrict__ tie_cnt,
                                                              const unsigned int* __restrict__ tie_off,
                                                              unsigned long long* __restrict__ counts) {
  __shared__ unsigned int s_red[kSweepThreads / 32];
  const int t = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const RiglSel s = sel[si];
    if (PHASE == 1 && s.none) continue;               // GROW leaves such a segment as the DROP wrote it
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    unsigned int key[kRiglPer];
    const unsigned int elig = rigl_load<PHASE>(sg, base, n_in, key);
    unsigned int picked = 0;
    if (!s.none) {
      const unsigned int T = s.prefix;
      unsigned int ord = 0;
      if (tie_cnt[tile]) {                              // this tile holds ties at T: their rank in the segment
        unsigned int mine = 0, tot;
#pragma unroll
        for (int j = 0; j < kRiglPer; ++j) mine += ((elig >> j) & 1u) && key[j] == T;
        ord = tie_off[tile] + block_excl_scan_u32(mine, s_red, &tot);
      }
#pragma unroll
      for (int j = 0; j < kRiglPer; ++j) {
        if (!((elig >> j) & 1u)) continue;
        if (key[j] < T) picked |= 1u << j;
        else if (key[j] == T) { if ((unsigned long long)ord < s.k_rem) picked |= 1u << j; ++ord; }
      }
    }
    const int j0 = t * kRiglPer;
    float* o = sg.mo + base + j0;
    if (PHASE == 0) {
      const unsigned int keep = elig & ~picked;
      if (n_in - j0 >= kRiglPer && (((uintptr_t)o) & 15) == 0) {
#pragma unroll
        for (int q = 0; q < kRiglPer / 4; ++q)
          ((float4*)o)[q] = make_float4((float)((keep >> (4 * q)) & 1u), (float)((keep >> (4 * q + 1)) & 1u),
                                        (float)((keep >> (4 * q + 2)) & 1u), (float)((keep >> (4 * q + 3)) & 1u));
      } else {
        for (int j = 0; j < kRiglPer && j0 + j < n_in; ++j) o[j] = (float)((keep >> j) & 1u);
      }
    } else {
#pragma unroll
      for (int j = 0; j < kRiglPer; ++j)
        if ((picked >> j) & 1u) o[j] = 1.f;
    }
    const unsigned int tot = block_sum_u32(__popc(picked), s_red);
    if (t == 0 && tot) atomicAdd(&counts[2 * si + PHASE], (unsigned long long)tot);
  }
}

// mask <- new; where new != 0 and old == 0 the weight and its optimizer state (if any) restart from 0.
// Seg: m = mask (written), g = new mask, w = weight (written), buf = first state array (nullable).
// xs: the further state arrays, xs[j * n_seg + i] = state j + 1 of segment i (nullable entries), n_xs of them per segment.
__global__ void __launch_bounds__(kSweepThreads) k_rigl_apply(const Seg* __restrict__ segs, int n_seg, long long tiles,
                                                              float* const* __restrict__ xs, int n_xs) {
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int si = find_seg(segs, n_seg, tile);
    const Seg sg = segs[si];
    const long long base = (tile - sg.tile0) * kTileElems;
    const long long rem = sg.n - base;
    const int n_in = rem < kTileElems ? (int)rem : kTileElems;
    float* m = const_cast<float*>(sg.m) + base;
    float* w = const_cast<float*>(sg.w) + base;
    float* buf = sg.buf ? sg.buf + base : nullptr;
    const float* nm = sg.g + base;
    for (int i = threadIdx.x; i < n_in; i += kSweepThreads) {
      const float old = m[i], nw = nm[i];
      if (nw != 0.f && old == 0.f) {
        w[i] = 0.f;
        if (buf) buf[i] = 0.f;
        for (int j = 0; j < n_xs; ++j) {
          float* x = xs[(size_t)j * n_seg + si];
          if (x) x[base + i] = 0.f;
        }
      }
      if (__float_as_uint(nw) != __float_as_uint(old)) m[i] = nw;
    }
  }
}

struct RiglWs {
  Seg* segs; RiglSel* sel; unsigned int* hist; unsigned int* tie_cnt; unsigned int* tie_off;
};

static long long rigl_max_tiles(int n_seg, long long total) { return total / kTileElems + n_seg + 1; }

template <int PHASE>
static int rigl_phase(const RiglWs& w, int n_seg, long long tiles, unsigned long long* counts, cudaStream_t st) {
  const int grid = sweep_grid(tiles);
  RiglSel* sel = w.sel + (size_t)PHASE * n_seg;
  const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
  for (int p = 0; p < 3; ++p) {
    k_rigl_hist<PHASE><<<grid, kSweepThreads, 0, st>>>(w.segs, n_seg, tiles, sel, shifts[p], bits[p], w.hist);
    k_rigl_pick<<<n_seg, kSweepThreads, 0, st>>>(w.hist, sel, PHASE == 1 ? w.sel : nullptr, shifts[p], bits[p], p == 0);
  }
  k_rigl_ties<PHASE><<<grid, kSweepThreads, 0, st>>>(w.segs, n_seg, tiles, sel, w.tie_cnt);
  k_rigl_tie_scan<<<n_seg, kSweepThreads, 0, st>>>(w.segs, sel, w.tie_cnt, w.tie_off);
  k_rigl_write<PHASE><<<grid, kSweepThreads, 0, st>>>(w.segs, n_seg, tiles, sel, w.tie_cnt, w.tie_off, counts);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // namespace tp

using namespace tp;

extern "C" {

size_t tp_topk_workspace_bytes(int n_seg, int64_t total_numel) {
  size_t b = 0;
  b += align_up(sizeof(Seg) * (size_t)(n_seg > 0 ? n_seg : 1), 256);
  b += align_up(align_up(sizeof(SelState), 256) + sizeof(unsigned int) * 4 * kDigitBins, 256);
  b += align_up(sizeof(unsigned int) * kCand2, 256);
  b += align_up(sizeof(uint2) * (size_t)cand_cap(total_numel), 256);
  return b + 1024;
}

static int topk_common(const void* const* w, const void* const* g, const void* const* m, void* const* mask_out,
                       const int64_t* numel, int n_seg, int64_t k, int score_kind, float* thr_out, void* ws, size_t ws_bytes,
                       int table_cached, bool do_enqueue, bool do_finish, int64_t* info_out, cudaStream_t st) {
  if (!m || !numel || n_seg <= 0 || !thr_out || !ws) return TP_ERR_INVALID;
  if (!table_cached && (!w || (score_kind != TP_SCORE_MAG && !g))) return TP_ERR_INVALID;
  if (score_kind < 0 || score_kind > 2) return TP_ERR_INVALID;
  long long N = 0, tiles = 0;
  for (int i = 0; i < n_seg; ++i) { if (numel[i] < 0) return TP_ERR_INVALID; N += numel[i]; tiles += (numel[i] + kTileElems - 1) / kTileElems; }
  if (k < 1 || k > N) return TP_ERR_K_RANGE;          // torch.kthvalue raises (pruning_utils.py:79)
  if (N >= (1ll << 32)) return TP_ERR_UNSUPPORTED;    // candidate records carry 32-bit indices
  TopkWs t;
  int rc = carve_topk_ws(ws, ws_bytes, n_seg, N, &t); if (rc) return rc;
  const bool write = mask_out != nullptr;
  if (do_enqueue) {
    if (!table_cached) {
      Arena ar(ws, ws_bytes);
      Seg* d_segs = nullptr;
      rc = upload_segs(ar, w, g, m, mask_out, nullptr, numel, n_seg, &d_segs, nullptr, nullptr, st); if (rc) return rc;
      if (d_segs != t.segs) return TP_ERR_WORKSPACE;
    }
#define TP_ENQ(KIND) (write ? enqueue_topk<KIND, true>(t, n_seg, tiles, N, k, thr_out, st) : enqueue_topk<KIND, false>(t, n_seg, tiles, N, k, thr_out, st))
    rc = score_kind == TP_SCORE_MAG ? TP_ENQ(TP_SCORE_MAG) : (score_kind == TP_SCORE_SNIP ? TP_ENQ(TP_SCORE_SNIP) : TP_ENQ(TP_SCORE_SYNFLOW));
#undef TP_ENQ
    if (rc) return rc;
  }
  if (do_finish) {
    switch (score_kind) {
      case TP_SCORE_MAG: return finish_topk<TP_SCORE_MAG>(t, n_seg, tiles, k, write, thr_out, info_out, st);
      case TP_SCORE_SNIP: return finish_topk<TP_SCORE_SNIP>(t, n_seg, tiles, k, write, thr_out, info_out, st);
      default: return finish_topk<TP_SCORE_SYNFLOW>(t, n_seg, tiles, k, write, thr_out, info_out, st);
    }
  }
  return TP_OK;
}

int tp_topk_threshold_mask(const void* const* w, const void* const* g, const void* const* m,
                           void* const* mask_out, const int64_t* numel, int n_seg,
                           int64_t k, int score_kind, float* thr_out,
                           void* ws, size_t ws_bytes, int64_t* info_out, void* stream) {
  return topk_common(w, g, m, mask_out, numel, n_seg, k, score_kind, thr_out, ws, ws_bytes, 0, true, true, info_out, (cudaStream_t)stream);
}

int tp_topk_enqueue(const void* const* w, const void* const* g, const void* const* m,
                    void* const* mask_out, const int64_t* numel, int n_seg,
                    int64_t k, int score_kind, float* thr_out,
                    void* ws, size_t ws_bytes, int table_cached, void* stream) {
  return topk_common(w, g, m, mask_out, numel, n_seg, k, score_kind, thr_out, ws, ws_bytes, table_cached, true, false, nullptr, (cudaStream_t)stream);
}

int tp_topk_finish(const void* const* m, void* const* mask_out, const int64_t* numel, int n_seg,
                   int64_t k, int score_kind, float* thr_out,
                   void* ws, size_t ws_bytes, int64_t* info_out, void* stream) {
  return topk_common(nullptr, nullptr, m, mask_out, numel, n_seg, k, score_kind, thr_out, ws, ws_bytes, 1, false, true, info_out, (cudaStream_t)stream);
}

int tp_apply_threshold(const void* const* w, const void* const* g, const void* const* m,
                       void* const* mask_out, const int64_t* numel, int n_seg,
                       int score_kind, const float* thr, void* ws, size_t ws_bytes, void* stream) {
  if (!w || !m || !mask_out || !numel || n_seg <= 0 || !thr || !ws) return TP_ERR_INVALID;
  if (score_kind != TP_SCORE_MAG && !g) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  int rc = upload_segs(ar, w, g, m, mask_out, nullptr, numel, n_seg, &d_segs, &tiles, nullptr, st);
  if (rc) return rc;
  if (tiles == 0) return TP_OK;
  const int grid = sweep_grid(tiles);
  if (score_kind == TP_SCORE_MAG) k_apply<TP_SCORE_MAG><<<grid, kSweepThreads, 0, st>>>(d_segs, n_seg, tiles, thr);
  else if (score_kind == TP_SCORE_SNIP) k_apply<TP_SCORE_SNIP><<<grid, kSweepThreads, 0, st>>>(d_segs, n_seg, tiles, thr);
  else if (score_kind == TP_SCORE_SYNFLOW) k_apply<TP_SCORE_SYNFLOW><<<grid, kSweepThreads, 0, st>>>(d_segs, n_seg, tiles, thr);
  else return TP_ERR_INVALID;
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_count_zeros(const void* const* m, const int64_t* numel, int n_seg,
                   int64_t* zeros_out, void* ws, size_t ws_bytes, void* stream) {
  if (!m || !numel || n_seg <= 0 || !zeros_out || !ws) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  int rc = upload_segs(ar, nullptr, nullptr, m, nullptr, nullptr, numel, n_seg, &d_segs, &tiles, nullptr, st);
  if (rc) return rc;
  TP_CUDA_CHECK(cudaMemsetAsync(zeros_out, 0, sizeof(int64_t) * (size_t)(n_seg + 1), st));
  if (tiles == 0) return TP_OK;
  k_count_zeros<<<sweep_grid(tiles), kSweepThreads, 0, st>>>(d_segs, n_seg, tiles, (unsigned long long*)zeros_out);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

size_t tp_rigl_workspace_bytes(int n_seg, int64_t total_numel) {
  const size_t ns = (size_t)(n_seg > 0 ? n_seg : 1);
  const size_t tiles = (size_t)rigl_max_tiles((int)ns, total_numel);
  return align_up(sizeof(Seg) * ns, 256) + align_up(sizeof(RiglSel) * 2 * ns, 256) + align_up(sizeof(unsigned int) * 2048 * ns, 256) +
         2 * align_up(sizeof(unsigned int) * tiles, 256) + 1024;
}

int tp_rigl_select(const void* const* w, const void* const* g, const void* const* mask, void* const* new_mask_out,
                   const int64_t* numel, const int64_t* k, int n_seg, int64_t* counts_out, void* ws, size_t ws_bytes,
                   void* stream) {
  if (!w || !g || !mask || !new_mask_out || !numel || !k || n_seg <= 0 || !counts_out || !ws) return TP_ERR_INVALID;
  for (int i = 0; i < n_seg; ++i) {
    if (!w[i] || !g[i] || !mask[i] || !new_mask_out[i]) return TP_ERR_INVALID;
    if (numel[i] < 0 || numel[i] > (1ll << 31) || k[i] < 0) return TP_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  RiglWs t;
  long long tiles = 0, total = 0;
  int rc = upload_segs(ar, w, g, mask, new_mask_out, nullptr, numel, n_seg, &t.segs, &tiles, &total, st);
  if (rc) return rc;
  t.sel = (RiglSel*)ar.take(sizeof(RiglSel) * 2 * (size_t)n_seg);
  t.hist = (unsigned int*)ar.take(sizeof(unsigned int) * 2048 * (size_t)n_seg);
  t.tie_cnt = (unsigned int*)ar.take(sizeof(unsigned int) * (size_t)(tiles > 0 ? tiles : 1));
  t.tie_off = (unsigned int*)ar.take(sizeof(unsigned int) * (size_t)(tiles > 0 ? tiles : 1));
  if (!t.sel || !t.hist || !t.tie_cnt || !t.tie_off) return TP_ERR_WORKSPACE;
  std::vector<RiglSel> h(2 * (size_t)n_seg);
  for (int p = 0; p < 2; ++p)
    for (int i = 0; i < n_seg; ++i) {
      RiglSel& s = h[(size_t)p * n_seg + i];
      s = RiglSel{};
      s.k = (unsigned long long)k[i];
      s.k_rem = s.k;
      s.none = k[i] == 0;
    }
  // pageable source: the runtime stages the bytes before returning, so `h` may die.
  TP_CUDA_CHECK(cudaMemcpyAsync(t.sel, h.data(), sizeof(RiglSel) * h.size(), cudaMemcpyHostToDevice, st));
  TP_CUDA_CHECK(cudaMemsetAsync(t.hist, 0, sizeof(unsigned int) * 2048 * (size_t)n_seg, st));   // the picks clear it after use
  TP_CUDA_CHECK(cudaMemsetAsync(counts_out, 0, sizeof(int64_t) * 2 * (size_t)n_seg, st));
  if (tiles == 0) return TP_OK;
  rc = rigl_phase<0>(t, n_seg, tiles, (unsigned long long*)counts_out, st); if (rc) return rc;
  return rigl_phase<1>(t, n_seg, tiles, (unsigned long long*)counts_out, st);
}

int tp_rigl_apply_states(void* const* mask, const void* const* new_mask, void* const* w, void* const* states, int n_states,
                         const int64_t* numel, int n_seg, void* ws, size_t ws_bytes, void* stream) {
  if (!mask || !new_mask || !w || !numel || n_seg <= 0 || !ws || n_states < 0 || (n_states > 0 && !states)) return TP_ERR_INVALID;
  for (int i = 0; i < n_seg; ++i)
    if (!mask[i] || !new_mask[i] || !w[i] || numel[i] < 0 || numel[i] > (1ll << 31)) return TP_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(ws, ws_bytes);
  Seg* d_segs = nullptr; long long tiles = 0;
  int rc = upload_segs(ar, (const void* const*)w, new_mask, (const void* const*)mask, nullptr, n_states > 0 ? states : nullptr,
                       numel, n_seg, &d_segs, &tiles, nullptr, st);
  if (rc) return rc;
  // states past the first: a pointer array behind the segment table
  const int n_xs = n_states > 1 ? n_states - 1 : 0;
  float** d_xs = nullptr;
  if (n_xs > 0) {
    d_xs = (float**)ar.take(sizeof(float*) * (size_t)n_xs * n_seg);
    if (!d_xs) return TP_ERR_WORKSPACE;
    // pageable source: the runtime stages the bytes before returning
    TP_CUDA_CHECK(cudaMemcpyAsync(d_xs, states + n_seg, sizeof(float*) * (size_t)n_xs * n_seg, cudaMemcpyHostToDevice, st));
  }
  if (tiles == 0) return TP_OK;
  k_rigl_apply<<<sweep_grid(tiles), kSweepThreads, 0, st>>>(d_segs, n_seg, tiles, d_xs, n_xs);
  TP_LAUNCH_CHECK();
  return TP_OK;
}

int tp_rigl_apply(void* const* mask, const void* const* new_mask, void* const* w, void* const* momentum,
                  const int64_t* numel, int n_seg, void* ws, size_t ws_bytes, void* stream) {
  return tp_rigl_apply_states(mask, new_mask, w, momentum, momentum ? 1 : 0, numel, n_seg, ws, ws_bytes, stream);
}

}  // extern "C"
