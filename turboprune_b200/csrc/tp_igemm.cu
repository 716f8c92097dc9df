// Masked implicit-GEMM convolution / linear for sm_90a: TMA (tiled + im2col) -> 128B-swizzled
// shared memory -> wgmma (bf16 x bf16 -> fp32 in registers) -> epilogue.
//
// Replaces F.conv2d / F.linear / F.conv1d(k=1) on the masked weight and their autograd
// backward (utils/mask_layers.py:26-34, :70, :110-118 of the reference).  The mask never
// appears here as a separate pass: fprop/dgrad consume bf16 weights that were masked while
// being staged (tp_stage_weights), wgrad applies the mask in its finalize step.
//
// Two persistent, warp-specialised kernels (1 CTA / SM):
//   k_igemm_fwd (384 threads, ping-pong consumers):
//     warpgroup 0    : TMA producer (one lane; the warpgroup gives its registers up to the consumers)
//     warpgroups 1, 2: consumers; the CTA's work items alternate between them and each owns its whole 128 x BLOCK_N
//                      tile (MMA and epilogue).  Their mainloops take turns, so one warpgroup's epilogue runs under
//                      the other's MMAs and the tensor cores do not wait for the epilogue.
//   k_igemm_wgrad (288 threads):
//     warps 0..7     : two consumer warpgroups; warpgroup g issues the wgmma of rows 64g .. 64g+63 of the 128-row
//                      tile, then stores its fragments (the K loops are long, the epilogue is one store)
//     warp 8         : TMA producer (one elected lane)
//
//   k_igemm_fwd  : D[pixels, Cout] = A[pixels, K] * W[Cout, K]^T          (fprop, dgrad)
//                  A tile 128 pixels x 64 channels by TMA im2col (any r,s,stride,pad) or by
//                  a plain 2-D TMA box (1x1/s1 convs, linear); both K-major, SWIZZLE_128B.
//   k_igemm_wgrad: D[Cout, (tap,cin)] = dY^T[Cout, pixels] * Xcol[pixels, (tap,cin)]
//                  contraction over pixels: both operands MN-major, SWIZZLE_128B; split-K
//                  partials in fp32, summed in fixed order + masked + permuted to OIHW by
//                  k_wgrad_finalize (deterministic, no atomics).
#include "tp_common.cuh"
#include "tp_ptx.cuh"
#include <cuda.h>
#include <mutex>

namespace tp {
using namespace ptx;

constexpr int kBlockM = 128;         // two wgmma M = 64 halves
constexpr int kBlockK = 64;          // 64 bf16 = 128 B = one swizzle row
constexpr int kConsumers = 256;      // two consumer warpgroups
constexpr int kThreads = kConsumers + 32;   // k_igemm_wgrad: + the TMA producer warp
constexpr int kProducerWarp = kConsumers / 32;
constexpr int kFwdThreads = 3 * 128;        // k_igemm_fwd: producer warpgroup + two consumer warpgroups
constexpr int kMaxTaps = 64;

// Registers per thread after the k_igemm_fwd warpgroups re-balance them: the launch gives 168 to each of the 384 threads
// (65536 / 384, rounded down to a multiple of 8), and an increase waits until the producer's decrease has freed enough,
// so the two must add up to no more than the launch allocation.  The producer gets 56, not the usual 40: its K walk keeps
// the KSkip state, the im2col coordinates and (MULTI) the class decode live, and ptxas spills it to local memory at 40
// (every instantiation) and at 48 (both MULTI instantiations).  224 is what is left for the consumers, enough for the 128
// accumulators of BLOCK_N = 128 plus the epilogue without spills.
constexpr int kFwdProducerRegs = 56, kFwdConsumerRegs = 224;
static_assert(kFwdProducerRegs * 128 + kFwdConsumerRegs * 256 <= 168 * kFwdThreads, "fwd register split");

// smem pipeline depth of the fwd kernel: stage = A tile (16 KB) + weight tile (8 or 16 KB)
__host__ __device__ constexpr int fwd_stages(int block_n) { return block_n == 128 ? 5 : 8; }
// epilogue staging tile of one consumer warpgroup: 128 rows x BLOCK_N bf16, as 64-column sub-tiles of 16 KB
__host__ __device__ constexpr int fwd_stg_bytes(int block_n) { return kBlockM * block_n * 2; }
// fwd smem: the stages, both consumers' staging tiles, alignment slack and barriers
__host__ __device__ constexpr int fwd_smem(int block_n) {
  return fwd_stages(block_n) * (kBlockM * kBlockK * 2 + block_n * kBlockK * 2) + 2 * fwd_stg_bytes(block_n) + 1024 + 512;
}

struct TapEntry { uint16_t off_w, off_h; int32_t kofs; };

constexpr int kMaxCls = 4;

// One "class" of output pixels.  fprop and stride-1 dgrad have a single class (every output pixel, every tap).  The
// dgrad of a strided convolution splits dX into stride_h x stride_w parity classes: class (a, b) = the input pixels
// (stride*h' + a, stride*w' + b), each a stride-1 gather over dY with its own subset of taps (possibly none: those
// pixels only receive the fused addend, or zero).  All classes run in ONE launch: a work item is (class, M tile, N tile).
struct ClsEntry {
  int M;                    // iteration pixels of this class (n_img * P_it * Q_it)
  int P_it, Q_it;           // iteration grid per image
  int ntaps, tap0;          // taps[tap0 .. tap0 + ntaps)
  int base_w, base_h;       // im2col coordinate of iteration pixel (p,q): base + q*step
  int oah, oaw;             // output pixel = (p*osh + oah, q*osw + oaw)
  int tile0, m_groups;      // first work item of the class; M tiles it has
};

struct FwdParams {
  int M, N;                 // iteration pixels (all classes), output channels
  int ncls;
  ClsEntry cls[kMaxCls];
  int cchunks;              // K loop = ntaps x cchunks blocks of 64 channels
  int a_mode;               // 0: tiled 2-D A[M, K];  1: im2col 4-D
  int step_w, step_h;
  long long out_img_pix;    // output pixels per image
  int out_row_pix;          // output pixels per row
  int osh, osw;
  int linear;               // output pixel index == iteration pixel index (single class, unit output stride)
  int ldc;                  // elements between consecutive output pixels
  int staged_store;         // 1: epilogue stages 32x64 sub-tiles in smem and writes them as full 128-byte rows
  __nv_bfloat16* out;
  const float* bias;
  const __nv_bfloat16* addend;   // optional: out = acc (+ bias) + addend[pixel][channel] (same layout as out)
  float* stats;                  // optional (linear output only): per-channel sum / sum of squares of the bf16 outputs
                                 // of every 32-row group, [ceil(M/128)*4][2][N] fp32 — BatchNorm statistics without
                                 // another pass over the activation (SURVEY.md §8(f) row 1)
  // BNB instantiation (dgrad whose output is the gradient of a BatchNorm+ReLU output, no residual): the epilogue turns dz into
  // g = dz * [y*scale + shift > 0] (the forward's own ReLU decision) and accumulates the BatchNorm backward sums of g
  const __nv_bfloat16* bn_y;     // the BatchNorm INPUT y (same layout as out)
  const float* bn_weight; const float* bn_bias; const float* bn_mean; const float* bn_invstd;   // per channel (weight / bias may be NULL)
  const uint32_t* kmask;         // optional K-block occupancy of the weight operand: [ceil(N/64)][kmask_words] bitmasks over
  int kmask_words;               // 64-column K blocks (tp_stage_weights); empty blocks are neither loaded nor multiplied
  TapEntry taps[kMaxTaps];
};

// The staging call leaves the number of empty blocks behind the last mask row: zero (any iid unstructured mask) means
// the K loop needs no per-block test at all.
__device__ __forceinline__ const uint32_t* live_kmask(const uint32_t* km, int words, int N) {
  if (km && __ldg(km + (size_t)((N + 63) >> 6) * words) == 0u) return nullptr;
  return km;
}

// Which K blocks of an output-channel tile hold any non-zero weight: the OR of the occupancy words of the tile's 64-row
// groups.  Producer and MMA thread walk the K loop with one of these each and must take identical decisions: both ask
// take().
struct KSkip {
  const uint32_t* base; int words, g0, g1; int cur_w; uint32_t bits;
  __device__ __forceinline__ void begin(const uint32_t* km, int wds, int n0, int block_n, int N) {
    base = km; words = wds; cur_w = -1; bits = 0u;
    g0 = n0 >> 6; g1 = min((min(n0 + block_n, N) + 63) >> 6, ((N + 63) >> 6));
  }
  __device__ __forceinline__ bool on(int kb) {
    const int wi = kb >> 5;
    if (wi != cur_w) {
      cur_w = wi; bits = 0u;
      if (wi < words) for (int g = g0; g < g1; ++g) bits |= __ldg(base + (size_t)g * words + wi);
      else bits = 0xffffffffu;                    // a block outside the mask (never produced by the staging kernels): dense
    }
    return (bits >> (kb & 31)) & 1u;
  }
  // process K block kb?  Yes when its bit is set, or when it is the tile's last block (`last`) and no block was
  // processed yet (`any`): the accumulator must be written at least once.
  __device__ __forceinline__ bool take(int kb, bool last, bool any) { return on(kb) || (last && !any); }
};

struct WgParams {
  int Mc;                   // Cout
  int Kpix;                 // contraction length = n_img * P_it * Q_it (dY pixels)
  int P_it, Q_it;
  int chunks, cchunks;      // N axis = chunks of 64 K-columns; chunk -> (tap = chunk / cchunks, cc = chunk % cchunks)
  int nb;                   // chunks per N tile (1..4)
  int b_mode;               // 0: tiled 2-D Xcol[pixels, Kcols];  1: im2col over X
  int base_w, base_h, step_w, step_h;
  int m_tiles, n_tiles, splits, kb_per_split, kblocks;
  float* partial;           // [m_tiles*n_tiles*splits][128][nb*64]
  const uint32_t* kmask;    // optional: the fprop occupancy mask of this layer's weights ([ceil(Cout/64)][kmask_words] bits over
  int kmask_words;          // 64-column blocks of (tap, cin)): an output tile whose blocks are all masked out is not computed
  TapEntry taps[kMaxTaps];
};

// wgrad work item: split `split` (K blocks kb0 .. kb1-1) of output tile `tile` = (m_t, n_t), which covers 128 output
// channels x the nvalid 64-column chunks from chunk0.
struct WgItem {
  int split, tile, m_t, n_t, chunk0, nvalid, kb0, kb1;
  // the output-tile part (nb chunks per N tile, `chunks` in all); the finalize kernel, which knows the tile directly,
  // uses it alone
  __device__ __forceinline__ void set_tile(int m, int n, int m_tiles, int nb, int chunks) {
    m_t = m; n_t = n; tile = n * m_tiles + m;
    chunk0 = n * nb; nvalid = min(nb, chunks - chunk0);
  }
  // true when every 64x64 block of the tile is empty in the occupancy mask, i.e. every mask entry under it is zero
  // (tp_stage_weights marks a block occupied as soon as one mask entry is non-zero) — dW = mask * (...) is zero there
  // whatever the activations are.  The producer, the consumers and the finalize kernel all skip such tiles.
  __device__ __forceinline__ bool empty(const uint32_t* __restrict__ km, int words, int Mc) const {
    const int row_groups = (Mc + 63) >> 6;
    for (int r = 2 * m_t; r < 2 * m_t + 2 && r < row_groups; ++r)
      for (int c = chunk0; c < chunk0 + nvalid; ++c)
        if ((__ldg(km + (size_t)r * words + (c >> 5)) >> (c & 31)) & 1u) return false;
    return true;
  }
};

// Work item -> WgItem (nb: chunks per N tile).  Split-major order: the CTAs running at the same time work on the SAME
// pixel range for different (m, n) tiles, so each X / dY chunk comes from HBM once and from L2 for the siblings
// (tile-major order re-reads them from HBM).
__device__ __forceinline__ WgItem wg_item(const WgParams& p, int nb, int item) {
  WgItem w;
  const int ntile = p.m_tiles * p.n_tiles;
  w.split = item / ntile;
  const int tile = item - w.split * ntile, n_t = tile / p.m_tiles;
  w.set_tile(tile - n_t * p.m_tiles, n_t, p.m_tiles, nb, p.chunks);
  w.kb0 = w.split * p.kb_per_split; w.kb1 = min(p.kblocks, w.kb0 + p.kb_per_split);
  return w;
}

__device__ __forceinline__ void decompose_pixel(int m, int P, int Q, int& n, int& p, int& q) {
  q = m % Q; int t = m / Q; p = t % P; n = t / P;
}

// ============================================================================================
struct AMaps { CUtensorMap m[kMaxCls]; };      // activation-side tensor map of every class

// work item -> (class, M tile, N tile); identical in both roles
__device__ __forceinline__ void decode_tile(const FwdParams& p, int tile, int n_tiles, int& c, int& m_g, int& n_t) {
  c = 0;
#pragma unroll
  for (int j = 1; j < kMaxCls; ++j) if (j < p.ncls && tile >= p.cls[j].tile0) c = j;
  const int local = tile - p.cls[c].tile0;
  m_g = local / n_tiles; n_t = local - m_g * n_tiles;     // m-major: CTAs running together share A tiles, weights stay in L2
}

// A K block of the fwd GEMM for one consumer warpgroup: D[128 x BLOCK_N] (+)= A[128 x 64] * B[BLOCK_N x 64]^T, both
// K-major; rows 0..63 accumulate into acc[0 .. BLOCK_N/2), rows 64..127 into acc[BLOCK_N/2 .. BLOCK_N).
// T = float: the same block as 32 fp32 channels per 128-B row, four TF32 k8 MMAs per 64-row half.
template <int BLOCK_N, typename T = __nv_bfloat16>
__device__ __forceinline__ void fwd_mma_block(float (&acc)[BLOCK_N], uint32_t a_addr, uint32_t b_addr, uint32_t accumulate) {
  const uint64_t adesc = make_smem_desc(a_addr, 16, 1024);
  const uint64_t adesc_hi = make_smem_desc(a_addr + 64 * kBlockK * 2, 16, 1024);
  const uint64_t bdesc = make_smem_desc(b_addr, 16, 1024);
#pragma unroll
  for (int k = 0; k < kBlockK / 16; ++k) {
    // advance 16 elements (32 B) along K inside the 128-B swizzle row: +2 in 16-B units
    if constexpr (sizeof(T) == 4) {           // 8 tf32 elements: also 32 B
      if constexpr (BLOCK_N == 128) {
        wgmma_m64n128_tf32(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
        wgmma_m64n128_tf32(acc + BLOCK_N / 2, adesc_hi + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
      } else {
        wgmma_m64n64_tf32(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
        wgmma_m64n64_tf32(acc + BLOCK_N / 2, adesc_hi + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
      }
    } else if constexpr (BLOCK_N == 128) {
      wgmma_m64n128<0, 0>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
      wgmma_m64n128<0, 0>(acc + BLOCK_N / 2, adesc_hi + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
    } else {
      wgmma_m64n64<0, 0>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
      wgmma_m64n64<0, 0>(acc + BLOCK_N / 2, adesc_hi + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), accumulate | (uint32_t)k);
    }
  }
}

// MULTI = false: one class of output pixels (fprop, stride-1 dgrad) — the class decode, the per-row destination
// arithmetic and the "class without taps" handling are compiled out.
//
// BNB = true (single class, linear output): the BatchNorm backward reduction of the layer that FEEDS this convolution is
// done here, in the dgrad epilogue, instead of by k_bn_bwd_reduce (one read of dz and one of y per such layer less, one
// launch less): after the bf16 gradient sub-tile has been staged, each lane re-reads it row-coalesced together with the
// matching y values, applies the ReLU gate, stores g and adds sum(g), sum(g * xhat) of its 8 channels x 8 rows; rows are
// then combined by the same fixed-order xor tree as the forward statistics.  Output: g, and [32-row group][2][N] partials.
//
// Ping-pong: the CTA's w-th work item belongs to consumer warpgroup w & 1.  The two mainloops take turns through a pair
// of mbarriers (order_bar): a consumer starts its K loop once the other one has issued the last MMA of the previous
// item, so the MMAs of one tile run while the other warpgroup drains its epilogue.  With the turn it hands over the
// position in the stage ring (stage, phase) where its K loop ended, so neither consumer has to count the K blocks of
// the other's items (dense walk, K-block skipping and classes without taps all hand over the same way).  Taking turns
// is also what keeps the ring consistent: a consumer only waits on stages whose earlier fills have all been consumed.
//
// Epilogue, per 64-column chunk: every thread converts its own accumulator fragments (+ bias, + addend, round to bf16)
// and writes them into the warpgroup's 128 x 64 bf16 staging tile (16-byte chunk j of row r at chunk j ^ (r & 7):
// conflict-free for the fragment stores and for the row reads); after a warpgroup barrier, warp q reads rows
// 32q .. 32q+31 back row-coalesced for full-line stores, the BatchNorm statistics and the BNB gate.
//
// T = float (TF32 mode): activations, weights and the output are fp32 (p.out points to float).  The stage ring is the
// same bytes: a 128-B swizzle row holds 32 fp32 instead of 64 bf16, so a K block is 32 channels and cchunks counts
// 32-channel blocks.  Operands are read by TMA as plain FLOAT32 (not the TFLOAT32 map type, which may round), and the
// tensor core truncates each to its upper 19 bits (tp_ptx.cuh).  No K-block skipping (dense walk).  The epilogue adds
// the bias and stores each thread's fragments directly: a quad of lanes writes two adjacent fp32 of 4 consecutive column
// pairs, i.e. one full 32-byte sector per row, so no staging tile is needed.  No statistics, BNB or addend epilogue:
// the fp32 model runs BatchNorm, ReLU and the residual add as separate fp32 ops.
template <int BLOCK_N, bool MULTI, bool BNB, typename T = __nv_bfloat16>
__global__ void __launch_bounds__(kFwdThreads, 1)
k_igemm_fwd(const __grid_constant__ AMaps tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ FwdParams p) {
  static_assert(BLOCK_N == 64 || BLOCK_N == 128, "wgmma N of the fwd kernel");
  static_assert(!BNB || !MULTI, "BatchNorm-backward epilogue: single class");
  constexpr bool kF32 = sizeof(T) == 4;
  static_assert(!kF32 || !BNB, "fp32 operands: no BatchNorm-backward epilogue");
  constexpr int kKe = 128 / (int)sizeof(T);                // channels of one K block: one 128-B swizzle row
  constexpr int kABytes = kBlockM * kBlockK * 2;           // 16 KB
  constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  constexpr int kStageBytes = kABytes + kBBytes;
  constexpr int kStages = fwd_stages(BLOCK_N);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  pdl_trigger();
  constexpr int kStgBytes = fwd_stg_bytes(BLOCK_N);
  constexpr int kChunkStg = kBlockM * 64 * 2;                         // one 64-column sub-tile of the staging tile
  uint8_t* const stg_base = smem + kStages * kStageBytes;             // one staging tile per consumer (1024-B aligned)
  uint64_t* full_bar = (uint64_t*)(stg_base + 2 * kStgBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* order_bar = empty_bar + kStages;                          // [consumer]: its turn to run a mainloop
  int* ring_pos = (int*)(order_bar + 2);                              // stage * 2 + phase handed over with the turn

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (p.N + BLOCK_N - 1) / BLOCK_N;
  // work items: (class) x (M tile) x (N tile), classes back to back
  const int total_tiles = p.cls[p.ncls - 1].tile0 + p.cls[p.ncls - 1].m_groups * n_tiles;
  const int my_items = total_tiles > (int)blockIdx.x ? (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  // the w-th work item of this CTA
  auto get_tile = [&](int w, int& ci, int& m_g, int& n_t) {
    ci = 0;
    const int tile = (int)blockIdx.x + w * (int)gridDim.x;
    if (MULTI) decode_tile(p, tile, n_tiles, ci, m_g, n_t);
    else { m_g = tile / n_tiles; n_t = tile - m_g * n_tiles; }   // m-major: CTAs running together share A tiles, weights stay in L2
  };

  if (threadIdx.x == 0) {
    for (int j = 0; j < p.ncls; ++j) prefetch_tmap(&tmA.m[j]);
    prefetch_tmap(&tmB);
    // empty: one arrival by the consumer warpgroup whose MMAs have read the stage
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 1); }
    mbar_init(&order_bar[0], 1); mbar_init(&order_bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // barrier set-up and descriptor prefetch above overlap the previous grid's tail; global memory from here on

  if (warp < 4) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<kFwdProducerRegs>();
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t* const km = kF32 ? nullptr : live_kmask(p.kmask, p.kmask_words, p.N);
      for (int w = 0; w < my_items; ++w) {
        int ci, m_g, n_t; get_tile(w, ci, m_g, n_t);
        const ClsEntry& ce = p.cls[MULTI ? ci : 0];
        const CUtensorMap* const mapA = &tmA.m[MULTI ? ci : 0];
        const int m0 = m_g * kBlockM;
        int cn = 0, cp = 0, cq = 0;
        if (p.a_mode == 1) decompose_pixel(m0, ce.P_it, ce.Q_it, cn, cp, cq);
        const int cw = ce.base_w + cq * p.step_w, ch = ce.base_h + cp * p.step_h;
        auto load_block = [&](const TapEntry& te, int cc) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * kStageBytes;
          uint8_t* sB = sA + kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          if (p.a_mode == 1)
            tma_load_im2col_4d(sA, mapA, &full_bar[stage], cc * kKe, cw, ch, cn, te.off_w, te.off_h);
          else
            tma_load_2d(sA, mapA, &full_bar[stage], te.kofs + cc * kKe, m0);
          tma_load_2d(sB, &tmB, &full_bar[stage], te.kofs + cc * kKe, n_t * BLOCK_N);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        };
        const int tap_base = MULTI ? ce.tap0 : 0;     // single class: a static table offset (no dependent parameter load)
        if (!km) {
          // dense walk — nested tap / channel-chunk loops: no integer division on the single producer thread
          for (int tap = 0; tap < ce.ntaps; ++tap) {
            const TapEntry te = p.taps[tap_base + tap];
            for (int cc = 0; cc < p.cchunks; ++cc) load_block(te, cc);
          }
        } else {
          // some weight blocks are empty: all-zero blocks are neither loaded nor multiplied
          KSkip ks; bool any = false;
          ks.begin(km, p.kmask_words, n_t * BLOCK_N, BLOCK_N, p.N);
          for (int tap = 0; tap < ce.ntaps; ++tap) {
            const TapEntry te = p.taps[tap_base + tap];
            for (int cc = 0; cc < p.cchunks; ++cc) {
              const bool last = tap == ce.ntaps - 1 && cc == p.cchunks - 1;
              if (!ks.take((te.kofs >> 6) + cc, last, any)) continue;
              any = true;
              load_block(te, cc);
            }
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers: MMA and epilogue of every other work item ------------------------------
    setmaxnreg_inc<kFwdConsumerRegs>();
    const int cw = (warp >> 2) - 1;           // consumer warpgroup: work items cw, cw + 2, cw + 4, ...
    const int q = warp & 3;                   // epilogue: rows 32q .. 32q+31 of the tile, one per lane
    const int wtid = threadIdx.x & 127;
    const int bar_id = 1 + cw;                // warpgroup-local named barrier
    const uint32_t* const km = kF32 ? nullptr : live_kmask(p.kmask, p.kmask_words, p.N);
    const uint32_t stg = smem_u32(stg_base + cw * kStgBytes);
    // fragment rows of this thread: fr0 + 8h + 64mh (h, mh in {0, 1}); their swizzle key (row & 7) is lane / 4
    const int fr0 = q * 16 + (lane >> 2);
    const uint32_t fsw = (uint32_t)(lane >> 2);
    const uint32_t frag_base = stg + (uint32_t)(fr0 * 128 + (lane & 3) * 4);
    // row-read geometry of this lane: rows r_in + 4i of the warp's 32, 16-byte column c16 of each 128-byte row
    const int r_in = lane >> 3, c16 = lane & 7;
    const uint32_t buf = stg + (uint32_t)(q * 32 * 128);
    const uint32_t rd_even = buf + r_in * 128 + ((uint32_t)(c16 ^ r_in) << 4);          // rows r_in + 8j
    const uint32_t rd_odd = buf + (r_in + 4) * 128 + ((uint32_t)(c16 ^ (r_in + 4)) << 4);  // rows r_in + 4 + 8j
    for (int it = 0, w = cw; w < my_items; ++it, w += 2) {
      int ci, m_g, n_t; get_tile(w, ci, m_g, n_t);
      const ClsEntry& ce = p.cls[MULTI ? ci : 0];
      const bool has_acc = MULTI ? ce.ntaps > 0 : true;   // a class no tap reaches: the accumulator was never written, its value is zero
      const int m_t = m_g;

      // ---- mainloop, in turn with the other consumer ----
      int stage = 0; uint32_t phase = 0;
      const int turn = it + cw;               // turns of this consumer before this item (item 0 needs none)
      if (turn > 0) {
        mbar_wait(&order_bar[cw], (uint32_t)((turn - 1) & 1));
        const int pos = *(volatile int*)ring_pos;
        stage = pos >> 1; phase = (uint32_t)(pos & 1);
      }
      // every warp of the warpgroup has taken its turn and read the ring position before one thread passes the turn on
      // (which rewrites the position and may let the other consumer complete the next phase of order_bar[cw]); the
      // MMAs do not order this: an item of one K block passes the turn before its MMA is known to be issued by all warps
      bar_sync(bar_id, 128);
      auto pass_turn = [&]() {
        if (wtid == 0) { *(volatile int*)ring_pos = stage * 2 + (int)phase; mbar_arrive(&order_bar[cw ^ 1]); }
      };
      float acc[BLOCK_N];
      if (has_acc) {
#pragma unroll
        for (int i = 0; i < BLOCK_N; ++i) acc[i] = 0.f;
        int prev = -1;                        // stage of the previous K block: freed once its MMAs have completed
        auto mma_block = [&](uint32_t accumulate) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t s_addr = smem_u32(smem + stage * kStageBytes);
          wgmma_fence();
          fwd_mma_block<BLOCK_N, T>(acc, s_addr, s_addr + kABytes, accumulate);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && wtid == 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        };
        // one walk with a single MMA call site (two would make ptxas serialise the wgmma pipeline)
        KSkip ks; uint32_t any = 0;
        if (km) ks.begin(km, p.kmask_words, n_t * BLOCK_N, BLOCK_N, p.N);
        for (int tap = 0; tap < ce.ntaps; ++tap) {
          const int kb0 = p.taps[(MULTI ? ce.tap0 : 0) + tap].kofs >> 6;
          for (int cc = 0; cc < p.cchunks; ++cc) {
            const bool last = tap == ce.ntaps - 1 && cc == p.cchunks - 1;
            if (km && !ks.take(kb0 + cc, last, any)) continue;
            mma_block(any);
            any = 1;
          }
        }
        pass_turn();                          // every MMA of this tile is issued: the other consumer's K loop may start
        wgmma_wait<0>();
        acc_fence(acc);
        if (prev >= 0 && wtid == 0) mbar_arrive(&empty_bar[prev]);
      } else {
        pass_turn();
      }

      // ---- epilogue ----
      const long long wrow0 = (long long)m_t * kBlockM + q * 32;        // first row of this warp's 32
      const int rows_left = (int)(ce.M - wrow0 < 32 ? (ce.M - wrow0 < 0 ? 0 : ce.M - wrow0) : 32);
      const long long ldc = p.ldc;
      const int N = p.N;
      // element offset of output row i (rows r_in + 4i): the iteration pixel itself for a single class; for parity classes
      // the destination pixel — ONE division chain for the first row, the other seven follow by stepping 4 pixels
      long long ooff[MULTI ? 8 : 1];
      const long long rbase = (wrow0 + r_in) * ldc + c16 * 8;
      if (MULTI && p.staged_store) {
        int n, pp, qq; decompose_pixel((int)(wrow0 + r_in), ce.P_it, ce.Q_it, n, pp, qq);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const long long px = (long long)n * p.out_img_pix + (long long)(pp * p.osh + ce.oah) * p.out_row_pix + (qq * p.osw + ce.oaw);
          ooff[i] = px * ldc + c16 * 8;
          qq += 4;
          while (qq >= ce.Q_it) { qq -= ce.Q_it; if (++pp == ce.P_it) { pp = 0; ++n; } }
        }
      }
      auto row_off = [&](int i) -> long long { return MULTI ? ooff[MULTI ? i : 0] : rbase + (long long)(i * 4) * ldc; };
      if constexpr (kF32) {
        // fp32 output: (+ bias) and direct stores of the fragments; a parity class no tap reaches is written as zeros
        float* const out = reinterpret_cast<float*>(p.out);
        const bool pair_ok = (p.ldc & 1) == 0 && (((uintptr_t)out) & 7) == 0;
#pragma unroll
        for (int mh = 0; mh < 2; ++mh)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m_t * kBlockM + fr0 + 8 * h + 64 * mh;
            if (row >= ce.M) continue;
            long long opix = row;
            if (MULTI || !p.linear) {
              int n, pp, qq; decompose_pixel(row, ce.P_it, ce.Q_it, n, pp, qq);
              opix = (long long)n * p.out_img_pix + (long long)(pp * p.osh + ce.oah) * p.out_row_pix + (qq * p.osw + ce.oaw);
            }
            float* const orow = out + opix * p.ldc;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
              const int n = n_t * BLOCK_N + 8 * j + 2 * (lane & 3);
              if (n >= N) continue;
              const int i = mh * (BLOCK_N / 2) + 4 * j + 2 * h;
              float f0 = has_acc ? acc[i] : 0.f, f1 = has_acc ? acc[i + 1] : 0.f;
              if (p.bias && has_acc) {
                f0 += p.bias[n];
                if (n + 1 < N) f1 += p.bias[n + 1];
              }
              if (n + 1 < N && pair_ok) *reinterpret_cast<float2*>(orow + n) = make_float2(f0, f1);
              else {
                orow[n] = f0;
                if (n + 1 < N) orow[n + 1] = f1;
              }
            }
          }
        continue;
      }
      if (MULTI && !has_acc) {
        // parity class no tap reaches (e.g. 3 of the 4 classes of a 1x1 stride-2 convolution): dX there is the fused addend
        // or zero — plain coalesced copies / stores
        if (p.staged_store) {
#pragma unroll 1
          for (int c = 0; c < BLOCK_N; c += 64) {
            const int n0 = n_t * BLOCK_N + c;
            if (n0 >= N) break;
            if (n0 + c16 * 8 + 8 > N) continue;
            uint4 z[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              z[i] = make_uint4(0u, 0u, 0u, 0u);
              if (p.addend && i * 4 + r_in < rows_left) z[i] = *reinterpret_cast<const uint4*>(p.addend + row_off(i) + n0);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (i * 4 + r_in < rows_left) *reinterpret_cast<uint4*>(p.out + row_off(i) + n0) = z[i];
          }
        } else {
          const int row = m_t * kBlockM + wtid;
          if (row < ce.M) {
            int n, pp, qq; decompose_pixel(row, ce.P_it, ce.Q_it, n, pp, qq);
            const long long opix = (long long)n * p.out_img_pix + (long long)(pp * p.osh + ce.oah) * p.out_row_pix + (qq * p.osw + ce.oaw);
            for (int j = n_t * BLOCK_N; j < min(p.N, (n_t + 1) * BLOCK_N); ++j)
              p.out[opix * p.ldc + j] = p.addend ? p.addend[opix * p.ldc + j] : __float2bfloat16_rn(0.f);
          }
        }
        continue;
      }
      if (p.staged_store) {
        // fragments -> bf16 staging tile -> coalesced global stores, so every output line leaves the SM as full 128-byte
        // rows instead of scattered 4-byte pieces.  The staging tile is addressed through the shared window (st/ld.shared,
        // not generic loads and stores, which are slower on shared memory).
        __nv_bfloat16* const gout = p.out;
        const __nv_bfloat16* const gadd = p.addend;
        const float* bias = p.bias;
        float* stats = p.stats ? p.stats + (long long)(m_t * 4 + q) * 2 * N + c16 * 8 : nullptr;
        if (gadd) {
          // addend tile, coalesced (8 lanes cover one 128-byte row, 4 rows per instruction), staged into the warp's own
          // 32 rows; the fragment pass below reads it back at its fragment positions
          __syncwarp();                       // the warp's row reads of the previous tile are done
#pragma unroll
          for (int ch = 0; ch < BLOCK_N / 64; ++ch) {
            const int n0 = n_t * BLOCK_N + ch * 64;
            if (n0 >= N) break;
            const bool col_ok = n0 + c16 * 8 + 8 <= N;
            uint4 a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              a[i] = make_uint4(0u, 0u, 0u, 0u);
              if (i * 4 + r_in < rows_left && col_ok) a[i] = *reinterpret_cast<const uint4*>(gadd + row_off(i) + n0);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) sts128(((i & 1) ? rd_odd : rd_even) + (uint32_t)(ch * kChunkStg + (i >> 1) * 1024), a[i]);
          }
        }
        // the staging tile is free (every warp has read the previous tile back) and the staged addend is visible
        bar_sync(bar_id, 128);
#pragma unroll
        for (int ch = 0; ch < BLOCK_N / 64; ++ch) {
          const int n0 = n_t * BLOCK_N + ch * 64;
          if (n0 >= N) break;
#pragma unroll
          for (int mh = 0; mh < 2; ++mh)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const int i = mh * (BLOCK_N / 2) + 4 * (ch * 8 + j) + 2 * h;
                float f0 = acc[i], f1 = acc[i + 1];
                const int n = n0 + 8 * j + 2 * (lane & 3);
                if (bias) {
                  if (n < N) f0 += bias[n];
                  if (n + 1 < N) f1 += bias[n + 1];
                }
                const uint32_t addr = frag_base + (uint32_t)(ch * kChunkStg + (64 * mh + 8 * h) * 128) + (((uint32_t)j ^ fsw) << 4);
                if (gadd) {       // fused skip-gradient accumulation, in fp32 before the one rounding to bf16
                  const uint32_t a = lds32(addr);
                  const float2 t2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a));
                  f0 += t2.x; f1 += t2.y;
                }
                const __nv_bfloat162 hv = __floats2bfloat162_rn(f0, f1);
                sts32(addr, *reinterpret_cast<const uint32_t*>(&hv));
              }
        }
        bar_sync(bar_id, 128);
#pragma unroll 1
        for (int ch = 0; ch < BLOCK_N / 64; ++ch) {
          const int n0 = n_t * BLOCK_N + ch * 64;
          if (n0 >= N) break;
          const bool col_ok = n0 + c16 * 8 + 8 <= N;
          // smem -> global, coalesced: 8 lanes write one full 128-byte output row, 4 rows per instruction.
          // Plain stores are fire-and-forget, so the staging tile is free again after this read-back
          // (a TMA store here would make every tile wait for the previous store to drain).
          uint4 o[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] = lds128(((i & 1) ? rd_odd : rd_even) + (uint32_t)(ch * kChunkStg + (i >> 1) * 1024));
          // per-channel sums of the row-coalesced view: this lane owns channels n0 + c16*8 .. +8 of rows r_in + 4i.
          // BNB: sum g and sum g * xhat of the gradient, gated before it is stored; otherwise (stats) the BatchNorm batch statistics sum o and
          // sum o^2 of exactly the values stored (bf16-rounded).  A fixed-order xor tree over the 4 row groups finishes
          // the 32 rows.
          float s1[8], s2[8];
#pragma unroll
          for (int qq = 0; qq < 8; ++qq) { s1[qq] = 0.f; s2[qq] = 0.f; }
          if (BNB) {
            uint4 yv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              yv[i] = make_uint4(0u, 0u, 0u, 0u);
              if (i * 4 + r_in < rows_left && col_ok) yv[i] = *reinterpret_cast<const uint4*>(p.bn_y + row_off(i) + n0);
            }
            float sc[8], sf[8], is_[8], nm[8];
            if (col_ok) {
              const int cb = n0 + c16 * 8;
#pragma unroll
              for (int qq = 0; qq < 8; qq += 4) {
                const float4 one4 = make_float4(1.f, 1.f, 1.f, 1.f), zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
                const float4 a4 = p.bn_weight ? *reinterpret_cast<const float4*>(p.bn_weight + cb + qq) : one4;
                const float4 b4 = p.bn_bias ? *reinterpret_cast<const float4*>(p.bn_bias + cb + qq) : zero4;
                const float4 m4 = *reinterpret_cast<const float4*>(p.bn_mean + cb + qq), i4 = *reinterpret_cast<const float4*>(p.bn_invstd + cb + qq);
                is_[qq] = i4.x; is_[qq + 1] = i4.y; is_[qq + 2] = i4.z; is_[qq + 3] = i4.w;
                nm[qq] = m4.x; nm[qq + 1] = m4.y; nm[qq + 2] = m4.z; nm[qq + 3] = m4.w;
                // scale / shift exactly as k_bn_finalize_stats computed them for the forward apply pass
                sc[qq] = a4.x * i4.x; sc[qq + 1] = a4.y * i4.y; sc[qq + 2] = a4.z * i4.z; sc[qq + 3] = a4.w * i4.w;
                sf[qq] = fmaf(-m4.x, sc[qq], b4.x); sf[qq + 1] = fmaf(-m4.y, sc[qq + 1], b4.y);
                sf[qq + 2] = fmaf(-m4.z, sc[qq + 2], b4.z); sf[qq + 3] = fmaf(-m4.w, sc[qq + 3], b4.w);
              }
            } else {
#pragma unroll
              for (int qq = 0; qq < 8; ++qq) { sc[qq] = 0.f; sf[qq] = 0.f; is_[qq] = 0.f; nm[qq] = 0.f; }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              if (i * 4 + r_in < rows_left) {
                __nv_bfloat162* gh = reinterpret_cast<__nv_bfloat162*>(&o[i]);
                const __nv_bfloat162* yh = reinterpret_cast<const __nv_bfloat162*>(&yv[i]);
#pragma unroll
                for (int qq = 0; qq < 4; ++qq) {
                  float2 d2 = __bfloat1622float2(gh[qq]);
                  const float2 y2 = __bfloat1622float2(yh[qq]);
                  // the forward wrote z = max(fma(y, scale, shift), 0): same expression, same operands -> same decision
                  if (!(fmaf(y2.x, sc[2 * qq], sf[2 * qq]) > 0.f)) d2.x = 0.f;
                  if (!(fmaf(y2.y, sc[2 * qq + 1], sf[2 * qq + 1]) > 0.f)) d2.y = 0.f;
                  gh[qq] = __floats2bfloat162_rn(d2.x, d2.y);                    // exact: d2 is a bf16 value or zero
                  s1[2 * qq] += d2.x;     s2[2 * qq] = fmaf(d2.x, (y2.x - nm[2 * qq]) * is_[2 * qq], s2[2 * qq]);
                  s1[2 * qq + 1] += d2.y; s2[2 * qq + 1] = fmaf(d2.y, (y2.y - nm[2 * qq + 1]) * is_[2 * qq + 1], s2[2 * qq + 1]);
                }
              }
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (i * 4 + r_in < rows_left && col_ok) *reinterpret_cast<uint4*>(gout + row_off(i) + n0) = o[i];
          if (!BNB && stats) {       // after the stores, so that they leave while the sums are computed
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              if (i * 4 + r_in < rows_left) {
                const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&o[i]);
#pragma unroll
                for (int qq = 0; qq < 4; ++qq) {
                  const float2 t2 = __bfloat1622float2(h2[qq]);
                  s1[2 * qq] += t2.x; s2[2 * qq] = fmaf(t2.x, t2.x, s2[2 * qq]);
                  s1[2 * qq + 1] += t2.y; s2[2 * qq + 1] = fmaf(t2.y, t2.y, s2[2 * qq + 1]);
                }
              }
            }
          }
          if (BNB || stats) {
#pragma unroll
            for (int qq = 0; qq < 8; ++qq) {
              s1[qq] += __shfl_xor_sync(0xffffffffu, s1[qq], 8);  s2[qq] += __shfl_xor_sync(0xffffffffu, s2[qq], 8);
              s1[qq] += __shfl_xor_sync(0xffffffffu, s1[qq], 16); s2[qq] += __shfl_xor_sync(0xffffffffu, s2[qq], 16);
            }
            if (r_in == 0 && col_ok) {
              float4* d1 = reinterpret_cast<float4*>(stats + n0);
              float4* d2 = reinterpret_cast<float4*>(stats + N + n0);
              d1[0] = make_float4(s1[0], s1[1], s1[2], s1[3]); d1[1] = make_float4(s1[4], s1[5], s1[6], s1[7]);
              d2[0] = make_float4(s2[0], s2[1], s2[2], s2[3]); d2[1] = make_float4(s2[4], s2[5], s2[6], s2[7]);
            }
          }
        }
      } else {
        // generic output mapping: every thread stores its own fragments (4 rows, 2 adjacent columns per 8)
#pragma unroll
        for (int mh = 0; mh < 2; ++mh)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m_t * kBlockM + fr0 + 8 * h + 64 * mh;
            if (row >= ce.M) continue;
            long long opix = row;
            if (MULTI || !p.linear) {
              int n, pp, qq; decompose_pixel(row, ce.P_it, ce.Q_it, n, pp, qq);
              opix = (long long)n * p.out_img_pix + (long long)(pp * p.osh + ce.oah) * p.out_row_pix + (qq * p.osw + ce.oaw);
            }
            __nv_bfloat16* const orow = p.out + opix * p.ldc;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int n = n_t * BLOCK_N + 8 * j + 2 * (lane & 3) + e;
                if (n >= N) continue;
                float f = acc[mh * (BLOCK_N / 2) + 4 * j + 2 * h + e];
                if (p.bias) f += p.bias[n];
                if (p.addend) f += __bfloat162float(p.addend[opix * p.ldc + n]);
                orow[n] = __float2bfloat16_rn(f);
              }
          }
      }
    }
  }
}

// ============================================================================================
// One warpgroup's share of a K block of the wgrad GEMM: D[64 x NB*64] (+)= dY^T[64 couts x 64 pixels] *
// Xcol[64 pixels x NB*64], both operands MN-major (64 MN elements per 128-B row, 8 pixel rows per 1024-B atom,
// 64-column chunks 8 KB apart).
template <int NB>
__device__ __forceinline__ void wgrad_mma_block(float (&acc)[NB * 32], uint32_t a_addr, uint32_t b_addr, bool first) {
  constexpr uint32_t kChunk = 64 * kBlockK * 2;
#pragma unroll
  for (int k = 0; k < kBlockK / 16; ++k) {
    // 16 K rows = 2 swizzle atoms = 2048 B
    const uint32_t acc_on = (!first || k > 0) ? 1u : 0u;
    const uint64_t adesc = make_smem_desc(a_addr + (uint32_t)(2048 * k), kChunk, 1024);
    const uint32_t bk = b_addr + (uint32_t)(2048 * k);
    if constexpr (NB >= 2) wgmma_m64n128<1, 1>(acc, adesc, make_smem_desc(bk, kChunk, 1024), acc_on);
    else wgmma_m64n64<1, 1>(acc, adesc, make_smem_desc(bk, kChunk, 1024), acc_on);
    if constexpr (NB == 4) wgmma_m64n128<1, 1>(acc + 64, adesc, make_smem_desc(bk + 2 * kChunk, kChunk, 1024), acc_on);
    if constexpr (NB == 3) wgmma_m64n64<1, 1>(acc + 64, adesc, make_smem_desc(bk + 2 * kChunk, kChunk, 1024), acc_on);
  }
}

template <int NB>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm_wgrad(const __grid_constant__ CUtensorMap tmA /* dY [Kpix, Cout] */,
              const __grid_constant__ CUtensorMap tmB /* X im2col or Xcol tiled */,
              const __grid_constant__ WgParams p) {
  constexpr int kABytes = kBlockM * kBlockK * 2;          // 2 boxes of [64 pixels x 64 couts] = 16 KB
  constexpr int kChunkBytes = 64 * kBlockK * 2;           // 8 KB per 64-column chunk
  constexpr int kMaxNb = 4;
  constexpr int kStageBytes = kABytes + kMaxNb * kChunkBytes;   // 48 KB
  constexpr int kStages = 4;
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int items = p.m_tiles * p.n_tiles * p.splits;
  constexpr int ncols = NB * 64;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA); prefetch_tmap(&tmB);
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumers / 128); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  const uint32_t* const km = live_kmask(p.kmask, p.kmask_words, p.Mc);     // null: no empty block anywhere (or no mask given)

  if (warp == kProducerWarp) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const WgItem it = wg_item(p, NB, item);
        if (km && it.empty(km, p.kmask_words, p.Mc)) continue;
        const int m_t = it.m_t, chunk0 = it.chunk0, nvalid = it.nvalid, kb0 = it.kb0, kb1 = it.kb1;
        // Everything that needs an integer division is hoisted out of the K loop (one producer thread
        // feeds the whole SM): per-chunk (tap, channel) coordinates once per item, and the pixel
        // coordinate of a K block advanced incrementally by 64 = sn*P*Q + sp*Q + sq.
        int c_c[4]; uint16_t c_ow[4], c_oh[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int chunk = min(chunk0 + j, p.chunks - 1), tap = chunk / p.cchunks;
          c_c[j] = (chunk - tap * p.cchunks) * 64; c_ow[j] = p.taps[tap].off_w; c_oh[j] = p.taps[tap].off_h;
        }
        int cn, cp, cq; decompose_pixel(kb0 * kBlockK, p.P_it, p.Q_it, cn, cp, cq);
        const int sq = kBlockK % p.Q_it, t1 = kBlockK / p.Q_it, sp = t1 % p.P_it, sn = t1 / p.P_it;
        for (int kb = kb0; kb < kb1; ++kb) {
          const int pix0 = kb * kBlockK;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], kABytes + nvalid * kChunkBytes);
          uint8_t* sA = smem + stage * kStageBytes;
          uint8_t* sB = sA + kABytes;
          tma_load_2d(sA, &tmA, &full_bar[stage], m_t * kBlockM, pix0);
          tma_load_2d(sA + kChunkBytes, &tmA, &full_bar[stage], m_t * kBlockM + 64, pix0);
          if (p.b_mode == 1) {
            const int cw = p.base_w + cq * p.step_w, ch = p.base_h + cp * p.step_h;
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (j < nvalid)
                tma_load_im2col_4d(sB + j * kChunkBytes, &tmB, &full_bar[stage], c_c[j], cw, ch, cn, c_ow[j], c_oh[j]);
            cq += sq; if (cq >= p.Q_it) { cq -= p.Q_it; cp += 1; }
            cp += sp; if (cp >= p.P_it) { cp -= p.P_it; cn += 1; }
            cn += sn;
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (j < nvalid) tma_load_2d(sB + j * kChunkBytes, &tmB, &full_bar[stage], (chunk0 + j) * 64, pix0);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    const int wg = warp >> 2;                 // rows (output channels) 64*wg .. 64*wg+63 of the tile
    int stage = 0; uint32_t phase = 0;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
      const WgItem it = wg_item(p, NB, item);
      if (km && it.empty(km, p.kmask_words, p.Mc)) continue;
      const int kb0 = it.kb0, kb1 = it.kb1;
      float acc[NB * 32];
#pragma unroll
      for (int i = 0; i < NB * 32; ++i) acc[i] = 0.f;
      int prev = -1;                          // stage of the previous K block: freed once its MMAs have completed
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * kStageBytes);
        wgmma_fence();
        wgrad_mma_block<NB>(acc, a_addr + (uint32_t)(wg * kChunkBytes), a_addr + kABytes, kb == kb0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      acc_fence(acc);
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      // fragments -> fp32 partial tile [128][ncols]: 4 lanes write 32 contiguous bytes of a row
      float* ptile = p.partial + ((long long)it.tile * p.splits + it.split) * kBlockM * ncols;
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < ncols / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float2*>(ptile + (long long)(r0 + 8 * h) * ncols + 8 * j + 2 * (lane & 3)) =
              make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}

// dW[co][ci][tap] (fp32 OIHW) = mask * sum_split partial   — fixed summation order (deterministic, no atomics).
// Grid (Cout, K chunks): a CTA owns KT = 256 / sl consecutive K columns (kk = tap*cin_p + ci) of one output channel;
// its 256 threads are KT k-lanes x `sl` split-lanes.  Split lane j folds splits j, j+sl, ... with eight independent
// loads in flight, the lanes are then combined in lane order.  (The first version looped over the K chunks inside one
// CTA per channel: 18 dependent rounds of L2/DRAM latency for a 3x3x64 layer.)
__global__ void __launch_bounds__(256) k_wgrad_finalize(const float* __restrict__ partial, const float* __restrict__ mask,
                                                        float* __restrict__ dw, int cout, int cin_real, int cin_p, int rs,
                                                        int nb, int m_tiles, int splits, int sl,
                                                        const uint32_t* __restrict__ kmask, int kmask_words) {
  pdl_enter();
  __shared__ float s_lane[256];
  const uint32_t* const km = live_kmask(kmask, kmask_words, cout);
  const int co = blockIdx.x;
  const int r = co % kBlockM;
  const int ktot = rs * cin_p;
  const int ncols = nb * 64;
  const int KT = 256 / sl;
  const int kl = threadIdx.x % KT, sj = threadIdx.x / KT;
  const int kk = blockIdx.y * KT + kl;
  const long long sstride = (long long)kBlockM * ncols;          // floats between consecutive splits of a tile
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  // a work item the GEMM skipped has no partials (the workspace holds whatever was there): its gradient is exactly zero
  bool skipped = false;
  if (kk < ktot) {
    const int chunk = kk >> 6;
    WgItem it; it.set_tile(co / kBlockM, chunk / nb, m_tiles, nb, (ktot + 63) >> 6);     // the tile holding (co, kk)
    skipped = km && it.empty(km, kmask_words, cout);
    if (!skipped) {
      const float* base = partial + (((long long)it.tile * splits) * kBlockM + r) * ncols + (chunk - it.chunk0) * 64 + (kk & 63);
      int sp = sj;
      for (; sp + 7 * sl < splits; sp += 8 * sl) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = __ldcs(base + (long long)(sp + j * sl) * sstride);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += v[j];
      }
      for (; sp < splits; sp += sl) a[0] += __ldcs(base + (long long)sp * sstride);
    }
  }
  s_lane[sj * KT + kl] = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]));
  __syncthreads();
  if (sj == 0 && kk < ktot) {
    float acc = 0.f;
    for (int j = 0; j < sl; ++j) acc += s_lane[j * KT + kl];
    const int tap = kk / cin_p, ci = kk - tap * cin_p;
    if (ci < cin_real) {
      const long long o = ((long long)co * cin_real + ci) * rs + tap;
      dw[o] = skipped ? 0.f : mask[o] * acc;
    }
  }
}

// db[c] = sum over pixels of dy[pix][c]  (bias gradient), dy bf16 [npix, ldc], c % 8 == 0.
// Two stages, both in fixed order (deterministic): every CTA of a (pixel split x channel tile) grid sums its pixels — a thread
// owns one 16-byte vector of 8 channels and walks the pixel axis, 4 rows in flight — into part[split][c]; a small kernel
// folds the splits.  (The first version ran ONE CTA per 32 channels over all pixels with 2-byte loads: most of the DeiT-S
// step.)
__global__ void __launch_bounds__(256) k_colsum_part(const __nv_bfloat16* __restrict__ dy, long long npix, int c, int ldc,
                                                     float* __restrict__ part) {
  pdl_enter();
  __shared__ float s_acc[256][9];
  const int tx = threadIdx.x, ty = threadIdx.y, TX = blockDim.x, TY = blockDim.y;
  const int cvec = blockIdx.y * TX + tx;
  const bool act = cvec * 8 < c;
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = 0.f;
  auto add8 = [&](const uint4& v) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); a[2 * i] += f.x; a[2 * i + 1] += f.y; }
  };
  if (act) {
    const long long stride = (long long)gridDim.x * TY;
    long long p = (long long)blockIdx.x * TY + ty;
    const __nv_bfloat16* src = dy + (size_t)cvec * 8;
    for (; p + 3 * stride < npix; p += 4 * stride) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const uint4*>(src + (size_t)(p + u * stride) * ldc);
#pragma unroll
      for (int u = 0; u < 4; ++u) add8(v[u]);
    }
    for (; p < npix; p += stride) add8(*reinterpret_cast<const uint4*>(src + (size_t)p * ldc));
  }
  const int tid = ty * TX + tx;
#pragma unroll
  for (int i = 0; i < 8; ++i) s_acc[tid][i] = a[i];
  __syncthreads();
  if (ty == 0 && act) {
    float r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = 0.f;
    for (int j = 0; j < TY; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) r[i] += s_acc[j * TX + tx][i];
#pragma unroll
    for (int i = 0; i < 8; ++i) part[(size_t)blockIdx.x * c + cvec * 8 + i] = r[i];
  }
}

__global__ void __launch_bounds__(256) k_colsum_fold(const float* __restrict__ part, int nparts, int c, float* __restrict__ db) {
  pdl_enter();
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int j = 0;
  for (; j + 3 < nparts; j += 4) {                    // four independent chains, combined in a fixed order
    s0 += part[(size_t)j * c + ch]; s1 += part[(size_t)(j + 1) * c + ch];
    s2 += part[(size_t)(j + 2) * c + ch]; s3 += part[(size_t)(j + 3) * c + ch];
  }
  for (; j < nparts; ++j) s0 += part[(size_t)j * c + ch];
  db[ch] = (s0 + s1) + (s2 + s3);
}

// ============================================================================================
// host side
// ============================================================================================
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                     const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encodeTiled = nullptr;
static PFN_encodeIm2col g_encodeIm2col = nullptr;
static int g_driver_version = 0;

static int load_driver_fns() {
  static std::once_flag once;
  static int rc = TP_OK;
  std::call_once(once, []() {
    void* f1 = nullptr; void* f2 = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f1, cudaEnableDefault, &q) != cudaSuccess || !f1 ||
        cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &f2, cudaEnableDefault, &q) != cudaSuccess || !f2) {
      set_last_cuda_error(cudaErrorUnknown, "cudaGetDriverEntryPoint(cuTensorMapEncode*)");
      rc = TP_ERR_CUDA;
      return;
    }
    g_encodeTiled = (PFN_encodeTiled)f1;
    g_encodeIm2col = (PFN_encodeIm2col)f2;
    cudaDriverGetVersion(&g_driver_version);
  });
  return rc;
}

static int fail_cu(CUresult r, const char* what) {
  static thread_local char buf[128];
  snprintf(buf, sizeof(buf), "%s -> CUresult %d", what, (int)r);
  set_last_cuda_error(cudaErrorInvalidValue, buf);
  return TP_ERR_CUDA;
}

// 2-D bf16 tensor [rows][cols] (cols contiguous, row stride ld elements), box = [box_rows][64 cols], SW128.
// f32: an fp32 tensor, box = [box_rows][32 cols] (the same 128-B rows).  FLOAT32, not TFLOAT32: the map type that rounds
// to tf32 on load is not used, the tensor core's truncation is the only operand rounding.
static int make_tiled_map(CUtensorMap* m, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_rows,
                          bool f32 = false) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * (f32 ? 4 : 2)};
  cuuint32_t box[2] = {f32 ? 32u : 64u, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encodeTiled(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr),
                             dims, strides, box, es,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail_cu(r, "cuTensorMapEncodeTiled");
  return TP_OK;
}

// im2col map over NHWC bf16 [n][h][w][c]: `pixels` consecutive iteration positions x 64 channels.
// Iteration grid (P_it x Q_it per image) starts at (base_h, base_w) and advances by (step_h, step_w).
// f32: NHWC fp32, 32 channels per pixel row (128 B).
static int make_im2col_map(CUtensorMap* m, const void* ptr, int n, int h, int w, int c,
                           int base_w, int base_h, int step_w, int step_h, int P_it, int Q_it, uint32_t pixels, bool f32 = false) {
  const cuuint64_t es_b = f32 ? 4 : 2;
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)c * es_b, (cuuint64_t)w * c * es_b, (cuuint64_t)h * w * c * es_b};
  // bounding box: base positions run from `lower` while < extent + upper  =>  count = Q_it
  int lower[2] = {base_w, base_h};
  int upper[2] = {(Q_it - 1) * step_w + 1 + base_w - w, (P_it - 1) * step_h + 1 + base_h - h};
  cuuint32_t es[4] = {1, (cuuint32_t)step_w, (cuuint32_t)step_h, 1};
  CUresult r = g_encodeIm2col(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr),
                              dims, strides, lower, upper,
                              f32 ? 32 : 64, pixels, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail_cu(r, "cuTensorMapEncodeIm2col");
  // Driver quirk (CUDA <= 13.1 drivers, see CUTLASS copy_traits_sm90_im2col.hpp): for tensors
  // smaller than 128 KiB bit 21 of the second descriptor word must be cleared.
  if (g_driver_version <= 13010 && (size_t)n * h * w * c * es_b < 131072)
    reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
  return TP_OK;
}

// Geometry of a layer's wgrad GEMM: output tiles of 128 channels x nb 64-column chunks of K = (tap, cin), 64-pixel K
// blocks, and the largest split count pick_wgrad_splits() may choose.  The workspace size and the launch both derive
// from this one definition.
struct WgGeom {
  int chunks, nb, m_tiles, n_tiles, kblocks, smax;
  size_t partial_bytes(int splits) const { return (size_t)m_tiles * n_tiles * splits * kBlockM * nb * 64 * sizeof(float); }
};

static WgGeom wgrad_geom(const tp_conv_desc* d) {
  WgGeom g;
  g.chunks = (d->r * d->s * d->cin + 63) / 64;
  g.nb = g.chunks >= 4 ? 4 : g.chunks;
  g.m_tiles = (d->cout + kBlockM - 1) / kBlockM;
  g.n_tiles = (g.chunks + g.nb - 1) / g.nb;
  g.kblocks = (int)(((long long)d->n * d->p * d->q + 63) / 64);
  g.smax = (2 * sm_count()) / (g.m_tiles * g.n_tiles);
  if (g.smax > g.kblocks) g.smax = g.kblocks;
  if (g.smax < 1) g.smax = 1;
  return g;
}

// Split-K factor of the wgrad GEMM.  Every (tile, split) item costs its share of the K loop plus a fixed 128 x nb*64
// fp32 partial tile (written once, read once by the finalize pass), so the cheapest choice is the SMALLEST split
// count that reaches the minimal makespan over the persistent CTAs — not "as many as fit in two waves": at a per-GPU
// batch of 64 the partial tiles were most of the wgrad traffic (54 layers x ~300 items x 128 KB, twice).
static int pick_wgrad_splits(const WgGeom& g) {
  const int sms = sm_count();
  const int tiles = g.m_tiles * g.n_tiles, kblocks = g.kblocks, nb = g.nb;
  // Relative costs (only their ratios decide): a 64-pixel K block (48 KB of operands, one 128 x nb*64 x 64 MMA group),
  // storing one partial tile from the accumulator registers to global, and the finalize traffic of one partial tile.
  // These weights were calibrated on an earlier GPU generation (where the partial tile was drained through tensor memory)
  // and are NOT re-fitted for H100.  Checked on an H100 SXM (700 W) by sweeping the split count of every ResNet-50 wgrad
  // layer: the splits chosen here cost 7.6 % (batch 512) and 6.4 % (batch 64) more wgrad + finalize time than the best
  // split of each layer; the model fills exactly one wave, while the measured optima scatter around it.
  const double c_kb = 0.30;
  const double c_part = 0.33 * nb;
  const double c_fin = 0.013 * nb;
  int best = 1; double best_cost = 1e30;
  for (int s = 1; s <= g.smax; ++s) {
    const int kb = (kblocks + s - 1) / s;
    const int s_eff = (kblocks + kb - 1) / kb;      // no empty splits
    const long long items = (long long)tiles * s_eff;
    const long long waves = (items + sms - 1) / sms;
    const double cost = (double)waves * (kb * c_kb + c_part) + (double)items * c_fin;
    if (cost < best_cost - 1e-9) { best_cost = cost; best = s_eff; }
  }
  return best;
}

static bool is_plain_gemm(const tp_conv_desc* d) {
  return d->r == 1 && d->s == 1 && d->stride_h == 1 && d->stride_w == 1 && d->pad_h == 0 && d->pad_w == 0;
}

// tap table of a single-class walk over an R x S filter whose K axis is (r, s, c) with c < cin: tap (r, s) gathers at
// im2col offset (s, r) and starts at K column (r*S + s) * cin
static void fill_taps(TapEntry* taps, int R, int S, int cin) {
  for (int r = 0; r < R; ++r) for (int s = 0; s < S; ++s) {
    TapEntry& t = taps[r * S + s];
    t.off_w = (uint16_t)s; t.off_h = (uint16_t)r; t.kofs = (r * S + s) * cin;
  }
}

static int pick_block_n(long long m_tiles, int n) {
  // favour wide tiles (fewer re-reads of the activation tile), but keep the last wave full.  128 is the widest tile:
  // a consumer warpgroup holds the whole 128 x BLOCK_N tile in fp32 registers (128 per thread at BLOCK_N = 128).
  const int sms = sm_count();
  int best = 64; double best_score = -1;
  const int cands[2] = {128, 64};
  const double weight[2] = {1.0, 0.82};
  for (int i = 0; i < 2; ++i) {
    int bn = cands[i];
    if (bn > 64 && n <= bn / 2) continue;
    long long tiles = m_tiles * ((n + bn - 1) / bn);
    long long waves = (tiles + sms - 1) / sms;
    double eff = (double)tiles / (double)(waves * sms) * weight[i];
    if (eff > best_score) { best_score = eff; best = bn; }
  }
  return best;
}

constexpr int kSmemMax = 232448;                 // 227 KB: the per-CTA opt-in limit of sm_90

template <int BN, bool MULTI, bool BNB = false, typename T = __nv_bfloat16>
static int launch_fwd(const AMaps& a, const CUtensorMap& b, FwdParams& p, cudaStream_t st) {
  constexpr int smem = fwd_smem(BN);
  static_assert(smem <= kSmemMax, "fwd smem budget");
  const int n_tiles = (p.N + BN - 1) / BN;
  static bool attr_set = false;
  if (!attr_set) {
    TP_CUDA_CHECK(cudaFuncSetAttribute(k_igemm_fwd<BN, MULTI, BNB, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  // work items: per class, (M tiles) x (N tiles), classes back to back
  long long ctiles = 0;
  for (int c = 0; c < p.ncls; ++c) {
    p.cls[c].m_groups = (int)((p.cls[c].M + kBlockM - 1) / kBlockM);
    if (ctiles > 0x7fffffffll) return TP_ERR_UNSUPPORTED;
    p.cls[c].tile0 = (int)ctiles;
    ctiles += (long long)p.cls[c].m_groups * n_tiles;
  }
  if (ctiles > 0x7fffffffll || ctiles <= 0) return TP_ERR_UNSUPPORTED;
  const int grid = (int)(ctiles < sm_count() ? ctiles : sm_count());
  TP_CUDA_CHECK(launch(k_igemm_fwd<BN, MULTI, BNB, T>, dim3(grid), dim3(kFwdThreads), (size_t)smem, st, a, b, p));
  TP_LAUNCH_CHECK();
  return TP_OK;
}

static int run_fwd(const AMaps& a, const CUtensorMap& b, FwdParams& p, int bn, cudaStream_t st, bool f32 = false) {
  // 16-byte aligned output rows -> the epilogue stages 32x64 sub-tiles through smem and writes full 128-byte lines
  // (for any pixel mapping: a strided dgrad's parity classes compute the destination pixel of each row)
  p.linear = p.ncls == 1 && p.osh == 1 && p.osw == 1 && p.cls[0].oah == 0 && p.cls[0].oaw == 0 &&
             p.out_row_pix == p.cls[0].Q_it && p.out_img_pix == (long long)p.cls[0].P_it * p.cls[0].Q_it;
  if (f32) {
    // fp32 operands and output: bias only (no statistics, BatchNorm gate or addend), fragments stored directly
    if (p.stats || p.bn_y || p.addend || p.kmask) return TP_ERR_UNSUPPORTED;
    p.staged_store = 0;
    if (!p.linear) {
      if (bn == 128) return launch_fwd<128, true, false, float>(a, b, p, st);
      return launch_fwd<64, true, false, float>(a, b, p, st);
    }
    if (bn == 128) return launch_fwd<128, false, false, float>(a, b, p, st);
    return launch_fwd<64, false, false, float>(a, b, p, st);
  }
  p.staged_store = (p.ldc % 8 == 0 && p.N % 8 == 0 && (((uintptr_t)p.out) & 15) == 0 &&
                    (!p.addend || (((uintptr_t)p.addend) & 15) == 0)) ? 1 : 0;
  if (p.stats && !(p.staged_store && p.linear)) return TP_ERR_UNSUPPORTED;
  // the general-mapping instantiation only where it is needed: parity classes, or a single class whose output is not
  // the iteration order itself
  const bool multi = !p.linear;
  if (multi) {
    if (bn == 128) return launch_fwd<128, true>(a, b, p, st);
    return launch_fwd<64, true>(a, b, p, st);
  }
  if (p.bn_y) {      // BatchNorm-backward epilogue (needs the linear staged path; the caller checked the shapes)
    if (!p.staged_store || !p.stats) return TP_ERR_UNSUPPORTED;
    if (bn == 128) return launch_fwd<128, false, true>(a, b, p, st);
    return launch_fwd<64, false, true>(a, b, p, st);
  }
  if (bn == 128) return launch_fwd<128, false>(a, b, p, st);
  return launch_fwd<64, false>(a, b, p, st);
}

template <int NB>
static int launch_wgrad(int grid, const CUtensorMap& ta, const CUtensorMap& tb, const WgParams& p, cudaStream_t st) {
  constexpr int smem = 4 * (kBlockM * kBlockK * 2 + 4 * 64 * kBlockK * 2) + 1024 + 256;
  static bool attr_set = false;
  if (!attr_set) {
    TP_CUDA_CHECK(cudaFuncSetAttribute(k_igemm_wgrad<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  TP_CUDA_CHECK(launch(k_igemm_wgrad<NB>, dim3(grid), dim3(kThreads), (size_t)smem, st, ta, tb, p));
  TP_LAUNCH_CHECK();
  return TP_OK;
}

}  // namespace tp

using namespace tp;

extern "C" {

size_t tp_conv_workspace_bytes(const tp_conv_desc* d, int op) {
  if (!d) return 0;
  if (op != 2) return 256;
  // wgrad: split-K partial tiles at the largest split count pick_wgrad_splits() may choose
  const WgGeom g = wgrad_geom(d);
  return g.partial_bytes(g.smax) + 1024;
}

size_t tp_conv_stats_rows(const tp_conv_desc* d) {
  if (!d) return 0;
  const long long M = (long long)d->n * d->p * d->q;
  return (size_t)((M + kBlockM - 1) / kBlockM) * 4;
}

int tp_conv_fprop(const tp_conv_desc* d, const void* x, const void* wf, const void* bias_f32,
                  void* y, void* ws, size_t ws_bytes, void* stream) {
  return tp_conv_fprop_stats(d, x, wf, nullptr, bias_f32, y, nullptr, ws, ws_bytes, stream);
}

static int conv_fprop_impl(const tp_conv_desc* d, const void* x, const void* wf, const void* kmask_f, const void* bias_f32,
                           void* y, void* stats, void* stream, bool f32);

int tp_conv_fprop_stats(const tp_conv_desc* d, const void* x, const void* wf, const void* kmask_f, const void* bias_f32,
                        void* y, void* stats, void* ws, size_t ws_bytes, void* stream) {
  (void)ws; (void)ws_bytes;
  return conv_fprop_impl(d, x, wf, kmask_f, bias_f32, y, stats, stream, false);
}

int tp_conv_fprop_f32(const tp_conv_desc* d, const void* x, const void* wf, const void* bias_f32, void* y, void* stream) {
  return conv_fprop_impl(d, x, wf, nullptr, bias_f32, y, nullptr, stream, true);
}

static int conv_fprop_impl(const tp_conv_desc* d, const void* x, const void* wf, const void* kmask_f, const void* bias_f32,
                           void* y, void* stats, void* stream, bool f32) {
  if (!d || !x || !wf || !y) return TP_ERR_INVALID;
  if (stats && (d->cout % 8 != 0 || (((uintptr_t)y) & 15) != 0 || (((uintptr_t)stats) & 15) != 0)) return TP_ERR_UNSUPPORTED;
  if (d->cin % 8 != 0 || d->r * d->s > kMaxTaps) return TP_ERR_UNSUPPORTED;
  if (d->r * d->s > 1 && d->cin % 64 != 0) return TP_ERR_UNSUPPORTED;
  int rc = load_driver_fns(); if (rc) return rc;
  rc = bind_device_of(d ? (const void*)x : nullptr); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FwdParams p = {};
  p.M = d->n * d->p * d->q; p.N = d->cout;
  p.ncls = 1;
  ClsEntry& ce = p.cls[0];
  ce.M = p.M; ce.P_it = d->p; ce.Q_it = d->q; ce.ntaps = d->r * d->s; ce.tap0 = 0; ce.oah = 0; ce.oaw = 0;
  const int ke = f32 ? 32 : 64;                  // channels per K block
  p.cchunks = (d->cin + ke - 1) / ke;
  p.out_img_pix = (long long)d->p * d->q; p.out_row_pix = d->q;
  p.osh = 1; p.osw = 1;
  p.ldc = d->cout; p.out = (__nv_bfloat16*)y; p.bias = (const float*)bias_f32;
  p.stats = (float*)stats;
  p.kmask = (const uint32_t*)kmask_f; p.kmask_words = (int)tp_kblock_mask_words((int64_t)d->r * d->s * d->cin);
  fill_taps(p.taps, d->r, d->s, d->cin);
  AMaps ta; CUtensorMap tb;
  if (is_plain_gemm(d)) {
    p.a_mode = 0;
    rc = make_tiled_map(&ta.m[0], x, (uint64_t)d->cin, (uint64_t)p.M, (uint64_t)d->cin, kBlockM, f32); if (rc) return rc;
  } else {
    p.a_mode = 1;
    ce.base_w = -d->pad_w; ce.base_h = -d->pad_h; p.step_w = d->stride_w; p.step_h = d->stride_h;
    rc = make_im2col_map(&ta.m[0], x, d->n, d->h, d->w, d->cin, ce.base_w, ce.base_h, p.step_w, p.step_h, d->p, d->q, kBlockM, f32);
    if (rc) return rc;
  }
  for (int c = 1; c < kMaxCls; ++c) ta.m[c] = ta.m[0];
  const int bn = pick_block_n((p.M + kBlockM - 1) / kBlockM, p.N);
  rc = make_tiled_map(&tb, wf, (uint64_t)d->r * d->s * d->cin, (uint64_t)d->cout, (uint64_t)d->r * d->s * d->cin, (uint32_t)bn, f32);
  if (rc) return rc;
  return run_fwd(ta, tb, p, bn, st, f32);
}

struct BnGate { const void* y; const float* weight; const float* bias; const float* mean; const float* invstd; float* partial; };

static int conv_dgrad_impl(const tp_conv_desc* d, const void* dy, const void* wd, const void* kmask_d, const void* addend,
                           void* dx, const BnGate* gate, void* stream, bool f32 = false);

int tp_conv_dgrad(const tp_conv_desc* d, const void* dy, const void* wd, const void* kmask_d, const void* addend,
                  void* dx, void* ws, size_t ws_bytes, void* stream) {
  (void)ws; (void)ws_bytes;
  return conv_dgrad_impl(d, dy, wd, kmask_d, addend, dx, nullptr, stream);
}

int tp_conv_dgrad_f32(const tp_conv_desc* d, const void* dy, const void* wd, void* dx, void* stream) {
  return conv_dgrad_impl(d, dy, wd, nullptr, nullptr, dx, nullptr, stream, true);
}

int tp_conv_dgrad_bnrelu(const tp_conv_desc* d, const void* dy, const void* wd, const void* kmask_d,
                         const void* bn_y, const void* bn_weight, const void* bn_bias, const void* bn_mean, const void* bn_invstd,
                         void* g, void* partial, void* stream) {
  if (!d || !bn_y || !bn_mean || !bn_invstd || !partial) return TP_ERR_INVALID;
  if (d->stride_h != 1 || d->stride_w != 1 || d->cin % 8 != 0) return TP_ERR_UNSUPPORTED;
  if ((((uintptr_t)bn_y) | ((uintptr_t)bn_weight) | ((uintptr_t)bn_bias) | ((uintptr_t)bn_mean) | ((uintptr_t)bn_invstd) | ((uintptr_t)partial)) & 15)
    return TP_ERR_UNSUPPORTED;
  BnGate bn = {bn_y, (const float*)bn_weight, (const float*)bn_bias, (const float*)bn_mean, (const float*)bn_invstd, (float*)partial};
  return conv_dgrad_impl(d, dy, wd, kmask_d, nullptr, g, &bn, stream);
}

size_t tp_conv_dgrad_partial_rows(const tp_conv_desc* d) {
  if (!d) return 0;
  const long long M = (long long)d->n * d->h * d->w;
  return (size_t)((M + kBlockM - 1) / kBlockM) * 4;
}

static int conv_dgrad_impl(const tp_conv_desc* d, const void* dy, const void* wd, const void* kmask_d, const void* addend,
                           void* dx, const BnGate* gate, void* stream, bool f32) {
  if (!d || !dy || !wd || !dx) return TP_ERR_INVALID;
  // here the contraction runs over (r', s', cout): channel count of dY must be TMA friendly
  const int cop = d->cout;                       // caller passes dY with cout % 8 == 0 (padded if needed)
  if (cop % 8 != 0 || d->r * d->s > kMaxTaps) return TP_ERR_UNSUPPORTED;
  if (d->r * d->s > 1 && cop % 64 != 0) return TP_ERR_UNSUPPORTED;
  int rc = load_driver_fns(); if (rc) return rc;
  rc = bind_device_of(d ? (const void*)dy : nullptr); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int R = d->r, S = d->s;
  const long long ktot = (long long)R * S * cop;
  const int sh = d->stride_h, sw = d->stride_w;
  FwdParams p = {};
  p.N = d->cin;
  p.cchunks = f32 ? (cop + 31) / 32 : (cop + 63) / 64;
  p.out_img_pix = (long long)d->h * d->w; p.out_row_pix = d->w;
  p.ldc = d->cin; p.out = (__nv_bfloat16*)dx; p.bias = nullptr; p.addend = (const __nv_bfloat16*)addend;
  p.kmask = (const uint32_t*)kmask_d; p.kmask_words = (int)tp_kblock_mask_words(ktot);
  p.step_w = 1; p.step_h = 1;
  if (gate) {
    p.bn_y = (const __nv_bfloat16*)gate->y; p.bn_weight = gate->weight; p.bn_bias = gate->bias; p.bn_mean = gate->mean; p.bn_invstd = gate->invstd;
    p.stats = gate->partial;
  }
  AMaps ta; CUtensorMap tb;
  if (sh == 1 && sw == 1) {
    // dX = conv(dY, rot180(W)^T) with padding (R-1-pad): wd is stored already rotated
    p.M = d->n * d->h * d->w;
    p.ncls = 1; p.osh = 1; p.osw = 1;
    ClsEntry& ce = p.cls[0];
    ce.M = p.M; ce.P_it = d->h; ce.Q_it = d->w; ce.ntaps = R * S; ce.tap0 = 0; ce.oah = 0; ce.oaw = 0;
    fill_taps(p.taps, R, S, cop);
    if (is_plain_gemm(d)) {
      p.a_mode = 0;
      rc = make_tiled_map(&ta.m[0], dy, (uint64_t)cop, (uint64_t)p.M, (uint64_t)cop, kBlockM, f32); if (rc) return rc;
    } else {
      p.a_mode = 1;
      ce.base_w = -(S - 1 - d->pad_w); ce.base_h = -(R - 1 - d->pad_h);
      rc = make_im2col_map(&ta.m[0], dy, d->n, d->p, d->q, cop, ce.base_w, ce.base_h, 1, 1, d->h, d->w, kBlockM, f32);
      if (rc) return rc;
    }
    for (int c = 1; c < kMaxCls; ++c) ta.m[c] = ta.m[0];
  } else {
    // strided conv: dX splits into stride_h x stride_w parity classes; each class is a stride-1 gather over dY with its
    // own subset of taps, written to every stride-th pixel.  ONE launch covers all classes (no memset / memcpy of dX,
    // no launch per class with scattered 16-byte stores); a class
    // no tap reaches is written by the epilogue alone (the fused addend, or zero).
    if (sh * sw > kMaxCls || R * S > kMaxTaps) return TP_ERR_UNSUPPORTED;
    p.a_mode = 1; p.osh = sh; p.osw = sw;
    int nc = 0, nt = 0; long long Mtot = 0;
    for (int a = 0; a < sh; ++a) for (int b = 0; b < sw; ++b) {
      const int Hc = (d->h - a + sh - 1) / sh, Wc = (d->w - b + sw - 1) / sw;   // pixels of this class
      if (Hc <= 0 || Wc <= 0) continue;
      ClsEntry& ce = p.cls[nc];
      ce.M = d->n * Hc * Wc; ce.P_it = Hc; ce.Q_it = Wc; ce.oah = a; ce.oaw = b; ce.tap0 = nt; ce.ntaps = 0;
      // taps: input row h = sh*h' + a receives dY row p = h' + (a + pad - r)/sh when divisible
      int dh_min = 1 << 30, dw_min = 1 << 30;
      for (int r = 0; r < R; ++r) if ((a + d->pad_h - r) % sh == 0) dh_min = min(dh_min, (a + d->pad_h - r) / sh);
      for (int s = 0; s < S; ++s) if ((b + d->pad_w - s) % sw == 0) dw_min = min(dw_min, (b + d->pad_w - s) / sw);
      if (dh_min != (1 << 30) && dw_min != (1 << 30)) {
        for (int r = 0; r < R; ++r) {
          if ((a + d->pad_h - r) % sh != 0) continue;
          for (int s = 0; s < S; ++s) {
            if ((b + d->pad_w - s) % sw != 0) continue;
            TapEntry& t = p.taps[nt++];
            t.off_h = (uint16_t)((a + d->pad_h - r) / sh - dh_min);
            t.off_w = (uint16_t)((b + d->pad_w - s) / sw - dw_min);
            t.kofs = ((R - 1 - r) * S + (S - 1 - s)) * cop;          // wd stores tap (r,s) at rotated position (R-1-r, S-1-s)
            ++ce.ntaps;
          }
        }
      } else { dh_min = 0; dw_min = 0; }
      ce.base_w = dw_min; ce.base_h = dh_min;
      rc = make_im2col_map(&ta.m[nc], dy, d->n, d->p, d->q, cop, ce.base_w, ce.base_h, 1, 1, Hc, Wc, kBlockM, f32); if (rc) return rc;
      Mtot += ce.M; ++nc;
    }
    if (nc == 0) return TP_OK;
    for (int c = nc; c < kMaxCls; ++c) ta.m[c] = ta.m[0];
    p.ncls = nc; p.M = (int)Mtot;
  }
  long long m_tiles = 0;
  for (int c = 0; c < p.ncls; ++c) m_tiles += (p.cls[c].M + kBlockM - 1) / kBlockM;
  const int bn = pick_block_n(m_tiles, p.N);
  rc = make_tiled_map(&tb, wd, (uint64_t)ktot, (uint64_t)d->cin, (uint64_t)ktot, (uint32_t)bn, f32); if (rc) return rc;
  return run_fwd(ta, tb, p, bn, st, f32);
}

int tp_conv_wgrad(const tp_conv_desc* d, const void* x, const void* dy, const void* mask, const void* kmask_f,
                  int cin_real, void* dw, void* db, void* ws, size_t ws_bytes, void* stream) {
  if (!d || !x || !dy || !mask || !dw || !ws) return TP_ERR_INVALID;
  if (d->cin % 8 != 0 || d->cout % 8 != 0 || d->r * d->s > kMaxTaps || cin_real > d->cin) return TP_ERR_UNSUPPORTED;
  if (d->r * d->s > 1 && d->cin % 64 != 0) return TP_ERR_UNSUPPORTED;
  int rc = load_driver_fns(); if (rc) return rc;
  rc = bind_device_of(d ? (const void*)x : nullptr); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int rs = d->r * d->s;
  WgParams p = {};
  p.Mc = d->cout;
  p.Kpix = d->n * d->p * d->q;
  p.P_it = d->p; p.Q_it = d->q;
  const WgGeom g = wgrad_geom(d);
  p.chunks = g.chunks;
  p.cchunks = (d->cin + 63) / 64;
  p.nb = g.nb;
  p.m_tiles = g.m_tiles;
  p.n_tiles = g.n_tiles;
  p.kblocks = g.kblocks;
  const int sms = sm_count();
  int splits = pick_wgrad_splits(g);
  p.kb_per_split = (p.kblocks + splits - 1) / splits;
  splits = (p.kblocks + p.kb_per_split - 1) / p.kb_per_split;     // no empty splits
  p.splits = splits;
  if (ws_bytes < g.partial_bytes(splits)) return TP_ERR_WORKSPACE;
  p.partial = (float*)ws;
  p.kmask = (const uint32_t*)kmask_f; p.kmask_words = (int)tp_kblock_mask_words((int64_t)rs * d->cin);
  fill_taps(p.taps, d->r, d->s, d->cin);
  CUtensorMap ta, tb;
  rc = make_tiled_map(&ta, dy, (uint64_t)d->cout, (uint64_t)p.Kpix, (uint64_t)d->cout, 64); if (rc) return rc;
  if (is_plain_gemm(d)) {
    p.b_mode = 0;
    rc = make_tiled_map(&tb, x, (uint64_t)d->cin, (uint64_t)p.Kpix, (uint64_t)d->cin, 64); if (rc) return rc;
  } else {
    p.b_mode = 1;
    p.base_w = -d->pad_w; p.base_h = -d->pad_h; p.step_w = d->stride_w; p.step_h = d->stride_h;
    rc = make_im2col_map(&tb, x, d->n, d->h, d->w, d->cin, p.base_w, p.base_h, p.step_w, p.step_h, d->p, d->q, 64);
    if (rc) return rc;
  }
  const int items = p.m_tiles * p.n_tiles * splits;
  const int grid = items < sms ? items : sms;
  switch (p.nb) {
    case 1: rc = launch_wgrad<1>(grid, ta, tb, p, st); break;
    case 2: rc = launch_wgrad<2>(grid, ta, tb, p, st); break;
    case 3: rc = launch_wgrad<3>(grid, ta, tb, p, st); break;
    default: rc = launch_wgrad<4>(grid, ta, tb, p, st); break;
  }
  if (rc) return rc;
  // split lanes only pay when there are many splits (skinny layers); wide-K layers keep all 256 threads on K
  const int sl = splits >= 64 ? 8 : (splits >= 32 ? 4 : (splits >= 16 ? 2 : 1));
  const int fin_kt = 256 / sl;
  launch(k_wgrad_finalize, dim3(d->cout, (rs * d->cin + fin_kt - 1) / fin_kt), 256, 0, st,
      p.partial, (const float*)mask, (float*)dw, d->cout, cin_real, d->cin, rs, p.nb, p.m_tiles, splits, sl,
      p.kmask, p.kmask_words);
  TP_LAUNCH_CHECK();
  if (db) {
    // the split-K partials are dead once the finalize above has run (same stream): the workspace holds the column partials now
    const int c = d->cout, cv = c / 8;
    int tx = 1;
    while (tx < cv && tx < 256) tx <<= 1;
    const int ty = 256 / tx, ctiles = (cv + tx - 1) / tx;
    long long gx = ((long long)p.Kpix + (long long)ty * 4 - 1) / ((long long)ty * 4);          // >= 4 pixel rows per thread
    const long long want = (long long)sms * 4 / ctiles, fit = (long long)(ws_bytes / ((size_t)c * sizeof(float)));
    if (gx > want) gx = want;
    if (gx > fit) gx = fit;
    if (gx < 1) gx = 1;
    if ((((uintptr_t)dy) & 15) != 0) return TP_ERR_INVALID;
    launch(k_colsum_part, dim3((unsigned)gx, (unsigned)ctiles), dim3(tx, ty), 0, st, (const __nv_bfloat16*)dy, (long long)p.Kpix, c, c, (float*)ws);
    launch(k_colsum_fold, (c + 255) / 256, 256, 0, st, (const float*)ws, (int)gx, c, (float*)db);
    TP_LAUNCH_CHECK();
  }
  return TP_OK;
}

}  // extern "C"
