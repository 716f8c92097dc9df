"""The mask top-k (k_topk_fused and its exact fallback) at training extents, bit for bit against an exact CPU selection.

The oracle is oracle/prune.py: scores are single IEEE fp32 multiplies (they round exactly as on the GPU), the k-th
smallest is np.partition on sortable keys and the mask is ``score <= thr``.  The threshold bits (any NaN matches any
NaN) and every mask element must be equal; there is no tolerance, a selection is either exact or wrong.

The kernel reaches its result along one of several paths: a candidate list staged in shared memory that may spill to
global memory, a one- or two-level radix resolve (shift0 = 0, 11 or 22), the ``thr = lo`` shortcut, an exact 3-pass
radix fallback with three separate triggers, and the host's apply pass for a NaN threshold.  Most of them only occur at
extents or in data shapes that small tests never build, so every call here also

- decodes the selection state the fused kernel left in the workspace (``ops.topk_state``, read before ``finish``,
  whose fallback rewrites it) and names the path it took;
- compares that state with a mirror of the host planning and of the kernel's bracket (``topk_plan``,
  ``sample_positions``, ``predict_state``): the coarse sample histogram, both bracket bins, lo / hi, the three counters
  and the second-level list size must be equal, so a recipe that stops reaching its path fails instead of quietly
  testing something easier.

The last test asserts that the union of the paths reached is the full list ``BRANCHES``.
"""
import math
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import prune as P

gpu = pytest.mark.gpu

MAG, SNIP, SYNFLOW = P.SCORE_MAG, P.SCORE_SNIP, P.SCORE_SYNFLOW
KRUN = 16                  # neighbouring elements per sample run (kRun)
SAMPLE_MAX = 1 << 20       # 2^kSampleBits
TILE = 4096                # kTileElems: the sweep's work item, counted from each segment's start
SMEM_CAND = 2048           # kSmemCand: candidate staging per CTA
CAND2 = 4096               # kCand2: capacity of the second-level list
SMEM_SEGS = 128            # kSmemSegs: larger segment tables are searched in global memory
NAN_KEY = 0x7FFFFFFF       # the GPU's canonical NaN: every NaN score has this key
N25 = 25_000_000

BRANCHES = [
    "shift0 = 11",
    "shift0 = 22",
    "shift0 = 0",
    "thr = lo",
    "lo = 0",
    "candidate spill to global memory",
    "fallback: list over cap",
    "fallback: n_cand2 > 4096",
    "fallback: bracket above k",
    "fallback: bracket below k",
    "NaN threshold, fast path",
    "NaN threshold after a fallback",
    "+inf threshold",
    "subnormal threshold",
    "segment table in global memory",
    "misaligned operands (scalar sample / sweep)",
    "S == N = 2^20",
    "S = 2^20 < N",
    "write_masks=False",
]
REACHED = {}               # branch -> ids of the cases that reached it
RAN = set()                # ids of the cases that completed


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _release_memory():
    """Every case frees its tensors before the next one (the GPU is shared; the VGG-16-sized case holds 2.2 GB)."""
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


# ---------------------------------------------------------------- mirror of the host planning and the kernel state -----
def topk_plan(sizes, k):
    """enqueue_topk / cand_cap of tp_prune.cu.  S = min(N, 2^20, grid * 4096): the grid is occupancy (<= 4) x SMs CTAs,
    at least 3 x 132 on an H100 (80 registers, 41 KB of shared memory per CTA), so S never hits the grid term there;
    every GPU case checks that through the size of the coarse sample histogram."""
    N = int(sum(sizes))
    S = min(N, SAMPLE_MAX)
    rs = min(max((k * S + N - 1) // N, 1), S)
    pq = rs / S
    delta = int(6.0 * math.sqrt(S * pq * (1.0 - pq)) + 8.0) + KRUN * len(sizes)
    return SimpleNamespace(N=N, S=S, rs=rs, delta=delta, r_lo=rs - delta, r_hi=rs + delta,
                           cap=min(max(N // 8, 1 << 16), 1 << 23), seg_smem=len(sizes) <= SMEM_SEGS)


def sample_positions(sizes):
    """Global indices of the elements P0 reads: G = ceil(S / 16) runs, run gi starts at e = gi * N // G, aligned down to
    16 inside its segment and clamped to (n - 16) & ~3 (or 0) at the segment's end; nvalid = min(16, n - l0, S - 16 gi).
    Clamped runs may repeat elements, exactly as the kernel's samples do."""
    sizes = np.asarray(sizes, dtype=np.int64)
    N = int(sizes.sum())
    S = min(N, SAMPLE_MAX)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    G = -(-S // KRUN)
    gi = np.arange(G, dtype=np.int64)
    e = gi * N // G
    si = np.searchsorted(starts, e, side="right") - 1         # find_seg_by_elem: the last segment starting at or before e
    n, st = sizes[si], starts[si]
    l0 = (e - st) & ~np.int64(KRUN - 1)
    l0 = np.where(l0 + KRUN > n, np.where(n >= KRUN, (n - KRUN) & ~np.int64(3), 0), l0)
    nvalid = np.minimum(np.minimum(KRUN, n - l0), S - KRUN * gi)
    u = np.arange(KRUN)
    return ((st + l0)[:, None] + u[None, :])[u[None, :] < nvalid[:, None]]


def raw_keys(scores):
    """The kernel's keys: the bit patterns of the non-negative scores, every NaN as the canonical 0x7fffffff."""
    k = np.concatenate([np.ascontiguousarray(s, dtype=np.float32).reshape(-1).view(np.uint32) for s in scores])
    k[k > np.uint32(0x7F800000)] = np.uint32(NAN_KEY)
    return k


def resolve_shift0(lo, hi):
    span = lo ^ ((hi - 1) & 0xFFFFFFFF)
    return ((span.bit_length() - 1) // 11) * 11 if span else 0


def _find_rank(h, rank):
    """block_find_rank: the smallest bin whose inclusive cumulative count reaches rank, and the count before it."""
    c = np.cumsum(h, dtype=np.int64)
    if rank < 1 or rank > c[-1]:
        return 0, 0
    b = int(np.searchsorted(c, rank, side="left"))
    return b, int(c[b] - h[b])


def predict_state(keys, sizes, k):
    """What k_topk_fused must leave in SelState for these keys (P0-P4), plus the largest number of candidates one sweep
    tile holds (more than kSmemCand forces the spill to global memory)."""
    pl = topk_plan(sizes, k)
    sk = keys[sample_positions(sizes)]
    coarse = sk >> np.uint32(20)
    hc = np.bincount(coarse, minlength=2048)
    rlo, rhi = max(pl.r_lo, 1), min(pl.r_hi, pl.S)
    c_lo, b_lo = _find_rank(hc, rlo)
    c_hi, b_hi = _find_rank(hc, rhi)
    f_lo = np.bincount((sk[coarse == c_lo] >> np.uint32(9)) & np.uint32(2047), minlength=2048)
    f_hi = np.bincount((sk[coarse == c_hi] >> np.uint32(9)) & np.uint32(2047), minlength=2048)
    lo = (c_lo << 20) | (_find_rank(f_lo, rlo - b_lo)[0] << 9)
    hi = ((((c_hi << 11) | _find_rank(f_hi, rhi - b_hi)[0]) + 1) << 9) & 0xFFFFFFFF
    if pl.r_lo < 1:
        lo = 0
    if pl.r_hi > pl.S or hi > 0x80000000 or hi == 0:
        hi = 0x80000000
    lo32, hi32 = np.uint32(lo), np.uint32(hi)
    inside = (keys > lo32) & (keys < hi32)
    n_lt, n_eq, n_cand = int(np.count_nonzero(keys < lo32)), int(np.count_nonzero(keys == lo32)), int(np.count_nonzero(inside))
    fallback = k <= n_lt or n_cand > pl.cap or k > n_lt + n_eq + n_cand
    n_cand2 = 0
    if not fallback and k > n_lt + n_eq:
        shift0 = resolve_shift0(lo, hi)
        if shift0 > 0:
            ck = keys[inside]
            d, _ = _find_rank(np.bincount((ck >> np.uint32(shift0)) & np.uint32(2047), minlength=2048), k - n_lt - n_eq)
            prefix = (0 if shift0 + 11 >= 32 else lo & ((0xFFFFFFFF << (shift0 + 11)) & 0xFFFFFFFF)) | (d << shift0)
            n_cand2 = int(np.count_nonzero((ck & np.uint32((0xFFFFFFFF << shift0) & 0xFFFFFFFF)) == np.uint32(prefix)))
            fallback = n_cand2 > CAND2
    tile_max, off = 0, 0
    for n in sizes:
        x = inside[off:off + n]
        if n:
            pad = np.zeros(-(-n // TILE) * TILE, dtype=np.int32)
            pad[:n] = x
            tile_max = max(tile_max, int(pad.reshape(-1, TILE).sum(1).max()))
        off += n
    return dict(plan=pl, n_samples=int(sk.size), hist_c=hc, c_lo=c_lo, c_hi=c_hi, before_lo=b_lo, before_hi=b_hi, lo=lo,
                hi=hi, n_lt=n_lt, n_eq=n_eq, n_cand=n_cand, n_cand2=n_cand2, fallback=fallback, tile_max=tile_max)


def kth_many(flat, ks):
    """The k-th smallest for several k from one np.partition on P.sortable_key (P.kth_smallest, vectorised over k)."""
    keys = P.sortable_key(flat)
    part = np.partition(keys, [k - 1 for k in ks])
    out = []
    for k in ks:
        kk = part[k - 1]
        if kk == np.uint32(0xFFFFFFFF):
            out.append(np.float32(np.nan))
            continue
        u = (kk ^ np.uint32(0x80000000)) if (kk & np.uint32(0x80000000)) else np.uint32(~kk)
        out.append(np.array([u], dtype=np.uint32).view(np.float32)[0])
    return out


def _same_thr(got, ref):
    got, ref = np.float32(got), np.float32(ref)
    return (np.isnan(got) and np.isnan(ref)) or got.view(np.uint32) == ref.view(np.uint32)


def _classify(st, info, k, thr, pred=None, keys=None):
    """The paths one call took, from the decoded state (and the host's info).  With ``pred`` the state must also equal
    the mirror's."""
    if pred is not None:
        assert int(st["hist"][:2048].sum()) == pred["n_samples"] and pred["n_samples"] <= pred["plan"].S
        assert np.array_equal(st["hist"][:2048].astype(np.int64), pred["hist_c"]), "coarse sample histogram"
        for f in ("c_lo", "c_hi", "before_lo", "before_hi", "lo", "hi", "n_lt", "n_eq", "n_cand", "n_cand2"):
            assert st[f] == pred[f], (f, st[f], pred[f])
        assert (st["status"] == 1) == pred["fallback"], (st["status"], pred["fallback"])
    assert info["path"] == (1 if st["status"] == 1 else 0)
    b = set()
    lo, n_lt, n_eq, n_cand = st["lo"], st["n_lt"], st["n_eq"], st["n_cand"]
    if st["status"] == 1:
        cap = topk_plan([1], 1).cap if pred is None else pred["plan"].cap
        if pred is not None and n_cand > cap:
            b.add("fallback: list over cap")
        if k <= n_lt:
            b.add("fallback: bracket above k")
        if k > n_lt + n_eq + n_cand:
            b.add("fallback: bracket below k")
        if not b and st["n_cand2"] > CAND2:
            b.add("fallback: n_cand2 > 4096")
        if info["nan_thr"]:
            b.add("NaN threshold after a fallback")
    else:
        assert st["status"] in (0, 2) and n_lt < k <= n_lt + n_eq + n_cand
        if k <= n_lt + n_eq:
            assert st["thr_key"] == lo
            b.add("thr = lo")
        else:
            b.add(f"shift0 = {resolve_shift0(lo, st['hi'])}")
        if lo == 0:
            b.add("lo = 0")
        if st["status"] == 2:
            assert info["nan_thr"]
            b.add("NaN threshold, fast path")
        if pred is not None and pred["tile_max"] > SMEM_CAND:
            b.add("candidate spill to global memory")
    bits = int(np.float32(thr).view(np.uint32))
    if bits == 0x7F800000:
        b.add("+inf threshold")
    if 0 < bits < 0x00800000:
        b.add("subnormal threshold")
    return b


def _record(case_id, branches):
    for x in branches:
        REACHED.setdefault(x, []).append(case_id)
    RAN.add(case_id)
    print(f"[topk] {case_id}: {', '.join(sorted(branches))}")


def _select(plan, k, ref_thr, scores, keys, sizes):
    """One call through TopKPlan: enqueue, read the state, finish; threshold and every mask element against the oracle."""
    plan.enqueue(k)
    torch.cuda.synchronize()
    st = plan.state()
    outs, thr, info = plan.finish(k)
    got = np.float32(thr.item())
    assert _same_thr(got, ref_thr), (k, got, ref_thr)
    for i, (o, s) in enumerate(zip(outs, scores)):
        assert np.array_equal(o.cpu().numpy().reshape(-1), P.apply_threshold(s, ref_thr)), (k, i)
    return _classify(st, info, k, got, predict_state(keys, sizes, k))


def test_plan_mirror_host_arithmetic():
    """The mirror against hand-derived values (no GPU)."""
    p = topk_plan([1 << 20], 1 << 19)
    assert (p.S, p.rs, p.delta, p.cap) == (1 << 20, 1 << 19, int(6 * 512 + 8) + 16, 1 << 17)
    p = topk_plan([25_000_000] * 2, 40_000_000)
    assert p.S == 1 << 20 and p.cap == 6_250_000 and p.delta == int(6 * math.sqrt((1 << 20) * 0.8 * 0.2) + 8) + 32
    assert topk_plan([1000], 10).cap == 1 << 16 and topk_plan([1 << 27], 1).cap == 1 << 23
    assert topk_plan([5], 5).r_hi > 5 and topk_plan([100], 1).r_lo < 1
    assert np.array_equal(sample_positions([1 << 20]), np.arange(1 << 20))                 # S == N: every element once
    sizes = [1, 3, 7, 15, 17, 4099, 1 << 20]
    pos = sample_positions(sizes)
    starts = np.concatenate([[0], np.cumsum(sizes)])
    assert pos.min() >= 0 and pos.max() < starts[-1] and pos.size <= 1 << 20
    seg = np.searchsorted(starts, pos, side="right") - 1
    for i, n in enumerate(sizes):                                                            # clamped runs stay inside
        inseg = pos[seg == i] - starts[i]
        assert inseg.size == 0 or (inseg.min() >= 0 and inseg.max() < n)
    keys = np.arange(1 << 20, dtype=np.uint32) * np.uint32(64)                               # distinct keys, no ties
    pr = predict_state(keys, [1 << 20], 1 << 19)
    assert not pr["fallback"] and pr["n_lt"] < (1 << 19) <= pr["n_lt"] + pr["n_eq"] + pr["n_cand"]
    assert pr["lo"] <= int(keys[(1 << 19) - 1]) < pr["hi"] and pr["lo"] % 512 == 0 and pr["hi"] % 512 == 0


# ---------------------------------------------------------------- recipes: one way to reach each path -------------------
def _g(seed):
    return torch.Generator().manual_seed(seed)


def _u(g, n, a, b):
    return torch.rand(n, generator=g, dtype=torch.float64).mul_(b - a).add_(a).float()


def _perm(g, x):
    return x[torch.randperm(x.numel(), generator=g)]


def _ones(ws):
    return [torch.ones_like(w) for w in ws]


def r_shift22():
    """Two clusters 18 octaves apart; k just inside the small upper one: the bracket spans both, so the top digit is
    bits [31:22] and two select digits follow over the few hundred candidates that share it."""
    g, nh = _g(1), 20_000
    w = _perm(g, torch.cat([_u(g, N25 - nh, 1e-3, 2e-3), _u(g, nh, 1e3, 2e3)]))
    return dict(kind=MAG, ws=[w], ks=[N25 - nh + 100], expect={"shift0 = 22"})


def r_shift0():
    """2 M values on 4096 consecutive ulps above 1.0 inside a wide population, k a quarter into them: lo and hi - 1 share
    every bit above 2^11, one digit (ties allowed) resolves the key."""
    g, nc = _g(2), 2_000_000
    nb = (N25 - nc) // 2
    cl = (torch.randint(0, 4096, (nc,), generator=g, dtype=torch.int32) + 0x3F800000).view(torch.float32)
    w = _perm(g, torch.cat([_u(g, nb, 0.0, 0.9), cl, _u(g, N25 - nc - nb, 1.1, 100.0)]))
    return dict(kind=MAG, ws=[w], ks=[nb + nc // 4], expect={"shift0 = 0"})


def r_ties_at_lo():
    """30 % of the scores are exactly 0.5 (a fine-bin edge: its low key bits are zero) and k falls inside them."""
    g, nt = _g(3), int(0.3 * N25)
    w = _perm(g, torch.cat([torch.full((nt,), 0.5), _u(g, N25 - nt, 0.0, 1.0)]))
    return dict(kind=MAG, ws=[w], ks=[N25 // 2], expect={"thr = lo"})


def r_sorted():
    """One sorted segment: the candidates are contiguous, whole sweep tiles of them."""
    g = _g(4)
    w = torch.sort(torch.randn(N25, generator=g).abs_() * 0.05).values
    return dict(kind=MAG, ws=[w], ks=[N25 // 2, N25 // 10], expect={"candidate spill to global memory"})


def r_ties_over_cap():
    """20 % of the scores equal 0.3 (not a bin edge): all of them are candidates, more than the list holds."""
    g, nt = _g(5), N25 // 5
    w = _perm(g, torch.cat([torch.full((nt,), 0.3), _u(g, N25 - nt, 0.0, 1.0)]))
    return dict(kind=MAG, ws=[w], ks=[int(0.8 * N25 * 0.3) + nt // 2], expect={"fallback: list over cap"})


def r_ties_in_cand2():
    """10 k copies of 0.3 between a low and a high cluster, k inside the copies: they all share the top digit."""
    g, nt = _g(6), 10_000
    nl = (N25 - nt) // 2
    w = _perm(g, torch.cat([_u(g, nl, 1e-3, 2e-3), torch.full((nt,), 0.3), _u(g, N25 - nt - nl, 1e3, 2e3)]))
    return dict(kind=MAG, ws=[w], ks=[nl + nt // 2], expect={"fallback: n_cand2 > 4096"})


def r_aliased_above():
    """The sampled positions hold large values, every other element is tiny: the bracket sits above the k-th key."""
    g = _g(7)
    pos = torch.from_numpy(sample_positions([N25]))
    w = _u(g, N25, 1e-7, 2e-7)
    w[pos] = _u(g, pos.numel(), 1.0, 2.0)
    return dict(kind=MAG, ws=[w], ks=[N25 // 5], expect={"fallback: bracket above k"})


def r_aliased_below():
    """The opposite aliasing: the bracket sits below the k-th key."""
    g = _g(8)
    pos = torch.from_numpy(sample_positions([N25]))
    w = _u(g, N25, 1.0, 2.0)
    w[pos] = _u(g, pos.numel(), 1e-7, 2e-7)
    return dict(kind=MAG, ws=[w], ks=[N25 // 2], expect={"fallback: bracket below k"})


def _synflow_nan(seed, frac):
    g = _g(seed)
    w = torch.randn(N25, generator=g).abs_() * 0.02
    gr = torch.randn(N25, generator=g) * 1e-3
    m = torch.ones(N25)
    idx = torch.randperm(N25, generator=g)[:int(frac * N25)]
    m[idx] = 0.0                                    # SynFlow's (m * g) * w with m = 0 at g = inf: NaN scores
    gr[idx] = float("inf")
    return w, gr, m


def r_nan_fast():
    w, gr, m = _synflow_nan(9, 0.05)
    return dict(kind=SYNFLOW, ws=[w], gs=[gr], ms=[m], ks=[N25 - 1000, N25 - int(0.05 * N25) + 10],
                expect={"NaN threshold, fast path"})


def r_nan_fallback():
    w, gr, m = _synflow_nan(10, 0.2)
    return dict(kind=SYNFLOW, ws=[w], gs=[gr], ms=[m], ks=[N25 - 1000], expect={"NaN threshold after a fallback"})


def r_inf_thr():
    g = _g(11)
    w = torch.randn(N25, generator=g) * 0.05
    w[torch.randperm(N25, generator=g)[:N25 // 100]] = float("inf")
    return dict(kind=MAG, ws=[w], ks=[N25 - N25 // 200], expect={"+inf threshold"})


def r_subnormal_thr():
    g = _g(12)
    w = torch.randn(N25, generator=g) * 0.05
    idx = torch.randperm(N25, generator=g)[:3 * N25 // 100]
    w[idx] = _u(g, idx.numel(), 1e-42, 1e-39) * torch.sign(torch.randn(idx.numel(), generator=g))
    return dict(kind=MAG, ws=[w], ks=[int(0.015 * N25), int(0.029 * N25)], expect={"subnormal threshold"})


def r_200_segments():
    """200 segments of 1 ... 300 k elements, sizes neither multiples of 4 nor of 16, per-segment scales, IMP-style masks."""
    g = _g(13)
    sizes = (torch.randint(0, 75_000, (195,), generator=g) * 4 + torch.randint(1, 4, (195,), generator=g)).tolist()
    sizes = [1, 3, 7, 15, 17] + sizes
    sizes = [sizes[i] for i in torch.randperm(len(sizes), generator=g).tolist()]
    ws = [torch.randn(n, generator=g) * 10 ** (-3 + 2 * torch.rand((), generator=g).item()) for n in sizes]
    ms = [(torch.rand(n, generator=g) < 0.7).float() for n in sizes]
    N = sum(sizes)
    return dict(kind=MAG, ws=ws, ms=ms, ks=[int(0.2 * N), int(0.5 * N), int(0.9 * N)],
                expect={"segment table in global memory"})


def r_misaligned():
    """SNIP over w, m, g and the output each a view at storage offset 1-3: every 16-byte path is off."""
    g = _g(14)
    sizes = [10_000_001, 7_654_321, 6_000_005]
    ws = [torch.randn(n, generator=g) * 0.05 for n in sizes]
    ms = [(torch.rand(n, generator=g) < 0.8).float() for n in sizes]
    gs = [torch.randn(n, generator=g) * 1e-3 * m for n, m in zip(sizes, ms)]
    N = sum(sizes)
    return dict(kind=SNIP, ws=ws, ms=ms, gs=gs, ks=[int(0.3 * N), int(0.9 * N)], views=True,
                expect={"misaligned operands (scalar sample / sweep)"})


def r_s_equals_n():
    g = _g(15)
    N = 1 << 20
    return dict(kind=MAG, ws=[torch.randn(N, generator=g) * 0.05], ks=[1, N // 2, N], expect={"S == N = 2^20"})


def r_s_below_n():
    g = _g(16)
    sizes = [1 << 19, (1 << 19) + 1]
    N = sum(sizes)
    return dict(kind=MAG, ws=[torch.randn(n, generator=g) * 0.05 for n in sizes], ks=[1, N // 2, N],
                expect={"S = 2^20 < N"})


def r_thr_only():
    g = _g(17)
    sizes = [9_000_000, 8_000_003, 8_000_000]
    return dict(kind=MAG, ws=[torch.randn(n, generator=g) * 0.05 for n in sizes], ks=[int(0.8 * sum(sizes))],
                write=False, expect={"write_masks=False"})


RECIPES = {f.__name__[2:]: f for f in (r_shift22, r_shift0, r_ties_at_lo, r_sorted, r_ties_over_cap, r_ties_in_cand2,
                                       r_aliased_above, r_aliased_below, r_nan_fast, r_nan_fallback, r_inf_thr,
                                       r_subnormal_thr, r_200_segments, r_misaligned, r_s_equals_n, r_s_below_n,
                                       r_thr_only)}


def _offset_view(t, off, dev):
    """t on the device as a contiguous view at storage offset ``off`` of a larger buffer (4-byte, not 16-byte aligned)."""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=dev)
    v = buf[off:off + t.numel()]
    v.copy_(t)
    assert v.is_contiguous() and v.storage_offset() == off
    return v


def _oracle(r):
    ws = [w.numpy() for w in r["ws"]]
    ms = [m.numpy() for m in r.get("ms") or _ones(r["ws"])]
    gs = None if r.get("gs") is None else [x.numpy() for x in r["gs"]]
    scores = P.layer_scores(ws, ms, gs, r["kind"])
    flat = np.concatenate([s.reshape(-1) for s in scores])
    return scores, kth_many(flat, r["ks"]), raw_keys(scores)


@gpu
@pytest.mark.parametrize("rid", list(RECIPES))
def test_topk_path_recipe(dev, rid):
    from turboprune_b200 import _cabi, ops
    r = RECIPES[rid]()
    kind, sizes = r["kind"], [w.numel() for w in r["ws"]]
    ms = r.get("ms") or _ones(r["ws"])
    scores, thrs, keys = _oracle(r)
    reached = set()
    if r.get("views"):
        tw = [_offset_view(w, 1, dev) for w in r["ws"]]
        tm = [_offset_view(m, 2, dev) for m in ms]
        tg = [_offset_view(x, 3, dev) for x in r["gs"]]
        reached.add("misaligned operands (scalar sample / sweep)")
    else:
        tw = [w.to(dev) for w in r["ws"]]
        tm = [m.to(dev) for m in ms]
        tg = None if r.get("gs") is None else [x.to(dev) for x in r["gs"]]
    if r.get("write", True):
        plan = ops.TopKPlan(tw, tm, gs=tg, kind=kind)
        if r.get("views"):                              # the outputs too: views at offset 1 of larger buffers
            plan.outs = [_offset_view(torch.zeros(n), 1, dev) for n in sizes]
            plan.args = plan.args[:3] + (_cabi.ptr_array(plan.outs),) + plan.args[4:]
        assert all(a.data_ptr() == b.data_ptr() for a, b in zip(plan.ws + plan.ms, tw + tm))   # .contiguous() kept the views
        for k, thr in zip(r["ks"], thrs):
            reached |= _select(plan, k, thr, scores, keys, sizes)
    else:
        for k, thr in zip(r["ks"], thrs):
            outs, t, info = ops.topk_threshold_mask(tw, tm, k, gs=tg, kind=kind, write_masks=False)
            assert outs is None and _same_thr(t.item(), thr)
            st = ops.topk_state(ops._workspace(0, dev, "topk"), len(sizes))
            reached |= _classify(st, info, k, np.float32(t.item()), predict_state(keys, sizes, k))
        reached.add("write_masks=False")
    N = sum(sizes)
    if len(sizes) > SMEM_SEGS:
        reached.add("segment table in global memory")
    if N == SAMPLE_MAX:
        reached.add("S == N = 2^20")
    if N == SAMPLE_MAX + 1:
        reached.add("S = 2^20 < N")
    _record(rid, reached)
    assert r["expect"] <= reached, (rid, sorted(reached))


# ---------------------------------------------------------------- production extents, through the product ---------------
@pytest.fixture(scope="module")
def r50(dev):
    """Seed-0 ResNet-50 (ImageNet configuration): 54 masked layers, 25.5 M weights."""
    import refshim
    from turboprune_b200.utils import custom_models as cm
    torch.manual_seed(0)
    model = cm.TorchVisionModel(refshim.make_cfg("resnet50", "imagenet")).to(dev)
    layers = [m for _, m in model._masked()]
    assert len(layers) == 54
    return model, layers


def _state_of_last_call(dev, n_seg):
    from turboprune_b200 import ops
    return ops.topk_state(ops._workspace(0, dev, "topk"), n_seg)


def _fallbacks_only_on_the_second_level(case_id, k, branches, fallbacks):
    """A realistic selection must never miss its bracket or overflow the candidate list.  The one fallback it may take
    today is the overflow of the 4096-key second-level list: when the bracket spans only a few 2^11-key blocks, more than
    4096 candidates share the top digit (the result stays exact; the cost is the 3-pass radix fallback).  Such calls are
    reported as a warning so that they stay visible."""
    fb = {b for b in branches if b.startswith("fallback")}
    assert fb <= {"fallback: n_cand2 > 4096"}, (case_id, k, fb)
    if fb:
        fallbacks.append(k)


@gpu
def test_imp_chain_resnet50(dev, r50):
    """prune_mag on ResNet-50 at densities 0.8^L, L = 1 ... 30, every level bit for bit against the oracle's own chain.
    No level may miss its bracket (see _fallbacks_only_on_the_second_level)."""
    from turboprune_b200 import ops
    from turboprune_b200.utils import pruning_utils as pu
    model, layers = r50
    for m in layers:
        m.mask = torch.ones_like(m.weight)
    ws = [m.weight.detach().cpu().numpy().reshape(-1) for m in layers]
    sizes = [w.size for w in ws]
    ms = [np.ones_like(w) for w in ws]
    density, reached, fallbacks = 1.0, set(), []
    for level in range(1, 31):
        density *= 0.8
        pu.prune_mag(model, density)
        info = model._last_prune_info
        st = _state_of_last_call(dev, len(layers))
        prev = ms
        ms, thr, k = P.prune_global(ws, prev, density)
        for i, (m, r) in enumerate(zip(layers, ms)):
            assert np.array_equal(m.mask.cpu().numpy().reshape(-1), r), (level, i)
        if info["path"] == 0:
            assert _same_thr(np.array([st["thr_key"]], np.uint32).view(np.float32)[0], thr), level
            pred = None
            if level in (1, 5, 10, 20, 25, 30):
                pred = predict_state(raw_keys(P.layer_scores(ws, prev)), sizes, k)
            b = _classify(st, info, k, thr, pred)
        else:   # the fallback inside the call rewrote the state: replay the level through TopKPlan to read the kernel's own
            scores = P.layer_scores(ws, prev)
            plan = ops.TopKPlan([m.weight.detach() for m in layers], [torch.from_numpy(x).to(dev) for x in prev])
            b = _select(plan, k, thr, scores, raw_keys(scores), sizes)
            del plan
        print(f"[topk] imp level {level}: k={k} {sorted(b)}")
        _fallbacks_only_on_the_second_level(f"imp level {level}", k, b, fallbacks)
        reached |= b
    if fallbacks:
        warnings.warn(f"ResNet-50 IMP: {len(fallbacks)} of 30 levels took the exact fallback (second-level list over "
                      f"4096 keys), k = {fallbacks}")
    _record("imp_chain_resnet50", reached)


@gpu
@pytest.mark.parametrize("crit", ["erk", "balanced"])
def test_per_layer_random_criteria_resnet50(dev, r50, crit, monkeypatch):
    """prune_random_erk / prune_random_balanced on ResNet-50 against P.prune_per_layer on the same noise.  Five layers
    exceed 2^20 elements (sampled selection), the 2048 -> 512 1x1 convolutions hold exactly 2^20 (S == N)."""
    from turboprune_b200 import ops
    from turboprune_b200.utils import pruning_utils as pu
    model, layers = r50
    for m in layers:
        m.mask = torch.ones_like(m.weight)
    calls = []
    real = ops.topk_threshold_mask

    def spy(ws, ms, k, gs=None, kind=MAG, write_masks=True):
        out = real(ws, ms, k, gs=gs, kind=kind, write_masks=write_masks)
        calls.append((k, _state_of_last_call(dev, len(ws)), out[2], np.float32(out[1].item())))
        return out

    monkeypatch.setattr(ops, "topk_threshold_mask", spy)
    density = 0.2
    torch.manual_seed(5)
    (pu.prune_random_erk if crit == "erk" else pu.prune_random_balanced)(model, density)
    torch.manual_seed(5)
    noises = [torch.randn_like(m.weight).cpu().numpy().reshape(-1) for m in layers]
    numels = [m.weight.numel() for m in layers]
    fracs = (P.erk_keep_probabilities([tuple(m.weight.shape) for m in layers], density) if crit == "erk"
             else P.balanced_keep_probabilities(numels, density))
    ones = [np.ones(n, np.float32) for n in numels]
    ref, ks = P.prune_per_layer(noises, ones, fracs)
    assert [c[0] for c in calls] == [k for k in ks if k > 0]
    reached, it, big = set(), iter(calls), 0
    for i, (m, r, k, z) in enumerate(zip(layers, ref, ks, noises)):
        assert np.array_equal(m.mask.cpu().numpy().reshape(-1), r), (crit, i)
        if k == 0:
            continue
        _, st, info, thr = next(it)
        s = P.score_mag(z, ones[i])
        assert _same_thr(thr, P.kth_smallest(s, k)), (crit, i)
        pred = None
        big += z.size > SAMPLE_MAX
        if z.size >= SAMPLE_MAX and info["path"] == 0:     # a fallback inside the call rewrites the state
            pred = predict_state(raw_keys([s]), [z.size], k)
        reached |= _classify(st, info, k, thr, pred)
    assert big == 5
    _record(f"per_layer_{crit}", reached)


@gpu
def test_snip_scores_resnet50_extents(dev, r50):
    """SNIP over ResNet-50's 54 layers: gradients at per-layer scales 1e-6 ... 1e-2 with exact zeros wherever the mask is
    zero (what the masked wgrad writes), k inside and beyond the zero scores."""
    from turboprune_b200 import ops
    _, layers = r50
    g = _g(21)
    ws = [m.weight.detach().cpu().reshape(-1) for m in layers]
    ms = [(torch.rand(w.numel(), generator=g) < 0.6).float() for w in ws]
    gs = [torch.randn(w.numel(), generator=g) * 10 ** (-6 + 4 * torch.rand((), generator=g).item()) * m
          for w, m in zip(ws, ms)]
    N = sum(w.numel() for w in ws)
    r = dict(kind=SNIP, ws=ws, ms=ms, gs=gs, ks=[int((1 - d) * N) for d in (0.7, 0.5, 0.2, 0.05, 0.01)])
    scores, thrs, keys = _oracle(r)
    plan = ops.TopKPlan([w.to(dev) for w in ws], [m.to(dev) for m in ms], gs=[x.to(dev) for x in gs], kind=SNIP)
    reached, fallbacks = set(), []
    for k, thr in zip(r["ks"], thrs):
        b = _select(plan, k, thr, scores, keys, [w.numel() for w in ws])
        _fallbacks_only_on_the_second_level("snip", k, b, fallbacks)
        reached |= b
    if fallbacks:
        warnings.warn(f"SNIP at ResNet-50 extents: the exact fallback (second-level list over 4096 keys) at k = {fallbacks}")
    _record("snip_resnet50", reached)


@gpu
def test_synflow_vgg16_bench_shape(dev):
    """SynFlow at the benchmark's VGG-16 size: 134.7 M elements in 16 segments (16 B per element), |w|, gradients over
    ten decades and some +inf; every mask element is compared."""
    from turboprune_b200 import ops
    torch.cuda.reset_peak_memory_stats()
    held = torch.cuda.memory_allocated()            # what earlier tests of the session still hold is not this case's
    n2, nseg = 134_657_728, 16
    sizes = [n2 // nseg] * (nseg - 1)
    sizes.append(n2 - sum(sizes))
    g = _g(22)
    ws = [torch.randn(n, generator=g).abs_() * 0.02 for n in sizes]
    gs = []
    for n in sizes:
        x = torch.randn(n, generator=g) * torch.pow(10.0, torch.empty(n).uniform_(-9.0, 1.0, generator=g))
        x[torch.randint(0, n, (64,), generator=g)] = float("inf")
        gs.append(x)
    ms = _ones(ws)
    r = dict(kind=SYNFLOW, ws=ws, ms=ms, gs=gs, ks=[int(0.95 * n2), int(0.5 * n2)])
    scores, thrs, keys = _oracle(r)
    plan = ops.TopKPlan([w.to(dev) for w in ws], [m.to(dev) for m in ms], gs=[x.to(dev) for x in gs], kind=SYNFLOW)
    del ws, gs, ms, r
    reached = set()
    for k, thr in zip((int(0.95 * n2), int(0.5 * n2)), thrs):
        reached |= _select(plan, k, thr, scores, keys, sizes)
    peak = torch.cuda.max_memory_allocated() - held
    print(f"[topk] synflow_vgg16: peak device memory of the case {peak / 2**30:.2f} GiB "
          f"({held / 2**30:.2f} GiB held by earlier tests)")
    assert peak < 3.5 * 2**30, (peak, held)
    _record("synflow_vgg16", reached)


@gpu
def test_topk_plan_cached_table(dev, r50):
    """TopKPlan as bench.py uses it: repeated run(k), IMP levels whose new masks are copied into the plan's input masks
    in place and read through the cached segment table, and a fallback followed by a fast-path call on the same plan
    (the state reset between calls)."""
    from turboprune_b200 import ops
    _, layers = r50
    ws = [m.weight.detach().reshape(-1).clone() for m in layers]
    wn = [w.cpu().numpy() for w in ws]
    sizes = [w.size for w in wn]
    plan = ops.TopKPlan(ws, _ones(ws))
    mn = [np.ones_like(w) for w in wn]
    density, reached = 1.0, set()
    for level in range(1, 4):
        density *= 0.8
        scores = P.layer_scores(wn, mn)
        k = int((1 - density) * sum(sizes))
        thr = kth_many(np.concatenate(scores), [k])[0]
        keys = raw_keys(scores)
        for _ in range(2 if level == 1 else 1):
            reached |= _select(plan, k, thr, scores, keys, sizes)
        mn = [P.apply_threshold(s, thr) for s in scores]
        for dst, src in zip(plan.ms, plan.outs):
            dst.copy_(src)
    r = r_ties_over_cap()
    half = N25 // 2
    r["ws"] = [r["ws"][0][:half], r["ws"][0][half:]]
    k_fb, k_fast = r["ks"][0], int(0.9 * N25)
    r["ks"] = [k_fb, k_fast]
    scores, thrs, keys = _oracle(r)
    plan = ops.TopKPlan([w.to(dev) for w in r["ws"]], [torch.ones(w.numel(), device=dev) for w in r["ws"]])
    paths = []
    for k, thr in ((k_fb, thrs[0]), (k_fast, thrs[1]), (k_fb, thrs[0]), (k_fast, thrs[1])):
        b = _select(plan, k, thr, scores, keys, [w.numel() for w in r["ws"]])
        paths.append("fallback: list over cap" in b)
        reached |= b
    assert paths == [True, False, True, False]
    _record("plan_cached_table", reached)


@gpu
def test_apply_threshold_and_count_zeros(dev):
    """tp_apply_threshold and tp_count_zeros at 25 M elements in 200 segments, on views at storage offsets 1-3.
    Thresholds: 0 (the k == 0 path of the random criteria), subnormal, +inf, NaN.  Counts are exact integers."""
    from turboprune_b200 import ops
    g = _g(23)
    sizes = (torch.randint(0, 62_500, (200,), generator=g) * 4 + torch.randint(1, 4, (200,), generator=g)).tolist()
    ws, ms, gs = [], [], []
    for n in sizes:
        w = torch.randn(n, generator=g) * 0.05
        w[::97] = 0.0
        w[5::89] = 3e-40
        w[7::1009] = float("inf")
        w[11::2003] = float("nan")
        ws.append(w)
        ms.append((torch.rand(n, generator=g) < 0.7).float())
        gs.append(torch.randn(n, generator=g) * 1e-3)
    tw = [_offset_view(w, 1, dev) for w in ws]
    tm = [_offset_view(m, 2, dev) for m in ms]
    tg = [_offset_view(x, 3, dev) for x in gs]
    wn, mn, gn = [w.numpy() for w in ws], [m.numpy() for m in ms], [x.numpy() for x in gs]
    for kind in (MAG, SNIP):
        scores = P.layer_scores(wn, mn, None if kind == MAG else gn, kind)
        for thr in (0.0, 3e-40, float("inf"), float("nan")):
            outs = ops.apply_threshold(tw, tm, torch.tensor(thr, device=dev), gs=None if kind == MAG else tg, kind=kind)
            ref = [P.apply_threshold(s, np.float32(thr)) for s in scores]
            for i, (o, r) in enumerate(zip(outs, ref)):
                assert np.array_equal(o.cpu().numpy(), r), (kind, thr, i)
            want = [int(np.count_nonzero(r == 0)) for r in ref]
            want.append(sum(want))
            assert ops.count_zeros(outs).tolist() == want, (kind, thr)
            views = [_offset_view(o, 1 + i % 3, dev) for i, o in enumerate(outs)]
            assert ops.count_zeros(views).tolist() == want, (kind, thr)
    _record("apply_and_count", set())


@gpu
def test_every_path_reached():
    """Union of the paths the cases above reached: every entry of BRANCHES."""
    expected = set(RECIPES) | {"imp_chain_resnet50", "per_layer_erk", "per_layer_balanced", "snip_resnet50",
                               "synflow_vgg16", "plan_cached_table", "apply_and_count"}
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if RAN != expected:
        pytest.skip(f"only part of the file ran (missing: {sorted(expected - RAN)})")
    table = "\n".join(f"  {b:45s} {', '.join(REACHED.get(b, ['-- not reached --']))}" for b in BRANCHES)
    print("[topk] paths reached:\n" + table, file=sys.stderr)
    missed = [b for b in BRANCHES if b not in REACHED]
    assert not missed, "paths no case reached: " + ", ".join(missed) + "\n" + table
