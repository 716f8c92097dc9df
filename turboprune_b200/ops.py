"""Torch-tensor front end of the C-ABI kernels (device memory / streams are torch's; the
arithmetic is ours).  Every function here launches hand-written sm_90a kernels through
``_cabi`` — there is no eager / CPU fallback.
"""
import ctypes
import math
import threading
from contextlib import contextmanager
from ctypes import c_void_p
from typing import Callable, NamedTuple, Optional

import numpy as np
import torch

from . import _cabi

_launches = 0          # number of OUR kernel-launching C-ABI calls (bench.py reports it)


# ---- compute precision of the masked layers ---------------------------------------------------------------------------
# bf16 (the default): bf16 operands and activations, as under the reference's bf16 autocast.  float32: fp32 activations,
# gradients and operands end to end, GEMMs on TF32 tensor cores — the reference's training_precision: float32 with
# allow_tf32 = True.  Thread-local like autocast; a masked layer reads it once in its forward and records it for its
# backward (autograd runs backward on its own thread, where the context is not set).
_precision = threading.local()


def current_precision():
    return getattr(_precision, "dtype", torch.bfloat16)


@contextmanager
def compute_precision(dtype):
    """Run the masked layers (and ``WeightStager.stage``) inside this block at ``dtype``: torch.bfloat16 or torch.float32."""
    if dtype not in (torch.bfloat16, torch.float32):
        raise ValueError(f"compute_precision: bfloat16 or float32, not {dtype}")
    prev = getattr(_precision, "dtype", None)
    _precision.dtype = dtype
    try:
        yield
    finally:
        if prev is None:
            del _precision.dtype
        else:
            _precision.dtype = prev


# ---- dense weight gradients --------------------------------------------------------------------------------------------
# Inside ``dense_weight_grad()`` the masked layers write the UNMASKED weight gradient wgrad(x, dy) (RigL's grow
# criterion needs |g| at pruned positions).  The forward is unchanged.  Read in the forward and kept in ctx, like the
# precision.
_dense_grad = threading.local()


def dense_grad_enabled():
    return getattr(_dense_grad, "on", False)


@contextmanager
def dense_weight_grad(on=True):
    """Masked layers whose forward runs inside this block produce the dense weight gradient in their backward."""
    prev = dense_grad_enabled()
    _dense_grad.on = bool(on)
    try:
        yield
    finally:
        _dense_grad.on = prev


_ones_cache = {}


def _ones_like_mask(m):
    """Cached all-ones fp32 mask of m's shape (the wgrad kernels take a mask; a dense gradient hands them this one)."""
    key = (tuple(m.shape), m.device)
    t = _ones_cache.get(key)
    if t is None:
        t = _ones_cache[key] = torch.ones(m.shape, dtype=torch.float32, device=m.device)
    return t


def _count(n=1):
    global _launches
    _launches += n


def launch_count() -> int:
    return _launches


class KernelTimer:
    """CUDA-event timing of the masked-GEMM C-ABI calls on the launching stream (bench.py uses it
    to report the dominant kernel's achieved TFLOP/s live, inside the timed region)."""

    def __init__(self):
        self.records = []          # (kind, flops, start_event, end_event)

    def totals(self):
        out = {}
        for kind, flops, e0, e1 in self.records:
            ms = e0.elapsed_time(e1)
            t = out.setdefault(kind, [0.0, 0.0, 0])
            t[0] += ms; t[1] += flops; t[2] += 1
        return out


_timer = None


def set_timer(timer):
    global _timer
    _timer = timer


class _Timed:
    def __init__(self, kind, desc, cin_real=None):
        self.on = _timer is not None
        if self.on:
            cin = desc.cin if cin_real is None else cin_real
            self.flops = 2.0 * desc.n * desc.p * desc.q * desc.cout * cin * desc.r * desc.s
            self.kind = kind

    def __enter__(self):
        if self.on:
            self.e0 = torch.cuda.Event(enable_timing=True); self.e0.record()

    def __exit__(self, *a):
        if self.on:
            e1 = torch.cuda.Event(enable_timing=True); e1.record()
            _timer.records.append((self.kind, self.flops, self.e0, e1))


_grad_ready_hook = None      # set by P2PGradReducer.arm(): called with the data_ptr of every gradient slot a kernel just filled


def set_grad_ready_hook(fn):
    global _grad_ready_hook
    _grad_ready_hook = fn


def get_grad_ready_hook():
    return _grad_ready_hook


def grad_ready(*slots):
    """Report gradients written straight into their persistent slots (no AccumulateGrad node runs for them, so
    autograd's own hooks never fire): lets the gradient exchange start a bucket while the backward pass continues."""
    if _grad_ready_hook is not None:
        for s in slots:
            if s is not None:
                _grad_ready_hook(s.data_ptr())


# ---- weight gradients on a side stream -------------------------------------------------------------------------------
# dW of a layer is needed by nobody before the gradient exchange / the optimizer, while dX is the critical path of the
# backward pass.  With WGRAD_SIDE_STREAM the wgrad GEMM + finalize of every masked layer go to one side stream behind an
# event of the compute stream; at small per-GPU batches (the 8-GPU operating point: 64 images) the kernels are one or two
# waves each and the two chains fill each other's gaps.  The operands are marked as used by the side stream (the caching
# allocator would otherwise hand their blocks to the next main-stream allocation while the side stream still reads them).
# Off unless a caller that also joins turns it on (BaseHarness._step_body does, around its backward pass).
WGRAD_SIDE_STREAM = False
_wgrad_streams = {}
_wgrad_pending = set()      # devices with weight gradients launched on the side stream since the last join


def set_wgrad_side_stream(on: bool):
    global WGRAD_SIDE_STREAM
    WGRAD_SIDE_STREAM = bool(on)


def _wgrad_stream(device):
    st = _wgrad_streams.get(device.index)
    if st is None:
        st = _wgrad_streams[device.index] = torch.cuda.Stream(device)
    return st


def join_wgrad(device=None):
    """Make the current stream wait for every weight gradient launched on the side stream since the last join.  Call
    after ``loss.backward()``, before anything consumes ``param.grad``."""
    for d in _wgrad_pending:
        if device is None or d == device:
            torch.cuda.current_stream(d).wait_stream(_wgrad_stream(d))
    _wgrad_pending.clear()


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("turboprune_b200 kernels need CUDA tensors (H100 / sm_90a); there is no CPU path")


_ws_cache = {}


def _workspace(nbytes: int, device, tag="default") -> torch.Tensor:
    """Grow-only per-(device, stream, tag) scratch buffer owned by Python."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream, tag)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 1 << 16), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


# ---------------------------------------------------------------------------------------------
# pruning
# ---------------------------------------------------------------------------------------------
def topk_threshold_mask(ws, ms, k, gs=None, kind=_cabi.TP_SCORE_MAG, write_masks=True):
    """Exact k-th smallest score over all layers + new masks (torch.kthvalue / torch.where parity).

    Returns (new_masks | None, thr (0-dim fp32 cuda tensor), info dict).  Raises RuntimeError for
    k outside [1, N] like torch.kthvalue does (the reference hits this for k == 0,
    utils/pruning_utils.py:78-79).
    """
    lib = _cabi.load()
    _require_cuda(*ws, *ms)
    dev = ws[0].device
    ws = [w.detach().contiguous() for w in ws]
    ms = [m.detach().contiguous() for m in ms]
    gs = None if gs is None else [g.detach().contiguous() for g in gs]
    for t in ws + ms + (gs or []):
        if t.dtype != torch.float32:
            raise TypeError("pruning kernels operate on fp32 weights / masks / grads")
    numel = [w.numel() for w in ws]
    total = sum(numel)
    outs = [torch.empty_like(m) for m in ms] if write_masks else None
    thr = torch.empty((), dtype=torch.float32, device=dev)
    nbytes = lib.tp_topk_workspace_bytes(len(ws), total)
    wsb = _workspace(nbytes, dev, "topk")
    info = (ctypes.c_int64 * 4)()
    with torch.cuda.device(dev):
        rc = lib.tp_topk_threshold_mask(
            _cabi.ptr_array(ws), _cabi.ptr_array(gs), _cabi.ptr_array(ms), _cabi.ptr_array(outs),
            _cabi.i64_array(numel), len(ws), int(k), int(kind), c_void_p(thr.data_ptr()),
            c_void_p(wsb.data_ptr()), wsb.numel(), info, _cabi.stream_ptr(dev))
    if rc == _cabi.TP_ERR_K_RANGE:
        raise RuntimeError(f"kthvalue(): selected number k out of range for dimension 0 (k={k}, N={total})")
    _cabi.check(rc, "tp_topk_threshold_mask")
    _count(1)
    return outs, thr, {"path": int(info[0]), "candidates": int(info[1]), "n_lt": int(info[2]), "nan_thr": bool(info[3])}


class TopKPlan:
    """Pre-marshalled ``tp_topk_threshold_mask`` call (pointer tables, outputs, workspace built once): ``run(k)`` is
    just the C-ABI call.  Used when the same tensors are pruned repeatedly (benchmarks, per-level IMP)."""

    def __init__(self, ws, ms, gs=None, kind=_cabi.TP_SCORE_MAG):
        self.lib = _cabi.load()
        self.dev = ws[0].device
        self.ws = [w.detach().contiguous() for w in ws]
        self.ms = [m.detach().contiguous() for m in ms]
        self.gs = None if gs is None else [g.detach().contiguous() for g in gs]
        self.outs = [torch.empty_like(m) for m in self.ms]
        self.thr = torch.empty((), dtype=torch.float32, device=self.dev)
        self.n = len(self.ws)
        self.total = sum(w.numel() for w in self.ws)
        self.kind = int(kind)
        self.wsb = torch.empty(self.lib.tp_topk_workspace_bytes(self.n, self.total), dtype=torch.uint8, device=self.dev)
        self.args = (_cabi.ptr_array(self.ws), _cabi.ptr_array(self.gs), _cabi.ptr_array(self.ms), _cabi.ptr_array(self.outs),
                     _cabi.i64_array([w.numel() for w in self.ws]))
        self.info = (ctypes.c_int64 * 4)()
        self._cached = False

    def enqueue(self, k):
        """Issue the whole fast path (one memset + one cooperative kernel) without blocking the stream.  The masks /
        threshold must not be consumed before ``finish(k)``."""
        with torch.cuda.device(self.dev):
            rc = self.lib.tp_topk_enqueue(*self.args, self.n, int(k), self.kind, c_void_p(self.thr.data_ptr()),
                                          c_void_p(self.wsb.data_ptr()), self.wsb.numel(), int(self._cached),
                                          _cabi.stream_ptr(self.dev))
        if rc == _cabi.TP_ERR_K_RANGE:
            raise RuntimeError(f"kthvalue(): selected number k out of range for dimension 0 (k={k}, N={self.total})")
        _cabi.check(rc, "tp_topk_enqueue")
        self._cached = True                      # the segment table now lives in the workspace
        _count(1)

    def finish(self, k):
        """Synchronise, read the status back, run the exact fallback if the bracket missed.  Returns (masks, thr, info)."""
        with torch.cuda.device(self.dev):
            rc = self.lib.tp_topk_finish(self.args[2], self.args[3], self.args[4], self.n, int(k), self.kind,
                                         c_void_p(self.thr.data_ptr()), c_void_p(self.wsb.data_ptr()), self.wsb.numel(),
                                         self.info, _cabi.stream_ptr(self.dev))
        _cabi.check(rc, "tp_topk_finish")
        return self.outs, self.thr, {"path": int(self.info[0]), "candidates": int(self.info[1]), "n_lt": int(self.info[2]),
                                     "nan_thr": bool(self.info[3])}

    def run(self, k):
        self.enqueue(k)
        return self.finish(k)

    def state(self):
        """The selection state the last ``enqueue`` left in the workspace (see ``topk_state``)."""
        return topk_state(self.wsb, self.n)


# SelState of tp_prune.cu: k, n_lt, n_eq, n_cand | lo, hi, thr_key, status | prefix, prefix_mask | c_lo, c_hi |
# before_lo, before_hi, k_rem, n_cand2 | barrier, pad | t_phase[8]
_SELSTATE = ("<QQQQ IIIi II II QQQQ II 8Q", ("k", "n_lt", "n_eq", "n_cand", "lo", "hi", "thr_key", "status", "prefix",
                                           "prefix_mask", "c_lo", "c_hi", "before_lo", "before_hi", "k_rem", "n_cand2",
                                           "barrier", "pad"))


def topk_state(wsb, n_seg):
    """Decode the top-k selection state from a workspace of ``tp_topk_*``: a dict of the SelState fields, ``t_phase``
    (the %globaltimer stamps of CTA 0) and ``hist`` (uint32 [8192]: the coarse sample histogram, the two fine ones and
    the candidates' top-digit histogram).  The state follows the segment table (64 B per segment) at a 256-byte
    boundary, its histograms at the next one.  Read it after ``enqueue`` and before ``finish``: the exact fallback
    that ``finish`` may run rewrites it."""
    import struct
    import numpy as np
    off = (64 * n_seg + 255) // 256 * 256
    raw = wsb[off:off + 256 + 4 * 4 * 2048].cpu().numpy().tobytes()
    fmt, names = _SELSTATE
    vals = struct.unpack_from(fmt.replace(" ", ""), raw, 0)
    st = dict(zip(names, vals[:len(names)]))
    st["t_phase"] = list(vals[len(names):])
    st["hist"] = np.frombuffer(raw, dtype=np.uint32, offset=256).copy()
    return st


def apply_threshold(ws, ms, thr, gs=None, kind=_cabi.TP_SCORE_MAG):
    lib = _cabi.load()
    _require_cuda(*ws, *ms, thr)
    dev = ws[0].device
    ws = [w.detach().contiguous() for w in ws]
    ms = [m.detach().contiguous() for m in ms]
    gs = None if gs is None else [g.detach().contiguous() for g in gs]
    outs = [torch.empty_like(m) for m in ms]
    thr = thr.to(device=dev, dtype=torch.float32).reshape(())
    wsb = _workspace(lib.tp_segtable_workspace_bytes(len(ws)), dev, "seg")
    with torch.cuda.device(dev):
        rc = lib.tp_apply_threshold(_cabi.ptr_array(ws), _cabi.ptr_array(gs), _cabi.ptr_array(ms), _cabi.ptr_array(outs),
                                    _cabi.i64_array([w.numel() for w in ws]), len(ws), int(kind),
                                    c_void_p(thr.data_ptr()), c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_apply_threshold")
    _count()
    return outs


def count_zeros(ms):
    """int64 cuda tensor [n+1]: zeros per mask and the total in the last slot. One launch, no sync."""
    lib = _cabi.load()
    _require_cuda(*ms)
    dev = ms[0].device
    ms = [m.detach().contiguous() for m in ms]
    out = torch.empty(len(ms) + 1, dtype=torch.int64, device=dev)
    wsb = _workspace(lib.tp_segtable_workspace_bytes(len(ms)), dev, "seg")
    with torch.cuda.device(dev):
        rc = lib.tp_count_zeros(_cabi.ptr_array(ms), _cabi.i64_array([m.numel() for m in ms]), len(ms),
                                c_void_p(out.data_ptr()), c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_count_zeros")
    _count()
    return out


def rigl_select(ws, gs, ms, new_ms, ks):
    """RigL drop-and-regrow selection for all layers in one launch sequence (no host sync): writes the mask after the
    update into ``new_ms`` (``ms`` is not written).  Per layer i: drop the ks[i] smallest |w| among ms[i] != 0, then grow
    the ks[i] largest |g| among the positions that are 0 after the drop; ties in flat-index order.  Returns an int64
    cuda tensor [n, 2] of (dropped, grown) counts."""
    lib = _cabi.load()
    _require_cuda(*ws, *gs, *ms, *new_ms)
    for t in list(ws) + list(gs) + list(ms) + list(new_ms):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError("rigl_select: contiguous fp32 weights / gradients / masks")
    dev = ws[0].device
    numel = [w.numel() for w in ws]
    if any(t.numel() != n for n, g, m, o in zip(numel, gs, ms, new_ms) for t in (g, m, o)):
        raise ValueError("rigl_select: weight, gradient and mask sizes differ")
    counts = torch.empty(len(ws), 2, dtype=torch.int64, device=dev)
    wsb = _workspace(lib.tp_rigl_workspace_bytes(len(ws), sum(numel)), dev, "rigl")
    with torch.cuda.device(dev):
        rc = lib.tp_rigl_select(_cabi.ptr_array(ws), _cabi.ptr_array(gs), _cabi.ptr_array(ms), _cabi.ptr_array(new_ms),
                                _cabi.i64_array(numel), _cabi.i64_array(ks), len(ws), c_void_p(counts.data_ptr()),
                                c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_rigl_select")
    _count(20)
    return counts


def rigl_apply(ms, new_ms, ws, bufs=None):
    """In place, one launch: ms <- new_ms; where new != 0 and old == 0, w = 0 and its momentum (``bufs[i]``, may be
    None) = 0."""
    lib = _cabi.load()
    _require_cuda(*ms, *new_ms, *ws)
    bufs = [None] * len(ms) if bufs is None else list(bufs)
    for t in list(ms) + list(new_ms) + list(ws) + [b for b in bufs if b is not None]:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError("rigl_apply: contiguous fp32 masks / weights / momenta")
    dev = ms[0].device
    wsb = _workspace(lib.tp_segtable_workspace_bytes(len(ms)), dev, "seg")
    with torch.cuda.device(dev):
        rc = lib.tp_rigl_apply(_cabi.ptr_array(ms), _cabi.ptr_array(new_ms), _cabi.ptr_array(ws), _cabi.ptr_array(bufs),
                               _cabi.i64_array([m.numel() for m in ms]), len(ms), c_void_p(wsb.data_ptr()), wsb.numel(),
                               _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_rigl_apply")
    _count()


def rigl_apply_states(ms, new_ms, ws, states):
    """``rigl_apply`` for any number of optimizer state arrays: ``states[j][i]`` is state j of layer i (None allowed).
    Where new != 0 and old == 0, w and every state restart at 0.  One launch."""
    lib = _cabi.load()
    _require_cuda(*ms, *new_ms, *ws)
    states = [list(s) for s in states]
    if any(len(s) != len(ms) for s in states):
        raise ValueError("rigl_apply_states: one state tensor (or None) per layer")
    for t in list(ms) + list(new_ms) + list(ws) + [b for s in states for b in s if b is not None]:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError("rigl_apply_states: contiguous fp32 masks / weights / optimizer states")
    dev = ms[0].device
    wsb = _workspace(lib.tp_segtable_workspace_bytes(len(ms) * max(len(states), 1)), dev, "seg")
    flat = [b for s in states for b in s]
    with torch.cuda.device(dev):
        rc = lib.tp_rigl_apply_states(_cabi.ptr_array(ms), _cabi.ptr_array(new_ms), _cabi.ptr_array(ws),
                                      _cabi.ptr_array(flat) if flat else None, len(states),
                                      _cabi.i64_array([m.numel() for m in ms]), len(ms), c_void_p(wsb.data_ptr()),
                                      wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_rigl_apply_states")
    _count()


# ---------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------
def sgd_momentum_step(params, grads, bufs, lr_dev, momentum, weight_decay, first_step, table_ws=None, table_cached=False):
    """One fused launch.  ``table_ws``: a persistent uint8 workspace owned by the optimizer; with
    ``table_cached`` the segment table already in it is reused (no H2D copy -> CUDA-graph capturable)."""
    lib = _cabi.load()
    dev = params[0].device
    wsb = table_ws if table_ws is not None else _workspace(lib.tp_segtable_workspace_bytes(len(params)), dev, "seg")
    with torch.cuda.device(dev):
        rc = lib.tp_sgd_momentum(_cabi.ptr_array(params), _cabi.ptr_array(grads), _cabi.ptr_array(bufs),
                                 _cabi.i64_array([p.numel() for p in params]), len(params),
                                 c_void_p(lr_dev.data_ptr()), float(momentum), float(weight_decay), int(bool(first_step)),
                                 int(bool(table_cached)), c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_sgd_momentum")
    _count()


def adamw_step(params, grads, exp_avgs, exp_avg_sqs, steps, inv_lr_dev, decay_dev, beta1, beta2, eps, table_ws=None,
               table_cached=False):
    """One fused AdamW step (step-count increment + update: two launches).  ``inv_lr_dev``: device fp32(1 / lr) and
    ``decay_dev``: device fp32(1 - lr * wd), or None for weight_decay == 0, both formed in double.  ``table_ws`` /
    ``table_cached``: as ``sgd_momentum_step``."""
    lib = _cabi.load()
    dev = params[0].device
    wsb = table_ws if table_ws is not None else _workspace(lib.tp_segtable_workspace_bytes(len(params)), dev, "seg")
    # a cached table needs no pointers (the call only counts tiles), which saves the host five pointer arrays per step
    ptrs = [None] * 5 if table_cached else [_cabi.ptr_array(ts) for ts in (params, grads, exp_avgs, exp_avg_sqs, steps)]
    with torch.cuda.device(dev):
        rc = lib.tp_adamw(*ptrs, _cabi.i64_array([p.numel() for p in params]),
                          len(params), c_void_p(inv_lr_dev.data_ptr()), c_void_p(decay_dev.data_ptr()) if decay_dev is not None else None,
                          float(beta1), float(beta2), float(eps), int(bool(table_cached)), c_void_p(wsb.data_ptr()),
                          wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_adamw")
    _count(2)


def schedulefree_step(params, grads, zs, scalars_dev, weight_decay, first_step, table_ws=None, table_cached=False):
    """One fused Schedule-Free SGD step (one launch).  ``scalars_dev``: device fp32 [3] = (lr, ckp1, alpha_y), each
    formed in double.  ``first_step``: the ``zs`` are uninitialised and start as copies of the params.  ``table_ws`` /
    ``table_cached``: as ``sgd_momentum_step``."""
    lib = _cabi.load()
    dev = params[0].device
    wsb = table_ws if table_ws is not None else _workspace(lib.tp_segtable_workspace_bytes(len(params)), dev, "seg")
    ptrs = [None] * 3 if table_cached else [_cabi.ptr_array(ts) for ts in (params, grads, zs)]
    with torch.cuda.device(dev):
        rc = lib.tp_schedulefree_sgd(*ptrs, _cabi.i64_array([p.numel() for p in params]), len(params),
                                     c_void_p(scalars_dev.data_ptr()), float(weight_decay), int(bool(first_step)),
                                     int(bool(table_cached)), c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_schedulefree_sgd")
    _count()


def schedulefree_swap(params, zs, weight, table_ws=None, table_cached=False):
    """``p.lerp_(z, weight)`` for every pair, bit for bit with torch's per-tensor lerp_, in one launch."""
    lib = _cabi.load()
    dev = params[0].device
    wsb = table_ws if table_ws is not None else _workspace(lib.tp_segtable_workspace_bytes(len(params)), dev, "seg")
    ptrs = [None] * 2 if table_cached else [_cabi.ptr_array(ts) for ts in (params, zs)]
    with torch.cuda.device(dev):
        rc = lib.tp_schedulefree_swap(*ptrs, _cabi.i64_array([p.numel() for p in params]), len(params), float(weight),
                                      int(bool(table_cached)), c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_schedulefree_swap")
    _count()


MUON_GRAM, MUON_POLY, MUON_UPDATE = 0, 1, 2


def _pad64(v):
    return (v + 63) // 64 * 64


def muon_ratio(a, b, adjust_lr_fn):
    """torch.optim.Muon's ``_adjust_lr`` factor for the 2-D shape [a, b] (``lr * ratio`` is the step's lr)."""
    if adjust_lr_fn is None or adjust_lr_fn == "original":
        return math.sqrt(max(1, a / b))
    if adjust_lr_fn == "match_rms_adamw":
        return 0.2 * math.sqrt(max(a, b))
    return 1.0


class MuonPlan:
    """Workspace layout and tile lists of one Muon step over layers of 2-D shapes ``shapes`` = [(a, b), ...].

    Layer l: X = U (a <= b) or U^T (a > b), [mp][np] = (min, max) padded up to 64, in the panel layout of
    include/turboprune_b200.h; its rows x0 / x1 (the ping-pong pair), g (G = X X^T) and h (H) follow one another in one
    bf16 workspace of ``rows`` x 64.  ``n_tiles`` 64 x 64 X tiles drive the elementwise launches (layer l from
    ``tile0[l]``).  ``gemm_tiles[(mode, src)]``: int32 [n, 8] tile list of a Newton-Schulz GEMM reading X buffer src (0
    or 1), longest K first; UPDATE writes buffer 1 - src."""

    def __init__(self, shapes):
        self.shapes = [(int(a), int(b)) for a, b in shapes]
        self.trans, self.mp, self.np, self.tile0, self.x = [], [], [], [], []
        self.g, self.h = [], []
        rows = tiles = 0
        for a, b in self.shapes:
            mp, np_ = _pad64(min(a, b)), _pad64(max(a, b))
            self.trans.append(a > b)
            self.mp.append(mp)
            self.np.append(np_)
            self.tile0.append(tiles)
            tiles += (mp // 64) * (np_ // 64)
            xr, gr = mp * np_ // 64, mp * mp // 64
            self.x.append((rows, rows + xr))
            self.g.append(rows + 2 * xr)
            self.h.append(rows + 2 * xr + gr)
            rows += 2 * xr + 2 * gr
        self.rows, self.n_tiles = rows, tiles
        self.gemm_tiles = {}
        for src in (0, 1):
            for mode in (MUON_GRAM, MUON_POLY, MUON_UPDATE):
                if mode == MUON_POLY and src == 1:
                    continue
                self.gemm_tiles[(mode, src)] = self._tiles(mode, src)

    def _tiles(self, mode, src):
        out = []
        for l in range(len(self.shapes)):
            mp, np_, g, h = self.mp[l], self.np[l], self.g[l], self.h[l]
            x, xo = self.x[l][src], self.x[l][1 - src]
            tm, tn = mp // 64, np_ // 64
            if mode == MUON_UPDATE:                  # X' = H X + a X: A = rows of H, B = 64 K rows of X's panel tn
                out += [(h + ti * 64, x + t * mp, mp, 64, tm, x + t * mp + ti * 64, xo + t * mp + ti * 64, -1)
                        for ti in range(tm) for t in range(tn)]
                continue
            src_rows, nk, dst = (x, tn, g) if mode == MUON_GRAM else (g, tm, h)
            for ti in range(tm):
                for tk in range(ti, tm):                 # upper tiles; each is mirrored into (tk, ti)
                    c0 = g + tk * mp + ti * 64 if mode == MUON_POLY else -1
                    out.append((src_rows + ti * 64, src_rows + tk * 64, mp, mp, nk, c0,
                                dst + tk * mp + ti * 64, dst + ti * mp + tk * 64))
        out.sort(key=lambda t: -t[4])                    # longest K first (stable)
        return np.asarray(out, dtype=np.int32).reshape(-1, 8)

    def ratios(self, adjust_lr_fn):
        return [muon_ratio(a, b, adjust_lr_fn) for a, b in self.shapes]

    def layer_table(self, ws, gs, bufs, adjust_lr_fn):
        """ctypes array of tp_muon_layer for the fp32 [a][b] weights / gradients / momentum buffers."""
        arr = (_cabi.MuonLayer * len(self.shapes))()
        for l, ((a, b), r) in enumerate(zip(self.shapes, self.ratios(adjust_lr_fn))):
            arr[l] = _cabi.MuonLayer(ws[l].data_ptr(), gs[l].data_ptr(), bufs[l].data_ptr(), a, b, int(self.trans[l]),
                                     self.mp[l], self.np[l], self.tile0[l], self.x[l][0], self.x[l][1], r)
        return arr


def muon_prepare(plan, xws, partial, norms, table_ws, ws, gs, bufs, momentum, nesterov, eps, adjust_lr_fn,
                 table_cached=False):
    """Momentum lerps, bf16(u) into X buffer 0, per-tile sums of squares and each layer's clamped bf16 norm into the fp32
    device tensor ``norms`` (one launch).  ``ws`` / ``gs`` / ``bufs``: contiguous fp32 [a][b] views; with
    ``table_cached`` they are not read (the table in ``table_ws``, which carries each layer's lr ratio, is reused)."""
    lib = _cabi.load()
    dev = xws.device
    layers = None if table_cached else plan.layer_table(ws, gs, bufs, adjust_lr_fn)
    with torch.cuda.device(dev):
        rc = lib.tp_muon_prepare(layers, len(plan.shapes), plan.n_tiles, int(bool(table_cached)), c_void_p(xws.data_ptr()),
                                 c_void_p(partial.data_ptr()), c_void_p(norms.data_ptr()), float(momentum),
                                 int(bool(nesterov)), float(eps), c_void_p(table_ws.data_ptr()), table_ws.numel(),
                                 _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_muon_prepare")
    _count()


def muon_normalize(plan, xws, norms, table_ws):
    lib = _cabi.load()
    dev = xws.device
    with torch.cuda.device(dev):
        rc = lib.tp_muon_normalize(len(plan.shapes), plan.n_tiles, c_void_p(xws.data_ptr()), c_void_p(norms.data_ptr()),
                                   c_void_p(table_ws.data_ptr()), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_muon_normalize")
    _count()


def muon_ns_gemm(mode, xws, tiles_dev, alpha, beta):
    """One Newton-Schulz GEMM over the int32 [n, 8] device tile list ``tiles_dev`` (see tp_muon_ns_gemm)."""
    lib = _cabi.load()
    dev = xws.device
    with torch.cuda.device(dev):
        rc = lib.tp_muon_ns_gemm(int(mode), c_void_p(xws.data_ptr()), xws.numel() // 64, c_void_p(tiles_dev.data_ptr()),
                                 tiles_dev.shape[0], float(alpha), float(beta), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_muon_ns_gemm")
    _count()


def muon_apply(plan, xws, which, lr_wd, table_ws):
    """w = w * fp32(1 - lr wd) + fp32(-(lr ratio)) * O; ``lr_wd``: float64 device tensor (lr, weight_decay)."""
    lib = _cabi.load()
    dev = xws.device
    with torch.cuda.device(dev):
        rc = lib.tp_muon_apply(len(plan.shapes), plan.n_tiles, c_void_p(xws.data_ptr()), int(which),
                               c_void_p(lr_wd.data_ptr()), c_void_p(table_ws.data_ptr()), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_muon_apply")
    _count()


# ---------------------------------------------------------------------------------------------
# masked convolution / linear
# ---------------------------------------------------------------------------------------------
def _round_up(x, m):
    return (x + m - 1) // m * m


def make_desc(n, h, w, cin, cout, r, s, stride, padding):
    sh, sw = stride
    ph, pw = padding
    p = (h + 2 * ph - r) // sh + 1
    q = (w + 2 * pw - s) // sw + 1
    return _cabi.ConvDesc(n, h, w, cin, cout, r, s, sh, sw, ph, pw, p, q)


def stem_geometry(cin, r, s):
    """(channels per tap, K of the stem GEMM): no channel padding inside a tap (cg = cin); K padded to a multiple of 8
    (the RGB 7x7 stem: 147 -> 152 columns)."""
    cg = cin
    return cg, _round_up(r * s * cg, 8)


KBLOCK_SKIP = True      # K-block occupancy masks: all-zero 64x64 weight blocks are neither loaded nor multiplied


def set_kblock_skip(on: bool):
    """Toggle tile skipping (benchmarks / parity tests compare both walks; results are bit-identical)."""
    global KBLOCK_SKIP
    KBLOCK_SKIP = bool(on)


def kmask_shapes(cout, cin, r, s, wf_ld, cout_p):
    """([row groups, words] of the fprop mask, [row groups, words] of the dgrad mask) — include/turboprune_b200.h."""
    words = lambda cols: ((cols + 63) // 64 + 31) // 32
    return ((cout + 63) // 64, words(wf_ld)), ((cin + 63) // 64, words(r * s * cout_p))


def kblock_occupancy(kmask, columns):
    """(empty, total) 64x64 weight blocks described by an occupancy mask over ``columns`` K columns (host sync)."""
    kb = (columns + 63) // 64
    rows = kmask_rows(kmask, columns)
    return int(kmask[-1].item()), rows.shape[0] * kb            # the staging call left the count behind the last row


def stage_weights(weight4d, mask4d, cin_p, need_dgrad, cout_p=None, wf_ld=0, want_kmask=None):
    """(mask*w) -> bf16 operand layouts wf [Cout, R*S*cin_p] (row stride ``wf_ld`` when given, zero tail) and
    (optionally) wd [cin, R*S*cout_p].  With ``want_kmask`` (default: the module switch) the K-block occupancy masks are
    produced too and ride along as ``wf.kmask`` / ``wd.kmask`` (uint32 tensors consumed by conv_fprop / conv_dgrad)."""
    lib = _cabi.load()
    cout, cin, r, s = weight4d.shape
    dev = weight4d.device
    if wf_ld and wf_ld > r * s * cin_p:
        wf = torch.zeros(cout, wf_ld, dtype=torch.bfloat16, device=dev)
    else:
        wf = torch.empty(cout, r * s * cin_p, dtype=torch.bfloat16, device=dev)
    wd = None
    cout_p = cout if cout_p is None else cout_p
    if need_dgrad:
        wd = torch.empty(cin, r * s * cout_p, dtype=torch.bfloat16, device=dev)
    kf = kd = None
    if KBLOCK_SKIP if want_kmask is None else want_kmask:
        sf, sd = kmask_shapes(cout, cin, r, s, wf.shape[1], cout_p)
        kf = torch.empty(sf[0] * sf[1] + 1, dtype=torch.int32, device=dev)      # [rows][words] + the empty-block count
        kd = torch.empty(sd[0] * sd[1] + 1, dtype=torch.int32, device=dev) if wd is not None else None
    with torch.cuda.device(dev):
        rc = lib.tp_stage_weights(c_void_p(weight4d.data_ptr()), c_void_p(mask4d.data_ptr()), cout, cin, r, s,
                                  c_void_p(wf.data_ptr()), cin_p, int(wf_ld), c_void_p(wd.data_ptr()) if wd is not None else None,
                                  cout_p, cin, c_void_p(kf.data_ptr()) if kf is not None else None,
                                  c_void_p(kd.data_ptr()) if kd is not None else None, _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_stage_weights")
    _count()
    wf.kmask = kf
    if wd is not None:
        wd.kmask = kd
    return wf, wd


def kmask_rows(kmask, columns):
    """[row groups, words] view of an occupancy mask buffer (its last element is the empty-block count)."""
    words = ((columns + 63) // 64 + 31) // 32
    return kmask[:-1].view(-1, words)


def padded_cin(cin, r, s):
    """Channel count the TMA layouts need: a multiple of 8 (16-byte rows), and of 64 when the filter has more than one
    tap (the K loop walks 64-channel blocks per tap).  Inputs in between (the reference wraps ANY nn.Conv2d,
    custom_models.py:64-107) are zero-padded to it while being laid out as NHWC bf16."""
    return _round_up(cin, 64 if r * s > 1 else 8)


class LayerPlan(NamedTuple):
    """Operand layout of a masked layer (see ``layer_plan``)."""
    cin_p: int          # input channels as laid out: padded to ``padded_cin``; for the stem, cg = cin channels per tap
    cout_p: int         # output channels the backward GEMMs walk (cout for the stem)
    has_wd: bool        # a dgrad operand exists: False exactly for the stem
    wf_ld: int          # row length of the fprop operand: taps * cin_p; for the stem, its K padded to 8 (kp)

    @property
    def stem(self):
        return not self.has_wd


def layer_plan(cout, cin, r, s, need_dx=False):
    """The operand layout of a masked layer with weight [cout, cin, r, s].  <= 8 input channels that do not fill one
    16-byte row (or sit under a multi-tap filter) and no input gradient wanted (the RGB stem): explicit im2col over
    ``stem_geometry`` columns and a plain GEMM, with no dgrad operand.  Everything else: the TMA layouts, the input
    channels zero-padded to ``padded_cin`` and Cout padded for the backward GEMMs, which walk it in 64-channel blocks
    per tap when the filter has more than one tap.  The WeightStager plans with ``need_dx=False``."""
    if cin <= 8 and (cin % 8 != 0 or r * s > 1) and not need_dx:
        cg, kp = stem_geometry(cin, r, s)
        return LayerPlan(cg, cout, False, kp)
    cin_p = padded_cin(cin, r, s)
    return LayerPlan(cin_p, _round_up(cout, 64 if r * s > 1 else 8), True, r * s * cin_p)


def _layer_descs(plan, weight_shape, x_shape, stride, padding):
    """(conv, fprop, wgrad, dgrad) descriptors of a masked layer run with ``plan``.  conv: the convolution over the input
    as laid out.  The stem runs fprop and wgrad as one GEMM over the im2col rows and has no dgrad; the TMA wgrad walks
    Cout padded to cout_p, and the dgrad also writes only the real input channels."""
    cout, cin, r, s = weight_shape
    n, _, h, w = x_shape
    desc = make_desc(n, h, w, plan.cin_p, cout, r, s, stride, padding)
    if plan.stem:
        gdesc = _cabi.ConvDesc(n * desc.p * desc.q, 1, 1, plan.wf_ld, cout, 1, 1, 1, 1, 0, 0, 1, 1)
        return desc, gdesc, gdesc, None
    padded = lambda c: _cabi.ConvDesc(n, h, w, c, plan.cout_p, r, s, desc.stride_h, desc.stride_w, desc.pad_h,
                                      desc.pad_w, desc.p, desc.q)
    wdesc = desc if plan.cout_p == cout else padded(plan.cin_p)
    return desc, desc, wdesc, wdesc if cin == plan.cin_p else padded(cin)


def _shape4(w):
    return tuple(w.shape) if w.dim() == 4 else (w.shape[0], w.shape[1], 1, 1)   # Linear [out, in] / Conv1d(k=1) [out, in, 1]


class Staged(NamedTuple):
    """The operands a ``WeightStager`` left for one layer's next forward, and the plan they are laid out for."""
    wf: torch.Tensor
    wd: Optional[torch.Tensor]
    plan: LayerPlan


class _Shadow:
    """The weight shadow at one precision: persistent operand buffers of every layer the batched kernel stages (bf16
    also: the K-block occupancy masks of all layers in ONE buffer, zeroed by a single memset node per step), the
    StageItem table over them and the kernel's workspace, which caches the table on the device."""

    def __init__(self, layers, dtype):
        dev = layers[0].weight.device
        self.staged = []                   # (layer, Staged); a layer left out stages its own operands in its forward
        for l in layers:
            w = l.weight
            if not w.is_cuda or w.dtype != torch.float32 or not w.is_contiguous():
                continue
            cout, cin, r, s = _shape4(w)
            plan = layer_plan(cout, cin, r, s)
            wf = torch.zeros(cout, plan.wf_ld, dtype=dtype, device=dev)
            wd = torch.zeros(cin, r * s * plan.cout_p, dtype=dtype, device=dev) if plan.has_wd else None
            self.staged.append((l, Staged(wf, wd, plan)))
        self.kmask_all = None
        if dtype == torch.bfloat16:
            sizes = []
            for l, st in self.staged:
                sf, sd = kmask_shapes(*_shape4(l.weight), st.plan.wf_ld, st.plan.cout_p)
                sizes.append((sf[0] * sf[1] + 1, sd[0] * sd[1] + 1 if st.wd is not None else 0))
            self.kmask_all = torch.zeros(max(sum(f + d for f, d in sizes), 1), dtype=torch.int32, device=dev)
            off = 0
            for (_, st), (f, d) in zip(self.staged, sizes):
                st.wf.kmask = self.kmask_all[off:off + f]
                if st.wd is not None:
                    st.wd.kmask = self.kmask_all[off + f:off + f + d]
                off += f + d
        lib = _cabi.load()
        self.ws = torch.empty(max(int(lib.tp_stage_batched_workspace_bytes(len(layers))), 256), dtype=torch.uint8, device=dev)
        self.key = self.items = None

    def set_table(self, key):
        items = (_cabi.StageItem * len(self.staged))()
        for it, (l, st) in zip(items, self.staged):
            it.w = l.weight.data_ptr(); it.mask = l.mask.data_ptr()
            it.wf = st.wf.data_ptr(); it.wd = st.wd.data_ptr() if st.wd is not None else None
            it.cout, it.cin, it.r, it.s = _shape4(l.weight)
            it.cin_p, it.cout_p, it.wf_ld = st.plan.cin_p, st.plan.cout_p, st.plan.wf_ld
            kf, kd = getattr(st.wf, "kmask", None), getattr(st.wd, "kmask", None)
            it.kmask_f = kf.data_ptr() if kf is not None else None
            it.kmask_d = kd.data_ptr() if kd is not None else None
        self.items, self.key = items, key


class WeightStager:
    """"Weight shadow" of a whole model, refreshed by ONE launch per optimizer step (SURVEY.md §8(f) row 2).

    ``stage()`` writes mask * w of every masked layer, at the current precision (bf16, or float32 inside
    ``compute_precision(torch.float32)``), into persistent fprop / dgrad operand buffers and hands them to the layers;
    each layer consumes its ``Staged`` pair in its next forward (exactly once) instead of launching its own staging
    kernel — the reference's per-layer ``mask * weight`` + autocast cast (mask_layers.py:25-34) become one kernel per
    step.  Call it right before the training forward; a forward without a preceding ``stage()`` (eval, pruning scores)
    stages per layer.  Pointers are re-checked every call (pruning replaces mask tensors), the device table is only
    re-uploaded when they changed, so the call is CUDA-graph capturable after a warm-up step."""

    def __init__(self, layers):
        self.layers = list(layers)
        self._shadows = {}                 # precision -> _Shadow

    def stage(self):
        lib = _cabi.load()
        for l in self.layers:                                  # masks created on the host move with the first use
            if l.mask.device != l.weight.device or l.mask.dtype != torch.float32 or not l.mask.is_contiguous():
                l.mask = l.mask.to(device=l.weight.device, dtype=torch.float32).contiguous()
        key = tuple((l.weight.data_ptr(), l.mask.data_ptr()) for l in self.layers)
        dtype = current_precision()
        sh = self._shadows.get(dtype)
        if sh is None:
            sh = self._shadows[dtype] = _Shadow(self.layers, dtype)
        cached = key == sh.key
        if not cached:
            sh.set_table(key)
        if not sh.staged:
            return
        dev = self.layers[0].weight.device
        with torch.cuda.device(dev):
            if dtype == torch.bfloat16:
                rc = lib.tp_stage_weights_batched(sh.items, len(sh.staged), int(cached), c_void_p(sh.kmask_all.data_ptr()),
                                                  sh.kmask_all.numel() * 4, c_void_p(sh.ws.data_ptr()), sh.ws.numel(),
                                                  _cabi.stream_ptr(dev))
                _cabi.check(rc, "tp_stage_weights_batched")
            else:
                rc = lib.tp_stage_weights_batched_f32(sh.items, len(sh.staged), int(cached), c_void_p(sh.ws.data_ptr()),
                                                      sh.ws.numel(), _cabi.stream_ptr(dev))
                _cabi.check(rc, "tp_stage_weights_batched_f32")
        _count()
        for l, st in sh.staged:
            l.__dict__["_tp_staged"] = st

    def shadow(self, dtype=torch.bfloat16):
        """(layer, Staged) of every layer ``stage()`` covers at ``dtype``; empty before the first ``stage()`` there."""
        sh = self._shadows.get(dtype)
        return list(sh.staged) if sh is not None else []

    def drop(self):
        """Take back what the last ``stage()`` handed out and no forward consumed."""
        for l in self.layers:
            l.__dict__.pop("_tp_staged", None)


def skipped_block_report(stager):
    """After ``stager.stage()``: per layer and in total, how many 64x64 blocks of the fprop weight operand are empty
    (never loaded / multiplied).  For iid unstructured masks this is ~0 at any density a 64x64 block survives
    (SURVEY.md Appendix B); dead filters / dead input channels are what produces skippable blocks."""
    rows, empty, total = [], 0, 0
    for l, st in stager.shadow(torch.bfloat16):
        e, t = kblock_occupancy(st.wf.kmask, st.wf.shape[1])
        rows.append((type(l).__name__, tuple(l.weight.shape), e, t))
        empty += e; total += t
    return {"empty_blocks": empty, "total_blocks": total, "fraction": empty / max(total, 1), "layers": rows}


def take_staged(layer):
    """The ``Staged`` operands a ``WeightStager`` left for this layer's next forward, or None; consumed exactly once.
    Operands staged at another precision than the current one are dropped."""
    st = layer.__dict__.pop("_tp_staged", None)
    return st if st is not None and st.wf.dtype == current_precision() else None


def to_nhwc_bf16(x, c_pad):
    """[N, C, H, W] (any strides; fp32 or bf16) -> contiguous NHWC bf16 [N, H, W, c_pad]."""
    lib = _cabi.load()
    n, c, h, w = x.shape
    if x.dtype == torch.bfloat16 and c == c_pad and x.permute(0, 2, 3, 1).is_contiguous():
        return x.permute(0, 2, 3, 1)
    if x.dtype not in (torch.float32, torch.bfloat16):
        x = x.float()
    out = torch.empty(n, h, w, c_pad, dtype=torch.bfloat16, device=x.device)
    sn, sc, sh, sw = x.stride()
    with torch.cuda.device(x.device):
        rc = lib.tp_to_nhwc_bf16(c_void_p(x.data_ptr()), 0 if x.dtype == torch.float32 else 1, sn, sc, sh, sw,
                                 n, c, h, w, c_void_p(out.data_ptr()), c_pad, _cabi.stream_ptr(x.device))
    _cabi.check(rc, "tp_to_nhwc_bf16")
    _count()
    return out


def empty_cl(n, c, h, w, device, dtype=torch.bfloat16):
    """[n, c, h, w] bf16 with channels_last strides: the memory IS an NHWC array, and the tensor is not a view
    (autograd forbids in-place ops such as nn.ReLU(inplace=True) on views created inside a custom Function)."""
    return torch.empty((n, c, h, w), dtype=dtype, device=device, memory_format=torch.channels_last)


def im2col_stem(x, desc, kp, cg):
    """[N, C<=8, H, W] fp32/bf16 (any strides) -> [N*P*Q, kp] bf16 im2col matrix (column tap*cg + channel), conversion fused in."""
    lib = _cabi.load()
    n, c, h, w = x.shape
    if x.dtype not in (torch.float32, torch.bfloat16):
        x = x.float()
    out = torch.empty(n * desc.p * desc.q, kp, dtype=torch.bfloat16, device=x.device)
    sn, sc, sh, sw = x.stride()
    with torch.cuda.device(x.device):
        rc = lib.tp_im2col_stem(c_void_p(x.data_ptr()), 0 if x.dtype == torch.float32 else 1, sn, sc, sh, sw, n, c, h, w,
                                desc.r, desc.s, cg, desc.stride_h, desc.stride_w, desc.pad_h, desc.pad_w, desc.p, desc.q,
                                c_void_p(out.data_ptr()), kp, _cabi.stream_ptr(x.device))
    _cabi.check(rc, "tp_im2col_stem")
    _count()
    return out


def conv_fprop(desc, x_nhwc, wf, bias=None, out=None, want_stats=False):
    """``want_stats``: also return the BatchNorm batch statistics of the output, written by the conv epilogue
    ([rows, 2, cout] fp32: per 32-pixel group and channel the sum and the sum of squares of the bf16 outputs)."""
    lib = _cabi.load()
    dev = x_nhwc.device
    y = out if out is not None else torch.empty(desc.n, desc.p, desc.q, desc.cout, dtype=torch.bfloat16, device=dev)
    stats = None
    if want_stats:
        stats = torch.empty(int(lib.tp_conv_stats_rows(ctypes.byref(desc))), 2, desc.cout, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev), _Timed("fprop", desc):
        km = getattr(wf, "kmask", None) if KBLOCK_SKIP else None
        rc = lib.tp_conv_fprop_stats(ctypes.byref(desc), c_void_p(x_nhwc.data_ptr()), c_void_p(wf.data_ptr()),
                                     c_void_p(km.data_ptr()) if km is not None else None,
                                     c_void_p(bias.data_ptr()) if bias is not None else None, c_void_p(y.data_ptr()),
                                     c_void_p(stats.data_ptr()) if stats is not None else None,
                                     None, 0, _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_conv_fprop")
    _count()
    return (y, stats) if want_stats else y


def conv_dgrad(desc, dy_nhwc, wd, addend=None, kmask=None):
    """dx = dgrad(dy) [+ addend]: ``addend`` (NHWC bf16, dx's shape) is accumulated in the kernel epilogue.
    ``kmask``: K-block occupancy mask of ``wd`` (defaults to the one riding on the tensor)."""
    lib = _cabi.load()
    dev = dy_nhwc.device
    dx = torch.empty(desc.n, desc.h, desc.w, desc.cin, dtype=torch.bfloat16, device=dev)
    with torch.cuda.device(dev), _Timed("dgrad", desc):
        km = (kmask if kmask is not None else getattr(wd, "kmask", None)) if KBLOCK_SKIP else None
        rc = lib.tp_conv_dgrad(ctypes.byref(desc), c_void_p(dy_nhwc.data_ptr()), c_void_p(wd.data_ptr()),
                               c_void_p(km.data_ptr()) if km is not None else None,
                               c_void_p(addend.data_ptr()) if addend is not None else None,
                               c_void_p(dx.data_ptr()), None, 0, _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_conv_dgrad")
    _count(1 if desc.stride_h == 1 and desc.stride_w == 1 else desc.stride_h * desc.stride_w)
    return dx


BN_BWD_FUSION = True     # dgrad epilogue does the BatchNorm backward reduction of the layer that feeds the convolution


def set_bn_bwd_fusion(on: bool):
    global BN_BWD_FUSION
    BN_BWD_FUSION = bool(on)


def conv_dgrad_bnrelu(desc, dy_nhwc, wd, bn_src, kmask=None):
    """dgrad whose result is the gradient of a BatchNorm+ReLU output: returns (g, partial) with g = dx * [z > 0] and the
    per-32-pixel partial sums (sum g, sum g * xhat) the BatchNorm backward needs; None when the shape has no staged path."""
    lib = _cabi.load()
    dev = dy_nhwc.device
    y, weight, bias, mean, invstd = bn_src[:5]
    g = torch.empty(desc.n, desc.h, desc.w, desc.cin, dtype=torch.bfloat16, device=dev)
    rows = int(lib.tp_conv_dgrad_partial_rows(ctypes.byref(desc)))
    partial = torch.empty(rows, 2, desc.cin, dtype=torch.float32, device=dev)
    km = (kmask if kmask is not None else getattr(wd, "kmask", None)) if KBLOCK_SKIP else None
    P = lambda t: c_void_p(t.data_ptr()) if t is not None else None
    with torch.cuda.device(dev), _Timed("dgrad", desc):
        rc = lib.tp_conv_dgrad_bnrelu(ctypes.byref(desc), P(dy_nhwc), P(wd), P(km), P(y), P(weight), P(bias), P(mean), P(invstd),
                                      P(g), P(partial), _cabi.stream_ptr(dev))
    if rc == -5:          # TP_ERR_UNSUPPORTED: no 16-byte aligned linear output for this shape
        return None
    _cabi.check(rc, "tp_conv_dgrad_bnrelu")
    _count()
    return g, partial


def conv_wgrad(desc, x_nhwc, dy_nhwc, mask4d, cin_real, want_db=False, dw_out=None, db_out=None, kmask=None):
    """``dw_out`` / ``db_out``: write the gradients straight into these (contiguous fp32) buffers — used with the
    persistent gradient arena so no separate accumulate kernel runs.  ``kmask``: the fprop occupancy mask staged for
    ``mask4d`` (``wf.kmask``): output tiles under all-zero mask blocks are skipped (their gradient is zero)."""
    lib = _cabi.load()
    dev = x_nhwc.device
    dw = dw_out if dw_out is not None else torch.empty(desc.cout, cin_real, desc.r, desc.s, dtype=torch.float32, device=dev)
    db = (db_out if db_out is not None else torch.empty(desc.cout, dtype=torch.float32, device=dev)) if want_db else None
    nbytes = lib.tp_conv_workspace_bytes(ctypes.byref(desc), 2)
    wsb = _workspace(nbytes, dev, "wgrad")
    with torch.cuda.device(dev), _Timed("wgrad", desc):
        km = kmask if KBLOCK_SKIP else None
        rc = lib.tp_conv_wgrad(ctypes.byref(desc), c_void_p(x_nhwc.data_ptr()), c_void_p(dy_nhwc.data_ptr()),
                               c_void_p(mask4d.data_ptr()), c_void_p(km.data_ptr()) if km is not None else None,
                               cin_real, c_void_p(dw.data_ptr()),
                               c_void_p(db.data_ptr()) if db is not None else None,
                               c_void_p(wsb.data_ptr()), wsb.numel(), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_conv_wgrad")
    _count(3 if want_db else 2)
    return dw, db


# ---- fp32 (TF32) masked layers: inside compute_precision(torch.float32) ------------------------------------------------
def stage_weights_f32(weight4d, mask4d, cin_p, need_dgrad, cout_p=None, wf_ld=0):
    """fp32 mask*w in the layouts of ``stage_weights`` (no occupancy masks)."""
    lib = _cabi.load()
    cout, cin, r, s = weight4d.shape
    dev = weight4d.device
    wf = torch.zeros(cout, wf_ld, dtype=torch.float32, device=dev) if wf_ld and wf_ld > r * s * cin_p else \
        torch.empty(cout, r * s * cin_p, dtype=torch.float32, device=dev)
    cout_p = cout if cout_p is None else cout_p
    wd = torch.empty(cin, r * s * cout_p, dtype=torch.float32, device=dev) if need_dgrad else None
    with torch.cuda.device(dev):
        rc = lib.tp_stage_weights_f32(c_void_p(weight4d.data_ptr()), c_void_p(mask4d.data_ptr()), cout, cin, r, s,
                                      c_void_p(wf.data_ptr()), cin_p, int(wf_ld), c_void_p(wd.data_ptr()) if wd is not None else None,
                                      cout_p, _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_stage_weights_f32")
    _count()
    return wf, wd


def to_nhwc_f32(x, c_pad):
    """[N, C, H, W] fp32 (any strides) -> NHWC fp32 [N, H, W, c_pad]: a view when x already is channels_last with C == c_pad."""
    n, c, h, w = x.shape
    if x.dtype != torch.float32:
        raise TypeError(f"to_nhwc_f32: fp32 input expected, got {x.dtype}")
    if c == c_pad and x.permute(0, 2, 3, 1).is_contiguous():
        return x.permute(0, 2, 3, 1)
    lib = _cabi.load()
    out = torch.empty(n, h, w, c_pad, dtype=torch.float32, device=x.device)
    sn, sc, sh, sw = x.stride()
    with torch.cuda.device(x.device):
        rc = lib.tp_to_nhwc_f32(c_void_p(x.data_ptr()), sn, sc, sh, sw, n, c, h, w, c_void_p(out.data_ptr()), c_pad,
                                _cabi.stream_ptr(x.device))
    _cabi.check(rc, "tp_to_nhwc_f32")
    _count()
    return out


def im2col_stem_f32(x, desc, kp, cg):
    """[N, C<=8, H, W] fp32 (any strides) -> [N*P*Q, kp] fp32 im2col matrix (the layout of ``im2col_stem``)."""
    lib = _cabi.load()
    n, c, h, w = x.shape
    out = torch.empty(n * desc.p * desc.q, kp, dtype=torch.float32, device=x.device)
    sn, sc, sh, sw = x.stride()
    with torch.cuda.device(x.device):
        rc = lib.tp_im2col_stem_f32(c_void_p(x.data_ptr()), sn, sc, sh, sw, n, c, h, w, desc.r, desc.s, cg, desc.stride_h,
                                    desc.stride_w, desc.pad_h, desc.pad_w, desc.p, desc.q, c_void_p(out.data_ptr()), kp,
                                    _cabi.stream_ptr(x.device))
    _cabi.check(rc, "tp_im2col_stem_f32")
    _count()
    return out


def conv_fprop_f32(desc, x_nhwc, wf, bias=None, out=None):
    lib = _cabi.load()
    dev = x_nhwc.device
    y = out if out is not None else torch.empty(desc.n, desc.p, desc.q, desc.cout, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev), _Timed("fprop", desc):
        rc = lib.tp_conv_fprop_f32(ctypes.byref(desc), c_void_p(x_nhwc.data_ptr()), c_void_p(wf.data_ptr()),
                                   c_void_p(bias.data_ptr()) if bias is not None else None, c_void_p(y.data_ptr()),
                                   _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_conv_fprop_f32")
    _count()
    return y


def conv_dgrad_f32(desc, dy_nhwc, wd):
    lib = _cabi.load()
    dev = dy_nhwc.device
    dx = torch.empty(desc.n, desc.h, desc.w, desc.cin, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev), _Timed("dgrad", desc):
        rc = lib.tp_conv_dgrad_f32(ctypes.byref(desc), c_void_p(dy_nhwc.data_ptr()), c_void_p(wd.data_ptr()),
                                   c_void_p(dx.data_ptr()), _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_conv_dgrad_f32")
    _count()
    return dx


def wgrad_split3(x, c_pad, lo_block):
    """fp32 [N, C, H, W] (any strides) -> NHWC bf16 [3N, H, W, c_pad]: image block ``lo_block`` holds bf16(v - bf16(v)),
    the other two bf16(v) (see ``conv_wgrad_f32``)."""
    lib = _cabi.load()
    n, c, h, w = x.shape
    out = torch.empty(3 * n, h, w, c_pad, dtype=torch.bfloat16, device=x.device)
    sn, sc, sh, sw = x.stride()
    with torch.cuda.device(x.device):
        rc = lib.tp_wgrad_split3(c_void_p(x.data_ptr()), sn, sc, sh, sw, n, c, h, w, c_void_p(out.data_ptr()), c_pad, int(lo_block),
                                 _cabi.stream_ptr(x.device))
    _cabi.check(rc, "tp_wgrad_split3")
    _count()
    return out


def split_stacks(desc, x, dy, dy_c_pad):
    """The bf16 stacks of the fp32 weight gradient: x [N, cin, H, W] as (hi, lo, hi), dy [N, cout, P, Q] as (hi, hi, lo)."""
    return wgrad_split3(x, desc.cin, 1), wgrad_split3(dy, dy_c_pad, 2)


def conv_wgrad_f32(desc, xs, dys, mask4d, cin_real, dw_out=None):
    """fp32 masked weight gradient from the stacks of ``split_stacks``: ONE bf16 ``conv_wgrad`` over 3N images sums
    x_hi dy_hi + x_lo dy_hi + x_hi dy_lo in its deterministic split-K fold (TF32 wgmma cannot read the MN-major operands
    of the pixel contraction).  hi + lo carries 16 significant bits, so each product is within about 2^-16 relative
    (the dropped x_lo dy_lo term and the rounding of lo) — closer than TF32's 2^-10 per operand.  No bias gradient here:
    the stacked column sum would count dy_hi twice."""
    d3 = _cabi.ConvDesc(3 * desc.n, desc.h, desc.w, desc.cin, desc.cout, desc.r, desc.s, desc.stride_h, desc.stride_w,
                        desc.pad_h, desc.pad_w, desc.p, desc.q)
    dw, _ = conv_wgrad(d3, xs, dys, mask4d, cin_real, False, dw_out=dw_out)
    return dw


def _check_f32(x, want_skip, want_stats):
    if want_skip or want_stats:
        raise RuntimeError("masked_conv2d at float32: the skip-gradient and BatchNorm-statistics epilogues exist in bf16 "
                           "only (a float32 model runs unfused)")
    if x.dtype != torch.float32:
        raise TypeError(f"masked layers at float32 need fp32 activations, got {x.dtype}")


class _Precision(NamedTuple):
    """What a masked layer does differently at each compute precision; ``MaskedConv2dFn`` is written once against it."""
    act: torch.dtype                # activations, operands and input gradients
    check: Callable                 # (x, want_skip, want_stats): raises for what this precision cannot run
    stage: Callable                 # per-layer staging, as ``stage_weights``
    nhwc: Callable                  # (x [N, C, H, W], c_pad) -> NHWC
    im2col: Callable                # the stem's im2col, as ``im2col_stem``
    fprop: Callable                 # (desc, x, wf, bias, out=y)
    dy: Callable                    # (dy, cout_p): the form of dy the backward works from
    dgrad: Callable                 # (desc, dy in that form, wd, addend, kmask) -> NHWC dx
    wgrad_operands: Callable        # (desc, x as logical NCHW, dy in that form) -> the GEMM operands, made on the current stream
    wgrad: Callable                 # (desc, x, dy, mask, cin_real, want_db, dw_out, db_out, kmask) -> (dw, db)
    colsum_db: bool                 # wgrad also forms the bias gradient, as the column sums of dy


_PRECISIONS = {
    # dy laid out once as NHWC bf16; one conv_wgrad, the bias gradient from its column sums
    torch.bfloat16: _Precision(
        act=torch.bfloat16, check=lambda x, want_skip, want_stats: None, stage=stage_weights, nhwc=to_nhwc_bf16,
        im2col=im2col_stem, fprop=conv_fprop, dy=to_nhwc_bf16, dgrad=conv_dgrad,
        wgrad_operands=lambda desc, x, dy: (x, dy), wgrad=conv_wgrad, colsum_db=True),
    # dy stays fp32 NCHW: dgrad lays it out, the weight gradient is one conv_wgrad over the split stacks of 3N images,
    # and the bias gradient is dy.sum in fp32
    torch.float32: _Precision(
        act=torch.float32, check=_check_f32, stage=stage_weights_f32, nhwc=to_nhwc_f32, im2col=im2col_stem_f32,
        fprop=conv_fprop_f32, dy=lambda dy, c_pad: dy.float(),
        dgrad=lambda desc, dy, wd, addend, kmask: conv_dgrad_f32(desc, to_nhwc_f32(dy, desc.cout), wd),
        wgrad_operands=lambda desc, x, dy: split_stacks(desc, x, dy, desc.cout),
        wgrad=lambda desc, xs, dys, mask, cin, want_db, dw_out=None, db_out=None, kmask=None:
            (conv_wgrad_f32(desc, xs, dys, mask, cin, dw_out=dw_out), None),
        colsum_db=False),
}


def _on_wgrad_stream(fn, *operands):
    """``fn()`` on the side stream, behind an event of the current stream.  Every operand is marked as in use by the side
    stream, so the caching allocator hands its block to no other allocation before the side stream is done with it: the
    operands are freed as soon as this GEMM is done, not at ``join_wgrad``."""
    dev = operands[0].device
    side = _wgrad_stream(dev)
    ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(dev))
    side.wait_event(ev)
    with torch.cuda.stream(side):
        out = fn()
    for t in operands:
        t.record_stream(side)
    _wgrad_pending.add(dev)
    return out


class MaskedConv2dFn(torch.autograd.Function):
    """y = conv2d(x, mask*w, b) with tensor-core operands and fp32 accumulation, at the current compute precision.

    Replaces ``F.conv2d(x, mask * weight, ...)`` under bf16 autocast (reference
    utils/mask_layers.py:23-34 executed inside base_harness.py:121-125) and its autograd
    backward: dX = dgrad(dY, mask*w), dW = mask * wgrad(x, dY) in fp32, db = sum dY.
    Activations stay NHWC (logical NCHW tensors with channels_last strides), bf16 or fp32.
    """

    @staticmethod
    def forward(ctx, x, weight, mask, bias, stride, padding, want_skip=False, grad_slots=None, staged=None, want_stats=False,
                bn_src=None):
        _require_cuda(x, weight, mask)
        P = ctx.prec = _PRECISIONS[current_precision()]    # read once, like dense: backward runs on autograd's thread
        P.check(x, want_skip, want_stats)
        ctx.dense = dense_grad_enabled()                  # dW = wgrad(x, dy), unmasked
        ctx.set_materialize_grads(False)
        ctx.want_skip = want_skip
        # (w_slot, b_slot): persistent arena slots; when given, backward writes dW / db there and returns None for
        # them (no AccumulateGrad add kernel; the slot IS param.grad)
        ctx.grad_slots = grad_slots
        cout, cin, r, s = weight.shape
        n = x.shape[0]
        need_dx = ctx.needs_input_grad[0]
        m32 = mask.detach().contiguous()
        plan = ctx.plan = layer_plan(cout, cin, r, s, need_dx)
        desc, fdesc, ctx.wdesc, ctx.xdesc = _layer_descs(plan, weight.shape, x.shape, stride, padding)
        if plan.stem:
            xin = P.im2col(x, desc, plan.wf_ld, plan.cin_p)
        else:
            xin = P.nhwc(x, plan.cin_p)      # channels cin..cin_p are zero (and so are the staged weights there)
        if staged is not None and staged.plan == plan:
            wf, wd = staged.wf, staged.wd    # refreshed by WeightStager.stage() for this step (one launch for all layers)
        else:
            # nothing staged (eval, pruning scores), or a stem layout for a layer whose input needs a gradient here
            wf, wd = P.stage(weight.detach().contiguous(), m32, plan.cin_p, need_dx, plan.cout_p,
                             wf_ld=plan.wf_ld if plan.stem else 0)
        y = empty_cl(n, cout, desc.p, desc.q, x.device, P.act)
        stats = None
        if want_stats:
            _, stats = conv_fprop(fdesc, xin, wf, bias, out=y, want_stats=True)
        else:
            P.fprop(fdesc, xin, wf, bias, out=y)
        # x is the output of a fused BatchNorm+ReLU (no residual): this layer's dgrad can do that BatchNorm's backward
        # reduction in its epilogue (stride 1, no channel padding, the NHWC buffers line up)
        ctx.bn_src = None
        if (bn_src is not None and BN_BWD_FUSION and need_dx and not want_skip and stride == (1, 1) and plan.cin_p == cin
                and bn_src[0].shape == xin.shape):
            ctx.bn_src = bn_src
        ctx.wd_kmask = getattr(wd, "kmask", None)      # attributes do not survive save_for_backward
        ctx.wf_kmask = getattr(wf, "kmask", None)      # wgrad skips tiles under all-zero mask blocks
        # wgrad reads the activation as a logical NCHW tensor; the stem's im2col rows are 1x1 images of kp channels
        ctx.save_for_backward(xin.view(-1, plan.wf_ld, 1, 1) if plan.stem else xin.permute(0, 3, 1, 2), m32, wd)
        ctx.desc = desc
        ctx.cin = cin
        ctx.has_bias = bias is not None
        ctx.x_dtype = x.dtype
        if want_skip:
            # second output = the input itself: whatever gradient reaches it (the identity path of a residual
            # block, or a downsample branch) comes back to backward() as ``dskip`` and is accumulated inside
            # the dgrad epilogue instead of by autograd's separate elementwise add
            if want_stats:
                ctx.mark_non_differentiable(stats)
                return y, x, stats
            return y, x
        if want_stats:
            ctx.mark_non_differentiable(stats)
            return y, stats
        return y

    @staticmethod
    def backward(ctx, dy, *rest):
        # outputs were (y [, x_skip] [, stats]); the statistics output is non-differentiable
        dskip = rest[0] if ctx.want_skip and rest else None
        if dy is None:          # only the skip output was used downstream
            return dskip, None, None, None, None, None, None, None, None, None, None
        P, plan, desc = ctx.prec, ctx.plan, ctx.desc
        cout = desc.cout
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_db = ctx.has_bias and ctx.needs_input_grad[3]
        want_db = need_db and P.colsum_db
        dyl = P.dy(dy, plan.cout_p)
        x, m32, wd = ctx.saved_tensors
        dx = dw = db = None
        db_in_slot = False          # the bias gradient already sits in param.grad's arena slot: return None for it
        if need_dx:
            addend = to_nhwc_bf16(dskip, ctx.cin) if dskip is not None else None
            fused = None
            if ctx.bn_src is not None and addend is None:
                fused = conv_dgrad_bnrelu(ctx.xdesc, dyl, wd, ctx.bn_src, kmask=ctx.wd_kmask)
            if fused is not None:
                g, partial = fused
                from . import fused_norm
                fused_norm.offer_partials(g, partial, ctx.bn_src[5])          # picked up by that BatchNorm's backward
                dx = g.permute(0, 3, 1, 2)
            else:
                # dX has the REAL channel count: the dgrad GEMM's N axis is cin, its K axis (taps x cout_p)
                dx = P.dgrad(ctx.xdesc, dyl, wd, addend, ctx.wd_kmask).permute(0, 3, 1, 2)
            if dx.dtype != ctx.x_dtype:
                dx = dx.to(ctx.x_dtype)
        if need_dw:
            xa, dya = P.wgrad_operands(ctx.wdesc, x, dyl)
            # dense: all-ones mask and no occupancy mask, so every tile of dW is computed
            m, kmask = (_ones_like_mask(m32), None) if ctx.dense else (m32, ctx.wf_kmask)
            if plan.stem:
                # all kp columns (tap, channel) of the im2col GEMM: back to OIHW and apply the mask (9.4 k elements)
                ones = torch.ones(cout, plan.wf_ld, 1, 1, dtype=torch.float32, device=m32.device)
                dwm, db = P.wgrad(ctx.wdesc, xa, dya, ones, plan.wf_ld, want_db)
                cin, r, s = m32.shape[1:]
                dw = dwm[:, :r * s * cin].reshape(cout, r * s, cin).permute(0, 2, 1).reshape(cout, cin, r, s)
                if not ctx.dense:
                    dw = dw * m32
            elif plan.cout_p != cout:
                m_p = torch.zeros(plan.cout_p, *m.shape[1:], dtype=torch.float32, device=m.device)
                m_p[:cout] = m
                dwp, dbp = P.wgrad(ctx.wdesc, xa, dya, m_p, ctx.cin, want_db)
                dw = dwp[:cout].contiguous()
                db = dbp[:cout].contiguous() if dbp is not None else None
            else:
                ws_, bs_ = ctx.grad_slots if ctx.grad_slots is not None else (None, None)
                dw_out = ws_ if ws_ is not None and ws_.is_contiguous() and ws_.numel() == m.numel() else None
                db_out = bs_ if want_db else None

                def run():
                    out = P.wgrad(ctx.wdesc, xa, dya, m, ctx.cin, want_db, dw_out, db_out, kmask)
                    grad_ready(dw_out, db_out)
                    return out
                if WGRAD_SIDE_STREAM and dw_out is not None and (db_out is not None or not want_db):
                    dw, db = _on_wgrad_stream(run, xa, dya, m)   # nothing of it flows back through autograd
                else:
                    dw, db = run()
                if dw_out is not None:
                    dw = None
                if db_out is not None:
                    db, db_in_slot = None, True
        if need_db and db is None and not db_in_slot:
            db = dy.float().sum(dim=(0, 2, 3))
        return dx, dw, None, db, None, None, None, None, None, None, None


def masked_conv2d(x, weight, mask, bias=None, stride=(1, 1), padding=(0, 0), want_skip=False, grad_slots=None, staged=None,
                  want_stats=False, bn_src=None):
    """Returns y, or (y, x_skip) with ``want_skip``, with the BatchNorm statistics tensor appended for ``want_stats``.
    ``bn_src``: what ``BatchNorm2dB200`` attaches to its BatchNorm+ReLU output (``x._tp_bn_src``)."""
    return MaskedConv2dFn.apply(x, weight, mask, bias, tuple(stride), tuple(padding), want_skip, grad_slots, staged, want_stats,
                                bn_src)


def masked_linear(x, weight2d, mask2d, bias=None, grad_slots=None, staged=None):
    """y = x @ (mask*w)^T + b for x [..., in]; runs as a 1x1 convolution over a [rows,1,1,in] image."""
    shp = x.shape
    x2 = x.reshape(-1, shp[-1])
    y = MaskedConv2dFn.apply(x2.view(x2.shape[0], x2.shape[1], 1, 1), weight2d.view(*weight2d.shape, 1, 1),
                             mask2d.view(*mask2d.shape, 1, 1), bias, (1, 1), (0, 0), False, grad_slots, staged)
    return y.reshape(*shp[:-1], weight2d.shape[0])
