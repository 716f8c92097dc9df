"""Data-parallel gradient exchange over NVLink peer memory (replaces DDP's Reducer + NCCL).

The reference wraps the model in ``DistributedDataParallel`` with default settings
(harness_definitions/base_harness.py:81): per-bucket ``grad / W`` -> ``ncclAllReduce(SUM)`` ->
copy back, plus a broadcast of every buffer (all masks!) from rank 0 on every forward.  Here:

  * gradients are packed into a few large buckets that live in *symmetric memory*
    (``torch.distributed._symmetric_memory``: every rank's bucket is mapped into every peer's
    address space over NVLink / NVSwitch);
  * one ``tp_p2p_allreduce_mask`` kernel per bucket reads the peers' copies directly, sums them
    in fixed rank order (bit-identical result on every rank), scales by 1/W, applies the mask
    and leaves the result in the local bucket — ``param.grad`` then simply views the bucket;
  * nothing else is exchanged: masks are deterministic functions of replica-identical state, so
    the reference's per-step mask broadcast disappears.  torch.distributed (NCCL) is only used
    for rendezvous and scalar reductions.
"""
import ctypes
from ctypes import c_void_p

import torch
import torch.distributed as dist

from . import _cabi, ops

PAD_FLOATS = 1024          # 4 KiB of signal-pad slots at the head of every symmetric bucket


def plan_buckets(numels, cap_elems):
    """Pure host logic: pack parameters (given in REVERSE registration order, i.e. the order gradients become
    ready) into buckets of at most ``cap_elems`` fp32 slots; every slot is padded to a multiple of 4 elements so it
    stays 16-byte aligned.  Returns [(indices, offsets, total_elems)].  Must be identical on every rank."""
    buckets, cur, offs, total = [], [], [], 0
    for i, n in enumerate(numels):
        slot = (n + 3) // 4 * 4
        if cur and total + slot > cap_elems:
            buckets.append((cur, offs, total)); cur, offs, total = [], [], 0
        cur.append(i); offs.append(total); total += slot
    if cur:
        buckets.append((cur, offs, total))
    return buckets


def shard_bounds(numel, world):
    """float4-granular shard [s0, s1) of every rank for the two-shot algorithm (mirrors k_p2p_allreduce<1>)."""
    n4 = numel // 4
    per = (n4 + world - 1) // world
    return [(min(n4, per * r) * 4, min(n4, min(n4, per * r) + per) * 4) for r in range(world)]


class GradArena:
    """Persistent, flat gradient storage for ONE rank: ``param.grad`` permanently views a 16-byte aligned slot of
    one fp32 buffer, ``zero()`` is a single memset.  Pointers never change, so the fused SGD keeps its device-side
    pointer table and the whole train step can be captured into a CUDA graph (autograd accumulates into the
    zeroed slots: 0 + g == g bit-exactly, same values as the reference's zero_grad + assign)."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        (idx, offs, total), = plan_buckets([p.numel() for p in self.params], 1 << 62)
        self.flat = torch.zeros(total, dtype=torch.float32, device=self.params[0].device)
        self.views = [self.flat[o:o + p.numel()].view_as(p) for o, p in zip(offs, self.params)]
        self.attach()

    def attach(self):
        for p, v in zip(self.params, self.views):
            p.grad = v
            p._tp_grad_slot = v          # masked layers / fused BN write their gradients straight into the slot

    def zero(self):
        self.flat.zero_()
        self.attach()


class P2PGradReducer:
    """Gradient mean over NVLink peer memory, one kernel per bucket, overlapped with the backward pass.

    ``algo``: "one_shot" | "two_shot" | "nvls" | "auto".  "nvls" is the two-shot schedule with the reduction and the
    broadcast done INSIDE the NVSwitch (``multimem.ld_reduce`` / ``multimem.st`` on the symmetric allocation's
    multicast address): rank r pulls the switch-reduced shard r, scales / masks it and stores it once to the
    multicast address.  The switch's summation order is fixed by the fabric, not by us: replicas stay
    bit-identical (every replica receives the value rank r computed), but against the fixed rank-order sum the result
    may differ in the last bits of the LARGEST summand for W > 2 (tested: |diff| <= 4 eps * sum_r |g_r| / W); "auto" uses
    it from 4 ranks on (TP_P2P_NVLS=0/1 overrides; the crossover was chosen on an earlier GPU generation and is not
    re-measured on H100).

    Overlap: the masked layers / fused BN (which write their gradients straight into the bucket slots) and autograd's
    post-accumulate hooks (all other parameters) report every finished gradient through ``notify``; when the last
    gradient of a bucket is in, that bucket's kernel is launched on a side stream behind an event of the compute
    stream, so it runs under the rest of the backward pass (the reference's DDP does the same with NCCL,
    base_harness.py:81,127).  ``reduce()`` after ``loss.backward()`` launches whatever is left and joins the side
    stream.  Under CUDA-graph capture the same calls become a forked branch of the graph.
    """

    def __init__(self, params, bucket_cap_mb=25.0, algo="auto", group=None, masks=None, overlap=True):
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group or dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.params = [p for p in params if p.requires_grad]
        self.algo = algo
        dev = self.params[0].device
        self.device = dev
        cap = int(bucket_cap_mb * 1024 * 1024 / 4)
        # reverse order (gradients become ready back to front), like DDP's bucket assignment
        rev = list(reversed(self.params))
        self.plan = plan_buckets([p.numel() for p in rev], cap)
        self.buckets = [[rev[i] for i in idx] for idx, _, _ in self.plan]
        self._bk = []
        self._slot_bucket = {}          # slot data_ptr -> bucket index
        for bi, plist in enumerate(self.buckets):
            offs, total = [], 0
            for p in plist:
                offs.append(total); total += (p.numel() + 3) // 4 * 4
            buf = symm_mem.empty(PAD_FLOATS + total, dtype=torch.float32, device=dev)
            buf.zero_()
            hdl = symm_mem.rendezvous(buf, self.group)
            ptrs = [int(x) for x in hdl.buffer_ptrs]
            data_ptrs = (c_void_p * self.world)(*[c_void_p(x + PAD_FLOATS * 4) for x in ptrs])
            pad_ptrs = (c_void_p * self.world)(*[c_void_p(x) for x in ptrs])
            mc = 0
            try:
                mc = int(hdl.multicast_ptr or 0)
            except Exception:
                mc = 0
            data = buf[PAD_FLOATS:]
            views = [data[o:o + p.numel()].view_as(p) for o, p in zip(offs, plist)]
            algo_id = self._algo_for(total, mc != 0)
            # one-shot: peers read my bucket while I produce the result, so it needs its own
            # output buffer; two-shot / nvls finish in place (only rank r ever reads shard r).
            out = torch.empty(total, dtype=torch.float32, device=dev) if algo_id == 0 else data
            out_views = [out[o:o + p.numel()].view_as(p) for o, p in zip(offs, plist)]
            for v in views:
                self._slot_bucket[v.data_ptr()] = bi
            self._bk.append(dict(buf=buf, hdl=hdl, data=data, views=views, numel=total, params=plist, offs=offs,
                                 data_ptrs=data_ptrs, pad_ptrs=pad_ptrs, mask=None, algo=algo_id, out=out,
                                 out_views=out_views, mc=(mc + PAD_FLOATS * 4) if mc else 0))
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.overlap = bool(overlap)
        self._side = torch.cuda.Stream(dev)
        self._pending = [set() for _ in self._bk]
        self._streams = [dict() for _ in self._bk]
        self._launched = [False] * len(self._bk)
        self._armed = False
        self._hooks = []
        if masks:
            self.set_masks(masks)
        torch.cuda.synchronize(dev)
        dist.barrier(self.group)

    # -- configuration -----------------------------------------------------------------------------------------
    def _algo_for(self, numel, has_mc):
        if self.algo == "one_shot":
            return 0
        if self.algo == "two_shot":
            return 1
        if self.algo == "nvls":
            if not has_mc:
                raise RuntimeError("P2PGradReducer(algo='nvls'): the symmetric allocation has no multicast address")
            return 2
        if numel * 4 <= (1 << 20):
            return 0
        import os
        # the in-switch path pays off with more ranks (on 2 GPUs two-shot was faster), so it starts at 4 ranks;
        # TP_P2P_NVLS=0/1 overrides
        nvls = os.environ.get("TP_P2P_NVLS")
        use = (self.world >= 4) if nvls is None else (nvls == "1")
        return 2 if (has_mc and use) else 1

    def set_masks(self, masks):
        """``masks``: {id(param): mask tensor}.  The kernel multiplies the averaged gradient by it while writing it
        back ("already-masked gradients", BASELINE.json north_star); parameters without an entry get ones."""
        for bk in self._bk:
            if not any(id(p) in masks for p in bk["params"]):
                bk["mask"] = None
                continue
            m = bk["mask"]
            if m is None:
                m = torch.ones(bk["numel"], dtype=torch.float32, device=self.device)
            for o, p in zip(bk["offs"], bk["params"]):
                if id(p) in masks:
                    m[o:o + p.numel()] = masks[id(p)].reshape(-1).to(device=self.device, dtype=torch.float32)
                else:
                    m[o:o + p.numel()] = 1.0
            bk["mask"] = m

    def set_model_masks(self, model):
        """Flat per-bucket copies of every masked layer's mask (call after pruning: once per level)."""
        from .utils.mask_layers import MASKED_LAYER_TYPES
        self.set_masks({id(m.weight): m.mask for m in model.modules() if isinstance(m, MASKED_LAYER_TYPES)})

    # -- overlap machinery -------------------------------------------------------------------------------------
    def _launch_bucket(self, bi, stream):
        lib = _cabi.load()
        bk = self._bk[bi]
        st = c_void_p(stream.cuda_stream)
        mask = c_void_p(bk["mask"].data_ptr()) if bk["mask"] is not None else None
        if bk["algo"] == 2:
            rc = lib.tp_p2p_allreduce_nvls(bk["data_ptrs"], bk["pad_ptrs"], c_void_p(bk["mc"]), self.rank, self.world,
                                           bk["numel"], mask, 1.0 / self.world, c_void_p(bk["out"].data_ptr()),
                                           20000, c_void_p(self.status.data_ptr()), st)
        else:
            rc = lib.tp_p2p_allreduce_mask(bk["data_ptrs"], bk["pad_ptrs"], self.rank, self.world, bk["numel"], mask,
                                           1.0 / self.world, c_void_p(bk["out"].data_ptr()), bk["algo"],
                                           20000, c_void_p(self.status.data_ptr()), st)
        _cabi.check(rc, "tp_p2p_allreduce")
        ops._count()
        self._launched[bi] = True

    def notify(self, slot_ptr):
        """A gradient living at ``slot_ptr`` (a bucket slot) is complete on the current stream."""
        if not self._armed:
            return
        bi = self._slot_bucket.get(slot_ptr)
        if bi is None:
            return
        seen = self._pending[bi]
        seen.add(slot_ptr)                           # a set, not a counter: a gradient reported twice counts once
        # gradients of one bucket are written on DIFFERENT streams (BatchNorm / bias gradients on the compute stream, weight
        # gradients on the wgrad side stream): the exchange has to wait for every stream that contributed, not only for the
        # one that happened to report last (found by the per-level replica checksum on 4 GPUs: ranks diverged)
        cur = torch.cuda.current_stream(self.device)
        self._streams[bi][cur.cuda_stream] = cur
        if len(seen) == len(self._bk[bi]["params"]) and not self._launched[bi]:
            for st in self._streams[bi].values():
                ev = torch.cuda.Event()
                ev.record(st)
                self._side.wait_event(ev)
            with torch.cuda.device(self.device):
                self._launch_bucket(bi, self._side)

    def arm(self):
        """Start counting finished gradients for this step (call after ``zero()``, before the backward pass)."""
        if not self.overlap:
            return
        if not self._hooks:
            for p in self.params:
                self._hooks.append(p.register_post_accumulate_grad_hook(self._post_acc))
        self._pending = [set() for _ in self._bk]
        self._streams = [dict() for _ in self._bk]
        self._launched = [False] * len(self._bk)
        self._armed = True
        ops.set_grad_ready_hook(self.notify)

    def _post_acc(self, p):
        g = p.grad
        if g is not None:
            self.notify(g.data_ptr())

    def close(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []
        if ops.get_grad_ready_hook() == self.notify:
            ops.set_grad_ready_hook(None)

    @torch.no_grad()
    def reduce(self):
        """Average gradients across ranks; afterwards every ``param.grad`` views its bucket slot.  Buckets whose
        kernel already went out during the backward pass are only joined."""
        ops.join_wgrad(self.device)
        armed, self._armed = self._armed, False
        cur = torch.cuda.current_stream(self.device)
        joined = False
        for bi, bk in enumerate(self._bk):
            if armed and self._launched[bi]:
                joined = True
                continue
            grads = [p.grad for p in bk["params"]]
            live = [(v, g) for v, g in zip(bk["views"], grads) if g is not None and g.data_ptr() != v.data_ptr()]
            if live:
                torch._foreach_copy_([v for v, _ in live], [g for _, g in live])
            for v, g in zip(bk["views"], grads):
                if g is None:
                    v.zero_()
            if joined:
                # keep the launch order identical on every rank: buckets launched late go to the side stream too
                ev = torch.cuda.Event(); ev.record(cur); self._side.wait_event(ev)
                with torch.cuda.device(self.device):
                    self._launch_bucket(bi, self._side)
            else:
                with torch.cuda.device(self.device):
                    self._launch_bucket(bi, cur)
        if joined:
            done = torch.cuda.Event(); done.record(self._side); cur.wait_event(done)
        for bk in self._bk:
            for p, v in zip(bk["params"], bk["out_views"]):
                p.grad = v

    def attach(self):
        """Make every ``param.grad`` a persistent view of its bucket slot (stable pointers: CUDA-graph capturable)."""
        for bk in self._bk:
            for p, v in zip(bk["params"], bk["views"]):
                p.grad = v
                p._tp_grad_slot = v

    def zero(self):
        for bk in self._bk:
            bk["data"].zero_()
        self.attach()

    def check_status(self):
        if int(self.status.item()) != 0:
            raise RuntimeError("tp_p2p_allreduce_mask: peer barrier timed out (a rank did not arrive)")


_REDUCERS = {}


def get_reducer(params, **kw):
    """One ``P2PGradReducer`` per (process, parameter set): the level loop builds a new harness around the SAME
    module every level (run_experiment.py:113-115 of the reference) — its symmetric buckets and rendezvous are
    reused instead of being allocated again 21 times."""
    params = [p for p in params if p.requires_grad]
    key = tuple((p.data_ptr(), p.numel()) for p in params)
    red = _REDUCERS.get(key)
    if red is None:
        for k in list(_REDUCERS):                   # a different model in the same process: drop the old buckets
            _REDUCERS.pop(k).close()
        red = _REDUCERS[key] = P2PGradReducer(params, **kw)
    return red
