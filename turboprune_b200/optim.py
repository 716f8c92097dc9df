"""Fused SGD(momentum, weight_decay) — one kernel launch for all parameters — and fused AdamW (``FusedAdamW``).

Same update rule and state layout as ``torch.optim.SGD`` as the reference configures it
(harness_definitions/standard_pruning_harness.py:70-75): ``g += wd*w; buf = mu*buf + g
(buf = g on the first step); w -= lr*buf``.  Masked weights keep decaying because the decay
acts on ``w`` itself.  ``state[p]['momentum_buffer']`` is kept so ``state_dict()`` stays
interchangeable with torch's optimizer (the reference saves optimizer_init.pt / _rewind.pt).

CUDA-graph friendly: the learning rate lives in a device scalar (``sync_lr()`` copies
``param_groups[i]['lr']`` into it; inside a captured step nothing is baked in), and the device-side
pointer table is re-uploaded only when a parameter / gradient / buffer pointer changed.
"""
import math

import torch

from . import _cabi, ops


class FusedSGD(torch.optim.Optimizer):
    def __init__(self, params, lr=0.1, momentum=0.0, weight_decay=0.0, capturable=False):
        defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay, dampening=0, nesterov=False,
                        maximize=False, foreach=None, differentiable=False, fused=None)
        super().__init__(params, defaults)
        self.capturable = capturable
        self._lr_dev = {}
        self._table = {}          # (group, first) -> (pointer signature, workspace tensor)

    def _lr_tensor(self, gi, dev):
        t = self._lr_dev.get((gi, dev))
        if t is None:
            t = self._lr_dev[(gi, dev)] = torch.full((), float(self.param_groups[gi]["lr"]), dtype=torch.float32, device=dev)
        return t

    def sync_lr(self):
        """Copy every group's host lr into its device scalar (call between graph replays)."""
        for (gi, dev), t in self._lr_dev.items():
            t.fill_(float(self.param_groups[gi]["lr"]))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            ps = [p for p in group["params"] if p.grad is not None]
            if not ps:
                continue
            new = [p for p in ps if "momentum_buffer" not in self.state[p]]
            if new and len(new) != len(ps):
                # a parameter got its first gradient late: step the newcomers separately
                self._launch(gi, group, [p for p in ps if "momentum_buffer" in self.state[p]], False)
                self._launch(gi, group, new, True)
            else:
                self._launch(gi, group, ps, bool(new))
        return loss

    def _launch(self, gi, group, ps, first):
        dev = ps[0].device
        lr_dev = self._lr_tensor(gi, dev)
        if not self.capturable:
            lr_dev.fill_(float(group["lr"]))
        for p in ps:
            if "momentum_buffer" not in self.state[p]:
                self.state[p]["momentum_buffer"] = torch.empty_like(p, memory_format=torch.contiguous_format)
        grads = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ps]
        bufs = [self.state[p]["momentum_buffer"] for p in ps]
        sig = tuple(t.data_ptr() for t in ps) + tuple(t.data_ptr() for t in grads) + tuple(t.data_ptr() for t in bufs)
        key = (gi, dev)
        cached = self._table.get(key)
        if cached is None or cached[1].numel() < _cabi.load().tp_segtable_workspace_bytes(len(ps)):
            ws = torch.empty(_cabi.load().tp_segtable_workspace_bytes(len(ps)), dtype=torch.uint8, device=dev)
            cached = (None, ws)
        hit = cached[0] == sig
        ops.sgd_momentum_step(ps, grads, bufs, lr_dev, group["momentum"], group["weight_decay"], first,
                              table_ws=cached[1], table_cached=hit)
        self._table[key] = (sig, cached[1])


class FusedAdamW(torch.optim.Optimizer):
    """torch.optim.AdamW (decoupled weight decay) in one fused launch per parameter group, bit for bit with
    ``torch.optim.AdamW(foreach=True, capturable=True)`` on the same GPU.

    Param-group keys, state keys (``step``: 0-dim fp32 device tensor, ``exp_avg``, ``exp_avg_sq``) and ``state_dict()``
    are torch's, so checkpoints load into either optimizer.  As in ``FusedSGD``, the learning rate (as ``1 / lr``) and
    the decay factor ``1 - lr * weight_decay`` (both formed in double, as torch does) live in device scalars that
    ``sync_lr()`` refreshes, and the pointer table is re-uploaded only when a pointer changed, so a captured step follows
    the LR schedule.  Each
    parameter keeps its own step count and bias corrections: a parameter whose first gradient arrives late starts at
    t = 1 in the same launch, because fresh state (m = v = 0, step = 0) makes its first update the general one.
    AMSGrad, ``maximize``, ``differentiable``, tensor lr / betas and complex parameters raise ``ValueError``."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, *,
                 maximize=False, foreach=None, capturable=False, differentiable=False, fused=None):
        if isinstance(lr, torch.Tensor) or any(isinstance(b, torch.Tensor) for b in betas):
            raise ValueError("FusedAdamW: lr and betas must be Python numbers (the device scalars are its own)")
        if amsgrad or maximize or differentiable:
            raise ValueError("FusedAdamW: amsgrad, maximize and differentiable are not supported")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=foreach, capturable=capturable, differentiable=False, fused=fused,
                        decoupled_weight_decay=True)
        super().__init__(params, defaults)
        for group in self.param_groups:
            if any(torch.is_complex(p) for p in group["params"]):
                raise ValueError("FusedAdamW: complex parameters are not supported")
        self.capturable = capturable
        self._lr_dev = {}         # (group, device) -> fp32 [1 / lr, 1 - lr * weight_decay]
        self._table = {}          # (group, device) -> (pointer signature, workspace tensor)

    def _scalars(self, gi, dev):
        t = self._lr_dev.get((gi, dev))
        if t is None:
            t = self._lr_dev[(gi, dev)] = torch.empty(2, dtype=torch.float32, device=dev)
            self._fill(gi, t)
        return t

    def _fill(self, gi, t):
        group = self.param_groups[gi]
        lr = float(group["lr"])
        # torch's _foreach_div_(x, lr) multiplies by fp32(1.0 / lr), the reciprocal taken in double
        t[0].fill_(1.0 / lr if lr != 0 else math.inf)
        t[1].fill_(1 - lr * group["weight_decay"])

    def sync_lr(self):
        """Copy every group's host lr (and its decay factor) into the device scalars (call between graph replays)."""
        for (gi, _), t in self._lr_dev.items():
            self._fill(gi, t)

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        # a checkpoint of a non-capturable torch optimizer keeps `step` on the host; the kernel counts on the device
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state.get(p)
                if st and "step" in st and (st["step"].device != p.device or st["step"].dtype != torch.float32):
                    st["step"] = st["step"].to(device=p.device, dtype=torch.float32)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            ps = [p for p in group["params"] if p.grad is not None]
            if ps:
                self._launch(gi, group, ps)
        return loss

    def _launch(self, gi, group, ps):
        dev = ps[0].device
        scal = self._scalars(gi, dev)
        if not self.capturable:
            self._fill(gi, scal)
        for p in ps:
            if p.grad.is_sparse:
                raise RuntimeError("FusedAdamW does not support sparse gradients")
            st = self.state[p]
            if len(st) == 0:
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise TypeError("FusedAdamW: contiguous fp32 parameters")
                st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        grads = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ps]
        ms = [self.state[p]["exp_avg"] for p in ps]
        vs = [self.state[p]["exp_avg_sq"] for p in ps]
        steps = [self.state[p]["step"] for p in ps]
        sig = tuple(t.data_ptr() for ts in (ps, grads, ms, vs, steps) for t in ts)
        key = (gi, dev)
        nbytes = _cabi.load().tp_segtable_workspace_bytes(len(ps))
        cached = self._table.get(key)
        if cached is None or cached[1].numel() < nbytes:
            cached = (None, torch.empty(nbytes, dtype=torch.uint8, device=dev))
        beta1, beta2 = group["betas"]
        ops.adamw_step(ps, grads, ms, vs, steps, scal[0], scal[1] if group["weight_decay"] != 0 else None,
                       beta1, beta2, group["eps"], table_ws=cached[1], table_cached=cached[0] == sig)
        self._table[key] = (sig, cached[1])
