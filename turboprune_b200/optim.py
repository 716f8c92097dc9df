"""Fused SGD(momentum, weight_decay) — one kernel launch for all parameters — fused AdamW (``FusedAdamW``), fused
Muon with AdamW for the remaining parameters (``FusedMuon``) and fused Schedule-Free SGD (``FusedScheduleFreeSGD``).

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


def _check_adamw(lr, betas, eps, weight_decay, amsgrad, maximize, differentiable):
    """torch.optim.AdamW's argument checks, and the options the fused kernel does not implement."""
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


class _AdamWGroups:
    """The AdamW launch of a parameter group (``tp_adamw``), shared by ``FusedAdamW`` and the AdamW groups of
    ``FusedMuon``.  Expects ``self._lr_dev`` / ``self._table`` dicts and ``self.capturable``."""

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

    def _steps_to_device(self):
        # a checkpoint of a non-capturable torch optimizer keeps `step` on the host; the kernel counts on the device
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state.get(p)
                if st and "step" in st and (st["step"].device != p.device or st["step"].dtype != torch.float32):
                    st["step"] = st["step"].to(device=p.device, dtype=torch.float32)

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


class FusedAdamW(_AdamWGroups, torch.optim.Optimizer):
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
        _check_adamw(lr, betas, eps, weight_decay, amsgrad, maximize, differentiable)
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

    def sync_lr(self):
        """Copy every group's host lr (and its decay factor) into the device scalars (call between graph replays)."""
        for (gi, _), t in self._lr_dev.items():
            self._fill(gi, t)

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._steps_to_device()

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


def _schedulefree_advance(group):
    """One step of a Schedule-Free group's host schedule, in Python floats as the schedulefree package writes it: commits
    ``k + 1``, ``lr_max``, ``weight_sum`` and ``scheduled_lr`` and returns the step's (lr, ckp1, alpha_y)."""
    k, warmup = group["k"], group["warmup_steps"]
    sched = (k + 1) / warmup if k < warmup else 1.0
    lr = group["lr"] * sched
    lr_max = group["lr_max"] = max(lr, group["lr_max"])
    weight = ((k + 1) ** group["r"]) * (lr_max ** group["weight_lr_power"])
    weight_sum = group["weight_sum"] = group["weight_sum"] + weight
    ckp1 = weight / weight_sum if weight_sum != 0 else 0
    group["scheduled_lr"] = lr
    group["k"] = k + 1
    return lr, ckp1, lr * (group["momentum"] * (1 - ckp1) - 1)


class FusedScheduleFreeSGD(torch.optim.Optimizer):
    """Schedule-Free SGD (Defazio et al. 2024, "The Road Less Scheduled"): the schedulefree package's ``SGDScheduleFree``
    with one fused launch per parameter group (``tp_schedulefree_sgd``, 20 B/elem), bit for bit with the package's
    foreach torch ops on the same GPU.  Group keys (``lr, momentum, weight_decay, warmup_steps, r, weight_lr_power, k,
    weight_sum, lr_max, scheduled_lr, train_mode, foreach``) and the per-parameter state ``z`` are the package's, so
    ``state_dict()`` keeps its layout.

    The parameters hold y while training and the average x = lerp(y, z, 1 - 1 / momentum) otherwise.  ``eval()`` moves
    them to x and ``train()`` back to y (``tp_schedulefree_swap``: one launch, eager, no host sync); each is a no-op when
    the optimizer is already in that mode, and ``step()`` raises outside train mode.  The optimizer starts in eval mode:
    call ``train()`` before training and ``eval()`` before evaluating or saving (the harness does both).

    The schedule (``k`` and the values formed from it) advances exactly once per update:
      * ``capturable=False``: ``step()`` advances it, fills the step's device scalars and launches;
      * ``capturable=True``: ``sync_lr()`` advances it and fills the device scalars (``fill_``, no host sync); ``step()``
        only launches, so it may run eagerly, be captured into a CUDA graph, or both, after one ``sync_lr()``, and a
        replay needs ``sync_lr()`` first.  Call ``sync_lr()`` once before every update.
    A parameter whose first gradient arrives late gets its ``z`` in a launch of its own.  The package also adds the
    weight decay into ``p.grad``; this optimizer leaves the gradient as it is.  Closures are not supported."""

    def __init__(self, params, lr=1.0, momentum=0.9, weight_decay=0, warmup_steps=0, r=0.0, weight_lr_power=2.0, *,
                 capturable=False):
        for name, v in (("lr", lr), ("momentum", momentum), ("weight_decay", weight_decay), ("warmup_steps", warmup_steps),
                        ("r", r), ("weight_lr_power", weight_lr_power)):
            if isinstance(v, torch.Tensor):
                raise ValueError(f"FusedScheduleFreeSGD: {name} must be a Python number (the device scalars are its own)")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if not 0.0 < momentum < 1.0:
            raise ValueError(f"Momentum must be between 0 and 1 exclusive: {momentum}")
        defaults = dict(lr=lr, momentum=momentum, r=r, k=0, warmup_steps=warmup_steps, train_mode=False,
                        weight_sum=0.0, lr_max=-1.0, scheduled_lr=0.0, weight_lr_power=weight_lr_power,
                        weight_decay=weight_decay, foreach=True)
        super().__init__(params, defaults)
        for group in self.param_groups:
            for p in group["params"]:
                if torch.is_complex(p) or p.dtype != torch.float32:
                    raise ValueError(f"FusedScheduleFreeSGD: fp32 parameters only, not {p.dtype}")
        self.capturable = capturable
        self._host = {}           # group -> the step's (lr, ckp1, alpha_y) as Python floats
        self._sc_dev = {}         # (group, device) -> fp32 [lr, ckp1, alpha_y]
        self._table = {}          # (group, device) / (group, device, "swap") -> (pointer signature, workspace)

    def _fill(self, gi, t):
        # three fill_ launches, no host-to-device copy; fill_ rounds each double to fp32 as Scalar.to<float>() does
        for i, v in enumerate(self._host[gi]):
            t[i].fill_(v)

    def sync_lr(self):
        """Capturable: advance every group's schedule by one update and refresh its device scalars (call once before
        every update, eager or replayed).  Without ``capturable`` ``step()`` does this and this call does nothing."""
        if not self.capturable:
            return
        for gi, group in enumerate(self.param_groups):
            self._host[gi] = _schedulefree_advance(group)
        for (gi, _), t in self._sc_dev.items():
            self._fill(gi, t)

    @torch.no_grad()
    def train(self):
        """Move every parameter with a ``z`` from x to y (lerp weight 1 - momentum) and enter train mode."""
        self._swap(True)

    @torch.no_grad()
    def eval(self):
        """Move every parameter with a ``z`` from y to x (lerp weight 1 - 1 / momentum) and enter eval mode."""
        self._swap(False)

    def _swap(self, to_train):
        for gi, group in enumerate(self.param_groups):
            if group["train_mode"] == to_train:
                continue
            ps = [p for p in group["params"] if "z" in self.state[p]]
            if ps:
                momentum = group["momentum"]
                zs = [self.state[p]["z"] for p in ps]
                ws, hit = self._workspace((gi, ps[0].device, "swap"), ps, zs)
                ops.schedulefree_swap(ps, zs, 1 - momentum if to_train else 1 - 1 / momentum, table_ws=ws, table_cached=hit)
            group["train_mode"] = to_train

    def _workspace(self, key, *lists):
        sig = tuple(t.data_ptr() for ts in lists for t in ts)
        nbytes = _cabi.load().tp_segtable_workspace_bytes(len(lists[0]))
        cached = self._table.get(key)
        if cached is None or cached[1].numel() < nbytes:
            cached = (None, torch.empty(nbytes, dtype=torch.uint8, device=lists[0][0].device))
        self._table[key] = (sig, cached[1])
        return cached[1], cached[0] == sig

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise NotImplementedError("FusedScheduleFreeSGD.step does not take a closure")
        if not self.param_groups[0]["train_mode"]:
            raise RuntimeError("FusedScheduleFreeSGD: step() outside train mode: call optimizer.train() before training "
                               "and optimizer.eval() before evaluating or saving")
        for gi, group in enumerate(self.param_groups):
            if not self.capturable:
                self._host[gi] = _schedulefree_advance(group)
            elif gi not in self._host:
                raise RuntimeError("FusedScheduleFreeSGD(capturable=True): call sync_lr() before every update")
            ps = [p for p in group["params"] if p.grad is not None]
            old = [p for p in ps if "z" in self.state[p]]
            new = [p for p in ps if "z" not in self.state[p]]
            if old:
                self._launch(gi, group, old, False)
            if new:
                self._launch(gi, group, new, True)

    def _launch(self, gi, group, ps, first):
        dev = ps[0].device
        sc = self._sc_dev.get((gi, dev))
        if sc is None:
            sc = self._sc_dev[(gi, dev)] = torch.empty(3, dtype=torch.float32, device=dev)
            self._fill(gi, sc)
        elif not self.capturable:
            self._fill(gi, sc)
        for p in ps:
            if p.grad.is_sparse:
                raise RuntimeError("FusedScheduleFreeSGD does not support sparse gradients")
            if not p.is_contiguous():
                raise TypeError("FusedScheduleFreeSGD: contiguous fp32 parameters")
            if first:
                self.state[p]["z"] = torch.empty_like(p, memory_format=torch.contiguous_format)
        grads = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ps]
        zs = [self.state[p]["z"] for p in ps]
        ws, hit = self._workspace((gi, dev), ps, grads, zs)
        ops.schedulefree_step(ps, grads, zs, sc, group["weight_decay"], first, table_ws=ws, table_cached=hit)


MUON_NS_COEFFICIENTS = (3.4445, -4.7750, 2.0315)      # torch.optim.Muon's defaults (Keller Jordan's quintic)


def _check_muon_group(group):
    lr, momentum, wd, fn = group["lr"], group["momentum"], group["weight_decay"], group["adjust_lr_fn"]
    if isinstance(lr, torch.Tensor):
        raise ValueError("FusedMuon: lr must be a Python number (the device scalars are its own)")
    if not 0.0 <= lr:
        raise ValueError(f"Learning rate should be >= 0 but is: {lr}")
    if not 0.0 <= momentum:
        raise ValueError(f"momentum should be >= 0 but is: {momentum}")
    if not 0.0 <= wd:
        raise ValueError(f"weight decay should be >= 0 but is: {wd}")
    if fn is not None and fn not in ("original", "match_rms_adamw"):
        raise ValueError(f"Adjust learning rate function {fn} is not supported")
    if group["ns_steps"] >= 100:
        raise ValueError("Number of steps must be less than 100 for computational efficiency")
    if len(group["ns_coefficients"]) != 3:
        raise ValueError("Coefficients must be a tuple of exactly 3 values")


class FusedMuon(_AdamWGroups, torch.optim.Optimizer):
    """torch.optim.Muon for the hidden weight matrices and torch.optim.AdamW for every other parameter, in a fixed
    number of launches per step: 4 + 3 * ns_steps for all Muon layers together (19 at the default five Newton-Schulz
    steps) and the two of ``tp_adamw`` for each AdamW group.

    A parameter ``p`` of a Muon group (``use_muon=True``, the default) is stepped as ``torch.optim.Muon`` steps the 2-D
    view ``p.view(p.shape[0], -1)``: a conv weight [Cout, Cin, R, S] as [Cout, Cin*R*S], a Conv1d classifier
    [out, in, 1] as [out, in]; its ``momentum_buffer`` has that 2-D shape, so a Muon group's state loads into
    ``torch.optim.Muon`` over the views (and back).  The lr ratio of ``adjust_lr_fn`` is torch's ``_adjust_lr`` on the
    2-D shape.  Constructor arguments, defaults and validation are torch's, except that any parameter of two or more
    dimensions is accepted.  The Newton-Schulz iteration runs in bf16 (fp32 accumulation) as torch's does; its GEMMs are
    this project's wgmma kernel, deterministic (no atomics, no split-K), so replicas stay bit-identical.

    Groups with ``use_muon=False`` carry torch.optim.AdamW's keys (``betas`` and ``eps`` default to ``adamw_betas`` /
    ``adamw_eps``; ``lr`` and ``weight_decay`` to this optimizer's) and state, and are stepped by the ``FusedAdamW``
    kernel, bit for bit with torch's capturable AdamW.

    Masked weights: as torch does, the orthogonalised update is dense, so a pruned weight moves although its gradient
    is 0.  The forward always uses ``mask * w`` and the pruning scores use ``|mask * w|``, so this is not observable.

    Capturable: lr and weight_decay live in float64 device scalars that ``sync_lr()`` refreshes with ``fill_`` (no host
    synchronisation); the apply kernel forms ``1 - lr * weight_decay`` and every ``-(lr * ratio)`` from them in double,
    as Python does.  The layer table is re-uploaded only when a pointer or ``adjust_lr_fn`` changed."""

    def __init__(self, params, lr=1e-3, weight_decay=0.1, momentum=0.95, nesterov=True,
                 ns_coefficients=MUON_NS_COEFFICIENTS, eps=1e-7, ns_steps=5, adjust_lr_fn=None, *,
                 adamw_betas=(0.9, 0.999), adamw_eps=1e-8, capturable=False):
        self.capturable = capturable
        self._lr_dev = {}         # AdamW groups: (group, device) -> fp32 [1 / lr, 1 - lr * weight_decay]
        self._table = {}          # AdamW groups: (group, device) -> (pointer signature, workspace tensor)
        self._muon = {}           # Muon groups: (group, device) -> plan, workspaces, device tile lists and scalars
        self._adamw_defaults = dict(lr=lr, betas=tuple(adamw_betas), eps=adamw_eps, weight_decay=weight_decay,
                                    amsgrad=False, maximize=False, foreach=None, capturable=capturable,
                                    differentiable=False, fused=None, decoupled_weight_decay=True)
        defaults = dict(lr=lr, weight_decay=weight_decay, momentum=momentum, nesterov=nesterov,
                        ns_coefficients=tuple(ns_coefficients), eps=eps, ns_steps=ns_steps, adjust_lr_fn=adjust_lr_fn)
        _check_muon_group(defaults)
        super().__init__(params, defaults)

    def add_param_group(self, param_group):
        use_muon = bool(param_group.get("use_muon", True))
        ps = param_group["params"]
        ps = [ps] if isinstance(ps, torch.Tensor) else list(ps)
        if any(torch.is_complex(p) for p in ps):
            raise ValueError("FusedMuon: complex parameters are not supported")
        group = dict(param_group, params=ps, use_muon=use_muon)
        saved = self.defaults
        if use_muon:
            for k, v in saved.items():
                group.setdefault(k, v)
            _check_muon_group(group)
            for p in ps:
                if p.ndim < 2:
                    raise ValueError(f"Muon only supports 2D parameters whereas we found a parameter with size: {p.size()}")
        else:
            for k, v in self._adamw_defaults.items():
                group.setdefault(k, v)
            # FusedAdamW's checks: amsgrad, maximize, differentiable and a tensor lr would otherwise be ignored
            _check_adamw(group["lr"], group["betas"], group["eps"], group["weight_decay"], group["amsgrad"],
                         group["maximize"], group["differentiable"])
        try:
            # torch fills missing keys from self.defaults: an AdamW group gets AdamW's
            self.defaults = saved if use_muon else self._adamw_defaults
            super().add_param_group(group)
        finally:
            self.defaults = saved

    def _muon_fill(self, gi, st):
        # two fill_ launches, no host-to-device copy: the apply kernel forms 1 - lr * wd and -(lr * ratio) in double
        group = self.param_groups[gi]
        st["lr_wd"][0].fill_(float(group["lr"]))
        st["lr_wd"][1].fill_(float(group["weight_decay"]))

    def sync_lr(self):
        """Copy every group's host lr (and the factors formed from it) into the device scalars (call between graph
        replays)."""
        for (gi, _), t in self._lr_dev.items():
            self._fill(gi, t)
        for (gi, _), st in self._muon.items():
            self._muon_fill(gi, st)

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._steps_to_device()

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
            if group["use_muon"]:
                self._muon_step(gi, group, ps)
            else:
                self._launch(gi, group, ps)
        return loss

    def _muon_state(self, gi, dev, shapes):
        st = self._muon.get((gi, dev))
        if st is None or st["shapes"] != shapes:
            plan = ops.MuonPlan(shapes)
            lib = _cabi.load()
            st = dict(shapes=shapes, plan=plan, sig=None,
                      xws=torch.zeros(plan.rows * 64, dtype=torch.bfloat16, device=dev),
                      partial=torch.empty(plan.n_tiles, dtype=torch.float32, device=dev),
                      table=torch.empty(lib.tp_muon_workspace_bytes(len(shapes)), dtype=torch.uint8, device=dev),
                      tiles={k: torch.from_numpy(v).to(dev) for k, v in plan.gemm_tiles.items()},
                      norms=torch.empty(len(shapes), dtype=torch.float32, device=dev),
                      lr_wd=torch.empty(2, dtype=torch.float64, device=dev))
            self._muon[(gi, dev)] = st
            self._muon_fill(gi, st)
        return st

    def _muon_step(self, gi, group, ps):
        dev = ps[0].device
        shapes = tuple((p.shape[0], p.numel() // p.shape[0]) for p in ps)
        st = self._muon_state(gi, dev, shapes)
        if not self.capturable:
            self._muon_fill(gi, st)
        ws, gs, bufs = [], [], []
        for p, (a, b) in zip(ps, shapes):
            if p.grad.is_sparse:
                raise RuntimeError("Muon does not support sparse gradients")
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise TypeError("FusedMuon: contiguous fp32 parameters")
            s = self.state[p]
            if "momentum_buffer" not in s:
                s["momentum_buffer"] = torch.zeros((a, b), dtype=torch.float32, device=dev)
            ws.append(p.view(a, b))
            gs.append((p.grad if p.grad.is_contiguous() else p.grad.contiguous()).view(a, b))
            bufs.append(s["momentum_buffer"].view(a, b))
        # the layer table carries the pointers and each layer's lr ratio
        sig = tuple(t.data_ptr() for ts in (ws, gs, bufs) for t in ts) + (group["adjust_lr_fn"],)
        plan, xws, table = st["plan"], st["xws"], st["table"]
        ops.muon_prepare(plan, xws, st["partial"], st["norms"], table, ws, gs, bufs, group["momentum"], group["nesterov"],
                         group["eps"], group["adjust_lr_fn"], table_cached=st["sig"] == sig)
        st["sig"] = sig
        ops.muon_normalize(plan, xws, st["norms"], table)
        a, b, c = group["ns_coefficients"]
        src = 0
        for _ in range(group["ns_steps"]):
            ops.muon_ns_gemm(ops.MUON_GRAM, xws, st["tiles"][(ops.MUON_GRAM, src)], 1.0, 0.0)
            ops.muon_ns_gemm(ops.MUON_POLY, xws, st["tiles"][(ops.MUON_POLY, 0)], c, b)
            ops.muon_ns_gemm(ops.MUON_UPDATE, xws, st["tiles"][(ops.MUON_UPDATE, src)], 1.0, a)
            src = 1 - src
        ops.muon_apply(plan, xws, src, st["lr_wd"], table)
