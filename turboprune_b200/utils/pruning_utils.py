"""Pruning criteria — drop-in for the reference's ``utils/pruning_utils.py``.

Public names and call signatures are the reference's (``prune_the_model`` and the
``prune_<method>`` family looked up by string, utils/pruning_utils.py:23-58).  The heavy part —
per-layer score temporaries, ``torch.cat``, single-CTA ``torch.kthvalue`` and per-layer
``torch.where`` (:73-87, :186-203, :263-283) — is one call into the sm_90a radix-select
kernels (``ops.topk_threshold_mask``), bit-exact with the reference's masks.

Things kept on purpose:
  * ``k = int((1 - density) * N)`` is computed on the host in float64 (:78);
  * ``k == 0`` raises like ``torch.kthvalue`` does (the reference's ``if not k < 1`` guard at :81
    comes after the call that raises);
  * ties at the threshold are pruned (``score <= thr``);
  * random criteria draw their noise / Bernoulli masks with torch's generator in the reference's
    order, because the RNG stream is part of mask parity (:112, :314; mask_layers.py:43);
  * an unknown method prints an error and returns (:33-37).
"""
from contextlib import nullcontext
from typing import Any, List

import torch
import torch.nn as nn
from torch.amp import autocast

from .. import _cabi, ops
from .mask_layers import MASKED_LAYER_TYPES, ConvMask, Conv1dMask, LinearMask  # noqa: F401


def _masked(model: nn.Module) -> List[nn.Module]:
    return [m for _, m in model.named_modules() if isinstance(m, MASKED_LAYER_TYPES)]


def get_dtype_amp(cfg):
    table = {"bfloat16": (torch.bfloat16, True), "float16": (torch.float16, True), "float32": (torch.float32, False)}
    return table.get(cfg.experiment_params.training_precision, (torch.float32, False))


def _compute_precision(precision):
    """float32 configs score with fp32 activations and gradients (TF32 GEMMs); the others with the default bf16 kernels."""
    return ops.compute_precision(torch.float32) if precision == torch.float32 else nullcontext()


def _global_prune(model: nn.Module, density: float, kind: int) -> nn.Module:
    layers = _masked(model)
    ws = [m.weight for m in layers]
    ms = [m.mask.to(m.weight.device) for m in layers]
    gs = None if kind == _cabi.TP_SCORE_MAG else [m.weight.grad for m in layers]
    total = sum(w.numel() for w in ws)
    k = int((1 - density) * total)
    new_masks, _, info = ops.topk_threshold_mask(ws, ms, k, gs=gs, kind=kind)   # raises for k == 0
    for m, nm in zip(layers, new_masks):
        m.mask = nm
    model._last_prune_info = info
    return model


def prune_mag(model: nn.Module, density: float) -> nn.Module:
    """Global magnitude pruning: scores |mask * w| (reference :61-89)."""
    return _global_prune(model, density, _cabi.TP_SCORE_MAG)


def prune_snip(cfg, model: nn.Module, trainloader: Any, density: float) -> nn.Module:
    """SNIP: one batch forward/backward, scores |(g * w) * mask| (reference :160-205)."""
    precision, use_amp = get_dtype_amp(cfg)
    dev = next(model.parameters()).device
    criterion = nn.CrossEntropyLoss()
    for images, target in trainloader:
        images = images.to(dev)
        target = target.to(dev).long()
        with _compute_precision(precision), autocast("cuda", dtype=precision, enabled=use_amp):
            model.zero_grad()
            criterion(model(images), target).backward()
        break
    return _global_prune(model, density, _cabi.TP_SCORE_SNIP)


def prune_synflow(cfg, model: nn.Module, trainloader: Any, density: float) -> nn.Module:
    """SynFlow (single shot): |theta| network, all-ones input, scores |(mask * g) * w| (reference :208-285).

    Like the reference this takes |.| of every state-dict tensor (BN buffers included), runs the
    forward in the model's current mode on a batch of one, and restores the signs afterwards.
    """
    precision, use_amp = get_dtype_amp(cfg)
    dev = next(model.parameters()).device
    with torch.no_grad():
        signs = {}
        for name, t in model.state_dict().items():
            signs[name] = torch.sign(t)
            t.abs_()
    for images, _ in trainloader:
        shape = [1] + list(images[0, :].shape)
        ones = torch.ones(shape, device=dev)
        with _compute_precision(precision), autocast("cuda", dtype=precision, enabled=use_amp):
            torch.sum(model(ones)).backward()
        break
    layers = _masked(model)
    ws = [m.weight for m in layers]
    ms = [m.mask.to(m.weight.device) for m in layers]
    gs = [m.weight.grad.clone() for m in layers]
    model.zero_grad()
    # scores must be taken on the linearised (|w|) weights, before the signs come back
    total = sum(w.numel() for w in ws)
    k = int((1 - density) * total)
    new_masks, _, info = ops.topk_threshold_mask(ws, ms, k, gs=gs, kind=_cabi.TP_SCORE_SYNFLOW)
    with torch.no_grad():
        for name, t in model.state_dict().items():
            t.mul_(signs[name])
    for m, nm in zip(layers, new_masks):
        m.mask = nm
    model._last_prune_info = info
    return model


def _per_layer_random(model: nn.Module, keep_fracs, noises) -> nn.Module:
    for m, frac, z in zip(_masked(model), keep_fracs, noises):
        n = m.weight.numel()
        k = int((1 - frac) * n)                      # fp32 tensor arithmetic for erk, float for balanced
        mask_in = m.mask.to(m.weight.device)
        if k == 0:
            zero = torch.zeros((), device=m.weight.device)
            m.mask = ops.apply_threshold([z], [mask_in], zero)[0]
        else:
            m.mask = ops.topk_threshold_mask([z], [mask_in], k)[0][0]
        print("Layer", type(m).__name__, " params ", k, n)
    return model


def _erk_fracs(layers, density):
    fracs, counts, total = [], [], 0
    for m in layers:
        fracs.append(torch.tensor(m.weight.shape).sum() / m.weight.numel())
        counts.append(m.weight.numel())
        total += m.weight.numel()
    kept = (torch.tensor(fracs) * torch.tensor(counts)).sum()
    c = (total * density) / kept
    return c, [torch.clamp(c * s, 0, 1) for s in fracs]


def _balanced_fracs(layers, density):
    total = sum(m.weight.numel() for m in layers)
    L = len(layers)
    X = density * total / L
    fracs = []
    for l, m in enumerate(layers):
        n = m.weight.numel()
        if X / n < 1.0:
            fracs.append(X / n)
        else:
            fracs.append(1)
            X = X + (X - m.mask.numel()) / (L - l)
    return fracs


def prune_random_erk(model: nn.Module, density: float) -> nn.Module:
    """Random pruning with ERK layer budgets, per-layer thresholds (reference :92-146)."""
    layers = _masked(model)
    noises = [torch.randn_like(m.weight) for m in layers]        # same draw order as the reference
    c, fracs = _erk_fracs(layers, density)
    print("Factor: ", c)
    return _per_layer_random(model, fracs, noises)


def prune_random_balanced(model: nn.Module, density: float) -> nn.Module:
    """Random pruning with balanced layer budgets (reference :288-347)."""
    layers = _masked(model)
    noises = [torch.randn_like(m.weight) for m in layers]
    return _per_layer_random(model, _balanced_fracs(layers, density), noises)


def prune_er_erk(model: nn.Module, er_sparse_init: float):
    """Erdos-Renyi-Kernel Bernoulli masks at init (reference :350-378)."""
    layers = _masked(model)
    _, fracs = _erk_fracs(layers, er_sparse_init)
    for m, p in zip(layers, fracs):
        m.set_er_mask(p)
    return model


def prune_er_balanced(model: nn.Module, er_sparse_init: float):
    """Balanced Bernoulli masks at init (reference :381-415)."""
    layers = _masked(model)
    for m, p in zip(layers, _balanced_fracs(layers, er_sparse_init)):
        m.set_er_mask(p)
    return model


def sync_masks_from_rank0(model: nn.Module) -> None:
    """Make rank 0's masks the masks of every replica (one packed broadcast per pruning step).

    The reference prunes on rank 0 only and lets the next DistributedDataParallel constructor broadcast the buffers
    (run_experiment.py:85-105,113; base_harness.py:81).  Here every rank runs the pruner, which is replica-identical
    for the magnitude criteria but NOT for SNIP (each rank scores its own first batch, pruning_utils.py:177-184) nor
    for the random criteria if the per-device RNG streams ever drift — so rank 0's result is imposed, as upstream."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    layers = _masked(model)
    flat = torch.cat([m.mask.reshape(-1).to(m.weight.device, torch.float32) for m in layers])
    dist.broadcast(flat, 0)
    off = 0
    for m in layers:
        n = m.mask.numel()
        m.mask = flat[off:off + n].view_as(m.weight).clone()
        off += n


def sync_masks_from_rank0_(masks) -> None:
    """In-place form of ``sync_masks_from_rank0``: rank 0's values are broadcast INTO the given tensors (one packed
    broadcast), so every pointer a captured CUDA graph or a cached table holds stays valid."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    masks = list(masks)
    flat = torch.cat([m.reshape(-1) for m in masks])
    dist.broadcast(flat, 0)
    off = 0
    for m in masks:
        n = m.numel()
        m.copy_(flat[off:off + n].view_as(m))
        off += n


@torch.no_grad()
def rigl_update(model: nn.Module, optimizer, k_per_layer, new_masks=None):
    """One RigL drop-and-regrow step (Evci et al. 2020) over the masked layers' current ``.grad``.

    The gradients must be dense: run the forward / backward inside ``ops.dense_weight_grad()``.  Per masked layer l,
    the k_per_layer[l] live weights of smallest |w| are dropped and as many pruned positions of largest |g| (the
    just-dropped ones included) are grown; ties go to the lower flat index.  Grown weights and their optimizer state
    (``momentum_buffer``, or AdamW's ``exp_avg`` and ``exp_avg_sq``, when there is one) restart at 0 in the same launch;
    regrown dropped weights keep theirs.
    Masks, weights and momenta are updated in place (``mask_layers.mask_epoch()`` does not change).  Under
    torch.distributed every rank selects, rank 0's result is broadcast, every rank applies it.  ``new_masks``:
    scratch tensors of the masks' shapes to reuse.  Returns an int64 cuda tensor [layers, 2] of (dropped, grown)."""
    layers = _masked(model)
    for m in layers:
        if m.weight.grad is None:
            raise RuntimeError("rigl_update: a masked layer has no gradient (run a backward pass inside "
                               "ops.dense_weight_grad() first)")
        if m.mask.device != m.weight.device or m.mask.dtype != torch.float32 or not m.mask.is_contiguous():
            m.mask = m.mask.to(device=m.weight.device, dtype=torch.float32).contiguous()
    ws = [m.weight.detach() for m in layers]
    gs = [m.weight.grad.contiguous() for m in layers]
    ms = [m.mask for m in layers]
    if new_masks is None:
        new_masks = [torch.empty_like(m) for m in ms]
    counts = ops.rigl_select(ws, gs, ms, new_masks, k_per_layer)
    sync_masks_from_rank0_(new_masks)
    state = getattr(optimizer, "state", {}) if optimizer is not None else {}
    per_layer = [state[m.weight] if m.weight in state else {} for m in layers]
    # every per-element state the optimizer keeps (SGD: momentum_buffer; AdamW: exp_avg, exp_avg_sq; Schedule-Free: z;
    # AdamW's per-parameter step is left alone); one state, or none at all, keeps the one-state apply
    keys = [k for k in _RIGL_RESTART_KEYS if any(k in st for st in per_layer)] or ["momentum_buffer"]
    states = [[st.get(k) for st in per_layer] for k in keys]
    if len(keys) == 1:
        ops.rigl_apply(ms, new_masks, ws, states[0])
    else:
        ops.rigl_apply_states(ms, new_masks, ws, states)
    return counts


_RIGL_RESTART_KEYS = ("momentum_buffer", "exp_avg", "exp_avg_sq", "z")


def prune_the_model(cfg, harness, target_density: float) -> None:
    """Dispatcher by ``cfg.pruning_params.prune_method`` (reference :23-58)."""
    # the reference unwraps DDP here (:25); our harness keeps the bare module and reduces gradients explicitly
    model = getattr(harness.model, "module", harness.model)
    console = harness.console
    method = cfg.pruning_params.prune_method
    loader = harness.train_loader if method in {"synflow", "snip"} else None
    before = model.get_overall_sparsity()
    fn = globals().get(f"prune_{method}")
    if not fn:
        console.print(f"[bold red]Error: Unknown pruning method '{method}'[/bold red]")
        return
    model = fn(cfg, model, loader, target_density) if loader else fn(model, target_density)
    if getattr(harness, "distributed", False):
        sync_masks_from_rank0(model)
    after = model.get_overall_sparsity()
    console.print(f"Initial Sparsity {before:.4f}  ->  Final Sparsity {after:.4f}")
    console.print(f"[bold green]Pruning completed using {method} method![/bold green]")
