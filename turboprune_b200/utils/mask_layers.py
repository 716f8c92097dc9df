"""Masked operators — drop-in for the reference's ``utils/mask_layers.py``.

Same class names, constructor arguments, parameter/buffer names (``weight``, ``bias``, fp32
``mask`` buffer with the weight's shape) and ``set_er_mask`` as the reference
(utils/mask_layers.py:10-128), so checkpoints, ``custom_models.replace_layers`` and the
``mask_layer_type`` string lookup keep working.  What changes is ``forward``: instead of
materialising ``mask * weight`` and calling cuDNN/cuBLAS, it launches the sm_90a
implicit-GEMM kernels (``turboprune_b200.ops``), which consume weights masked while they are
staged to bf16 and apply the mask to the weight gradient inside wgrad.

There is deliberately no CPU implementation here: CPU tensors raise.
"""
import torch
import torch.nn as nn

from .. import ops


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _live_slot(p):
    # the slot only counts while it still IS p.grad (zero_grad(set_to_none=True) or a user assignment detaches it)
    if p is None:
        return None
    slot = getattr(p, "_tp_grad_slot", None)
    g = p.grad
    if slot is None or g is None or g.data_ptr() != slot.data_ptr():
        return None
    return slot


def grad_slots(weight, bias):
    ws = _live_slot(weight)
    if ws is None:
        return None
    return (ws, _live_slot(bias))


def _slots(layer):
    """Persistent gradient slots attached by GradArena / P2PGradReducer (None when training with plain .grad)."""
    return grad_slots(layer.weight, layer.bias)


_MASK_EPOCH = [0]


def mask_epoch() -> int:
    """Bumped whenever any masked layer gets a NEW mask tensor (pruning assigns ``m.mask = ...`` like the reference,
    pruning_utils.py:87): captured CUDA graphs and cached pointer tables key on it."""
    return _MASK_EPOCH[0]


class _MaskMixin:
    def _init_mask(self):
        self.register_buffer("mask", torch.ones_like(self.weight))

    def __setattr__(self, name, value):
        if name == "mask":
            _MASK_EPOCH[0] += 1
        super().__setattr__(name, value)

    def set_er_mask(self, p) -> None:
        """Bernoulli(p) keep-mask drawn with torch's generator (bit-identical to the reference,
        utils/mask_layers.py:36-43: the RNG stream is part of the mask-parity contract)."""
        self.mask = torch.zeros_like(self.weight).bernoulli_(p)

    def _check_plain(self):
        if getattr(self, "groups", 1) != 1 or any(d != 1 for d in _pair(getattr(self, "dilation", 1))):
            raise NotImplementedError("grouped / dilated masked convolutions (the reference drops these too)")


class ConvMask(_MaskMixin, nn.Conv2d):
    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self._init_mask()

    def forward(self, x, want_skip=False, want_stats=False):
        """``want_skip=True`` additionally returns ``x`` as a second output whose gradient is accumulated inside
        this layer's dgrad kernel (used by the fused ResNet block forwards for the identity / downsample paths).
        ``want_stats=True`` appends the BatchNorm batch statistics of the output, computed in the conv epilogue
        (consumed by the BatchNorm2dB200 that follows: no separate statistics pass over the activation)."""
        self._check_plain()
        if isinstance(self.padding, str):
            raise NotImplementedError("string padding modes")
        return ops.masked_conv2d(x, self.weight, self.mask, self.bias, _pair(self.stride), _pair(self.padding), want_skip, _slots(self),
                                 ops.take_staged(self), want_stats, getattr(x, "_tp_bn_src", None))


class LinearMask(_MaskMixin, nn.Linear):
    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self._init_mask()

    def forward(self, x):
        return ops.masked_linear(x, self.weight, self.mask, self.bias, _slots(self), ops.take_staged(self))


class Conv1dMask(_MaskMixin, nn.Conv1d):
    """nn.Linear replacement with weight [out, in, 1] (reference: utils/mask_layers.py:82-119)."""

    def __init__(self, in_features: int, out_features: int, bias: bool = False):
        super().__init__(in_channels=in_features, out_channels=out_features, kernel_size=1, stride=1, bias=bias)
        self._init_mask()

    def forward(self, x):
        w = self.weight
        return ops.masked_linear(x, w.view(w.shape[0], w.shape[1]), self.mask.view(w.shape[0], w.shape[1]), self.bias, _slots(self), ops.take_staged(self))


MASKED_LAYER_TYPES = (ConvMask, Conv1dMask, LinearMask)
