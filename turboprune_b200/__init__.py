"""turboprune_b200 — H100-native (sm_90a) implementation of TurboPrune's masked-DDP hot path.

Host side mirrors the reference's surface (``utils.mask_layers``, ``utils.pruning_utils``,
``utils.custom_models``, ``harness_definitions``); the arithmetic runs in hand-written CUDA
kernels behind the C ABI declared in ``include/turboprune_b200.h``.
"""
from . import _cabi  # noqa: F401

__all__ = ["_cabi"]
