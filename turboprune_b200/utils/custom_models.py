"""Model wrappers — drop-in for the reference's ``utils/custom_models.py``.

``PruneModel`` / ``TorchVisionModel`` / ``CustomModel`` keep the reference's methods and
semantics (utils/custom_models.py:18-245): layers are re-created (not copied) in
``named_children`` order so a seeded build yields bit-identical initial weights; the mask-layer
class is looked up BY NAME in this module's namespace (``mask_layer_type`` from the config);
``get_overall_sparsity`` returns PERCENT; ``reset_weights`` rewinds everything except ``*mask``.

Differences: sparsity accounting is one kernel launch + one sync instead of one ``.item()``
per layer (reference :51-62), and the network is kept in channels_last so activations reach the
masked convolutions as NHWC bf16 without a layout pass.
"""
import os
from typing import Dict, Type

import torch
import torch.nn as nn
from torchvision import models

from .. import ops
from .mask_layers import *  # noqa: F401,F403  (string lookup of mask_layer_type happens in this namespace)
from .mask_layers import MASKED_LAYER_TYPES, ConvMask, Conv1dMask, LinearMask
from . import vit as _vit


class PruneModel(nn.Module):
    def __init__(self):
        super().__init__()
        self.model = None

    def prepare(self, cfg):
        raise NotImplementedError("Subclasses must implement prepare method")

    def forward(self, x):
        return self.model(x)

    # ---- sparsity accounting -------------------------------------------------------------
    def _masked(self):
        return [(n, m) for n, m in self.model.named_modules() if isinstance(m, MASKED_LAYER_TYPES)]

    def _zero_counts(self):
        layers = self._masked()
        if not layers:
            return layers, []
        masks = [m.mask for _, m in layers]
        if masks[0].is_cuda:
            counts = ops.count_zeros(masks).tolist()          # one launch, one sync
        else:   # masks not yet moved to the GPU (e.g. right after construction): exact integer count
            counts = [int((mk == 0).sum()) for mk in masks]
            counts.append(sum(counts))
        return layers, counts

    def get_overall_sparsity(self) -> float:
        layers, counts = self._zero_counts()
        total = sum(m.mask.numel() for _, m in layers)
        return (counts[-1] / total) * 100 if total > 0 else 0

    def print_layer_sparsity(self):
        layers, counts = self._zero_counts()
        print("Layer-wise Sparsity (%)")
        for (name, m), z in zip(layers, counts):
            print(f"  {name:40s} {(z / m.mask.numel()) * 100:6.2f}")

    # ---- layer replacement -----------------------------------------------------------------
    def replace_layers(self, layer_types_map: Dict[Type[nn.Module], Type[nn.Module]]):
        """Swap layers by type; new layers are freshly initialised (only geometry and the
        presence of a bias are carried over — groups / dilation are not, as in the reference)."""

        def build(child, old_type, new_type):
            if old_type == nn.Linear and new_type == Conv1dMask:
                return Conv1dMask(in_features=child.in_features, out_features=child.out_features,
                                  bias=child.bias is not None)
            if old_type == nn.Conv2d and issubclass(new_type, nn.Conv2d):
                return new_type(in_channels=child.in_channels, out_channels=child.out_channels,
                                kernel_size=child.kernel_size, stride=child.stride, padding=child.padding,
                                bias=child.bias is not None)
            return new_type(in_features=child.in_features, out_features=child.out_features,
                            bias=child.bias is not None)

        def walk(module):
            for name, child in module.named_children():
                for old_type, new_type in layer_types_map.items():
                    if isinstance(child, old_type):
                        setattr(module, name, build(child, old_type, new_type))
                        break
                else:
                    walk(child)

        walk(self)

    # ---- checkpoints -------------------------------------------------------------------------
    def load_model(self, load_path):
        from .harness_utils import load_checkpoint
        self.model.load_state_dict(load_checkpoint(load_path))

    def reset_weights(self, cfg, expt_dir: str) -> None:
        kind = cfg.pruning_params.training_type
        if kind == "imp":
            ckpt = "model_init.pt"
        elif kind == "wr":
            ckpt = "model_rewind.pt"
        else:
            return                                        # LRR / pruning at init: nothing to rewind
        from .harness_utils import load_checkpoint
        saved = load_checkpoint(os.path.join(expt_dir, "checkpoints", ckpt))
        live = self.model.state_dict()
        for name, tensor in saved.items():
            if name in live and live[name].shape == tensor.shape and not name.endswith("mask"):
                live[name].copy_(tensor)
        self.model.load_state_dict(live)

    def reset_masks(self):
        for _, m in self._masked():
            m.mask.fill_(1)

    def load_only_masks(self, load_path: str):
        from .harness_utils import load_checkpoint
        saved = load_checkpoint(load_path)
        live = self.model.state_dict()
        for name, tensor in saved.items():
            if name in live and live[name].shape == tensor.shape and name.endswith("mask"):
                live[name].copy_(tensor)
        self.model.load_state_dict(live)


class TorchVisionModel(PruneModel):
    def __init__(self, cfg):
        super().__init__()
        self.model_name = cfg.model_params.model_name
        self.mask_layer_type = cfg.model_params.mask_layer_type
        self.prepare(cfg)

    def prepare(self, cfg):
        if not hasattr(models, self.model_name):
            raise ValueError(f"Model {self.model_name} not found in torchvision.models.")
        self.model = getattr(models, self.model_name)(weights=None)
        dataset = cfg.dataset_params.dataset_name.lower()
        if dataset in ("cifar10", "cifar100"):
            self._prepare_for_cifar(dataset)
        self._replace_layers()
        # BatchNorm / ReLU / residual-add between the masked convs run as fused NHWC kernels
        # (same modules, parameters and state-dict keys; SURVEY.md §8(f) row 1).
        # Inside ops.compute_precision(torch.float32) (a float32 config's step) these modules run the reference's own
        # ATen ops instead: the fused kernels are bf16-only (fused_norm.fused_enabled).
        if getattr(cfg.model_params, "fuse_norm", True):
            from ..fused_norm import fuse_torchvision_blocks
            fuse_torchvision_blocks(self.model)
        # Parameters keep their default (OIHW-contiguous) strides; activations become
        # channels_last (NHWC) at the first masked convolution and stay that way.

    def _prepare_for_cifar(self, dataset: str):
        ncls = 10 if dataset == "cifar10" else 100
        if self.model_name.startswith("resnet"):
            self.model.conv1 = nn.Conv2d(3, 64, kernel_size=3, stride=1, padding=1, bias=False)
            self.model.maxpool = nn.Identity()
            self.model.fc = nn.Linear(self.model.fc.in_features, ncls)
        elif self.model_name.startswith("vgg"):
            self.model.features[0] = nn.Conv2d(3, 64, kernel_size=3, padding=1)
            if hasattr(self.model, "classifier"):
                if isinstance(self.model.classifier, nn.Sequential):
                    self.model.classifier[-1] = nn.Linear(self.model.classifier[-1].in_features, ncls)
                else:
                    self.model.classifier = nn.Linear(self.model.classifier.in_features, ncls)

    def _replace_layers(self):
        conv_cls = globals().get(self.mask_layer_type)
        self.replace_layers({nn.Linear: Conv1dMask, nn.Conv2d: conv_cls})


class CustomModel(PruneModel):
    """Non-torchvision models (DeiT): every nn.Linear becomes LinearMask (reference :223-245).

    The reference resolves the name among timm-based factories in ``utils/deit.py``; timm is not
    available here, so ``utils/vit.py`` provides an equivalent ViT definition with the same
    hyper-parameters (deit.py:92-112).
    """

    def __init__(self, cfg):
        super().__init__()
        self.model_name = cfg.model_params.model_name
        self.mask_layer_type = cfg.model_params.mask_layer_type
        self.prepare(cfg)

    def prepare(self, cfg=None):
        factory = getattr(_vit, self.model_name, None)
        if factory is None:
            raise ValueError(f"Model {self.model_name} not found in torchvision.models or in the custom_models definition.")
        self.model = factory()
        self.replace_layers({nn.Linear: LinearMask})
