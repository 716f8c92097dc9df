"""``PruningHarness`` — drop-in for the reference's ``harness_definitions/standard_pruning_harness.py``.

``PruningHarness(cfg, gpu_id, expt_dir, model=None)`` and ``.train_one_level(epochs_per_level, level)`` keep the
reference's behaviour (:28-50, :159-269): a fresh optimizer and LR schedule per level (momentum never carries
over), ``model_init.pt`` / ``optimizer_init.pt`` at level 0, ``model_rewind.pt`` at ``pruning_params.rewind_epoch``,
per-level CSV + summary CSV.  Optimizer = ``FusedSGD`` (same state-dict layout as torch.optim.SGD), or ``FusedAdamW``
(torch.optim.AdamW's) when ``optimizer_params.optimizer_name`` is ``AdamW``, or ``FusedMuon`` (Muon for the hidden masked
weights, AdamW for the rest) when it is ``MuonAdamW``.  Loaders: the
reference's device-resident CIFAR loader (``AirbenchLoaders``) when a CIFAR config names a ``dataset_params.dataloader_type``
other than ``synthetic`` (the reference's ``dp_cifar*.yaml`` say ``torch``); ``ImageFolderImagenet`` (GPU-decoded
ImageFolder tree) when an ImageNet config says ``dataloader_type: imagefolder``; otherwise (FFCV / WebDataset are out of
scope) the synthetic on-device generator.

``pruning_params.training_type: rigl`` trains with dynamic sparse masks (RigL, utils/rigl.py): on an update batch the
harness runs one eager forward / backward with dense weight gradients instead of the train step, drops and regrows
weights in place (``pruning_utils.rigl_update``), takes no optimizer step and zeroes the gradients.  Every other batch
is the ordinary train step, whose captured CUDA graph stays valid across updates.
"""
import csv
import os
import sys
from typing import Optional

import torch
import torch.nn as nn
from torch.amp import autocast

from ..optim import FusedAdamW, FusedMuon, FusedSGD
from ..utils import schedulers
from ..utils.custom_models import CustomModel, TorchVisionModel
from ..utils.dataset import AirbenchLoaders, ImageFolderImagenet, SyntheticLoaders
from ..utils.harness_utils import save_model
from ..utils.rigl import RiglSchedule, rigl_params
from .base_harness import BaseHarness


class PruningHarness(BaseHarness):
    def __init__(self, cfg, gpu_id: int, expt_dir, model: Optional[nn.Module] = None):
        self.gpu_id = gpu_id
        self.dataset_name = cfg.dataset_params.dataset_name.lower()
        self.use_compile = cfg.model_params.use_compile
        self.num_classes = 1000 if self.dataset_name.startswith("imagenet") else (100 if self.dataset_name.startswith("cifar100") else 10)
        local = int(os.environ.get("LOCAL_RANK", gpu_id))
        self.this_device = torch.device("cuda", local)
        self.prefix, self.expt_dir = expt_dir
        distributed = (cfg.experiment_params.distributed and torch.distributed.is_available()
                       and torch.distributed.is_initialized() and not self.dataset_name.startswith("cifar"))
        self._rigl_params = rigl_params(cfg)          # raises ValueError for a config RigL cannot start from
        self.rigl = None                               # this level's RiglSchedule (train_one_level / begin_rigl_level)
        super().__init__(cfg=cfg, device=self.this_device, model=model, distributed=distributed)

    def _create_model(self):
        try:
            model = TorchVisionModel(cfg=self.cfg)
        except ValueError:
            model = CustomModel(cfg=self.cfg)            # the reference's fallback (broken upstream) for DeiT names
        return model

    def _setup_dataloaders(self):
        kind = getattr(self.cfg.dataset_params, "dataloader_type", None)
        world = torch.distributed.get_world_size() if self.distributed else 1
        rank = torch.distributed.get_rank() if self.distributed else 0
        if self.dataset_name.startswith("cifar") and kind is not None and kind != "synthetic":
            loaders = AirbenchLoaders(self.cfg, self.device)          # reference :145-148; CIFAR never runs distributed
            print(f"Data: CifarLoader ({self.cfg.dataset_params.dataset_name}, {self.cfg.dataset_params.data_root_dir})",
                  file=sys.stderr)
        elif self.dataset_name.startswith("imagenet") and kind == "imagefolder":
            loaders = ImageFolderImagenet(self.cfg, self.device, world, rank)
            print(f"Data: ImageFolderImagenet ({self.cfg.dataset_params.data_root_dir}/{{train,val}}, rank {rank} of {world})",
                  file=sys.stderr)
        else:
            loaders = SyntheticLoaders(self.cfg, self.device, world, rank)
            print(f"Data: SyntheticLoaders ({self.cfg.dataset_params.dataset_name}-shaped on-device batches)", file=sys.stderr)
        return loaders.train_loader, loaders.test_loader

    def _setup_optimizer(self):
        o = self.cfg.optimizer_params
        if o.scheduler_type == "ScheduleFree":
            raise NotImplementedError("ScheduleFree optimizer (third-party package, off the benchmarked path)")
        # capturable: the learning rate is a device scalar refreshed by train_step (sync_lr), so the captured step
        # follows the per-iteration LR schedule without being re-recorded
        if o.get("optimizer_name", "SGD") == "AdamW":
            self.optimizer = FusedAdamW(self.model.parameters(), lr=o.lr, betas=tuple(o.get("betas") or (0.9, 0.999)),
                                        eps=o.get("eps") or 1e-8, weight_decay=o.weight_decay, capturable=True)
            return
        if o.get("optimizer_name", "SGD") == "MuonAdamW":
            self.optimizer = self._muon_adamw(o)
            return
        # SGD, and (as in the reference, whose harness builds SGD whatever the name says) every other name (Muon too)
        self.optimizer = FusedSGD(self.model.parameters(), lr=o.lr, momentum=o.momentum, weight_decay=o.weight_decay,
                                  capturable=True)

    def _muon_adamw(self, o):
        """Muon for the weights of every masked layer but the classifier (the last masked layer in module order, whose
        output width is the class count), AdamW for every other parameter: biases, norms, the classifier, DeiT's
        unmasked patch embedding.  One lr and one weight decay serve both groups: ``adjust_lr_fn`` defaults to
        ``match_rms_adamw``, which scales Muon's step to AdamW's update RMS."""
        from ..utils.mask_layers import MASKED_LAYER_TYPES
        masked = [m for m in self.model.modules() if isinstance(m, MASKED_LAYER_TYPES)]
        if not masked:
            raise ValueError("MuonAdamW: the model has no masked layer to train with Muon")
        head = masked[-1]
        num_classes = getattr(self, "num_classes", None)
        assert num_classes is None or head.weight.shape[0] == num_classes, \
            f"MuonAdamW: the last masked layer has {head.weight.shape[0]} outputs, not the {num_classes} classes"
        hidden = [m.weight for m in masked[:-1]]
        ids = {id(w) for w in hidden}
        rest = [p for p in self.model.parameters() if id(p) not in ids]
        groups = [dict(params=hidden, use_muon=True), dict(params=rest, use_muon=False)]
        return FusedMuon([g for g in groups if g["params"]], lr=o.lr, weight_decay=o.weight_decay, momentum=o.momentum,
                         nesterov=bool(o.get("nesterov", True)), ns_steps=int(o.get("ns_steps", 5)),
                         adjust_lr_fn=o.get("adjust_lr_fn", "match_rms_adamw"),
                         adamw_betas=tuple(o.get("betas") or (0.9, 0.999)), adamw_eps=o.get("eps") or 1e-8,
                         capturable=True)

    def _setup_scheduler(self, epochs_per_level):
        kind = self.cfg.optimizer_params.scheduler_type
        if kind == "OneCycleLR":
            self.scheduler = torch.optim.lr_scheduler.OneCycleLR(self.optimizer, max_lr=self.cfg.optimizer_params.lr,
                                                                 epochs=epochs_per_level, steps_per_epoch=len(self.train_loader))
        elif kind == "TriangularSchedule":
            self.scheduler = schedulers.TriangularSchedule(self.cfg, self.optimizer, len(self.train_loader), epochs_per_level)
        else:
            raise NotImplementedError(f"scheduler {kind}: its reference call site passes arguments the class does not accept")

    def train_one_level(self, epochs_per_level: int, level: int) -> None:
        rows = []
        model = self.model
        self._setup_optimizer()
        self._setup_scheduler(epochs_per_level)
        if self._rigl_params is not None:
            self.begin_rigl_level(epochs_per_level)
        ck = os.path.join(self.expt_dir, "checkpoints")
        art = os.path.join(self.expt_dir, "artifacts")
        if self.gpu_id == 0 and level == 0:
            save_model(self.model, os.path.join(ck, "model_init.pt"))
            torch.save(self.optimizer.state_dict(), os.path.join(art, "optimizer_init.pt"))
        rewind_epoch = getattr(self.cfg.pruning_params, "rewind_epoch", None)
        for epoch in range(epochs_per_level):
            self.epoch_counter += 1
            if self.gpu_id == 0:
                self.console.rule(f"Current Epoch: {epoch + 1}/{epochs_per_level}")
            metrics = {"epoch": int(self.epoch_counter), **self.train_epoch(), **self.test()}
            if self.gpu_id == 0 and rewind_epoch == epoch and level == 0:
                save_model(self.model, os.path.join(ck, "model_rewind.pt"))
                torch.save(self.optimizer.state_dict(), os.path.join(art, "optimizer_rewind.pt"))
            if self.gpu_id == 0:
                self.console.print({k: (round(v, 4) if isinstance(v, float) else v) for k, v in metrics.items()})
                rows.append({**metrics, "max_test_acc": max([r["test_acc"] for r in rows] + [metrics["test_acc"]]),
                             "sparsity": model.get_overall_sparsity()})
        if self.gpu_id == 0:
            path = os.path.join(self.expt_dir, "metrics", "level_wise_metrics", f"level_{level}_metrics.csv")
            with open(path, "w", newline="") as f:
                w = csv.DictWriter(f, fieldnames=list(rows[0].keys())); w.writeheader(); w.writerows(rows)
            summary = os.path.join(self.expt_dir, f"{self.prefix}_summary.csv")
            new = not os.path.exists(summary)
            with open(summary, "a", newline="") as f:
                w = csv.writer(f)
                if new:
                    w.writerow(["Level", "Sparsity", "Last_Test_Acc", "Max_Test_Acc"])
                w.writerow([level, model.get_overall_sparsity(), rows[-1]["test_acc"], max(r["test_acc"] for r in rows)])

    # ---- RigL: dynamic sparse masks within a level ---------------------------------------------------------------
    def _masked_layers(self):
        from ..utils.mask_layers import MASKED_LAYER_TYPES
        return [m for m in self.model.modules() if isinstance(m, MASKED_LAYER_TYPES)]

    def begin_rigl_level(self, epochs_per_level: int) -> None:
        """Start a RigL level of ``epochs_per_level * len(train_loader)`` batches: count every layer's active weights
        (one host sync; RigL keeps the counts) and allocate the scratch masks the updates reuse."""
        from .. import ops
        layers = self._masked_layers()
        for m in layers:
            if m.mask.device != m.weight.device or m.mask.dtype != torch.float32 or not m.mask.is_contiguous():
                m.mask = m.mask.to(device=m.weight.device, dtype=torch.float32).contiguous()
        zeros = ops.count_zeros([m.mask for m in layers]).cpu().tolist()
        self.rigl = RiglSchedule(*self._rigl_params, total_steps=epochs_per_level * len(self.train_loader))
        self.rigl_active = [m.mask.numel() - z for m, z in zip(layers, zeros)]
        self.rigl_step = 0                         # batches consumed in this level
        self.rigl_counts = None                    # (dropped, grown) per layer of the last update, int64 cuda [layers, 2]
        self._rigl_new = [torch.empty_like(m.mask) for m in layers]

    def train_step(self, batch):
        t = getattr(self, "rigl_step", None)
        if self.rigl is not None and self.rigl.is_update(t):
            out = self._rigl_update_step(batch, self.rigl.k_per_layer(t, self.rigl_active))
        else:
            out = super().train_step(batch)
        if self.rigl is not None:
            self.rigl_step = t + 1
        return out

    def _rigl_update_step(self, batch, k_per_layer):
        """Dense-gradient forward / backward, drop-and-regrow in place, no optimizer step.  Under torch.distributed
        every rank uses its own dense gradient (no exchange on this batch) and rank 0's masks are imposed."""
        from .. import fused_norm, ops
        from ..utils.pruning_utils import rigl_update
        inputs, targets = batch
        inputs, targets = inputs.to(self.device, non_blocking=True), targets.to(self.device, non_blocking=True)
        store = self._grad_store()
        store.zero()
        with self._compute_precision(), ops.dense_weight_grad():
            self._weight_stager().stage()
            with autocast(device_type="cuda", dtype=self.precision, enabled=self.use_amp):
                outputs = self.model(inputs)
                loss = self.criterion(outputs, targets)
            try:
                loss.backward()
            finally:
                ops.join_wgrad(self.device)
                fused_norm.drop_partials()
        self.rigl_counts = rigl_update(self.model, self.optimizer, k_per_layer, new_masks=self._rigl_new)
        if self.reducer is not None:
            self.reducer.set_model_masks(getattr(self.model, "model", self.model))     # in place: same buffers
        store.zero()
        self._drop_staged()                        # the next step restages the weights from the new masks
        self.train_accuracy.update(outputs.detach(), targets)
        return {"loss": loss.detach()}
