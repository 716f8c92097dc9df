"""Generic train / eval loop — drop-in for the reference's ``harness_definitions/base_harness.py``.

Same attributes and methods the driver relies on (``.model .train_loader .val_loader .distributed .console
.optimizer .scheduler``; ``train_step / test_step / train_epoch / test``, reference :115-245).  Differences:
  * the model is NOT wrapped in DistributedDataParallel: gradients are averaged by ``P2PGradReducer`` (one NVLink
    kernel per bucket, launched on a side stream as soon as the bucket's last gradient is written, i.e. under the
    rest of the backward pass); masks are broadcast once per pruning step, never per forward;
  * ``train_step`` owns the persistent gradient storage, the one-launch bf16 weight shadow and a CUDA-graph capture
    of the whole step (replayed from the third step of a level on);
  * the per-step ``loss.item()`` host sync (reference :134) is deferred: losses accumulate on the device and are
    read once per epoch;
  * accuracy is a two-integer device counter instead of torchmetrics (not installed);
  * a schedule-free optimizer (one with ``train()`` / ``eval()``) is put in train mode by ``train_step`` and in eval
    mode by ``test()``, so evaluation and the checkpoints saved after it see the averaged weights x (the reference never
    calls either, so its evaluation and checkpoints see the training iterate y).
"""
from contextlib import nullcontext

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.amp import autocast


class _Console:
    def print(self, *a, **k):
        print(*[str(x) for x in a])

    def rule(self, title=""):
        print("-" * 20, title, "-" * 20)


class _Accuracy:
    def __init__(self, device):
        self.stat = torch.zeros(2, dtype=torch.int64, device=device)

    def update(self, outputs, targets):
        self.stat[0] += (outputs.argmax(1) == targets).sum()
        self.stat[1] += targets.numel()

    def compute(self, distributed=False):
        s = self.stat.clone()
        if distributed:
            dist.all_reduce(s)
        return (s[0].float() / s[1].clamp(min=1).float())

    def reset(self):
        self.stat.zero_()


class BaseHarness:
    def __init__(self, cfg, device, model=None, distributed: bool = False):
        self.cfg = cfg
        self.device = device
        self.distributed = distributed
        self.epoch_counter = 0
        self.console = _Console()
        self.model = self._setup_model(model)
        self.criterion = nn.CrossEntropyLoss()
        self.train_accuracy = _Accuracy(self.device)
        self.test_accuracy = _Accuracy(self.device)
        self.train_loader, self.val_loader = self._setup_dataloaders()
        self.precision, self.use_amp = self._get_dtype_amp()
        self.reducer = None
        self._arena = None
        self._stager = None
        self._graph = None               # captured train step: dict(key, graph, x, t, loss)
        self._warm = {}
        self._capture_stream = None

    # the reference wraps in DDP here (base_harness.py:74-82); we keep the bare module and reduce explicitly
    def _setup_model(self, model):
        if model is None:
            model = self._create_model()
        return model.to(self.device)

    def _create_model(self):
        raise NotImplementedError

    def _setup_dataloaders(self):
        raise NotImplementedError

    def _get_dtype_amp(self):
        table = {"bfloat16": (torch.bfloat16, True), "float16": (torch.float16, True), "float32": (torch.float32, False)}
        return table.get(self.cfg.experiment_params.training_precision, (torch.float32, False))

    def _ensure_reducer(self):
        if self.distributed and self.reducer is None:
            from ..grad_exchange import get_reducer
            # one reducer per process and parameter set: the level loop builds a new harness around the same module
            # every level (reference run_experiment.py:113-115); the symmetric buckets are reused
            self.reducer = get_reducer(list(self.model.parameters()))
            inner = getattr(self.model, "model", self.model)
            self.reducer.set_model_masks(inner)          # masks of THIS level, applied while the mean is written back

    def _grad_store(self):
        if self.distributed:
            self._ensure_reducer()
            return self.reducer
        if self._arena is None:
            from ..grad_exchange import GradArena
            self._arena = GradArena(list(self.model.parameters()))
        return self._arena

    def _weight_stager(self):
        if self._stager is None:
            from .. import ops
            from ..utils.mask_layers import MASKED_LAYER_TYPES
            self._stager = ops.WeightStager([m for m in self.model.modules() if isinstance(m, MASKED_LAYER_TYPES)])
        return self._stager

    # ---- the train step (reference :115-134), owned by the harness: persistent gradient storage, one-launch weight
    # ---- shadow, gradient exchange overlapped with the backward pass, CUDA-graph replay ---------------------------
    def _step_body(self, inputs, targets):
        """zero_grad -> autocast forward -> CE -> backward (+ P2P gradient mean under it) -> SGD -> accuracy.
        Everything here is device work on the current stream (capturable: no host sync, no pointer changes)."""
        from .. import ops
        store = self._grad_store()
        store.zero()                       # one memset of the persistent gradient storage (param.grad views its slot)
        if self.distributed:
            store.arm()                    # finished gradients start their bucket's reduce on a side stream
        with self._compute_precision():
            self._weight_stager().stage()      # bf16(mask * w) operands of every masked layer: one launch
            with autocast(device_type="cuda", dtype=self.precision, enabled=self.use_amp):
                outputs = self.model(inputs)
                loss = self.criterion(outputs, targets)
            side_wgrad = bool(getattr(self.cfg.experiment_params, "wgrad_side_stream", True))
            ops.set_wgrad_side_stream(side_wgrad)     # weight gradients run on a side stream beside the dgrad chain ...
            try:
                loss.backward()
            finally:
                ops.set_wgrad_side_stream(False)
                ops.join_wgrad(self.device)           # ... and are joined before anything reads param.grad
                from .. import fused_norm
                fused_norm.drop_partials()
        if self.distributed:
            self.reducer.reduce()          # joins the side stream; leftover buckets go out here
        self.optimizer.step()
        self.train_accuracy.update(outputs.detach(), targets)
        return loss.detach()

    def _compute_precision(self):
        """training_precision: float32 runs the masked layers with fp32 operands on TF32 tensor cores (the reference's
        float32 mode with allow_tf32); every other precision keeps the default bf16 kernels."""
        if self.precision == torch.float32:
            from .. import ops
            return ops.compute_precision(torch.float32)
        return nullcontext()

    def _graph_enabled(self):
        return bool(getattr(self.cfg.experiment_params, "cuda_graph", True)) and hasattr(self.optimizer, "sync_lr")

    def _graph_key(self, inputs, targets):
        from ..utils import mask_layers
        return (tuple(inputs.shape), inputs.dtype, tuple(inputs.stride()), tuple(targets.shape), targets.dtype,
                id(self.optimizer), self.model.training, mask_layers.mask_epoch(), self.precision)

    def train_step(self, batch):
        """One optimisation step; returns ``{"loss": 0-dim device tensor}`` (the host sync of the reference's
        ``loss.item()``, :134, is left to the caller / deferred to the end of the epoch).

        Calls 1-3 with a given batch geometry run eagerly (the third on a side stream, then the step is captured);
        from then on a step is: copy the batch into the static buffers, refresh the device LR scalar, replay the graph.
        The capture is dropped when the batch geometry, the optimizer, train/eval mode or any mask tensor changes."""
        inputs, targets = batch
        inputs, targets = inputs.to(self.device, non_blocking=True), targets.to(self.device, non_blocking=True)
        if not inputs.is_cuda:
            raise RuntimeError("turboprune_b200: the train step needs CUDA tensors (H100 / sm_90a); there is no CPU path")
        self._optimizer_mode(train=True)  # in place: a captured step stays valid across the switches
        sync_lr = getattr(self.optimizer, "sync_lr", None)
        key = self._graph_key(inputs, targets)
        g = self._graph if self._graph_enabled() else None
        if g is not None and g["key"] == key:
            g["x"].copy_(inputs, non_blocking=True); g["t"].copy_(targets, non_blocking=True)
            sync_lr()
            g["graph"].replay()
            return {"loss": g["loss"]}
        if g is not None:                  # geometry / masks / optimizer changed: start over
            self._graph = None
            self._warm = {}
        if not self._graph_enabled():
            if sync_lr is not None:
                sync_lr()
            loss = self._step_body(inputs, targets)
            self._drop_staged()
            return {"loss": loss}
        n = self._warm.get(key, 0)
        self._warm[key] = n + 1
        cur = torch.cuda.current_stream(self.device)
        if sync_lr is not None:
            sync_lr()
        if n == 0:
            loss = self._step_body(inputs, targets)
            self._drop_staged()
            return {"loss": loss}
        # warm-up on the side stream the capture will fork from (allocator pools, workspaces and autograd's stream
        # bookkeeping must have seen it), then capture — this call's batch is trained by the eager run
        side = self._capture_stream
        if side is None:
            side = self._capture_stream = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            loss = self._step_body(inputs, targets)
        cur.wait_stream(side)
        if n >= 2:
            x = torch.empty_strided(inputs.shape, inputs.stride(), dtype=inputs.dtype, device=self.device)
            t = torch.empty_like(targets)
            x.copy_(inputs); t.copy_(targets)
            torch.cuda.synchronize(self.device)
            if self.distributed:
                dist.barrier()             # every rank enters the capture together (the captured step has peer barriers)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
                gl = self._step_body(x, t)
            self._graph = dict(key=key, graph=graph, x=x, t=t, loss=gl)
        self._drop_staged()
        return {"loss": loss}

    def _optimizer_mode(self, train: bool):
        """Schedule-free optimizers keep the weights at y to train and at the average x to evaluate; ``train()`` /
        ``eval()`` move them (no-ops when already there).  Other optimizers have neither method."""
        opt = getattr(self, "optimizer", None)
        fn = getattr(opt, "train" if train else "eval", None)
        if callable(fn) and callable(getattr(opt, "eval" if train else "train", None)):
            fn()

    def _drop_staged(self):
        """A staged operand pair must never outlive its step (a layer skipped by this forward would otherwise feed the
        next eval / pruning forward bf16 weights from before optimizer.step())."""
        if self._stager is not None:
            self._stager.drop()

    def test_step(self, batch):
        inputs, targets = batch
        inputs, targets = inputs.to(self.device, non_blocking=True), targets.to(self.device, non_blocking=True)
        with torch.no_grad(), self._compute_precision(), autocast(device_type="cuda", dtype=self.precision, enabled=self.use_amp):
            outputs = self.model(inputs)
            loss = self.criterion(outputs, targets)
            self.test_accuracy.update(outputs, targets)
        return {"loss": loss.detach()}

    def _epoch(self, loader, step_fn, acc, per_iter_sched):
        total = torch.zeros((), device=self.device)
        for batch in loader:
            total += step_fn(batch)["loss"].float()
            if per_iter_sched and self.scheduler is not None:
                self.scheduler.step()
        avg = total / max(1, len(loader))
        accuracy = acc.compute(self.distributed)
        if self.distributed:
            dist.all_reduce(avg, op=dist.ReduceOp.AVG)
        acc.reset()
        out = float(avg.item()), float(accuracy.item()) * 100           # the only host syncs of the epoch
        if self.reducer is not None:
            self.reducer.check_status()      # a peer-barrier timeout leaves gradients unreduced: fail, do not train on
        return out

    def train_epoch(self):
        self.model.train()
        per_iter = self.cfg.optimizer_params.scheduler_type in ("OneCycleLR", "TriangularSchedule", "TrapezoidalSchedule")
        loss, acc = self._epoch(self.train_loader, self.train_step, self.train_accuracy, per_iter)
        return {"train_loss": loss, "train_acc": acc}

    def test(self):
        self.model.eval()
        self._optimizer_mode(train=False)
        if self.distributed:        # the reference's DDP broadcasts rank 0's BN statistics on every forward
            for m in self.model.modules():
                if isinstance(m, nn.modules.batchnorm._BatchNorm) and m.running_mean is not None:
                    dist.broadcast(m.running_mean, 0); dist.broadcast(m.running_var, 0)
        loss, acc = self._epoch(self.val_loader, self.test_step, self.test_accuracy, False)
        return {"test_loss": loss, "test_acc": acc}
