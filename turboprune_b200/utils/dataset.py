"""Synthetic on-device generator standing in for the reference's loaders (utils/dataset.py: CifarLoader
:101-226, FFCVImagenet :347-430 — out of scope: they need the data sets / FFCV / network).

Same batch contract: an iterable of ``(images fp32 [B,3,H,W], labels int64 [B])`` with ``len()``; ImageNet-shaped
batches come channels_last like FFCV's ToTorchImage.  Seeded per rank; either a fixed number of distinct batches is
generated once and cycled (an epoch costs no host work), or (``dataset_params.synthetic_fresh``) every step draws a new
batch on the device.  ``DevicePrefetcher`` is the host->device leg for loaders that produce pinned host batches.
"""
from ctypes import c_void_p

import torch

from .. import _cabi, ops


# ---- airbench-style GPU augmentation (reference utils/dataset.py:38-98): same names, same draws, one fused kernel ------
def _ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else None


def _augment(src, out_hw, r, shifts=None, flip=None, corner_y=None, corner_x=None, cut_size=0):
    if not src.is_cuda:
        raise RuntimeError("turboprune_b200 augmentation kernels need CUDA tensors (H100 / sm_90a); there is no CPU path")
    lib = _cabi.load()
    src = src.contiguous().float()
    n, c = src.shape[:2]
    h, w = out_hw
    out = torch.empty(n, c, h, w, dtype=torch.float32, device=src.device)
    f8 = flip.to(torch.uint8).contiguous() if flip is not None else None
    sh = shifts.to(torch.int64).contiguous() if shifts is not None else None
    cy = corner_y.to(torch.int64).contiguous() if corner_y is not None else None
    cx = corner_x.to(torch.int64).contiguous() if corner_x is not None else None
    with torch.cuda.device(src.device):
        rc = lib.tp_cifar_augment(_ptr(src), _ptr(out), _ptr(sh), _ptr(f8), _ptr(cy), _ptr(cx), int(cut_size), n, c, h, w, int(r),
                                  _cabi.stream_ptr(src.device))
    _cabi.check(rc, "tp_cifar_augment")
    ops._count()
    return out


def batch_flip_lr(inputs):
    """reference :38-40 — the flip mask is drawn with torch's generator on the inputs' device, like upstream."""
    flip_mask = torch.rand(len(inputs), device=inputs.device) < 0.5
    return _augment(inputs, inputs.shape[-2:], 0, flip=flip_mask)


def batch_crop(images, crop_size):
    """reference :43-69 — random translation: a crop_size window of the padded images at a per-image shift."""
    r = (images.size(-1) - crop_size) // 2
    shifts = torch.randint(-r, r + 1, size=(len(images), 2), device=images.device)
    return _augment(images, (crop_size, crop_size), r, shifts=shifts)


def batch_cutout(inputs, size):
    """reference :72-98 — one size x size square per image zeroed."""
    n, c, h, w = inputs.shape
    corner_y = torch.randint(0, h - size + 1, size=(n,), device=inputs.device)
    corner_x = torch.randint(0, w - size + 1, size=(n,), device=inputs.device)
    return _augment(inputs, (h, w), 0, corner_y=corner_y, corner_x=corner_x, cut_size=size)


def augment_epoch(padded, crop_size, flip=True, cutout=0):
    """CifarLoader.__iter__ (:204-221, random-flip branch) for one epoch in ONE pass: the draws are made in the
    reference's order (crop shifts, flip mask, cutout corners), the pixels move once instead of three times."""
    n = len(padded)
    r = (padded.size(-1) - crop_size) // 2
    shifts = torch.randint(-r, r + 1, size=(n, 2), device=padded.device) if r > 0 else None
    flip_mask = (torch.rand(n, device=padded.device) < 0.5) if flip else None
    cy = cx = None
    if cutout > 0:
        cy = torch.randint(0, crop_size - cutout + 1, size=(n,), device=padded.device)
        cx = torch.randint(0, crop_size - cutout + 1, size=(n,), device=padded.device)
    return _augment(padded, (crop_size, crop_size), r, shifts=shifts, flip=flip_mask, corner_y=cy, corner_x=cx, cut_size=cutout)


def synth_normal_(out, seed, counter_offset=0, raw_words=False):
    """Fill ``out`` (fp32, dense memory) with the Philox4x32-10 / Box-Muller stream (element order = memory order)."""
    lib = _cabi.load()
    with torch.cuda.device(out.device):
        rc = lib.tp_synth_normal(_ptr(out), out.numel(), int(seed), int(counter_offset), int(bool(raw_words)), _cabi.stream_ptr(out.device))
    _cabi.check(rc, "tp_synth_normal")
    ops._count()
    return out


def synth_labels_(out, num_classes, seed, counter_offset=0):
    lib = _cabi.load()
    with torch.cuda.device(out.device):
        rc = lib.tp_synth_labels(_ptr(out), out.numel(), int(num_classes), int(seed), int(counter_offset), _cabi.stream_ptr(out.device))
    _cabi.check(rc, "tp_synth_labels")
    ops._count()
    return out


class SyntheticLoader:
    """``fresh=True``: every iteration draws a new batch on the device (Philox, seeded per rank — SURVEY.md §8(d));
    otherwise ``distinct`` batches are generated once and cycled."""

    def __init__(self, batch_size, steps, shape, num_classes, device, seed=0, distinct=4, channels_last=False, fresh=False):
        self.gen = torch.Generator(device=device).manual_seed(seed)
        self.seed, self._ctr = int(seed), 0
        self.steps = steps
        self.batch_size, self.shape, self.num_classes, self.device = batch_size, tuple(shape), num_classes, device
        self.channels_last = channels_last
        self.fresh = fresh
        self.batches = [] if fresh else [self._draw() for _ in range(min(distinct, steps))]

    def _draw(self):
        c, h, w = self.shape
        dev = torch.device(self.device)
        if dev.type == "cuda":
            # our generator: Philox4x32-10 -> Box-Muller straight into the batch buffer, a fresh counter range per batch
            shp = (self.batch_size, h, w, c) if self.channels_last else (self.batch_size, c, h, w)
            x = torch.empty(shp, dtype=torch.float32, device=dev)
            t = torch.empty(self.batch_size, dtype=torch.int64, device=dev)
            synth_normal_(x, self.seed, self._ctr)
            synth_labels_(t, self.num_classes, self.seed ^ 0x5DEECE66D, self._ctr)
            self._ctr += (x.numel() + 3) // 4
            return (x.permute(0, 3, 1, 2) if self.channels_last else x), t
        if self.channels_last:       # NHWC memory, logical NCHW (what FFCV's ToTorchImage hands over, dataset.py:391)
            x = torch.randn(self.batch_size, h, w, c, device=self.device, generator=self.gen).permute(0, 3, 1, 2)
        else:
            x = torch.randn(self.batch_size, c, h, w, device=self.device, generator=self.gen)
        return x, torch.randint(0, self.num_classes, (self.batch_size,), device=self.device, generator=self.gen)

    def __len__(self):
        return self.steps

    def __iter__(self):
        for i in range(self.steps):
            yield self._draw() if self.fresh else self.batches[i % len(self.batches)]


class DevicePrefetcher:
    """Wraps an iterable of HOST batches (pinned ``(images, labels)``) and yields device batches: batch i+1 crosses PCIe
    on a copy stream while step i computes (two staging slots, guarded by events).  Stands where the reference's
    loaders hand over device tensors (FFCV ``ToDevice(non_blocking=True)``, dataset.py:385-430)."""

    def __init__(self, host_loader, device):
        self.loader, self.device = host_loader, device
        self.copy_stream = torch.cuda.Stream(device)
        self.slots = [None, None]
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.consumed = [torch.cuda.Event(), torch.cuda.Event()]

    def __len__(self):
        return len(self.loader)

    def _issue(self, j, batch):
        x, t = batch
        if self.slots[j] is None or self.slots[j][0].shape != x.shape:
            self.slots[j] = (torch.empty_strided(x.shape, x.stride(), dtype=x.dtype, device=self.device),
                             torch.empty(t.shape, dtype=t.dtype, device=self.device))
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.consumed[j])
            self.slots[j][0].copy_(x, non_blocking=True); self.slots[j][1].copy_(t, non_blocking=True)
            self.ready[j].record(self.copy_stream)

    def __iter__(self):
        cur = torch.cuda.current_stream(self.device)
        for ev in self.consumed:
            ev.record(cur)
        it = iter(self.loader)
        nxt = next(it, None)
        if nxt is None:
            return
        self._issue(0, nxt)
        i = 0
        while nxt is not None:
            j = i % 2
            nxt = next(it, None)
            if nxt is not None:
                self._issue(1 - j, nxt)              # overlaps with the step consuming slot j
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(self.ready[j])
            yield self.slots[j]
            self.consumed[j].record(torch.cuda.current_stream(self.device))
            i += 1


class SyntheticLoaders:
    """train_loader / test_loader pair sized from the config (dataset_params.total_batch_size // world_size,
    reference dataset.py:411)."""

    def __init__(self, cfg, device, world_size=1, rank=0):
        name = cfg.dataset_params.dataset_name.lower()
        ncls = 1000 if name.startswith("imagenet") else (100 if name.startswith("cifar100") else 10)
        shape = (3, 224, 224) if name.startswith("imagenet") else (3, 32, 32)
        bs = max(1, cfg.dataset_params.total_batch_size // world_size)
        steps = int(getattr(cfg.dataset_params, "synthetic_steps_per_epoch", 8))
        seed = cfg.experiment_params.seed * world_size + rank
        fresh = bool(getattr(cfg.dataset_params, "synthetic_fresh", False))
        self.train_loader = SyntheticLoader(bs, steps, shape, ncls, device, seed, channels_last=name.startswith("imagenet"),
                                            fresh=fresh)
        self.test_loader = SyntheticLoader(bs, max(1, steps // 4), shape, ncls, device, seed + 7919,
                                           channels_last=name.startswith("imagenet"))
