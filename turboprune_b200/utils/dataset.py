"""Data loaders of the reference's ``utils/dataset.py``, device-resident.

* ``CifarLoader`` / ``AirbenchLoaders`` (reference :101-256): the airbench CIFAR-10/100 loader, same names, constructor
  arguments, random draws and batches.  The data set lives on the GPU; each batch is ONE ``tp_cifar_augment`` launch
  that gathers the permuted source images and applies the epoch's translate / flip / cutout on the way, so an epoch
  never writes an augmented copy of the whole data set and never waits on the host.
* ``ImageFolderLoader`` / ``ImageFolderImagenet``: ImageNet from the standard ImageFolder tree
  ``{root}/{train,val}/<wnid>/*.JPEG`` with the transforms of the reference's FFCV pipelines (:347-430): files read by a
  thread pool, decoded batched on the GPU (nvjpeg through torchvision), and every batch's crops resized, mirrored and
  normalised by ONE ``tp_resized_crop`` launch, prepared on a side stream while the caller trains on the previous batch.
* ``SyntheticLoaders``: the on-device generator standing in for loaders whose data is not at hand (the FFCV beton and
  WebDataset readers, :347-546, are out of scope; benchmarks and synthetic configs use it for every data set).

Same batch contract throughout: an iterable of ``(images fp32 [B,3,H,W], labels int64 [B])`` with ``len()``;
ImageNet-shaped synthetic batches come channels_last like FFCV's ToTorchImage.  Synthetic loaders are seeded per rank;
either a fixed number of distinct batches is generated once and cycled (an epoch costs no host work), or
(``dataset_params.synthetic_fresh``) every step draws a new batch on the device.  ``DevicePrefetcher`` is the
host->device leg for loaders that produce pinned host batches.
"""
import math
import os
import queue
import sys
import threading
from concurrent.futures import ThreadPoolExecutor
from ctypes import c_float, c_void_p, sizeof
from functools import lru_cache
from math import ceil

import numpy as np
import torch

from .. import _cabi, ops


# ---- airbench-style GPU augmentation (reference utils/dataset.py:38-98): same names, same draws, one fused kernel ------
def _ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else None


def _augment(src, out_hw, r, shifts=None, flip=None, corner_y=None, corner_x=None, cut_size=0, idx=None):
    """One ``tp_cifar_augment`` launch.  ``idx`` (int64 [B] on the device): output image j is built from source image
    ``idx[j]``, and every draw is indexed by the source image; without it the output has one image per source."""
    if not src.is_cuda:
        raise RuntimeError("turboprune_b200 augmentation kernels need CUDA tensors (H100 / sm_90a); there is no CPU path")
    lib = _cabi.load()
    src = src.contiguous().float()
    c = src.shape[1]
    ix = idx.to(torch.int64).contiguous() if idx is not None else None
    n = len(ix) if ix is not None else src.shape[0]
    h, w = out_hw
    out = torch.empty(n, c, h, w, dtype=torch.float32, device=src.device)
    f8 = flip.to(torch.uint8).contiguous() if flip is not None else None
    sh = shifts.to(torch.int64).contiguous() if shifts is not None else None
    cy = corner_y.to(torch.int64).contiguous() if corner_y is not None else None
    cx = corner_x.to(torch.int64).contiguous() if corner_x is not None else None
    with torch.cuda.device(src.device):
        rc = lib.tp_cifar_augment(_ptr(src), _ptr(out), _ptr(ix), _ptr(sh), _ptr(f8), _ptr(cy), _ptr(cx), int(cut_size), n, c, h, w, int(r),
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


# ---- the airbench CIFAR loader (reference utils/dataset.py:101-256) ---------------------------------------------------
CIFAR10_MEAN = torch.tensor((0.4914, 0.4822, 0.4465))
CIFAR10_STD = torch.tensor((0.2470, 0.2435, 0.2616))
CIFAR100_MEAN = torch.tensor((0.5071, 0.4867, 0.4408))
CIFAR100_STD = torch.tensor((0.2675, 0.2565, 0.2761))


def cifar_variant(dataset):
    """``"CIFAR10"`` / ``"CIFAR100"`` in any case -> (canonical name, sub-directory, mean, std)."""
    name = str(dataset).upper()
    if name == "CIFAR10":
        return name, "cifar10", CIFAR10_MEAN, CIFAR10_STD
    if name == "CIFAR100":
        return name, "cifar100", CIFAR100_MEAN, CIFAR100_STD
    raise ValueError(f"CifarLoader: unknown data set {dataset!r} (CIFAR10 or CIFAR100)")


def _load_cifar_cache(path, dataset, train, device):
    """The reference's cache ``{path}/{cifar10|cifar100}/{CIFAR10|CIFAR100}_{train|test}.pt`` (uint8 images [N,32,32,3],
    labels, classes), built with torchvision on first use under a file lock, written to a temporary file and renamed."""
    from filelock import FileLock
    name, sub, _, _ = cifar_variant(dataset)
    root = os.path.join(path, sub)
    os.makedirs(root, exist_ok=True)
    data_path = os.path.join(root, f"{name}_{'train' if train else 'test'}.pt")
    with FileLock(data_path + ".lock"):
        if not os.path.exists(data_path):
            import torchvision
            cls = torchvision.datasets.CIFAR10 if name == "CIFAR10" else torchvision.datasets.CIFAR100
            dset = cls(root, download=True, train=train)
            tmp = data_path + ".tmp"
            torch.save({"images": torch.tensor(dset.data), "labels": torch.tensor(dset.targets), "classes": dset.classes}, tmp)
            os.rename(tmp, data_path)
        return torch.load(data_path, map_location=device)


class CifarLoader:
    """Drop-in for the reference's ``CifarLoader`` (utils/dataset.py:101-226): same constructor, ``len()``, random draws
    (torch's generator on the data's device, in the reference's order) and batches, bit for bit.

    ``dataset`` is ``"CIFAR10"`` or ``"CIFAR100"``, matched case-insensitively; any other name raises.  (The reference
    takes every name other than exactly ``"CIFAR10"`` for CIFAR-100.)  ``device``: where the data set lives, by default
    the current CUDA device.

    The first ``iter()`` normalises the images with the reference's own ops (``/255``, torchvision's ``normalize``),
    applies the random pre-flip when ``aug["flip"]`` is set and reflect-pads by ``aug["translate"]``; only the last of
    these tensors is kept (train: 50,000 x 3 x 36 x 36 fp32).  Every epoch then draws the crop shifts
    (``randint(-r, r+1, (N, 2))``), the flip mask (without ``altflip``) and the cutout corners for the whole data set,
    then the permutation, exactly as the reference does; with ``altflip`` odd epochs are mirrored.  Each batch is one
    ``tp_cifar_augment`` launch over a slice of the permutation plus ``labels[idx]``: no host sync, no whole-data-set
    copy per epoch.  Unshuffled loaders without augmentation (the test loader) yield views of the normalised images.
    """

    def __init__(self, path, train=True, batch_size=500, aug=None, drop_last=None, shuffle=None, altflip=False,
                 dataset="CIFAR10", device=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise RuntimeError("turboprune_b200 CifarLoader keeps the data set on a CUDA device (H100 / sm_90a)")
        self.dataset, _, self.mean, self.std = cifar_variant(dataset)
        data = _load_cifar_cache(path, self.dataset, train, self.device)
        self.epoch = 0
        self.images, self.labels, self.classes = data["images"], data["labels"], data["classes"]
        self.num_images, self.crop_size = len(self.images), int(self.images.shape[-2])
        self.aug = aug or {}
        for k in self.aug.keys():
            assert k in ["flip", "translate", "cutout"], "Unrecognized key: %s" % k
        self.batch_size = batch_size
        self.drop_last = train if drop_last is None else drop_last
        self.shuffle = train if shuffle is None else shuffle
        self.altflip = altflip
        self.source = None              # what the batches read: padded (translate), pre-flipped or normalised images
        self._all = None                # uint8 ones [N]: the altflip mirror of odd epochs

    def __len__(self):
        n = self.num_images
        return n // self.batch_size if self.drop_last else ceil(n / self.batch_size)

    def _prepare(self):
        """Epoch 0 (reference :193-201): normalise, random pre-flip, reflect-pad; keep only what the batches read."""
        from torchvision.transforms import functional as TF
        images = TF.normalize((self.images / 255).permute(0, 3, 1, 2), self.mean, self.std)
        self.images = None
        if self.aug.get("flip", False):
            images = batch_flip_lr(images)
        pad = self.aug.get("translate", 0)
        if pad > 0:
            images = torch.nn.functional.pad(images, (pad,) * 4, "reflect")
        self.source = images.contiguous()
        if self.aug.get("flip", False) and self.altflip:
            self._all = torch.ones(self.num_images, dtype=torch.uint8, device=self.device)

    def __iter__(self):
        if self.epoch == 0:
            self._prepare()
        n, dev, crop = self.num_images, self.device, self.crop_size
        r = self.aug.get("translate", 0)
        shifts = torch.randint(-r, r + 1, size=(n, 2), device=dev) if r > 0 else None
        flip = None
        if self.aug.get("flip", False):
            if self.altflip:
                flip = self._all if self.epoch % 2 == 1 else None
            else:
                flip = (torch.rand(n, device=dev) < 0.5).to(torch.uint8)
        cut = self.aug.get("cutout", 0)
        cy = cx = None
        if cut > 0:
            cy = torch.randint(0, crop - cut + 1, size=(n,), device=dev)
            cx = torch.randint(0, crop - cut + 1, size=(n,), device=dev)
        self.epoch += 1
        plain = shifts is None and flip is None and cy is None
        if plain and not self.shuffle:
            for i in range(len(self)):
                s = slice(i * self.batch_size, (i + 1) * self.batch_size)
                yield self.source[s], self.labels[s]
            return
        indices = (torch.randperm if self.shuffle else torch.arange)(n, device=dev)
        for i in range(len(self)):
            idx = indices[i * self.batch_size:(i + 1) * self.batch_size]
            yield (_augment(self.source, (crop, crop), r, shifts=shifts, flip=flip, corner_y=cy, corner_x=cx, cut_size=cut, idx=idx),
                   self.labels.index_select(0, idx))


class AirbenchLoaders:
    """train_loader / test_loader pair of the reference (utils/dataset.py:229-256): ``dataset_params.data_root_dir``,
    ``total_batch_size`` and ``dataset_name``; translate 2 + alternating flip for training, unshuffled test set."""

    def __init__(self, cfg, device=None):
        print("Using the Airbench CIFAR loader (https://github.com/KellerJordan/cifar10-airbench), device-resident")
        dp = cfg.dataset_params
        self.train_loader = CifarLoader(path=dp.data_root_dir, batch_size=dp.total_batch_size, train=True,
                                        aug={"flip": True, "translate": 2}, altflip=True, dataset=dp.dataset_name, device=device)
        self.test_loader = CifarLoader(path=dp.data_root_dir, batch_size=dp.total_batch_size, train=False,
                                       dataset=dp.dataset_name, device=device)


# ---- ImageNet from an ImageFolder tree (reference utils/dataset.py:347-430 reads FFCV betons written from it) ----------
IMAGENET_MEAN = tuple(v * 255 for v in (0.485, 0.456, 0.406))     # reference :28-29, already scaled to 0..255
IMAGENET_STD = tuple(v * 255 for v in (0.229, 0.224, 0.225))
DEFAULT_CROP_RATIO = 224 / 256


def resized_crop(images, boxes, flips, size=224, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """One ``tp_resized_crop`` launch on the current stream.  ``images``: list of uint8 [3, H, W] contiguous CUDA
    tensors; ``boxes``: int [B, 4] (top, left, h, w) per image, inside it; ``flips``: bool [B].  Returns fp32
    [B, 3, size, size] with channels_last strides: each box resized like
    ``F.interpolate(box, (size, size), mode="bilinear", antialias=True)``, mirrored where flipped, then
    ``(v - mean) / std``."""
    if not images or not images[0].is_cuda:
        raise RuntimeError("turboprune_b200 resized_crop needs CUDA images (H100 / sm_90a); there is no CPU path")
    dev, n = images[0].device, len(images)
    boxes, flips = torch.as_tensor(boxes).tolist(), torch.as_tensor(flips).tolist()
    if len(boxes) != n or len(flips) != n:
        raise ValueError("resized_crop: one box and one flip per image")
    table = torch.empty(n * sizeof(_cabi.CropEntry), dtype=torch.uint8, pin_memory=True)
    entries = (_cabi.CropEntry * n).from_address(table.data_ptr())
    for i, (img, (t, l, h, w), f) in enumerate(zip(images, boxes, flips)):
        if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[0] != 3 or not img.is_contiguous() or img.device != dev:
            raise ValueError(f"resized_crop: image {i} must be uint8 [3, H, W] contiguous on {dev}")
        H, W = img.shape[1:]
        if not (h >= 1 and w >= 1 and 0 <= t and t + h <= H and 0 <= l and l + w <= W and w <= 1023 * size):
            raise ValueError(f"resized_crop: box {(t, l, h, w)} of image {i} does not fit its {H} x {W} image")
        entries[i] = _cabi.CropEntry(img.data_ptr(), H, W, t, l, h, w, int(bool(f)), 0)
    dtab = table.to(dev, non_blocking=True)
    out = torch.empty(n, size, size, 3, dtype=torch.float32, device=dev)
    lib = _cabi.load()
    with torch.cuda.device(dev):
        rc = lib.tp_resized_crop(_ptr(dtab), n, int(size), (c_float * 3)(*mean), (c_float * 3)(*std), _ptr(out),
                                 _cabi.stream_ptr(dev))
    _cabi.check(rc, "tp_resized_crop")
    ops._count()
    return out.permute(0, 3, 1, 2)


def random_resized_crop_boxes(hw, u_area, u_ratio, u_off, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3)):
    """torchvision's / FFCV's ``RandomResizedCrop`` box draw, vectorised over images, from pre-drawn uniforms in [0, 1):
    ``hw`` int [B, 2] image extents, ``u_area`` / ``u_ratio`` float64 [B, 10] (one pair per attempt), ``u_off`` float64
    [B, 2].  Attempt k: area = H*W*U(scale), aspect = exp(U(log ratio)), w = round(sqrt(area*aspect)),
    h = round(sqrt(area/aspect)); the first attempt with 0 < w <= W and 0 < h <= H wins and is placed at a uniform
    offset; without one, the ratio-clamped centre crop.  Returns int64 [B, 4] (top, left, h, w)."""
    hw = torch.as_tensor(hw, dtype=torch.float64)
    H, W = hw[:, :1], hw[:, 1:]
    target = H * W * (scale[0] + (scale[1] - scale[0]) * u_area)
    lr0, lr1 = math.log(ratio[0]), math.log(ratio[1])
    ar = torch.exp(lr0 + (lr1 - lr0) * u_ratio)
    w = torch.round(torch.sqrt(target * ar))
    h = torch.round(torch.sqrt(target / ar))
    ok = (w > 0) & (w <= W) & (h > 0) & (h <= H)
    k = ok.to(torch.int8).argmax(1, keepdim=True)                  # first accepted attempt (0 when none is)
    hit = ok.any(1)
    H, W = H.squeeze(1), W.squeeze(1)
    w, h = w.gather(1, k).squeeze(1), h.gather(1, k).squeeze(1)
    top = torch.minimum(torch.floor(u_off[:, 0] * (H - h + 1)), H - h)
    left = torch.minimum(torch.floor(u_off[:, 1] * (W - w + 1)), W - w)
    in_ratio = W / H
    tall, wide = in_ratio < min(ratio), in_ratio > max(ratio)
    fw = torch.where(wide, torch.round(H * max(ratio)), W)
    fh = torch.where(tall, torch.round(W / min(ratio)), H)
    box = torch.stack([torch.where(hit, top, torch.div(H - fh, 2, rounding_mode="floor")),
                       torch.where(hit, left, torch.div(W - fw, 2, rounding_mode="floor")),
                       torch.where(hit, h, fh), torch.where(hit, w, fw)], 1)
    return box.to(torch.int64)


def center_crop_box(H, W, ratio=DEFAULT_CROP_RATIO):
    """FFCV's ``CenterCropRGBImageDecoder`` box: a c x c square, c = int(ratio * min(H, W)) (at least 1), centred."""
    c = max(1, int(ratio * min(H, W)))
    return (H - c) // 2, (W - c) // 2, c, c


@lru_cache(maxsize=4)
def scan_image_folder(root):
    """``torchvision.datasets.ImageFolder``'s index of ``root``: sorted class directories give class i, files in its
    order.  Returns (classes, relative paths as a bytes array, labels int64 array); cached per root."""
    from torchvision.datasets.folder import IMG_EXTENSIONS, find_classes, make_dataset
    classes, to_idx = find_classes(root)
    samples = make_dataset(root, to_idx, IMG_EXTENSIONS)
    if not samples:
        raise FileNotFoundError(f"ImageFolderLoader: no images under {root}")
    rel = np.array([os.fsencode(os.path.relpath(p, root)) for p, _ in samples])
    return tuple(classes), rel, np.array([c for _, c in samples], dtype=np.int64)


def _jpeg_components(data):
    """Number of colour components from the first SOF marker of JPEG bytes (uint8 tensor); None if it is not a JPEG
    nvjpeg can be handed (no SOI, or no frame header found)."""
    b = data[:65536].numpy().tobytes()
    if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
        return None
    i = 2
    while i + 9 < len(b):
        if b[i] != 0xFF:
            return None
        m = b[i + 1]
        if m == 0xFF:
            i += 1
            continue
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            return b[i + 9]
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7:
            i += 2
            continue
        i += 2 + (b[i + 2] << 8 | b[i + 3])
    return None


_warned_files = set()


def decode_images(datas, device, names=None):
    """Raw file bytes (uint8 CPU tensors) -> list of uint8 [3, H, W] RGB tensors on ``device``, plus a bool per image
    telling whether it went through the CPU.  JPEGs with 1 or 3 components are decoded by nvjpeg in one batched call;
    what nvjpeg cannot take (CMYK, PNG or other data named .JPEG, a file the batched call rejects) is decoded by
    torchvision's CPU ``decode_image`` and uploaded.  A file no decoder accepts becomes a mean-coloured 8 x 8 image,
    with a warning, so that one bad file never fails a batch."""
    from torchvision.io import ImageReadMode, decode_image, decode_jpeg
    out, on_cpu = [None] * len(datas), [False] * len(datas)
    gpu = [i for i, d in enumerate(datas) if _jpeg_components(d) in (1, 3)]
    if gpu:
        try:
            dec = decode_jpeg([datas[i] for i in gpu], mode=ImageReadMode.RGB, device=device)
        except RuntimeError:
            dec = []
            for i in gpu:
                try:
                    dec.append(decode_jpeg(datas[i], mode=ImageReadMode.RGB, device=device))
                except RuntimeError:
                    dec.append(None)
        for i, x in zip(gpu, dec):
            if x is not None and x.dim() == 3 and x.shape[0] == 3:
                out[i] = x.contiguous()
    for i, x in enumerate(out):
        if x is not None:
            continue
        on_cpu[i] = True
        try:
            x = decode_image(datas[i], mode=ImageReadMode.RGB)
        except RuntimeError:
            name = names[i] if names is not None else i
            if name not in _warned_files:
                _warned_files.add(name)
                print(f"ImageFolderLoader: cannot decode {name}; using a blank image", file=sys.stderr)
            x = torch.tensor([round(m) for m in IMAGENET_MEAN], dtype=torch.uint8).view(3, 1, 1).expand(3, 8, 8)
        out[i] = x.contiguous().pin_memory().to(device, non_blocking=True)
    return out, on_cpu


def _read_file(path):
    with open(path, "rb") as f:
        return torch.frombuffer(bytearray(f.read()), dtype=torch.uint8)


class ImageFolderLoader:
    """One split of an ImageFolder tree as an iterable of ``(images fp32 [B, 3, S, S] channels_last, labels int64 [B])``
    on ``device``, B = ``total_batch_size // world_size``: the batch contract of the reference's FFCV loaders
    (utils/dataset.py:380-430).

    ``train=True``: every epoch one permutation seeded by ``(seed, epoch)``, the same on every rank; global batch g is
    ``perm[g*T:(g+1)*T]`` (T = total_batch_size) and rank r takes its r-th slice of B; ``drop_last``, so
    ``len() = N // T``.  Each image gets a RandomResizedCrop(S, scale=(0.08, 1), ratio=(3/4, 4/3)) box and a flip with
    p = 0.5, drawn on the host from the same generator for the whole global batch (a sample's draws do not depend on the
    world size).  ``train=False``: images ``i % world_size == rank`` in order, FFCV's centre crop (ratio 224/256), no
    flip, the last partial batch kept, so the ranks' counts add up to the whole split.

    Batch i+1 is read (``num_workers`` threads), decoded and cropped on a side stream by a producer thread while the
    caller uses batch i; the caller's stream waits on an event before it sees a batch, and ``record_stream`` keeps each
    batch alive until the caller's work on it is done.  ``last_indices`` / ``last_boxes`` / ``last_flips`` describe the
    batch last handed out (sample indices into ``labels``, (top, left, h, w) per image, mirrored or not)."""

    def __init__(self, root, train, total_batch_size, device=None, num_workers=8, seed=0, world_size=1, rank=0,
                 size=224):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise RuntimeError("turboprune_b200 ImageFolderLoader decodes and crops on a CUDA device (H100 / sm_90a)")
        if not 0 <= rank < world_size or total_batch_size < world_size:
            raise ValueError(f"ImageFolderLoader: rank {rank} of {world_size} with total batch {total_batch_size}")
        self.root, self.train, self.size = os.fspath(root), bool(train), int(size)
        self.classes, self.paths, self.labels = scan_image_folder(self.root)
        self.total_batch_size, self.batch_size = int(total_batch_size), int(total_batch_size) // world_size
        self.world_size, self.rank, self.seed = world_size, rank, int(seed)
        self.num_workers = max(1, int(num_workers))
        self.epoch = 0
        self.last_indices = self.last_boxes = self.last_flips = None

    def __len__(self):
        n = len(self.labels)
        if self.train:
            return n // self.total_batch_size
        return ceil(len(range(self.rank, n, self.world_size)) / self.batch_size)

    def _plan(self, epoch):
        """Per batch: (sample indices [B], uniforms for this rank's slice or None)."""
        n, B = len(self.labels), self.batch_size
        if not self.train:
            idx = torch.arange(self.rank, n, self.world_size)
            for i in range(len(self)):
                yield idx[i * B:(i + 1) * B], None
            return
        g = torch.Generator().manual_seed(((self.seed << 32) + epoch) & (2 ** 64 - 1))
        perm, T = torch.randperm(n, generator=g), self.total_batch_size
        s = slice(self.rank * B, (self.rank + 1) * B)
        for i in range(len(self)):
            u = [torch.rand(T, k, generator=g, dtype=torch.float64)[s] for k in (10, 10, 2, 1)]
            yield perm[i * T:(i + 1) * T][s], u

    def _batch(self, idx, u, datas):
        """Decode, draw the boxes, one crop launch, labels: all on the current (side) stream."""
        names = [self.paths[i] for i in idx.tolist()]
        images, _ = decode_images(datas, self.device, names)
        cur = torch.cuda.current_stream(self.device)
        for x in images:
            x.record_stream(cur)          # nvjpeg may allocate on its own stream; the crop reads on this one
        hw = torch.tensor([x.shape[1:] for x in images], dtype=torch.int64)
        if u is None:
            boxes = torch.tensor([center_crop_box(h, w) for h, w in hw.tolist()], dtype=torch.int64)
            flips = torch.zeros(len(images), dtype=torch.bool)
        else:
            boxes = random_resized_crop_boxes(hw, u[0], u[1], u[2])
            flips = u[3][:, 0] < 0.5
        x = resized_crop(images, boxes, flips, self.size)
        y = torch.from_numpy(self.labels[idx.numpy()]).pin_memory().to(self.device, non_blocking=True)
        return x, y, (idx, boxes, flips)

    def _produce(self, epoch, q, stop):
        try:
            side = torch.cuda.Stream(self.device)
            with ThreadPoolExecutor(self.num_workers) as pool, torch.cuda.device(self.device), torch.cuda.stream(side):
                read = lambda idx: [pool.submit(_read_file, os.path.join(self.root, os.fsdecode(self.paths[i])))
                                    for i in idx.tolist()]
                plan = self._plan(epoch)
                nxt = next(plan, None)
                pending = read(nxt[0]) if nxt is not None else None
                while nxt is not None and not stop.is_set():
                    idx, u = nxt
                    nxt = next(plan, None)
                    datas = [f.result() for f in pending]
                    pending = read(nxt[0]) if nxt is not None else None      # the next batch's files meanwhile
                    x, y, meta = self._batch(idx, u, datas)
                    ev = torch.cuda.Event()
                    ev.record(side)
                    item = (x, y, ev, meta)
                    while not stop.is_set():
                        try:
                            q.put(item, timeout=0.1)
                            break
                        except queue.Full:
                            pass
                if pending is not None:
                    for f in pending:
                        f.cancel()
        except BaseException as e:               # handed to the consumer, which raises it
            q.put(e)
            return
        q.put(None)

    def __iter__(self):
        epoch = self.epoch
        self.epoch += 1
        q, stop = queue.Queue(maxsize=1), threading.Event()
        worker = threading.Thread(target=self._produce, args=(epoch, q, stop), daemon=True,
                                  name=f"ImageFolderLoader-{'train' if self.train else 'val'}")
        worker.start()
        try:
            while True:
                item = q.get()
                if item is None:
                    return
                if isinstance(item, BaseException):
                    raise item
                x, y, ev, meta = item
                cur = torch.cuda.current_stream(self.device)
                cur.wait_event(ev)
                x.record_stream(cur); y.record_stream(cur)
                self.last_indices, self.last_boxes, self.last_flips = meta
                yield x, y
        finally:
            stop.set()
            while worker.is_alive():
                try:
                    q.get(timeout=0.1)
                except queue.Empty:
                    pass
            worker.join()


class ImageFolderImagenet:
    """train_loader / test_loader pair over ``{dataset_params.data_root_dir}/{train,val}``, the shape of the
    reference's ``FFCVImagenet`` (utils/dataset.py:347-430): batch ``total_batch_size // world_size``, ``num_workers``
    reading threads, seeded by ``experiment_params.seed``."""

    def __init__(self, cfg, device, world_size=1, rank=0):
        dp = cfg.dataset_params
        kw = dict(total_batch_size=dp.total_batch_size, device=device, num_workers=getattr(dp, "num_workers", 8),
                  seed=cfg.experiment_params.seed, world_size=world_size, rank=rank)
        self.train_loader = ImageFolderLoader(os.path.join(dp.data_root_dir, "train"), train=True, **kw)
        self.test_loader = ImageFolderLoader(os.path.join(dp.data_root_dir, "val"), train=False, **kw)
