"""Data loaders of the reference's ``utils/dataset.py``, device-resident.

* ``CifarLoader`` / ``AirbenchLoaders`` (reference :101-256): the airbench CIFAR-10/100 loader, same names, constructor
  arguments, random draws and batches.  The data set lives on the GPU; each batch is ONE ``tp_cifar_augment`` launch
  that gathers the permuted source images and applies the epoch's translate / flip / cutout on the way, so an epoch
  never writes an augmented copy of the whole data set and never waits on the host.
* ``SyntheticLoaders``: the on-device generator standing in for loaders whose data is not at hand (ImageNet's FFCV /
  WebDataset loaders, :347-546, are out of scope; benchmarks and synthetic configs use it for every data set).

Same batch contract throughout: an iterable of ``(images fp32 [B,3,H,W], labels int64 [B])`` with ``len()``;
ImageNet-shaped synthetic batches come channels_last like FFCV's ToTorchImage.  Synthetic loaders are seeded per rank;
either a fixed number of distinct batches is generated once and cycled (an epoch costs no host work), or
(``dataset_params.synthetic_fresh``) every step draws a new batch on the device.  ``DevicePrefetcher`` is the
host->device leg for loaders that produce pinned host batches.
"""
import os
from ctypes import c_void_p
from math import ceil

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
