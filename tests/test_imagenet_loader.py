"""The ImageFolder ImageNet loader (turboprune_b200.utils.dataset.ImageFolderLoader) and its crop kernel tp_resized_crop.

CPU: the vectorised RandomResizedCrop draw equals the scalar restatement in tests/imagenet_loader_oracle.py on the same
uniforms (every fallback branch included), class indices equal torchvision's ImageFolder, the JPEG header probe routes
files correctly.  GPU: the kernel against F.interpolate(antialias=True) in float64, loader batches against that oracle on
the loader's own boxes, rank coverage, odd files, determinism, and a run of run_experiment.main that learns.
"""
import csv
import os

import numpy as np
import pytest
import torch

import imagenet_loader_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def _save(path, arr, mode="RGB", fmt="JPEG", **kw):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    img = Image.fromarray(arr)
    if mode != img.mode:
        img = img.convert(mode)
    img.save(path, fmt, **kw)


def _tree(root, sizes, seed=0):
    """{root}/<wnid>/img_k.JPEG: sizes[c] lists the (H, W) of class c's images; random-texture RGB JPEGs, quality 90."""
    rng = np.random.default_rng(seed)
    for c, hws in enumerate(sizes):
        for k, (h, w) in enumerate(hws):
            arr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            _save(os.path.join(root, f"n{c:08d}", f"img_{k}.JPEG"), arr, quality=90)


# ---------------------------------------------------------------- CPU --------------------------------------------------
def test_box_draw_equals_scalar_restatement():
    from turboprune_b200.utils import dataset as ds
    g = torch.Generator().manual_seed(5)
    hw = [(375, 500), (500, 375), (3000, 4000), (7, 300), (300, 7), (1, 1), (1, 500), (224, 224), (64, 48)]
    hw = torch.tensor(hw * 40 + [(int(a), int(b)) for a, b in torch.randint(1, 2000, (200, 2), generator=g)])
    n = len(hw)
    ua, ur = torch.rand(n, 10, generator=g, dtype=torch.float64), torch.rand(n, 10, generator=g, dtype=torch.float64)
    uo = torch.rand(n, 2, generator=g, dtype=torch.float64)
    # forced failures of all ten attempts: largest area and extreme aspect on a tall, a wide and an in-range image
    forced = torch.tensor([(100, 10), (10, 100), (50, 50), (2000, 100), (100, 2000), (400, 400)])
    hw = torch.cat([hw, forced])
    fa = torch.full((len(forced), 10), 0.999999, dtype=torch.float64)
    fr = torch.tensor([[1.0 - 1e-9] * 10, [0.0] * 10, [1.0 - 1e-9] * 10] * 2, dtype=torch.float64)
    ua, ur = torch.cat([ua, fa]), torch.cat([ur, fr])
    uo = torch.cat([uo, torch.rand(len(forced), 2, generator=g, dtype=torch.float64)])
    got = ds.random_resized_crop_boxes(hw, ua, ur, uo)
    branches = set()
    for i, (h, w) in enumerate(hw.tolist()):
        want = O.rrc_box(h, w, ua[i], ur[i], uo[i])
        assert tuple(got[i].tolist()) == want, (i, h, w)
        t, l, bh, bw = want
        assert 0 <= t and t + bh <= h and 0 <= l and l + bw <= w and bh >= 1 and bw >= 1, (i, h, w, want)
        if i >= n:
            branches.add("tall" if w / h < 3 / 4 else "wide" if w / h > 4 / 3 else "in-range")
            assert (t, l) == ((h - bh) // 2, (w - bw) // 2), "a forced failure must take the centre-crop fallback"
    assert branches == {"tall", "wide", "in-range"}


def test_center_box_is_ffcvs():
    from turboprune_b200.utils import dataset as ds
    for h, w in [(375, 500), (500, 375), (224, 224), (256, 256), (3000, 4000), (7, 300)]:
        assert ds.center_crop_box(h, w) == O.center_box(h, w)


def test_class_indices_match_torchvision_image_folder(tmp_path):
    from torchvision.datasets import ImageFolder
    from turboprune_b200.utils import dataset as ds
    rng = np.random.default_rng(1)
    root = tmp_path / "train"
    for wnid in ["n09999999", "n01440764", "n02102040", "n01443537"]:
        for k in range(int(rng.integers(1, 5))):
            _save(str(root / wnid / f"{wnid}_{k}.JPEG"), rng.integers(0, 256, (9, 11, 3), dtype=np.uint8))
    _save(str(root / "n01440764" / "a.png"), rng.integers(0, 256, (9, 11, 3), dtype=np.uint8), fmt="PNG")
    (root / "n01440764" / "notes.txt").write_text("not an image")
    ref = ImageFolder(str(root))
    classes, paths, labels = ds.scan_image_folder(str(root))
    assert list(classes) == ref.classes == sorted(ref.classes)
    assert labels.tolist() == ref.targets
    assert [os.path.join(str(root), os.fsdecode(p)) for p in paths] == [p for p, _ in ref.samples]


def _odd_files(root):
    """Grayscale, CMYK, progressive and PNG-named-.JPEG files, plus a plain RGB JPEG."""
    from PIL import Image
    rng = np.random.default_rng(2)          # a smooth field: decoders differ most in chroma upsampling of noise
    arr = np.asarray(Image.fromarray(rng.integers(0, 256, (4, 5, 3), dtype=np.uint8)).resize((53, 37), Image.BILINEAR))
    files = {"rgb": dict(), "gray": dict(mode="L"), "cmyk": dict(mode="CMYK"), "progressive": dict(progressive=True),
             "png": dict(fmt="PNG")}
    out = {}
    for name, kw in files.items():
        p = os.path.join(root, "n00000000", f"{name}.JPEG")
        _save(p, arr, quality=90, **kw) if kw.get("fmt") != "PNG" else _save(p, arr, fmt="PNG")
        out[name] = p
    return out


def test_jpeg_header_probe(tmp_path):
    from turboprune_b200.utils import dataset as ds
    files = _odd_files(str(tmp_path))
    comps = {k: ds._jpeg_components(ds._read_file(p)) for k, p in files.items()}
    assert comps == {"rgb": 3, "gray": 1, "cmyk": 4, "progressive": 3, "png": None}


# ---------------------------------------------------------------- GPU --------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked ImageNet loader tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


KERNEL_ERR_BAR = 1e-5


@pytest.mark.gpu
def test_resized_crop_kernel_against_float64(dev):
    """Downscales up to 17.9x, upscales, full images, 1-pixel-wide and 1-pixel-high boxes, flips."""
    from turboprune_b200.utils import dataset as ds
    g = torch.Generator().manual_seed(11)
    cases = [((3000, 4000), (0, 0, 3000, 4000), False), ((3000, 4000), (0, 0, 3000, 4000), True),
             ((3000, 4000), (17, 3, 2983, 3990), True), ((7, 300), (0, 0, 7, 300), False),
             ((7, 300), (2, 100, 1, 1), True), ((375, 500), (10, 20, 300, 1), False), ((375, 500), (10, 20, 1, 300), True),
             ((375, 500), (100, 200, 20, 30), True), ((375, 500), (0, 0, 375, 500), False), ((224, 224), (0, 0, 224, 224), True),
             ((500, 375), (37, 11, 449, 337), False), ((1200, 900), (5, 7, 1190, 223), True), ((230, 2500), (0, 0, 230, 2500), False)]
    images = [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8).to(dev) for (h, w), _, _ in cases]
    boxes = torch.tensor([b for _, b, _ in cases])
    flips = torch.tensor([f for _, _, f in cases])
    out = ds.resized_crop(images, boxes, flips)
    assert out.shape == (len(cases), 3, 224, 224) and out.is_contiguous(memory_format=torch.channels_last)
    errs = []
    for i, (img, b, f) in enumerate(zip(images, boxes.tolist(), flips.tolist())):
        want = O.resized_crop(img, b, f)
        errs.append((out[i].cpu().double() - want).abs().max().item())
    print(f"tp_resized_crop max |error| per case vs float64: {['%.2e' % e for e in errs]}")
    assert max(errs) <= KERNEL_ERR_BAR, errs


@pytest.mark.gpu
def test_resized_crop_identity_is_exact(dev):
    from turboprune_b200.utils import dataset as ds
    img = torch.randint(0, 256, (3, 224, 224), generator=torch.Generator().manual_seed(3), dtype=torch.uint8).to(dev)
    out = ds.resized_crop([img, img], [(0, 0, 224, 224)] * 2, [False, True])
    mean = torch.tensor(ds.IMAGENET_MEAN, dtype=torch.float32, device=dev).view(3, 1, 1)
    std = torch.tensor(ds.IMAGENET_STD, dtype=torch.float32, device=dev).view(3, 1, 1)
    want = (img.float() - mean) / std
    assert torch.equal(out[0], want) and torch.equal(out[1], want.flip(-1))


@pytest.mark.gpu
def test_resized_crop_rejects_boxes_outside_the_image(dev):
    from turboprune_b200.utils import dataset as ds
    img = torch.zeros(3, 10, 10, dtype=torch.uint8, device=dev)
    for box in [(0, 0, 11, 10), (-1, 0, 5, 5), (0, 6, 5, 5), (0, 0, 0, 5)]:
        with pytest.raises(ValueError):
            ds.resized_crop([img], [box], [False])


@pytest.fixture(scope="module")
def small_tree(tmp_path_factory):
    """3 classes, 7 train and 5 val images each, sizes from 40 x 300 to 420 x 380."""
    root = tmp_path_factory.mktemp("imagenet_small")
    rng = np.random.default_rng(4)
    for split, per in (("train", 7), ("val", 5)):
        sizes = [[(int(rng.integers(40, 421)), int(rng.integers(40, 421))) for _ in range(per)] for _ in range(3)]
        sizes[0][0] = (40, 300)
        _tree(str(root / split), sizes, seed=len(split))
    return root


def _decode_like_loader(loader, idx, dev):
    from torchvision.io import ImageReadMode, decode_jpeg
    from turboprune_b200.utils import dataset as ds
    datas = [ds._read_file(os.path.join(loader.root, os.fsdecode(loader.paths[i]))) for i in idx]
    return decode_jpeg(datas, mode=ImageReadMode.RGB, device=dev)


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["train", "val"])
def test_loader_batches_equal_oracle(dev, small_tree, split):
    from turboprune_b200.utils import dataset as ds
    loader = ds.ImageFolderLoader(small_tree / split, train=split == "train", total_batch_size=4, device=dev, num_workers=3,
                                  seed=9)
    n = len(loader.labels)
    assert len(loader) == (n // 4 if split == "train" else -(-n // 4)) and (split == "train" or n % 4 == 3)
    worst, count = 0.0, 0
    for e in range(2):
        for x, y in loader:
            idx = loader.last_indices.tolist()
            assert x.shape[1:] == (3, 224, 224) and x.is_contiguous(memory_format=torch.channels_last)
            assert y.tolist() == loader.labels[idx].tolist()
            images = _decode_like_loader(loader, idx, dev)
            for j, img in enumerate(images):
                box, flip = loader.last_boxes[j].tolist(), bool(loader.last_flips[j])
                if split == "val":
                    assert tuple(box) == O.center_box(*img.shape[1:]) and not flip
                worst = max(worst, (x[j].cpu().double() - O.resized_crop(img, box, flip)).abs().max().item())
            count += len(idx)
    print(f"{split}: {count} images, max |error| vs float64 oracle {worst:.2e}")
    assert count == 2 * (len(loader) * 4 if split == "train" else n)
    assert worst <= KERNEL_ERR_BAR


@pytest.mark.gpu
def test_two_ranks_cover_the_splits(dev, small_tree):
    from turboprune_b200.utils import dataset as ds
    kw = dict(total_batch_size=4, device=dev, num_workers=2, seed=1, world_size=2)
    tr = [ds.ImageFolderLoader(small_tree / "train", train=True, rank=r, **kw) for r in (0, 1)]
    n = len(tr[0].labels)
    for epoch in range(2):
        seen = []
        for loader in tr:
            mine = []
            for x, y in loader:
                assert x.shape[0] == 2 and y.tolist() == loader.labels[loader.last_indices.numpy()].tolist()
                mine += loader.last_indices.tolist()
            assert len(mine) == len(loader) * 2 and len(loader) == n // 4
            seen.append(set(mine))
            assert len(set(mine)) == len(mine)
        assert not seen[0] & seen[1] and len(seen[0] | seen[1]) == (n // 4) * 4
    va = [ds.ImageFolderLoader(small_tree / "val", train=False, rank=r, **kw) for r in (0, 1)]
    got = []
    for loader in va:
        for x, y in loader:
            got += loader.last_indices.tolist()
            assert y.tolist() == loader.labels[loader.last_indices.numpy()].tolist()
    assert sorted(got) == list(range(len(va[0].labels)))


@pytest.mark.gpu
def test_odd_files_decode_to_rgb(dev, tmp_path):
    from torchvision.io import ImageReadMode, decode_image
    from turboprune_b200.utils import dataset as ds
    files = _odd_files(str(tmp_path))
    names = list(files)
    datas = [ds._read_file(files[k]) for k in names]
    imgs, on_cpu = ds.decode_images(datas, dev, names)
    for k, img, cpu in zip(names, imgs, on_cpu):
        want = decode_image(datas[names.index(k)], mode=ImageReadMode.RGB)
        assert img.is_cuda and img.dtype == torch.uint8 and img.shape == (3, 37, 53), k
        diff = (img.cpu().int() - want.int()).abs()
        print(f"{k}: {'CPU fallback' if cpu else 'nvjpeg'}, max |diff| vs CPU decode_image {diff.max().item()}")
        if cpu:
            assert torch.equal(img.cpu(), want), k
        else:
            # nvjpeg and libjpeg-turbo upsample chroma differently (mean 4.2 measured on this file); a channel-order
            # or colour-space mistake is an order of magnitude larger
            assert diff.float().mean() < 10, k
    assert on_cpu[names.index("png")] and on_cpu[names.index("cmyk")] and not on_cpu[names.index("rgb")]
    # a batch holding every odd file (and one that no decoder takes) goes through the loader's batched path whole
    bad = torch.frombuffer(bytearray(b"\xff\xd8\xff\xc0 truncated"), dtype=torch.uint8)
    imgs, on_cpu = ds.decode_images(datas + [bad], dev, names + ["bad"])
    assert all(x.shape[0] == 3 for x in imgs) and on_cpu[-1]
    out = ds.resized_crop(imgs, [(0, 0, x.shape[1], x.shape[2]) for x in imgs], [False] * len(imgs))
    assert torch.isfinite(out).all()


@pytest.mark.gpu
def test_same_seed_same_batches(dev, small_tree):
    from turboprune_b200.utils import dataset as ds
    mk = lambda: ds.ImageFolderLoader(small_tree / "train", train=True, total_batch_size=4, device=dev, num_workers=4, seed=3)
    a, b = mk(), mk()
    epochs = []
    for _ in range(2):
        xa = [(x.clone(), y.clone()) for x, y in a]
        xb = [(x.clone(), y.clone()) for x, y in b]
        assert all(torch.equal(p, q) and torch.equal(s, t) for (p, s), (q, t) in zip(xa, xb))
        epochs.append(torch.cat([x for x, _ in xa]))
    assert not torch.equal(epochs[0], epochs[1])


def _learnable_tree(root, per_class, seed):
    """4 classes: red / green / blue / yellow base colours with class-specific stripes, random sizes and aspects."""
    rng = np.random.default_rng(seed)
    colours = np.array([[200, 40, 40], [40, 190, 60], [50, 60, 210], [220, 200, 40]])
    for c in range(4):
        for k in range(per_class):
            h, w = int(rng.integers(64, 320)), int(rng.integers(64, 320))
            arr = colours[c][None, None, :] + rng.normal(0, 20, (h, w, 3))
            yy, xx = np.mgrid[:h, :w]
            arr[((xx + yy * (c % 2)) // (6 + 4 * c)) % 2 == 0] += 30
            _save(os.path.join(root, f"n{c:08d}", f"{k}.JPEG"), arr.clip(0, 255).astype(np.uint8), quality=90)


TEST_ACC_BAR = 90.0          # chance is 25 %


@pytest.mark.gpu
def test_run_experiment_trains_on_the_image_folder_loader(dev, tmp_path, capfd):
    """The reference's imagenet_er_balanced config with dataloader_type=imagefolder and ResNet-18, one level, over a
    learnable fabricated tree: ImageFolderImagenet is selected and test accuracy clears the bar."""
    import run_experiment
    from turboprune_b200.utils import config as C
    data = tmp_path / "data"
    _learnable_tree(str(data / "train"), 100, 0)
    _learnable_tree(str(data / "val"), 25, 1)
    cfg = C.compose("imagenet_er_balanced", ["model_params=mp_resnet18", "dataset_params.dataloader_type=imagefolder",
                                             f"dataset_params.data_root_dir={data}", "dataset_params.total_batch_size=32",
                                             "dataset_params.num_workers=4", "+pruning_params.target_sparsity=0.5",
                                             "experiment_params.epochs_per_level=16", "optimizer_params.lr=0.05", "experiment_params.distributed=false",
                                             f"experiment_params.base_dir={tmp_path / 'experiments'}"],
                    os.path.join(G, "reference_conf"))
    prefix, expt = run_experiment.main(cfg)
    err = capfd.readouterr().err
    assert "Data: ImageFolderImagenet" in err and "Data: SyntheticLoaders" not in err
    summary = list(csv.DictReader(open(os.path.join(expt, f"{prefix}_summary.csv"))))
    accs = [float(r["Last_Test_Acc"]) for r in summary]
    rows = list(csv.DictReader(open(os.path.join(expt, "metrics", "level_wise_metrics", "level_0_metrics.csv"))))
    print(f"test accuracy: {accs}; per epoch: {rows}")
    assert len(rows) == 16 and len(accs) == 1 and accs[0] >= TEST_ACC_BAR, accs


@pytest.mark.gpu
def test_other_imagenet_configs_keep_synthetic_loaders(dev, tmp_path):
    import refshim
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import dataset as ds
    for extra in ({}, {"dataloader_type": "synthetic"}, {"dataloader_type": "ffcv"}, {"dataloader_type": "webdataset"}):
        cfg = refshim.make_cfg("resnet18", "imagenet")
        cfg["dataset_params"].update(extra, data_root_dir=str(tmp_path / "absent"), total_batch_size=8)
        h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("t", str(tmp_path)))
        assert isinstance(h.train_loader, ds.SyntheticLoader) and isinstance(h.val_loader, ds.SyntheticLoader)
    assert not os.path.exists(tmp_path / "absent")
