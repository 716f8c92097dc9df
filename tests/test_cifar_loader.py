"""The device-resident CIFAR loader (reference utils/dataset.py:101-256).

CPU: the torch restatement in tests/cifar_loader_oracle.py reproduces the reference loader's batches
(cifar_loader_small.npz, written by tests/golden/make_cifar_loader_golden.py running the unmodified reference on a
fabricated cache) bit for bit.  GPU: the product loader equals the restatement
run on the device from the same seed at full CIFAR extents, never syncs with the host between batches, and trains a
learnable fabricated data set through run_experiment.main.
"""
import csv
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def _write_cache(root, name, split, images, labels, ncls):
    sub = os.path.join(root, name.lower())
    os.makedirs(sub, exist_ok=True)
    torch.save({"images": images.cpu(), "labels": labels.cpu(), "classes": [str(i) for i in range(ncls)]},
               os.path.join(sub, f"{name.upper()}_{split}.pt"))


# ---------------------------------------------------------------- CPU --------------------------------------------------
def test_restatement_reproduces_reference_loader_fixture():
    import cifar_loader_oracle as D
    z = np.load(os.path.join(G, "cifar_loader_small.npz"))
    bs, epochs = int(z["batch_size"]), int(z["epochs"])
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(int(z["seed"]))
        tr = torch.from_numpy(z["train.images"]); tl = torch.from_numpy(z["train.labels"])
        for e, batches in enumerate(D.cifar_loader_epochs(tr, tl, "CIFAR10", bs, True, epochs)):
            assert len(batches) == int(z["train.len"]) == 5
            for i, (x, y) in enumerate(batches):
                assert np.array_equal(x.numpy(), z[f"train.e{e}.b{i}.x"]), (e, i)
                assert np.array_equal(y.numpy(), z[f"train.e{e}.b{i}.y"]), (e, i)
        assert e == epochs - 1
    te = torch.from_numpy(z["test.images"]); tl = torch.from_numpy(z["test.labels"])
    for batches in D.cifar_loader_epochs(te, tl, "CIFAR10", bs, False, 2):
        assert len(batches) == int(z["test.len"]) == 3 and [len(x) for x, _ in batches] == [8, 8, 4]
        for i, (x, y) in enumerate(batches):
            assert np.array_equal(x.numpy(), z[f"test.b{i}.x"]) and np.array_equal(y.numpy(), z[f"test.b{i}.y"]), i


def test_dataset_names_are_case_insensitive():
    from turboprune_b200.utils import dataset as ds
    assert ds.cifar_variant("cifar10")[:2] == ("CIFAR10", "cifar10")
    assert ds.cifar_variant("Cifar100")[:2] == ("CIFAR100", "cifar100")
    assert torch.equal(ds.cifar_variant("CIFAR100")[2], ds.CIFAR100_MEAN)
    with pytest.raises(ValueError):
        ds.cifar_variant("cifar10-c")


# ---------------------------------------------------------------- GPU --------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked CIFAR loader tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def full_cache(tmp_path_factory):
    """50,000 train / 10,000 test random uint8 images under both names, as the reference's cache files."""
    root = str(tmp_path_factory.mktemp("cifar_full"))
    g = torch.Generator().manual_seed(17)
    data = {}
    for name, ncls in (("CIFAR10", 10), ("CIFAR100", 100)):
        for split, n in (("train", 50_000), ("test", 10_000)):
            images = torch.randint(0, 256, (n, 32, 32, 3), generator=g, dtype=torch.uint8)
            labels = torch.randint(0, ncls, (n,), generator=g)
            _write_cache(root, name, split, images, labels, ncls)
            data[name, split] = images, labels
    return root, data


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["CIFAR10", "cifar100"])
def test_loader_equals_restatement_at_full_extents(dev, full_cache, name):
    """Four epochs (the epoch-0 pre-flip, both altflip parities) of AirbenchLoaders' train loader and the test loader:
    every batch and label bit-identical to the restatement on the device, from the same CUDA seed, with the same
    number of draws (the generator states agree after every epoch)."""
    import cifar_loader_oracle as D
    from turboprune_b200.utils import dataset as ds
    root, data = full_cache
    images, labels = data[name.upper(), "train"]
    train = ds.CifarLoader(root, train=True, batch_size=512, aug={"flip": True, "translate": 2}, altflip=True, dataset=name,
                           device=dev)
    assert len(train) == 97 and 50_000 - 97 * 512 == 336
    with torch.random.fork_rng(devices=[dev]):
        torch.cuda.manual_seed(1000 + len(name))
        ref = D.cifar_loader_epochs(images.to(dev), labels.to(dev), name, 512, True, 4)
        for e in range(4):
            before = torch.cuda.get_rng_state(dev)
            got = list(train)
            after = torch.cuda.get_rng_state(dev)
            torch.cuda.set_rng_state(before, dev)
            want = next(ref)
            assert torch.equal(torch.cuda.get_rng_state(dev), after), f"epoch {e}: different number of draws"
            assert len(got) == len(want) == 97
            assert all(x.shape == (512, 3, 32, 32) and x.is_contiguous() for x, _ in got)
            assert torch.equal(torch.cat([x for x, _ in got]), torch.cat([x for x, _ in want])), f"epoch {e}: images"
            assert torch.equal(torch.cat([y for _, y in got]), torch.cat([y for _, y in want])), f"epoch {e}: labels"
    timages, tlabels = data[name.upper(), "test"]
    test = ds.CifarLoader(root, train=False, batch_size=512, dataset=name, device=dev)
    got = list(test)
    want = next(D.cifar_loader_epochs(timages.to(dev), tlabels.to(dev), name, 512, False, 1))
    assert len(test) == len(got) == 20 and len(got[-1][0]) == 272
    for (x, y), (xr, yr) in zip(got, want):
        assert torch.equal(x, xr) and torch.equal(y, yr)


@pytest.mark.gpu
def test_batches_after_the_first_never_sync(dev, full_cache):
    from turboprune_b200.utils import dataset as ds
    root, _ = full_cache
    train = ds.CifarLoader(root, train=True, batch_size=512, aug={"flip": True, "translate": 2}, altflip=True, device=dev)
    test = ds.CifarLoader(root, train=False, batch_size=512, device=dev)
    for loader in (train, train, test):          # epoch 0 (prepares), epoch 1 (mirrored), the test set
        it = iter(loader)
        first = next(it)
        count = 1
        torch.cuda.set_sync_debug_mode("error")
        try:
            for _ in it:
                count += 1
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert count == len(loader) and first[0].shape[1:] == (3, 32, 32)


@pytest.mark.gpu
def test_augment_kernel_gathers_by_source_index(dev):
    """tp_cifar_augment with idx (repeats, translate, flip, cutout; and a plain gather) equals the oracle on the gathered
    arrays: output j is source idx[j] with source idx[j]'s draws."""
    from oracle import data as D
    from turboprune_b200.utils import dataset as ds
    g = torch.Generator().manual_seed(8)
    src = torch.randn(37, 3, 40, 40, generator=g)
    idx = torch.cat([torch.randint(0, 37, (45,), generator=g), torch.tensor([5, 5, 5, 36, 0])])
    sh = torch.randint(-4, 5, (37, 2), generator=g)
    fm = torch.rand(37, generator=g) < 0.5
    cy = torch.randint(0, 25, (37,), generator=g); cx = torch.randint(0, 25, (37,), generator=g)
    out = ds._augment(src.to(dev), (32, 32), 4, shifts=sh.to(dev), flip=fm.to(dev), corner_y=cy.to(dev), corner_x=cx.to(dev),
                      cut_size=8, idx=idx.to(dev))
    i = idx.numpy()
    ref = D.augment(src.numpy()[i], 32, sh.numpy()[i], fm.numpy()[i], 8, cy.numpy()[i], cx.numpy()[i])
    assert out.shape == (50, 3, 32, 32) and np.array_equal(out.cpu().numpy(), ref)
    plain = ds._augment(src.to(dev), (40, 40), 0, idx=idx.to(dev))
    assert np.array_equal(plain.cpu().numpy(), src.numpy()[i])


def _learnable_cache(root, n_train, n_test, seed=3):
    """10 classes: a class colour plus per-pixel noise, clipped to uint8."""
    g = torch.Generator().manual_seed(seed)
    colours = torch.randint(40, 216, (10, 3), generator=g).float()
    for split, n in (("train", n_train), ("test", n_test)):
        labels = torch.randint(0, 10, (n,), generator=g)
        x = colours[labels].view(n, 1, 1, 3) + 32 * torch.randn(n, 32, 32, 3, generator=g)
        _write_cache(root, "CIFAR10", split, x.round().clamp(0, 255).to(torch.uint8), labels, 10)


TEST_ACC_BAR = 90.0            # measured 100.0 % at both levels on an H100 80GB HBM3 (700 W); chance is 10 %


@pytest.mark.gpu
def test_run_experiment_trains_on_the_cifar_loader(dev, tmp_path, capfd):
    """The reference's own cifar10_er_erk config (dataloader_type: torch), composed as SURVEY.md Appendix D config 1,
    on a fabricated learnable cache: CifarLoader is selected, both levels write their CSVs, test accuracy clears the bar."""
    import run_experiment
    from turboprune_b200.utils import config as C
    data = tmp_path / "data"
    _learnable_cache(str(data), 10_240, 2_000)
    cfg = C.compose("cifar10_er_erk", ["pruning_params=iterative_imp", "pruning_params.target_sparsity=0.2",
                                       "experiment_params.epochs_per_level=4", f"dataset_params.data_root_dir={data}",
                                       f"experiment_params.base_dir={tmp_path / 'experiments'}"],
                    os.path.join(G, "reference_conf"))
    assert cfg.dataset_params.dataloader_type == "torch"
    prefix, expt = run_experiment.main(cfg)
    err = capfd.readouterr().err
    assert "Data: CifarLoader" in err and "Data: SyntheticLoaders" not in err
    for level in (0, 1):
        rows = list(csv.DictReader(open(os.path.join(expt, "metrics", "level_wise_metrics", f"level_{level}_metrics.csv"))))
        assert len(rows) == 4
    summary = list(csv.DictReader(open(os.path.join(expt, f"{prefix}_summary.csv"))))
    accs = [float(r["Last_Test_Acc"]) for r in summary]
    print(f"test accuracy per level: {accs}")
    assert [r["Level"] for r in summary] == ["0", "1"] and min(accs) >= TEST_ACC_BAR, accs


@pytest.mark.gpu
def test_configs_without_a_loader_type_keep_synthetic_loaders(dev, tmp_path):
    import refshim
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import dataset as ds
    for extra in ({}, {"dataloader_type": "synthetic"}):
        cfg = refshim.make_cfg("resnet18", "cifar10")
        cfg["dataset_params"].update(extra, data_root_dir=str(tmp_path / "absent"))
        h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("t", str(tmp_path)))
        assert isinstance(h.train_loader, ds.SyntheticLoader) and isinstance(h.val_loader, ds.SyntheticLoader)
    assert not os.path.exists(tmp_path / "absent")
