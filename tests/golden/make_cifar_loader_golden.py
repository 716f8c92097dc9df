#!/usr/bin/env python
"""Generate ``cifar_loader_small.npz`` by EXECUTING THE UNMODIFIED REFERENCE's CifarLoader on CPU.

The reference's CifarLoader (utils/dataset.py:101-226) with AirbenchLoaders' arguments (:243-256): translate 2 +
random pre-flip + altflip for the training loader, plain and unshuffled for the test loader.  It runs over a fabricated
cache of 40 train / 20 test uint8 images in the reference's format, batch 8, three epochs; the file holds the source
data, the seed and every batch.  The reference loads its cache onto 'cuda'; torch.load is pointed at the CPU while it
runs (the reference source stays untouched).

Run only in the build container:  python tests/golden/make_cifar_loader_golden.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refshim  # noqa: E402


def gen_cifar_loader():
    ds = refshim.load_reference_dataset()
    g = torch.Generator().manual_seed(5)
    out, seed, bs, epochs = {}, 1234, 8, 3
    with tempfile.TemporaryDirectory() as root:
        os.makedirs(os.path.join(root, "cifar10"))
        for split, n in (("train", 40), ("test", 20)):
            images = torch.randint(0, 256, (n, 32, 32, 3), generator=g, dtype=torch.uint8)
            labels = torch.randint(0, 10, (n,), generator=g)
            torch.save({"images": images, "labels": labels, "classes": [str(i) for i in range(10)]},
                       os.path.join(root, "cifar10", f"CIFAR10_{split}.pt"))
            out[f"{split}.images"], out[f"{split}.labels"] = images.numpy(), labels.numpy()
        real_load = torch.load
        torch.load = lambda *a, **k: real_load(*a, **{**k, "map_location": "cpu"})
        try:
            train = ds.CifarLoader(root, batch_size=bs, train=True, aug={"flip": True, "translate": 2}, altflip=True,
                                   dataset="CIFAR10")
            test = ds.CifarLoader(root, batch_size=bs, train=False, dataset="CIFAR10")
        finally:
            torch.load = real_load
        out["seed"], out["batch_size"], out["epochs"] = np.array(seed), np.array(bs), np.array(epochs)
        out["train.len"], out["test.len"] = np.array(len(train)), np.array(len(test))
        torch.manual_seed(seed)
        for e in range(epochs):
            for i, (x, y) in enumerate(train):
                out[f"train.e{e}.b{i}.x"], out[f"train.e{e}.b{i}.y"] = x.contiguous().numpy(), y.numpy()
            for i, (x, y) in enumerate(test):           # no draws: every epoch yields the same batches
                if e == 0:
                    out[f"test.b{i}.x"], out[f"test.b{i}.y"] = x.contiguous().numpy(), y.numpy()
                else:
                    assert np.array_equal(x.numpy(), out[f"test.b{i}.x"]) and np.array_equal(y.numpy(), out[f"test.b{i}.y"])
    path = os.path.join(HERE, "cifar_loader_small.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    gen_cifar_loader()
