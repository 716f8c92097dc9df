#!/usr/bin/env python
"""Generate ``reference_live.npz`` and ``reference_conf/`` by running the UNMODIFIED reference on CPU.

The tests used to compare against a live import of the reference tree whenever one was mounted next to the
repository; these fixtures hold exactly what those comparisons read from it, so the comparisons run everywhere:

  reference_live.npz
    sd_sha256.keys / .values    "<tag>.<key>" -> sha256 of every state-dict tensor of the reference's seed-0 ResNet-18 / CIFAR-10
                                (TorchVisionModel), after construction (tag "init") and after prune_er_erk /
                                prune_er_balanced (seed 5)
    rn18.sparsity.<fn>          get_overall_sparsity() after each of those
    rn18.x, rn18.logits         an input batch and the reference model's eval-mode output on it
    rn18.mag08.masks_sha256     sha256 of the reference's masks after prune_mag(0.8)
    crop.pad, crop.shifts, crop.out   utils/dataset.py batch_crop under torch.manual_seed(8)
  reference_conf/               the reference's own YAML configuration files the config composer is tested on

Run from the repository root with the reference checked out at $TURBOPRUNE_REFERENCE (default /root/reference).
"""
import hashlib
import os
import shutil
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refshim  # noqa: E402

CONF_FILES = ["cifar10_er_erk.yaml", "imagenet_er_balanced.yaml", "dataset_params/dp_cifar10.yaml",
              "dataset_params/dp_imagenet_ffcv.yaml", "dataset_params/dp_imagenet_wds.yaml",
              "optimizer_params/sgd_cifar10.yaml", "optimizer_params/sgd_imagenet.yaml",
              "experiment_params/ep_cifar10.yaml", "experiment_params/ep_imagenet.yaml",
              "model_params/mp_resnet18.yaml", "model_params/mp_resnet50.yaml",
              "pruning_params/pai_er_erk.yaml", "pruning_params/pai_er_balanced.yaml",
              "pruning_params/iterative_imp.yaml", "pruning_params/iterative_wr.yaml", "cyclic_training/ct_no_cyclic.yaml"]


def sha(t) -> str:
    a = t.detach().cpu().contiguous().numpy() if torch.is_tensor(t) else np.ascontiguousarray(t)
    return hashlib.sha256(a.tobytes()).hexdigest()


def main():
    out, hashes = {}, {}
    ml, rpu, rcm = refshim.load_reference()
    torch.manual_seed(0)
    r = rcm.TorchVisionModel(refshim.make_cfg("resnet18", "cifar10"))
    for k, v in r.state_dict().items():
        hashes[f"init.{k}"] = sha(v)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 32, 32, generator=g)
    r.eval()
    with torch.no_grad():
        out["rn18.x"] = x.numpy()
        out["rn18.logits"] = r(x).numpy()
    torch.manual_seed(0)
    r2 = rcm.TorchVisionModel(refshim.make_cfg("resnet18", "cifar10"))
    rpu.prune_mag(r2, 0.8)
    hh = hashlib.sha256()
    for m in r2.model.modules():
        if isinstance(m, (ml.ConvMask, ml.Conv1dMask, ml.LinearMask)):
            hh.update(np.ascontiguousarray(m.mask.numpy()).tobytes())
    out["rn18.mag08.masks_sha256"] = hh.hexdigest()
    for fn in ("prune_er_erk", "prune_er_balanced"):
        torch.manual_seed(5)
        getattr(rpu, fn)(r, 0.2)
        for k, v in r.state_dict().items():
            hashes[f"{fn}.{k}"] = sha(v)
        out[f"rn18.sparsity.{fn}"] = np.float64(r.get_overall_sparsity())

    ds = refshim.load_reference_dataset()
    g = torch.Generator().manual_seed(3)
    imgs = torch.randn(5, 3, 10, 10, generator=g)
    pad = torch.nn.functional.pad(imgs, (3,) * 4, "reflect")
    torch.manual_seed(8)
    out["crop.out"] = ds.batch_crop(pad, 10).numpy()
    torch.manual_seed(8)
    out["crop.shifts"] = torch.randint(-3, 4, size=(5, 2)).numpy()
    out["crop.pad"] = pad.numpy()
    out["sd_sha256.keys"] = np.array(list(hashes))
    out["sd_sha256.values"] = np.array(list(hashes.values()))
    np.savez_compressed(os.path.join(HERE, "reference_live.npz"), **{k: np.asarray(v) for k, v in out.items()})

    dst = os.path.join(HERE, "reference_conf")
    for f in CONF_FILES:
        os.makedirs(os.path.dirname(os.path.join(dst, f)), exist_ok=True)
        shutil.copyfile(os.path.join(refshim.REFERENCE_ROOT, "conf", f), os.path.join(dst, f))
    print("wrote reference_live.npz and reference_conf/")


if __name__ == "__main__":
    main()
