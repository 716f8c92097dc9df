#!/usr/bin/env python
"""What the device-resident CIFAR loader costs a training epoch (1 GPU).

    python tools/cifar_epoch_bench.py [--rounds R]

ResNet-18 / CIFAR-10 at ERK 80 % sparsity, batch 512, bf16, through ``PruningHarness.train_epoch`` (CUDA-graph replay)
on a fabricated 50,000 / 10,000-image uint8 cache written to a temporary directory.  Alternating, one epoch each, it
records:
  * the epoch's wall time with ``CifarLoader`` and with ``SyntheticLoaders`` (97 steps each, the same harness step);
  * the loader alone: wall time to produce one epoch's batches (ended by a device synchronise) and, in a profiled pass
    of its own, the device time of its kernels;
  * the torch restatement of the reference loader's op sequence (tests/cifar_loader_oracle.py: one cropped copy of the
    whole data set, a mirrored copy on odd epochs, then the batch gathers), its wall time per epoch.
Prints the GPU's name and power limit and one JSON line.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q or "nvidia-smi unavailable"}


def synced(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "cifar_epoch_bench needs a GPU"
    import refshim
    import cifar_loader_oracle as D
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import custom_models as cm, dataset as ds, pruning_utils as pu

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    print(f"GPU: {info['name']} | name, power limit, max SM clock: {info['nvidia_smi']}", flush=True)
    with tempfile.TemporaryDirectory() as root:
        g = torch.Generator().manual_seed(0)
        for split, n in (("train", 50_000), ("test", 10_000)):
            os.makedirs(os.path.join(root, "cifar10"), exist_ok=True)
            torch.save({"images": torch.randint(0, 256, (n, 32, 32, 3), generator=g, dtype=torch.uint8),
                        "labels": torch.randint(0, 10, (n,), generator=g), "classes": [str(i) for i in range(10)]},
                       os.path.join(root, "cifar10", f"CIFAR10_{split}.pt"))

        def harness(model, real):
            cfg = refshim.make_cfg("resnet18", "cifar10", precision="bfloat16")
            cfg["optimizer_params"].update(lr=0.05)
            cfg["dataset_params"].update(synthetic_steps_per_epoch=97, data_root_dir=root)
            if real:
                cfg["dataset_params"]["dataloader_type"] = "torch"
            h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("cifarbench", root), model=model)
            h._setup_optimizer()
            h.scheduler = None            # constant LR: the schedule's host arithmetic is the same for both loaders
            return h

        torch.manual_seed(0)
        model = cm.TorchVisionModel(refshim.make_cfg("resnet18", "cifar10"))
        pu.prune_er_erk(model, 0.2)
        real, synth = harness(model, True), harness(copy.deepcopy(model), False)   # each with its own gradient arena
        assert isinstance(real.train_loader, ds.CifarLoader) and isinstance(synth.train_loader, ds.SyntheticLoader)
        assert len(real.train_loader) == len(synth.train_loader) == 97
        loader = ds.CifarLoader(root, train=True, batch_size=512, aug={"flip": True, "translate": 2}, altflip=True, device=dev)
        train = torch.load(os.path.join(root, "cifar10", "CIFAR10_train.pt"), map_location=dev)
        restated = D.cifar_loader_epochs(train["images"], train["labels"], "CIFAR10", 512, True, 2 * args.rounds + 2)

        for h in (real, synth):          # warm-up: preparation, graph capture, allocator pools
            synced(h.train_epoch)
        synced(lambda: list(loader)); synced(lambda: next(restated))
        rec = {k: [] for k in ("epoch_s_cifar", "epoch_s_synthetic", "loader_epoch_ms", "restated_reference_epoch_ms")}
        for _ in range(args.rounds):
            rec["epoch_s_cifar"].append(synced(real.train_epoch)[0])
            rec["epoch_s_synthetic"].append(synced(synth.train_epoch)[0])
            for _ in range(2):           # both altflip parities
                rec["loader_epoch_ms"].append(synced(lambda: list(loader))[0] * 1e3)
                rec["restated_reference_epoch_ms"].append(synced(lambda: next(restated))[0] * 1e3)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            synced(lambda: list(loader))
        dev_us = sum(getattr(e, "self_device_time_total", 0) for e in prof.key_averages())

    med = {k: statistics.median(v) for k, v in rec.items()}
    line = {
        "gpu": info, "workload": "resnet18 cifar10 ERK-80% bf16, batch 512, 97 steps/epoch, PruningHarness.train_epoch",
        "rounds": args.rounds, "median": med, "samples": rec,
        "loader_overhead_s_per_epoch": med["epoch_s_cifar"] - med["epoch_s_synthetic"],
        "loader_device_ms_per_epoch": dev_us / 1e3,
    }
    print(f"epoch wall time: CifarLoader {med['epoch_s_cifar']:.3f} s, SyntheticLoaders {med['epoch_s_synthetic']:.3f} s; "
          f"loader alone {med['loader_epoch_ms']:.1f} ms wall, {dev_us / 1e3:.1f} ms device; "
          f"restated reference loader {med['restated_reference_epoch_ms']:.1f} ms", flush=True)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
