#!/usr/bin/env python
"""What the ImageFolder ImageNet loader delivers, and what it costs a ResNet-50 epoch (1 GPU).

    python tools/imagenet_loader_bench.py [--root DIR] [--images 5000] [--large 8] [--workers 16] [--rounds 3]

Without ``--root`` it writes an ImageNet-like tree to a temporary directory with PIL: ``--images`` JPEGs of about
500 x 375 (either orientation, +-20 %), quality 90, over 100 class directories, ``--large`` of them 3000 x 4000, plus a
500-image val split.  Then, batch 512:
  * the train loader's own rate: wall time of whole epochs (ended by a device synchronise), images per second;
  * where the time goes, phase by phase on the same batches run serially: file reads (``--workers`` threads), batched
    nvjpeg decode (ended by a synchronise), and the ``tp_resized_crop`` launch (CUDA events), with the kernel's bytes
    (each box's uint8 pixels once plus the fp32 output) over its time;
  * ResNet-50 ERK-80 % bf16 epochs through ``PruningHarness.train_epoch`` with this loader and with ``SyntheticLoaders``
    (same steps per epoch), alternating rounds.
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
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
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


def write_tree(root, n, n_large, seed):
    """Smooth colour fields plus noise, so the JPEGs are about as large as photographs of the same size."""
    from PIL import Image

    def one(k):
        rng = np.random.default_rng(seed * 1_000_003 + k)
        if k < n_large:
            h, w = 3000, 4000
        else:
            a, b = int(375 * rng.uniform(0.8, 1.2)), int(500 * rng.uniform(0.8, 1.2))
            h, w = (a, b) if rng.random() < 0.75 else (b, a)
        base = Image.fromarray(rng.integers(0, 256, (12, 16, 3), dtype=np.uint8)).resize((w, h), Image.BILINEAR)
        arr = np.asarray(base, dtype=np.float32) + rng.normal(0, 10, (h, w, 3))
        d = os.path.join(root, f"n{k % 100:08d}")
        os.makedirs(d, exist_ok=True)
        Image.fromarray(arr.clip(0, 255).astype(np.uint8)).save(os.path.join(d, f"img_{k}.JPEG"), quality=90)

    with ThreadPoolExecutor(os.cpu_count() or 8) as pool:
        list(pool.map(one, range(n)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=None, help="an ImageFolder tree with train/ and val/ (default: write one)")
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--large", type=int, default=8)
    ap.add_argument("--workers", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "imagenet_loader_bench needs a GPU"
    import refshim
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import custom_models as cm, dataset as ds, pruning_utils as pu

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    print(f"GPU: {info['name']} | name, power limit, max SM clock: {info['nvidia_smi']}", flush=True)
    tmp = None
    root = args.root
    if root is None:
        tmp = tempfile.TemporaryDirectory()
        root = tmp.name
        t = time.perf_counter()
        write_tree(os.path.join(root, "train"), args.images, args.large, 0)
        write_tree(os.path.join(root, "val"), 500, 0, 1)
        print(f"wrote {args.images} + 500 JPEGs in {time.perf_counter() - t:.1f} s", flush=True)
    B = 512
    loader = ds.ImageFolderLoader(os.path.join(root, "train"), train=True, total_batch_size=B, device=dev,
                                  num_workers=args.workers, seed=0)
    n_batches = len(loader)
    file_mb = sum(os.path.getsize(os.path.join(loader.root, os.fsdecode(p))) for p in loader.paths) / 1e6

    # ---- the loader alone -------------------------------------------------------------------------------------------
    synced(lambda: sum(1 for _ in loader))                     # warm-up: nvjpeg handles, allocator, module load
    epoch_s = [synced(lambda: sum(1 for _ in loader))[0] for _ in range(args.rounds)]

    # ---- phases, serially, on the same batches ----------------------------------------------------------------------
    phases = {"read_ms": [], "decode_ms": [], "crop_ms": [], "crop_bytes": []}
    plan = list(loader._plan(99))
    with ThreadPoolExecutor(args.workers) as pool:
        for idx, u in plan[:min(len(plan), 6)]:
            paths = [os.path.join(loader.root, os.fsdecode(loader.paths[i])) for i in idx.tolist()]
            t0 = time.perf_counter()
            datas = list(pool.map(ds._read_file, paths))
            t1 = time.perf_counter()
            dt, (images, _) = synced(lambda: ds.decode_images(datas, dev))
            hw = torch.tensor([x.shape[1:] for x in images])
            boxes = ds.random_resized_crop_boxes(hw, u[0], u[1], u[2])
            flips = u[3][:, 0] < 0.5
            ds.resized_crop(images, boxes, flips)               # warm
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 20
            e0.record()
            for _ in range(reps):
                ds.resized_crop(images, boxes, flips)
            e1.record()
            torch.cuda.synchronize()
            phases["read_ms"].append((t1 - t0) * 1e3)
            phases["decode_ms"].append(dt * 1e3)
            phases["crop_ms"].append(e0.elapsed_time(e1) / reps)
            phases["crop_bytes"].append(int((boxes[:, 2] * boxes[:, 3]).sum()) * 3 + B * 3 * 224 * 224 * 4)

    # ---- ResNet-50 epochs: this loader against SyntheticLoaders -----------------------------------------------------
    def harness(model, real):
        cfg = refshim.make_cfg("resnet50", "imagenet", precision="bfloat16")
        cfg["optimizer_params"].update(lr=0.05, weight_decay=5e-5)
        cfg["dataset_params"].update(synthetic_steps_per_epoch=n_batches, data_root_dir=root, num_workers=args.workers)
        if real:
            cfg["dataset_params"]["dataloader_type"] = "imagefolder"
        h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("imagenetbench", root), model=model)
        h._setup_optimizer()
        h.scheduler = None
        return h

    torch.manual_seed(0)
    model = cm.TorchVisionModel(refshim.make_cfg("resnet50", "imagenet"))
    pu.prune_er_erk(model, 0.2)
    real, synth = harness(model, True), harness(copy.deepcopy(model), False)
    assert isinstance(real.train_loader, ds.ImageFolderLoader) and isinstance(synth.train_loader, ds.SyntheticLoader)
    for h in (real, synth):
        synced(h.train_epoch)
    rec = {"epoch_s_imagefolder": [], "epoch_s_synthetic": []}
    for _ in range(args.rounds):
        rec["epoch_s_imagefolder"].append(synced(real.train_epoch)[0])
        rec["epoch_s_synthetic"].append(synced(synth.train_epoch)[0])
    if tmp is not None:
        tmp.cleanup()

    med = {k: statistics.median(v) for k, v in {**phases, **rec, "loader_epoch_s": epoch_s}.items()}
    imgs = n_batches * B
    line = {
        "gpu": info, "images": len(loader.labels), "large_3000x4000": args.large if args.root is None else None,
        "file_MB": round(file_mb, 1), "batch": B, "batches_per_epoch": n_batches, "read_threads": args.workers,
        "loader_img_per_s": imgs / med["loader_epoch_s"],
        "phase_ms_per_batch": {k: med[k] for k in ("read_ms", "decode_ms", "crop_ms")},
        "phase_img_per_s": {k: B / med[k] * 1e3 for k in ("read_ms", "decode_ms", "crop_ms")},
        "crop_kernel_GB_per_s": med["crop_bytes"] / (med["crop_ms"] * 1e-3) / 1e9,
        "train_img_per_s": {"imagefolder": imgs / med["epoch_s_imagefolder"], "synthetic": imgs / med["epoch_s_synthetic"]},
        "samples": {**rec, "loader_epoch_s": epoch_s, **phases},
    }
    print(f"loader alone {line['loader_img_per_s']:.0f} img/s; per batch: read {med['read_ms']:.1f} ms, decode "
          f"{med['decode_ms']:.1f} ms, crop kernel {med['crop_ms']:.3f} ms ({line['crop_kernel_GB_per_s']:.0f} GB/s); "
          f"ResNet-50 epoch {med['epoch_s_imagefolder']:.3f} s with ImageFolderLoader vs {med['epoch_s_synthetic']:.3f} s "
          f"synthetic ({n_batches} steps)", flush=True)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
