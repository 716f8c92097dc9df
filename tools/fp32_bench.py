#!/usr/bin/env python
"""ResNet-50 ERK-80 % train step at training_precision: float32 — this repo's fp32 path against the reference's eager fp32
execution model, alternately in the same process on the same GPU.

    python tools/fp32_bench.py [batch=256] [rounds=3] [steps=10]

This repo: ``PruningHarness.train_step`` with a float32 config (TF32 masked GEMMs, split-stack wgrad, ATen BatchNorm /
ReLU / pooling, fused SGD, CUDA-graph replay).  Reference model: the oracle's restatement of the reference's module graph
(oracle/model.py) on cuda, channels_last, cuDNN on ``mask * w`` with TF32 allowed (as the reference sets it), ATen
BatchNorm, ``torch.optim.SGD``.  Prints one JSON line: img/s of both per round, the per-GEMM kernel times of one eager
step of this repo (CUDA events around each masked-GEMM call), the peak device memory of each path, and the GPU name and
power limit.
"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch


def timed(fn, steps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except Exception:
        return None


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from oracle import model as OM, prune as OP
    import refshim
    from turboprune_b200 import ops
    from turboprune_b200.utils import custom_models as cm

    torch.manual_seed(0)
    ref = OM.build("resnet50", "imagenet")
    shapes = [tuple(m.weight.shape) for _, m in OM.masked_layers(ref)]
    torch.manual_seed(1)
    OM.set_er_masks(ref, OP.erk_keep_probabilities(shapes, 0.2))
    state = {k: v.clone() for k, v in ref.state_dict().items()}
    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(B, 3, 224, 224, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 1000, (B,), device=dev, generator=g)

    # reference execution model, fp32 with TF32 convolutions / matmuls
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    ref = ref.to(dev).to(memory_format=torch.channels_last).train()
    opt = torch.optim.SGD(ref.parameters(), lr=0.2, momentum=0.9, weight_decay=1e-4)

    def ref_step():
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(ref(x), t)
        loss.backward()
        opt.step()
        return loss

    # this repo, float32 config
    cfg = refshim.make_cfg("resnet50", "imagenet", precision="float32")
    cfg["optimizer_params"].update(lr=0.2, weight_decay=1e-4)
    torch.manual_seed(0)
    mine = cm.TorchVisionModel(cfg)
    mine.model.load_state_dict(state)
    h = refshim.make_harness(cfg, mine, B)

    def my_step():
        return h.train_step((x, t))["loss"]

    peak = {}
    for name, fn in (("reference_eager_fp32_tf32", ref_step), ("this_repo_fp32", my_step)):
        torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        for _ in range(4):                   # warm-up (cuDNN autotuning; this repo: eager steps, then the graph capture)
            fn()
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 30
    res = {"reference_eager_fp32_tf32": [], "this_repo_fp32": []}
    for _ in range(rounds):
        for name, fn in (("reference_eager_fp32_tf32", ref_step), ("this_repo_fp32", my_step)):
            res[name].append(B / timed(fn, steps) * 1e3)

    # per-GEMM kernel times of one eager step (no graph): fprop / dgrad / wgrad calls of the masked layers
    h.cfg["experiment_params"]["cuda_graph"] = False
    timer = ops.KernelTimer()
    ops.set_timer(timer)
    h.cfg["experiment_params"]["wgrad_side_stream"] = False
    my_step()
    torch.cuda.synchronize()
    ops.set_timer(None)
    gemm = {k: {"ms": round(v[0], 3), "calls": v[2], "tflops": round(v[1] / v[0] / 1e9, 1)} for k, v in timer.totals().items()}
    print(json.dumps({
        "workload": f"resnet50 ERK-80 train step, B={B}, training_precision float32, SGD(0.9, 1e-4)",
        "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
        "img_s": {k: [round(v, 1) for v in vs] for k, vs in res.items()},
        "img_s_median": {k: round(statistics.median(vs), 1) for k, vs in res.items()},
        "this_repo_gemm_ms_per_eager_step": gemm,
        "peak_gib_above_start": {k: round(v, 2) for k, v in peak.items()},
    }))


if __name__ == "__main__":
    main()
