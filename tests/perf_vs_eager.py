#!/usr/bin/env python
"""Reference-style GPU eager path vs this repo's path on the same GPU (SURVEY.md §8(d), last row).

The reference is a GPU framework: on an H100 it would run the masked layers as ``F.conv2d(x, mask * w)`` on
cuDNN under bf16 autocast, torchvision BatchNorm/ReLU, ``torch.optim.SGD`` (mask_layers.py:26-34,
base_harness.py:115-134).  The reference is not part of this repository, so the oracle's restatement of that
module graph (oracle/model.py — the same torch ops, validated against the reference's recorded outputs in tests/) is moved to
``cuda`` and timed here: this is the "kernel to beat".  It lives under tests/ because it executes oracle/ code;
it is a script (not collected by pytest):

    python tests/perf_vs_eager.py [per_gpu_batch=256] [steps=10]

Prints one JSON line: eager img/s, this repo's eager (no CUDA graph) and graph-replay img/s for the same model,
masks, batch and optimizer settings.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch


def timed(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    dev = torch.device("cuda", 0)
    from oracle import model as OM, prune as OP
    import refshim
    from turboprune_b200.utils import custom_models as cm
    from turboprune_b200.grad_exchange import GradArena
    from turboprune_b200.optim import FusedSGD

    torch.manual_seed(0)
    ref = OM.build("resnet50", "imagenet")
    shapes = [tuple(m.weight.shape) for _, m in OM.masked_layers(ref)]
    probs = OP.erk_keep_probabilities(shapes, 0.2)
    torch.manual_seed(1)
    OM.set_er_masks(ref, probs)
    state = {k: v.clone() for k, v in ref.state_dict().items()}

    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(B, 3, 224, 224, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    t = torch.randint(0, 1000, (B,), device=dev, generator=g)

    # ---- reference-style eager path: cuDNN convs on mask*w, ATen BN/ReLU, torch SGD -------------------------
    ref = ref.to(dev).to(memory_format=torch.channels_last).train()
    opt = torch.optim.SGD(ref.parameters(), lr=0.2, momentum=0.9, weight_decay=1e-4)
    torch.backends.cudnn.benchmark = True

    def ref_step():
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(ref(x), t)
        loss.backward()
        opt.step()
        return loss

    ms_ref = timed(ref_step, steps)
    loss_ref = float(ref_step())
    del ref, opt
    torch.cuda.empty_cache()

    # ---- this repo: same weights, masks, batch --------------------------------------------------------------
    torch.manual_seed(0)
    mine = cm.TorchVisionModel(refshim.make_cfg("resnet50", "imagenet"))
    mine.model.load_state_dict(state)            # same keys as the reference's inner torchvision model (masks included)
    mine = mine.to(dev).train()
    opt2 = FusedSGD(mine.parameters(), lr=0.2, momentum=0.9, weight_decay=1e-4, capturable=True)
    arena = GradArena(list(mine.parameters()))

    def my_step():
        arena.zero()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(mine(x), t)
        loss.backward()
        opt2.step()
        return loss

    ms_eager = timed(my_step, steps)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        my_step()
    torch.cuda.current_stream(dev).wait_stream(side)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, capture_error_mode="thread_local"):
        loss_t = my_step()
    ms_graph = timed(gr.replay, steps)
    print(json.dumps({
        "workload": f"resnet50 ERK-80 train step, B={B}, bf16 autocast, SGD(0.9, 1e-4), 1x {torch.cuda.get_device_name()}",
        "reference_style_eager_cudnn": {"ms_per_step": ms_ref, "img_s": B / ms_ref * 1e3, "loss_after": loss_ref},
        "this_repo_eager": {"ms_per_step": ms_eager, "img_s": B / ms_eager * 1e3},
        "this_repo_cuda_graph": {"ms_per_step": ms_graph, "img_s": B / ms_graph * 1e3, "loss_last": float(loss_t)},
        "speedup_graph_vs_reference_eager": ms_ref / ms_graph,
    }))


if __name__ == "__main__":
    main()
