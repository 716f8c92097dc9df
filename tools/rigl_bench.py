#!/usr/bin/env python
"""Cost of RigL drop-and-regrow on the GPU.

    python tools/rigl_bench.py [reps=20] [rounds=3] [batch=256] [steps=12] [interval=4]

1. ``ops.rigl_select`` + ``ops.rigl_apply`` over all 54 masked layers of ResNet-50 with ERK masks at 80 % sparsity
   (25.5 M weights), k = floor(0.3 n_active) per layer: CUDA-event time per call, the bytes the kernels move (counted
   from the passes they make, see ``select_bytes``) and the resulting GB/s.
2. Images/s of a RigL epoch against a static-mask epoch of the same ResNet-50 ERK-80 model through
   ``PruningHarness.train_epoch`` on synthetic ImageNet-shaped batches, alternating the two, ``rounds`` times each.  A
   RigL update batch runs an eager dense-gradient forward / backward and the selection instead of the captured step.

Prints one JSON line with the GPU name and power limit.
"""
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except Exception:
        return None


def select_bytes(numel, active, ks):
    """Bytes read and written by one tp_rigl_select: per phase three histogram passes, one tie-count pass and one write
    pass over the two fp32 operands (DROP: mask, w; GROW: new mask, g); DROP writes every new-mask element, GROW only
    the grown ones."""
    n = sum(numel)
    drop = 5 * 8 * n + 4 * n
    grow = 5 * 8 * n + 4 * sum(ks)
    return drop + grow


def apply_bytes(numel):
    """tp_rigl_apply reads mask and new mask; it writes only changed mask elements and grown weights / momenta, and the
    timed calls hand it new == old, so they write nothing."""
    return 8 * sum(numel)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    batch = int(sys.argv[3]) if len(sys.argv) > 3 else 256
    steps = int(sys.argv[4]) if len(sys.argv) > 4 else 12
    interval = int(sys.argv[5]) if len(sys.argv) > 5 else 4
    if not torch.cuda.is_available():
        raise SystemExit("rigl_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import refshim
    from turboprune_b200 import ops
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu

    # ---- 1. select + apply at ResNet-50 ERK-80 extents
    torch.manual_seed(0)
    model = cm.TorchVisionModel(refshim.make_cfg("resnet50", "imagenet")).to(dev)
    pu.prune_er_erk(model, 0.2)
    layers = [m for _, m in model._masked()]
    ws = [m.weight.detach() for m in layers]
    gs = [torch.randn_like(w) for w in ws]
    ms = [m.mask.contiguous() for m in layers]
    bufs = [torch.randn_like(w) for w in ws]
    numel = [w.numel() for w in ws]
    active = [int(m.sum()) for m in ms]
    ks = [int(math.floor(0.3 * a)) for a in active]
    news = [torch.empty_like(m) for m in ms]
    # apply with new == old changes nothing, so the same inputs can be timed again and again
    for _ in range(3):
        ops.rigl_select(ws, gs, ms, news, ks)
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    sel_ms, app_ms = [], []
    for _ in range(reps):
        e[0].record()
        ops.rigl_select(ws, gs, ms, news, ks)
        e[1].record()
        ops.rigl_apply(ms, ms, ws, bufs)
        e[2].record()
        torch.cuda.synchronize()
        sel_ms.append(e[0].elapsed_time(e[1]))
        app_ms.append(e[1].elapsed_time(e[2]))
    sel_ms.sort(); app_ms.sort()
    sel, app = sel_ms[len(sel_ms) // 2], app_ms[len(app_ms) // 2]
    sb, ab = select_bytes(numel, active, ks), apply_bytes(numel)
    kernel = {"layers": len(layers), "weights": sum(numel), "select_ms_median": round(sel, 4), "select_ms_min": round(sel_ms[0], 4),
              "apply_ms_median": round(app, 4), "select_bytes": sb, "apply_bytes": ab,
              "select_GBps": round(sb / sel / 1e6, 1), "apply_GBps": round(ab / app / 1e6, 1)}
    del model, layers, ws, gs, ms, bufs, news
    torch.cuda.empty_cache()

    # ---- 2. RigL epoch vs static-mask epoch through train_epoch
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.pruning_utils import prune_the_model

    def harness(rigl):
        over = [f"dataset_params.total_batch_size={batch}", f"dataset_params.synthetic_steps_per_epoch={steps}",
                "experiment_params.distributed=false", "experiment_params.base_dir=/tmp/rigl_bench"]
        if rigl:
            over += ["pruning_params=rigl_erk_80", f"pruning_params.rigl_update_interval={interval}",
                     "pruning_params.rigl_end_fraction=1.0"]
        cfg = C.compose("synthetic_rn50_erk80", over, os.path.join(ROOT, "conf_b200"))
        torch.manual_seed(0)
        h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("bench", "/tmp/rigl_bench"))
        prune_the_model(cfg=cfg, harness=h, target_density=0.2)
        h._setup_optimizer()
        h._setup_scheduler(1)
        if rigl:
            h.begin_rigl_level(rounds + 1)            # the schedule spans every timed epoch
        return h

    hs = {"static": harness(False), "rigl": harness(True)}
    for h in hs.values():
        h.train_epoch()                              # warm-up: capture, allocator pools
    torch.cuda.synchronize()
    ips = {k: [] for k in hs}
    for _ in range(rounds):
        for name, h in hs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h.train_epoch()                          # ends in a host sync (the epoch's loss / accuracy)
            torch.cuda.synchronize()
            ips[name].append(round(batch * steps / (time.perf_counter() - t0), 1))
    r = hs["rigl"].rigl
    updates = sum(1 for t in range(steps * (rounds + 1)) if r.is_update(t))
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "select_apply": kernel,
           "epoch": {"batch": batch, "steps_per_epoch": steps, "rigl_interval": interval, "rigl_updates_total": updates,
                     "img_per_s": ips}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
