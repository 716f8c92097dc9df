#!/usr/bin/env python
"""Cost of the fused AdamW step on the GPU.

    python tools/adamw_bench.py [reps=50] [rounds=5] [batch=256] [steps=8]

1. One optimizer step over ResNet-50's 161 parameters (25.6 M values) and DeiT-S's 152 (22.1 M): ``FusedAdamW`` against
   ``torch.optim.AdamW`` foreach-capturable and fused-capturable, on the same parameters and gradients, alternating the
   three ``rounds`` times.  Each step is timed with CUDA events two ways: replays of a CUDA graph of one step (device
   time, what the harness's captured train step pays) and eager ``step()`` calls back to back (host + device).  The
   step moves 28 B per value (read w, g, m, v; write w, m, v); GB/s and the share of the H100 SXM data-sheet 3.35 TB/s
   are computed from that and the graph-replay time.
2. The DeiT-S train step (``PruningHarness.train_epoch``, synthetic ImageNet-shaped batches, bf16, SNIP 50 %) with
   optimizer_name AdamW against SGD, alternating, ``rounds`` epochs of ``steps`` batches each.

Prints one JSON line with the GPU name and power limit.
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
BYTES_PER_VALUE = 28


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except Exception:
        return None


def param_list(model):
    if model == "resnet50":
        import torchvision
        with torch.device("meta"):
            net = torchvision.models.resnet50()
    else:
        from turboprune_b200.utils import vit
        with torch.device("meta"):
            net = vit.local_deit_small_patch16_224()
    return [tuple(p.shape) for p in net.parameters()]


def time_optimizers(model, reps, rounds, dev):
    from turboprune_b200.grad_exchange import plan_buckets
    from turboprune_b200.optim import FusedAdamW
    shapes = param_list(model)
    g = torch.Generator(device=dev).manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(s, generator=g, device=dev) * 0.02) for s in shapes]
    numels = [p.numel() for p in params]
    (_, offs, total), = plan_buckets(numels, 1 << 62)
    flat = torch.randn(total, generator=g, device=dev) * 1e-3          # gradients: views into one buffer, as in training
    for p, o, n in zip(params, offs, numels):
        p.grad = flat[o:o + n].view_as(p)
    kw = dict(lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.05)
    opts = {"fused_adamw": FusedAdamW(params, capturable=True, **kw),
            "torch_foreach_capturable": torch.optim.AdamW(params, foreach=True, capturable=True, **kw),
            "torch_fused_capturable": torch.optim.AdamW(params, fused=True, capturable=True, **kw)}
    graphs = {}
    side = torch.cuda.Stream(dev)
    for name, o in opts.items():
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(3):                      # state, pointer tables, allocator pools
                o.step()
        torch.cuda.current_stream(dev).wait_stream(side)
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            o.step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {k: {"graph": [], "eager": []} for k in opts}
    for _ in range(rounds):
        for name, o in opts.items():
            for mode in ("graph", "eager"):
                run = graphs[name].replay if mode == "graph" else o.step
                for _ in range(3):
                    run()
                torch.cuda.synchronize()
                e0.record()
                for _ in range(reps):
                    run()
                e1.record()
                torch.cuda.synchronize()
                res[name][mode].append(e0.elapsed_time(e1) / reps)
    n = sum(numels)
    out = {"params": len(params), "values": n, "bytes_per_step": BYTES_PER_VALUE * n}
    for name, r in res.items():
        gm = sorted(r["graph"])[len(r["graph"]) // 2]
        em = sorted(r["eager"])[len(r["eager"]) // 2]
        gbps = BYTES_PER_VALUE * n / (gm * 1e-3) / 1e9
        out[name] = {"graph_ms_median": round(gm, 4), "graph_ms_min": round(min(r["graph"]), 4),
                     "eager_ms_median": round(em, 4), "GBps": round(gbps, 1),
                     "share_of_3.35TBps": round(gbps * 1e9 / HBM_BYTES_PER_S, 3)}
    out["fused_vs_torch_fused_graph"] = round(out["fused_adamw"]["graph_ms_median"] / out["torch_fused_capturable"]["graph_ms_median"], 3)
    del opts, graphs, params, flat
    torch.cuda.empty_cache()
    return out


def time_train_step(batch, steps, rounds):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.pruning_utils import prune_the_model

    def harness(opt):
        over = [f"dataset_params.total_batch_size={batch}", f"dataset_params.synthetic_steps_per_epoch={steps}",
                "experiment_params.base_dir=/tmp/adamw_bench"]
        if opt == "sgd":
            over += ["optimizer_params=sgd_triangular"]
        cfg = C.compose("synthetic_deit_s_snip50_adamw", over, os.path.join(ROOT, "conf_b200"))
        torch.manual_seed(0)
        h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("bench", "/tmp/adamw_bench"))
        prune_the_model(cfg=cfg, harness=h, target_density=0.5)
        h._setup_optimizer()
        h._setup_scheduler(rounds + 1)
        return h

    hs = {"adamw": harness("adamw"), "sgd": harness("sgd")}
    for h in hs.values():
        h.train_epoch()                              # warm-up: capture, allocator pools
    torch.cuda.synchronize()
    ips = {k: [] for k in hs}
    for _ in range(rounds):
        for name, h in hs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h.train_epoch()
            torch.cuda.synchronize()
            ips[name].append(round(batch * steps / (time.perf_counter() - t0), 1))
    med = {k: sorted(v)[len(v) // 2] for k, v in ips.items()}
    return {"batch": batch, "steps_per_epoch": steps, "optimizer": {k: type(h.optimizer).__name__ for k, h in hs.items()},
            "img_per_s": ips, "img_per_s_median": med, "adamw_over_sgd": round(med["adamw"] / med["sgd"], 3)}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    batch = int(sys.argv[3]) if len(sys.argv) > 3 else 256
    steps = int(sys.argv[4]) if len(sys.argv) > 4 else 8
    if not torch.cuda.is_available():
        raise SystemExit("adamw_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for model in ("resnet50", "deit_s"):
        out[model] = time_optimizers(model, reps, rounds, dev)
    out["deit_s_train_step"] = time_train_step(batch, steps, rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
