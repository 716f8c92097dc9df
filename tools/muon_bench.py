#!/usr/bin/env python
"""Cost of the fused Muon + AdamW step on the GPU.

    python tools/muon_bench.py [reps=20] [rounds=3] [batch=128] [steps=6]

1. One optimizer step over ResNet-50's and DeiT-S's parameters: ``FusedMuon`` (Muon for the weights the harness puts
   in the Muon group: every conv / linear weight but the classifier and DeiT's patch embedding; AdamW for the rest),
   replayed from a CUDA graph and called eagerly, against ``torch.optim.Muon`` on the 2-D views plus
   ``torch.optim.AdamW(fused=True, capturable=True)`` on the rest, eagerly and (when torch's step captures) from a
   graph.  Alternating, ``rounds`` times; CUDA events.
2. The 3 * 5 Newton-Schulz GEMM launches alone (CUDA events).  Their FLOP rate counts the work the kernel does: 2 * 64^3
   per K block of every tile of the 64-padded tile lists, upper-triangle tiles only for G and H (the "with the symmetric
   halves, 64-padded" count), as a share of the 989 TFLOP/s bf16 dense data-sheet figure of the H100 SXM.
3. The ResNet-50 ERK-80 % and DeiT-S SNIP-50 % train steps (``PruningHarness.train_epoch``, synthetic ImageNet-shaped
   batches, bf16) with optimizer_name MuonAdamW against SGD, alternating, ``rounds`` epochs of ``steps`` batches each.

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

import torch

BF16_FLOPS = 989e12              # H100 SXM data sheet, dense bf16


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except Exception:
        return None


def named_params(model):
    if model == "resnet50":
        import torchvision
        with torch.device("meta"):
            net = torchvision.models.resnet50()
        head = "fc.weight"
    else:
        from turboprune_b200.utils import vit
        with torch.device("meta"):
            net = vit.local_deit_small_patch16_224()
        head = "head.weight"
    named = [(n, tuple(p.shape)) for n, p in net.named_parameters()]
    # the masked layers' weights: not the classifier, DeiT's patch embedding, cls_token or pos_embed
    return named, [len(s) >= 2 and n.endswith("weight") and n != head and "patch_embed" not in n for n, s in named]


def _time(run, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _capture(step, dev):
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return g


def time_optimizers(model, reps, rounds, dev):
    from turboprune_b200 import ops
    from turboprune_b200.optim import FusedMuon
    named, is_muon = named_params(model)
    gen = torch.Generator(device=dev).manual_seed(0)
    init = [torch.randn(s, generator=gen, device=dev) * 0.02 for _, s in named]
    grads = [torch.randn(s, generator=gen, device=dev) * 1e-3 for _, s in named]
    kw = dict(lr=5e-4, weight_decay=0.05)
    ps = [torch.nn.Parameter(v.clone()) for v in init]
    for p, g in zip(ps, grads):
        p.grad = g
    mine = FusedMuon([dict(params=[p for p, m in zip(ps, is_muon) if m]),
                      dict(params=[p for p, m in zip(ps, is_muon) if not m], use_muon=False)],
                     adjust_lr_fn="match_rms_adamw", capturable=True, **kw)
    rv = [torch.nn.Parameter(v.clone().view(v.shape[0], -1)) for v, m in zip(init, is_muon) if m]
    for v, g in zip(rv, [g for g, m in zip(grads, is_muon) if m]):
        v.grad = g.view(v.shape)
    ra = [torch.nn.Parameter(v.clone()) for v, m in zip(init, is_muon) if not m]
    for p, g in zip(ra, [g for g, m in zip(grads, is_muon) if not m]):
        p.grad = g
    t_muon = torch.optim.Muon(rv, adjust_lr_fn="match_rms_adamw", **kw)
    t_adamw = torch.optim.AdamW(ra, fused=True, capturable=True, **kw)

    def torch_step():
        t_muon.step()
        t_adamw.step()

    runs = {"fused_graph": _capture(mine.step, dev).replay, "fused_eager": mine.step, "torch_eager": torch_step}
    try:
        runs["torch_graph"] = _capture(torch_step, dev).replay
    except Exception as e:            # torch's step may not capture: report it
        runs["torch_graph"] = None
        torch_graph_error = f"{type(e).__name__}: {e}"[:200]
    # the 15 Newton-Schulz launches alone, on the workspace the fused step left
    st = next(iter(mine._muon.values()))
    a, b, c = mine.param_groups[0]["ns_coefficients"]

    def ns():
        src = 0
        for _ in range(5):
            ops.muon_ns_gemm(ops.MUON_GRAM, st["xws"], st["tiles"][(ops.MUON_GRAM, src)], 1.0, 0.0)
            ops.muon_ns_gemm(ops.MUON_POLY, st["xws"], st["tiles"][(ops.MUON_POLY, 0)], c, b)
            ops.muon_ns_gemm(ops.MUON_UPDATE, st["xws"], st["tiles"][(ops.MUON_UPDATE, src)], 1.0, a)
            src = 1 - src
    runs["ns_gemms"] = ns
    res = {k: [] for k, r in runs.items() if r is not None}
    for _ in range(rounds):
        for k in res:
            res[k].append(round(_time(runs[k], reps), 4))
    plan = st["plan"]
    flops = sum(2 * 64 ** 3 * int(t[:, 4].sum()) for k, t in plan.gemm_tiles.items() if k[1] == 0) * 5
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    out = {"muon_layers": len(plan.shapes), "muon_values": sum(a * b for a, b in plan.shapes),
           "values": sum(math.prod(s) for _, s in named), "ms": res, "ms_median": med,
           "ns_gflop_per_step_64padded_symmetric": round(flops / 1e9, 1),
           "ns_tflops": round(flops / (med["ns_gemms"] * 1e-3) / 1e12, 1),
           "ns_share_of_989": round(flops / (med["ns_gemms"] * 1e-3) / BF16_FLOPS, 3),
           "fused_graph_vs_torch_eager": round(med["fused_graph"] / med["torch_eager"], 3)}
    if "torch_graph" in med:
        out["fused_graph_vs_torch_graph"] = round(med["fused_graph"] / med["torch_graph"], 3)
    else:
        out["torch_graph_error"] = torch_graph_error
    del mine, t_muon, t_adamw, runs
    torch.cuda.empty_cache()
    return out


def time_train_step(config, density, batch, steps, rounds):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.pruning_utils import prune_the_model

    def harness(opt):
        over = [f"dataset_params.total_batch_size={batch}", f"dataset_params.synthetic_steps_per_epoch={steps}",
                "experiment_params.base_dir=/tmp/muon_bench", "experiment_params.distributed=false"]
        if opt == "sgd":
            over += ["optimizer_params=sgd_triangular"]
        cfg = C.compose(config, over, os.path.join(ROOT, "conf_b200"))
        torch.manual_seed(0)
        h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("bench", "/tmp/muon_bench"))
        prune_the_model(cfg=cfg, harness=h, target_density=density)
        h._setup_optimizer()
        h._setup_scheduler(rounds + 1)
        return h

    hs = {"muon_adamw": harness("muon"), "sgd": harness("sgd")}
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
    out = {"batch": batch, "steps_per_epoch": steps, "optimizer": {k: type(h.optimizer).__name__ for k, h in hs.items()},
           "img_per_s": ips, "img_per_s_median": med, "muon_over_sgd": round(med["muon_adamw"] / med["sgd"], 3)}
    del hs
    torch.cuda.empty_cache()
    return out


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    batch = int(sys.argv[3]) if len(sys.argv) > 3 else 128
    steps = int(sys.argv[4]) if len(sys.argv) > 4 else 6
    if not torch.cuda.is_available():
        raise SystemExit("muon_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for model in ("resnet50", "deit_s"):
        out[model] = time_optimizers(model, reps, rounds, dev)
    out["rn50_erk80_train_step"] = time_train_step("synthetic_rn50_erk80_muon", 0.2, batch, steps, rounds)
    out["deit_s_snip50_train_step"] = time_train_step("synthetic_deit_s_snip50_muon", 0.5, batch, steps, rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
