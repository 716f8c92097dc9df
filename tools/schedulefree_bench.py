#!/usr/bin/env python
"""Cost of the fused Schedule-Free SGD step and of its train / eval switch on the GPU.

    python tools/schedulefree_bench.py [reps=50] [rounds=5] [batch=512] [steps=12]

1. One optimizer step over ResNet-50's 161 parameters (25.6 M values) and DeiT-S's 152 (22.1 M): ``FusedScheduleFreeSGD``
   against the schedulefree package's foreach torch sequence (weight decay add, lerp, add, sub) on copies of the same
   tensors with fixed step scalars, alternating ``rounds`` times.  Each is timed with CUDA events as replays of a CUDA
   graph of one step (device time) and as eager calls back to back (host + device; the fused one includes ``sync_lr``).
   The fused step moves 20 B per value (read y, g, z; write y, z); GB/s and the share of the H100 SXM data-sheet
   3.35 TB/s are computed from that and the graph-replay time.
2. The eval() + train() pair: the fused swap (one launch each, 12 B per value) against one ``p.lerp_(z, w)`` per
   parameter, timed eagerly.
3. The ResNet-50 ERK-80 % train step (``PruningHarness.train_epoch``, synthetic ImageNet-shaped batches, bf16, captured
   and replayed) with scheduler_type ScheduleFree against SGD: one harness, the optimizer swapped every round (each
   round re-captures in an untimed epoch, then times an epoch of ``steps`` replays).

Prints one JSON line with the GPU name and power limit.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
STEP_BYTES, SWAP_BYTES = 20, 12


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


def _time(run, reps, e0, e1):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _med(v):
    return sorted(v)[len(v) // 2]


def time_optimizer(model, reps, rounds, dev):
    from turboprune_b200.grad_exchange import plan_buckets
    from turboprune_b200.optim import FusedScheduleFreeSGD
    shapes = param_list(model)
    g = torch.Generator(device=dev).manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(s, generator=g, device=dev) * 0.02) for s in shapes]
    numels = [p.numel() for p in params]
    (_, offs, total), = plan_buckets(numels, 1 << 62)
    flat = torch.randn(total, generator=g, device=dev) * 1e-3          # gradients: views into one buffer, as in training
    for p, o, n in zip(params, offs, numels):
        p.grad = flat[o:o + n].view_as(p)
    lr, momentum, wd = 1e-3, 0.9, 5e-4
    opt = FusedScheduleFreeSGD(params, lr=lr, momentum=momentum, weight_decay=wd, warmup_steps=0, capturable=True)
    opt.train()
    # the package's foreach sequence on copies (it adds the decay into the gradient; that drift does not change the time)
    ys = [p.detach().clone() for p in params]
    zs = [p.detach().clone() for p in params]
    gs = [p.grad.clone() for p in params]
    ckp1 = 0.01
    alpha_y = lr * (momentum * (1 - ckp1) - 1)

    def torch_step():
        torch._foreach_add_(gs, ys, alpha=wd)
        torch._foreach_lerp_(ys, zs, weight=ckp1)
        torch._foreach_add_(ys, gs, alpha=alpha_y)
        torch._foreach_sub_(zs, gs, alpha=lr)

    def fused_eager():
        opt.sync_lr()
        opt.step()

    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(3):                                   # state, pointer tables, allocator pools
            fused_eager()
            torch_step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graphs = {"fused": torch.cuda.CUDAGraph(), "torch_foreach": torch.cuda.CUDAGraph()}
    opt.sync_lr()
    with torch.cuda.graph(graphs["fused"]):
        opt.step()
    with torch.cuda.graph(graphs["torch_foreach"]):
        torch_step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    eager = {"fused": fused_eager, "torch_foreach": torch_step}
    res = {k: {"graph": [], "eager": []} for k in graphs}
    moms = {"fused": [], "torch_lerp_loop": []}
    zlist = [opt.state[p]["z"] for p in params]

    def fused_swap():
        opt.eval()
        opt.train()

    def torch_swap():
        with torch.no_grad():
            for p, z in zip(params, zlist):
                p.lerp_(z, 1 - 1 / momentum)
            for p, z in zip(params, zlist):
                p.lerp_(z, 1 - momentum)

    for _ in range(rounds):
        for name in graphs:
            res[name]["graph"].append(_time(graphs[name].replay, reps, e0, e1))
            res[name]["eager"].append(_time(eager[name], reps, e0, e1))
        moms["fused"].append(_time(fused_swap, reps, e0, e1))
        moms["torch_lerp_loop"].append(_time(torch_swap, reps, e0, e1))
    n = sum(numels)
    out = {"params": len(params), "values": n, "step_bytes": STEP_BYTES * n}
    for name, r in res.items():
        gm, em = _med(r["graph"]), _med(r["eager"])
        gbps = STEP_BYTES * n / (gm * 1e-3) / 1e9
        out[name] = {"graph_ms_median": round(gm, 4), "graph_ms_min": round(min(r["graph"]), 4),
                     "eager_ms_median": round(em, 4), "GBps_on_20B": round(gbps, 1),
                     "share_of_3.35TBps": round(gbps * 1e9 / HBM_BYTES_PER_S, 3)}
    out["torch_over_fused_graph"] = round(out["torch_foreach"]["graph_ms_median"] / out["fused"]["graph_ms_median"], 3)
    sw = {k: _med(v) / 2 for k, v in moms.items()}               # one switch = half of an eval() + train() pair
    out["swap"] = {"fused_ms_median": round(sw["fused"], 4), "torch_lerp_loop_ms_median": round(sw["torch_lerp_loop"], 4),
                   "fused_GBps_on_12B": round(SWAP_BYTES * n / (sw["fused"] * 1e-3) / 1e9, 1),
                   "launches": {"fused": 1, "torch_lerp_loop": len(params)}}
    del opt, graphs, params, flat, ys, zs, gs, zlist
    torch.cuda.empty_cache()
    return out


def time_train_step(batch, steps, rounds):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils import custom_models as cm
    from turboprune_b200.utils import pruning_utils as pu
    tmp = tempfile.mkdtemp(prefix="schedulefree_bench_")

    def cfg(name):
        return C.compose(name, [f"dataset_params.total_batch_size={batch}", f"dataset_params.synthetic_steps_per_epoch={steps}",
                                "experiment_params.distributed=false", f"experiment_params.base_dir={tmp}"],
                         os.path.join(ROOT, "conf_b200"))

    cfgs = {"schedulefree": cfg("synthetic_rn50_erk80_schedulefree"), "sgd": cfg("synthetic_rn50_erk80")}
    torch.manual_seed(0)
    model = cm.TorchVisionModel(cfgs["sgd"])
    torch.manual_seed(1)
    pu.prune_er_erk(model, 0.2)
    h = PruningHarness(cfg=cfgs["sgd"], gpu_id=0, expt_dir=("bench", tmp), model=model)
    opts, scheds = {}, {}
    for name, c in cfgs.items():
        h.cfg = c
        h._setup_optimizer()
        h._setup_scheduler(2 * rounds + 2)
        opts[name], scheds[name] = h.optimizer, h.scheduler
    ips = {k: [] for k in cfgs}
    losses = {k: [] for k in cfgs}
    for _ in range(rounds):
        for name in cfgs:
            h.cfg, h.optimizer, h.scheduler = cfgs[name], opts[name], scheds[name]
            h.train_epoch()                                  # re-captures for this optimizer (untimed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = h.train_epoch()
            torch.cuda.synchronize()
            ips[name].append(round(batch * steps / (time.perf_counter() - t0), 1))
            losses[name].append(round(out["train_loss"], 4))
    med = {k: _med(v) for k, v in ips.items()}
    return {"batch": batch, "steps_per_epoch": steps, "optimizer": {k: type(o).__name__ for k, o in opts.items()},
            "img_per_s": ips, "img_per_s_median": med, "train_loss": losses,
            "schedulefree_over_sgd": round(med["schedulefree"] / med["sgd"], 3)}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    batch = int(sys.argv[3]) if len(sys.argv) > 3 else 512
    steps = int(sys.argv[4]) if len(sys.argv) > 4 else 12
    if not torch.cuda.is_available():
        raise SystemExit("schedulefree_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for model in ("resnet50", "deit_s"):
        out[model] = time_optimizer(model, reps, rounds, dev)
    out["resnet50_erk80_train_step"] = time_train_step(batch, steps, rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
