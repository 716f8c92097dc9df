#!/usr/bin/env python
"""BASELINE.json configs 3, 4 and 5 through the product surface, measured (the headline bench.py line is config 2).

    python tools/config_bench.py [3] [4] [5] [rn50tail]          (1 GPU; under torchrun the level loop of config 3 is data parallel)

  3  ResNet-50 IMP + weight rewinding, 20 prune cycles (21 levels, target sparsity 0.988, rewind_epoch 0) through
     run_experiment.main on synthetic ImageNet-shaped batches: wall time per level, time of the prune step (global
     magnitude top-k over 25.5 M weights + rewind), final sparsity, replica checksums (N > 1).
  4  VGG-16 / CIFAR-100 shape, SynFlow one-shot to 95 % sparsity, B = 512: train-step images/s with and without
     K-block skipping, and the honest count of skippable 64x64 weight blocks.
  5  DeiT-small, SNIP to 50 % sparsity, per-GPU batch 64 (masked-Linear path): train-step images/s.
  rn50tail  ResNet-50 at the IMP tail (density 0.012, magnitude pruning of the seed-0 network): images/s with / without
     K-block skipping + skippable-block count.

One JSON line per config on stdout (rank 0).
"""
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist


def _harness(cfg, model, batch):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    cfg["dataset_params"]["total_batch_size"] = batch
    cfg["dataset_params"]["synthetic_steps_per_epoch"] = 4
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("cfgbench", tempfile.gettempdir()), model=model)
    h._setup_optimizer()
    h.model.train()
    return h


def _throughput(h, batch, steps=20, warmup=6):
    steps = int(os.environ.get("TP_CFG_STEPS", steps)); warmup = int(os.environ.get("TP_CFG_WARMUP", warmup))   # short runs under ncu
    it = iter(h.train_loader)
    b0 = next(it)
    for _ in range(warmup):
        h.train_step(b0)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        loss = h.train_step(b0)["loss"]
    b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    return {"ms_per_step": ms, "images_per_s": batch / ms * 1e3, "loss": float(loss.item()), "cuda_graph": h._graph is not None}


def _skip_compare(cfg, model, batch):
    """Train-step rate with the K-block skip on and off (separate harnesses: the capture bakes the choice in)."""
    import copy
    from turboprune_b200 import ops
    out = {}
    for on in (True, False):
        ops.set_kblock_skip(on)
        try:
            h = _harness(copy.deepcopy(cfg), copy.deepcopy(model), batch)
            out["skip_on" if on else "skip_off"] = _throughput(h, batch)
            if on:
                h._weight_stager().stage()
                rep = ops.skipped_block_report(h._weight_stager())
                h._drop_staged()
                out["weight_blocks_64x64"] = {"empty": rep["empty_blocks"], "total": rep["total_blocks"], "fraction": rep["fraction"],
                                              "worst_layers": sorted(((e / max(t, 1), n, list(s)) for n, s, e, t in rep["layers"]), reverse=True)[:4]}
            del h
            torch.cuda.empty_cache()
        finally:
            ops.set_kblock_skip(True)
    return out


def config4():
    import refshim
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    from turboprune_b200.utils.dataset import SyntheticLoader
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = refshim.make_cfg("vgg16", "cifar100", precision="bfloat16", prune_method="synflow")
    cfg["optimizer_params"].update(lr=0.05)
    torch.manual_seed(0)
    model = cm.TorchVisionModel(cfg).to(dev).train()
    loader = SyntheticLoader(512, 1, (3, 32, 32), 100, dev, seed=1)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    pu.prune_synflow(cfg, model, loader, 0.05)
    torch.cuda.synchronize(); t_prune = time.perf_counter() - t0
    res = {"config": "4: VGG-16 CIFAR-100-shape, SynFlow one-shot 95 % sparsity, B=512, bf16", "sparsity_percent": model.get_overall_sparsity(),
           "prune_synflow_s": t_prune, "prune_info": getattr(model, "_last_prune_info", None)}
    dens = {n: float(m.mask.mean()) for n, m in model._masked()}
    res["layer_density_min_max"] = [min(dens.values()), max(dens.values())]
    res.update(_skip_compare(cfg, model, 512))
    return res


def config5():
    """1 process: per-GPU batch 64 on one GPU.  Under torchrun: data parallel over all ranks (BASELINE.json config 5), SNIP
    scored on every rank's first batch, rank 0's masks imposed, gradient exchange over NVLink under the backward pass."""
    import refshim
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    from turboprune_b200.utils.dataset import SyntheticLoader
    world = int(os.environ.get("WORLD_SIZE", "1")); rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", torch.cuda.current_device())
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    cfg = refshim.make_cfg("local_deit_small_patch16_224", "imagenet", mask_layer_type="LinearMask", precision="bfloat16", prune_method="snip")
    cfg["optimizer_params"].update(lr=0.01)
    cfg["experiment_params"]["distributed"] = world > 1
    torch.manual_seed(0)
    model = cm.CustomModel(cfg).to(dev).train()
    loader = SyntheticLoader(64, 1, (3, 224, 224), 1000, dev, seed=1 + rank)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    pu.prune_snip(cfg, model, loader, 0.5)
    pu.sync_masks_from_rank0(model)
    torch.cuda.synchronize(); t_prune = time.perf_counter() - t0
    model.zero_grad(set_to_none=True)
    res = {"config": f"5: DeiT-small, SNIP 50 % sparsity, per-GPU batch 64, bf16 (masked Linear path), {world} GPU(s)",
           "sparsity_percent": model.get_overall_sparsity(), "prune_snip_s": t_prune}
    h = _harness(cfg, model, 64 * world)
    if world > 1:
        dist.barrier()
    r = _throughput(h, 64)
    if world > 1:
        ms = torch.tensor([r["ms_per_step"]], device=dev); dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        r["ms_per_step"] = float(ms.item()); r["images_per_s"] = 64 * world / r["ms_per_step"] * 1e3
        h.reducer.check_status()
    res.update(r)
    flops = 3 * 2 * 4.183e9                     # SURVEY.md §8(d): masked linears fwd 4.183 GMAC/img, x3 for fwd + dgrad + wgrad
    res["masked_linear_tflops"] = res["images_per_s"] * flops / 1e12
    if world > 1:
        dist.barrier()
    return res if rank == 0 else None


def rn50tail():
    import refshim
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = refshim.make_cfg("resnet50", "imagenet", precision="bfloat16")
    cfg["optimizer_params"].update(weight_decay=1e-4)
    torch.manual_seed(0)
    model = cm.TorchVisionModel(cfg).to(dev).train()
    pu.prune_mag(model, 0.012)                  # the density of IMP level 20 (0.8^20), one shot on the seed-0 network
    res = {"config": "ResNet-50 ImageNet-shape at the IMP-tail density 0.012 (global magnitude), B=256, bf16",
           "sparsity_percent": model.get_overall_sparsity()}
    res.update(_skip_compare(cfg, model, 256))
    return res


def config3():
    import run_experiment
    from turboprune_b200.utils import config as C
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    per_gpu = 64
    steps = 6
    base = tempfile.mkdtemp(prefix="tp_cfg3_") if rank == 0 else tempfile.gettempdir()
    cfg = C.compose("synthetic_rn50_erk80", [
        "pruning_params=imp_one_cycle", "pruning_params.target_sparsity=0.988", "pruning_params.training_type=wr",
        "+pruning_params.rewind_epoch=0", f"dataset_params.total_batch_size={per_gpu * world}",
        f"dataset_params.synthetic_steps_per_epoch={steps}", f"experiment_params.distributed={'true' if world > 1 else 'false'}",
        "optimizer_params.weight_decay=1e-4", f"experiment_params.base_dir={base}"], os.path.join(ROOT, "conf_b200"))
    marks = []
    real_prune = run_experiment.prune_the_model

    def timed_prune(**kw):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        real_prune(**kw)
        torch.cuda.synchronize(); marks.append(time.perf_counter() - t0)
    run_experiment.prune_the_model = timed_prune
    torch.cuda.synchronize() if torch.cuda.is_initialized() else None
    t0 = time.perf_counter()
    prefix, expt = run_experiment.main(cfg)
    total = time.perf_counter() - t0
    if rank != 0:
        return None
    import csv
    rows = list(csv.DictReader(open(os.path.join(expt, f"{prefix}_summary.csv"))))
    return {"config": f"3: ResNet-50 IMP + weight rewinding, 20 prune cycles (21 levels) on {world} GPU(s), synthetic ImageNet-shape, "
                      f"per-GPU batch {per_gpu}, {steps} steps/level",
            "levels": len(rows), "final_sparsity_percent": float(rows[-1]["Sparsity"]), "wall_s": total, "s_per_level": total / max(len(rows), 1),
            "prune_step_s_median": sorted(marks)[len(marks) // 2] if marks else None, "prune_steps": len(marks),
            "sparsity_by_level": [round(float(r["Sparsity"]), 3) for r in rows]}


def main():
    which = [a for a in sys.argv[1:]] or ["4", "5", "rn50tail", "3"]
    if "LOCAL_RANK" in os.environ:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    rank = int(os.environ.get("RANK", "0"))
    for w in which:
        fn = {"3": config3, "4": config4, "5": config5, "rn50tail": rn50tail}[w]
        if w not in ("3", "5") and rank != 0:
            continue
        res = fn()
        if res is not None:
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
