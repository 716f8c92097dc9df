#!/usr/bin/env python
"""Level loop — drop-in for the reference's ``run_experiment.py`` (:21-133) on the H100 hot path.

    python run_experiment.py --config-name=cifar10_er_erk [--config-path=/path/to/TurboPrune/conf] group.key=value ...
    torchrun --nproc_per_node=N run_experiment.py --config-name=imagenet_er_balanced ...

Differences from the reference, all on purpose: the Hydra CLI is a small composer (hydra is not installed);
pruning runs on every rank and rank 0's masks are then broadcast once (packed, 102 MB for ResNet-50) — the
reference prunes on rank 0 and lets the next DDP constructor broadcast all 204 MB of state, and DDP re-broadcasts
every buffer on every forward; a per-level replica checksum guards the invariant; wandb logging is not part of the
path.  Checkpoint files, names and formats are the reference's.
"""
import os
import sys

import torch
import torch.distributed as dist

from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
from turboprune_b200.utils import config as tp_config
from turboprune_b200.utils.harness_utils import gen_expt_dir, generate_densities, save_config, save_model, set_seed
from turboprune_b200.utils.pruning_utils import prune_the_model
from turboprune_b200.utils.rigl import rigl_params


def check_replicas(model, what):
    """Data-parallel invariant: weights and masks are bit-identical on every rank (same seed, bit-identical gradient
    mean, deterministic kernels; masks imposed from rank 0 after pruning).  One checksum per rank and level — the
    cheap stand-in for DDP's per-forward buffer broadcast, which hid such divergence upstream."""
    with torch.no_grad():
        parts = [p.detach().double().sum() for p in model.parameters()]
        parts += [m.mask.double().sum() for _, m in model._masked()]
        mine = torch.stack(parts).sum().reshape(1)
    allv = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
    dist.all_gather(allv, mine)
    if not all(torch.equal(allv[0], v) for v in allv):
        raise RuntimeError(f"replicas diverged ({what}): checksums {[float(v) for v in allv]}")


def main(cfg):
    launched = "LOCAL_RANK" in os.environ or "RANK" in os.environ
    cifar = cfg.dataset_params.dataset_name.lower().startswith("cifar")
    if launched and cifar:
        if int(os.environ.get("LOCAL_RANK", 0)) == 0:
            print("CIFAR datasets do not support distributed training. Please run without torchrun/distributed launch.")
        sys.exit(1)                                           # reference run_experiment.py:25-37
    use_distributed = cfg.experiment_params.distributed and not cifar and launched
    rigl_params(cfg)                                          # a RigL config needs a one-shot initial mask: fail before training
    set_seed(cfg)
    if use_distributed:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
        dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
        rank, world = dist.get_rank(), dist.get_world_size()
    else:
        rank, world = 0, 1
    packaged = None
    if rank == 0:
        print(f"Training on {world} GPUs")
        packaged = gen_expt_dir(cfg)
        save_config(packaged[1], cfg)
    if use_distributed:
        box = [packaged]
        dist.broadcast_object_list(box, src=0)
        packaged = box[0]
    harness = PruningHarness(cfg=cfg, gpu_id=rank, expt_dir=packaged)
    model = harness.model
    at_init = cfg.pruning_params.training_type in ("at_init", "rigl")     # RigL: the one-shot mask at level 0, one level
    densities = generate_densities(cfg=cfg, current_sparsity=model.get_overall_sparsity())
    ckpt = os.path.join(packaged[1], "checkpoints")
    for level, density in enumerate(densities):
        if level == 0:
            if at_init:
                prune_the_model(cfg=cfg, harness=harness, target_density=density)
            elif rank == 0:
                save_model(model, os.path.join(ckpt, "model_init.pt"))
        elif not at_init:
            if use_distributed:
                dist.barrier()                                # rank 0 finished writing model_level_{level-1}.pt
            model.load_model(os.path.join(ckpt, f"model_level_{level - 1}.pt"))
            prune_the_model(cfg=cfg, harness=harness, target_density=density)
            model.reset_weights(cfg=cfg, expt_dir=packaged[1])
        if rank == 0:
            print(f"Model Sparsity check: {model.get_overall_sparsity():.2f}%")
        harness = PruningHarness(cfg=cfg, model=model, expt_dir=packaged, gpu_id=rank)
        harness.train_one_level(epochs_per_level=cfg.experiment_params.epochs_per_level, level=level)
        if use_distributed:
            check_replicas(harness.model, f"after level {level}")
        if rank == 0:
            save_model(harness.model, os.path.join(ckpt, f"model_level_{level}.pt"))
            print(f"Training level {level} complete, moving on to {level + 1}")
    if use_distributed:
        dist.barrier()
        dist.destroy_process_group()
    return packaged


if __name__ == "__main__":
    name, conf_dir, overrides = tp_config.parse_cli()
    here = os.path.dirname(os.path.abspath(__file__))
    conf_dir = conf_dir or os.environ.get("TURBOPRUNE_CONF") or (os.path.join(here, "conf") if os.path.isdir(os.path.join(here, "conf")) else os.path.join(here, "conf_b200"))
    main(tp_config.compose(name, overrides, conf_dir))
