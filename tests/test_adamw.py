"""AdamW (``optimizer_params.optimizer_name: AdamW``): the configuration and the optimizer's interface on the CPU, and on an
H100 the fused kernel bit for bit against ``torch.optim.AdamW(foreach=True, capturable=True)`` at ResNet-50 and DeiT-S
extents, state-dict interchange in both directions, the harness's captured train step, RigL's state reset and the level
loop."""
import copy
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONF = os.path.join(ROOT, "conf_b200")
REF_CONF = os.path.join(ROOT, "tests", "golden", "reference_conf")
NEW_SYMBOLS = ("tp_adamw", "tp_rigl_apply_states")


# ---------------------------------------------------------------- CPU ------------------------------------------------------
def test_adamw_abi_symbols_declared_and_built():
    from turboprune_b200 import _cabi
    header = open(os.path.join(ROOT, "include", "turboprune_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _cabi.SIGNATURES, name
    lib = _cabi.load()                                     # every SIGNATURES entry resolves in the sm_90a library
    for name in NEW_SYMBOLS:
        assert getattr(lib, name) is not None
    assert lib.tp_abi_version() == 11


def _harness_optimizer(cfg):
    """The optimizer PruningHarness._setup_optimizer builds for ``cfg`` (CPU parameters: construction touches no GPU)."""
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    h = PruningHarness.__new__(PruningHarness)
    h.cfg = cfg
    h.model = torch.nn.Linear(4, 3)
    h._setup_optimizer()
    return h.optimizer


def test_config_selects_the_optimizer():
    from turboprune_b200.optim import FusedAdamW, FusedSGD
    from turboprune_b200.utils import config as C
    c = C.compose("synthetic_deit_s_snip50_adamw", [], CONF)
    assert c.model_params.model_name == "local_deit_small_patch16_224" and c.pruning_params.prune_method == "snip"
    assert c.pruning_params.target_sparsity == 0.5
    opt = _harness_optimizer(c)
    assert type(opt) is FusedAdamW
    g = opt.param_groups[0]
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"], g["capturable"]) == (5e-4, (0.9, 0.999), 1e-8, 0.05, True)
    # the reference's own tree: the name switches the optimizer; betas / eps default to torch's
    c = C.compose("cifar10_er_erk", ["optimizer_params.optimizer_name=AdamW", "optimizer_params.lr=1e-3",
                                     "optimizer_params.weight_decay=0.02"], REF_CONF)
    opt = _harness_optimizer(c)
    g = opt.param_groups[0]
    assert type(opt) is FusedAdamW
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"]) == (1e-3, (0.9, 0.999), 1e-8, 0.02)
    c = C.compose("cifar10_er_erk", ["optimizer_params.optimizer_name=AdamW", "+optimizer_params.betas=[0.8,0.99]",
                                     "+optimizer_params.eps=1e-6"], REF_CONF)
    assert _harness_optimizer(c).param_groups[0]["betas"] == (0.8, 0.99)
    assert _harness_optimizer(c).param_groups[0]["eps"] == 1e-6
    # SGD stays SGD: the shipped configs (no optimizer_name key), the reference's SGD configs, and any other name
    for name in ("synthetic_rn18_imp", "synthetic_rn18_rigl", "synthetic_rn50_erk80"):
        c = C.compose(name, [], CONF)
        assert "optimizer_name" not in c.optimizer_params
        opt = _harness_optimizer(c)
        assert type(opt) is FusedSGD and opt.param_groups[0]["momentum"] == 0.9
    for name in ("cifar10_er_erk", "imagenet_er_balanced"):
        assert type(_harness_optimizer(C.compose(name, [], REF_CONF))) is FusedSGD
    assert type(_harness_optimizer(C.compose("cifar10_er_erk", ["optimizer_params.optimizer_name=Muon"], REF_CONF))) is FusedSGD


def test_fused_adamw_interface_matches_torch():
    from turboprune_b200.optim import FusedAdamW
    ps = [torch.nn.Parameter(torch.zeros(3))]
    mine = FusedAdamW(ps, lr=1e-3, weight_decay=0.05, capturable=True)
    ref = torch.optim.AdamW(ps, lr=1e-3, weight_decay=0.05, capturable=True)
    assert set(mine.param_groups[0]) == set(ref.param_groups[0])
    assert {k: v for k, v in mine.param_groups[0].items() if k != "params"} == \
        {k: v for k, v in ref.param_groups[0].items() if k != "params"}
    assert hasattr(mine, "sync_lr")
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(differentiable=True), dict(lr=torch.tensor(1e-3)),
               dict(betas=(torch.tensor(0.9), 0.999)), dict(betas=(1.0, 0.999)), dict(lr=-1.0)):
        with pytest.raises(ValueError):
            FusedAdamW(ps, **kw)
    with pytest.raises(ValueError):
        FusedAdamW([torch.nn.Parameter(torch.zeros(3, dtype=torch.complex64))])


# ---------------------------------------------------------------- GPU ------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _param_list(model):
    if model == "resnet50":
        import torchvision
        with torch.device("meta"):
            net = torchvision.models.resnet50()
    else:
        from turboprune_b200.utils import vit
        with torch.device("meta"):
            net = vit.local_deit_small_patch16_224()
    return [(name, tuple(p.shape)) for name, p in net.named_parameters()]


def _init(named, g, dev):
    out = []
    for name, shape in named:
        if len(shape) > 1:
            v = torch.randn(shape, generator=g, device=dev) * (2.0 / math.prod(shape[1:])) ** 0.5
        elif name.endswith("weight"):
            v = 1 + 0.1 * torch.randn(shape, generator=g, device=dev)
        else:
            v = 0.1 * torch.randn(shape, generator=g, device=dev)
        out.append(v)
    return out


def _erk80(named, g, dev):
    """Bernoulli ERK masks at 80 % sparsity for every weight of two or more dimensions (None elsewhere)."""
    shapes = [s for _, s in named if len(s) > 1]
    fr = [sum(s) / math.prod(s) for s in shapes]
    c = 0.2 * sum(math.prod(s) for s in shapes) / sum(f * math.prod(s) for f, s in zip(fr, shapes))
    out = []
    for _, s in named:
        if len(s) > 1:
            p = min(1.0, c * sum(s) / math.prod(s))
            out.append((torch.rand(s, generator=g, device=dev) < p).float())
        else:
            out.append(None)
    return out


def _diff(what, a, r):
    bad = a.reshape(-1).view(torch.int32) != r.reshape(-1).view(torch.int32)
    if bool(bad.any()):
        j = int(bad.nonzero()[0])
        return (f"{what}: {int(bad.sum())} of {a.numel()} differ from torch.optim.AdamW, first at {j}: "
                f"fused {float(a.reshape(-1)[j])!r}, torch {float(r.reshape(-1)[j])!r}")
    return None


def _compare_adamw(opt, ropt, mine, ref, named, tag):
    for p, rp, (name, _) in zip(mine, ref, named):
        msg = _diff(f"{tag} {name} weight", p.detach(), rp.detach())
        assert msg is None, msg
        st, rst = opt.state.get(p, {}), ropt.state.get(rp, {})
        assert set(st) == set(rst), (tag, name, sorted(st), sorted(rst))
        for key in ("exp_avg", "exp_avg_sq", "step"):
            if key in st:
                assert st[key].device == p.device and st[key].dtype == torch.float32
                msg = _diff(f"{tag} {name} {key}", st[key], rst[key])
                assert msg is None, msg


ADAMW_VARIANTS = ["eager", "cuda-graph", "misaligned-grad", "late-param", "weight-decay-0", "masked", "large-step"]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ADAMW_VARIANTS)
@pytest.mark.parametrize("model", ["resnet50", "deit_s"])
def test_fused_adamw_bit_identical_to_torch(dev, model, variant):
    """FusedAdamW(capturable=True) against torch.optim.AdamW(foreach=True, capturable=True) on the same GPU, over
    ResNet-50's 161 parameters (25,557,032 values) and DeiT-S's 152 (22,050,664): weight, exp_avg, exp_avg_sq and step
    bit-identical after each of four steps, weight decay 0.05, the learning rate changed between steps through sync_lr.
    Gradients are views into one plan_buckets flat buffer (16-byte aligned slots: every full tile is vectorised).

    - cuda-graph: step 1 eager (uploads the table), then one captured step replayed for steps 2-4;
    - misaligned-grad: the largest gradient sits 4 bytes off 16-byte alignment (scalar path);
    - late-param: the largest parameter gets its first gradient at step 2 and starts at t = 1;
    - weight-decay-0: no decay multiply;
    - masked: gradients zero under ERK-80 masks: exp_avg and exp_avg_sq stay exactly 0 there, the weights only decay;
    - large-step: both optimizers loaded from one state dict with step = 10000 (pow far from t = 1)."""
    from turboprune_b200.grad_exchange import plan_buckets
    from turboprune_b200.optim import FusedAdamW
    named = _param_list(model)
    n_total = sum(math.prod(s) for _, s in named)
    assert (len(named), n_total) == ((161, 25_557_032) if model == "resnet50" else (152, 22_050_664))
    g = torch.Generator(device=dev).manual_seed(7)
    init = _init(named, g, dev)
    mine = [torch.nn.Parameter(v.clone()) for v in init]
    ref = [torch.nn.Parameter(v.clone()) for v in init]
    del init
    numels = [p.numel() for p in mine]
    (_, offs, total), = plan_buckets(numels, 1 << 62)
    flat = torch.zeros(total, device=dev)
    views = [flat[o:o + n].view_as(p) for o, n, p in zip(offs, numels, mine)]
    big = max(range(len(mine)), key=lambda i: numels[i])
    if variant == "misaligned-grad":
        spare = torch.zeros(numels[big] + 1, device=dev)
        views[big] = spare[1:].view_as(mine[big])
    for i, v in enumerate(views):
        assert v.data_ptr() % 16 == (4 if variant == "misaligned-grad" and i == big else 0), named[i][0]
    masks = _erk80(named, g, dev) if variant == "masked" else [None] * len(named)
    late = big if variant == "late-param" else None
    wd = 0.0 if variant == "weight-decay-0" else 0.05
    lrs = (1e-3, 8e-4, 6e-4, 4e-4)
    opt = FusedAdamW(mine, lr=lrs[0], betas=(0.9, 0.999), eps=1e-8, weight_decay=wd, capturable=True)
    ropt = torch.optim.AdamW(ref, lr=lrs[0], betas=(0.9, 0.999), eps=1e-8, weight_decay=wd, foreach=True, capturable=True)

    def grads(step):
        for i, (p, rp, v, m, (name, _)) in enumerate(zip(mine, ref, views, masks, named)):
            gv = torch.randn(v.shape, generator=g, device=dev) * (1e-2 if name.endswith("bias") else 3e-3)
            if m is not None:
                gv.mul_(m)
            if step == 0 and i == late:
                p.grad = rp.grad = None
                continue
            v.copy_(gv)
            p.grad, rp.grad = v, gv

    if variant == "large-step":
        # one step of torch's optimizer fills the state; both start from it with step = 10000
        grads(0)
        ropt.step()
        sd = ropt.state_dict()
        for st in sd["state"].values():
            st["step"].fill_(10000.0)
        with torch.no_grad():
            for p, rp in zip(mine, ref):
                p.copy_(rp)
        opt.load_state_dict(copy.deepcopy(sd))
        ropt.load_state_dict(copy.deepcopy(sd))
        _compare_adamw(opt, ropt, mine, ref, named, "loaded")
    graph = None
    for step in range(4):
        grads(step)
        for grp in opt.param_groups + ropt.param_groups:
            grp["lr"] = lrs[step]
        opt.sync_lr()
        if variant == "cuda-graph" and step >= 1:
            if graph is None:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    opt.step()
            graph.replay()
        else:
            opt.step()
        ropt.step()
        _compare_adamw(opt, ropt, mine, ref, named, f"{variant}, step {step + 1}")
        if variant == "late-param":
            assert (late in [i for i, p in enumerate(mine) if p in opt.state]) == (step >= 1)
            if step >= 1:
                assert float(opt.state[mine[late]]["step"]) == step
    want_step = 10004.0 if variant == "large-step" else 4.0
    assert float(opt.state[mine[0]]["step"]) == want_step
    if variant == "masked":
        n = 0
        for p, m in zip(mine, masks):
            if m is not None:
                off = m == 0
                assert float(opt.state[p]["exp_avg"][off].abs().sum()) == 0.0
                assert float(opt.state[p]["exp_avg_sq"][off].abs().sum()) == 0.0
                assert int((opt.state[p]["exp_avg_sq"][~off] == 0).sum()) == 0
                n += int(off.sum())
        assert n > 0.7 * n_total


@pytest.mark.gpu
def test_fused_adamw_many_steps_and_learning_rates(dev):
    """300 steps of a small parameter set (a vectorised 4096-value tile plus a scalar tail, and a 3-value bias) with a
    new learning rate at every step from a triangular schedule: every step count t = 1..300 meets a different lr, so the
    bias corrections and the division by lr are checked over many (t, lr) pairs, eagerly and through a replayed graph."""
    from turboprune_b200.optim import FusedAdamW
    named = [("w", (5, 4096 + 3)), ("bias", (3,))]
    g = torch.Generator(device=dev).manual_seed(5)
    init = _init(named, g, dev)
    for use_graph in (False, True):
        mine = [torch.nn.Parameter(v.clone()) for v in init]
        ref = [torch.nn.Parameter(v.clone()) for v in init]
        opt = FusedAdamW(mine, lr=1e-3, weight_decay=0.05, capturable=True)
        ropt = torch.optim.AdamW(ref, lr=1e-3, weight_decay=0.05, foreach=True, capturable=True)
        gs = [torch.zeros_like(p) for p in mine]
        for p, rp, gv in zip(mine, ref, gs):
            p.grad, rp.grad = gv, gv
        graph = None
        for step in range(300):
            for gv in gs:
                gv.copy_(torch.randn(gv.shape, generator=g, device=dev) * 3e-3)
            lr = 1e-3 * float(np.interp(step, [0, 60, 300], [0.2, 1.0, 0.0]))
            for grp in opt.param_groups + ropt.param_groups:
                grp["lr"] = lr
            opt.sync_lr()
            if use_graph and step >= 1:
                if graph is None:
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        opt.step()
                graph.replay()
            else:
                opt.step()
            ropt.step()
            _compare_adamw(opt, ropt, mine, ref, named, f"graph={use_graph} step {step + 1} lr {lr!r}")


@pytest.mark.gpu
def test_state_dict_interchange_both_ways(dev):
    """DeiT-S parameters: FusedAdamW's state dict loads into torch.optim.AdamW and torch's into FusedAdamW; after the
    swap both chains keep stepping bit-identically (each state tensor, including step, is the other's)."""
    from turboprune_b200.optim import FusedAdamW
    named = _param_list("deit_s")
    g = torch.Generator(device=dev).manual_seed(11)
    init = _init(named, g, dev)
    a = [torch.nn.Parameter(v.clone()) for v in init]             # FusedAdamW, then torch
    b = [torch.nn.Parameter(v.clone()) for v in init]             # torch, then FusedAdamW
    del init
    kw = dict(lr=5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.05, capturable=True)
    oa, ob = FusedAdamW(a, **kw), torch.optim.AdamW(b, foreach=True, **kw)
    for step in range(4):
        if step == 2:
            sa, sb = oa.state_dict(), ob.state_dict()
            assert set(sa["state"][0]) == set(sb["state"][0]) == {"step", "exp_avg", "exp_avg_sq"}
            assert set(sa["param_groups"][0]) == set(sb["param_groups"][0])
            oa = torch.optim.AdamW(a, foreach=True, **kw)
            oa.load_state_dict(copy.deepcopy(sa))
            ob = FusedAdamW(b, **kw)
            ob.load_state_dict(copy.deepcopy(sb))
            assert isinstance(oa, torch.optim.AdamW) and isinstance(ob, FusedAdamW)
        for pa, pb in zip(a, b):
            gv = torch.randn(pa.shape, generator=g, device=dev) * 3e-3
            pa.grad, pb.grad = gv, gv.clone()
        for grp in oa.param_groups + ob.param_groups:
            grp["lr"] = 5e-4 * (1 - 0.1 * step)
        for o in (oa, ob):
            if hasattr(o, "sync_lr"):
                o.sync_lr()
        oa.step()
        ob.step()
        fused, torch_opt, pf, pt = (oa, ob, a, b) if isinstance(oa, FusedAdamW) else (ob, oa, b, a)
        _compare_adamw(fused, torch_opt, pf, pt, named, f"step {step + 1}")


HARNESS_CASES = [("local_deit_small_patch16_224", "imagenet", "LinearMask", 8), ("resnet18", "cifar10", "ConvMask", 64)]


def _adamw_harness(case, tmp_path):
    from refshim import make_cfg, make_harness
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    model_name, data, mlt, batch = case
    cfg = make_cfg(model_name, data, mask_layer_type=mlt, precision="bfloat16")
    cfg["optimizer_params"].update(optimizer_name="AdamW", lr=1e-3, weight_decay=0.05)
    torch.manual_seed(0)
    model = cm.CustomModel(cfg) if mlt == "LinearMask" else cm.TorchVisionModel(cfg)
    torch.manual_seed(1)
    pu.prune_er_erk(model, 0.3)
    return make_harness(cfg, model, batch, str(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("case", HARNESS_CASES, ids=["deit_s.b8", "resnet18.b64"])
def test_harness_adamw_graph_step_matches_torch(dev, case, tmp_path):
    """bf16 PruningHarness.train_step with optimizer_name AdamW: six steps, the CUDA graph captured on the third and
    replayed on the fourth to sixth (the eager step body is not entered again), the learning rate changed before every
    step.  The same harness with its optimizer replaced by torch.optim.AdamW(foreach=True, capturable=True), which steps
    eagerly, ends every step with bit-identical parameters."""
    from turboprune_b200.optim import FusedAdamW
    model_name, data, _, batch = case
    h = _adamw_harness(case, tmp_path)
    assert isinstance(h.optimizer, FusedAdamW)
    h2 = _adamw_harness(case, tmp_path)
    h2.optimizer = torch.optim.AdamW(h2.model.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.05,
                                     foreach=True, capturable=True)
    assert not h2._graph_enabled() and h._graph_enabled()
    entered = []
    body = h._step_body
    h._step_body = lambda *a: (entered.append(1), body(*a))[1]
    size = 32 if data == "cifar10" else 224
    gen = torch.Generator().manual_seed(3)
    h.model.train(); h2.model.train()
    graph = None
    for step in range(6):
        x = torch.randn(batch, 3, size, size, generator=gen).cuda()
        t = torch.randint(0, 10, (batch,), generator=gen).cuda()
        for o in (h.optimizer, h2.optimizer):
            for grp in o.param_groups:
                grp["lr"] = 1e-3 * (1 - 0.1 * step)
        n_before = len(entered)
        h.train_step((x, t))
        h2.train_step((x, t))
        if step == 2:
            assert h._graph is not None, "the step is captured on the third call"
            graph = h._graph["graph"]
        if step >= 3:
            assert h._graph["graph"] is graph and len(entered) == n_before, "the captured step is replayed"
        torch.cuda.synchronize()
        for (name, p), p2 in zip(h.model.named_parameters(), h2.model.parameters()):
            msg = _diff(f"{model_name} step {step + 1} {name}", p.detach(), p2.detach())
            assert msg is None, msg
    assert h2._graph is None
    assert float(h.optimizer.state[next(h.model.parameters())]["step"]) == 6.0


def _rigl_adamw_harness(tmp_path):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.harness_utils import set_seed
    from turboprune_b200.utils.pruning_utils import prune_the_model
    cfg = C.compose("synthetic_rn18_rigl", ["optimizer_params=adamw_triangular", "dataset_params.total_batch_size=64",
                                            "dataset_params.synthetic_steps_per_epoch=15", "pruning_params.rigl_update_interval=3",
                                            f"experiment_params.base_dir={tmp_path}"], CONF)
    set_seed(cfg)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)))
    prune_the_model(cfg=cfg, harness=h, target_density=0.2)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)), model=h.model)
    h._setup_optimizer()
    h._setup_scheduler(1)
    h.begin_rigl_level(1)
    return h


@pytest.mark.gpu
def test_rigl_update_resets_adamw_state(dev, tmp_path):
    """synthetic_rn18_rigl with optimizer_params=adamw_triangular: after every update, grown positions have w = m = v = 0,
    every other element of every parameter and of its exp_avg / exp_avg_sq is bit-unchanged and no step count moved; the
    graph captured before the first update is replayed after the last.  A second harness runs the level through
    train_epoch."""
    from turboprune_b200.optim import FusedAdamW
    h = _rigl_adamw_harness(tmp_path)
    assert isinstance(h.optimizer, FusedAdamW) and h.rigl.update_batches() == [3, 6, 9]
    layers = h._masked_layers()
    lw = {id(m.weight) for m in layers}
    params = list(h.model.parameters())
    h.model.train()
    graph, updates, held = None, 0, 0
    for t, batch in enumerate(h.train_loader):
        is_update = h.rigl.is_update(t)
        if is_update:
            if graph is None:
                assert h._graph is not None
                graph = h._graph["graph"]
            old_mask = [m.mask.clone() for m in layers]
            before = [(p.detach().clone(), {k: v.clone() for k, v in h.optimizer.state[p].items()}) for p in params]
        h.train_step(batch)
        h.scheduler.step()
        if not is_update:
            continue
        updates += 1
        grown_of = {id(m.weight): (m.mask != 0) & (o == 0) for m, o in zip(layers, old_mask)}
        n_grown = 0
        for p, (w0, st0) in zip(params, before):
            st = h.optimizer.state[p]
            assert torch.equal(st["step"], st0["step"])
            keep = ~grown_of[id(p)] if id(p) in lw else torch.ones_like(p, dtype=torch.bool)
            for now, was in ((p.detach(), w0), (st["exp_avg"], st0["exp_avg"]), (st["exp_avg_sq"], st0["exp_avg_sq"])):
                assert torch.equal(now[keep].view(torch.int32), was[keep].view(torch.int32))
                if id(p) in lw:
                    assert float(now[~keep].abs().sum()) == 0.0
            n_grown += int((~keep).sum()) if id(p) in lw else 0
        assert n_grown > 0
        # grown positions that held state: weights dropped by an earlier update (their m, v only decay while masked)
        held += sum(int((st0["exp_avg_sq"][grown_of[id(p)]] != 0).sum()) for p, (_, st0) in zip(params, before) if id(p) in lw)
    assert updates == 3 and h._graph is not None and h._graph["graph"] is graph
    assert held > 0, "no update regrew a weight with non-zero optimizer state"

    h2 = _rigl_adamw_harness(tmp_path)
    out = h2.train_epoch()
    assert h2.rigl_step == 15 and h2.rigl_counts is not None and h2._graph is not None
    assert all(math.isfinite(float(v)) for v in out.values() if isinstance(v, (int, float)))


@pytest.mark.gpu
def test_run_experiment_deit_adamw_level(dev, tmp_path):
    """run_experiment.main on synthetic_deit_s_snip50_adamw (a few batches of 8) completes the level and writes an
    optimizer_init.pt that torch.optim.AdamW.load_state_dict accepts."""
    import run_experiment
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils import custom_models as cm
    cfg = C.compose("synthetic_deit_s_snip50_adamw", ["dataset_params.total_batch_size=8",
                                                      "dataset_params.synthetic_steps_per_epoch=4",
                                                      f"experiment_params.base_dir={tmp_path}"], CONF)
    prefix, expt = run_experiment.main(cfg)
    assert os.path.isfile(os.path.join(expt, "metrics", "level_wise_metrics", "level_0_metrics.csv"))
    sd = torch.load(os.path.join(expt, "artifacts", "optimizer_init.pt"), map_location="cpu")
    assert sd["param_groups"][0]["weight_decay"] == 0.05 and tuple(sd["param_groups"][0]["betas"]) == (0.9, 0.999)
    model = cm.CustomModel(cfg=cfg)
    ref = torch.optim.AdamW(model.parameters())
    ref.load_state_dict(sd)
    assert ref.param_groups[0]["lr"] == sd["param_groups"][0]["lr"]
