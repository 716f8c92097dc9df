"""Schedule-Free SGD (``optimizer_params.scheduler_type: ScheduleFree``): the configuration, the host schedule and the
optimizer's interface on the CPU, and on an H100 the fused step and the train / eval switch bit for bit against a torch
restatement of the schedulefree package's SGDScheduleFree (tests/schedulefree_oracle.py), the harness's captured train
step, RigL's state reset and the level loop."""
import copy
import math
import os
import re

import numpy as np
import pytest
import torch

from schedulefree_oracle import SGDScheduleFreeReference, schedule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONF = os.path.join(ROOT, "conf_b200")
REF_CONF = os.path.join(ROOT, "tests", "golden", "reference_conf")
NEW_SYMBOLS = ("tp_schedulefree_sgd", "tp_schedulefree_swap")
GROUP_KEYS = {"params", "lr", "momentum", "weight_decay", "warmup_steps", "r", "weight_lr_power", "k", "weight_sum",
              "lr_max", "scheduled_lr", "train_mode", "foreach"}


# ---------------------------------------------------------------- CPU ------------------------------------------------------
def test_schedulefree_abi_symbols_declared_and_built():
    from turboprune_b200 import _cabi
    header = open(os.path.join(ROOT, "include", "turboprune_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _cabi.SIGNATURES, name
    lib = _cabi.load()
    for name in NEW_SYMBOLS:
        assert getattr(lib, name) is not None
    assert lib.tp_abi_version() == 11


def _harness(cfg):
    """PruningHarness._setup_optimizer and _setup_scheduler for ``cfg`` (CPU parameters: construction touches no GPU)."""
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    h = PruningHarness.__new__(PruningHarness)
    h.cfg = cfg
    h.model = torch.nn.Linear(4, 3)
    h._setup_optimizer()
    return h


def test_config_selects_schedulefree():
    from turboprune_b200.optim import FusedAdamW, FusedScheduleFreeSGD, FusedSGD
    from turboprune_b200.utils import config as C
    c = C.compose("synthetic_rn50_erk80_schedulefree", [], CONF)
    assert c.model_params.model_name == "resnet50" and c.pruning_params.target_sparsity == 0.8
    h = _harness(c)
    h._setup_scheduler(1)
    assert type(h.optimizer) is FusedScheduleFreeSGD and h.scheduler is None and h.optimizer.capturable
    g = h.optimizer.param_groups[0]
    assert (g["lr"], g["momentum"], g["weight_decay"], g["warmup_steps"]) == (1.0, 0.9, 5e-4, 50)
    # the reference's tree: ScheduleFree builds SGDScheduleFree whatever optimizer_name says, with its lr / momentum / wd
    for name in ("SGD", "AdamW", "MuonAdamW"):
        c = C.compose("cifar10_er_erk", ["optimizer_params.scheduler_type=ScheduleFree", "+optimizer_params.warmup_steps=7",
                                         f"optimizer_params.optimizer_name={name}"], REF_CONF)
        h = _harness(c)
        h._setup_scheduler(1)
        g = h.optimizer.param_groups[0]
        assert type(h.optimizer) is FusedScheduleFreeSGD and h.scheduler is None, name
        o = c.optimizer_params
        assert (g["lr"], g["momentum"], g["weight_decay"], g["warmup_steps"]) == (o.lr, o.momentum, o.weight_decay, 7)
        assert (g["r"], g["weight_lr_power"], g["k"], g["train_mode"]) == (0.0, 2.0, 0, False)
    # the reference's configs have no warmup_steps: the error names the key
    c = C.compose("cifar10_er_erk", ["optimizer_params.scheduler_type=ScheduleFree"], REF_CONF)
    with pytest.raises(ValueError, match=r"optimizer_params\.warmup_steps"):
        _harness(c)
    # every other config builds what it built before
    for name in ("synthetic_rn18_imp", "synthetic_rn18_rigl", "synthetic_rn50_erk80"):
        assert type(_harness(C.compose(name, [], CONF)).optimizer) is FusedSGD
    assert type(_harness(C.compose("synthetic_deit_s_snip50_adamw", [], CONF)).optimizer) is FusedAdamW
    for name in ("cifar10_er_erk", "imagenet_er_balanced"):
        assert type(_harness(C.compose(name, [], REF_CONF)).optimizer) is FusedSGD


SCHEDULES = [dict(warmup_steps=w, r=r, weight_lr_power=p) for w in (0, 1, 7) for r in (0.0, 0.5) for p in (2.0, 1.0)]


@pytest.mark.parametrize("kw", SCHEDULES, ids=lambda kw: "w{warmup_steps}-r{r}-p{weight_lr_power}".format(**kw))
@pytest.mark.parametrize("lr", [0.5, 0.0])
def test_host_schedule_matches_the_restatement(kw, lr):
    """k = 0 .. 10,000 through sync_lr (capturable): the group's k, weight_sum, lr_max and scheduled_lr equal the
    restatement's after every update, and the three fp32 device scalars it fills are np.float32 of the restatement's
    doubles.  The lr changes at k = 5000; lr = 0 takes the ckp1 = 0 branch."""
    from turboprune_b200.optim import FusedScheduleFreeSGD
    opt = FusedScheduleFreeSGD([torch.nn.Parameter(torch.zeros(3))], lr=lr, momentum=0.9, capturable=True, **kw)
    ref = dict(opt.param_groups[0], params=None)
    g = opt.param_groups[0]
    t = torch.empty(3, dtype=torch.float32)
    for k in range(10001):
        if k == 5000:
            g["lr"] = ref["lr"] = lr * 0.3
        opt.sync_lr()
        want = schedule(ref)
        for key in ("k", "weight_sum", "lr_max", "scheduled_lr"):
            assert g[key] == ref[key], (k, key, g[key], ref[key])
        opt._fill(0, t)
        assert np.array_equal(t.numpy().view(np.int32), np.array([np.float32(v) for v in want]).view(np.int32)), (k, want)
    assert g["k"] == 10001
    if lr == 0.0:
        assert g["weight_sum"] == 0.0 and t[1].item() == 0.0


def test_state_dict_keys_and_round_trip():
    from turboprune_b200.optim import FusedScheduleFreeSGD
    ps = [torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(3))]
    kw = dict(lr=0.3, momentum=0.85, weight_decay=1e-4, warmup_steps=5)
    mine, ref = FusedScheduleFreeSGD(ps, capturable=True, **kw), SGDScheduleFreeReference(ps, **kw)
    assert set(mine.param_groups[0]) == set(ref.param_groups[0]) == GROUP_KEYS
    assert {k: v for k, v in mine.param_groups[0].items() if k != "params"} == \
        {k: v for k, v in ref.param_groups[0].items() if k != "params"}
    for _ in range(9):
        mine.sync_lr()
    for p in ps:
        mine.state[p]["z"] = p.detach() * 2
    sd = mine.state_dict()
    assert set(sd["state"][0]) == {"z"} and set(sd["param_groups"][0]) == GROUP_KEYS
    fresh = FusedScheduleFreeSGD(ps, capturable=True, **kw)
    fresh.load_state_dict(copy.deepcopy(sd))
    for key in GROUP_KEYS - {"params"}:
        assert fresh.param_groups[0][key] == mine.param_groups[0][key], key
    assert fresh.param_groups[0]["k"] == 9
    for p in ps:
        assert torch.equal(fresh.state[p]["z"], mine.state[p]["z"])
    ref.load_state_dict(copy.deepcopy(sd))                      # the restatement takes the same layout
    assert ref.param_groups[0]["k"] == 9


def test_interface_and_refusals():
    from turboprune_b200.optim import FusedScheduleFreeSGD
    ps = [torch.nn.Parameter(torch.zeros(3))]
    for kw in (dict(momentum=0.0), dict(momentum=1.0), dict(momentum=-0.5), dict(lr=-1.0), dict(weight_decay=-1e-4),
               dict(lr=torch.tensor(1.0)), dict(momentum=torch.tensor(0.9)), dict(weight_decay=torch.tensor(0.0))):
        with pytest.raises(ValueError):
            FusedScheduleFreeSGD(ps, **kw)
    for dtype in (torch.complex64, torch.float64, torch.bfloat16):
        with pytest.raises(ValueError):
            FusedScheduleFreeSGD([torch.nn.Parameter(torch.zeros(3, dtype=dtype))])
    opt = FusedScheduleFreeSGD(ps, capturable=True)
    assert opt.param_groups[0]["train_mode"] is False
    with pytest.raises(RuntimeError, match="train mode"):
        opt.step()
    opt.eval()                                                  # no-ops: already in eval mode, and no z yet
    opt.train()
    opt.train()
    assert opt.param_groups[0]["train_mode"] is True and torch.equal(ps[0].detach(), torch.zeros(3))
    with pytest.raises(RuntimeError, match="sync_lr"):
        opt.step()
    with pytest.raises(NotImplementedError):
        opt.step(lambda: 0.0)
    plain = FusedScheduleFreeSGD(ps)
    plain.sync_lr()                                             # without capturable, step() advances the schedule
    assert plain.param_groups[0]["k"] == 0


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


def _diff(what, a, r):
    bad = a.reshape(-1).view(torch.int32) != r.reshape(-1).view(torch.int32)
    if bool(bad.any()):
        j = int(bad.nonzero()[0])
        return (f"{what}: {int(bad.sum())} of {a.numel()} differ from the restatement, first at {j}: "
                f"fused {float(a.reshape(-1)[j])!r}, torch {float(r.reshape(-1)[j])!r}")
    return None


def _compare(opt, ropt, mine, ref, names, tag):
    for p, rp, name in zip(mine, ref, names):
        msg = _diff(f"{tag} {name} y", p.detach(), rp.detach())
        assert msg is None, msg
        st, rst = opt.state.get(p, {}), ropt.state.get(rp, {})
        assert set(st) == set(rst), (tag, name, sorted(st), sorted(rst))
        if "z" in st:
            msg = _diff(f"{tag} {name} z", st["z"], rst["z"])
            assert msg is None, msg
    for key in ("k", "weight_sum", "lr_max", "scheduled_lr", "train_mode"):
        assert opt.param_groups[0][key] == ropt.param_groups[0][key], (tag, key)


STEP_VARIANTS = ["eager", "eager-capturable", "cuda-graph", "misaligned-grad", "late-param", "late-param-graph"]


@pytest.mark.gpu
@pytest.mark.parametrize("wd", [5e-4, 0.0])
@pytest.mark.parametrize("variant", STEP_VARIANTS)
@pytest.mark.parametrize("model", ["resnet50", "deit_s"])
def test_fused_step_bit_identical_to_the_restatement(dev, model, variant, wd):
    """FusedScheduleFreeSGD against the torch restatement on the same GPU, over ResNet-50's 161 parameters and DeiT-S's
    152: y and z bit-identical after each of five steps with warmup_steps = 2 (the step scalars change every step across
    the warm-up, then only through ckp1), the lr changed before the fifth step.

    - eager: capturable=False, step() advances the schedule; eager-capturable: sync_lr() then step();
    - cuda-graph: step 1 eager, one step captured and replayed for steps 2-5;
    - misaligned-grad: the largest gradient sits 4 bytes off 16-byte alignment (scalar path);
    - late-param: the largest parameter gets its first gradient at step 3 (z created from y in a launch of its own);
      late-param-graph: the same, step 4 eager over every parameter (it uploads the pointer table), step 5 captured and
      replayed."""
    from turboprune_b200.optim import FusedScheduleFreeSGD
    named = _param_list(model)
    assert len(named) == (161 if model == "resnet50" else 152)
    names = [n for n, _ in named]
    g = torch.Generator(device=dev).manual_seed(7)
    init = _init(named, g, dev)
    mine = [torch.nn.Parameter(v.clone()) for v in init]
    ref = [torch.nn.Parameter(v.clone()) for v in init]
    del init
    big = max(range(len(mine)), key=lambda i: mine[i].numel())
    grads = [torch.zeros_like(p) for p in mine]
    if variant == "misaligned-grad":
        grads[big] = torch.zeros(mine[big].numel() + 1, device=dev)[1:].view_as(mine[big])
        assert grads[big].data_ptr() % 16 == 4
    late = big if variant.startswith("late-param") else None
    capture_at = {"cuda-graph": 1, "late-param-graph": 4}.get(variant)
    kw = dict(lr=0.5, momentum=0.9, weight_decay=wd, warmup_steps=2)
    opt = FusedScheduleFreeSGD(mine, capturable=variant != "eager", **kw)
    ropt = SGDScheduleFreeReference(ref, **kw)
    opt.train()
    ropt.train()
    graph = None
    for step in range(5):
        for i, (p, rp, gv, name) in enumerate(zip(mine, ref, grads, names)):
            if i == late and step < 2:
                p.grad = rp.grad = None
                continue
            gv.copy_(torch.randn(gv.shape, generator=g, device=dev) * (1e-2 if name.endswith("bias") else 3e-3))
            p.grad, rp.grad = gv, gv.clone()
        if step == 4:
            opt.param_groups[0]["lr"] = ropt.param_groups[0]["lr"] = 0.35
        opt.sync_lr()
        if capture_at is not None and step >= capture_at:
            if graph is None:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    opt.step()
            graph.replay()
        else:
            opt.step()
        ropt.step()
        _compare(opt, ropt, mine, ref, names, f"{variant}, step {step + 1}")
        if late is not None:
            assert ("z" in opt.state[mine[late]]) == (step >= 2)
    assert opt.param_groups[0]["k"] == 5


@pytest.mark.gpu
@pytest.mark.parametrize("momentum", [0.9, 0.95])
@pytest.mark.parametrize("model", ["resnet50", "deit_s"])
def test_train_eval_switch_equals_per_tensor_lerp(dev, model, momentum):
    """eval() and train() against the restatement's per-tensor ``p.lerp_(z, w)``, every bit: both are no-ops before the
    first step, a repeated call is a no-op, and only parameters with a z move (one never has a gradient)."""
    from turboprune_b200.optim import FusedScheduleFreeSGD
    named = _param_list(model)
    names = [n for n, _ in named]
    g = torch.Generator(device=dev).manual_seed(3)
    init = _init(named, g, dev)
    mine = [torch.nn.Parameter(v.clone()) for v in init]
    ref = [torch.nn.Parameter(v.clone()) for v in init]
    kw = dict(lr=0.5, momentum=momentum, weight_decay=5e-4, warmup_steps=1)
    opt, ropt = FusedScheduleFreeSGD(mine, capturable=True, **kw), SGDScheduleFreeReference(ref, **kw)
    for o in (opt, ropt):
        o.eval(); o.train(); o.eval(); o.train()
    _compare(opt, ropt, mine, ref, names, "before the first step")
    for p, v in zip(mine, init):
        assert torch.equal(p.detach(), v)
    for step in range(3):
        for i, (p, rp) in enumerate(zip(mine, ref)):
            if i == 0:
                continue
            gv = torch.randn(p.shape, generator=g, device=dev) * 3e-3
            p.grad, rp.grad = gv, gv.clone()
        opt.sync_lr()
        opt.step()
        ropt.step()
    assert "z" not in opt.state[mine[0]]
    for what in ("eval", "eval again", "train", "train again", "eval"):
        getattr(opt, what.split()[0])()
        getattr(ropt, what.split()[0])()
        _compare(opt, ropt, mine, ref, names, what)
    assert torch.equal(mine[0].detach(), init[0])


def _sf_harness(tmp_path, lr=0.2):
    from refshim import make_cfg, make_harness
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    cfg = make_cfg("resnet18", "cifar10", mask_layer_type="ConvMask", precision="bfloat16")
    cfg["optimizer_params"].update(scheduler_type="ScheduleFree", lr=lr, momentum=0.9, weight_decay=5e-4, warmup_steps=3)
    torch.manual_seed(0)
    model = cm.TorchVisionModel(cfg)
    torch.manual_seed(1)
    pu.prune_er_erk(model, 0.3)
    return make_harness(cfg, model, 64, str(tmp_path))


@pytest.mark.gpu
def test_harness_train_step_matches_the_restatement(dev, tmp_path):
    """bf16 ResNet-18 PruningHarness.train_step with ScheduleFree: eight steps (eager, side-stream warm-up, capture, then
    replays; warm-up over three steps), test() after the fifth.  The same harness with the restatement as its optimizer
    and cuda_graph false ends every step, and the test(), with bit-identical parameters; both groups count eight updates."""
    from turboprune_b200.optim import FusedScheduleFreeSGD
    h = _sf_harness(tmp_path)
    h2 = _sf_harness(tmp_path)
    assert isinstance(h.optimizer, FusedScheduleFreeSGD)
    o = h2.cfg.optimizer_params
    h2.optimizer = SGDScheduleFreeReference(h2.model.parameters(), lr=o.lr, momentum=o.momentum,
                                            weight_decay=o.weight_decay, warmup_steps=o.warmup_steps)
    h2.cfg.experiment_params["cuda_graph"] = False
    assert h._graph_enabled() and not h2._graph_enabled()
    entered = []
    body = h._step_body
    h._step_body = lambda *a: (entered.append(1), body(*a))[1]
    gen = torch.Generator().manual_seed(3)
    graph = None

    def same(tag):
        torch.cuda.synchronize()
        for (name, p), p2 in zip(h.model.named_parameters(), h2.model.parameters()):
            msg = _diff(f"{tag} {name}", p.detach(), p2.detach())
            assert msg is None, msg

    for step in range(8):
        h.model.train(); h2.model.train()
        x = torch.randn(64, 3, 32, 32, generator=gen).cuda()
        t = torch.randint(0, 10, (64,), generator=gen).cuda()
        n_before = len(entered)
        h.train_step((x, t))
        h2.train_step((x, t))
        assert h.optimizer.param_groups[0]["train_mode"] and h2.optimizer.param_groups[0]["train_mode"]
        if step == 2:
            assert h._graph is not None
            graph = h._graph["graph"]
        if step >= 3:
            assert h._graph["graph"] is graph and len(entered) == n_before, "the captured step is replayed"
        same(f"step {step + 1}")
        if step == 4:
            h.test(); h2.test()
            assert not h.optimizer.param_groups[0]["train_mode"]
            same("test() after step 5")
    assert h.optimizer.param_groups[0]["k"] == h2.optimizer.param_groups[0]["k"] == 8


def _rigl_sf_harness(tmp_path):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.harness_utils import set_seed
    from turboprune_b200.utils.pruning_utils import prune_the_model
    cfg = C.compose("synthetic_rn18_rigl", ["optimizer_params=schedulefree_sgd", "optimizer_params.lr=0.2",
                                            "dataset_params.total_batch_size=64", "dataset_params.synthetic_steps_per_epoch=12",
                                            "pruning_params.rigl_update_interval=3", f"experiment_params.base_dir={tmp_path}"],
                    CONF)
    set_seed(cfg)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)))
    prune_the_model(cfg=cfg, harness=h, target_density=0.2)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)), model=h.model)
    h._setup_optimizer()
    h._setup_scheduler(1)
    h.begin_rigl_level(1)
    return h


@pytest.mark.gpu
def test_rigl_update_restarts_y_and_z(dev, tmp_path):
    """synthetic_rn18_rigl with optimizer_params=schedulefree_sgd: after every update, grown positions have y = z = 0,
    every other element of every parameter and of its z is bit-unchanged, k did not move, and the graph captured before
    the first update is replayed after the last."""
    from turboprune_b200.optim import FusedScheduleFreeSGD
    h = _rigl_sf_harness(tmp_path)
    assert isinstance(h.optimizer, FusedScheduleFreeSGD) and h.scheduler is None
    layers = h._masked_layers()
    lw = {id(m.weight) for m in layers}
    params = list(h.model.parameters())
    h.model.train()
    graph, updates, steps = None, 0, 0
    for t, batch in enumerate(h.train_loader):
        is_update = h.rigl.is_update(t)
        if is_update:
            if graph is None:
                assert h._graph is not None
                graph = h._graph["graph"]
            old_mask = [m.mask.clone() for m in layers]
            before = [(p.detach().clone(), h.optimizer.state[p]["z"].clone()) for p in params]
            k0 = h.optimizer.param_groups[0]["k"]
        h.train_step(batch)
        if not is_update:
            steps += 1
            continue
        updates += 1
        assert h.optimizer.param_groups[0]["k"] == k0
        grown_of = {id(m.weight): (m.mask != 0) & (o == 0) for m, o in zip(layers, old_mask)}
        n_grown = 0
        for p, (y0, z0) in zip(params, before):
            keep = ~grown_of[id(p)] if id(p) in lw else torch.ones_like(p, dtype=torch.bool)
            for now, was in ((p.detach(), y0), (h.optimizer.state[p]["z"], z0)):
                assert torch.equal(now[keep].view(torch.int32), was[keep].view(torch.int32))
                if id(p) in lw:
                    assert float(now[~keep].abs().sum()) == 0.0
            n_grown += int((~keep).sum()) if id(p) in lw else 0
        assert n_grown > 0
    assert updates >= 2 and h._graph is not None and h._graph["graph"] is graph
    assert h.optimizer.param_groups[0]["k"] == steps


@pytest.mark.gpu
def test_run_experiment_two_levels_evaluate_and_save_x(dev, tmp_path, monkeypatch):
    """run_experiment.main on synthetic_rn18_imp with optimizer_params=schedulefree_sgd, two levels: every test() runs
    in eval mode at x = lerp(y, z, 1 - 1 / momentum) (per-tensor torch lerp_ of the weights test() was entered with),
    model_level_0.pt holds the x of level 0's last test(), and optimizer_init.pt loads into a fresh optimizer."""
    import run_experiment
    from turboprune_b200.harness_definitions.base_harness import BaseHarness
    from turboprune_b200.optim import FusedScheduleFreeSGD
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils import custom_models as cm
    from turboprune_b200.utils.harness_utils import unwrap
    cfg = C.compose("synthetic_rn18_imp", ["optimizer_params=schedulefree_sgd", "optimizer_params.lr=0.2",
                                           "dataset_params.total_batch_size=64", "dataset_params.synthetic_steps_per_epoch=4",
                                           f"experiment_params.base_dir={tmp_path}"], CONF)
    seen = []
    test = BaseHarness.test

    def checked_test(self):
        opt = self.optimizer
        assert isinstance(opt, FusedScheduleFreeSGD) and opt.param_groups[0]["train_mode"]
        m = opt.param_groups[0]["momentum"]
        want = {}
        for name, p in self.model.named_parameters():
            x = p.detach().clone()
            if "z" in opt.state[p]:
                x.lerp_(opt.state[p]["z"], 1 - 1 / m)
            want[name] = x
        modes = []
        step = self.test_step
        self.test_step = lambda b: (modes.append(opt.param_groups[0]["train_mode"]), step(b))[1]
        try:
            out = test(self)
        finally:
            del self.test_step
        assert modes and not any(modes), "test() ran in train mode"
        for name, p in self.model.named_parameters():
            msg = _diff(f"x of {name}", p.detach(), want[name])
            assert msg is None, msg
        seen.append({k: v.cpu() for k, v in unwrap(self.model).state_dict().items()})
        return out

    monkeypatch.setattr(BaseHarness, "test", checked_test)
    prefix, expt = run_experiment.main(cfg)
    assert len(seen) == 2, "one test() per level"
    saved = torch.load(os.path.join(expt, "checkpoints", "model_level_0.pt"), map_location="cpu")
    assert set(saved) == set(seen[0])
    for k, v in seen[0].items():
        assert torch.equal(saved[k], v), k
    sd = torch.load(os.path.join(expt, "artifacts", "optimizer_init.pt"), map_location="cpu")
    assert sd["param_groups"][0]["k"] == 0 and sd["param_groups"][0]["warmup_steps"] == 50
    model = cm.TorchVisionModel(cfg)
    fresh = FusedScheduleFreeSGD(model.parameters(), lr=0.1, momentum=0.5)
    fresh.load_state_dict(sd)
    assert fresh.param_groups[0]["lr"] == 0.2 and fresh.param_groups[0]["momentum"] == 0.9


@pytest.mark.gpu
def test_schedulefree_two_ranks_stay_identical(dev, tmp_path):
    """torchrun on 2 GPUs, synthetic_rn50_erk80_schedulefree with ResNet-18: the replicas' x (after test()) stay
    bit-identical (the per-level replica checksum).  Skipped on one GPU."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = 29800 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "run_experiment.py"),
           "--config-name=synthetic_rn50_erk80_schedulefree", f"--config-path={CONF}", "model_params=resnet18_convmask",
           "optimizer_params.lr=0.2", "dataset_params.total_batch_size=32", "dataset_params.synthetic_steps_per_epoch=5",
           f"experiment_params.base_dir={tmp_path}"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
