"""RigL dynamic sparse training (Evci et al. 2020): the schedule, the configuration, the numpy oracle of one update, and
on an H100 the select / apply kernels bit for bit against that oracle at ResNet-50 ERK-80 extents, the dense weight
gradient of the masked layers, and the harness and level loop training with drop-and-regrow updates."""
import math
import os

import numpy as np
import pytest
import torch

import rigl_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONF = os.path.join(ROOT, "conf_b200")
REF_CONF = os.path.join(ROOT, "tests", "golden", "reference_conf")


# ---------------------------------------------------------------- CPU: schedule and configuration ------------------------
def test_schedule_matches_hand_computed_values():
    from turboprune_b200.utils.rigl import RiglSchedule
    s = RiglSchedule(interval=3, drop_fraction=0.3, end_fraction=0.75, total_steps=20)     # T_end = floor(15.0) = 15
    assert s.t_end == 15
    assert s.update_batches() == [3, 6, 9, 12]
    assert not s.is_update(0) and not s.is_update(15) and not s.is_update(18) and not s.is_update(4)
    # f(t) = 0.15 (1 + cos(pi t / 15)); k = floor(f * n)
    assert s.fraction(0) == pytest.approx(0.3)
    assert s.fraction(3) == 0.3 / 2 * (1 + math.cos(math.pi * 3 / 15))
    assert s.k_per_layer(3, [1000, 7, 0]) == [271, 1, 0]           # f(3) = 0.27135...
    assert s.k_per_layer(6, [1000]) == [196]                        # f(6) = 0.19635...
    assert s.k_per_layer(9, [1000]) == [103]                        # f(9) = 0.10365...
    assert s.k_per_layer(12, [1000, 100]) == [28, 2]                # f(12) = 0.02865...
    s = RiglSchedule(interval=2, drop_fraction=0.5, end_fraction=0.5, total_steps=9)       # T_end = floor(4.5) = 4
    assert s.t_end == 4 and s.update_batches() == [2]
    assert s.k_per_layer(2, [10]) == [2]                            # f(2) = 0.25 (1 + cos(pi / 2)) = 0.25


def test_config_composition_and_overrides():
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.harness_utils import generate_densities
    from turboprune_b200.utils.rigl import RiglSchedule, rigl_params
    c = C.compose("synthetic_rn18_rigl", [], CONF)
    assert c.pruning_params.training_type == "rigl" and c.pruning_params.prune_method == "er_erk"
    assert rigl_params(c) == (100, 0.3, 0.75)
    assert generate_densities(c, 0.0) == [1 - 0.8]                  # one level, like at_init
    c = C.compose("synthetic_rn18_rigl", ["pruning_params.rigl_update_interval=7", "pruning_params.rigl_drop_fraction=0.5"], CONF)
    assert rigl_params(c) == (7, 0.5, 0.75)
    # the reference's own tree has no RigL keys: training_type switches it on, the rest are added with '+' or defaulted
    c = C.compose("cifar10_er_erk", ["pruning_params.training_type=rigl"], REF_CONF)
    assert rigl_params(c) == (100, 0.3, 0.75)
    c = C.compose("cifar10_er_erk", ["pruning_params.training_type=rigl", "+pruning_params.rigl_update_interval=50",
                                     "+pruning_params.rigl_end_fraction=0.5"], REF_CONF)
    assert rigl_params(c) == (50, 0.3, 0.5)
    assert RiglSchedule.from_cfg(c, 1000).update_batches() == list(range(50, 500, 50))
    c = C.compose("imagenet_er_balanced", ["pruning_params.training_type=rigl", "+pruning_params.rigl_drop_fraction=0.1"], REF_CONF)
    assert c.pruning_params.prune_method == "er_balanced" and rigl_params(c) == (100, 0.1, 0.75)
    assert rigl_params(C.compose("cifar10_er_erk", [], REF_CONF)) is None


def test_iterative_prune_method_is_refused():
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.rigl import rigl_params
    for method in ("mag", "random_erk", "random_balanced"):
        c = C.compose("synthetic_rn18_rigl", [f"pruning_params.prune_method={method}"], CONF)
        with pytest.raises(ValueError, match="one-shot"):
            rigl_params(c)
    c = C.compose("synthetic_rn18_imp", ["pruning_params.training_type=rigl"], CONF)
    with pytest.raises(ValueError):
        rigl_params(c)


def test_run_experiment_refuses_before_training(tmp_path):
    import run_experiment
    from turboprune_b200.utils import config as C
    c = C.compose("synthetic_rn18_imp", ["pruning_params.training_type=rigl", f"experiment_params.base_dir={tmp_path}"], CONF)
    with pytest.raises(ValueError):
        run_experiment.main(c)
    assert not os.listdir(tmp_path)                                 # nothing was written


def _check_counts(m, new, nd, ng, k):
    assert int((m != 0).sum()) == int((new != 0).sum())
    assert nd == ng == min(k, int((m != 0).sum()))


def test_oracle_on_tie_heavy_cases():
    n = 64
    idx = np.arange(n)
    m = (idx % 3 != 0).astype(np.float32)                          # 42 active
    # all-equal |w|: the lowest active indices are dropped; all-equal |g|: the lowest free indices are grown
    w = np.where(idx % 2 == 0, 0.5, -0.5).astype(np.float32)
    g = np.full(n, 2.0, np.float32)
    new, nd, ng = O.select(w, g, m, 5)
    drop = np.flatnonzero(m != 0)[:5]
    free = np.flatnonzero((m == 0) | np.isin(idx, drop))[:5]
    want = (m != 0) & ~np.isin(idx, drop) | np.isin(idx, free)
    assert np.array_equal(new, want.astype(np.float32)) and nd == ng == 5
    # zero gradients everywhere: the grow still takes k positions, lowest index first (dropped ones included)
    new, nd, ng = O.select(w, np.zeros(n, np.float32), m, 5)
    assert np.array_equal(new, want.astype(np.float32))
    # NaN: |w| = NaN is the largest key (dropped last), |g| = NaN the largest (grown first)
    w2 = np.linspace(1, 2, n).astype(np.float32)
    w2[1] = np.nan
    g2 = np.zeros(n, np.float32)
    g2[0] = -np.nan
    g2[3] = np.inf
    new, nd, ng = O.select(w2, g2, m, int((m != 0).sum()) - 1)
    assert new[1] == 1 and new[0] == 1 and new[3] == 1           # NaN weight kept; NaN and inf gradients grown first
    # k = 0: nothing moves
    new, nd, ng = O.select(w2, g2, m, 0)
    assert np.array_equal(new, m) and nd == ng == 0
    # k = n_active: every active weight is dropped, and the grow picks the k largest |g| over the whole layer
    gg = np.arange(n, dtype=np.float32)[::-1].copy()
    new, nd, ng = O.select(w, gg, m, 42)
    assert np.array_equal(new, (idx < 42).astype(np.float32)) and nd == ng == 42
    # a dense layer: the k weakest go, and come back where |g| is largest (here: where they were)
    md = np.ones(n, np.float32)
    new, nd, ng = O.select(np.arange(n, dtype=np.float32), np.arange(n, dtype=np.float32), md, 10)
    assert np.array_equal(new, md) and nd == ng == 10
    # apply: only positions that were 0 and are 1 now restart
    m0 = np.array([1, 0, 0, 1], np.float32)
    nm = np.array([0, 1, 0, 1], np.float32)
    mm, ww, bb = O.apply(m0, nm, np.array([1, 2, 3, 4], np.float32), np.array([5, 6, 7, 8], np.float32))
    assert mm.tolist() == [0, 1, 0, 1] and ww.tolist() == [1, 0, 3, 4] and bb.tolist() == [5, 0, 7, 8]
    for k in (0, 1, 7, 42, 100):
        new, nd, ng = O.select(w, g, m, k)
        _check_counts(m, new, nd, ng, k)


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


def _rn50_erk80_layers():
    """(weight shape, mask) of every masked layer of the ImageNet ResNet-50 with ERK masks at 80 % sparsity (CPU)."""
    import refshim
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    torch.manual_seed(0)
    model = cm.TorchVisionModel(refshim.make_cfg("resnet50", "imagenet"))
    pu.prune_er_erk(model, 0.2)
    return [m.mask.clone() for _, m in model._masked()]


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


@pytest.mark.gpu
def test_select_apply_bit_exact_at_resnet50_extents(dev):
    """All 54 masked layers of ResNet-50 ERK-80 (25.5 M weights) in one select + one apply: every mask element, every
    zeroed weight and momentum and every (dropped, grown) count equals the oracle.  Weights are quantised to a few
    hundred values and ~30 % of the gradients are exactly zero, so ties are everywhere; layer 0 has k = 0, layer 1
    k = n_active, the fc layer is dense, the largest 3x3 layer has one |w| value for all weights (its ties straddle
    hundreds of 4096-element tiles), layer 4 carries NaN and inf weights and gradients."""
    from turboprune_b200 import ops
    masks = _rn50_erk80_layers()
    assert len(masks) == 54 and abs(sum(m.numel() for m in masks) - 25.5e6) < 0.1e6
    masks[-1] = torch.ones_like(masks[-1])                          # a dense layer
    tie_layer = max(range(len(masks) - 1), key=lambda i: masks[i].numel())
    gen = torch.Generator().manual_seed(1)
    ws, gs, bufs = [], [], []
    for i, m in enumerate(masks):
        w = (torch.randint(-300, 301, m.shape, generator=gen).float() / 64)
        g = (torch.randint(-200, 201, m.shape, generator=gen).float() / 128)
        g[torch.rand(m.shape, generator=gen) < 0.3] = 0.0
        if i == tie_layer:
            w = torch.where(torch.rand(m.shape, generator=gen) < 0.5, 0.25, -0.25)
        if i == 4:
            w.view(-1)[::997] = float("nan"); w.view(-1)[5::1009] = float("inf")
            g.view(-1)[::1013] = float("nan"); g.view(-1)[7::1019] = float("-inf")
        ws.append(w); gs.append(g); bufs.append(torch.randn(m.shape, generator=gen))
    active = [int(m.sum()) for m in masks]
    ks = [int(math.floor(0.3 * a)) for a in active]
    ks[0] = 0
    ks[1] = active[1]
    assert ks[tie_layer] > 4 * 4096
    # oracle
    want = []
    for w, g, m, b, k in zip(ws, gs, masks, bufs, ks):
        new, nd, ng = O.select(w.numpy(), g.numpy(), m.numpy(), k)
        mm, ww, bb = O.apply(m.numpy(), new, w.numpy(), b.numpy())
        want.append((mm, ww, bb, nd, ng))
    d = lambda ts: [t.to(dev).contiguous() for t in ts]
    dws, dgs, dms, dbufs = d(ws), d(gs), d(masks), d(bufs)
    news = [torch.empty_like(m) for m in dms]
    counts = ops.rigl_select(dws, dgs, dms, news, ks)
    # the select leaves the masks alone
    for m, dm in zip(masks, dms):
        assert torch.equal(m, dm.cpu())
    ops.rigl_apply(dms, news, dws, dbufs)
    counts = counts.cpu().numpy()
    for i, (mm, ww, bb, nd, ng) in enumerate(want):
        assert np.array_equal(_bits(news[i]).reshape(-1), mm.view(np.int32)), f"layer {i}: new mask"
        assert np.array_equal(_bits(dms[i]).reshape(-1), mm.view(np.int32)), f"layer {i}: mask after apply"
        assert np.array_equal(_bits(dws[i]).reshape(-1), ww.view(np.int32)), f"layer {i}: weights"
        assert np.array_equal(_bits(dbufs[i]).reshape(-1), bb.view(np.int32)), f"layer {i}: momentum"
        assert (counts[i, 0], counts[i, 1]) == (nd, ng), (i, counts[i], nd, ng)
        assert int(dms[i].sum()) == active[i]
    assert counts[0].tolist() == [0, 0] and counts[1].tolist() == [active[1], active[1]]
    assert any(not torch.equal(m.to(dev), dm) for m, dm in zip(masks, dms))
    # the same call again on the same inputs is bit-identical (integer atomics only)
    news2 = [torch.empty_like(m) for m in dms]
    ops.rigl_select(dws, dgs, dms, news2, ks)
    ops.rigl_select(dws, dgs, dms, news, ks)
    assert all(torch.equal(a, b) for a, b in zip(news, news2))


# integer operands: every product and partial sum of the weight gradient is exact (see test_kernel_exactness.py)
DENSE_CASES = [
    # name, kind, n, hw, cin, cout, k, stride, pad
    ("conv3x3.s2", "conv", 32, 28, 128, 128, 3, 2, 1),
    ("conv1x1", "conv", 32, 14, 256, 128, 1, 1, 0),
    ("stem7x7.s2", "stem", 8, 224, 3, 64, 7, 2, 3),
    ("linear", "linear", 8 * 197, None, 384, 1152, 1, 1, 0),
]


def _dense_case(dev, case, dense, precision):
    from turboprune_b200 import ops
    from turboprune_b200.utils.mask_layers import ConvMask, LinearMask
    name, kind, n, hw, cin, cout, k, st, pad = case
    g = torch.Generator(device=dev).manual_seed(cin + cout + n)
    ints = lambda shape: torch.randint(-1, 2, shape, generator=g, device=dev).float()
    if kind == "linear":
        layer = LinearMask(in_features=cin, out_features=cout, bias=True).to(dev)
    else:
        layer = ConvMask(in_channels=cin, out_channels=cout, kernel_size=k, stride=st, padding=pad, bias=False).to(dev)
    with torch.no_grad():
        layer.weight.copy_(torch.randint(0, 2, layer.weight.shape, generator=g, device=dev).float() * 2 - 1)
    m = (torch.rand(layer.weight.shape, generator=g, device=dev) < 0.3).float()
    if kind == "conv":
        m[:64] = 0                                                  # a dead row group: the occupancy mask skips its dW tiles
    layer.mask = m
    x = ints((8, 197, cin) if kind == "linear" else (n, cin, hw, hw))
    if kind == "conv":
        x = x.contiguous(memory_format=torch.channels_last).requires_grad_(True)
    ctx = ops.compute_precision(precision)
    with ctx, ops.dense_weight_grad(dense):
        xin = x if precision == torch.float32 or kind == "stem" else x.detach().to(torch.bfloat16).requires_grad_(x.requires_grad)
        y = layer(xin)
        dy = ints(tuple(y.shape)).to(y.dtype)
        if kind != "linear":
            dy = dy.contiguous(memory_format=torch.channels_last)
        y.backward(dy)
    # exact float64 weight gradient
    x64, dy64 = x.detach().double(), dy.double()
    if kind == "linear":
        dw64 = (dy64.reshape(-1, cout).t() @ x64.reshape(-1, cin))
    else:
        from torch.nn.grad import conv2d_weight
        dw64 = conv2d_weight(x64, layer.weight.shape, dy64, st, pad)
    return layer.weight.grad.detach().clone(), m, dw64


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("case", DENSE_CASES, ids=[c[0] for c in DENSE_CASES])
def test_dense_weight_gradient(dev, case, precision):
    """Inside ``dense_weight_grad()``: at kept positions dW equals the normal masked gradient bit for bit, at pruned
    positions it equals float64 (the operands keep every partial sum exact)."""
    masked, m, _ = _dense_case(dev, case, False, precision)
    dense, m2, dw64 = _dense_case(dev, case, True, precision)
    assert torch.equal(m, m2)
    keep, pruned = m != 0, m == 0
    assert float(masked[pruned].abs().max()) == 0.0
    assert torch.equal(dense[keep].view(torch.int32), masked[keep].view(torch.int32)), "kept positions differ"
    want = torch.round(dw64)[pruned].float()
    assert torch.equal(dense[pruned], want), f"pruned positions: {int((dense[pruned] != want).sum())} differ"
    assert int((want != 0).sum()) > want.numel() // 4                # the check is not about zeros


def _rigl_cfg(tmp_path, overrides=()):
    from turboprune_b200.utils import config as C
    return C.compose("synthetic_rn18_rigl", ["dataset_params.total_batch_size=64", "dataset_params.synthetic_steps_per_epoch=15",
                                             "pruning_params.rigl_update_interval=3", f"experiment_params.base_dir={tmp_path}",
                                             *overrides], CONF)


def _rigl_harness(cfg, tmp_path):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.utils.harness_utils import set_seed
    from turboprune_b200.utils.pruning_utils import prune_the_model
    set_seed(cfg)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)))
    prune_the_model(cfg=cfg, harness=h, target_density=0.2)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)), model=h.model)
    h._setup_optimizer()
    h._setup_scheduler(1)
    h.begin_rigl_level(1)
    return h


@pytest.mark.gpu
def test_harness_rigl_level(dev, tmp_path):
    """ResNet-18 CIFAR shape, ERK 80 %, dT = 3 over 15 batches (updates at t = 3, 6, 9): per-layer active counts stay
    constant, masks change, grown weights and momenta are 0 right after an update, the CUDA graph captured before the
    first update is the one replayed after the last, ``mask_epoch()`` never moves, and a run without CUDA graphs ends with
    bit-identical weights and masks."""
    from turboprune_b200.utils import mask_layers
    cfg = _rigl_cfg(tmp_path)
    h = _rigl_harness(cfg, tmp_path)
    assert h.rigl.update_batches() == [3, 6, 9]
    layers = h._masked_layers()
    active = [int(m.mask.sum()) for m in layers]
    assert active == h.rigl_active
    epoch0 = mask_layers.mask_epoch()
    h.model.train()
    graph, updates = None, 0
    for t, batch in enumerate(h.train_loader):
        is_update = h.rigl.is_update(t)
        if is_update:
            old = [m.mask.clone() for m in layers]
            if graph is None:
                assert h._graph is not None, "the step is captured before the first update"
                graph = h._graph["graph"]
        h.train_step(batch)
        h.scheduler.step()
        if is_update:
            updates += 1
            changed = 0
            for m, o, a in zip(layers, old, active):
                assert int(m.mask.sum()) == a
                grown = (m.mask != 0) & (o == 0)
                changed += int(grown.sum())
                assert float(m.weight.detach()[grown].abs().sum()) == 0.0
                buf = h.optimizer.state[m.weight]["momentum_buffer"]
                assert float(buf[grown].abs().sum()) == 0.0
            counts = h.rigl_counts.cpu()
            assert torch.equal(counts[:, 0], counts[:, 1])
            assert changed > 0 and int(counts[:, 1].sum()) >= changed
        assert mask_layers.mask_epoch() == epoch0
    assert updates == 3 and h.rigl_step == 15
    assert h._graph is not None and h._graph["graph"] is graph        # captured once, replayed across all updates
    torch.cuda.synchronize()
    w1 = [p.detach().clone() for p in h.model.parameters()]
    m1 = [m.mask.clone() for m in layers]
    # the same level without CUDA graphs
    cfg2 = _rigl_cfg(tmp_path, ["experiment_params.cuda_graph=false"]) if hasattr(cfg.experiment_params, "cuda_graph") else \
        _rigl_cfg(tmp_path, ["+experiment_params.cuda_graph=false"])
    h2 = _rigl_harness(cfg2, tmp_path)
    h2.train_epoch()
    assert h2._graph is None and h2.rigl_step == 15
    for a, b in zip(w1, h2.model.parameters()):
        assert torch.equal(a.view(torch.int32), b.detach().view(torch.int32))
    for a, m in zip(m1, h2._masked_layers()):
        assert torch.equal(a, m.mask)


@pytest.mark.gpu
def test_run_experiment_rigl_level(dev, tmp_path):
    """run_experiment.main with synthetic_rn18_rigl trains one level with updates and writes the level CSV and
    model_level_0.pt, whose masks keep the ERK per-layer counts."""
    import run_experiment
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    cfg = C.compose("synthetic_rn18_rigl", ["dataset_params.total_batch_size=64", "dataset_params.synthetic_steps_per_epoch=8",
                                            "pruning_params.rigl_update_interval=2", f"experiment_params.base_dir={tmp_path}"], CONF)
    prefix, expt = run_experiment.main(cfg)
    assert os.path.isfile(os.path.join(expt, "metrics", "level_wise_metrics", "level_0_metrics.csv"))
    sd = torch.load(os.path.join(expt, "checkpoints", "model_level_0.pt"), map_location="cpu")
    init = torch.load(os.path.join(expt, "checkpoints", "model_init.pt"), map_location="cpu")
    # model_init.pt holds the ERK masks the level started from: per layer, Bernoulli draws at the ERK densities
    ref = cm.TorchVisionModel(cfg=cfg)
    _, fracs = pu._erk_fracs([m for _, m in ref._masked()], 0.2)
    names = [n + ".mask" for n, _ in ref._masked()]
    for name, p in zip(names, fracs):
        n, kept, p = init[name].numel(), int(init[name].sum()), float(p)
        assert abs(kept - p * n) <= 6 * math.sqrt(n * p * (1 - p)) + 1, (name, kept, p * n)
    got = {k: int(sd[k].sum()) for k in names}
    assert got == {k: int(init[k].sum()) for k in names}             # RigL moved weights, never changed a layer's count
    changed = sum(int((sd[k] != init[k]).sum()) for k in names)
    assert changed > 0, "no mask changed during the level"


@pytest.mark.gpu
def test_rigl_two_ranks_stay_identical(dev, tmp_path):
    """torchrun on 2 GPUs, ImageNet-shaped ResNet-18 with RigL updates at t = 1, 2: every rank selects on its own dense
    gradient, rank 0's masks are imposed in place, and the per-level replica checksum holds.  Skipped on one GPU."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = 29700 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "run_experiment.py"), "--config-name=synthetic_rn50_erk80",
           f"--config-path={CONF}", "model_params=resnet18_convmask", "pruning_params=rigl_erk_80",
           "pruning_params.rigl_update_interval=1", "dataset_params.total_batch_size=32",
           "dataset_params.synthetic_steps_per_epoch=5", f"experiment_params.base_dir={tmp_path}"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
