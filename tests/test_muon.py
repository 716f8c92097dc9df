"""Muon (``optimizer_params.optimizer_name: MuonAdamW``): the configuration, the group split and the plan on the CPU; on an
H100 the Newton-Schulz GEMM bit for bit against float64 on exact operands, the prepare / normalize / apply kernels
against torch's ops, the whole step against ``torch.optim.Muon`` + ``torch.optim.AdamW`` at ResNet-50 and DeiT-S extents,
the harness's captured step, RigL's state reset and the level loop."""
import math
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONF = os.path.join(ROOT, "conf_b200")
NEW_SYMBOLS = ("tp_muon_workspace_bytes", "tp_muon_prepare", "tp_muon_normalize", "tp_muon_ns_gemm", "tp_muon_apply")
MODELS = {"resnet18": ("resnet18", "cifar10", "ConvMask", 10), "resnet50": ("resnet50", "imagenet", "ConvMask", 1000),
          "vgg16": ("vgg16", "cifar100", "ConvMask", 100),
          "deit_s": ("local_deit_small_patch16_224", "imagenet", "LinearMask", 1000)}


# ---------------------------------------------------------------- CPU ------------------------------------------------------
def test_muon_abi_symbols_declared_and_built():
    from turboprune_b200 import _cabi
    header = open(os.path.join(ROOT, "include", "turboprune_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _cabi.SIGNATURES, name
    lib = _cabi.load()
    for name in NEW_SYMBOLS:
        assert getattr(lib, name) is not None
    assert lib.tp_abi_version() == 11
    assert lib.tp_muon_workspace_bytes(3) >= 3 * __import__("ctypes").sizeof(_cabi.MuonLayer)


def _model(key):
    from refshim import make_cfg
    from turboprune_b200.utils import custom_models as cm
    name, data, mlt, _ = MODELS[key]
    cfg = make_cfg(name, data, mask_layer_type=mlt, precision="bfloat16")
    cfg["optimizer_params"].update(optimizer_name="MuonAdamW", lr=5e-4, momentum=0.95, weight_decay=0.05)
    torch.manual_seed(0)
    return cfg, (cm.CustomModel(cfg) if mlt == "LinearMask" else cm.TorchVisionModel(cfg))


def _harness_optimizer(cfg, model, num_classes):
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    h = PruningHarness.__new__(PruningHarness)
    h.cfg, h.model, h.num_classes = cfg, model, num_classes
    h._setup_optimizer()
    return h.optimizer


@pytest.mark.parametrize("key", sorted(MODELS))
def test_muon_adamw_group_split(key):
    """Every masked weight but the classifier's is in the Muon group; the classifier, biases, norms and (DeiT-S) the
    unmasked patch embedding are in the AdamW group."""
    from turboprune_b200.optim import FusedMuon
    from turboprune_b200.utils.mask_layers import MASKED_LAYER_TYPES
    cfg, model = _model(key)
    opt = _harness_optimizer(cfg, model, MODELS[key][3])
    assert type(opt) is FusedMuon and len(opt.param_groups) == 2
    muon, adamw = opt.param_groups
    assert muon["use_muon"] and not adamw["use_muon"]
    masked = [m for m in model.modules() if isinstance(m, MASKED_LAYER_TYPES)]
    assert [id(p) for p in muon["params"]] == [id(m.weight) for m in masked[:-1]]
    assert masked[-1].weight.shape[0] == MODELS[key][3]
    assert any(p is masked[-1].weight for p in adamw["params"])
    ids = {id(p) for g in opt.param_groups for p in g["params"]}
    assert ids == {id(p) for p in model.parameters()} and len(muon["params"]) + len(adamw["params"]) == len(ids)
    assert (muon["lr"], muon["weight_decay"], muon["momentum"], muon["nesterov"], muon["ns_steps"],
            muon["adjust_lr_fn"]) == (5e-4, 0.05, 0.95, True, 5, "match_rms_adamw")
    assert (adamw["lr"], adamw["weight_decay"], adamw["betas"], adamw["eps"]) == (5e-4, 0.05, (0.9, 0.999), 1e-8)
    adamw_ids = {id(p) for p in adamw["params"]}
    emb = [p for n, p in model.named_parameters() if "patch_embed" in n]
    assert (len(emb) > 0) == (key == "deit_s") and all(id(p) in adamw_ids for p in emb)


def test_muon_configs_and_the_name_muon_stays_sgd():
    from turboprune_b200.optim import FusedSGD
    from turboprune_b200.utils import config as C
    for name, model in (("synthetic_deit_s_snip50_muon", "local_deit_small_patch16_224"),
                        ("synthetic_rn50_erk80_muon", "resnet50")):
        c = C.compose(name, [], CONF)
        o = c.optimizer_params
        assert c.model_params.model_name == model
        assert (o.optimizer_name, o.lr, o.weight_decay, o.momentum, o.scheduler_type) == \
            ("MuonAdamW", 5e-4, 0.05, 0.95, "TriangularSchedule")
    cfg, model = _model("resnet18")
    cfg["optimizer_params"]["optimizer_name"] = "Muon"
    assert type(_harness_optimizer(cfg, model, 10)) is FusedSGD


def test_muon_plan_shapes_tiles_and_ratios():
    from torch.optim._muon import _adjust_lr
    from turboprune_b200 import ops
    shapes = [(64, 147), (64, 27), (384, 768), (1536, 384), (2048, 512), (2048, 1024), (4096, 25088)]
    plan = ops.MuonPlan(shapes)
    assert plan.trans == [False, True, False, True, True, True, False]
    assert plan.mp == [64, 64, 384, 384, 512, 1024, 4096]
    assert plan.np == [192, 64, 768, 1536, 2048, 2048, 25088]
    assert plan.tile0[0] == 0 and plan.n_tiles == sum(m * n // 4096 for m, n in zip(plan.mp, plan.np))
    for (mode, src), t in plan.gemm_tiles.items():
        tm = [m // 64 for m in plan.mp]
        want = sum(k * (k + 1) // 2 for k in tm) if mode != ops.MUON_UPDATE else plan.n_tiles
        assert t.shape == (want, 8), (mode, src)
        assert list(t[:, 4]) == sorted(t[:, 4], reverse=True)          # longest K first
        assert t[:, :2].min() >= 0 and (t[:, :2] + (t[:, 4:5] - 1) * t[:, 2:4] + 64).max() <= plan.rows
    for fn in (None, "original", "match_rms_adamw"):
        for (a, b), r in zip(shapes, plan.ratios(fn)):
            assert 1e-3 * r == _adjust_lr(1e-3, fn, torch.Size((a, b)))


def test_fused_muon_interface_matches_torch():
    from turboprune_b200.optim import FusedMuon
    ps = [torch.nn.Parameter(torch.zeros(4, 3))]
    mine, ref = FusedMuon(ps), torch.optim.Muon(ps)
    g = mine.param_groups[0]
    assert set(g) - {"use_muon"} == set(ref.param_groups[0]) and g["use_muon"]
    assert {k: v for k, v in g.items() if k not in ("params", "use_muon")} == \
        {k: v for k, v in ref.param_groups[0].items() if k != "params"}
    assert hasattr(mine, "sync_lr")
    FusedMuon([torch.nn.Parameter(torch.zeros(4, 3, 3, 3))])                       # ndim >= 2 is accepted
    mixed = FusedMuon([dict(params=ps), dict(params=[torch.nn.Parameter(torch.zeros(3))], use_muon=False)], lr=0.1)
    aw = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(3))], lr=0.1, weight_decay=0.1)
    assert set(mixed.param_groups[1]) - {"use_muon"} == set(aw.param_groups[0])
    assert (mixed.param_groups[1]["eps"], mixed.param_groups[1]["betas"]) == (1e-8, (0.9, 0.999))
    for kw, pat in ((dict(lr=-1.0), "Learning rate"), (dict(momentum=-0.1), "momentum"), (dict(weight_decay=-1.0), "weight decay"),
                    (dict(adjust_lr_fn="bogus"), "not supported")):
        with pytest.raises(ValueError, match=pat):
            FusedMuon(ps, **kw)
        with pytest.raises(ValueError, match=pat):
            torch.optim.Muon(ps, **kw)
    with pytest.raises(ValueError, match="less than 100"):
        FusedMuon(ps, ns_steps=100)
    one = [torch.nn.Parameter(torch.zeros(3))]
    for kw in (dict(lr=-1.0), dict(eps=-1.0), dict(weight_decay=-1.0), dict(betas=(1.0, 0.999)), dict(amsgrad=True),
               dict(maximize=True), dict(differentiable=True), dict(lr=torch.tensor(1e-3))):
        with pytest.raises(ValueError):                    # an AdamW group is held to FusedAdamW's checks
            FusedMuon([dict(params=ps), dict(params=one, use_muon=False, **kw)])
    with pytest.raises(ValueError, match="2D parameters"):
        FusedMuon([torch.nn.Parameter(torch.zeros(3))])
    with pytest.raises(ValueError, match="2D parameters"):
        torch.optim.Muon([torch.nn.Parameter(torch.zeros(3))])


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


def _panel(xws, row0, mp, np_):
    """[mp][np] view of the panel-layout matrix at workspace row row0."""
    return xws.view(-1, 64)[row0:row0 + mp * np_ // 64].view(np_ // 64, mp, 64).permute(1, 0, 2).reshape(mp, np_)


def _put(xws, row0, m):
    mp, np_ = m.shape
    xws.view(-1, 64)[row0:row0 + mp * np_ // 64] = m.reshape(mp, np_ // 64, 64).permute(1, 0, 2).reshape(-1, 64)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


# one 2-D Muon shape per distinct (mp, np, transposed) of the four models' Muon groups (test_exact_shapes_cover_the_models
# pins the list to the models): the stems 64 x 27 (CIFAR, transposed) and 64 x 147 (ResNet-50), ResNet-50's 1x1
# expansions (transposed), m = 1024, DeiT-S's qkv (transposed), proj, fc1 (transposed) and fc2, VGG-16's 4096 x 4096 and
# 4096 x 25088 classifier layers (K = 25088: 392 K blocks per gram tile)
EXACT_SHAPES = [(64, 64), (64, 27), (128, 64), (64, 147), (64, 256), (256, 64), (64, 576), (128, 256), (256, 128),
                (128, 512), (512, 128), (128, 576), (128, 1152), (256, 512), (512, 256), (256, 1024), (1024, 256),
                (256, 1152), (256, 2304), (384, 384), (1152, 384), (384, 1536), (1536, 384), (512, 1024), (1024, 512),
                (512, 2048), (2048, 512), (512, 2304), (512, 4608), (2048, 1024), (4096, 4096), (4096, 25088)]


def _padded_keys(shapes):
    from turboprune_b200 import ops
    plan = ops.MuonPlan(shapes)
    return set(zip(plan.mp, plan.np, plan.trans))


def test_exact_shapes_cover_the_models():
    """EXACT_SHAPES holds exactly one shape per distinct padded (mp, np, transposed) of the Muon groups the harness builds
    for ResNet-18 (CIFAR), ResNet-50, VGG-16 (CIFAR) and DeiT-S."""
    keys = set()
    for key in MODELS:
        cfg, model = _model(key)
        opt = _harness_optimizer(cfg, model, MODELS[key][3])
        keys |= _padded_keys([(p.shape[0], p.numel() // p.shape[0]) for p in opt.param_groups[0]["params"]])
    assert _padded_keys(EXACT_SHAPES) == keys and len(EXACT_SHAPES) == len(keys)


def _exact_bound(a, b):
    """Largest sum of |products| of a @ b.T (float64): below 2^24 every fp32 partial sum of the GEMM is exact."""
    return float((a.abs() @ b.abs().T).max())


@pytest.mark.gpu
def test_ns_gemm_modes_exact_on_integer_operands(dev):
    """GRAM, POLY and UPDATE over one tile list covering every shape at once, on integer operands whose fp32 partial sums
    are exact (asserted first), with dyadic alpha / beta: each output equals float64 rounded once to bf16, bit for bit;
    G and H are exactly symmetric and their padding is zero."""
    from turboprune_b200 import ops
    plan = ops.MuonPlan(EXACT_SHAPES)
    xws = torch.full((plan.rows * 64,), float("nan"), dtype=torch.bfloat16, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    tiles = {k: torch.from_numpy(v).to(dev) for k, v in plan.gemm_tiles.items()}

    def sym(mp, m, lim):
        g = torch.zeros(mp, mp, dtype=torch.float64, device=dev)
        s = torch.randint(-lim, lim + 1, (m, m), generator=gen, device=dev).double()
        g[:m, :m] = torch.triu(s) + torch.triu(s, 1).T
        return g

    X, Gs, Hs = [], [], []
    for l, (a, b) in enumerate(plan.shapes):
        m, n, mp, np_ = min(a, b), max(a, b), plan.mp[l], plan.np[l]
        x = torch.zeros(mp, np_, dtype=torch.float64, device=dev)
        x[:m, :n] = torch.randint(-2, 3, (m, n), generator=gen, device=dev).double()
        g = sym(mp, m, 8)
        assert _exact_bound(x, x) < 2 ** 24 and 0.5 * _exact_bound(g, g) + 16 < 2 ** 24
        _put(xws, plan.x[l][0], x.bfloat16())
        _put(xws, plan.g[l], g.bfloat16())
        X.append(x); Gs.append(g)
    # POLY (G is the random symmetric matrix), then GRAM (overwrites G)
    ops.muon_ns_gemm(ops.MUON_POLY, xws, tiles[(ops.MUON_POLY, 0)], 0.5, -2.0)
    ops.muon_ns_gemm(ops.MUON_GRAM, xws, tiles[(ops.MUON_GRAM, 0)], 1.0, 0.0)
    torch.cuda.synchronize()
    for l, (a, b) in enumerate(plan.shapes):
        mp = plan.mp[l]
        x, g = X[l], Gs[l]
        h = _panel(xws, plan.h[l], mp, mp)
        assert torch.equal(_bits(h), _bits((0.5 * g @ g - 2.0 * g).bfloat16())), (a, b, "POLY")
        assert torch.equal(_bits(h), _bits(h.T)), (a, b, "H symmetric")
        gg = _panel(xws, plan.g[l], mp, mp)
        assert torch.equal(_bits(gg), _bits((x @ x.T).bfloat16())), (a, b, "GRAM")
        assert torch.equal(_bits(gg), _bits(gg.T)), (a, b, "G symmetric")
        # UPDATE's H: small symmetric integers, so that H X stays exact at K = mp
        hs = sym(mp, min(a, b), 4)
        assert 0.25 * _exact_bound(hs, X[l].T) + 6 < 2 ** 24
        _put(xws, plan.h[l], hs.bfloat16())
        Hs.append(hs)
    ops.muon_ns_gemm(ops.MUON_UPDATE, xws, tiles[(ops.MUON_UPDATE, 0)], 0.25, 3.0)
    torch.cuda.synchronize()
    for l, (a, b) in enumerate(plan.shapes):
        x1_ref = (0.25 * Hs[l] @ X[l] + 3.0 * X[l]).bfloat16()
        assert torch.equal(_bits(_panel(xws, plan.x[l][1], plan.mp[l], plan.np[l])), _bits(x1_ref)), (a, b, "UPDATE")


def _opt_state(opt, gi=0):
    return next(st for (g, _), st in opt._muon.items() if g == gi)


def _final_x(opt, l, gi=0):
    """Layer l's O (the last Newton-Schulz iterate) as the [a][b] float64 matrix the apply kernel reads."""
    st = _opt_state(opt, gi)
    plan = st["plan"]
    ns = opt.param_groups[gi]["ns_steps"]
    a, b = plan.shapes[l]
    x = _panel(st["xws"], plan.x[l][ns % 2], plan.mp[l], plan.np[l]).double()
    x = x[:min(a, b), :max(a, b)]
    return x.T if plan.trans[l] else x


@pytest.mark.gpu
@pytest.mark.parametrize("nesterov", [True, False])
def test_prepare_and_normalize_match_torch(dev, nesterov):
    """The momentum buffer is torch's lerp_ bit for bit, X is bf16(lerp) (transposed where a > b) with zero padding,
    the norm and the scaled X are exact on operands whose sum of squares is exact, within one bf16 ulp on random ones,
    and a zero gradient gives X = 0 without NaN."""
    from turboprune_b200.optim import FusedMuon
    shapes = [(64, 147), (64, 27), (300, 100), (96, 200), (1024, 9216), (9216, 640)]    # up to 2304 tiles in one fold
    gen = torch.Generator(device=dev).manual_seed(1)
    for kind in ("exact", "random", "zero"):
        ps = [torch.nn.Parameter(torch.randn(s, generator=gen, device=dev)) for s in shapes]
        opt = FusedMuon(ps, lr=0.01, momentum=0.9, nesterov=nesterov, ns_steps=0)
        bufs = [torch.randn(s, generator=gen, device=dev) for s in shapes]
        for p, bf in zip(ps, bufs):
            if kind == "exact":            # bf16 integers: u = g (momentum buffer = g too), sums of squares exact
                p.grad = torch.randint(-4, 5, p.shape, generator=gen, device=dev).float()
                bf.copy_(p.grad)
            elif kind == "zero":
                p.grad = torch.zeros_like(p)
                bf.zero_()
            else:
                p.grad = torch.randn(p.shape, generator=gen, device=dev)
            opt.state[p]["momentum_buffer"] = bf.clone()
        opt.step()
        torch.cuda.synchronize()
        st = _opt_state(opt)
        plan = st["plan"]
        for l, (p, bf) in enumerate(zip(ps, bufs)):
            ref_buf = bf.clone().lerp_(p.grad, 1 - 0.9)
            assert torch.equal(_bits(opt.state[p]["momentum_buffer"]), _bits(ref_buf)), (kind, l)
            u = p.grad.lerp(ref_buf, 0.9) if nesterov else ref_buf
            xb = u.bfloat16()
            xb = xb.T if plan.trans[l] else xb
            nrm = xb.norm().clamp(min=1e-7)
            ref = xb.clone().div_(nrm)
            x = _panel(st["xws"], plan.x[l][0], plan.mp[l], plan.np[l])
            m, n = xb.shape
            assert float(x[m:].abs().sum()) == 0 and float(x[:, n:].abs().sum()) == 0, (kind, l, "padding")
            got = x[:m, :n]
            assert not torch.isnan(got).any()
            # the norm the kernel divided by (fp32 holding a bf16 value), and X = bf16(x / n) with it, bit for bit
            nk = st["norms"][l]
            assert torch.equal(nk.bfloat16().float(), nk), (kind, l)
            assert torch.equal(_bits(got), _bits((xb.float() / nk).bfloat16())), (kind, l)
            if kind == "zero":
                assert float(got.abs().sum()) == 0 and float(nk) == float(torch.tensor(1e-7).bfloat16())
            elif kind == "exact":
                assert float(nk) == float(nrm)
                assert torch.equal(_bits(got), _bits(ref)), (kind, l)
            else:
                # within one bf16 ulp (of the smaller of the two) of torch's norm
                ulp = 2.0 ** (math.floor(math.log2(min(float(nk), float(nrm)))) - 7)
                assert abs(float(nk) - float(nrm)) <= ulp, (kind, l, float(nk), float(nrm))


def _ns_restated(u, coef, steps, eps):
    """torch's _zeropower_via_newtonschulz in float64 with bf16 rounding at the same points."""
    a, b, c = coef
    x = u.bfloat16()
    tr = u.shape[0] > u.shape[1]
    x = (x.T if tr else x).double()
    n = torch.sqrt((x ** 2).sum()).bfloat16().double().clamp(min=eps).bfloat16().double()
    x = (x / n).bfloat16().double()
    for _ in range(steps):
        g = (x @ x.T).bfloat16().double()
        h = (c * g @ g + b * g).bfloat16().double()
        x = (a * x + h @ x).bfloat16().double()
    return x.T if tr else x


def _rel(x, r):
    return float(torch.linalg.norm(x - r) / torch.linalg.norm(r))


def _named(model):
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


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["resnet50", "deit_s"])
def test_fused_muon_step_against_torch(dev, model):
    """Three steps over ResNet-50's / DeiT-S's parameters with ERK-80 % masked gradients: momentum buffers and the AdamW
    group bit for bit with torch.optim.Muon (on the 2-D views) + torch.optim.AdamW; w bit for bit with torch's mul_ /
    add_ on the kernel's own O; each layer's O within max(1.5 x torch's distance, 2^-8) of the float64 restatement; a
    second optimizer gives identical bits, and a CUDA-graph replay of the step equals the eager step."""
    from turboprune_b200.optim import FusedMuon
    from torch.optim._muon import _zeropower_via_newtonschulz
    named, is_muon = _named(model)
    gen = torch.Generator(device=dev).manual_seed(7)
    init = [torch.randn(s, generator=gen, device=dev) * 0.05 for _, s in named]
    masks = [(torch.rand(s, generator=gen, device=dev) > 0.8).float() if m else None for (_, s), m in zip(named, is_muon)]
    lr, wd = 2e-3, 0.05

    def build():
        ps = [torch.nn.Parameter(v.clone()) for v in init]
        groups = [dict(params=[p for p, m in zip(ps, is_muon) if m]), dict(params=[p for p, m in zip(ps, is_muon) if not m], use_muon=False)]
        return ps, FusedMuon(groups, lr=lr, weight_decay=wd, adjust_lr_fn="match_rms_adamw", capturable=True)

    mine, opt = build()
    mine2, opt2 = build()
    ref = [torch.nn.Parameter(v.clone()) for v in init]
    rm = [p for p, m in zip(ref, is_muon) if m]
    rviews = [torch.nn.Parameter(p.detach().view(p.shape[0], -1).clone()) for p in rm]        # the 2-D views, as leaves
    ropt = torch.optim.Muon(rviews, lr=lr, weight_decay=wd, adjust_lr_fn="match_rms_adamw")
    raw = torch.optim.AdamW([p for p, m in zip(ref, is_muon) if not m], lr=lr, weight_decay=wd, foreach=True, capturable=True)
    spread = []
    for step in range(3):
        grads = [torch.randn(p.shape, generator=gen, device=dev) * (m if m is not None else 1) for p, m in zip(mine, masks)]
        before = [p.detach().clone() for p in mine]
        for ps in (mine, mine2, ref):
            for p, g in zip(ps, grads):
                p.grad = g.clone()
        for v, p in zip(rviews, rm):
            v.grad = p.grad.view(v.shape)
        opt.step(); opt2.step(); ropt.step(); raw.step()
        torch.cuda.synchronize()
        mi = 0
        for i, (p, p2, r, (name, _)) in enumerate(zip(mine, mine2, ref, named)):
            assert torch.equal(_bits(p.detach()), _bits(p2.detach())), f"{name}: two runs differ"
            if not is_muon[i]:
                assert torch.equal(_bits(p.detach()), _bits(r.detach())), f"{name}: AdamW group differs from torch"
                continue
            v = rviews[mi]
            buf = opt.state[p]["momentum_buffer"]
            assert torch.equal(_bits(buf), _bits(ropt.state[v]["momentum_buffer"])), f"{name} step {step}: momentum"
            o = _final_x(opt, mi)
            a, b = v.shape
            want = before[i].view(a, b).clone().mul_(1 - lr * wd).add_(o.bfloat16(), alpha=-(lr * 0.2 * math.sqrt(max(a, b))))
            assert torch.equal(_bits(p.detach().view(a, b)), _bits(want)), f"{name} step {step}: apply"
            u = v.grad.lerp(buf, 0.95)
            r_ = _ns_restated(u, (3.4445, -4.7750, 2.0315), 5, 1e-7)
            d_mine = _rel(o, r_)
            d_torch = _rel(_zeropower_via_newtonschulz(u, (3.4445, -4.7750, 2.0315), 5, 1e-7).double(), r_)
            spread.append((d_mine, d_torch))
            assert d_mine <= max(1.5 * d_torch, 2.0 ** -8), f"{name} step {step}: {d_mine} vs torch {d_torch}"
            mi += 1
    print(f"\n{model}: kernel distance max {max(s[0] for s in spread):.3e}, torch distance max {max(s[1] for s in spread):.3e}")

    # a captured step replays to the bits of the eager one
    state = [p.detach().clone() for p in mine]
    bufs = {k: {n: t.clone() for n, t in v.items()} for k, v in opt.state.items()}
    opt.step()
    eager = [p.detach().clone() for p in mine]
    for p, s0 in zip(mine, state):
        p.data.copy_(s0)
    for k, v in bufs.items():
        for n, t in v.items():
            opt.state[k][n].copy_(t)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        opt.step()
    torch.cuda.current_stream().wait_stream(s)
    for p, s0 in zip(mine, state):          # capture does not run the step: start from the same state again
        p.data.copy_(s0)
    for k, v in bufs.items():
        for n, t in v.items():
            opt.state[k][n].copy_(t)
    g.replay()
    torch.cuda.synchronize()
    for p, e, (name, _) in zip(mine, eager, named):
        assert torch.equal(_bits(p.detach()), _bits(e)), f"{name}: graph replay differs from the eager step"


@pytest.mark.gpu
def test_padding_stays_zero_from_a_poisoned_workspace(dev):
    from turboprune_b200.optim import FusedMuon
    shapes = [(64, 147), (64, 27), (1536, 384), (100, 300)]
    gen = torch.Generator(device=dev).manual_seed(3)
    ps = [torch.nn.Parameter(torch.randn(s, generator=gen, device=dev)) for s in shapes]
    opt = FusedMuon(ps, lr=0.01)
    for p in ps:
        p.grad = torch.randn(p.shape, generator=gen, device=dev)
    opt.step()
    st = _opt_state(opt)
    st["xws"].fill_(float("nan"))
    opt.step()
    torch.cuda.synchronize()
    plan = st["plan"]
    for l, (a, b) in enumerate(shapes):
        m, n = min(a, b), max(a, b)
        for buf in (0, 1):
            x = _panel(st["xws"], plan.x[l][buf], plan.mp[l], plan.np[l])
            assert float(x[m:].abs().sum()) == 0 and float(x[:, n:].abs().sum()) == 0, (a, b, buf)
        for row0 in (plan.g[l], plan.h[l]):
            gm = _panel(st["xws"], row0, plan.mp[l], plan.mp[l])
            assert float(gm[m:].abs().sum()) == 0 and float(gm[:, m:].abs().sum()) == 0
        assert not torch.isnan(_final_x(opt, l)).any() and torch.isfinite(ps[l]).all()


# ---------------------------------------------------------------- harness --------------------------------------------------
def _muon_harness(key, batch, tmp_path, precision="bfloat16", graph=True):
    from refshim import make_cfg, make_harness
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    name, data, mlt, _ = MODELS[key]
    cfg = make_cfg(name, data, mask_layer_type=mlt, precision=precision)
    cfg["optimizer_params"].update(optimizer_name="MuonAdamW", lr=2e-3, momentum=0.95, weight_decay=0.05)
    cfg["experiment_params"]["cuda_graph"] = graph
    torch.manual_seed(0)
    model = cm.CustomModel(cfg) if mlt == "LinearMask" else cm.TorchVisionModel(cfg)
    torch.manual_seed(1)
    pu.prune_er_erk(model, 0.3)
    return make_harness(cfg, model, batch, str(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [("deit_s", 8), ("resnet18", 64)], ids=["deit_s.b8", "resnet18.b64"])
def test_harness_muon_graph_step(dev, case, tmp_path):
    """bf16 PruningHarness.train_step with MuonAdamW: five steps, captured on the third call and then replayed, equal
    the cuda_graph: false harness bit for bit.  The last (replayed) step is taken again by torch.optim.Muon (on 2-D copies
    of the Muon weights) + torch.optim.AdamW(foreach, capturable) from the state before it, on the harness's gradients:
    momentum buffers and the AdamW group equal torch's bit for bit, and each Muon weight differs from torch's by at most
    the distance bar (relative to torch's update) plus torch's own distance from the float64 restatement."""
    from torch.optim._muon import _zeropower_via_newtonschulz
    from turboprune_b200.optim import FusedMuon
    key, batch = case
    h = _muon_harness(key, batch, tmp_path)
    h2 = _muon_harness(key, batch, tmp_path, graph=False)
    assert isinstance(h.optimizer, FusedMuon) and h._graph_enabled() and not h2._graph_enabled()
    size = 32 if key == "resnet18" else 224
    gen = torch.Generator().manual_seed(3)
    h.model.train(); h2.model.train()
    for step in range(5):
        x = torch.randn(batch, 3, size, size, generator=gen).cuda()
        t = torch.randint(0, 10, (batch,), generator=gen).cuda()
        for o in (h.optimizer, h2.optimizer):
            for grp in o.param_groups:
                grp["lr"] = 2e-3 * (1 - 0.1 * step)
        opt = h.optimizer
        if step == 4:                        # the state before the last step, for torch's optimizers
            w0 = {p: p.detach().clone() for g in opt.param_groups for p in g["params"]}
            st0 = {p: {k: v.clone() for k, v in opt.state[p].items()} for p in w0}
        h.train_step((x, t))
        h2.train_step((x, t))
        torch.cuda.synchronize()
        for (name, p), p2 in zip(h.model.named_parameters(), h2.model.parameters()):
            assert torch.equal(_bits(p.detach()), _bits(p2.detach())), f"{key} step {step + 1} {name}"
    assert h._graph is not None and h2._graph is None
    lr, wd = 2e-3 * (1 - 0.1 * 4), 0.05
    muon_ps, adamw_ps = opt.param_groups[0]["params"], opt.param_groups[1]["params"]
    views = [torch.nn.Parameter(w0[p].view(p.shape[0], -1).clone()) for p in muon_ps]
    ropt = torch.optim.Muon(views, lr=lr, weight_decay=wd, momentum=0.95, adjust_lr_fn="match_rms_adamw")
    for v, p in zip(views, muon_ps):
        v.grad = p.grad.reshape(v.shape).clone()
        ropt.state[v]["momentum_buffer"] = st0[p]["momentum_buffer"].clone()
    aws = [torch.nn.Parameter(w0[p].clone()) for p in adamw_ps]
    raw = torch.optim.AdamW(aws, lr=lr, weight_decay=wd, foreach=True, capturable=True)
    for q, p in zip(aws, adamw_ps):
        q.grad = p.grad.clone()
        raw.state[q] = {k: v.clone() for k, v in st0[p].items()}
    ropt.step(); raw.step()
    torch.cuda.synchronize()
    for q, p in zip(aws, adamw_ps):
        assert torch.equal(_bits(p.detach()), _bits(q.detach())), (key, "AdamW group", tuple(p.shape))
    for l, (v, p) in enumerate(zip(views, muon_ps)):
        buf = opt.state[p]["momentum_buffer"]
        assert torch.equal(_bits(buf), _bits(ropt.state[v]["momentum_buffer"])), (key, l, "momentum")
        u = v.grad.lerp(buf, 0.95)
        r_ = _ns_restated(u, (3.4445, -4.7750, 2.0315), 5, 1e-7)
        d_torch = _rel(_zeropower_via_newtonschulz(u, (3.4445, -4.7750, 2.0315), 5, 1e-7).double(), r_)
        bar = max(1.5 * d_torch, 2.0 ** -8)
        assert _rel(_final_x(opt, l), r_) <= bar, (key, l)
        decayed = w0[p].view(v.shape) * (1 - lr * wd)
        upd = torch.linalg.norm((v.detach() - decayed).double())          # torch's lr * ratio * |O_torch|
        diff = torch.linalg.norm((p.detach().view(v.shape) - v.detach()).double())
        assert float(diff) <= (bar + d_torch) * float(upd) * 1.01 + 1e-12, (key, l, float(diff / upd))


@pytest.mark.gpu
def test_harness_muon_float32_step(dev, tmp_path):
    h = _muon_harness("resnet18", 32, tmp_path, precision="float32")
    h.model.train()
    before = [p.detach().clone() for p in h.model.parameters()]
    x, t = torch.randn(32, 3, 32, 32).cuda(), torch.randint(0, 10, (32,)).cuda()
    h.train_step((x, t))
    torch.cuda.synchronize()
    assert all(torch.isfinite(p).all() for p in h.model.parameters())
    assert all(not torch.equal(p.detach(), b) for p, b in zip(h.optimizer.param_groups[0]["params"], before))


@pytest.mark.gpu
def test_rigl_update_resets_muon_momentum(dev, tmp_path):
    """synthetic_rn18_rigl with MuonAdamW: a RigL update zeroes the weight and momentum of grown positions of the Muon
    layers (exp_avg / exp_avg_sq of the classifier) and leaves every other element alone."""
    from turboprune_b200.harness_definitions.standard_pruning_harness import PruningHarness
    from turboprune_b200.optim import FusedMuon
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils.harness_utils import set_seed
    from turboprune_b200.utils.pruning_utils import prune_the_model
    cfg = C.compose("synthetic_rn18_rigl", ["optimizer_params=muon_adamw_triangular", "dataset_params.total_batch_size=64",
                                            "dataset_params.synthetic_steps_per_epoch=6", "pruning_params.rigl_update_interval=3",
                                            f"experiment_params.base_dir={tmp_path}"], CONF)
    set_seed(cfg)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)))
    prune_the_model(cfg=cfg, harness=h, target_density=0.2)
    h = PruningHarness(cfg=cfg, gpu_id=0, expt_dir=("rigl", str(tmp_path)), model=h.model)
    h._setup_optimizer()
    h._setup_scheduler(1)
    h.begin_rigl_level(1)
    assert isinstance(h.optimizer, FusedMuon)
    layers = h._masked_layers()
    lw = {id(m.weight) for m in layers}
    params = list(h.model.parameters())
    h.model.train()
    updates = 0
    for t, batch in enumerate(h.train_loader):
        is_update = h.rigl.is_update(t)
        if is_update:
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
            keep = ~grown_of[id(p)] if id(p) in lw else torch.ones_like(p, dtype=torch.bool)
            pairs = [(p.detach(), w0)] + [(st[k].view(p.shape), st0[k].view(p.shape)) for k in ("momentum_buffer", "exp_avg", "exp_avg_sq") if k in st]
            for now, was in pairs:
                assert torch.equal(now[keep].view(torch.int32), was[keep].view(torch.int32))
                if id(p) in lw:
                    assert float(now[~keep].abs().sum()) == 0.0
            n_grown += int((~keep).sum()) if id(p) in lw else 0
        assert n_grown > 0
    assert updates >= 1


@pytest.mark.gpu
def test_run_experiment_deit_muon_level(dev, tmp_path):
    """run_experiment.main on synthetic_deit_s_snip50_muon (a few batches of 8) completes the level and writes an
    optimizer_init.pt that loads back into FusedMuon."""
    import run_experiment
    from turboprune_b200.optim import FusedMuon
    from turboprune_b200.utils import config as C
    from turboprune_b200.utils import custom_models as cm
    cfg = C.compose("synthetic_deit_s_snip50_muon", ["dataset_params.total_batch_size=8",
                                                     "dataset_params.synthetic_steps_per_epoch=4",
                                                     f"experiment_params.base_dir={tmp_path}"], CONF)
    prefix, expt = run_experiment.main(cfg)
    assert os.path.isfile(os.path.join(expt, "metrics", "level_wise_metrics", "level_0_metrics.csv"))
    sd = torch.load(os.path.join(expt, "artifacts", "optimizer_init.pt"), map_location="cpu")
    assert [g["use_muon"] for g in sd["param_groups"]] == [True, False]
    assert sd["param_groups"][0]["adjust_lr_fn"] == "match_rms_adamw" and sd["param_groups"][1]["eps"] == 1e-8
    model = cm.CustomModel(cfg=cfg)
    masked = [m.weight for m in model.modules() if hasattr(m, "mask")]
    rest = [p for p in model.parameters() if all(p is not w for w in masked[:-1])]
    opt = FusedMuon([dict(params=masked[:-1]), dict(params=rest, use_muon=False)])
    opt.load_state_dict(sd)
    assert opt.param_groups[0]["lr"] == sd["param_groups"][0]["lr"]
