"""training_precision: float32 — fp32 activations and gradients end to end, masked GEMMs on TF32 tensor cores.

Exactness.  Operands are integers, so the exact result is known and an fp32 kernel must reproduce it bit for bit:
masked weights are in {-1, 0, 1} and every partial sum stays an integer below 2^22 (S = sum |a| |b| is asserted per
element, in float64).  For fprop and dgrad the activations / output gradients are odd integers in [257, 1023]: exact in
TF32 (11 significant bits), NOT representable in bf16 (8 significant bits), so a path that silently goes through bf16
fails.  For wgrad (a bf16 GEMM over the three-way split stacks, see ops.conv_wgrad_f32) x holds odd integers up to 2^15
(hi + lo is exact, x is not bf16) and dy is sparse in {-1, 0, 1} (dy_lo = 0).  Every case asserts its kernel path
through the mirrors of the host planning in test_kernel_exactness / test_fwd_pingpong.

Error bounds.  On random fp32 operands fprop / dgrad stay within 2^-9 S + K 2^-23 S (TF32 truncation of both operands
plus fp32 accumulation) and wgrad within 2^-15 S.  The bf16 path exceeds the TF32 bound on operands bf16 must round.
"""
import ctypes
import os
import re
import threading
from contextlib import nullcontext
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from test_fwd_pingpong import _dgrad_tapped, _fprop_items, _sms
from test_kernel_exactness import wgrad_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT = 2.0 ** 22


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


# ---------------------------------------------------------------- CPU-only ----------------------------------------------
NEW_SYMBOLS = ["tp_conv_fprop_f32", "tp_conv_dgrad_f32", "tp_wgrad_split3", "tp_stage_weights_f32",
               "tp_stage_weights_batched_f32", "tp_to_nhwc_f32", "tp_im2col_stem_f32"]


def test_fp32_abi_symbols_declared():
    from turboprune_b200 import _cabi
    header = open(os.path.join(ROOT, "include", "turboprune_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _cabi.SIGNATURES, name
    core = open(os.path.join(ROOT, "turboprune_b200", "csrc", "tp_core.cu")).read()
    assert "int tp_abi_version(void) { return 11; }" in core


def test_compute_precision_is_thread_local_and_nests():
    from turboprune_b200 import ops
    assert ops.current_precision() == torch.bfloat16
    seen = []
    with ops.compute_precision(torch.float32):
        assert ops.current_precision() == torch.float32
        t = threading.Thread(target=lambda: seen.append(ops.current_precision()))
        t.start(); t.join()
        with ops.compute_precision(torch.bfloat16):
            assert ops.current_precision() == torch.bfloat16
        assert ops.current_precision() == torch.float32
    assert ops.current_precision() == torch.bfloat16
    assert seen == [torch.bfloat16]
    with pytest.raises(ValueError):
        with ops.compute_precision(torch.float16):
            pass


def test_fused_modules_take_the_aten_path_at_float32():
    """The fused modules are bf16-only: inside an fp32 context BatchNorm2dB200, MaxPool2dB200 and the fused block forwards
    run ATen's ops (same modules and state dict, the choice is made per forward)."""
    from refshim import make_cfg
    from turboprune_b200 import fused_norm, ops
    from turboprune_b200.fused_norm import BatchNorm2dB200
    from turboprune_b200.utils import custom_models as cm
    m = cm.TorchVisionModel(make_cfg("resnet18", "cifar10", precision="float32"))
    assert any(isinstance(x, BatchNorm2dB200) for x in m.modules())
    assert fused_norm.fused_enabled()
    with ops.compute_precision(torch.float32):
        assert not fused_norm.fused_enabled()
    bn = BatchNorm2dB200(8)
    x = torch.randn(2, 8, 4, 4)
    with ops.compute_precision(torch.float32):
        z = bn(x, residual=x, relu=True)
    assert torch.equal(z, torch.relu(torch.nn.BatchNorm2d(8)(x) + x))


def test_fused_batchnorm_raises_inside_fp32_context():
    from turboprune_b200 import ops
    from turboprune_b200.fused_norm import _BNFn
    x = torch.zeros(2, 8, 4, 4)
    w, b = torch.ones(8), torch.zeros(8)
    rm, rv = torch.zeros(8), torch.ones(8)
    with ops.compute_precision(torch.float32):
        with pytest.raises(RuntimeError, match="bf16-only"):
            _BNFn.apply(x, None, w, b, rm, rv, None, 0.1, 1e-5, True, True)


def test_bf16_configs_never_enter_the_context(monkeypatch):
    from turboprune_b200 import ops
    from turboprune_b200.harness_definitions.base_harness import BaseHarness
    from turboprune_b200.utils import pruning_utils as pu
    entered = []
    real = ops.compute_precision
    monkeypatch.setattr(ops, "compute_precision", lambda d: (entered.append(d), real(d))[1])
    for dt in (torch.bfloat16, torch.float16):
        assert isinstance(BaseHarness._compute_precision(SimpleNamespace(precision=dt)), nullcontext)
        assert isinstance(pu._compute_precision(dt), nullcontext)
    assert entered == []
    with BaseHarness._compute_precision(SimpleNamespace(precision=torch.float32)):
        assert ops.current_precision() == torch.float32
    with pu._compute_precision(torch.float32):
        assert ops.current_precision() == torch.float32
    assert entered == [torch.float32, torch.float32]


# ---------------------------------------------------------------- operands ----------------------------------------------
def _odd(g, shape, lo, hi, dev):
    """fp32 odd integers with |v| in [lo, hi] and random signs."""
    v = torch.randint(lo // 2, (hi - 1) // 2 + 1, shape, generator=g, device=dev) * 2 + 1
    s = torch.randint(0, 2, shape, generator=g, device=dev) * 2 - 1
    return (v * s).float()


def _not_bf16(t, what):
    assert bool((t.bfloat16().float() != t).all()), f"{what}: some operands are bf16-representable"


def _tf32_exact(t, what):
    b = t.view(torch.int32) & 0x1FFF
    assert int(b.abs().max()) == 0, f"{what}: operands need more than TF32's 11 significant bits"


def _same(got, want, what):
    bad = got.double() != want
    n = int(bad.sum())
    if n:
        i = tuple(bad.nonzero()[0].tolist())
        pytest.fail(f"{what}: {n} of {bad.numel()} elements differ; first at {i}: {float(got[i])!r} vs {float(want[i])!r}")


def _sparse_signs(g, shape, q, dev):
    keep = (torch.rand(shape, generator=g, device=dev) < q).float()
    return keep * ((torch.randint(0, 2, shape, generator=g, device=dev) * 2 - 1).float())


def _layer(x, w, m, b, stride, pad, kind):
    from turboprune_b200 import ops
    if kind == "linear":
        return ops.masked_linear(x, w, m, b)
    return ops.masked_conv2d(x, w, m, b, (stride, stride), (pad, pad))


# (id, kind, batch, extent, cin, cout, k, stride, pad, bias)
CASES = [
    ("l1.1x1.256-64.b512", "conv", 512, 56, 256, 64, 1, 1, 0, False),
    ("l1.3x3.64.b512", "conv", 512, 56, 64, 64, 3, 1, 1, False),
    ("l2.3x3.128.s2.b256", "conv", 256, 56, 128, 128, 3, 2, 1, True),
    ("l3.1x1.512-1024.s2.b128", "conv", 128, 28, 512, 1024, 1, 2, 0, False),
    ("stem.7x7.s2.224.b64", "stem", 64, 224, 3, 64, 7, 2, 3, False),
    ("fc.2048-1000.b512", "linear", 512, None, 2048, 1000, 1, 1, 0, True),
    ("deit.qkv.384-1152", "linear", 8 * 197, None, 384, 1152, 1, 1, 0, True),
]


def _operands(g, case, dev, wgrad):
    name, kind, n, hw, cin, cout, k, st, pad, has_bias = case
    if kind == "linear":
        xshape = (n, cin)
        w = (torch.randint(-1, 2, (cout, cin), generator=g, device=dev)).float()
        m = (torch.rand(cout, cin, generator=g, device=dev) < 0.5).float()
    else:
        xshape = (n, cin, hw, hw)
        w = (torch.randint(-1, 2, (cout, cin, k, k), generator=g, device=dev)).float()
        m = (torch.rand(cout, cin, k, k, generator=g, device=dev) < 0.5).float()
    if wgrad:
        x = _odd(g, xshape, 257, 2 ** 15 - 1, dev)
    else:
        x = _odd(g, xshape, 257, 1023, dev)
    if kind != "linear":
        x = x.contiguous(memory_format=torch.channels_last)
    b = torch.randint(-8, 9, (cout,), generator=g, device=dev).float() if has_bias else None
    return x, w, m, b


def _ref_conv(x64, w64, st, pad, kind):
    return x64 @ w64.t() if kind == "linear" else F.conv2d(x64, w64, None, st, pad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fp32_fprop_dgrad_exact(dev, case):
    """y and dx of one masked layer, through MaskedConv2dFn at float32, equal float64 bit for bit on TF32-exact operands
    bf16 cannot hold."""
    from turboprune_b200 import ops
    name, kind, n, hw, cin, cout, k, st, pad, has_bias = case
    sms = _sms()
    if kind == "conv" and n == 512:
        items, _ = _fprop_items(n, hw, cout, k, k, st, pad)
        assert items > 40 * sms, items                    # many work items per CTA: both ping-pong consumers cycle
    if kind == "conv" and st == 2:
        assert sum(_dgrad_tapped(k, k, st, pad)) == (4 if k == 3 else 1)   # 1x1 s2: three parity classes write zeros
    g = torch.Generator(device=dev).manual_seed(len(name) * 7 + n)
    x, w, m, b = _operands(g, case, dev, wgrad=False)
    _not_bf16(x, "x"); _tf32_exact(x, "x")
    stem = kind == "stem"
    x.requires_grad_(not stem)
    with ops.compute_precision(torch.float32):
        y = _layer(x, w, m, b, st, pad, kind)
        assert y.dtype == torch.float32
        dy = _odd(g, tuple(y.shape), 257, 1023, dev)
        _not_bf16(dy, "dy")
        if not stem:
            (dx,) = torch.autograd.grad(y, x, dy)
            assert dx.dtype == torch.float32
    wm = (w * m).double()
    x64 = x.detach().double()
    S = _ref_conv(x64.abs(), wm.abs(), st, pad, kind)
    assert float(S.max()) <= EXACT
    ref = _ref_conv(x64, wm, st, pad, kind)
    if b is not None:
        ref = ref + (b.double() if kind == "linear" else b.double().view(1, -1, 1, 1))
    _same(y.detach(), torch.round(ref), f"{name} fprop")
    del S, ref
    if not stem:
        dy64 = dy.double()
        if kind == "linear":
            S, ref = dy64.abs() @ wm.abs(), dy64 @ wm
        else:
            S = conv2d_input(x64.shape, wm.abs(), dy64.abs(), st, pad)
            ref = conv2d_input(x64.shape, wm, dy64, st, pad)
        assert float(S.max()) <= EXACT
        _same(dx, torch.round(ref), f"{name} dgrad")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fp32_wgrad_exact(dev, case):
    """dW (through the three-way split stacks and ONE bf16 wgrad over 3n images) and db equal float64 bit for bit;
    masked weights get exactly zero."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    name, kind, n, hw, cin, cout, k, st, pad, has_bias = case
    g = torch.Generator(device=dev).manual_seed(len(name) * 11 + n)
    x, w, m, b = _operands(g, case, dev, wgrad=True)
    _not_bf16(x, "x")
    w.requires_grad_(True)
    if b is not None:
        b.requires_grad_(True)
    with ops.compute_precision(torch.float32):
        y = _layer(x, w, m, b, st, pad, kind)
    npix = y.numel() // cout
    # the GEMM the split runs: 3 * npix pixels; its plan (split-K, split lanes) is the bf16 kernel's for that extent
    if kind == "stem":
        kp = ops.stem_geometry(cin, k, k)[1]
        d3 = ops._cabi.ConvDesc(3 * npix, 1, 1, kp, cout, 1, 1, 1, 1, 0, 0, 1, 1)
        kcols = kp
    else:
        cin_p = ops.padded_cin(cin, k, k) if kind == "conv" else ops.padded_cin(cin, 1, 1)
        kk = k if kind == "conv" else 1
        d3 = ops.make_desc(3 * n, hw or 1, hw or 1, cin_p, cout, kk, kk, (st, st), (pad, pad))
        kcols = kk * kk * cin_p
    plan = wgrad_plan(3 * npix, kcols, cout, _sms())
    assert lib.tp_conv_workspace_bytes(ctypes.byref(d3), 2) == plan.ws_bytes
    assert plan.splits >= 1 and plan.kblocks == (3 * npix + 63) // 64
    q = min(1 / 64, 2.0 ** 21 / (npix * 2 ** 15))          # sparse dy: every partial sum of dW stays below 2^22
    dy = _sparse_signs(g, tuple(y.shape), q, dev)
    if kind != "linear":
        dy = dy.contiguous(memory_format=torch.channels_last)
    with ops.compute_precision(torch.float32):
        grads = torch.autograd.grad(y, [w] + ([b] if b is not None else []), dy)
    x64, dy64 = x.double(), dy.double()
    if kind == "linear":
        ref, S = dy64.t() @ x64, dy64.abs().t() @ x64.abs()
    else:
        ref = conv2d_weight(x64, w.shape, dy64, st, pad)
        S = conv2d_weight(x64.abs(), w.shape, dy64.abs(), st, pad)
    assert float(S.max()) <= EXACT, float(S.max())
    _same(grads[0], torch.round(ref) * m.double(), f"{name} wgrad")
    assert bool((grads[0][m == 0] == 0).all())
    if b is not None:
        dims = (0,) if kind == "linear" else (0, 2, 3)
        _same(grads[1], dy64.sum(dims), f"{name} bias gradient")


@pytest.mark.gpu
def test_fp32_error_bounds_and_bf16_differs(dev):
    """Random fp32 operands: TF32 fprop / dgrad within 2^-9 S + K 2^-23 S of float64, the split wgrad within 2^-15 S.
    On operands 3/4 of a bf16 ulp above a bf16 value (exact in TF32), the bf16 path exceeds the TF32 bound."""
    from turboprune_b200 import ops
    n, hw, cin, cout, k = 32, 28, 128, 128, 3
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn(n, cin, hw, hw, generator=g, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = torch.randn(cout, cin, k, k, generator=g, device=dev).requires_grad_(True)
    m = (torch.rand(cout, cin, k, k, generator=g, device=dev) < 0.5).float()
    dy = torch.randn(n, cout, hw, hw, generator=g, device=dev)
    K = cin * k * k
    with ops.compute_precision(torch.float32):
        y = ops.masked_conv2d(x, w, m, None, (1, 1), (1, 1))
        dx, dw = torch.autograd.grad(y, [x, w], dy)
    x64, w64, dy64 = x.detach().double(), (w.detach() * m).double(), dy.double()
    tol = 2.0 ** -9 + K * 2.0 ** -23
    S = F.conv2d(x64.abs(), w64.abs(), None, 1, 1)
    err = (y.detach().double() - F.conv2d(x64, w64, None, 1, 1)).abs()
    assert bool((err <= tol * S).all()), float((err / S).max())
    S = conv2d_input(x64.shape, w64.abs(), dy64.abs(), 1, 1)
    err = (dx.double() - conv2d_input(x64.shape, w64, dy64, 1, 1)).abs()
    assert bool((err <= tol * S).all()), float((err / S).max())
    S = conv2d_weight(x64.abs(), w.shape, dy64.abs(), 1, 1)
    err = (dw.double() - conv2d_weight(x64, w.shape, dy64, 1, 1) * m.double()).abs()
    assert bool((err <= 2.0 ** -15 * S).all()), float((err / S).max())

    # operands bf16 must round up by 1/4 of its ulp, exactly representable in TF32
    base = 1 + torch.randint(0, 32, (n, cin, hw, hw), generator=g, device=dev).float() * 2.0 ** -7
    xb = (base + 0.75 * 2.0 ** -7).contiguous(memory_format=torch.channels_last)
    wb = 1 + (torch.randint(0, 32, (cout, cin, k, k), generator=g, device=dev).float() + 0.75) * 2.0 ** -7
    _tf32_exact(xb, "x"); _tf32_exact(wb, "w"); _not_bf16(xb, "x")
    ref = F.conv2d(xb.double(), (wb * m).double(), None, 1, 1)
    S = F.conv2d(xb.double(), (wb * m).double().abs(), None, 1, 1)
    with ops.compute_precision(torch.float32):
        y32 = ops.masked_conv2d(xb, wb, m, None, (1, 1), (1, 1))
    y16 = ops.masked_conv2d(xb, wb, m, None, (1, 1), (1, 1))          # default precision: bf16
    assert y16.dtype == torch.bfloat16 and y32.dtype == torch.float32
    assert bool(((y32.double() - ref).abs() <= K * 2.0 ** -23 * S).all())
    assert bool(((y16.double() - ref).abs() > tol * S).any())


# ---------------------------------------------------------------- harness -----------------------------------------------
class _Recorder:
    """Wraps the loaded C library: records the name of every entry point called."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("tp_"):
            return fn

        def call(*a):
            self.calls.append(name)
            return fn(*a)
        return call


BF16_ENTRIES = {"tp_conv_fprop", "tp_conv_fprop_stats", "tp_conv_dgrad", "tp_conv_dgrad_bnrelu", "tp_to_nhwc_bf16",
                "tp_stage_weights", "tp_stage_weights_batched", "tp_im2col_stem", "tp_bn_forward", "tp_bn_forward_ext",
                "tp_bn_backward", "tp_bn_backward_ext", "tp_maxpool_forward", "tp_maxpool_backward"}

HARNESS_CASES = [("resnet18", "cifar10", "ConvMask", 64), ("resnet50", "imagenet", "ConvMask", 32),
                 ("vgg16", "cifar10", "ConvMask", 64), ("local_deit_small_patch16_224", "imagenet", "LinearMask", 16)]


def _harness(case, tmp_path, precision="float32"):
    from refshim import make_cfg, make_harness
    from turboprune_b200.utils import custom_models as cm, pruning_utils as pu
    model_name, data, mlt, batch = case
    cfg = make_cfg(model_name, data, mask_layer_type=mlt, precision=precision)
    cfg["optimizer_params"].update(lr=0.05, weight_decay=5e-4)
    torch.manual_seed(0)
    model = cm.CustomModel(cfg) if mlt == "LinearMask" else cm.TorchVisionModel(cfg)
    torch.manual_seed(1)
    pu.prune_er_erk(model, 0.3)
    return cfg, model, make_harness(cfg, model, batch, str(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("case", HARNESS_CASES, ids=[c[0] for c in HARNESS_CASES])
def test_fp32_train_step_matches_oracle(dev, case, tmp_path, monkeypatch):
    """One PruningHarness.train_step at float32: loss within 1e-3 of the CPU oracle in fp32, an fp32 loss tensor, no bf16
    conv / BatchNorm / layout entry point called, and only fp32 outputs seen by forward hooks."""
    from oracle.train import train_step
    from turboprune_b200 import _cabi
    import copy
    cfg, model, h = _harness(case, tmp_path)
    ref = copy.deepcopy(model.model).cpu().float()
    for mod in ref.modules():            # the oracle: the same masked graph, fp32 eager on the CPU
        if hasattr(mod, "mask"):
            mod.forward = _cpu_masked_forward(mod)
    opt_ref = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=5e-4)
    model_name, data, _, batch = case
    size = 32 if data.startswith("cifar") else 224
    g = torch.Generator().manual_seed(2)
    x = torch.randn(batch, 3, size, size, generator=g)
    t = torch.randint(0, 10, (batch,), generator=g)
    ref.train()
    l_ref, _ = train_step(ref, opt_ref, x, t, use_amp=False)
    rec = _Recorder(_cabi.load())
    monkeypatch.setattr(_cabi, "_lib", rec)
    dtypes = set()
    hooks = [mod.register_forward_hook(lambda mod, i, o: dtypes.add(o.dtype) if torch.is_tensor(o) else None)
             for mod in h.model.modules()]
    try:
        loss = h.train_step((x.cuda(), t.cuda()))["loss"]
        torch.cuda.synchronize()
    finally:
        for hk in hooks:
            hk.remove()
    assert loss.dtype == torch.float32
    rel = abs(float(loss) - float(l_ref)) / abs(float(l_ref))
    assert rel <= 1e-3, (float(loss), float(l_ref))
    assert not (set(rec.calls) & BF16_ENTRIES), sorted(set(rec.calls) & BF16_ENTRIES)
    assert "tp_conv_fprop_f32" in rec.calls and "tp_wgrad_split3" in rec.calls and "tp_conv_wgrad" in rec.calls
    assert dtypes <= {torch.float32, torch.int64}, dtypes


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bfloat16", "float32"])
@pytest.mark.parametrize("case", HARNESS_CASES, ids=[c[0] for c in HARNESS_CASES])
def test_train_step_consumes_the_weight_shadow(dev, case, precision, tmp_path, monkeypatch):
    """In a train step every masked layer runs on the operands of the one-launch weight shadow: no layer stages its own
    (tp_stage_weights / tp_stage_weights_f32), at either precision."""
    from turboprune_b200 import _cabi
    _, _, h = _harness(case, tmp_path, precision)
    _, data, _, batch = case
    size = 32 if data.startswith("cifar") else 224
    g = torch.Generator().manual_seed(2)
    x = torch.randn(batch, 3, size, size, generator=g)
    t = torch.randint(0, 10, (batch,), generator=g)
    rec = _Recorder(_cabi.load())
    monkeypatch.setattr(_cabi, "_lib", rec)
    h.train_step((x.cuda(), t.cuda()))
    torch.cuda.synchronize()
    batched = "tp_stage_weights_batched" if precision == "bfloat16" else "tp_stage_weights_batched_f32"
    assert rec.calls.count(batched) == 1
    assert not {"tp_stage_weights", "tp_stage_weights_f32"} & set(rec.calls), sorted(set(rec.calls))


def _cpu_masked_forward(mod):
    """F.conv2d / F.linear on mask * w in fp32 (the fused block forwards may also ask a convolution for its input back)."""
    def fwd(x, want_skip=False, want_stats=False):
        w = mod.weight * mod.mask
        if isinstance(mod, torch.nn.Conv1d):
            return F.linear(x, w.view(w.shape[0], w.shape[1]), mod.bias)
        if isinstance(mod, torch.nn.Linear):
            return F.linear(x, w, mod.bias)
        y = F.conv2d(x, w, mod.bias, mod.stride, mod.padding)
        assert not want_stats
        return (y, x) if want_skip else y
    return fwd


@pytest.mark.gpu
def test_fp32_graph_replay_and_side_stream_equal_eager(dev, tmp_path):
    """float32 ResNet-18: a CUDA-graph replay of the step equals the eager step bit for bit (loss and updated weights),
    and side-stream wgrad equals main-stream wgrad bit for bit."""
    case = HARNESS_CASES[0]
    g = torch.Generator().manual_seed(3)
    x = torch.randn(64, 3, 32, 32, generator=g).cuda()
    t = torch.randint(0, 10, (64,), generator=g).cuda()
    res = {}
    for mode in ("graph", "eager", "eager_main"):
        cfg, model, h = _harness(case, tmp_path)
        cfg["experiment_params"]["cuda_graph"] = mode == "graph"
        cfg["experiment_params"]["wgrad_side_stream"] = mode != "eager_main"
        losses = [h.train_step((x, t))["loss"].clone() for _ in range(4)]
        torch.cuda.synchronize()
        res[mode] = (torch.stack(losses), [p.detach().clone() for p in h.model.parameters()])
    for other in ("eager", "eager_main"):
        assert torch.equal(res["graph"][0], res[other][0]), other
        assert all(torch.equal(a, b) for a, b in zip(res["graph"][1], res[other][1])), other


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["snip", "synflow"])
def test_fp32_snip_synflow_masks(dev, method, tmp_path):
    """SNIP and SynFlow at float32 score through the fp32 path and produce masks of the requested density."""
    from turboprune_b200 import _cabi
    from turboprune_b200.utils import pruning_utils as pu
    cfg, model, h = _harness(HARNESS_CASES[0], tmp_path)
    rec = _Recorder(_cabi.load())
    old = _cabi._lib
    _cabi._lib = rec
    try:
        fn = getattr(pu, f"prune_{method}")
        fn(cfg, h.model, h.train_loader, 0.2)
    finally:
        _cabi._lib = old
    assert "tp_conv_fprop_f32" in rec.calls and not (set(rec.calls) & BF16_ENTRIES)
    layers = [m for _, m in h.model._masked()]
    total = sum(m.mask.numel() for m in layers)
    kept = sum(int(m.mask.sum()) for m in layers)
    assert abs(kept / total - 0.2) < 1e-3, kept / total


@pytest.mark.gpu
def test_fp32_run_experiment_two_levels(dev, tmp_path):
    """run_experiment.main completes two IMP levels with a float32 synthetic CIFAR config and writes its CSVs."""
    import csv
    import run_experiment
    from turboprune_b200.utils import config as C
    cfg = C.compose("synthetic_rn18_imp", ["dataset_params.total_batch_size=64", "dataset_params.synthetic_steps_per_epoch=3",
                                           "experiment_params.training_precision=float32",
                                           f"experiment_params.base_dir={tmp_path}"], os.path.join(ROOT, "conf_b200"))
    prefix, expt = run_experiment.main(cfg)
    rows = list(csv.DictReader(open(os.path.join(expt, f"{prefix}_summary.csv"))))
    assert [r["Level"] for r in rows] == ["0", "1"]
    assert abs(float(rows[1]["Sparsity"]) - 20.0) < 1e-3
