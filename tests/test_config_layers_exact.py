"""Exactness of the masked layers of the CIFAR ResNet-18, VGG-16 (CIFAR-100) and DeiT-S train steps, at bf16 and
float32, against float64.

test_kernel_exactness.py, test_step_kernels_exact.py and test_fp32_training.py check the kernels at ResNet-50's
ImageNet extents.  The other models the configs train reach geometries those tables do not: 4x4 and 2x2 extents (one
128-pixel M tile spans 8 or 32 images; most taps of a 2x2 output read padding), classifiers whose output channels are
padded for the backward GEMMs (512 -> 10: cout_p 16; 4096 -> 100: cout_p 104), a K of 25 088 (VGG's classifier[0]:
392 K blocks, 3136 wgrad tiles, a 411 MB split-K workspace), biases with dgrad at CIFAR extents, ResNet-18's BasicBlock
epilogues and BatchNorm extents, and DeiT-S's linears (a head of 1000 rows: 7 full 128-row tiles and 104 more).

The tables list every masked-layer geometry of each model at the per-GPU batch of 512, the epilogues the train step
runs on it and the wgrad plan it reaches on a 132-SM H100.  A CPU test pins the geometries to the models; GPU tests pin
every C-ABI convolution call (descriptor and epilogue operands) and every BatchNorm call of a real step to the tables.
Each row is then checked with the methods of the files above:

- bf16: integer operands, S <= 2^22 quanta asserted first, fprop / dgrad / wgrad / bias gradient bit for bit against
  float64 (convolutions through ops.conv_*, stems and linears through the layers' autograd path);
- float32: TF32-exact operands bf16 cannot hold for fprop / dgrad, the split stacks for wgrad, bit for bit;
- through the weight shadow: a WeightStager stages, the weights and the mask change in place, it stages again, and the
  layer runs on the staged operands; the result equals the per-layer run bit for bit and the float64 result;
- ResNet-18's BatchNorm calls and the fused BatchNorm-backward dgrad epilogue of each stage's conv2.
"""
import ctypes
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from test_fp32_training import _Recorder, _not_bf16, _odd, _sparse_signs, _tf32_exact
from test_fwd_pingpong import _sms
from test_kernel_exactness import (H100_SMS, _assert_plan, _bounded, _check_row_stats, _exact, _ints, _kill_blocks,
                                   _nchw64, _per_batch, _same, _signs, bnb_dgrad_check, wgrad_plan)
from test_step_kernels_exact import BnCase, _missed_bn_paths, _table_keys, bn_backward_check, bn_forward_check, bn_geom


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _release_memory():
    """Every case frees its tensors before the next one (the GPU is shared; VGG's classifier[0] needs a few GB)."""
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


# ---------------------------------------------------------------- the tables -------------------------------------------------
# kind: "stem" (im2col GEMM, no dgrad), "conv" (TMA implicit GEMM), "fc" (Conv1dMask), "linear" (LinearMask).
# hw: input extent of a convolution; tokens per image of a linear.  epi: what the train step adds to the plain GEMMs,
# s = BatchNorm statistics in the fprop epilogue, a = the skip gradient added in the dgrad epilogue, b = the fused
# BatchNorm-backward dgrad epilogue (conv_dgrad_bnrelu, checked by test_rn18_bn_backward_dgrad_epilogue_exact).
# plan: (wgrad splits, split lanes, K blocks per split, K blocks of the last split) of the bf16 wgrad at ``batch`` on 132
# SMs.  f32_batch: the batch of the float32 cases (the float64 references of every row fit at 512).
Row = namedtuple("Row", "id kind batch hw cin cout k stride pad bias epi plan f32_batch")

RN18 = [
    Row("rn18.stem.3x3.32", "stem", 512, 32, 3, 64, 3, 1, 1, False, "s", (131, 8, 63, 2), 512),
    Row("rn18.l1.3x3.64@32", "conv", 512, 32, 64, 64, 3, 1, 1, False, "sab", (44, 4, 187, 151), 512),
    Row("rn18.l2.0.3x3.64-128.s2@32", "conv", 512, 32, 64, 128, 3, 2, 1, False, "sa", (44, 4, 47, 27), 512),
    Row("rn18.l2.3x3.128@16", "conv", 512, 16, 128, 128, 3, 1, 1, False, "sab", (26, 2, 79, 73), 512),
    Row("rn18.l2.ds.1x1.64-128.s2@32", "conv", 512, 32, 64, 128, 1, 2, 0, False, "s", (128, 8, 16, 16), 512),
    Row("rn18.l3.0.3x3.128-256.s2@16", "conv", 512, 16, 128, 256, 3, 2, 1, False, "sa", (13, 1, 40, 32), 512),
    Row("rn18.l3.3x3.256@8", "conv", 512, 8, 256, 256, 3, 1, 1, False, "sab", (7, 1, 74, 68), 512),
    Row("rn18.l3.ds.1x1.128-256.s2@16", "conv", 512, 16, 128, 256, 1, 2, 0, False, "s", (57, 4, 9, 8), 512),
    Row("rn18.l4.0.3x3.256-512.s2@8", "conv", 512, 8, 256, 512, 3, 2, 1, False, "sa", (3, 1, 43, 42), 512),
    # P*Q = 16: one 128-pixel M tile spans 8 images
    Row("rn18.l4.3x3.512@4", "conv", 512, 4, 512, 512, 3, 1, 1, False, "sab", (3, 1, 43, 42), 512),
    Row("rn18.l4.ds.1x1.256-512.s2@8", "conv", 512, 8, 256, 512, 1, 2, 0, False, "s", (13, 1, 10, 8), 512),
    # cout 10 padded to cout_p 16 for the backward GEMMs
    Row("rn18.fc.512-10", "fc", 512, 1, 512, 10, 1, 1, 0, True, "", (4, 1, 2, 2), 512),
]
VGG = [
    Row("vgg.stem.3x3.32", "stem", 512, 32, 3, 64, 3, 1, 1, True, "", (131, 8, 63, 2), 512),
    Row("vgg.3x3.64@32", "conv", 512, 32, 64, 64, 3, 1, 1, True, "", (44, 4, 187, 151), 512),
    Row("vgg.3x3.64-128@16", "conv", 512, 16, 64, 128, 3, 1, 1, True, "", (44, 4, 47, 27), 512),
    Row("vgg.3x3.128@16", "conv", 512, 16, 128, 128, 3, 1, 1, True, "", (26, 2, 79, 73), 512),
    Row("vgg.3x3.128-256@8", "conv", 512, 8, 128, 256, 3, 1, 1, True, "", (13, 1, 40, 32), 512),
    Row("vgg.3x3.256@8", "conv", 512, 8, 256, 256, 3, 1, 1, True, "", (7, 1, 74, 68), 512),
    Row("vgg.3x3.256-512@4", "conv", 512, 4, 256, 512, 3, 1, 1, True, "", (3, 1, 43, 42), 512),
    Row("vgg.3x3.512@4", "conv", 512, 4, 512, 512, 3, 1, 1, True, "", (3, 1, 43, 42), 512),
    # P*Q = 4: one M tile spans 32 images, 5 of the 9 taps of every output pixel read padding
    Row("vgg.3x3.512@2", "conv", 512, 2, 512, 512, 3, 1, 1, True, "", (1, 1, 32, 32), 512),
    # K = 25 088 (392 K blocks); wgrad: 3136 tiles in one split, a 411 MB workspace
    Row("vgg.fc0.25088-4096", "fc", 512, 1, 25088, 4096, 1, 1, 0, True, "", (1, 1, 8, 8), 512),
    Row("vgg.fc1.4096-4096", "fc", 512, 1, 4096, 4096, 1, 1, 0, True, "", (1, 1, 8, 8), 512),
    # cout 100 padded to cout_p 104
    Row("vgg.fc2.4096-100", "fc", 512, 1, 4096, 100, 1, 1, 0, True, "", (2, 1, 4, 4), 512),
]
DEIT = [
    # 512 x 197 = 100 864 rows: 788 full M tiles
    Row("deit.qkv.384-1152", "linear", 512, 197, 384, 1152, 1, 1, 0, True, "", (7, 1, 226, 220), 512),
    Row("deit.proj.384-384", "linear", 512, 197, 384, 384, 1, 1, 0, True, "", (22, 2, 72, 64), 512),
    Row("deit.fc1.384-1536", "linear", 512, 197, 384, 1536, 1, 1, 0, True, "", (5, 1, 316, 312), 512),
    Row("deit.fc2.1536-384", "linear", 512, 197, 1536, 384, 1, 1, 0, True, "", (7, 1, 226, 220), 512),
    # 1000 output rows: 7 full 128-row tiles + 104
    Row("deit.head.384-1000", "linear", 512, 1, 384, 1000, 1, 1, 0, True, "", (2, 1, 4, 4), 512),
]
# not a train-step batch: 37 x 197 = 7289 rows = 56 full M tiles + 121 rows
DEIT_RAGGED = Row("deit.fc2.1536-384.b37", "linear", 37, 197, 1536, 384, 1, 1, 0, True, "", (6, 1, 19, 19), 37)
MODELS = {"resnet18": RN18, "vgg16": VGG, "deit_s": DEIT}
ALL_ROWS = RN18 + VGG + DEIT + [DEIT_RAGGED]
CONV_ROWS = [r for r in ALL_ROWS if r.kind == "conv"]
LAYER_ROWS = [r for r in ALL_ROWS if r.kind != "conv"]
# conv rows that also run through the weight shadow (every stem and linear row does)
SHADOW_CONVS = {"rn18.l4.3x3.512@4", "vgg.3x3.512@2"}
SHADOW_ROWS = [r for r in ALL_ROWS if r.id in SHADOW_CONVS]

# (model, make_cfg arguments, input extent)
MODEL_CFGS = {"resnet18": (("resnet18", "cifar10", "ConvMask"), 32), "vgg16": (("vgg16", "cifar100", "ConvMask"), 32),
              "deit_s": (("local_deit_small_patch16_224", "imagenet", "LinearMask"), 224)}


def _cout_p(row):
    """cout as the backward GEMMs walk it (ops.layer_plan): a multiple of 8, of 64 under a multi-tap filter."""
    if row.kind == "stem":
        return row.cout
    m = 64 if row.k > 1 else 8
    return (row.cout + m - 1) // m * m


def _pq(row):
    return (row.hw + 2 * row.pad - row.k) // row.stride + 1 if row.kind in ("stem", "conv") else 1


def _kcols(row):
    """K columns of the wgrad GEMM: the stem's im2col width (taps * cin padded to 8), else taps * cin."""
    kk = row.k * row.k * row.cin
    return (kk + 7) // 8 * 8 if row.kind == "stem" else kk


def _npix(row, n):
    return n * (_pq(row) ** 2 if row.kind in ("stem", "conv") else row.hw)


def _seed(*parts):
    return sum(ord(c) for c in "/".join(map(str, parts)))


# ---------------------------------------------------------------- CPU: the tables against the models ------------------------
def _geometry(row):
    kind = "linear" if row.kind in ("fc", "linear") else row.kind
    return (kind, row.hw, row.cin, row.cout, row.k, row.stride, row.pad, row.bias)


def _record_geometries(model_key, monkeypatch):
    """Masked-layer geometries of one CPU forward of the model (fuse_norm off), recorded in place of ops.masked_conv2d /
    ops.masked_linear (which compute F.conv2d / F.linear of the masked weight instead)."""
    from refshim import make_cfg
    from turboprune_b200 import ops
    from turboprune_b200.utils import custom_models as cm
    (name, data, mlt), hw = MODEL_CFGS[model_key]
    seen = set()

    def conv(x, w, m, b=None, stride=(1, 1), padding=(0, 0), *a, **k):
        cout, cin, r, s = w.shape
        assert x.shape[2] == x.shape[3] and r == s and stride[0] == stride[1] and padding[0] == padding[1]
        kind = "stem" if ops.layer_plan(cout, cin, r, s, x.requires_grad).stem else "conv"
        seen.add((kind, x.shape[2], cin, cout, r, stride[0], padding[0], b is not None))
        return F.conv2d(x, w * m, b, stride, padding)

    def linear(x, w, m, b=None, *a, **k):
        seen.add(("linear", math.prod(x.shape[1:-1]), w.shape[1], w.shape[0], 1, 1, 0, b is not None))
        return F.linear(x, w * m, b)

    monkeypatch.setattr(ops, "masked_conv2d", conv)
    monkeypatch.setattr(ops, "masked_linear", linear)
    cfg = make_cfg(name, data, mask_layer_type=mlt, precision="bfloat16")
    cfg["model_params"]["fuse_norm"] = False
    torch.manual_seed(0)
    model = cm.CustomModel(cfg) if mlt == "LinearMask" else cm.TorchVisionModel(cfg)
    model.model(torch.randn(1, 3, hw, hw))
    return seen


@pytest.mark.parametrize("model_key", list(MODELS))
def test_tables_list_every_masked_layer_geometry(model_key, monkeypatch):
    """The table of each model is exactly the set of its masked-layer geometries (input extent or tokens per image, cin,
    cout, kernel, stride, padding, bias, stem or not), in both directions, with one row per geometry."""
    seen = _record_geometries(model_key, monkeypatch)
    want = [_geometry(r) for r in MODELS[model_key]]
    assert len(set(want)) == len(want)
    assert seen == set(want), f"in the model only: {sorted(seen - set(want))}; in the table only: {sorted(set(want) - seen)}"
    assert len(want) == {"resnet18": 12, "vgg16": 12, "deit_s": 5}[model_key]


def test_config_wgrad_plans_on_h100():
    """The mirror of the wgrad host code gives every row the plan its table states on a 132-SM H100, and the rows reach
    what the tables say they reach."""
    for r in ALL_ROWS:
        plan = wgrad_plan(_npix(r, r.batch), _kcols(r), _cout_p(r), H100_SMS)
        assert (plan.splits, plan.sl, plan.kbps, plan.last) == r.plan, r.id
    fc0 = next(r for r in VGG if r.cin == 25088)
    p = wgrad_plan(_npix(fc0, 512), _kcols(fc0), fc0.cout, H100_SMS)
    assert (fc0.cin + 63) // 64 == 392 and p.tiles == 3136 and p.splits == 1 and 410e6 < p.ws_bytes < 412e6
    assert {_cout_p(r) for r in ALL_ROWS if _cout_p(r) != r.cout} == {16, 104}
    assert all(_npix(r, 512) % 128 == 0 for r in DEIT) and _npix(DEIT_RAGGED, 37) % 128 == 121
    assert {_pq(r) ** 2 for r in CONV_ROWS if r.stride == 1} >= {16, 4}
    assert {p[1] for p in (r.plan for r in ALL_ROWS)} == {1, 2, 4, 8}


# ---------------------------------------------------------------- bf16 convolutions -------------------------------------------
def _synflow_mask(m, g):
    """SynFlow-like structure at 95 % sparsity: 5 % of the weights live, dead filters (output channels 64..127 and a few
    single ones) and a dead block of input channels (0..63 under every tap), so whole 64x64 blocks of the fprop, dgrad and
    wgrad operands are empty."""
    m.mul_((torch.rand(m.shape, generator=g, device=m.device) < 0.1).float())
    m[64:128] = 0
    m[[3, m.shape[0] - 7]] = 0
    m[:, :64] = 0


# (row, structured zeros): every conv row with the mask at 50 %, plus VGG's small extents at 95 % with SynFlow's structure
# and a whole empty wgrad tile at 2x2
CONV_CASES = [(r, None) for r in CONV_ROWS] + [(r, "synflow") for r in VGG if r.id in ("vgg.3x3.128@16", "vgg.3x3.512@4",
                                                                                         "vgg.3x3.512@2")] \
    + [(r, "tile") for r in VGG if r.id == "vgg.3x3.512@2"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=[r.id + (f".{d}" if d else "") for r, d in CONV_CASES])
def test_conv_bf16_exact(dev, case):
    """fprop (+ bias, + the epilogue statistics where the step asks for them), dgrad (+ the skip addend where the step
    adds one) and wgrad (+ the bias gradient) of one convolution row through ops.conv_* equal the exact result bit for
    bit; with structured zeros both K-block walks run and the occupancy masks report empty blocks.  The split-K
    workspace is NaN before every wgrad call."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    row, dead = case
    n, hw, cin, cout, k, st, pad = row.batch, row.hw, row.cin, row.cout, row.k, row.stride, row.pad
    sms = _sms()
    desc = ops.make_desc(n, hw, hw, cin, cout, k, k, (st, st), (pad, pad))
    plan = wgrad_plan(n * desc.p * desc.q, k * k * cin, cout, sms)
    assert lib.tp_conv_workspace_bytes(ctypes.byref(desc), 2) == plan.ws_bytes
    _assert_plan(plan, row.plan, sms)
    stats, has_add = "s" in row.epi, "a" in row.epi

    g = torch.Generator(device=dev).manual_seed(_seed(row.id, dead))
    x = _ints(g, (n, hw, hw, cin), -1, 1, dev)
    w = _signs(g, (cout, cin, k, k), dev)
    m = (torch.rand(cout, cin, k, k, generator=g, device=dev) < 0.5).float()
    if dead == "synflow":
        _synflow_mask(m, g)
    else:
        _kill_blocks(m, dead)
    bias = torch.randint(-8, 9, (cout,), generator=g, device=dev).float() if row.bias else None
    dy = _ints(g, (n, desc.p, desc.q, cout), -1, 1, dev)
    add = _ints(g, (n, hw, hw, cin), -8, 8, dev) if has_add else None

    outs = {}
    for skip in ((True, False) if dead else (True,)):
        ops.set_kblock_skip(skip)
        try:
            wf, wd = ops.stage_weights(w, m, cin, True, cout)
            if dead and skip:
                assert ops.kblock_occupancy(wf.kmask, wf.shape[1])[0] > 0
                assert ops.kblock_occupancy(wd.kmask, wd.shape[1])[0] > 0
            o = {}
            o["y"], o["stats"] = ops.conv_fprop(desc, x, wf, bias, want_stats=True) if stats else (ops.conv_fprop(desc, x, wf, bias), None)
            o["dx"] = ops.conv_dgrad(desc, dy, wd, addend=add)
            wsb = ops._workspace(lib.tp_conv_workspace_bytes(ctypes.byref(desc), 2), dev, "wgrad")
            wsb[: wsb.numel() // 4 * 4].view(torch.float32).fill_(float("nan"))
            o["dw"], o["db"] = ops.conv_wgrad(desc, x, dy, m, cin, want_db=row.bias, kmask=wf.kmask if skip else None)
            outs[skip] = o
            del wf, wd
        finally:
            ops.set_kblock_skip(True)

    wm = (w * m).double()
    dw_ref = torch.zeros(cout, cin, k, k, dtype=torch.float64, device=dev)
    dw_s = torch.zeros_like(dw_ref)
    for sl in _per_batch(n, hw * hw * max(cin, cout)):
        x64, dy64 = _nchw64(x[sl]), _nchw64(dy[sl])
        S = F.conv2d(x64.abs(), wm.abs(), None, st, pad)
        _bounded(S, 1.0, "fprop")
        ref = _exact(F.conv2d(x64, wm, None, st, pad), 1.0)
        if bias is not None:
            ref += bias.double().view(1, -1, 1, 1)
        ref, S = ref.permute(0, 2, 3, 1).to(torch.bfloat16), S.permute(0, 2, 3, 1)
        for skip, o in outs.items():
            _same(o["y"][sl], ref, S, f"{row.id} fprop (K-block skipping {skip})")
        S = conv2d_input(x64.shape, wm.abs(), dy64.abs(), st, pad)
        _bounded(S, 1.0, "dgrad")
        ref = _exact(conv2d_input(x64.shape, wm, dy64, st, pad), 1.0)
        if add is not None:
            ref += _nchw64(add[sl])
        ref, S = ref.permute(0, 2, 3, 1).to(torch.bfloat16), S.permute(0, 2, 3, 1)
        for skip, o in outs.items():
            _same(o["dx"][sl], ref, S, f"{row.id} dgrad (K-block skipping {skip})")
        del S, ref
        dw_ref += conv2d_weight(x64, w.shape, dy64, st, pad)
        dw_s += conv2d_weight(x64.abs(), w.shape, dy64.abs(), st, pad)
        del x64, dy64
    _bounded(dw_s, 1.0, "wgrad")
    dw_ref = _exact(dw_ref, 1.0) * m.double()
    db_ref, db_s = dy.double().sum(dim=(0, 1, 2)), dy.abs().double().sum(dim=(0, 1, 2))
    _bounded(db_s, 1.0, "bias gradient")
    for skip, o in outs.items():
        _same(o["dw"], dw_ref, dw_s, f"{row.id} wgrad (K-block skipping {skip})")
        if row.bias:
            _same(o["db"], db_ref, db_s, f"{row.id} bias gradient")
        if stats:
            _check_row_stats(o["y"], o["stats"], f"{row.id} epilogue statistics")


# ---------------------------------------------------------------- layers through autograd ------------------------------------
def _make_layer(row, dev):
    from turboprune_b200.utils.mask_layers import Conv1dMask, ConvMask, LinearMask
    if row.kind in ("stem", "conv"):
        layer = ConvMask(in_channels=row.cin, out_channels=row.cout, kernel_size=row.k, stride=row.stride, padding=row.pad,
                         bias=row.bias)
    elif row.kind == "fc":
        layer = Conv1dMask(row.cin, row.cout, bias=row.bias)
    else:
        layer = LinearMask(in_features=row.cin, out_features=row.cout, bias=row.bias)
    return layer.to(dev)


def _set(layer, w, m, b):
    """Weights, mask and bias of the layer, written in place (the weight shadow keeps the tensors' addresses)."""
    with torch.no_grad():
        layer.weight.copy_(w.view(layer.weight.shape))
        layer.mask.copy_(m.view(layer.mask.shape))
        if b is not None:
            layer.bias.copy_(b)


def _x_shape(row, n):
    if row.kind in ("stem", "conv"):
        return (n, row.cin, row.hw, row.hw)
    return (n, row.hw, row.cin) if row.hw > 1 else (n, row.cin)


def _y_shape(row, n):
    if row.kind in ("stem", "conv"):
        return (n, row.cout, _pq(row), _pq(row))
    return (n, row.hw, row.cout) if row.hw > 1 else (n, row.cout)


def _run_layer(layer, row, x, dy, dtype, shadow=None):
    """y, dx (None for the stem), dW, db of the layer at ``dtype`` through autograd.  ``shadow``: (w0, m0): first a
    WeightStager over [another layer, this layer] stages from w0 / m0, then the layer's own weights and mask are written
    back in place and it stages again; the forward must consume the staged operands (no per-layer staging call)."""
    from turboprune_b200 import _cabi, ops
    layer.weight.grad = None
    if layer.bias is not None:
        layer.bias.grad = None
    x = x.detach().clone()
    if row.kind in ("stem", "conv"):
        x = x.contiguous(memory_format=torch.channels_last)
    x.requires_grad_(row.kind != "stem")
    with ops.compute_precision(dtype):
        if shadow is not None:
            w1, m1 = layer.weight.detach().clone(), layer.mask.clone()
            other = _make_layer(Row("other", "conv", 1, 8, 64, 64, 3, 1, 1, False, "", None, 1), x.device)
            stager = ops.WeightStager([other, layer])
            _set(layer, *shadow, None)
            stager.stage()
            _set(layer, w1, m1, None)              # the same tensors: the cached StageItem table is reused
            stager.stage()
            assert "_tp_staged" in layer.__dict__
            rec = _Recorder(_cabi.load())
            with pytest.MonkeyPatch.context() as mp:
                mp.setattr(_cabi, "_lib", rec)
                y = layer(x)
            assert not {"tp_stage_weights", "tp_stage_weights_f32"} & set(rec.calls), rec.calls
            assert "_tp_staged" not in layer.__dict__
            stager.drop()
        else:
            y = layer(x)
        assert y.dtype == dtype
    y.backward(dy)
    return (y.detach(), x.grad if row.kind != "stem" else None, layer.weight.grad.view(row.cout, row.cin, row.k, row.k),
            layer.bias.grad if layer.bias is not None else None)


def _ref64(row, x, wm, dy):
    """float64 y, dx, dW (unmasked), db and their S (the same sums of the absolute operands), from NCHW / [rows, cin]."""
    out = {}
    if row.kind in ("stem", "conv"):
        x64, dy64 = x.double(), dy.double()
        st, pad = row.stride, row.pad
        out["y"] = (F.conv2d(x64, wm, None, st, pad), F.conv2d(x64.abs(), wm.abs(), None, st, pad))
        if row.kind == "conv":
            out["dx"] = (conv2d_input(x64.shape, wm, dy64, st, pad), conv2d_input(x64.shape, wm.abs(), dy64.abs(), st, pad))
        out["dw"] = (conv2d_weight(x64, wm.shape, dy64, st, pad), conv2d_weight(x64.abs(), wm.shape, dy64.abs(), st, pad))
        out["db"] = (dy64.sum(dim=(0, 2, 3)), dy64.abs().sum(dim=(0, 2, 3)))
        return out
    x64, dy64, w2 = x.reshape(-1, row.cin).double(), dy.reshape(-1, row.cout).double(), wm.view(row.cout, row.cin)
    out["y"] = (x64 @ w2.t(), x64.abs() @ w2.abs().t())
    out["dx"] = (dy64 @ w2, dy64.abs() @ w2.abs())
    out["dw"] = ((dy64.t() @ x64).view(wm.shape), (dy64.abs().t() @ x64.abs()).view(wm.shape))
    out["db"] = (dy64.sum(0), dy64.abs().sum(0))
    return out


def _check_layer(row, got, x, w, m, b, dy, dtype, what):
    """Every output of _run_layer against float64: y / dx rounded to bf16 (bf16) or exact (float32), dW exact and masked
    (exactly cout rows for a padded classifier; masked weights exactly 0), db exact."""
    y, dx, dw, db = got
    wm = (w * m).double()
    ref = _ref64(row, x, wm, dy)
    rnd = (lambda t: t.to(torch.bfloat16)) if dtype == torch.bfloat16 else (lambda t: t)
    v, S = ref["y"]
    _bounded(S, 1.0, f"{what} fprop")
    v = _exact(v, 1.0)
    if b is not None:
        v = v + (b.double().view(1, -1, 1, 1) if row.kind in ("stem", "conv") else b.double())
    _same(y.reshape(v.shape), rnd(v), S, f"{what} output")
    if dx is not None:
        v, S = ref["dx"]
        _bounded(S, 1.0, f"{what} dgrad")
        _same(dx.reshape(v.shape), rnd(_exact(v, 1.0)), S, f"{what} input gradient")
    v, S = ref["dw"]
    assert tuple(dw.shape) == tuple(w.shape) == (row.cout, row.cin, row.k, row.k), (tuple(dw.shape), row.cout)
    _bounded(S, 1.0, f"{what} wgrad")
    _same(dw, _exact(v, 1.0) * m.double(), S, f"{what} weight gradient")
    assert bool((dw[m == 0] == 0).all())
    if b is not None:
        v, S = ref["db"]
        assert tuple(db.shape) == (row.cout,)
        _bounded(S, 1.0, f"{what} bias gradient")
        _same(db, v, S, f"{what} bias gradient")


def _bitwise(a, b, what):
    for name, u, v in zip(("output", "input gradient", "weight gradient", "bias gradient"), a, b):
        if u is None or v is None:
            assert u is None and v is None, (what, name)
            continue
        _same(u, v.double(), None, f"{what}: {name} through the weight shadow against the per-layer run")


def _bf16_operands(row, g, dev, n):
    w = _signs(g, (row.cout, row.cin, row.k, row.k), dev)
    m = (torch.rand(row.cout, row.cin, row.k, row.k, generator=g, device=dev) < 0.5).float()
    b = torch.randint(-8, 9, (row.cout,), generator=g, device=dev).float() if row.bias else None
    x = _ints(g, _x_shape(row, n), -1, 1, dev)
    if row.kind == "stem":
        x = x.float()                                  # fp32 input: the stem converts while gathering
    dy = _ints(g, _y_shape(row, n), -1, 1, dev)
    if row.kind in ("stem", "conv"):
        dy = dy.contiguous(memory_format=torch.channels_last)
    return w, m, b, x, dy


BF16_LAYER_CASES = LAYER_ROWS + SHADOW_ROWS


@pytest.mark.gpu
@pytest.mark.parametrize("row", BF16_LAYER_CASES, ids=[r.id for r in BF16_LAYER_CASES])
def test_layer_bf16_exact(dev, row):
    """Stems, classifiers and linears (and one convolution per model) at bf16 through the layers' own autograd path:
    output, input gradient, weight gradient and bias gradient equal the exact result bit for bit; a padded classifier
    returns exactly cout rows of dW and db.  Then the same operands through the weight shadow (staged from other
    weights and another mask first, written in place, staged again): bit for bit the per-layer result."""
    n = row.batch
    sms = _sms()
    plan = wgrad_plan(_npix(row, n), _kcols(row), _cout_p(row), sms)
    _assert_plan(plan, row.plan, sms)
    g = torch.Generator(device=dev).manual_seed(_seed(row.id, "bf16"))
    w, m, b, x, dy = _bf16_operands(row, g, dev, n)
    layer = _make_layer(row, dev)
    _set(layer, w, m, b)
    per_layer = _run_layer(layer, row, x, dy, torch.bfloat16)
    _check_layer(row, per_layer, x, w, m, b, dy, torch.bfloat16, row.id)
    w0 = _signs(g, w.shape, dev) * 2
    m0 = (torch.rand(m.shape, generator=g, device=dev) < 0.7).float()
    shadow = _run_layer(layer, row, x, dy, torch.bfloat16, shadow=(w0, m0))
    _bitwise(shadow, per_layer, row.id)


# ---------------------------------------------------------------- float32 ------------------------------------------------------
F32_XMAX = {"vgg.fc0.25088-4096": 511}       # K = 25 088: odd |x| up to 511 keeps S below 2^22 (asserted)


@pytest.mark.gpu
@pytest.mark.parametrize("row", ALL_ROWS, ids=[r.id for r in ALL_ROWS])
def test_layer_fp32_exact(dev, row):
    """Every row at float32 through MaskedConv2dFn, with the method of test_fp32_training:

    - fprop / dgrad: odd integers in [257, 1023] (511 for K = 25 088) for x and dy, exact in TF32 and not in bf16, weights
      in {-1, 0, 1}: y and dx equal float64 bit for bit; the stem, the linears and one conv per model then run again
      through the weight shadow and equal that run bit for bit;
    - wgrad: x odd up to 2^15 (not bf16; hi + lo exact), dy sparse signs: dW (one bf16 wgrad over the 3N-image split
      stacks, its plan mirrored against the library's workspace size) and db equal float64 bit for bit."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    n = row.f32_batch
    g = torch.Generator(device=dev).manual_seed(_seed(row.id, "fp32"))
    w = torch.randint(-1, 2, (row.cout, row.cin, row.k, row.k), generator=g, device=dev).float()
    m = (torch.rand(w.shape, generator=g, device=dev) < 0.5).float()
    b = torch.randint(-8, 9, (row.cout,), generator=g, device=dev).float() if row.bias else None
    layer = _make_layer(row, dev)
    _set(layer, w, m, b)

    x = _odd(g, _x_shape(row, n), 257, F32_XMAX.get(row.id, 1023), dev)
    _not_bf16(x, "x"); _tf32_exact(x, "x")
    dy = _odd(g, _y_shape(row, n), 257, 1023, dev)
    _not_bf16(dy, "dy")
    got = _run_layer(layer, row, x, dy, torch.float32)
    # y and dx (the weight gradient is checked on the operands of the split-stack run below)
    wm = (w * m).double()
    ref = _ref64(row, x, wm, dy)
    v, S = ref["y"]
    _bounded(S, 1.0, "fp32 fprop")
    if b is not None:
        v = v + (b.double().view(1, -1, 1, 1) if row.kind in ("stem", "conv") else b.double())
    _same(got[0].reshape(v.shape), torch.round(v), S, f"{row.id} float32 fprop")
    if row.kind != "stem":
        v, S = ref["dx"]
        _bounded(S, 1.0, "fp32 dgrad")
        _same(got[1].reshape(v.shape), torch.round(v), S, f"{row.id} float32 dgrad")
    del ref, v, S
    if row.kind != "conv" or row.id in SHADOW_CONVS:
        w0 = torch.randint(-2, 3, w.shape, generator=g, device=dev).float()
        m0 = (torch.rand(m.shape, generator=g, device=dev) < 0.7).float()
        shadow = _run_layer(layer, row, x, dy, torch.float32, shadow=(w0, m0))
        _bitwise(shadow[:2], got[:2], f"{row.id} float32")

    # weight and bias gradients from the split stacks
    npix = _npix(row, n)
    if row.kind == "stem":
        d3 = ops._cabi.ConvDesc(3 * npix, 1, 1, _kcols(row), row.cout, 1, 1, 1, 1, 0, 0, 1, 1)
    elif row.kind == "conv":
        d3 = ops.make_desc(3 * n, row.hw, row.hw, row.cin, row.cout, row.k, row.k, (row.stride,) * 2, (row.pad,) * 2)
    else:
        d3 = ops._cabi.ConvDesc(3 * npix, 1, 1, row.cin, _cout_p(row), 1, 1, 1, 1, 0, 0, 1, 1)
    plan = wgrad_plan(3 * npix, _kcols(row), _cout_p(row), _sms())
    assert lib.tp_conv_workspace_bytes(ctypes.byref(d3), 2) == plan.ws_bytes
    x = _odd(g, _x_shape(row, n), 257, 2 ** 15 - 1, dev)
    _not_bf16(x, "x")
    q = min(1 / 64, 2.0 ** 21 / (npix * 2 ** 15))
    dy = _sparse_signs(g, _y_shape(row, n), q, dev)
    got = _run_layer(layer, row, x, dy, torch.float32)
    ref = _ref64(row, x, wm, dy)
    v, S = ref["dw"]
    _bounded(S, 1.0, "fp32 wgrad")
    assert tuple(got[2].shape) == tuple(w.shape)
    _same(got[2], torch.round(v) * m.double(), S, f"{row.id} float32 wgrad")
    assert bool((got[2][m == 0] == 0).all())
    if b is not None:
        v, S = ref["db"]
        assert tuple(got[3].shape) == (row.cout,)
        _same(got[3], v, S, f"{row.id} float32 bias gradient")


# ---------------------------------------------------------------- ResNet-18 BatchNorm ------------------------------------------
# The BatchNorm calls of a ResNet-18 CIFAR step at batch 512 (every forward takes the conv epilogue's statistics rows).
# Backward: bn1 of every block feeds conv2 (stride 1), whose dgrad does its reduction ("ext"); the stem's BatchNorm feeds
# layer1.0.conv1, which adds the skip gradient instead, so it recomputes its gate from y ("relu2").
RN18_BN_TABLE = [
    BnCase("rn18.stem.bn1", 512 * 32 * 32, 64, True, False, "relu2", False),
    BnCase("rn18.l1.bn1", 512 * 32 * 32, 64, True, False, "ext", False),
    BnCase("rn18.l1.bn2+id", 512 * 32 * 32, 64, True, True, "relu1+dres", False),
    BnCase("rn18.l2.bn1", 512 * 16 * 16, 128, True, False, "ext", False),
    BnCase("rn18.l2.bn2+id", 512 * 16 * 16, 128, True, True, "relu1+dres", False),
    BnCase("rn18.l2.ds", 512 * 16 * 16, 128, False, False, "relu0", False),
    BnCase("rn18.l3.bn1", 512 * 8 * 8, 256, True, False, "ext", False),
    BnCase("rn18.l3.bn2+id", 512 * 8 * 8, 256, True, True, "relu1+dres", False),
    BnCase("rn18.l3.ds", 512 * 8 * 8, 256, False, False, "relu0", False),
    BnCase("rn18.l4.bn1", 512 * 4 * 4, 512, True, False, "ext", False),
    BnCase("rn18.l4.bn2+id", 512 * 4 * 4, 512, True, True, "relu1+dres", False),
    BnCase("rn18.l4.ds", 512 * 4 * 4, 512, False, False, "relu0", False),
]
# paths of _missed_bn_paths a row does not reach on 132 SMs: at M = 8192, C = 512 the grid (512 x 4 threads) covers the
# pixels exactly, so neither pixel loop has a tail; every other row reaches every path
RN18_BN_MISSED = {c.id: (["4-row tail loop", "2-row tail loop"] if c.M == 8192 else []) for c in RN18_BN_TABLE}


def test_rn18_bn_geom_on_h100():
    """The paths each ResNet-18 BatchNorm row reaches on a 132-SM H100, as the table states; both ways of folding the
    external rows occur (fold groups at M >= 128 k, a direct fold below)."""
    for c in RN18_BN_TABLE:
        assert _missed_bn_paths(bn_geom(c.M, c.C, H100_SMS), c) == RN18_BN_MISSED[c.id], c.id
    assert {bn_geom(c.M, c.C, H100_SMS).fold_ext for c in RN18_BN_TABLE if c.bwd == "ext"} == {True, False}


def _rn18_bn_geom(case):
    from turboprune_b200 import _cabi
    sms = _sms()
    geom = bn_geom(case.M, case.C, sms)
    assert int(_cabi.load().tp_bn_workspace_bytes(case.M, case.C)) == geom.ws_bytes
    if sms == H100_SMS:
        assert _missed_bn_paths(geom, case) == RN18_BN_MISSED[case.id]
    return geom


@pytest.mark.gpu
@pytest.mark.parametrize("case", RN18_BN_TABLE, ids=[c.id for c in RN18_BN_TABLE])
def test_rn18_bn_forward_exact(dev, case):
    """The checks of test_step_kernels_exact.test_bn_forward_exact at ResNet-18's BatchNorm extents."""
    bn_forward_check(dev, case, _rn18_bn_geom(case))


@pytest.mark.gpu
@pytest.mark.parametrize("case", RN18_BN_TABLE, ids=[c.id for c in RN18_BN_TABLE])
def test_rn18_bn_backward_exact(dev, case):
    """The checks of test_step_kernels_exact.test_bn_backward_exact at ResNet-18's BatchNorm extents."""
    bn_backward_check(dev, case, _rn18_bn_geom(case))


RN18_BNB_CASES = [("rn18.l1.conv2.64@32", 512, 32, 64, 64, 3), ("rn18.l2.conv2.128@16", 512, 16, 128, 128, 3),
                  ("rn18.l3.conv2.256@8", 512, 8, 256, 256, 3), ("rn18.l4.conv2.512@4", 512, 4, 512, 512, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", RN18_BNB_CASES, ids=[c[0] for c in RN18_BNB_CASES])
def test_rn18_bn_backward_dgrad_epilogue_exact(dev, case):
    """The checks of test_kernel_exactness.test_bn_backward_dgrad_epilogue_exact on conv2 of each ResNet-18 stage."""
    bnb_dgrad_check(dev, case)


# ---------------------------------------------------------------- GPU: the tables against real steps ------------------------
def _desc(d):
    return tuple(getattr(d, f) for f, _ in type(d)._fields_)


def _expected_conv_calls(rows, n, dtype):
    """Every (entry point, ConvDesc fields, epilogue operands) a forward and backward at batch n makes for these rows.
    The stem runs fprop and wgrad as one GEMM over n P Q im2col rows of K = taps * cin padded to 8; a linear is a 1x1
    convolution over its rows; the backward GEMMs walk cout_p output channels; the float32 weight gradient is one bf16
    wgrad over the 3n images of the split stacks, without a bias gradient."""
    want = set()
    for r in rows:
        pq, cp = _pq(r), _cout_p(r)
        if r.kind == "stem":
            f = (n * pq * pq, 1, 1, _kcols(r), r.cout, 1, 1, 1, 1, 0, 0, 1, 1)
            wd = f
        elif r.kind == "conv":
            f = (n, r.hw, r.hw, r.cin, r.cout, r.k, r.k, r.stride, r.stride, r.pad, r.pad, pq, pq)
            wd = f[:4] + (cp,) + f[5:]
        else:
            f = (n * r.hw, 1, 1, r.cin, r.cout, 1, 1, 1, 1, 0, 0, 1, 1)
            wd = f[:4] + (cp,) + f[5:]
        if dtype == torch.bfloat16:
            want.add(("fprop", f, r.bias, "s" in r.epi))
            want.add(("wgrad", wd, r.bias))
            if r.kind != "stem":
                if "b" in r.epi:
                    want.add(("dgrad_bnrelu", wd))
                if "a" in r.epi:
                    want.add(("dgrad", wd, True))
                if not set(r.epi) & set("ab"):
                    want.add(("dgrad", wd, False))
        else:
            want.add(("fprop_f32", f, r.bias))
            want.add(("wgrad", (3 * wd[0],) + wd[1:], False))
            if r.kind != "stem":
                want.add(("dgrad_f32", wd))
    return want


def _model(model_key, dtype, dev):
    from refshim import make_cfg
    from turboprune_b200.utils import custom_models as cm
    (name, data, mlt), hw = MODEL_CFGS[model_key]
    torch.manual_seed(0)
    cfg = make_cfg(name, data, mask_layer_type=mlt, precision="bfloat16" if dtype == torch.bfloat16 else "float32")
    model = cm.CustomModel(cfg) if mlt == "LinearMask" else cm.TorchVisionModel(cfg)
    return model.to(dev).train(), hw


def _step(model, hw, n, dtype, dev):
    from turboprune_b200 import ops
    x = torch.randn(n, 3, hw, hw, device=dev).contiguous(memory_format=torch.channels_last)
    if dtype == torch.bfloat16:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(x)
    else:
        with ops.compute_precision(torch.float32):
            out = model(x)
    out.float().square().mean().backward()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("model_key", list(MODELS))
def test_conv_calls_match_the_tables(dev, model_key, dtype, monkeypatch):
    """One forward and backward of the model at batch 2 with the convolution entry points wrapped: the set of (entry
    point, ConvDesc read through the byref argument, epilogue operands present: bias, statistics, skip addend) the step
    issues equals the set the table gives at batch 2, in both directions."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    n = 2
    seen = set()

    def record(name, key):
        fn = getattr(lib, name)

        def wrapped(*a):
            seen.add(key(a))
            return fn(*a)
        monkeypatch.setattr(lib, name, wrapped)

    record("tp_conv_fprop_stats", lambda a: ("fprop", _desc(a[0]._obj), a[4] is not None, a[6] is not None))
    record("tp_conv_dgrad", lambda a: ("dgrad", _desc(a[0]._obj), a[4] is not None))
    record("tp_conv_dgrad_bnrelu", lambda a: ("dgrad_bnrelu", _desc(a[0]._obj)))
    record("tp_conv_wgrad", lambda a: ("wgrad", _desc(a[0]._obj), a[7] is not None))
    record("tp_conv_fprop_f32", lambda a: ("fprop_f32", _desc(a[0]._obj), a[3] is not None))
    record("tp_conv_dgrad_f32", lambda a: ("dgrad_f32", _desc(a[0]._obj)))
    model, hw = _model(model_key, dtype, dev)
    _step(model, hw, n, dtype, dev)
    want = _expected_conv_calls(MODELS[model_key], n, dtype)
    assert seen == want, f"issued but not in the table: {sorted(seen - want)}; in the table but not issued: {sorted(want - seen)}"


@pytest.mark.gpu
def test_bn_case_table_matches_resnet18_step(dev, monkeypatch):
    """One ResNet-18 CIFAR forward and backward at batch 2 (bf16) with the BatchNorm entry points wrapped: every
    (entry point, M scaled to batch 512, C, ReLU mode, residual) the step issues is a row of RN18_BN_TABLE, and every
    row is issued."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    n = 2
    s = 512 // n
    seen = set()

    def record(name, key):
        fn = getattr(lib, name)

        def wrapped(*a):
            seen.add(key(a))
            return fn(*a)
        monkeypatch.setattr(lib, name, wrapped)

    record("tp_bn_forward_ext", lambda a: ("forward", a[3] * s, a[4], bool(a[13]), a[1] is not None, a[16] is not None))
    record("tp_bn_forward", lambda a: ("forward", a[3] * s, a[4], bool(a[13]), a[1] is not None, False))
    record("tp_bn_backward", lambda a: ("backward", a[3] * s, a[4], int(a[9]), a[11] is not None))
    record("tp_bn_backward_ext", lambda a: ("backward_ext", a[2] * s, a[3]))
    model, hw = _model("resnet18", torch.bfloat16, dev)
    _step(model, hw, n, torch.bfloat16, dev)
    want = set().union(*(_table_keys(c) for c in RN18_BN_TABLE))
    assert seen == want, f"issued but not in the table: {sorted(seen - want)}; in the table but not issued: {sorted(want - seen)}"
