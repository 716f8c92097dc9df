"""Work-item scheduling of the fprop / dgrad kernel: the CTA's work items alternate between two consumer warpgroups,
which take turns running their K loops and hand the position in the shared stage ring over with the turn.  These
cases put that hand-over at its edges and check the results against the oracle or against the dense walk:
CTAs with a single item and with an odd number of items, consecutive items with different K-block counts, and
strided dgrad whose parity classes have no taps (items without a K loop) between classes with taps.

The kernel is persistent with grid = min(items, SMs) and CTA b runs items b, b + grid, b + 2 grid, ...; the helpers
below count the items the way the host code does (tp_igemm.cu: pick_block_n, launch_fwd, conv_dgrad_impl), so every
case asserts the item count it needs instead of silently running one item per CTA."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a = a.detach().float().cpu(); b = b.detach().float().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _block_n(m_tiles, n):
    """pick_block_n: the tile width whose last wave is fullest, 64-wide tiles weighted 0.82."""
    sms, best, best_score = _sms(), 64, -1.0
    for bn, weight in ((128, 1.0), (64, 0.82)):
        if bn > 64 and n <= bn // 2:
            continue
        tiles = m_tiles * ((n + bn - 1) // bn)
        eff = tiles / (math.ceil(tiles / sms) * sms) * weight
        if eff > best_score:
            best_score, best = eff, bn
    return best


def _items(class_pixels, n):
    """(work items, N tiles) of one launch: per class ceil(M / 128) M tiles x the N tiles, classes back to back."""
    m_tiles = [(m + 127) // 128 for m in class_pixels]
    n_tiles = (n + _block_n(sum(m_tiles), n) - 1) // _block_n(sum(m_tiles), n)
    return sum(m_tiles) * n_tiles, n_tiles


def _fprop_items(n, hw, cout, r, s, stride, pad):
    p = (hw + 2 * pad - r) // stride + 1
    q = (hw + 2 * pad - s) // stride + 1
    return _items([n * p * q], cout)


def _dgrad_items(n, hw, cin, stride):
    """dgrad of a stride-s convolution: s x s parity classes of the input pixels (one class at stride 1)."""
    cls = [n * ((hw - a + stride - 1) // stride) * ((hw - b + stride - 1) // stride) for a in range(stride) for b in range(stride)]
    return _items([m for m in cls if m > 0], cin)


def _dgrad_tapped(r, s, stride, pad):
    """Which parity classes (a, b), in launch order, have at least one tap."""
    return [any((a + pad - i) % stride == 0 for i in range(r)) and any((b + pad - j) % stride == 0 for j in range(s))
            for a in range(stride) for b in range(stride)]


def _conv_vs_oracle(n, hw, cin, cout, r, s, stride, pad, seed, addend=False):
    """fprop (with the epilogue's BatchNorm statistics) and dgrad (optionally with the fused addend) of one masked
    convolution against the oracle on the same bf16 operands."""
    from turboprune_b200 import ops
    from oracle import mask_ops as R
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, hw, hw, generator=g).to(torch.bfloat16)
    wt = torch.randn(cout, cin, r, s, generator=g) / (cin * r * s) ** 0.5
    mk = (torch.rand(cout, cin, r, s, generator=g) < 0.3).float()
    desc = ops.make_desc(n, hw, hw, cin, cout, r, s, (stride, stride), (pad, pad))
    xn = x.cuda().permute(0, 2, 3, 1).contiguous()
    wf, wd = ops.stage_weights(wt.cuda(), mk.cuda(), cin, True, cout)
    y, stats = ops.conv_fprop(desc, xn, wf, want_stats=True)
    yr = R.masked_conv2d(x.float(), wt, mk, None, stride, pad, bf16_operands=True)
    assert _rel(y.permute(0, 3, 1, 2), yr) < 4e-3
    # the statistics are sums of exactly the bf16 values stored
    yf = y.float().reshape(-1, cout)
    assert torch.allclose(stats[:, 0].sum(0), yf.sum(0), rtol=1e-4, atol=1e-2)
    assert torch.allclose(stats[:, 1].sum(0), (yf * yf).sum(0), rtol=1e-4, atol=1e-2)
    dy = torch.randn(yr.shape, generator=g).to(torch.bfloat16)
    add = torch.randn(n, hw, hw, cin, generator=g).to(torch.bfloat16) if addend else None
    dx = ops.conv_dgrad(desc, dy.cuda().permute(0, 2, 3, 1).contiguous(), wd, addend=add.cuda() if addend else None)
    dxr, _, _ = R.masked_conv2d_grads(x.float(), wt, mk, dy.float(), stride, pad, bf16_operands=True, has_bias=False)
    if addend:
        dxr = dxr + add.permute(0, 3, 1, 2).float()
    assert _rel(dx.permute(0, 3, 1, 2), dxr) < 4e-3


@pytest.mark.parametrize("items_per_sm", ["few", "odd"])
def test_item_counts_per_cta(dev, items_per_sm):
    """1x1 convolution with 64 channels in and out, one 128-pixel M tile per two 8x8 images: 'few' gives most CTAs one
    item and a few CTAs two (fewer items than 2 x grid), 'odd' gives one CTA four items and every other CTA three."""
    sms = _sms()
    tiles = sms + 5 if items_per_sm == "few" else 3 * sms + 1
    n = 2 * tiles
    for items, _ in (_fprop_items(n, 8, 64, 1, 1, 1, 0), _dgrad_items(n, 8, 64, 1)):
        assert items == tiles
    _conv_vs_oracle(n, 8, 64, 64, 1, 1, 1, 0, seed=tiles, addend=True)


@pytest.mark.parametrize("case", [(256, 14, 64, 128, 2, 1, 2, 0), (256, 14, 64, 128, 1, 1, 2, 0), (192, 14, 64, 64, 3, 3, 2, 1)])
def test_strided_dgrad_classes_without_taps(dev, case):
    """Strided dgrad, all parity classes in one launch, at least three items per CTA.  2x1 stride 2: classes (0,1) and
    (1,1) have no taps and alternate with the two that do, so a CTA runs a tapped item, a tapless one, a tapped one.
    1x1 stride 2: tapped items, then three classes of tapless ones.  3x3 stride 2: 1, 2, 2 and 4 taps per class."""
    n, hw, cin, cout, r, s, stride, pad = case
    items, _ = _dgrad_items(n, hw, cin, stride)
    assert items > 2 * _sms(), (items, _sms())
    tapped = _dgrad_tapped(r, s, stride, pad)
    if (r, s) == (2, 1):
        assert tapped == [True, False, True, False]
        # the CTA whose items are the first tiles of classes 0, 1, 2 meets tapped -> tapless -> tapped
        per_class = items // 4
        assert per_class <= _sms() < 2 * per_class <= 2 * _sms() < 3 * per_class
    elif (r, s) == (1, 1):
        assert tapped == [True, False, False, False]
    _conv_vs_oracle(n, hw, cin, cout, r, s, stride, pad, seed=sum(case), addend=True)


@pytest.mark.parametrize("case", [(160, 12, 192, 576, 3, 1, 1), (128, 14, 576, 192, 1, 1, 0)])
def test_alternating_kblock_counts_bit_identical_to_dense_walk(dev, case):
    """An occupancy mask whose empty 64x64 weight blocks differ between output-channel tiles, at several items per CTA.
    With 576 GEMM columns (fprop of the first case, dgrad of the second) the N-tile count (5 or 9) does not divide the
    grid, so consecutive items of a CTA fall on different N tiles and have different K-block counts.  fprop and dgrad
    with block skipping equal the dense walk bit for bit; the dense walk matches the oracle."""
    from turboprune_b200 import ops
    from oracle import mask_ops as R
    n, hw, cin, cout, k, s, p = case
    sms = _sms()
    f_items, f_nt = _fprop_items(n, hw, cout, k, k, s, p)
    d_items, d_nt = _dgrad_items(n, hw, cin, s)
    assert f_items > 2 * sms and d_items > 2 * sms, (f_items, d_items, sms)
    wide_nt = f_nt if cout == 576 else d_nt
    assert sms % wide_nt != 0, (sms, wide_nt)              # consecutive items of a CTA: different N tiles
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(n, cin, hw, hw, generator=g).to(torch.bfloat16)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    mk = (torch.rand(cout, cin, k, k, generator=g) < 0.3).float()
    for j in range(0, cout, 64):            # output-channel group j/64 loses (j/64) % 4 of its first input-channel blocks
        mk[j:j + 64, :64 * ((j // 64) % 4)] = 0
    for j in range(0, cin, 64):             # and the dgrad operand: input-channel group j/64 loses output-channel blocks
        mk[:64 * ((j // 64) % 3), j:j + 64] = 0
    desc = ops.make_desc(n, hw, hw, cin, cout, k, k, (s, s), (p, p))
    xn = x.cuda().permute(0, 2, 3, 1).contiguous()
    dy = torch.randn(n, cout, desc.p, desc.q, generator=g).to(torch.bfloat16)
    dyn = dy.cuda().permute(0, 2, 3, 1).contiguous()
    outs = {}
    for skip in (True, False):
        ops.set_kblock_skip(skip)
        try:
            wf, wd = ops.stage_weights(wt.cuda(), mk.cuda(), cin, True, cout)
            if skip:
                assert ops.kblock_occupancy(wf.kmask, wf.shape[1])[0] > 0 and ops.kblock_occupancy(wd.kmask, wd.shape[1])[0] > 0
            outs[skip] = (ops.conv_fprop(desc, xn, wf), ops.conv_dgrad(desc, dyn, wd))
        finally:
            ops.set_kblock_skip(True)
    for a, b in zip(outs[True], outs[False]):
        assert torch.equal(a, b)
    yr = R.masked_conv2d(x.float(), wt, mk, None, s, p, bf16_operands=True)
    dxr, _, _ = R.masked_conv2d_grads(x.float(), wt, mk, dy.float(), s, p, bf16_operands=True, has_bias=False)
    assert _rel(outs[False][0].permute(0, 3, 1, 2), yr) < 4e-3
    assert _rel(outs[False][1].permute(0, 3, 1, 2), dxr) < 4e-3
