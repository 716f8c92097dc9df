"""Exactness of the BatchNorm apply / backward, max-pool and SGD kernels of the train step, against float64.

Same method as test_kernel_exactness.py: operands are chosen so that the exact result is known, every fp32 partial sum
is asserted exact first (S = sum |terms| <= 2^22 quanta), and the kernel output is compared with float64 torch on the GPU,
bit for bit where the arithmetic is exact and against a stated bar where it is not (rsqrtf, divisions by M).

- BatchNorm forward (tp_bn_forward_ext, tp_bn_forward): y takes bf16 integers and the external statistics rows are the
  exact per-32-row sums of y, so save_mean is float32(sum / M) bit for bit.  z is reproduced from the kernel's own scale
  and shift (read from the workspace): bf16(relu(fp32(fp32(fma(y, scale, shift)) + residual))), every fp32 rounding
  taken from the exact float64 value (products of fp32 and small integers are exact in float64; sums are split exactly
  with TwoSum, see _fma32), so z must match bit for bit.
- BatchNorm backward (tp_bn_backward): mean, invstd, weight and bias are dyadic, so the ReLU gate, x-hat, sum g and
  sum g * x-hat are exact; dweight, dbias and dres must equal float64, and dy must equal
  bf16(fma(k0, g, fma(k1, y, k2))) from the kernel's own coefficients.
- The cases are the ResNet-50 BatchNorm layers at batch 512, and every case asserts through a mirror of bn_geom which
  kernel paths it reaches (unrolled pixel loops and their tails, the unrolled 32-lane fold, the external-row fold).  A
  real ResNet-50 step checks that the table lists exactly the BatchNorm calls the step makes.
- Max-pool: post-ReLU integer inputs (half zeros: ties and all-zero windows everywhere), y, the arg-max and dx against
  float64 torch, bit for bit.
- SGD: FusedSGD against torch.optim.SGD (foreach) on ResNet-50's parameter list, weights and momentum buffers bit for bit.
"""
import math
import warnings
from collections import namedtuple
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from test_fwd_pingpong import _sms
from test_kernel_exactness import EXACT, _bounded, _ints, _per_batch, _ptr, _same

H100_SMS = 132              # the BatchNorm plans in the case table are the ones a 132-SM H100 runs
MOMENTUM, EPS = 0.1, 1e-5


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: the gpu-marked tests need an H100")
    from turboprune_b200 import _cabi
    _cabi.load()
    return torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _release_memory():
    """Every case frees its tensors before the next one (the GPU is shared; the stem tensors are 822 MB each)."""
    yield
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


# ---------------------------------------------------------------- mirror of the BatchNorm host code ----------------------
def bn_geom(M, C, sms):
    """bn_geom of tp_bn.cu: (tx, ty) threads per CTA, ctiles channel tiles, grid_x CTAs along the pixels.  Each thread
    walks pixels p0, p0 + stride, ... (stride = grid_x * ty); the statistics / apply kernels take 4 rows per unrolled
    iteration, the backward kernels 2.  ``loop4`` / ``loop2``: (unrolled iterations every thread runs, pixels left to the
    tail loops).  The finalize kernels fold grid_x partial rows (backward) with 32 lanes, 4 rows per unrolled step."""
    cv = C // 8
    tx = 1
    while tx < cv and tx < 256:
        tx <<= 1
    ty = 256 // tx
    ctiles = (cv + tx - 1) // tx
    want = max(1, sms * 4 // ctiles)
    grid_x = max(1, min(((M + ty - 1) // ty + 3) // 4, want))
    stride = grid_x * ty
    full, rest = divmod(M, stride)          # threads p0 < rest walk full + 1 rows, the others full rows

    def loop(u):
        return full // u, rest * ((full + 1) % u) + (stride - rest) * (full % u)

    ext_rows = (M + 127) // 128 * 4         # the conv epilogue's statistics rows (one per 32 pixels, whole 128-pixel tiles)
    groups = (ext_rows + 1023) // 1024
    return SimpleNamespace(tx=tx, ty=ty, ctiles=ctiles, grid_x=grid_x, stride=stride, loop4=loop(4), loop2=loop(2),
                           ext_rows=ext_rows, fold_ext=groups > 1, fwd_nparts=groups if groups > 1 else ext_rows,
                           ws_bytes=grid_x * 2 * C * 4 + 5 * C * 4 + 1024)


def _missed_bn_paths(geom, case):
    """Paths a case exists for that it does not reach under ``geom``: the unrolled pixel loops and their tails (4-row
    statistics / apply kernels, 2-row backward kernels), the unrolled 32-lane fold of the finalize kernels (nparts > 96;
    with external rows it folds either the k_bn_fold_ext groups or, for <= 1024 rows, the rows themselves)."""
    missed = []
    for name, (iters, tail) in (("4-row", geom.loop4), ("2-row", geom.loop2)):
        if iters < 1:
            missed.append(f"{name} unrolled loop")
        if tail <= 0:
            missed.append(f"{name} tail loop")
    ext_bwd = case.bwd == "ext"
    if (case.two_pass or not ext_bwd) and geom.grid_x <= 96:
        missed.append("unrolled fold of the grid_x partial rows")
    if not case.two_pass and not geom.fold_ext and geom.fwd_nparts <= 96:
        missed.append("unrolled fold of the external rows")
    return missed


# (id, M at batch 512, C, forward ReLU, residual, backward path, two-pass statistics)
# backward: "relu2" = tp_bn_backward with the gate recomputed from y, "relu1+dres" = gate from z and the residual gradient,
# "relu0" = no activation, "ext" = tp_bn_backward_ext: the consuming conv's dgrad already gated the gradient and wrote
# per-32-pixel partial sums, the GPU case feeds exact ones (k_bn_fold_ext or a direct fold, k_bn_finalize_bwd,
# k_bn_bwd_apply<0, false>)
BnCase = namedtuple("BnCase", "id M C relu res bwd two_pass")
BN_TABLE = [
    BnCase("stem.bn1", 512 * 112 * 112, 64, True, False, "relu2", False),
    BnCase("l1.bn1-bn2", 512 * 56 * 56, 64, True, False, "ext", False),
    BnCase("l1.bn3+id", 512 * 56 * 56, 256, True, True, "relu1+dres", False),
    BnCase("l1.ds", 512 * 56 * 56, 256, False, False, "relu0", False),
    BnCase("l2.0.bn1", 512 * 56 * 56, 128, True, False, "relu2", False),          # feeds the stride-2 conv2
    BnCase("l2.bn1-bn2", 512 * 28 * 28, 128, True, False, "ext", False),
    BnCase("l2.bn3+id", 512 * 28 * 28, 512, True, True, "relu1+dres", False),
    BnCase("l2.ds", 512 * 28 * 28, 512, False, False, "relu0", False),
    BnCase("l3.0.bn1", 512 * 28 * 28, 256, True, False, "relu2", False),
    BnCase("l3.bn1-bn2", 512 * 14 * 14, 256, True, False, "ext", False),
    BnCase("l3.bn3+id", 512 * 14 * 14, 1024, True, True, "relu1+dres", False),
    BnCase("l3.ds", 512 * 14 * 14, 1024, False, False, "relu0", False),
    BnCase("l4.0.bn1", 512 * 14 * 14, 512, True, False, "relu2", False),
    BnCase("l4.bn1-bn2", 512 * 7 * 7, 512, True, False, "ext", False),
    BnCase("l4.bn3+id", 512 * 7 * 7, 2048, True, True, "relu1+dres", False),       # ty = 1
    BnCase("l4.ds", 512 * 7 * 7, 2048, False, False, "relu0", False),
]
BN_EXTRA = [
    BnCase("c192.inactive-lanes", 8 * 56 * 56, 192, True, False, "relu2", False),  # tx = 32 lanes for 24 vectors
    BnCase("two-pass.b64-l2", 64 * 28 * 28, 256, True, True, "relu1+dres", True),
    # accepted by the C ABI, never issued by BatchNorm2dB200
    BnCase("abi.relu0+res", 25000, 256, False, True, "relu0+dres", False),
    BnCase("abi.relu2+res", 25000, 256, True, True, "relu2+dres", False),
]
BN_CASES = BN_TABLE + BN_EXTRA
BWD_MODES = {"relu2": (2, False), "ext": (2, False), "relu1+dres": (1, True), "relu0": (0, False),
             "relu0+dres": (0, True), "relu2+dres": (2, True)}


def test_bn_geom_mirror_on_h100():
    """The mirror of bn_geom gives the 132-SM plans below, and every case reaches the paths it is meant to."""
    g = bn_geom(512 * 112 * 112, 64, H100_SMS)
    assert (g.tx, g.ty, g.ctiles, g.grid_x, g.stride) == (8, 32, 1, 528, 16896)
    assert g.loop4 == (95, 2048) and g.loop2 == (190, 2048)
    plans = {(25088, 2048): (256, 1, 1, 528), (25088, 192): (32, 8, 1, 528), (1000, 64): (8, 32, 1, 8),
             (256, 4096): (256, 1, 2, 64), (1 << 20, 4096): (256, 1, 2, 264), (100352, 512): (64, 4, 1, 528)}
    for (M, C), want in plans.items():
        g = bn_geom(M, C, H100_SMS)
        assert (g.tx, g.ty, g.ctiles, g.grid_x) == want, (M, C)
    for c in BN_CASES:
        assert _missed_bn_paths(bn_geom(c.M, c.C, H100_SMS), c) == [], c.id
    # both ways of folding the external rows occur, in the forward and in tp_bn_backward_ext
    folds = {bn_geom(c.M, c.C, H100_SMS).fold_ext for c in BN_CASES if not c.two_pass}
    assert folds == {True, False}
    assert {bn_geom(c.M, c.C, H100_SMS).fold_ext for c in BN_CASES if c.bwd == "ext"} == {True, False}


# ---------------------------------------------------------------- helpers ---------------------------------------------------
def _f32_ulp(v):
    """Spacing of fp32 numbers at |v| (float64 tensor)."""
    _, ex = torch.frexp(v.abs())
    return torch.where(v == 0, 2.0 ** -149, torch.ldexp(torch.ones_like(v), (ex - 24).clamp_min(-149)))


def _fma32(a, b, c):
    """fp32 of the exact a * b + c, rounded once as fmaf rounds it (a * b must be exact in float64: fp32 times fp32, or
    times a small integer).  TwoSum splits the sum into float64 s + e exactly; s rounded to fp32 is the correctly rounded
    result unless s lies exactly halfway between two fp32 numbers, and there the sign of e decides."""
    p, c = a.double() * b.double(), c.double()
    s = p + c
    v = s - p
    e = (p - (s - v)) + (c - v)
    f = s.float()
    fd = f.double()
    up = s > fd
    g = torch.nextafter(f, torch.where(up, float("inf"), float("-inf")).float())
    mid = (s != fd) & ((s - fd) == (g.double() - fd) / 2)
    return torch.where(mid & (e != 0) & ((e > 0) == up), g, f)


def _within_ulps(got, want, ulps, what, scale=None):
    """|got - want| <= ulps fp32 ulp of ``scale`` (default |want|), per channel."""
    ref = want.abs() if scale is None else scale
    err = (got.double() - want).abs() / _f32_ulp(ref)
    worst = float(err.max())
    assert worst <= ulps, f"{what}: {worst:.2f} fp32 ulp (bar {ulps}) at channel {int(err.argmax())}"
    return worst


def _rows(M, C):
    """Pixel chunks of about 2^23 elements for the float64 passes."""
    step = max(32, (1 << 23) // C // 32 * 32)
    return [(p, min(M, p + step)) for p in range(0, M, step)]


def _sparse_ints(g, M, C, m, density, dev):
    """[M, C] bf16 integers in [-m, m], each kept with probability ``density`` (generated in chunks)."""
    out = torch.empty(M, C, dtype=torch.bfloat16, device=dev)
    for p0, p1 in _rows(M, C):
        v = _ints(g, (p1 - p0, C), -m, m, dev)
        if density < 1:
            v *= (torch.rand(p1 - p0, C, generator=g, device=dev) < density).to(torch.bfloat16)
        out[p0:p1] = v
    return out


def _bn_y(g, M, C, dev):
    """bf16 integer activations: [-m, m] with the widest m in {8, 4, 2, 1} that keeps sum y^2 per channel well below
    2^22; at the stem extent {-1, 0, 1} with half of them zero."""
    for m in (8, 4, 2, 1):
        if M * m * (m + 1) / 3 <= 0.8 * EXACT:
            return _sparse_ints(g, M, C, m, 1.0, dev), m
    return _sparse_ints(g, M, C, 1, 0.5, dev), 1


def _stream(dev):
    from turboprune_b200 import _cabi
    return _cabi.stream_ptr(dev)


def _zeros(t):
    """Number of zeros of an [M, C] tensor, counted in chunks (no full-size temporaries)."""
    return sum(int(torch.count_nonzero(t[p0:p1] == 0)) for p0, p1 in _rows(*t.shape))


def _ws(lib, M, C, dev):
    """Workspace filled with NaN, so that a coefficient read before it is written shows up."""
    ws = torch.empty(int(lib.tp_bn_workspace_bytes(M, C)), dtype=torch.uint8, device=dev)
    ws.view(torch.float32).fill_(float("nan"))
    return ws


def _geom_checked(lib, case):
    """The mirror matches the library's workspace size on this device.  On a 132-SM H100 the case must reach every path
    it exists for; the grid depends on the SM count, so on other devices a path it misses is reported as a warning
    (the exactness checks still run)."""
    sms = _sms()
    geom = bn_geom(case.M, case.C, sms)
    assert int(lib.tp_bn_workspace_bytes(case.M, case.C)) == geom.ws_bytes
    missed = _missed_bn_paths(geom, case)
    if sms == H100_SMS:
        assert not missed, (case.id, missed)
    elif missed:
        warnings.warn(f"{case.id}: on {sms} SMs this case does not reach: {', '.join(missed)}")
    return geom


def _ext_rows(y, rows):
    """Per-32-row sums of y and y^2 ([rows, 2, C] fp32, rows past the last pixel zero), as the conv epilogue writes
    them (exact for integer y: every row sum is far below 2^24)."""
    M, C = y.shape
    ext = torch.zeros(rows, 2, C, dtype=torch.float32, device=y.device)
    for p0, p1 in _rows(M, C):
        seg = y[p0:p1].double()
        pad = (-seg.shape[0]) % 32
        if pad:
            seg = torch.cat([seg, seg.new_zeros(pad, C)])
        seg = seg.view(-1, 32, C)
        ext[p0 // 32:p0 // 32 + seg.shape[0], 0] = seg.sum(1).float()
        ext[p0 // 32:p0 // 32 + seg.shape[0], 1] = (seg * seg).sum(1).float()
    return ext


def _bn_forward(lib, dev, y, res, z, relu, w, b, rm, rv, nbt, sm, si, ext, ws, training=True):
    M, C = y.shape
    with torch.cuda.device(dev):
        stream = _stream(dev)
        if ext is not None:
            rc = lib.tp_bn_forward_ext(_ptr(y), _ptr(res), _ptr(z), M, C, _ptr(w), _ptr(b), _ptr(rm), _ptr(rv), _ptr(nbt),
                                       MOMENTUM, EPS, int(training), int(relu), _ptr(sm), _ptr(si), _ptr(ext), ext.shape[0],
                                       _ptr(ws), ws.numel(), stream)
        else:
            rc = lib.tp_bn_forward(_ptr(y), _ptr(res), _ptr(z), M, C, _ptr(w), _ptr(b), _ptr(rm), _ptr(rv), _ptr(nbt),
                                   MOMENTUM, EPS, int(training), int(relu), _ptr(sm), _ptr(si), _ptr(ws), ws.numel(), stream)
    assert rc == 0, f"tp_bn_forward: {rc}"


def _bn_backward(lib, dev, dz, z, y, relu, w, b, mean, inv, dy, dres, dw, db, ws):
    M, C = y.shape
    with torch.cuda.device(dev):
        rc = lib.tp_bn_backward(_ptr(dz), _ptr(z), _ptr(y), M, C, _ptr(w), _ptr(b), _ptr(mean), _ptr(inv), relu, _ptr(dy),
                                _ptr(dres), _ptr(dw), _ptr(db), _ptr(ws), ws.numel(), _stream(dev))
    assert rc == 0, f"tp_bn_backward: {rc}"


def _gated_partials(dz, y, sc, sf, mean, inv, rows):
    """What the dgrad epilogue hands to tp_bn_backward_ext: g = dz * [fma(y, scale, shift) > 0] (bf16) and per 32 pixels
    [sum g, sum g * xhat] ([rows, 2, C] fp32, rows past the last pixel zero); exact for the dyadic operands used here."""
    M, C = y.shape
    g = torch.empty_like(dz)
    partial = torch.zeros(rows, 2, C, dtype=torch.float32, device=y.device)
    m64, i64 = mean.double(), inv.double()
    for p0, p1 in _rows(M, C):
        yy = y[p0:p1].double()
        gg = torch.where(yy * sc + sf > 0, dz[p0:p1].double(), 0.0)
        g[p0:p1] = gg.to(torch.bfloat16)
        gx = gg * (yy - m64) * i64
        pad = (-gg.shape[0]) % 32
        if pad:
            gg, gx = torch.cat([gg, gg.new_zeros(pad, C)]), torch.cat([gx, gx.new_zeros(pad, C)])
        r0, n = p0 // 32, gg.shape[0] // 32
        partial[r0:r0 + n, 0] = gg.view(n, 32, C).sum(1).float()
        partial[r0:r0 + n, 1] = gx.view(n, 32, C).sum(1).float()
    return g, partial


def _coefs(ws, geom, C, k):
    """k consecutive [C] float vectors after the grid_x * 2 * C partial sums: forward scale, shift; backward k0, k1, k2,
    forward scale, forward shift."""
    off = geom.grid_x * 2 * C
    f = ws.view(torch.float32)
    return [f[off + i * C:off + (i + 1) * C].clone() for i in range(k)]


def _check_z(z, y, res, relu, scale, shift, what):
    """z == bf16([relu](fp32(fp32(fma(y, scale, shift)) [+ residual]))), every rounding from the exact value."""
    M, C = y.shape
    for p0, p1 in _rows(M, C):
        t = _fma32(y[p0:p1], scale, shift)
        if res is not None:
            t = _fma32(t, torch.ones_like(scale), res[p0:p1])
        if relu:
            t = t.clamp_min(0)
        _same(z[p0:p1], t.to(torch.bfloat16), None, what)


# ---------------------------------------------------------------- BatchNorm forward -----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", BN_CASES, ids=[c.id for c in BN_CASES])
def test_bn_forward_exact(dev, case):
    """Training-mode BatchNorm forward from external statistics rows (tp_bn_forward_ext: k_bn_fold_ext or a direct
    fold, k_bn_finalize_stats, k_bn_apply) or from its own two-pass statistics (tp_bn_forward: k_bn_stats), then one
    eval-mode call (k_bn_eval_coeffs, k_bn_apply) with the updated running statistics.

    - external rows: save_mean == float32(s1 / M) bit for bit (s1 the exact sum); save_invstd within 4 fp32 ulp of
      1 / sqrt(var + eps) from the exact sums (rsqrtf is specified to 2 ulp);
    - two-pass (shifted sums, divisions by M in fp32): |mean error| <= 2^-23 (|mean| + 2 |s1' / M|), invstd within
      (2 kappa + 4) 2^-23 relative, kappa = E[(y - shift)^2] / var (the cancellation of the shifted variance);
    - running_mean / running_var (unbiased, torch's momentum rule) within 2 fp32 ulp of float64 evaluated from the
      kernel's mean and the variance (the two-pass bar adds the variance error), num_batches_tracked + 1;
    - scale == fp32(w * invstd), shift == fp32(b - mean * scale) from save_mean / save_invstd, and z bit for bit."""
    from turboprune_b200 import _cabi
    bn_forward_check(dev, case, _geom_checked(_cabi.load(), case))


def bn_forward_check(dev, case, geom):
    """The checks of test_bn_forward_exact for one BnCase whose bn_geom plan ``geom`` the caller has asserted."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    M, C = case.M, case.C
    g = torch.Generator(device=dev).manual_seed(M + C)
    y, _ = _bn_y(g, M, C, dev)
    res = _ints(g, (M, C), -8, 8, dev) if case.res else None
    s1 = torch.zeros(C, dtype=torch.float64, device=dev)
    s2 = torch.zeros_like(s1)
    for p0, p1 in _rows(M, C):
        yy = y[p0:p1].double()
        s1 += yy.sum(0)
        s2 += (yy * yy).sum(0)
    _bounded(s2, 1.0, "sum y^2")                         # also bounds sum |y| and every fp32 partial sum of the folds
    ext = None if case.two_pass else _ext_rows(y, geom.ext_rows)
    w = torch.rand(C, generator=g, device=dev) * 1.5 + 0.5
    b = torch.rand(C, generator=g, device=dev) * 2 - 1
    rm0 = torch.randn(C, generator=g, device=dev) * 0.1
    rv0 = torch.rand(C, generator=g, device=dev) * 1.5 + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.full((1,), 7, dtype=torch.int64, device=dev)
    sm, si = torch.empty(C, device=dev), torch.empty(C, device=dev)
    z = torch.empty_like(y)
    ws = _ws(lib, M, C, dev)
    _bn_forward(lib, dev, y, res, z, case.relu, w, b, rm, rv, nbt, sm, si, ext, ws)
    assert int(nbt) == 8

    # statistics
    mean = s1 / M
    var = (s2 * M - s1 * s1) / (M * M)                 # both products exact in float64 (< 2^53): one rounding
    inv = 1.0 / torch.sqrt(var + float(torch.tensor(EPS)))
    if case.two_pass:
        sh = y[0].double()
        dm = s1 / M - sh
        kappa = (s2 - 2 * sh * s1 + M * sh * sh) / M / var
        assert float(kappa.max()) <= 8, "the shifted sums cancel too much for the stated bar"
        err = (sm.double() - mean).abs() - 2.0 ** -23 * (mean.abs() + 2 * dm.abs())
        assert float(err.max()) <= 0, f"{case.id}: save_mean outside its bar at channel {int(err.argmax())}"
        rel = (si.double() - inv).abs() / inv / ((2 * kappa + 4) * 2.0 ** -23)
        assert float(rel.max()) <= 1, f"{case.id}: save_invstd outside its bar ({float(rel.max()):.2f} of it)"
        var_err = var * (2 * kappa + 2) * 2.0 ** -23
    else:
        _same(sm, mean.float(), None, f"{case.id} save_mean")
        _within_ulps(si, inv, 4, f"{case.id} save_invstd")
        var_err = torch.zeros_like(var)
    m = float(torch.tensor(MOMENTUM))
    unb = var.float().double() * M / (M - 1)
    rm_terms = ((1 - m) * rm0.double(), m * sm.double())
    rv_terms = ((1 - m) * rv0.double(), m * unb)
    for got, (a, c), extra, what in ((rm, rm_terms, 0.0, "running_mean"), (rv, rv_terms, m * var_err * M / (M - 1), "running_var")):
        bar = 2 * _f32_ulp(a.abs() + c.abs()) + extra
        err = (got.double() - (a + c)).abs() / bar
        assert float(err.max()) <= 1, f"{case.id} {what}: {float(err.max()):.2f} of the bar at channel {int(err.argmax())}"

    # the apply kernel's coefficients and z
    scale, shift = _coefs(ws, geom, C, 2)
    _same(scale, (w.double() * si.double()).float(), None, f"{case.id} scale")
    _same(shift, _fma32(-sm, scale, b), None, f"{case.id} shift")
    _check_z(z, y, res, case.relu, scale, shift, f"{case.id} z (training)")

    # eval mode from the running statistics just written
    ws.view(torch.float32).fill_(float("nan"))
    _bn_forward(lib, dev, y, res, z, case.relu, w, b, rm, rv, None, None, None, None, ws, training=False)
    scale, shift = _coefs(ws, geom, C, 2)
    _within_ulps(scale, w.double() / torch.sqrt(rv.double() + float(torch.tensor(EPS))), 4, f"{case.id} eval scale")
    _same(shift, _fma32(-rm, scale, b), None, f"{case.id} eval shift")
    _check_z(z, y, res, case.relu, scale, shift, f"{case.id} z (eval)")


# ---------------------------------------------------------------- BatchNorm backward ----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", BN_CASES, ids=[c.id for c in BN_CASES])
def test_bn_backward_exact(dev, case):
    """tp_bn_backward (k_bn_bwd_reduce, k_bn_finalize_bwd, k_bn_bwd_apply) with dyadic statistics and affine parameters
    (the "ext" rows: tp_bn_backward_ext from the gated gradient g and its exact per-32-pixel partial sums, as the
    consuming conv's dgrad epilogue hands them over):
    means on a 1/4 grid (y == mean ties, xhat == 0 and gates exactly at zero occur), invstd a power of two, so the gate
    fma(y, w * invstd, fma(-mean, w * invstd, b)) > 0 and g * xhat are exact; dz in {-1, 0, 1} at a density that keeps
    S <= 2^22 quanta for sum g and sum g * xhat (asserted).

    - dweight == sum g * xhat and dbias == sum g exactly; dres == dz * gate exactly;
    - k0 == fp32(w * invstd) exactly; k1 and k2 within 4 fp32 ulp of float64 from the exact sums (k2: ulp of
      |k0 mean(g)| + |k1 mean|, its two terms can cancel); the forward scale / shift copies used by the relu = 2 apply
      exactly;
    - dy == bf16(fma(k0, g, fma(k1, y, k2))) from the kernel's coefficients, bit for bit (roundings as in _fma32)."""
    from turboprune_b200 import _cabi
    bn_backward_check(dev, case, _geom_checked(_cabi.load(), case))


def bn_backward_check(dev, case, geom):
    """The checks of test_bn_backward_exact for one BnCase whose bn_geom plan ``geom`` the caller has asserted."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    M, C = case.M, case.C
    relu, want_dres = BWD_MODES[case.bwd]
    g_ = torch.Generator(device=dev).manual_seed(M + C + 1)
    y, ymax = _bn_y(g_, M, C, dev)
    pick = lambda vals: torch.tensor(vals, device=dev)[torch.randint(0, len(vals), (C,), generator=g_, device=dev)]
    w = pick([-1.0, 0.5, 1.0, 1.5, 2.0])
    inv = pick([0.125, 0.25, 0.5])
    b = pick([0.0, 0.0, 0.125, -0.25]) * w * inv         # gate: (y - mean + b / scale) * scale > 0, open and closed in every channel
    mean = torch.randint(-2 * ymax, 2 * ymax + 1, (C,), generator=g_, device=dev).float() / 4
    sc64, sf64 = w.double() * inv.double(), b.double() - mean.double() * w.double() * inv.double()
    xmax = (ymax + ymax / 2) * 0.5                     # largest |xhat|
    dens = min(0.5, 0.8 * EXACT / (M * xmax * 32))
    dz = _sparse_ints(g_, M, C, 1, dens, dev)
    res = _ints(g_, (M, C), -8, 8, dev) if (relu == 1 and case.res) else None
    z = None
    if relu == 1:
        z = torch.empty_like(y)
        for p0, p1 in _rows(M, C):
            t = y[p0:p1].double() * sc64 + sf64
            if res is not None:
                t += res[p0:p1].double()
            z[p0:p1] = t.clamp_min(0).to(torch.bfloat16)
        del res
    dy = torch.empty_like(y)
    dres = torch.empty_like(y) if want_dres else None
    dwt, dbs = torch.empty(C, device=dev), torch.empty(C, device=dev)
    ws = _ws(lib, M, C, dev)
    if case.bwd == "ext":
        g, partial = _gated_partials(dz, y, sc64, sf64, mean, inv, geom.ext_rows)
        with torch.cuda.device(dev):
            rc = lib.tp_bn_backward_ext(_ptr(g), _ptr(y), M, C, _ptr(w), _ptr(b), _ptr(mean), _ptr(inv), _ptr(partial),
                                        partial.shape[0], _ptr(dy), _ptr(dwt), _ptr(dbs), _ptr(ws), ws.numel(), _stream(dev))
        assert rc == 0, f"tp_bn_backward_ext: {rc}"
        del g, partial
    else:
        _bn_backward(lib, dev, dz, z, y, relu, w, b, mean, inv, dy, dres, dwt, dbs, ws)

    k0, k1, k2, fsc, fsf = _coefs(ws, geom, C, 5)
    sums = torch.zeros(4, C, dtype=torch.float64, device=dev)      # sum g, sum g*xhat, sum |g|, sum |g*xhat|
    m64, i64 = mean.double(), inv.double()
    for p0, p1 in _rows(M, C):
        yy, d = y[p0:p1].double(), dz[p0:p1].double()
        if relu == 1:
            gate = z[p0:p1].double() > 0
        elif relu == 2:
            gate = yy * sc64 + sf64 > 0
        else:
            gate = torch.ones_like(d, dtype=torch.bool)
        gg = torch.where(gate, d, 0.0)
        gx = gg * (yy - m64) * i64
        sums += torch.stack([gg.sum(0), gx.sum(0), gg.abs().sum(0), gx.abs().sum(0)])
        if dres is not None:
            _same(dres[p0:p1], gg.to(torch.bfloat16), None, f"{case.id} dres")
        _same(dy[p0:p1], _fma32(k0, gg, _fma32(k1, yy, k2)).to(torch.bfloat16), None, f"{case.id} dy")
    sg, sgx, sga, sgxa = sums
    _bounded(sga, 1.0, "sum g")
    _bounded(sgxa, 2.0 ** -5, "sum g * xhat")          # xhat is a multiple of 1/32
    assert float(sga.min()) > 0, "every channel needs a non-zero gated gradient"
    _same(dbs, sg, sga, f"{case.id} dbias")
    _same(dwt, sgx, sgxa, f"{case.id} dweight")
    _same(k0, sc64, None, f"{case.id} k0")
    _same(fsc, sc64, None, f"{case.id} forward scale copy")
    _same(fsf, _fma32(-mean, k0, b), None, f"{case.id} forward shift copy")
    k1_64 = -sc64 * i64 * (sgx / M)
    _within_ulps(k1, k1_64, 4, f"{case.id} k1")
    a, c = -sc64 * (sg / M), -k1_64 * m64
    _within_ulps(k2, a + c, 4, f"{case.id} k2", scale=a.abs() + c.abs())


# ---------------------------------------------------------------- one gate, four places ------------------------------------
GATE_CASES = [("stem.bn1", 512 * 112 * 112, 64), ("l2.0.bn1", 512 * 56 * 56, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GATE_CASES, ids=[c[0] for c in GATE_CASES])
def test_relu_gate_same_in_forward_and_backward(dev, case):
    """With the statistics the forward actually produced (real-valued y, non-dyadic mean / invstd), the backward with
    the gate read from z (relu = 1) and with the gate recomputed from y (relu = 2) give bit-identical dy, dweight and
    dbias: the forward apply, k_bn_bwd_reduce<2> and k_bn_bwd_apply<2> evaluate the same gate."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    name, M, C = case
    geom = bn_geom(M, C, _sms())
    g = torch.Generator(device=dev).manual_seed(M + 3)
    mu = torch.randn(C, generator=g, device=dev) * 0.5
    sd = torch.rand(C, generator=g, device=dev) * 1.5 + 0.5
    y = torch.empty(M, C, dtype=torch.bfloat16, device=dev)
    for p0, p1 in _rows(M, C):
        y[p0:p1] = (torch.randn(p1 - p0, C, generator=g, device=dev) * sd + mu).to(torch.bfloat16)
    ext = _ext_rows(y, geom.ext_rows)
    w = torch.rand(C, generator=g, device=dev) * 1.5 + 0.5
    b = torch.randn(C, generator=g, device=dev) * 0.5
    sm, si = torch.empty(C, device=dev), torch.empty(C, device=dev)
    z = torch.empty_like(y)
    ws = _ws(lib, M, C, dev)
    _bn_forward(lib, dev, y, None, z, True, w, b, torch.zeros(C, device=dev), torch.ones(C, device=dev), None, sm, si, ext, ws)
    del ext
    closed = _zeros(z) / z.numel()
    assert 0.2 < closed < 0.8, closed
    dz = _sparse_ints(g, M, C, 1, 1.0, dev)
    out = []
    for relu in (1, 2):
        dy = torch.empty_like(y)
        dwt, dbs = torch.empty(C, device=dev), torch.empty(C, device=dev)
        _bn_backward(lib, dev, dz, z if relu == 1 else None, y, relu, w, b, sm, si, dy, None, dwt, dbs, ws)
        out.append((dy, dwt, dbs))
    (dy1, dw1, db1), (dy2, dw2, db2) = out
    if not torch.equal(dy1.view(torch.int16), dy2.view(torch.int16)):
        nbad = sum(int(torch.count_nonzero(dy1[p0:p1].view(torch.int16) != dy2[p0:p1].view(torch.int16))) for p0, p1 in _rows(M, C))
        pytest.fail(f"{name}: dy differs in {nbad} elements between the gate from z and the gate from y")
    assert torch.equal(dw1.view(torch.int32), dw2.view(torch.int32)) and torch.equal(db1.view(torch.int32), db2.view(torch.int32))


@pytest.mark.gpu
def test_bnb_epilogue_gate_same_as_forward(dev):
    """The BatchNorm-backward gate of the dgrad epilogue (ops.conv_dgrad_bnrelu) fed the y, save_mean and save_invstd of a
    real forward (ResNet-50 l1 3x3 64 at batch 256): g == dx * (z > 0) bit for bit, z the forward's output."""
    from turboprune_b200 import ops
    lib = ops._cabi.load()
    n, hw, c, k = 256, 56, 64, 3
    M = n * hw * hw
    geom = bn_geom(M, c, _sms())
    g = torch.Generator(device=dev).manual_seed(256)
    y = (torch.randn(M, c, generator=g, device=dev) * 1.3 + 0.2).to(torch.bfloat16)
    w_bn = torch.rand(c, generator=g, device=dev) * 1.5 + 0.5
    b_bn = torch.randn(c, generator=g, device=dev) * 0.5
    sm, si = torch.empty(c, device=dev), torch.empty(c, device=dev)
    z = torch.empty_like(y)
    ws = _ws(lib, M, c, dev)
    _bn_forward(lib, dev, y, None, z, True, w_bn, b_bn, torch.zeros(c, device=dev), torch.ones(c, device=dev), None, sm, si,
                _ext_rows(y, geom.ext_rows), ws)
    desc = ops.make_desc(n, hw, hw, c, c, k, k, (1, 1), (1, 1))
    wc = (torch.randint(0, 2, (c, c, k, k), generator=g, device=dev) * 2 - 1).float()
    mc = (torch.rand(c, c, k, k, generator=g, device=dev) < 0.5).float()
    _, wd = ops.stage_weights(wc, mc, c, True, c)
    dyc = _ints(g, (n, hw, hw, c), -1, 1, dev)
    out = ops.conv_dgrad_bnrelu(desc, dyc, wd, (y.view(n, hw, hw, c), w_bn, b_bn, sm, si))
    assert out is not None, "the fused path must exist for this shape"
    gated = out[0].view(M, c)
    dx = ops.conv_dgrad(desc, dyc, wd).view(M, c)
    want = torch.where(z > 0, dx, torch.zeros_like(dx))
    _same(gated, want, None, "dgrad epilogue gate against the forward's z")
    assert 0.2 < _zeros(z) / z.numel() < 0.8


# ---------------------------------------------------------------- the table against a real ResNet-50 step -----------------
def _table_keys(c):
    fwd = ("forward", c.M, c.C, c.relu, c.res, not c.two_pass)
    if c.bwd == "ext":
        return {fwd, ("backward_ext", c.M, c.C)}
    relu, dres = BWD_MODES[c.bwd]
    return {fwd, ("backward", c.M, c.C, relu, dres)}


@pytest.mark.gpu
def test_bn_case_table_matches_resnet50_step(dev, monkeypatch):
    """One ResNet-50 forward and backward at batch 2 (224 x 224, bf16 autocast) through fuse_torchvision_blocks, with the
    BatchNorm entry points wrapped: every (entry point, M per image scaled to batch 512, C, ReLU mode, residual) the
    step issues is a row of BN_TABLE, and every row of BN_TABLE is issued."""
    import refshim
    from turboprune_b200 import _cabi
    from turboprune_b200.utils import custom_models as cm
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
    torch.manual_seed(0)
    model = cm.TorchVisionModel(refshim.make_cfg("resnet50", "imagenet")).to(dev).train()
    x = torch.randn(n, 3, 224, 224, device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(x)
    out.float().square().mean().backward()
    torch.cuda.synchronize()
    want = set().union(*(_table_keys(c) for c in BN_TABLE))
    assert seen == want, f"issued but not in the table: {sorted(seen - want)}; in the table but not issued: {sorted(want - seen)}"


# ---------------------------------------------------------------- max-pool ----------------------------------------------------
# (id, n, c, h, w, k, stride, pad)
POOL_CASES = [
    ("stem.3x3s2p1.512x64x112", 512, 64, 112, 112, 3, 2, 1),              # k_maxpool_*_321
    ("vgg.2x2s2.64@32", 512, 64, 32, 32, 2, 2, 0),                         # VGG-16 CIFAR pools: the generic kernels
    ("vgg.2x2s2.128@16", 512, 128, 16, 16, 2, 2, 0),
    ("vgg.2x2s2.256@8", 512, 256, 8, 8, 2, 2, 0),
    ("vgg.2x2s2.512@4", 512, 512, 4, 4, 2, 2, 0),
    ("vgg.2x2s2.512@2", 512, 512, 2, 2, 2, 2, 0),
    ("clip.3x3s1p1", 16, 64, 23, 17, 3, 1, 1),
    ("clip.3x3s2p0", 16, 64, 23, 17, 3, 2, 0),
    ("clip.2x2s1p0", 16, 64, 23, 17, 2, 1, 0),
    ("odd.3x3s2p1", 16, 64, 23, 17, 3, 2, 1),                              # k_maxpool_*_321 with clipped last windows
]


def _pool(lib, dev, x, k, st, pad, dy=None):
    n, h, w, c = x.shape
    p, q = (h + 2 * pad - k) // st + 1, (w + 2 * pad - k) // st + 1
    y = torch.empty(n, p, q, c, dtype=torch.bfloat16, device=dev)
    idx = torch.empty(n, p, q, c, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        assert lib.tp_maxpool_forward(_ptr(x), _ptr(y), _ptr(idx), n, h, w, c, k, st, pad, p, q, _stream(dev)) == 0
        dx = None
        if dy is not None:
            dx = torch.empty_like(x)
            assert lib.tp_maxpool_backward(_ptr(dy), _ptr(idx), _ptr(dx), n, h, w, c, k, st, pad, p, q, _stream(dev)) == 0
    return y, idx, dx


def _flat_index(idx, k, st, pad, w):
    """uint8 window index r * k + s -> torch's flat input index (h0 + r) * W + (w0 + s)."""
    n, p, q, c = idx.shape
    ii = idx.long()
    r, s = ii // k, ii % k
    h0 = (torch.arange(p, device=idx.device) * st - pad).view(1, p, 1, 1)
    w0 = (torch.arange(q, device=idx.device) * st - pad).view(1, 1, q, 1)
    return (h0 + r) * w + (w0 + s)


def _check_pool(y, idx, dx, x, dy, k, st, pad, what):
    n, h, w, c = x.shape
    for sl in _per_batch(n, h * w * c):
        x64 = x[sl].permute(0, 3, 1, 2).double().contiguous()
        yr, ir = F.max_pool2d(x64, k, st, pad, return_indices=True)
        yr, irn = yr.permute(0, 2, 3, 1), ir.permute(0, 2, 3, 1)
        both_nan = torch.isnan(y[sl].double()) & torch.isnan(yr)
        bad = ~both_nan & (y[sl].double() != yr)
        assert not bool(bad.any()), f"{what}: y differs in {int(bad.sum())} elements, first at {bad.nonzero()[0].tolist()}"
        got = _flat_index(idx[sl], k, st, pad, w)
        bad = got != irn
        assert not bool(bad.any()), (f"{what}: arg-max differs in {int(bad.sum())} elements, first at {bad.nonzero()[0].tolist()}: "
                                     f"kernel {int(got[bad][0])}, torch {int(irn[bad][0])}")
        dy64 = dy[sl].permute(0, 3, 1, 2).double().contiguous()
        dxr = torch.ops.aten.max_pool2d_with_indices_backward(dy64, x64, [k, k], [st, st], [pad, pad], [1, 1], False, ir)
        _same(dx[sl], dxr.permute(0, 2, 3, 1).to(torch.bfloat16), None, f"{what}: dx")
        del x64, yr, ir, dy64, dxr


@pytest.mark.gpu
@pytest.mark.parametrize("case", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_maxpool_exact(dev, case):
    """Max-pool forward and backward on post-ReLU-like input (bf16 integers in [-2, 3] clamped at 0: half zeros, so ties
    and all-zero windows are the normal case) against float64 torch: y bit-identical, the saved window index equal to
    torch's arg-max everywhere (first maximum wins, ties included), dx for integer dy in [-4, 4] bit-identical to torch's
    float64 backward rounded to bf16 (sums of at most 9 such values are exact)."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    name, n, c, h, w, k, st, pad = case
    g = torch.Generator(device=dev).manual_seed(n * c + h + k)
    x = _ints(g, (n, h, w, c), -2, 3, dev).clamp_min(0)
    p, q = (h + 2 * pad - k) // st + 1, (w + 2 * pad - k) // st + 1
    dy = _ints(g, (n, p, q, c), -4, 4, dev)
    y, idx, dx = _pool(lib, dev, x, k, st, pad, dy)
    assert int(torch.count_nonzero(y == 0)) > y.numel() // 1000, "all-zero windows must occur"
    _check_pool(y, idx, dx, x, dy, k, st, pad, name)


@pytest.mark.gpu
@pytest.mark.parametrize("geom", [(3, 2, 1), (3, 1, 1), (2, 2, 0)], ids=["3x3s2p1", "3x3s1p1", "2x2s2p0"])
def test_maxpool_nan_and_inf(dev, geom):
    """NaN propagates with torch's index (a later NaN in the window wins, as in ATen's `val > max || isnan(val)`), and a
    window that is all -inf (inside the image, and clipped at the corner) takes its first in-bounds tap."""
    from turboprune_b200 import _cabi
    lib = _cabi.load()
    k, st, pad = geom
    g = torch.Generator(device=dev).manual_seed(k + st)
    n, h, w, c = 2, 11, 11, 16
    x = _ints(g, (n, h, w, c), -2, 3, dev).clamp_min(0)
    x[0, 3, 4, :8] = float("nan")
    x[0, 5, 5] = float("nan")
    x[0, 5, 6] = float("nan")
    x[1, 0, 0, 8:] = float("nan")
    x[1, 4:9, 4:9] = float("-inf")
    x[1, 0:2, 8:11] = float("-inf")
    p, q = (h + 2 * pad - k) // st + 1, (w + 2 * pad - k) // st + 1
    dy = _ints(g, (n, p, q, c), -4, 4, dev)
    y, idx, dx = _pool(lib, dev, x, k, st, pad, dy)
    assert bool(torch.isnan(y.float()).any()) and bool(torch.isneginf(y.float()).any())
    _check_pool(y, idx, dx, x, dy, k, st, pad, f"nan/-inf {geom}")


# ---------------------------------------------------------------- SGD ----------------------------------------------------------
def _resnet50_params():
    import torchvision
    with torch.device("meta"):
        net = torchvision.models.resnet50()
    return [(name, tuple(p.shape)) for name, p in net.named_parameters()]


SGD_VARIANTS = ["eager", "cuda-graph", "misaligned-grad", "late-param"]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", SGD_VARIANTS)
def test_fused_sgd_bit_identical_to_torch(dev, variant):
    """FusedSGD(capturable=True) on ResNet-50's 161 parameters (25.5 M values; lr 0.2, momentum 0.9, weight decay 5e-4,
    the ResNet-50 recipe) against torch.optim.SGD(foreach=True) on the same GPU: weights and momentum buffers
    bit-identical after each of three steps (the first without momentum), with the learning rate changed between steps
    through sync_lr.  The gradients are views into one flat buffer with 16-byte aligned slots, laid out as grad_exchange
    lays them out, so every full 4096-element tile of a weight takes k_sgd's vectorised path.

    - cuda-graph: step 1 eager (uploads the segment table), then one captured step replayed for steps 2 and 3 (the
      cached table, the learning rate read from the device scalar);
    - misaligned-grad: the largest gradient sits 4 bytes off 16-byte alignment, so its full tiles take the scalar path;
    - late-param: the largest parameter gets its first gradient at step 2 (FusedSGD.step's first-step split)."""
    from turboprune_b200.grad_exchange import plan_buckets
    from turboprune_b200.optim import FusedSGD
    named = _resnet50_params()
    assert len(named) == 161 and sum(math.prod(s) for _, s in named) == 25_557_032
    g = torch.Generator(device=dev).manual_seed(50)
    init = []
    for name, shape in named:
        if len(shape) > 1:
            v = torch.randn(shape, generator=g, device=dev) * (2.0 / math.prod(shape[1:])) ** 0.5
        elif name.endswith("weight"):
            v = 1 + 0.1 * torch.randn(shape, generator=g, device=dev)
        else:
            v = 0.1 * torch.randn(shape, generator=g, device=dev)
        init.append(v)
    mine = [torch.nn.Parameter(v.clone()) for v in init]
    ref = [torch.nn.Parameter(v.clone()) for v in init]
    del init
    numels = [p.numel() for p in mine]
    (_, offs, total), = plan_buckets(numels, 1 << 62)
    flat = torch.zeros(total, device=dev)
    views = [flat[o:o + p.numel()].view_as(p) for o, p in zip(offs, mine)]
    big = max(range(len(mine)), key=lambda i: numels[i])
    if variant == "misaligned-grad":
        spare = torch.zeros(numels[big] + 1, device=dev)
        views[big] = spare[1:].view_as(mine[big])
    for i, v in enumerate(views):
        off = v.data_ptr() % 16
        assert off == (4 if variant == "misaligned-grad" and i == big else 0), (named[i][0], off)
    late = big if variant == "late-param" else None
    lrs = (0.2, 0.15, 0.1)
    opt = FusedSGD(mine, lr=lrs[0], momentum=0.9, weight_decay=5e-4, capturable=True)
    ropt = torch.optim.SGD(ref, lr=lrs[0], momentum=0.9, weight_decay=5e-4, foreach=True)
    graph = None
    for step in range(3):
        for i, (p, rp, v, (name, _)) in enumerate(zip(mine, ref, views, named)):
            gv = torch.randn(v.shape, generator=g, device=dev) * (1e-2 if name.endswith("bias") else 3e-3)
            if step == 0 and i == late:
                p.grad = rp.grad = None
                continue
            v.copy_(gv)
            p.grad, rp.grad = v, gv
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
        for i, (p, rp) in enumerate(zip(mine, ref)):
            name = named[i][0]
            pairs = [("weight", p.detach(), rp.detach())]
            b, rb = opt.state[p].get("momentum_buffer"), ropt.state[rp].get("momentum_buffer")
            assert (b is None) == (rb is None) == (step == 0 and i == late), (name, step)
            if b is not None:
                pairs.append(("momentum_buffer", b, rb))
            for what, a, r in pairs:
                bad = a.view(torch.int32) != r.view(torch.int32)
                if bool(bad.any()):
                    j = int(bad.flatten().nonzero()[0])
                    pytest.fail(f"{variant}, step {step + 1}, {name} {what}: {int(bad.sum())} of {a.numel()} elements differ from "
                                f"torch.optim.SGD, first at {j}: fused {float(a.flatten()[j])!r}, torch {float(r.flatten()[j])!r}")
