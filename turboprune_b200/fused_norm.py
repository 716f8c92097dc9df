"""Fused BatchNorm (+ residual) (+ ReLU) for the NHWC bf16 activation path (SURVEY.md §8(f) row 1).

``BatchNorm2dB200`` is a drop-in ``nn.BatchNorm2d`` subclass (same parameters / buffers / state-dict
keys); ``fuse_torchvision_blocks`` rebinds the ``forward`` of torchvision's ResNet blocks and VGG
``features`` so that ``bn -> relu`` and ``bn -> (+identity) -> relu`` run as ONE apply kernel (and one
backward pair) instead of separate ATen batch_norm / relu / add kernels.  The module graph the reference
builds (utils/custom_models.py:184) and its state dict are unchanged.
"""
import types
from ctypes import c_void_p

import torch
import torch.nn as nn

from . import _cabi, ops
from .utils.mask_layers import grad_slots


def _ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else None


# Partial sums offered by a dgrad that already did a BatchNorm's backward reduction (ops.conv_dgrad_bnrelu): keyed by the
# storage pointer of the gated gradient, validated by the token of the BatchNorm forward call they belong to.
_PARTIALS = {}


def offer_partials(g, partial, token):
    # g is kept alive (its address cannot be recycled) and its version counter remembered: when the BatchNorm output has a
    # second consumer, autograd may ACCUMULATE the other gradient in place into g — same address, different content
    _PARTIALS[g.data_ptr()] = (partial, token, g, g._version)


def drop_partials():
    _PARTIALS.clear()


def fused_enabled():
    """The fused NHWC kernels are bf16-only: inside ``ops.compute_precision(torch.float32)`` the modules of this file run
    the reference's own ATen ops (BatchNorm, ReLU, the residual add, max-pool) on the fp32 channels_last activations."""
    return ops.current_precision() != torch.float32


class _BNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, nbt, momentum, eps, training, relu, grad_slots=None, ext_stats=None,
                saved=None):
        if ops.current_precision() == torch.float32:
            raise RuntimeError("fused BatchNorm is bf16-only: at float32 BatchNorm2dB200 runs ATen's batch_norm")
        lib = _cabi.load()
        ctx.set_materialize_grads(False)
        ctx.grad_slots = grad_slots
        ctx.token = saved[3] if saved is not None else None
        n, c, h, w = x.shape
        xn = saved[0] if saved is not None else ops.to_nhwc_bf16(x, c)
        rn = ops.to_nhwc_bf16(residual, c) if residual is not None else None
        m = n * h * w
        dev = x.device
        z = ops.empty_cl(n, c, h, w, dev)
        save_mean = (saved[1] if saved is not None else torch.empty(c, dtype=torch.float32, device=dev)) if training else None
        save_invstd = (saved[2] if saved is not None else torch.empty(c, dtype=torch.float32, device=dev)) if training else None
        wsb = ops._workspace(lib.tp_bn_workspace_bytes(m, c), dev, "bn")
        with torch.cuda.device(dev):
            use_ext = ext_stats is not None and training
            rc = lib.tp_bn_forward_ext(_ptr(xn), _ptr(rn), _ptr(z), m, c, _ptr(weight), _ptr(bias), _ptr(running_mean),
                                       _ptr(running_var), _ptr(nbt), float(momentum), float(eps), int(training), int(relu),
                                       _ptr(save_mean), _ptr(save_invstd), _ptr(ext_stats) if use_ext else None,
                                       ext_stats.shape[0] if use_ext else 0, _ptr(wsb), wsb.numel(), _cabi.stream_ptr(dev))
        _cabi.check(rc, "tp_bn_forward")
        ops._count(3 if training else 2)
        if training:
            # ReLU gate: recomputed from y in the backward unless a residual was added (then z itself is needed)
            ctx.relu = 0 if not relu else (1 if residual is not None else 2)
            ctx.save_for_backward(xn, z.permute(0, 2, 3, 1) if ctx.relu == 1 else None, weight, bias, save_mean, save_invstd)
            ctx.has_res = residual is not None
            ctx.res_dtype = residual.dtype if residual is not None else None
            ctx.x_dtype = x.dtype
        return z

    @staticmethod
    def backward(ctx, dz):
        lib = _cabi.load()
        xn, z, weight, bias, save_mean, save_invstd = ctx.saved_tensors
        n, h, w, c = xn.shape
        m = n * h * w
        dev = xn.device
        dzn = ops.to_nhwc_bf16(dz, c)
        dy = torch.empty_like(xn)
        dres = torch.empty_like(xn) if ctx.has_res else None
        ws_, bs_ = ctx.grad_slots if ctx.grad_slots is not None else (None, None)
        direct = ws_ is not None and bs_ is not None
        dweight = ws_ if direct else torch.empty(c, dtype=torch.float32, device=dev)
        dbias = bs_ if direct else torch.empty(c, dtype=torch.float32, device=dev)
        wsb = ops._workspace(lib.tp_bn_workspace_bytes(m, c), dev, "bn")
        hint = _PARTIALS.pop(dzn.data_ptr(), None) if _PARTIALS else None
        if hint is not None and (hint[1] is not ctx.token or hint[2]._version != hint[3] or ctx.relu != 2 or ctx.has_res):
            hint = None          # not ours, or summed with another consumer's gradient in place: treat it as the raw dz (always right:
                                 # gating an already gated gradient changes nothing)
        with torch.cuda.device(dev):
            if hint is not None:
                # the dgrad that produced dz already gated it and summed it: fold, coefficients, apply
                rc = lib.tp_bn_backward_ext(_ptr(dzn), _ptr(xn), m, c, _ptr(weight), _ptr(bias), _ptr(save_mean), _ptr(save_invstd),
                                            _ptr(hint[0]), hint[0].shape[0], _ptr(dy), _ptr(dweight), _ptr(dbias), _ptr(wsb),
                                            wsb.numel(), _cabi.stream_ptr(dev))
            else:
                rc = lib.tp_bn_backward(_ptr(dzn), _ptr(z), _ptr(xn), m, c, _ptr(weight), _ptr(bias), _ptr(save_mean), _ptr(save_invstd),
                                        int(ctx.relu), _ptr(dy), _ptr(dres), _ptr(dweight), _ptr(dbias), _ptr(wsb), wsb.numel(),
                                        _cabi.stream_ptr(dev))
        _cabi.check(rc, "tp_bn_backward")
        ops._count(3)
        gx = dy.permute(0, 3, 1, 2)
        if gx.dtype != ctx.x_dtype:
            gx = gx.to(ctx.x_dtype)
        gr = dres.permute(0, 3, 1, 2) if dres is not None else None
        if gr is not None and gr.dtype != ctx.res_dtype:
            gr = gr.to(ctx.res_dtype)
        if direct:
            dweight = dbias = None
            ops.grad_ready(ws_, bs_)
        return gx, gr, dweight, dbias, None, None, None, None, None, None, None, None, None, None


class BatchNorm2dB200(nn.BatchNorm2d):
    """nn.BatchNorm2d whose CUDA path is the fused sm_90a kernel; ``forward(x, residual=None, relu=False)``."""

    def forward(self, x, residual=None, relu=False, ext_stats=None):
        """``ext_stats``: batch statistics of ``x`` already computed by the producing convolution's epilogue."""
        training = self.training or not self.track_running_stats
        # eval-mode BN inside an autograd graph is not on the hot path: leave it to torch
        # momentum=None means a cumulative moving average in torch (factor 1/num_batches_tracked): not on the hot path
        if (not x.is_cuda or not fused_enabled() or x.shape[1] % 8 != 0 or (not training and torch.is_grad_enabled() and x.requires_grad)
                or (self.momentum is None and training and self.track_running_stats)):
            y = super().forward(x)
            if residual is not None:
                y = y + residual
            return torch.relu(y) if relu else y
        momentum = 0.0 if self.momentum is None else self.momentum
        slots = grad_slots(self.weight, self.bias)
        saved = None
        if training and relu and residual is None and ops.BN_BWD_FUSION and torch.is_grad_enabled():
            # BatchNorm+ReLU whose output feeds a masked convolution: that convolution's dgrad can do this layer's backward
            # reduction in its epilogue — it needs y, the batch statistics and the affine parameters
            c = x.shape[1]
            with torch.no_grad():
                xn = ops.to_nhwc_bf16(x.detach(), c)
            saved = (xn, torch.empty(c, dtype=torch.float32, device=x.device),
                     torch.empty(c, dtype=torch.float32, device=x.device), object())
        z = _BNFn.apply(x, residual, self.weight, self.bias, self.running_mean, self.running_var,
                        self.num_batches_tracked if (training and self.track_running_stats) else None,
                        momentum, self.eps, training, relu, slots, ext_stats, saved)
        if saved is not None:
            z._tp_bn_src = (saved[0], self.weight, self.bias, saved[1], saved[2], saved[3])
        return z


class _MaxPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad):
        lib = _cabi.load()
        n, c, h, w = x.shape
        xn = ops.to_nhwc_bf16(x, c)
        p = (h + 2 * pad - k) // stride + 1
        q = (w + 2 * pad - k) // stride + 1
        y = ops.empty_cl(n, c, p, q, x.device)
        idx = torch.empty(n, p, q, c, dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            rc = lib.tp_maxpool_forward(_ptr(xn), _ptr(y), _ptr(idx), n, h, w, c, k, stride, pad, p, q, _cabi.stream_ptr(x.device))
        _cabi.check(rc, "tp_maxpool_forward")
        ops._count()
        ctx.save_for_backward(idx)
        ctx.geom = (n, h, w, c, k, stride, pad, p, q)
        ctx.x_dtype = x.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _cabi.load()
        (idx,) = ctx.saved_tensors
        n, h, w, c, k, stride, pad, p, q = ctx.geom
        dyn = ops.to_nhwc_bf16(dy, c)
        dx = torch.empty(n, h, w, c, dtype=torch.bfloat16, device=dy.device)
        with torch.cuda.device(dy.device):
            rc = lib.tp_maxpool_backward(_ptr(dyn), _ptr(idx), _ptr(dx), n, h, w, c, k, stride, pad, p, q, _cabi.stream_ptr(dy.device))
        _cabi.check(rc, "tp_maxpool_backward")
        ops._count()
        gx = dx.permute(0, 3, 1, 2)
        return (gx if gx.dtype == ctx.x_dtype else gx.to(ctx.x_dtype)), None, None, None


class MaxPool2dB200(nn.MaxPool2d):
    """nn.MaxPool2d whose CUDA/NHWC path is the sm_90a kernel pair (square window, no dilation / ceil_mode)."""

    def forward(self, x):
        k, s, p = self.kernel_size, self.stride, self.padding
        simple = all(isinstance(v, int) for v in (k, s, p)) and self.dilation == 1 and not self.ceil_mode and not self.return_indices
        if not (simple and x.is_cuda and fused_enabled() and x.dim() == 4 and x.shape[1] % 8 == 0 and k * k <= 255):
            return super().forward(x)
        return _MaxPoolFn.apply(x, k, s, p)


# ---- fused forwards for the torchvision graphs the reference instantiates ------------------------------
def _stats_ok(conv, bn, x):
    """conv -> bn can hand the batch statistics over through the conv epilogue (training-mode fused BN on CUDA)."""
    from .utils.mask_layers import ConvMask
    return (isinstance(conv, ConvMask) and isinstance(bn, BatchNorm2dB200) and x.is_cuda and fused_enabled() and conv.out_channels % 8 == 0
            and (bn.training or not bn.track_running_stats) and not isinstance(conv.padding, str))


def _conv_bn(conv, bn, x, residual=None, relu=False, skip=False):
    """bn(conv(x)) [+ residual] [relu] with the statistics taken from the conv epilogue when possible.
    ``skip=True`` also returns the aliased input whose gradient lands in conv's dgrad epilogue."""
    fuse = _stats_ok(conv, bn, x)
    xs = x
    if skip:
        from .utils.mask_layers import ConvMask
        skip = isinstance(conv, ConvMask) and x.requires_grad and x.shape[1] % 64 == 0 and fused_enabled()
    if fuse:
        outs = conv(x, want_skip=skip, want_stats=True)
        y, stats = outs[0], outs[-1]
        if skip:
            xs = outs[1]
        z = bn(y, residual=residual, relu=relu, ext_stats=stats)
    else:
        if skip:
            y, xs = conv(x, want_skip=True)
        else:
            y = conv(x)
        z = bn(y, residual=residual, relu=relu)
    return z, xs


def _downsample(ds, identity):
    if isinstance(ds, nn.Sequential) and len(ds) == 2:
        return _conv_bn(ds[0], ds[1], identity)[0]
    return ds(identity)


def _basic_block_forward(self, x):
    out, identity = _conv_bn(self.conv1, self.bn1, x, relu=True, skip=True)
    if self.downsample is not None:
        identity = _downsample(self.downsample, identity)
    return _conv_bn(self.conv2, self.bn2, out, residual=identity, relu=True)[0]


def _bottleneck_forward(self, x):
    out, identity = _conv_bn(self.conv1, self.bn1, x, relu=True, skip=True)
    out = _conv_bn(self.conv2, self.bn2, out, relu=True)[0]
    if self.downsample is not None:
        identity = _downsample(self.downsample, identity)
    return _conv_bn(self.conv3, self.bn3, out, residual=identity, relu=True)[0]


def _resnet_forward_impl(self, x):
    x = _conv_bn(self.conv1, self.bn1, x, relu=True)[0]
    x = self.maxpool(x)
    x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
    x = torch.flatten(self.avgpool(x), 1)
    return self.fc(x)


class _FusedSeq(nn.Sequential):
    """nn.Sequential that runs `BatchNorm2dB200 -> ReLU` pairs as one fused call (VGG-BN features)."""

    def forward(self, x):
        mods = list(self)
        i = 0
        while i < len(mods):
            m = mods[i]
            if i + 1 < len(mods) and _stats_ok(m, mods[i + 1], x):          # conv -> BN [-> ReLU]
                relu = i + 2 < len(mods) and isinstance(mods[i + 2], nn.ReLU)
                x = _conv_bn(m, mods[i + 1], x, relu=relu)[0]; i += 3 if relu else 2
            elif isinstance(m, BatchNorm2dB200) and i + 1 < len(mods) and isinstance(mods[i + 1], nn.ReLU):
                x = m(x, relu=True); i += 2
            else:
                x = m(x); i += 1
        return x


def convert_batchnorm(module: nn.Module):
    """Replace every nn.BatchNorm2d by BatchNorm2dB200 (same init: ones / zeros, no RNG consumed)."""
    for name, child in module.named_children():
        if type(child) is nn.BatchNorm2d:
            new = BatchNorm2dB200(child.num_features, eps=child.eps, momentum=child.momentum, affine=child.affine,
                                  track_running_stats=child.track_running_stats)
            new.load_state_dict(child.state_dict())
            new.train(child.training)
            setattr(module, name, new)
        elif type(child) is nn.MaxPool2d:
            setattr(module, name, MaxPool2dB200(child.kernel_size, child.stride, child.padding, child.dilation,
                                                child.return_indices, child.ceil_mode))
        else:
            convert_batchnorm(child)
    return module


def fuse_torchvision_blocks(net: nn.Module):
    from torchvision.models.resnet import BasicBlock, Bottleneck, ResNet
    from torchvision.models.vgg import VGG
    convert_batchnorm(net)
    for m in net.modules():
        if type(m) is BasicBlock:
            m.forward = types.MethodType(_basic_block_forward, m)
        elif type(m) is Bottleneck:
            m.forward = types.MethodType(_bottleneck_forward, m)
    if isinstance(net, ResNet) and isinstance(net.bn1, BatchNorm2dB200):
        net._forward_impl = types.MethodType(_resnet_forward_impl, net)
    if isinstance(net, VGG) and type(net.features) is nn.Sequential:
        net.features.__class__ = _FusedSeq
    return net
