"""torch.autograd.Function wrappers: one node per hot-path block, forward and backward both made of
libsmaat_b200.so kernels (functional.py).  They make the drop-in modules differentiable so the
reference's training loops (`loss.backward()` in train_SmaAtUNet.py:55, Lightning's automatic
optimisation over UNetBase.training_step, regression_lightning.py:67-77) run unchanged.
"""
from __future__ import annotations

import torch

from . import functional as Fn
from . import ops


def _check_saved(ctx, what):
    """The block Functions keep their activations in a plain dict (a dozen tensors plus scalars) that is released by the
    first backward -- the same contract as torch's saved tensors, with torch's wording for the error."""
    if ctx.saved is None:
        raise RuntimeError(f"Trying to backward through the graph a second time ({what} block of smaat_unet_b200): the saved "
                           "activations were freed by the first backward; retain_graph=True is not supported by these blocks.")


class DoubleConvDSFn(torch.autograd.Function):
    """(DS conv => BN => ReLU) * 2 over the virtual concat [x, x1]."""

    @staticmethod
    def params(mod):
        ds0, bn0, ds1, bn1 = mod.double_conv[0], mod.double_conv[1], mod.double_conv[3], mod.double_conv[4]
        out = []
        for ds, bn in ((ds0, bn0), (ds1, bn1)):
            for p in (ds.depthwise.weight, ds.depthwise.bias, ds.pointwise.weight, ds.pointwise.bias, bn.weight, bn.bias):
                if p is None:
                    raise NotImplementedError("DoubleConvDS without conv bias / BN affine parameters is not supported in the autograd path")
                out.append(p)
        return out

    @staticmethod
    def run(mod, x, x1=None):
        return DoubleConvDSFn.apply(mod, x, x1, *DoubleConvDSFn.params(mod))

    @staticmethod
    def forward(ctx, mod, x, x1, *params):
        x = ops._dense(x, "x")
        x1 = ops._dense(x1, "x1") if x1 is not None else None
        out, saved = Fn.double_conv_fwd(mod, x, x1)
        ctx.mod, ctx.saved = mod, saved
        return out

    @staticmethod
    def backward(ctx, g):
        need = ctx.needs_input_grad
        _check_saved(ctx, "DoubleConvDS")
        dx, dx1, pg = Fn.double_conv_bwd(ctx.mod, ctx.saved, g, need_x=need[1], need_x1=need[2])
        ctx.saved = None
        # gradients that went straight into a session's flat bucket (functional.set_grad_sinks) bypass AccumulateGrad
        pg = [pgi if (need[3 + i] and not Fn.is_sunk(prm)) else None for i, (pgi, prm) in enumerate(zip(pg, DoubleConvDSFn.params(ctx.mod)))]
        return (None, dx if need[1] else None, dx1 if need[2] else None, *pg)


class DoubleConvFn(torch.autograd.Function):
    """(Conv2d 3x3 => BN => ReLU) * 2 over the virtual concat [x, x1] (unet_parts.py:8-25)."""

    @staticmethod
    def params(mod):
        c0, bn0, c1, bn1 = mod.double_conv[0], mod.double_conv[1], mod.double_conv[3], mod.double_conv[4]
        out = []
        for p in (c0.weight, c0.bias, bn0.weight, bn0.bias, c1.weight, c1.bias, bn1.weight, bn1.bias):
            if p is None:
                raise NotImplementedError("DoubleConv without conv bias / BN affine parameters is not supported in the autograd path")
            out.append(p)
        return out

    @staticmethod
    def run(mod, x, x1=None):
        return DoubleConvFn.apply(mod, x, x1, *DoubleConvFn.params(mod))

    @staticmethod
    def forward(ctx, mod, x, x1, *params):
        x = ops._dense(x, "x")
        x1 = ops._dense(x1, "x1") if x1 is not None else None
        out, saved = Fn.dense_double_conv_fwd(mod, x, x1)
        ctx.mod, ctx.saved = mod, saved
        return out

    @staticmethod
    def backward(ctx, g):
        need = ctx.needs_input_grad
        _check_saved(ctx, "DoubleConv")
        dx, dx1, pg = Fn.dense_double_conv_bwd(ctx.mod, ctx.saved, g, need_x=need[1], need_x1=need[2])
        ctx.saved = None
        pg = [pgi if (need[3 + i] and not Fn.is_sunk(prm)) else None for i, (pgi, prm) in enumerate(zip(pg, DoubleConvFn.params(ctx.mod)))]
        return (None, dx if need[1] else None, dx1 if need[2] else None, *pg)


class DSConvFn(torch.autograd.Function):
    """A standalone DepthwiseSeparableConv (layers.py:47-50): depthwise then pointwise, both biases, no BN/activation."""

    @staticmethod
    def run(mod, x):
        for p in (mod.depthwise.bias, mod.pointwise.bias):
            if p is None:
                raise NotImplementedError("DepthwiseSeparableConv without conv biases is not supported in the autograd path")
        return DSConvFn.apply(mod, x, mod.depthwise.weight, mod.depthwise.bias, mod.pointwise.weight, mod.pointwise.bias)

    @staticmethod
    def forward(ctx, mod, x, *params):
        x = ops._dense(x, "x")
        d, z = Fn.ds_conv_fwd(mod, x)              # unfused: the depthwise result is needed by the weight gradient
        ctx.mod = mod
        ctx.save_for_backward(x, d)
        return z

    @staticmethod
    def backward(ctx, g):
        x, d = ctx.saved_tensors
        mod, need = ctx.mod, ctx.needs_input_grad
        g = ops._dense(g, "grad_output")
        zeros = lambda p: torch.zeros(p.shape, device=p.device, dtype=torch.float32)
        dWd, dbd, dWp, dbp = zeros(mod.depthwise.weight), zeros(mod.depthwise.bias), zeros(mod.pointwise.weight), zeros(mod.pointwise.bias)
        dd = Fn.pw_bwd(g, d, mod.pointwise.weight, dWp, dbp)
        dx, _ = Fn.dw_bwd(dd, mod.depthwise.weight, x, None, None, None, mod.kernels_per_layer, dWd, dbd, need_input=need[1])
        grads = [dWd, dbd, dWp, dbp]
        return (None, dx if need[1] else None, *[gi if need[2 + i] else None for i, gi in enumerate(grads)])


class CBAMFn(torch.autograd.Function):
    @staticmethod
    def params(mod):
        ca, sp = mod.channel_att, mod.spatial_att
        return [ca.MLP[1].weight, ca.MLP[1].bias, ca.MLP[3].weight, ca.MLP[3].bias, sp.conv.weight, sp.bn.weight, sp.bn.bias]

    @staticmethod
    def run(mod, x):
        return CBAMFn.apply(mod, x, *CBAMFn.params(mod))

    @staticmethod
    def forward(ctx, mod, x, *params):
        out, saved = Fn.cbam_fwd(mod, ops._dense(x, "x"))
        ctx.mod, ctx.saved = mod, saved
        return out

    @staticmethod
    def backward(ctx, g):
        _check_saved(ctx, "CBAM")
        dx, pg = Fn.cbam_bwd(ctx.mod, ctx.saved, g)
        ctx.saved = None
        need = ctx.needs_input_grad
        prms = CBAMFn.params(ctx.mod)
        return (None, dx if need[1] else None, *[p if (need[2 + i] and not Fn.is_sunk(prms[i])) else None for i, p in enumerate(pg)])


class MaxPool2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = ops._dense(x, "x")
        ctx.save_for_backward(x)
        return ops.maxpool2(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return Fn.maxpool2_bwd(x, g)


class Upsample2xPadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, Ho, Wo):
        ctx.in_shape = tuple(x.shape)
        return ops.upsample2x_pad(x, Ho, Wo)

    @staticmethod
    def backward(ctx, g):
        return Fn.upsample2x_pad_bwd(g, ctx.in_shape), None, None


class ConvT2x2PadFn(torch.autograd.Function):
    """nn.ConvTranspose2d(Cin, Cout, 2, stride=2) + F.pad to (Ho, Wo) (parts_ds.py:72-73, 76-81): one pointwise GEMM to the
    4 Cout packed taps + a pixel shuffle; backward = the gather transpose + the pointwise backward + the weight un-pack."""

    @staticmethod
    def forward(ctx, x, weight, bias, Ho, Wo, wp, w_split):
        x = ops._dense(x, "x")
        Cout = weight.shape[1]
        t = ops.pw1x1(x, wp, None, None, False, w_split=w_split)
        ctx.save_for_backward(x, weight, wp, *([bias] if bias is not None else []))
        ctx.has_bias, ctx.out_hw = bias is not None, (Ho, Wo)
        return ops.pixel_shuffle2_pad(t, bias.detach() if bias is not None else None, Cout, Ho, Wo)

    @staticmethod
    def backward(ctx, g):
        from . import _lib
        x, weight, wp = ctx.saved_tensors[:3]
        bias = ctx.saved_tensors[3] if ctx.has_bias else None
        B, Cin, H, W = x.shape
        Cout = weight.shape[1]
        Ho, Wo = ctx.out_hw
        lib = _lib.load()
        g, gbs = ops._nchw_bstride(g, "grad_output")
        dt = torch.empty((B, 4 * Cout, H, W), device=x.device, dtype=torch.float32)
        ops._call("smaat_pixel_shuffle2_pad_bwd", 8 * dt.numel(), 0, lib.smaat_pixel_shuffle2_pad_bwd, ops._ptr(g), gbs, ops._ptr(dt), B, Cout, H, W, Ho,
                  Wo, ops._stream())
        dwp = torch.zeros_like(wp)
        dbp = torch.zeros(4 * Cout, device=x.device, dtype=torch.float32)
        dx = Fn.pw_bwd(dt, x, wp, dwp, dbp, need_input=ctx.needs_input_grad[0])
        dW = Fn._zeros_like_param(weight)
        db = Fn._zeros_like_param(bias) if bias is not None else None
        ops._call("smaat_convt2x2_unpack_wgrad", 8 * dwp.numel(), 0, lib.smaat_convt2x2_unpack_wgrad, ops._ptr(dwp), ops._ptr(dbp), ops._ptr(dW), ops._ptr(db),
                  Cin, Cout, ops._stream())
        return (dx, None if Fn.is_sunk(weight) else dW, (db if (bias is not None and not Fn.is_sunk(bias)) else None), None, None, None, None)


class OutConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        x = ops._dense(x, "x")
        ctx.save_for_backward(x, weight, *([bias] if bias is not None else []))
        ctx.has_bias = bias is not None
        return ops.outconv(x, weight.detach(), bias.detach() if bias is not None else None)

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors[:2]
        bias = ctx.saved_tensors[2] if ctx.has_bias else None
        dx, dW, db = Fn.outconv_bwd(x, weight, g, need_x=ctx.needs_input_grad[0], bias=bias)
        return dx, (None if Fn.is_sunk(weight) else dW), (db if (ctx.has_bias and not Fn.is_sunk(bias)) else None)
