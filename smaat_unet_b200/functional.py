"""Block-level forward (train / eval-with-grad) and backward passes built from the C-ABI kernels.

These are the bodies of the ``torch.autograd.Function``s in ``autograd.py``; ``modules.py`` routes
here whenever batch statistics or gradients are needed (inference without grad keeps the fused,
BN-folded fast path).  Every function only enqueues kernels from libsmaat_b200.so -- there is no
PyTorch arithmetic fallback; torch supplies memory, streams and the autograd tape.

Reference semantics restated (file:line under /root/reference):
  DoubleConvDS  models/unet_parts_depthwise_separable.py:17-36   CBAM  models/layers.py:90-141
  DoubleConv    models/unet_parts.py:15-22
  BatchNorm2d train mode: batch mean / biased variance normalise, running stats get the unbiased
  variance with momentum 0.1 (SURVEY 8a row a4).
"""
from __future__ import annotations

import torch

from . import ops


def _p(t):
    return None if t is None else t.detach()


_RECOMPUTE_DW = False


def set_recompute_depthwise(flag: bool) -> bool:
    """Trade ~7 % step time for ~45 % less saved-activation memory in the training path: the depthwise
    results (k x the input channels, the largest tensors the DoubleConvDS backward keeps) are dropped after
    the forward and recomputed by the same kernel call right before the pointwise weight-gradient GEMM
    needs them (bit-identical: same kernel, same inputs).  Returns the previous setting."""
    global _RECOMPUTE_DW
    old, _RECOMPUTE_DW = _RECOMPUTE_DW, bool(flag)
    return old


def get_recompute_depthwise() -> bool:
    return _RECOMPUTE_DW


def bn_scale_shift(bn, stats, count):
    """(scale, shift, mean, invstd) that realise ``bn`` on the tensor whose fp64 statistics are ``stats``.
    Train mode: batch statistics (and running-stat update); eval mode: running statistics."""
    use_batch = bn.training or not bn.track_running_stats or bn.running_mean is None
    if use_batch:
        return ops.bn_finalize(stats, count, bn, save=True)
    dev = bn.running_mean.device
    scale, shift = ops.bn_fold(_p(bn.weight), _p(bn.bias), bn.running_mean, bn.running_var, None, bn.eps)
    ones = torch.ones(bn.num_features, device=dev)
    invstd, _ = ops.bn_fold(ones, torch.zeros_like(ones), bn.running_mean, bn.running_var, None, bn.eps)
    return scale, shift, bn.running_mean, invstd


def ds_conv_fwd(ds, x, x1=None, in_scale=None, in_shift=None, stats=None):
    """DepthwiseSeparableConv (layers.py:47-50), unfused so that the depthwise result is available to the
    backward pass: returns (d, z) with z = pointwise(d) + bias (pre-BatchNorm)."""
    ds._check()
    d = ops.dw3x3(x, _p(ds.depthwise.weight), _p(ds.depthwise.bias), ds.kernels_per_layer, x1=x1, in_scale=in_scale, in_shift=in_shift)
    mode = ops.get_pointwise_mode()
    z = ops.pw1x1(d, _p(ds.pointwise.weight), None, _p(ds.pointwise.bias), False, mode=mode, w_split=ds.pw_operands(), stats=stats)
    return d, z


def double_conv_fwd(mod, x, x1=None):
    """DoubleConvDS forward with explicit BatchNorm (batch statistics in train mode).  Returns (out, saved)."""
    ds0, bn0, ds1, bn1 = mod.double_conv[0], mod.double_conv[1], mod.double_conv[3], mod.double_conv[4]
    B, _, H, W = x.shape
    n = B * H * W
    S0 = ops.new_stats(bn0.num_features, x.device)
    S1 = ops.new_stats(bn1.num_features, x.device)
    d0, z0 = ds_conv_fwd(ds0, x, x1=x1, stats=S0)
    sc0, sh0, m0, i0 = bn_scale_shift(bn0, S0, n)
    d1, z1 = ds_conv_fwd(ds1, z0, in_scale=sc0, in_shift=sh0, stats=S1)   # BN+ReLU of z0 applied on load
    if _RECOMPUTE_DW:
        # [Running the fused depthwise->pointwise kernel here instead (nothing to keep, so nothing to write) was tried: with the
        # extra BN+ReLU materialisation it needs it measured 41.4 ms per step against 39.2 ms for this plain drop-and-recompute.]
        d0 = d1 = None
    sc1, sh1, m1, i1 = bn_scale_shift(bn1, S1, n)
    out = ops.affine_act(z1, sc1, sh1, "relu")
    saved = dict(x=x, x1=x1, d0=d0, z0=z0, sc0=sc0, sh0=sh0, m0=m0, i0=i0, d1=d1, z1=z1, sc1=sc1, sh1=sh1, m1=m1, i1=i1, n=n)
    return out, saved


def dense_double_conv_fwd(mod, x, x1=None):
    """DoubleConv forward (unet_parts.py:15-22) over [x, x1] with explicit BatchNorm (batch statistics in train mode).
    The second conv's input relu(BN0(z0)) is materialised (affine_act): its weight gradient needs it.  Returns (out, saved)."""
    bn0, bn1 = mod.double_conv[1], mod.double_conv[4]
    B, _, H, W = x.shape
    n = B * H * W
    S0 = ops.new_stats(bn0.num_features, x.device)
    S1 = ops.new_stats(bn1.num_features, x.device)
    z0 = mod.conv(0, x, x1, shift=_p(mod.double_conv[0].bias), stats=S0)
    sc0, sh0, m0, i0 = bn_scale_shift(bn0, S0, n)
    a0 = ops.affine_act(z0, sc0, sh0, "relu")
    z1 = mod.conv(3, a0, shift=_p(mod.double_conv[3].bias), stats=S1)
    sc1, sh1, m1, i1 = bn_scale_shift(bn1, S1, n)
    out = ops.affine_act(z1, sc1, sh1, "relu")
    saved = dict(x=x, x1=x1, z0=z0, a0=a0, sc0=sc0, sh0=sh0, m0=m0, i0=i0, z1=z1, sc1=sc1, sh1=sh1, m1=m1, i1=i1, n=n)
    return out, saved


def cbam_fwd(mod, x):
    """CBAM forward (layers.py:138-141) with the spatial gate's BatchNorm2d(1) in either mode.  Returns (out, saved)."""
    ca, sa_mod = mod.channel_att, mod.spatial_att
    avg, mx = ops.cbam_pool(x)
    l1, l2 = ca.MLP[1], ca.MLP[3]
    sc = ops.cbam_mlp(avg, mx, _p(l1.weight), _p(l1.bias), _p(l2.weight), _p(l2.bias))
    pooled = ops.cbam_reduce(x, sc)
    _, raw = ops.cbam_gate(pooled, _p(sa_mod.conv.weight), None, want_raw=True)
    B, _, H, W = x.shape
    bn = sa_mod.bn
    S = ops.channel_stats(raw)
    g_sc, g_sh, g_m, g_i = bn_scale_shift(bn, S, B * H * W)
    sa = ops.affine_act(raw, g_sc, g_sh, "sigmoid")
    out = ops.cbam_scale(x, sc, sa)
    saved = dict(x=x, avg=avg, mx=mx, sc=sc, pooled=pooled, raw=raw, sa=sa, g_sc=g_sc, g_sh=g_sh, g_m=g_m, g_i=g_i)
    return out, saved


# =============================================================================================
# backward building blocks (thin wrappers over the C ABI; accumulate-into semantics noted)
# =============================================================================================
from . import _lib  # noqa: E402

_ptr, _call, _stream = ops._ptr, ops._call, ops._stream


# Gradient sinks: a training session (train.TrainSession) owns ONE flat gradient bucket; registering its views here makes
# every backward kernel accumulate a parameter's gradient straight into its slot of the bucket (zeroed once per step by
# the session) -- no per-parameter zero-fill, no autograd AccumulateGrad copy, no gather before the all-reduce.
_grad_sink = {}


def add_grad_sinks(params, views):
    """params[i]'s gradient is accumulated into views[i] (same shape) by the block backward passes.  Returns the keys to
    hand to remove_grad_sinks (a parameter is identified by its storage address: it must stay alive while registered)."""
    keys = []
    for p, v in zip(params, views):
        _grad_sink[p.data_ptr()] = v
        keys.append(p.data_ptr())
    return keys


def remove_grad_sinks(keys):
    for k in keys:
        _grad_sink.pop(k, None)


def is_sunk(p):
    return p is not None and p.data_ptr() in _grad_sink


def _zeros_like_param(p):
    v = _grad_sink.get(p.data_ptr())
    if v is not None:
        return v
    return torch.zeros(p.shape, device=p.device, dtype=torch.float32)


def bn_act_bwd(dy, z, scale, shift, gamma, mean, invstd, count, train, act, dgamma, dbeta, dz_sum=None):
    """dL/dz for a = act(BN(z)) given dL/da; accumulates dgamma/dbeta (may be None) and, into ``dz_sum``, the per-channel
    sum of dz (the bias gradient of the conv that produced z) without another pass over dz."""
    B, C, H, W = z.shape
    P = H * W
    lib = _lib.load()
    sums = torch.zeros(2 * C, device=z.device, dtype=torch.float64)
    _call("smaat_bn_act_bwd_reduce", 8 * B * C * P, 0, lib.smaat_bn_act_bwd_reduce, _ptr(dy), _ptr(z), _ptr(scale), _ptr(shift),
          _ptr(sums), B, C, P, act, _stream())
    a = torch.empty(C, device=z.device)
    b = torch.empty_like(a)
    cc = torch.empty_like(a)
    _call("smaat_bn_bwd_coeffs", 64 * C, 0, lib.smaat_bn_bwd_coeffs, _ptr(sums), float(count), _ptr(gamma), _ptr(mean), _ptr(invstd),
          int(bool(train)), _ptr(a), _ptr(b), _ptr(cc), _ptr(dgamma), _ptr(dbeta), _ptr(dz_sum), C, _stream())
    dz = torch.empty_like(z)
    _call("smaat_bn_act_bwd_apply", 12 * B * C * P, 0, lib.smaat_bn_act_bwd_apply, _ptr(dy), _ptr(z), _ptr(scale), _ptr(shift), _ptr(a),
          _ptr(b), _ptr(cc), _ptr(dz), B, C, P, act, _stream())
    return dz


def pw_bwd(dz, d, weight, dW, db, need_input=True):
    """Pointwise 1x1 backward: returns dL/dd (tensor-core GEMM with W^T) and accumulates dW, db."""
    B, Cout, H, W = dz.shape
    K = d.shape[1]
    P = H * W
    lib = _lib.load()
    m = ops.wgrad_mode(ops.PW_MODES[ops.get_pointwise_mode()])
    if m != 0 and P % 4 == 0 and K >= 8 and Cout >= 8:      # tensor cores: split-K over pixels, register accumulators, fp32 atomics to merge
        _call(f"smaat_pw1x1_bwd_weight_tc[K{K}_N{Cout}_P{P}]", 4 * B * P * (K + Cout), 2 * B * P * K * Cout, lib.smaat_pw1x1_bwd_weight_tc,
              _ptr(dz), _ptr(d), _ptr(dW), _ptr(db), B, K, Cout, P, m, _stream())
    else:
        _call(f"smaat_pw1x1_bwd_weight[K{K}_N{Cout}_P{P}]", 4 * B * P * (K + Cout), 2 * B * P * K * Cout, lib.smaat_pw1x1_bwd_weight,
              _ptr(dz), _ptr(d), _ptr(dW), _ptr(db), B, K, Cout, P, _stream())
    if not need_input:
        return None
    w2d = weight.detach().reshape(Cout, K)
    wt = torch.empty((K, Cout), device=dz.device, dtype=torch.float32)
    _call("smaat_transpose", 8 * K * Cout, 0, lib.smaat_transpose, _ptr(w2d), _ptr(wt), Cout, K, _stream())
    return ops.pw1x1(dz, wt, None, None, False)          # dd[b] = W^T dz[b]: the forward kernel with K and Cout swapped


def dw_bwd(dd, dw_weight, x0, x1, in_scale, in_shift, k, dWdw, dbdw, need_input=True):
    """Depthwise 3x3 backward: accumulates weight/bias grads; returns (dx0, dx1) split over the virtual concat."""
    B, KC, H, W = dd.shape
    x0c, bs0, x1c, C1, bs1 = ops._concat_operands(x0, x1)
    C0 = x0c.shape[1]
    lib = _lib.load()
    _call("smaat_dw3x3_bwd_weight", 4 * B * H * W * (KC + C0 + C1), 20 * B * H * W * KC, lib.smaat_dw3x3_bwd_weight, _ptr(dd), _ptr(x0c),
          C0, bs0, _ptr(x1c), C1, bs1, _ptr(in_scale), _ptr(in_shift), _ptr(dWdw), _ptr(dbdw), B, H, W, k, _stream())
    if not need_input:
        return None, None
    dx0 = torch.empty((B, C0, H, W), device=dd.device, dtype=torch.float32)
    dx1 = torch.empty((B, C1, H, W), device=dd.device, dtype=torch.float32) if C1 else None
    _call("smaat_dw3x3_bwd_input", 4 * B * H * W * (KC + C0 + C1), 18 * B * H * W * KC, lib.smaat_dw3x3_bwd_input, _ptr(dd),
          _ptr(dw_weight.detach()), _ptr(dx0), C0, C0 * H * W, _ptr(dx1), C1, C1 * H * W, B, H, W, k, _stream())
    return dx0, dx1


def double_conv_bwd(mod, saved, g, need_x=True, need_x1=True):
    """Backward of double_conv_fwd.  Returns (dx, dx1, [12 parameter grads in DoubleConvDSFn.PARAMS order])."""
    ds0, bn0, ds1, bn1 = mod.double_conv[0], mod.double_conv[1], mod.double_conv[3], mod.double_conv[4]
    s = saved
    n = s["n"]
    k = ds0.kernels_per_layer
    g = ops._dense(g, "grad_output")

    def grads(ds, bn):
        return [_zeros_like_param(ds.depthwise.weight), _zeros_like_param(ds.depthwise.bias), _zeros_like_param(ds.pointwise.weight),
                _zeros_like_param(ds.pointwise.bias), _zeros_like_param(bn.weight), _zeros_like_param(bn.bias)]

    g0, g1 = grads(ds0, bn0), grads(ds1, bn1)
    tr0 = bn0.training or not bn0.track_running_stats
    tr1 = bn1.training or not bn1.track_running_stats
    # second DS conv: out = relu(BN1(z1)), z1 = pw(d1) + b, d1 = dw(relu(BN0(z0)))
    dz1 = bn_act_bwd(g, s["z1"], s["sc1"], s["sh1"], bn1.weight.detach(), s["m1"], s["i1"], n, tr1, 1, g1[4], g1[5], dz_sum=g1[3])
    d1 = s["d1"]
    if d1 is None:                                                      # set_recompute_depthwise: same kernel call as the forward's
        d1 = ops.dw3x3(s["z0"], _p(ds1.depthwise.weight), _p(ds1.depthwise.bias), k, in_scale=s["sc0"], in_shift=s["sh0"])
    dd1 = pw_bwd(dz1, d1, ds1.pointwise.weight, g1[2], None)           # bias gradient = sum dz: from the BN sums above
    del d1
    da0, _ = dw_bwd(dd1, ds1.depthwise.weight, s["z0"], None, s["sc0"], s["sh0"], k, g1[0], g1[1])
    # first DS conv
    dz0 = bn_act_bwd(da0, s["z0"], s["sc0"], s["sh0"], bn0.weight.detach(), s["m0"], s["i0"], n, tr0, 1, g0[4], g0[5], dz_sum=g0[3])
    need_in = need_x or (s["x1"] is not None and need_x1)
    d0 = s["d0"]
    if d0 is None:
        d0 = ops.dw3x3(s["x"], _p(ds0.depthwise.weight), _p(ds0.depthwise.bias), k, x1=s["x1"])
    dd0 = pw_bwd(dz0, d0, ds0.pointwise.weight, g0[2], None)
    del d0
    dx, dx1 = dw_bwd(dd0, ds0.depthwise.weight, s["x"], s["x1"], None, None, k, g0[0], g0[1], need_input=need_in)
    return dx, dx1, g0 + g1


def conv3x3_bwd(mod, idx, dz, x0, x1, dW, need_input=True):
    """Backward of DoubleConv conv ``idx`` over [x0, x1]: accumulates dW; returns (dx0, dx1).  The input gradient is the
    forward kernel on dz with the flipped, transposed weight; it splits over the virtual concat as channel views."""
    ops.conv3x3_bwd_weight(dz, x0, x1, dW)
    if not need_input:
        return None, None
    C0, C1 = x0.shape[1], (x1.shape[1] if x1 is not None else 0)
    wt, wops = mod.packed(idx, C0, C1, flip_transpose=True)
    dx = ops.conv3x3(dz, wt, C0 + C1, None, None, False, w_split=wops)
    return (dx[:, :C0], dx[:, C0:]) if C1 else (dx, None)


def dense_double_conv_bwd(mod, saved, g, need_x=True, need_x1=True):
    """Backward of dense_double_conv_fwd.  Returns (dx, dx1, [8 parameter grads in DoubleConvFn.PARAMS order])."""
    c0, bn0, c1, bn1 = mod.double_conv[0], mod.double_conv[1], mod.double_conv[3], mod.double_conv[4]
    s = saved
    n = s["n"]
    g = ops._dense(g, "grad_output")
    pg = [_zeros_like_param(p) for p in (c0.weight, c0.bias, bn0.weight, bn0.bias, c1.weight, c1.bias, bn1.weight, bn1.bias)]
    tr0 = bn0.training or not bn0.track_running_stats
    tr1 = bn1.training or not bn1.track_running_stats
    # second conv: out = relu(BN1(z1)), z1 = conv(a0) + b1; the conv bias gradient is sum dz1, from the BN sums
    dz1 = bn_act_bwd(g, s["z1"], s["sc1"], s["sh1"], bn1.weight.detach(), s["m1"], s["i1"], n, tr1, 1, pg[6], pg[7], dz_sum=pg[5])
    da0, _ = conv3x3_bwd(mod, 3, dz1, s["a0"], None, pg[4])
    del dz1
    # first conv: a0 = relu(BN0(z0)), z0 = conv([x, x1]) + b0
    dz0 = bn_act_bwd(da0, s["z0"], s["sc0"], s["sh0"], bn0.weight.detach(), s["m0"], s["i0"], n, tr0, 1, pg[2], pg[3], dz_sum=pg[1])
    del da0
    need_in = need_x or (s["x1"] is not None and need_x1)
    dx, dx1 = conv3x3_bwd(mod, 0, dz0, s["x"], s["x1"], pg[0], need_input=need_in)
    return dx, dx1, pg


def cbam_bwd(mod, saved, g):
    """Backward of cbam_fwd.  Returns (dx, [7 parameter grads in CBAMFn.PARAMS order])."""
    s = saved
    x, sc, sa = s["x"], s["sc"], s["sa"]
    B, C, H, W = x.shape
    P = H * W
    ca, sp = mod.channel_att, mod.spatial_att
    l1, l2, bn = ca.MLP[1], ca.MLP[3], sp.bn
    lib = _lib.load()
    g = ops._dense(g, "grad_output")
    dpre = torch.empty((B, 1, H, W), device=x.device)
    amax = torch.empty((B, H, W), device=x.device, dtype=torch.int32)
    _call("smaat_cbam_bwd_gate_in", 8 * B * C * P, 0, lib.smaat_cbam_bwd_gate_in, _ptr(g), _ptr(x), _ptr(sc), _ptr(sa), _ptr(dpre), _ptr(amax),
          B, C, P, _stream())
    d_bn_w, d_bn_b = _zeros_like_param(bn.weight), _zeros_like_param(bn.bias)
    train = bn.training or not bn.track_running_stats
    draw = bn_act_bwd(dpre, s["raw"], s["g_sc"], s["g_sh"], bn.weight.detach(), s["g_m"], s["g_i"], B * P, train, 0, d_bn_w, d_bn_b)
    dpooled = torch.empty((B, 2, H, W), device=x.device)
    d_conv = _zeros_like_param(sp.conv.weight)
    ks = sp.conv.weight.shape[-1]
    _call("smaat_cbam_gate_bwd", 16 * B * P, 0, lib.smaat_cbam_gate_bwd, _ptr(draw), _ptr(s["pooled"]), _ptr(sp.conv.weight.detach()),
          _ptr(dpooled), _ptr(d_conv), B, H, W, ks, _stream())
    dsc = torch.zeros((B, C), device=x.device)
    pkey = torch.zeros((B, C), device=x.device, dtype=torch.int64)     # packed (value, ~index) plane argmax of x
    _call("smaat_cbam_bwd_dsc", 8 * B * C * P, 0, lib.smaat_cbam_bwd_dsc, _ptr(g), _ptr(x), _ptr(sa), _ptr(dpooled), _ptr(amax), _ptr(dsc),
          _ptr(pkey), B, C, P, _stream())
    dw1, db1, dw2, db2 = (_zeros_like_param(l1.weight), _zeros_like_param(l1.bias), _zeros_like_param(l2.weight), _zeros_like_param(l2.bias))
    davg = torch.empty((B, C), device=x.device)
    dmx = torch.empty_like(davg)
    _call("smaat_cbam_mlp_bwd", 32 * B * C, 0, lib.smaat_cbam_mlp_bwd, _ptr(s["avg"]), _ptr(s["mx"]), _ptr(l1.weight.detach()),
          _ptr(l1.bias.detach()), _ptr(l2.weight.detach()), _ptr(sc), _ptr(dsc), _ptr(dw1), _ptr(db1), _ptr(dw2), _ptr(db2), _ptr(davg),
          _ptr(dmx), B, C, l1.weight.shape[0], _stream())
    dx = torch.empty_like(x)
    _call("smaat_cbam_bwd_dx", 8 * B * C * P, 0, lib.smaat_cbam_bwd_dx, _ptr(g), _ptr(sc), _ptr(sa), _ptr(dpooled), _ptr(amax), _ptr(davg),
          _ptr(dmx), _ptr(pkey), _ptr(dx), B, C, P, _stream())
    return dx, [dw1, db1, dw2, db2, d_conv, d_bn_w, d_bn_b]


def maxpool2_bwd(x, g):
    x = ops._dense(x, "x")
    g = ops._dense(g, "grad_output")
    B, C, H, W = x.shape
    dx = torch.empty_like(x)
    _call("smaat_maxpool2_bwd", 4 * B * C * (2 * H * W + (H // 2) * (W // 2)), 0, _lib.load().smaat_maxpool2_bwd, _ptr(x), _ptr(g), _ptr(dx),
          B * C, H, W, _stream())
    return dx


def upsample2x_pad_bwd(g, in_shape):
    g, gbs = ops._nchw_bstride(g, "grad_output")
    B, C, H, W = in_shape
    Ho, Wo = g.shape[2], g.shape[3]
    dx = torch.empty(in_shape, device=g.device, dtype=torch.float32)
    _call("smaat_upsample2x_pad_bwd", 4 * B * C * (H * W + Ho * Wo), 0, _lib.load().smaat_upsample2x_pad_bwd, _ptr(g), gbs, _ptr(dx), B, C, H, W,
          Ho, Wo, _stream())
    return dx


def outconv_bwd(x, weight, g, need_x=True, bias=None):
    x = ops._dense(x, "x")
    g = ops._dense(g, "grad_output")
    B, Cin, H, W = x.shape
    ncls = weight.shape[0]
    dx = torch.empty_like(x) if need_x else None
    dW = _zeros_like_param(weight)
    db = _zeros_like_param(bias) if bias is not None else torch.zeros(ncls, device=x.device)
    _call("smaat_outconv_bwd", 4 * B * H * W * (2 * Cin + ncls), 0, _lib.load().smaat_outconv_bwd, _ptr(g), _ptr(x), _ptr(weight.detach()),
          _ptr(dx), _ptr(dW), _ptr(db), B, Cin, ncls, H * W, _stream())
    return dx, dW, db
