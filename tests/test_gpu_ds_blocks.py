"""The SmaAt-UNet blocks' training step (forward + backward through autograd) against float64 at the block shapes
SmaAt_UNet(12, 1, kernels_per_layer=2) runs at 288x288, bilinear and transposed-conv up paths.

The kernel tests (test_gpu_ds_forward_kernels.py, test_gpu_backward_kernels.py) hold every entry point to float64 at these
shapes, but not the glue that chains them into one block step: functional.double_conv_fwd / double_conv_bwd, bn_scale_shift,
bn_act_bwd, pw_bwd, dw_bwd and the autograd Functions behind DoubleConvDS, DownDS, UpDS and OutConv.  The glue decides which
saved tensor feeds which kernel, the BatchNorm count, the BN0+ReLU prologue of the second depthwise backward, the pointwise
bias gradient taken from the BatchNorm backward's sums, the eval branch's inv-std, the [skip, up] split of the concat
gradient and the recompute-depthwise path.  The block tests elsewhere run on frames of at most 48x48, and the whole-network
tests at 288x288 sit under a noise-calibrated bound loose enough to pass a 1 % error in one block's gradient.

  A  the float64 block references, on the CPU: against autograd of oracle/torch_port.py's double_conv_ds / down_ds / up_ds
     (bilinear and transposed) on small shapes, train and eval, with tied 2x2 max-pool windows; and the fp32-coordinate
     bilinear upsample against F.interpolate
  B  train mode at every block of the network: output, input gradients (skip and low input of the up blocks), every
     parameter gradient (the transposed conv's and OutConv's included), running statistics, num_batches_tracked
  C  eval-mode BatchNorm with gradients on at inc, down4, up1 and up4: the conv-bias gradients are non-zero there, so the
     pointwise bias gradient (dz_sum of smaat_bn_bwd_coeffs) and the depthwise db are checked by value; running buffers stay
     bit-unchanged
  D  functional.set_recompute_depthwise(True) at inc and up4; gradient sinks (functional.add_grad_sinks) at up1

  block   input(s) (C @ plane)                 DoubleConvDS (k = 2)            conv plane   B
  inc     12 @ 288                             12 -> 64 -> 64                  288          2
  down1   64 @ 288 (max-pool)                  64 -> 128 -> 128                144          4
  down2   128 @ 144                            128 -> 256 -> 256               72           8
  down3   256 @ 72                             256 -> 512 -> 512               36           16
  down4   512 @ 36                             512 -> 512 -> 512               18           32
  up1     low 512 @ 18, skip 512 @ 36          [512 | 512] -> 512 -> 256       36           16
  up2     low 256 @ 36, skip 256 @ 72          [256 | 256] -> 256 -> 128       72           8
  up3     low 128 @ 72, skip 128 @ 144         [128 | 128] -> 128 -> 64        144          4
  up4     low 64 @ 144, skip 64 @ 288          [64 | 64] -> 64 -> 64           288          2
  outc    64 @ 288                             OutConv 64 -> 1                 288          2
  up1T    low 1024 @ 18, skip 512 @ 36         ConvT 1024 -> 512, [512 | 512] -> 512 -> 512     36    16
  up4T    low 128 @ 144, skip 64 @ 288         ConvT 128 -> 64, [64 | 64] -> 64 -> 64           288   2

The batch sizes are not bench.py's B = 32: they keep the largest float64 tensor of the references near 340 MB (the 256-channel
depthwise result of up4 at 288x288, B = 2) while every BatchNorm still normalises over >= 10 368 samples per channel.

Conventions:
  * the references are float64 autograd of F.conv2d(groups=Cin) (depthwise), a 1x1 F.conv2d (pointwise) and
    F.batch_norm(momentum=0.1, eps=1e-5) on float64 copies of the running buffers;
  * every selection is routed by the kernels' own decision, so that a value within rounding of a threshold cannot send the
    full upstream gradient down different paths: the first ReLU by the sign of z0 * sc0 + sh0 evaluated in float64 from the
    saved fp32 z0, sc0, sh0 (the product is exact, so the sign is that of the kernels' fmaf), the second ReLU by out > 0,
    the 2x2 max-pool by the first maximum of the fp32 input (row-major window order).  The ReLU routings may differ from
    the reference's own pre-activation signs only where the reference is within the routing bound of 0;
  * the bilinear upsample builds its source coordinates in fp32 as upsample.cu does (ry = (float)(H-1) / (float)(2H-1),
    sy = ry * (float)u): with exact coordinates the ~1e-5 coordinate rounding (test_gpu_backward_kernels.py part E) would
    set the floor of the block bound;
  * in train mode the four conv-bias gradients are mathematically zero (the batch mean cancels them): they are bounded
    relative to the block's largest gradient;
  * sunk gradients start from a non-zero pattern in the flat buffer and are checked as init + gradient;
  * errors are max |got - ref| / max |ref|, as tests/_util.assert_close measures them.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than 10x
above it:

  quantity                                               fp32                     tf32x3
                                                         observed / bound         observed / bound
  B-D  out, dx, parameter gradients, running statistics  4.2e-6 / 2e-5            1.1e-4 / 3e-4
       conv-bias gradients of train mode (zero), as a    4.9e-7 / 4e-6            2.3e-5 / 2e-4
       fraction of the block's largest gradient
       ReLU routings that differ: |pre| / max |pre|      6.1e-7 / 3e-6            5.2e-6 / 5e-5
                                                         (<= 8 per ReLU)          (<= 24 per ReLU)
  B    ConvTranspose2d bias gradient, train mode         6.7e-6 / 5e-5            3.2e-4 / 2e-3

The largest block errors are the pointwise weight gradients of the first DS conv in tf32x3 (the split-K tensor-core GEMM
over 41 472 .. 165 888 pixels, fed by a dz that already carries the forward's tf32x3 error).  The transposed conv's bias
gradient in train mode is the pixel sum of dL/d(up), which the BatchNorm cancels down to the depthwise conv's image-border
terms: the sum of |terms| is 280x (up1T) and 2 800x (up4T) its result, and that factor multiplies the elementwise error
of the gradient flowing in.  The summation itself is not the limit: against a float64 sum of the kernels' own dL/d(up) the
bias gradient is within 3.7e-6 in both modes.  num_batches_tracked and the eval-mode running buffers are exact.  The whole
file runs in 8-13 s on one H100 at a peak of 2.0-2.5 GiB allocated.
"""
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from smaat_unet_b200 import functional as Fn
from smaat_unet_b200 import ops

gpu = pytest.mark.gpu
KPL = 2                      # kernels_per_layer of the network under test
BN_EPS, BN_MOM = 1e-5, 0.1
MODES = ("fp32", "tf32x3")

# max |got - ref| / max |ref| bounds (see the module docstring for the observed figures)
ERR_BOUND = {
    "block": {"fp32": 2e-5, "tf32x3": 3e-4},        # out, dx, parameter gradients, running statistics
    "zero": {"fp32": 4e-6, "tf32x3": 2e-4},         # train-mode conv-bias gradients (mathematically 0), vs the largest gradient
    "routing": {"fp32": 3e-6, "tf32x3": 5e-5},      # |pre| / max |pre| where a kernel ReLU routing differs from the reference's
    "convt_bias": {"fp32": 5e-5, "tf32x3": 2e-3},   # train-mode ConvTranspose2d bias gradient: a near-cancelling sum
}

# the parameters in autograd.DoubleConvDSFn.params order and the running buffers, relative to the DoubleConvDS
PARAM_KEYS = [key for i in (0, 3) for key in (f"double_conv.{i}.depthwise.weight", f"double_conv.{i}.depthwise.bias",
                                              f"double_conv.{i}.pointwise.weight", f"double_conv.{i}.pointwise.bias",
                                              f"double_conv.{i + 1}.weight", f"double_conv.{i + 1}.bias")]
BUF_KEYS = ["double_conv.1.running_mean", "double_conv.1.running_var", "double_conv.4.running_mean", "double_conv.4.running_var"]
ZERO_IN_TRAIN = {"double_conv.0.depthwise.bias", "double_conv.0.pointwise.bias", "double_conv.3.depthwise.bias",
                 "double_conv.3.pointwise.bias"}
PREFIX = {"inc": "", "down": "maxpool_conv.1.", "up": "conv.", "upT": "conv."}     # the DoubleConvDS inside each block kind


# ------------------------------------------------------------------------------------------------------------------ helpers
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=g, device=g.device) * scale + shift


def _rand(shape, g, lo=0.0, hi=1.0):
    return torch.rand(shape, generator=g, device=g.device) * (hi - lo) + lo


def _rel(got, ref):
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _check(got, ref, tol, what):
    e = _rel(got, ref)
    print(f"ERR {what}: {e:.3e} (bound {tol:.1e})")
    assert e == e and e <= tol, f"{what}: max rel err {e:.3e} > {tol:.1e}"
    return e


# ------------------------------------------------------------------------------------------------------ float64 references
def ds_conv_ref(x, dw_w, dw_b, pw_w, pw_b):
    """DepthwiseSeparableConv: 3x3 depthwise (kernels_per_layer outputs per channel), then the 1x1 pointwise conv."""
    return F.conv2d(F.conv2d(x, dw_w, dw_b, padding=1, groups=x.shape[1]), pw_w, pw_b)


def double_conv_ds_ref(x, params, bufs, masks, training):
    """(DS conv => BatchNorm2d => ReLU) x 2 with the ReLUs routed by the given 0/1 masks.  ``params`` in PARAM_KEYS order;
    ``bufs`` (float64 running mean / var of both BatchNorms) are updated in place in train mode.  Returns (out, (pre0, pre1))
    with pre the BatchNorm outputs."""
    dw0, db0, pw0, pb0, g0, b0, dw1, db1, pw1, pb1, g1, b1 = params
    n0 = F.batch_norm(ds_conv_ref(x, dw0, db0, pw0, pb0), bufs[0], bufs[1], g0, b0, training=training, momentum=BN_MOM, eps=BN_EPS)
    n1 = F.batch_norm(ds_conv_ref(n0 * masks[0], dw1, db1, pw1, pb1), bufs[2], bufs[3], g1, b1, training=training, momentum=BN_MOM,
                      eps=BN_EPS)
    return n1 * masks[1], (n0, n1)


def _windows(x):
    B, C, H, W = x.shape
    Ho, Wo = H // 2, W // 2
    return x[:, :, :2 * Ho, :2 * Wo].reshape(B, C, Ho, 2, Wo, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, Ho, Wo, 4)


def maxpool2_first_index(x):
    """(B, C, H/2, W/2, 1) position 0..3 of the first maximum of each 2x2 window, row-major."""
    w = _windows(x)
    ar = torch.arange(4, device=x.device)
    return torch.where(w == w.amax(dim=4, keepdim=True), ar, 4).amin(dim=4, keepdim=True)


def maxpool2_ref(x, idx):
    """MaxPool2d(2) routed by ``idx`` (maxpool2_first_index): the gradient goes to that one window position."""
    return _windows(x).gather(4, idx).squeeze(4)


def _lerp_matrix(n, coords, device):
    """(2n, n) float64 matrix of align_corners=True bilinear x2 along one axis: output u reads s = u (n-1) / (2n-1) as
    (1 - l) v[i] + l v[min(i + 1, n - 1)], i = min(floor(s), n - 1), l = s - i.  coords="fp32" forms s as upsample.cu does:
    the ratio (float)(n-1) / (float)(2n-1) and its product with (float)u each rounded to fp32."""
    u = torch.arange(2 * n)
    if coords == "fp32":
        r = torch.tensor(float(n - 1), dtype=torch.float32) / torch.tensor(float(2 * n - 1), dtype=torch.float32)
        s = (r * u.float()).double()
    else:
        s = u.double() * (n - 1) / (2 * n - 1)
    i0 = s.floor().long().clamp(max=n - 1)
    lam = s - i0.double()
    m = torch.zeros(2 * n, n, dtype=torch.float64)
    m.index_put_((u, i0), 1 - lam, accumulate=True)
    m.index_put_((u, (i0 + 1).clamp(max=n - 1)), lam, accumulate=True)
    return m.to(device)


def upsample2x_ref(x, coords="fp32"):
    """nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True) as two float64 matrix products (see _lerp_matrix)."""
    H, W = x.shape[2:]
    return _lerp_matrix(H, coords, x.device) @ x @ _lerp_matrix(W, coords, x.device).t()


def pad_to(t, Ho, Wo):
    dY, dX = Ho - t.shape[2], Wo - t.shape[3]
    return F.pad(t, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])


def block_input_ref(kind, inputs, idx=None, up=None, coords="fp32"):
    """The DoubleConvDS input of a block: x (inc), the routed max-pool of x (down), or [skip, pad(up(low))] (up: bilinear;
    upT: ConvTranspose2d(k=2, s=2) with ``up`` = (weight, bias))."""
    if kind == "inc":
        return inputs[0]
    if kind == "down":
        return maxpool2_ref(inputs[0], idx)
    low, skip = inputs
    u = F.conv_transpose2d(low, up[0], up[1], stride=2) if kind == "upT" else upsample2x_ref(low, coords)
    return torch.cat([skip, pad_to(u, skip.shape[2], skip.shape[3])], dim=1)


# ============================================================================================= A: the references on the CPU
# (kind, block constructor args, input shapes): small shapes; "up_ds_bilinear_pad" pads the upsampled map to an odd skip
REF_CASES = {
    "double_conv_ds": ("inc", (5, 8), [(2, 5, 9, 11)]),
    "down_ds": ("down", (6, 8), [(2, 6, 10, 12)]),
    "up_ds_bilinear": ("up", (8, 6), [(2, 4, 5, 6), (2, 4, 10, 12)]),
    "up_ds_bilinear_pad": ("up", (8, 6), [(2, 4, 5, 6), (2, 4, 11, 13)]),
    "up_ds_transposed": ("upT", (8, 6), [(2, 8, 5, 6), (2, 4, 11, 13)]),
}


def _make_block(kind, cin, cout):
    if kind == "inc":
        return S.DoubleConvDS(cin, cout, kernels_per_layer=KPL)
    if kind == "down":
        return S.DownDS(cin, cout, kernels_per_layer=KPL)
    if kind == "outc":
        return S.OutConv(cin, cout)
    return S.UpDS(cin, cout, bilinear=(kind == "up"), kernels_per_layer=KPL)


def _init_block(mod, g):
    """Weights at fan-in scale, conv biases 0.3 N(0, 1), randomised BatchNorm affine and running buffers."""
    with torch.no_grad():
        for m in mod.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.ConvTranspose2d)):
                fan_in = m.weight.shape[0] if isinstance(m, torch.nn.ConvTranspose2d) else m.weight[0].numel()
                m.weight.copy_(_randn(m.weight.shape, g, fan_in ** -0.5))
                m.bias.copy_(_randn(m.bias.shape, g, 0.3))
            elif isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(_rand(m.weight.shape, g, 0.5, 1.5))
                m.bias.copy_(_randn(m.bias.shape, g, 0.3))
                m.running_mean.copy_(_randn(m.running_mean.shape, g, 0.1))
                m.running_var.copy_(_rand(m.running_var.shape, g, 0.5, 1.5))


def _port_masks(inner, sd, p, training):
    """The port's own ReLU routing: the signs of its two BatchNorm outputs (on a throwaway copy of the running buffers)."""
    sd = {k: v.detach().clone() for k, v in sd.items()}
    n0 = TP._bn(TP.ds_conv(inner, sd, p + ".double_conv.0"), sd, p + ".double_conv.1", training)
    n1 = TP._bn(TP.ds_conv(F.relu(n0), sd, p + ".double_conv.3"), sd, p + ".double_conv.4", training)
    return (n0 > 0).double(), (n1 > 0).double()


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("case", list(REF_CASES))
def test_block_references_match_the_torch_port(case, training):
    """Float64 on the CPU: with the masks and the max-pool argmax taken from the reference's own values, the block
    references (exact upsample coordinates) and autograd of oracle/torch_port.py agree on the output, every input and
    parameter gradient and the running buffers to 1e-12."""
    kind, (cin, cout), shapes = REF_CASES[case]
    g = torch.Generator().manual_seed(len(case) * 7 + training)
    mod = _make_block(kind, cin, cout)
    _init_block(mod, g)
    names = dict(mod.named_parameters())
    sd = {}
    for k, v in mod.state_dict().items():
        v = v.detach().clone()
        v = v.double() if v.is_floating_point() else v
        sd["blk." + k] = v.requires_grad_(True) if k in names else v
    q = "blk." + PREFIX[kind]
    bufs = [sd[q + k].clone() for k in BUF_KEYS]             # before the port updates its own in place
    xs = [torch.relu(_randn(s, g)).double() for s in shapes]      # about half exact zeros
    if kind == "down":
        xs[0][:, :, 2:4, 4:6] = 0.0                      # an all-zero window in every plane besides the ReLU's own: 4-way ties
    xp = [x.clone().requires_grad_(True) for x in xs]
    if kind == "inc":
        yp = TP.double_conv_ds(xp[0], sd, "blk", training)
    elif kind == "down":
        yp = TP.down_ds(xp[0], sd, "blk", training)
    else:
        yp = TP.up_ds(xp[0], xp[1], sd, "blk", training)
    gout = _randn(yp.shape, g).double()
    yp.backward(gout)

    idx = None
    if kind == "down":
        idx = maxpool2_first_index(xs[0])
        ties = (_windows(xs[0]) == _windows(xs[0]).amax(dim=4, keepdim=True)).sum(dim=4) > 1
        assert int(ties.sum()) > xs[0].shape[0] * xs[0].shape[1], "the pooled map must have tied windows"
    up = [sd["blk.up.weight"].detach().clone().requires_grad_(True), sd["blk.up.bias"].detach().clone().requires_grad_(True)] \
        if kind == "upT" else None
    with torch.no_grad():
        inner = block_input_ref(kind, xs, idx, up, coords="exact")
    masks = _port_masks(inner, sd, q[:-1], training)
    params = [sd[q + k].detach().clone().requires_grad_(True) for k in PARAM_KEYS]
    xr = [x.clone().requires_grad_(True) for x in xs]
    y, _ = double_conv_ds_ref(block_input_ref(kind, xr, idx, up, coords="exact"), params, bufs, masks, training)
    y.backward(gout)

    assert _rel(y.detach(), yp.detach()) <= 1e-12
    for a, b in zip(xr, xp):
        assert _rel(a.grad, b.grad) <= 1e-12
    gmax = max(p.grad.abs().max().item() for p in params)
    for k, p in zip(PARAM_KEYS, params):
        if training and k in ZERO_IN_TRAIN:     # rounding noise around 0 on both sides: against the largest gradient
            assert (p.grad - sd[q + k].grad).abs().max().item() <= 1e-12 * gmax, k
        else:
            assert _rel(p.grad, sd[q + k].grad) <= 1e-12, k
    for k, b in zip(BUF_KEYS, bufs):
        assert _rel(b, sd[q + k]) <= 1e-12, k
    if up is not None:
        assert _rel(up[0].grad, sd["blk.up.weight"].grad) <= 1e-12
        assert _rel(up[1].grad, sd["blk.up.bias"].grad) <= 1e-12


@pytest.mark.parametrize("H, W", [(5, 7), (1, 3), (18, 18), (144, 144), (72, 36)])
def test_upsample_reference_coordinates(H, W):
    """upsample2x_ref with exact coordinates is F.interpolate(bilinear, align_corners=True) in float64; with fp32
    coordinates it reproduces torch's fp32 CPU upsample (the same fp32 coordinate rounding) to fp32 arithmetic noise, and
    stays within the coordinate rounding of the exact one."""
    g = torch.Generator().manual_seed(H * 131 + W)
    x = _randn((2, 3, H, W), g).double()
    exact = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
    assert _rel(upsample2x_ref(x, "exact"), exact) <= 1e-12
    f32 = upsample2x_ref(x, "fp32")
    torch_f32 = F.interpolate(x.float(), scale_factor=2, mode="bilinear", align_corners=True)
    assert _rel(torch_f32, f32) <= 1e-6
    assert _rel(f32, exact) <= 2.0 ** -22 * max(H, W)     # |s32 - s| <= ~2^-23 s, slope <= 2 max |x|


# ================================================================================================= B-D: blocks on the H100
# name: (kind, in channels, out channels, conv plane, B).  up: UpDS(in, out) bilinear, low in // 2 @ plane / 2 and skip
# in // 2 @ plane; upT: UpDS(in, out, bilinear=False), low in @ plane / 2 and skip in // 2 @ plane
BLOCKS = {
    "inc": ("inc", 12, 64, 288, 2),
    "down1": ("down", 64, 128, 144, 4),
    "down2": ("down", 128, 256, 72, 8),
    "down3": ("down", 256, 512, 36, 16),
    "down4": ("down", 512, 512, 18, 32),
    "up1": ("up", 1024, 256, 36, 16),
    "up2": ("up", 512, 128, 72, 8),
    "up3": ("up", 256, 64, 144, 4),
    "up4": ("up", 128, 64, 288, 2),
    "outc": ("outc", 64, 1, 288, 2),
    "up1T": ("upT", 1024, 512, 36, 16),
    "up4T": ("upT", 128, 64, 288, 2),
}


def _relu_map(shape, g):
    """A DoubleConvDS output: ReLU of a BatchNorm'd map, about half exact zeros."""
    return torch.relu(_randn(shape, g))


def _cbam_map(shape, g):
    """A CBAM output: a ReLU'd map scaled by a channel gate and a spatial gate in (0, 1), non-negative with many zeros."""
    B, C, H, W = shape
    return _relu_map(shape, g) * _rand((B, C, 1, 1), g, 0.2, 1.0) * _rand((B, 1, H, W), g, 0.1, 1.0)


def _block_inputs(kind, cin, H, B, g):
    if kind == "inc":
        return [_rand((B, cin, H, H), g)]                                    # radar frames in [0, 1)
    if kind == "down":
        return [_relu_map((B, cin, 2 * H, 2 * H), g)]
    if kind == "outc":
        return [_relu_map((B, cin, H, H), g)]
    low_c = cin // 2 if kind == "up" else cin
    return [_cbam_map((B, low_c, H // 2, H // 2), g), _cbam_map((B, cin // 2, H, H), g)]


def _run_block(mod, kind, xs):
    if kind in ("inc", "down", "outc"):
        return mod(xs[0])
    return mod(xs[0], xs[1])


def _block_step(name, mode, training=True, recompute=False, sink=False):
    """One block forward + backward through autograd on the GPU, then the float64 reference; checks everything."""
    kind, cin, cout, H, B = BLOCKS[name]
    g = _gen(1000 + list(BLOCKS).index(name))
    mod = _make_block(kind, cin, cout).cuda()
    _init_block(mod, g)
    mod.train(training)
    xs = [t.requires_grad_(True) for t in _block_inputs(kind, cin, H, B, g)]
    gout = _randn((B, cout, H, H), g)
    q = PREFIX[kind]
    params = [mod.get_parameter(q + k) for k in PARAM_KEYS]
    bufs = [mod.get_buffer(q + k).detach().double().clone() for k in BUF_KEYS]
    bufs32 = [mod.get_buffer(q + k).detach().clone() for k in BUF_KEYS]
    nbts = [mod.get_buffer(q + f"double_conv.{i}.num_batches_tracked") for i in (1, 4)]
    up_params = [mod.up.weight, mod.up.bias] if kind == "upT" else []
    idx = maxpool2_first_index(xs[0].detach()) if kind == "down" else None
    keys = None
    if sink:          # one flat bucket, pre-filled with a non-zero pattern, sliced into a view per parameter
        flat = 0.5 + 0.25 * torch.sin(0.37 * torch.arange(sum(p.numel() for p in params), device="cuda", dtype=torch.float32))
        views, off = [], 0
        for p in params:
            views.append(flat[off:off + p.numel()].view(p.shape))
            off += p.numel()
        inits = [v.clone() for v in views]
    old_mode = ops.get_pointwise_mode()
    ops.set_pointwise_mode(mode)
    old_rc = Fn.set_recompute_depthwise(recompute)
    try:
        y = _run_block(mod, kind, xs)
        s = y.grad_fn.saved
        if recompute:
            assert s["d0"] is None and s["d1"] is None
        # the kernels' routing: BN0+ReLU as fmaf(z0, sc0, sh0) > 0 (exact product in float64), BN1+ReLU as out > 0
        m0 = (s["z0"].double() * s["sc0"].double().view(1, -1, 1, 1) + s["sh0"].double().view(1, -1, 1, 1)) > 0
        masks = (m0.double(), (y.detach() > 0).double())
        del s, m0
        if sink:
            keys = Fn.add_grad_sinks(params, views)
        y.backward(gout)
    finally:
        if keys is not None:
            Fn.remove_grad_sinks(keys)
        Fn.set_recompute_depthwise(old_rc)
        ops.set_pointwise_mode(old_mode)
    y = y.detach()

    # float64 reference
    pr = [p.detach().double().requires_grad_(True) for p in params]
    ur = [p.detach().double().requires_grad_(True) for p in up_params]
    xr = [x.detach().double().requires_grad_(True) for x in xs]
    inner = block_input_ref(kind, xr, idx, ur)
    inner.retain_grad()
    yr, pre = double_conv_ds_ref(inner, pr, bufs, masks, training)
    yr.backward(gout.double())
    what = f"{name} {mode}{'' if training else ' eval'}{' recompute' if recompute else ''}{' sinks' if sink else ''}"
    tol, tol_route = ERR_BOUND["block"][mode], ERR_BOUND["routing"][mode]
    for mk, n, nm in zip(masks, pre, ("relu0", "relu1")):         # the routings may differ only within the bound of 0
        n = n.detach()
        off = (mk > 0) != (n > 0)
        worst = float(n[off].abs().max()) / float(n.abs().max()) if bool(off.any()) else 0.0
        print(f"ERR {what} {nm} routing: {int(off.sum())} differ, at |pre| <= {worst:.3e} of max (bound {tol_route:.1e})")
        assert worst <= tol_route, f"{what}: {nm} routing differs at |pre| = {worst:.3e} of its max"
    del pre, masks
    _check(y, yr, tol, f"{what} out")
    if kind in ("up", "upT"):
        _check(xs[1].grad, xr[1].grad, tol, f"{what} dskip")
        _check(xs[0].grad, xr[0].grad, tol, f"{what} dlow")
    else:
        _check(xs[0].grad, xr[0].grad, tol, f"{what} dx")
    gmax = max(p.grad.abs().max().item() for p in pr)
    for i, (k, p, r) in enumerate(zip(PARAM_KEYS, params, pr)):
        if sink:
            assert p.grad is None, f"{what}: {k} is sunk but has a .grad"
            got, i0 = views[i].double(), inits[i].double()
        else:
            got, i0 = p.grad.double(), torch.zeros_like(r.grad)
        if training and k in ZERO_IN_TRAIN:                       # mathematically zero: bounded against the largest gradient
            e = (got - i0).abs().max().item() / gmax
            tz = ERR_BOUND["zero"][mode]
            print(f"ERR {what} d{k} (zero, vs largest gradient): {e:.3e} (bound {tz:.1e})")
            assert e <= tz, f"{what} d{k}"
            continue
        _check(got, i0 + r.grad, tol, f"{what} d{k}{' (sunk)' if sink else ''}")
    if up_params:
        _check(up_params[0].grad, ur[0].grad, tol, f"{what} dup.weight")
        if training:
            # sum over pixels of dL/d(up): the train-mode BatchNorm makes the pointwise input gradient sum to 0 per channel,
            # so only the depthwise taps' image-border terms survive, and the sum is far smaller than the sum of its terms
            dup = inner.grad[:, xs[1].shape[1]:]
            cancel = dup.abs().sum(dim=(0, 2, 3)).max().item() / ur[1].grad.abs().max().item()
            _check(up_params[1].grad, ur[1].grad, ERR_BOUND["convt_bias"][mode], f"{what} dup.bias (sum |terms| / max |sum| = "
                   f"{cancel:.0f})")
        else:
            _check(up_params[1].grad, ur[1].grad, tol, f"{what} dup.bias")
    for k, b, b32 in zip(BUF_KEYS, bufs, bufs32):
        cur = mod.get_buffer(q + k)
        if training:
            _check(cur, b, tol, f"{what} {k}")
        else:
            assert torch.equal(cur, b32), f"{what}: eval changed {k}"
    for nbt in nbts:
        assert int(nbt) == (1 if training else 0)


def _outconv_step(mode):
    kind, cin, cout, H, B = BLOCKS["outc"]
    g = _gen(1000 + list(BLOCKS).index("outc"))
    mod = _make_block(kind, cin, cout).cuda()
    _init_block(mod, g)
    x = _block_inputs(kind, cin, H, B, g)[0].requires_grad_(True)
    gout = _randn((B, cout, H, H), g)
    old_mode = ops.get_pointwise_mode()
    ops.set_pointwise_mode(mode)
    try:
        y = mod(x)
        y.backward(gout)
    finally:
        ops.set_pointwise_mode(old_mode)
    w, b = (t.detach().double().requires_grad_(True) for t in (mod.conv.weight, mod.conv.bias))
    xr = x.detach().double().requires_grad_(True)
    yr = F.conv2d(xr, w, b)
    yr.backward(gout.double())
    what, tol = f"outc {mode}", ERR_BOUND["block"][mode]
    _check(y.detach(), yr, tol, f"{what} out")
    _check(x.grad, xr.grad, tol, f"{what} dx")
    _check(mod.conv.weight.grad, w.grad, tol, f"{what} dweight")
    _check(mod.conv.bias.grad, b.grad, tol, f"{what} dbias")


@gpu
@pytest.mark.parametrize("name", list(BLOCKS))
@pytest.mark.parametrize("mode", MODES)
def test_block_train_step_at_network_shapes(name, mode):
    """B: train-mode forward + backward of each block of SmaAt_UNet(12, 1, k=2) at 288x288 through autograd."""
    if name == "outc":
        _outconv_step(mode)
    else:
        _block_step(name, mode)


@gpu
@pytest.mark.parametrize("name", ["inc", "down4", "up1", "up4"])
@pytest.mark.parametrize("mode", MODES)
def test_block_eval_batchnorm_with_gradients(name, mode):
    """C: eval-mode BatchNorm with gradients on: the conv-bias gradients (dz_sum, the depthwise db) are non-zero and held
    to the ordinary bound; the running buffers come back bit-unchanged."""
    _block_step(name, mode, training=False)


@gpu
@pytest.mark.parametrize("name", ["inc", "up4"])
@pytest.mark.parametrize("mode", MODES)
def test_block_recompute_depthwise(name, mode):
    """D: set_recompute_depthwise(True) keeps no depthwise result and recomputes both in the backward."""
    _block_step(name, mode, recompute=True)


@gpu
def test_block_gradient_sinks():
    """D: every DoubleConvDS gradient of up1 accumulated into views of one flat buffer; .grad stays None."""
    _block_step("up1", "tf32x3", sink=True)
