"""Each kernel of the dense UNet / UNetAttention path against a float64 reference of the plain operation, at every 3x3 conv
layer shape UNet(12, 1) runs at 288x288 (bilinear and transposed-conv up path alike) and at the edges where the kernels
switch variants.

test_gpu_dense.py checks these kernels on small planes (H, W <= 20, fewer tiles than SMs) and the whole network at 288x288
under a network-level bound; neither gives a CTA several tiles (the halo and weight rings wrapping across tiles), reaches
the ragged patches of the production planes, the 8 channel passes of a 1024-channel input gradient, or the production
split-K count of the weight gradient.  Here every entry point is called directly (through ``ops`` / ``functional`` or the
C ABI) and compared with a float64 reference computed on the GPU:

  A  smaat_conv3x3_fwd: every conv layer, fp32 (CUDA cores), tf32 and tf32x3, eval epilogue (scale, shift, ReLU) and train
     epilogue (shift = conv bias, BatchNorm statistics)
  B  the input gradient: the forward kernel on dz with the flipped, transposed weight, split over the concat
  C  smaat_conv3x3_bwd_weight: tensor cores (tf32, tf32x3) and CUDA cores (fp32)
  D  smaat_conv3x3_pack_weight, smaat_convt2x2_pack_weight, smaat_pixel_shuffle2_pad_fwd (bit-exact), and the whole
     ConvTranspose2d(k=2, s=2) + pad up path as Up(bilinear=False) runs it
  E  refusals, Cout > 1024, strided inputs, batch independence and repeatability
  F  DoubleConv train-mode forward + backward through autograd at three production block shapes

Conventions:
  * the float64 references are DGEMMs over an explicit im2col (F.unfold): forward W . unfold(x), input gradient
    fold(W^T . dz), weight gradient dz . unfold(x)^T (test_reference_helpers_match_autograd checks them on the CPU);
  * tf32 mode hands both operands to the tensor core as raw fp32 bits; its reference takes the operands with the low 13
    mantissa bits cleared (TF32_ROUNDING), so the products are exact and the bound sits near fp32 accumulation noise;
    tf32x3 and fp32 are checked against the plain float64 reference;
  * accumulating outputs (dW) start from a non-zero buffer and are checked as init + gradient;
  * errors are max |got - ref| / max |ref|, as tests/_util.assert_close measures them;
  * a tf32 / tf32x3 request the tensor cores cannot take (the 18x18 layers, W % 4 == 2) runs on the CUDA cores and is held
    to the fp32 reference and bounds;
  * the DoubleConv reference routes its two ReLUs by the kernels' fp32 pre-activations (a value within rounding of 0 can
    land on either side, and the full upstream gradient follows it); the routings may differ only within the bound of 0.

The tensor core ignores the low 13 mantissa bits of a raw fp32 operand (truncation).  On three layers (64+64 -> 64 @288,
256 -> 128 @72, 512+512 -> 512 @36) the tf32 forward, input and weight gradients sit 1.7e-6 .. 2.4e-5 off the truncated-
operand reference and 7.8e-4 .. 9.6e-4 off a round-to-nearest one, about as far as from the exact operands.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (400 W power limit), no more than 10x
above it:

  quantity                                         fp32 (CUDA cores)   tf32              tf32x3
                                                   observed / bound    observed / bound  observed / bound
  A  forward y, eval and train epilogues           3.7e-6 / 2e-5       2.3e-5 / 1e-4     7.1e-5 / 3e-4
     BatchNorm sums of the train epilogue          3.8e-7 / 2e-6       2.0e-5 / 1e-4     6.2e-5 / 3e-4
  B  input gradient                                4.1e-6 / 2e-5       1.3e-5 / 6e-5     3.6e-5 / 2e-4
  C  weight gradient                               3.3e-6 / 2e-5       9.6e-6 / 5e-5     3.0e-5 / 2e-4
  D  transposed-conv up path                       1.4e-6 / 1e-5       2.5e-6 / 2e-5     9.0e-6 / 5e-5
  F  DoubleConv out, dx, parameter gradients,      3.3e-6 / 2e-5       -                 5.6e-5 / 3e-4
     running statistics
     ReLU routings that differ: |pre| / max        2.4e-7 (<= 2 per    -                 1.9e-5 (<= 19 per
                                                   ReLU)                                 ReLU)

The weight packings, the pixel shuffle, batch independence and repeated forwards are bit-exact.  The whole file runs in
~7 s on one H100 at a peak of 2.0 GiB allocated.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from smaat_unet_b200 import _lib, ops

gpu = pytest.mark.gpu
MODES = ("fp32", "tf32", "tf32x3")

# How the tensor core reads an fp32 bit pattern as a tf32 operand: "truncate" (low 13 mantissa bits ignored) or "nearest"
TF32_ROUNDING = "truncate"

# max |got - ref| / max |ref| bounds per quantity and arithmetic (see the module docstring for the observed figures)
ERR_BOUND = {
    "fwd": {"fp32": 2e-5, "tf32": 1e-4, "tf32x3": 3e-4},      # y, eval and train epilogues
    "stats": {"fp32": 2e-6, "tf32": 1e-4, "tf32x3": 3e-4},    # BatchNorm sums of the train epilogue
    "dgrad": {"fp32": 2e-5, "tf32": 6e-5, "tf32x3": 2e-4},
    "wgrad": {"fp32": 2e-5, "tf32": 5e-5, "tf32x3": 2e-4},
    "convt": {"fp32": 1e-5, "tf32": 2e-5, "tf32x3": 5e-5},
    "block": {"fp32": 2e-5, "tf32x3": 3e-4},                  # DoubleConv output, input and parameter gradients, running stats
}


# ------------------------------------------------------------------------------------------------------------------ helpers
def _p(t):
    return None if t is None else t.data_ptr()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=g, device="cuda") * scale + shift


def _rel(got, ref):
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _check(got, ref, tol, what):
    e = _rel(got, ref)
    print(f"ERR {what}: {e:.3e} (bound {tol:.1e})")
    assert e == e and e <= tol, f"{what}: max rel err {e:.3e} > {tol:.1e}"
    return e


def _offset(t):
    """A copy of ``t`` whose data starts one element past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def tf32(t, rounding=None):
    """fp32 -> the tf32 value the tensor core multiplies: low 13 mantissa bits cleared, after round-half-away-from-zero on
    the magnitude for ``rounding="nearest"``."""
    b = t.float().contiguous().view(torch.int32)
    if (rounding or TF32_ROUNDING) == "nearest":
        b = b + 0x1000
    return (b & -8192).view(torch.float32)


def _operands(mode, *ts):
    """float64 operands of the reference for the arithmetic ``mode`` ran in: tf32-rounded for the tensor cores' 'tf32', exact
    otherwise."""
    return [(tf32(t) if mode == "tf32" else t).double() for t in ts]


def _pad32(c):
    return (c + 31) // 32 * 32


# ---------------------------------------------------------------------------------------------- float64 references (GEMMs)
def conv3x3_ref(x, w):
    """nn.Conv2d(Cin, Cout, 3, padding=1, bias=False)(x) as one GEMM over an explicit im2col: W (Cout, 9 Cin) . unfold(x)."""
    B, _, H, W = x.shape
    Cout = w.shape[0]
    return (w.reshape(Cout, -1) @ F.unfold(x, 3, padding=1)).view(B, Cout, H, W)


def conv3x3_input_grad_ref(dz, w):
    """Input gradient of conv3x3_ref for output gradient dz: fold(W^T . dz)."""
    B, Cout, H, W = dz.shape
    return F.fold(w.reshape(Cout, -1).t() @ dz.reshape(B, Cout, H * W), (H, W), 3, padding=1)


def conv3x3_weight_grad_ref(dz, x):
    """Weight gradient of conv3x3_ref for output gradient dz: dz . unfold(x)^T, summed over the batch."""
    B, Cout, H, W = dz.shape
    return torch.einsum("bop,bkp->ok", dz.reshape(B, Cout, H * W), F.unfold(x, 3, padding=1)).view(Cout, x.shape[1], 3, 3)


def convt2x2_pad_ref(x, w, bias, Ho, Wo):
    """nn.ConvTranspose2d(Cin, Cout, 2, stride=2)(x) + F.pad to (Ho, Wo): one GEMM, the four taps never overlap."""
    B, _, H, W = x.shape
    Cout = w.shape[1]
    y = torch.einsum("bcij,cokl->boikjl", x, w).reshape(B, Cout, 2 * H, 2 * W) + bias.view(1, Cout, 1, 1)
    dY, dX = Ho - 2 * H, Wo - 2 * W
    return F.pad(y, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])


def test_reference_helpers_match_autograd():
    """The GEMM references against float64 autograd of F.conv2d / F.conv_transpose2d on the CPU, over a concat of two partial
    32-channel chunks and W % 4 != 0; and the tf32 operand rounding on hand-picked bit patterns."""
    gen = torch.Generator().manual_seed(3)
    for B, Cin, Cout, H, W in ((2, 12 + 20, 24, 7, 10), (1, 5, 9, 6, 8), (3, 8, 4, 5, 3)):
        x = torch.randn(B, Cin, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
        w = torch.randn(Cout, Cin, 3, 3, generator=gen, dtype=torch.float64, requires_grad=True)
        dz = torch.randn(B, Cout, H, W, generator=gen, dtype=torch.float64)
        z = F.conv2d(x, w, padding=1)
        z.backward(dz)
        xd, wd = x.detach(), w.detach()
        assert torch.allclose(conv3x3_ref(xd, wd), z.detach(), rtol=1e-12, atol=1e-12)
        assert torch.allclose(conv3x3_input_grad_ref(dz, wd), x.grad, rtol=1e-12, atol=1e-12)
        assert torch.allclose(conv3x3_weight_grad_ref(dz, xd), w.grad, rtol=1e-12, atol=1e-12)
    for B, Cin, Cout, H, W, Ho, Wo in ((2, 6, 4, 3, 5, 7, 13), (1, 3, 2, 4, 4, 8, 8)):
        x = torch.randn(B, Cin, H, W, generator=gen, dtype=torch.float64)
        w = torch.randn(Cin, Cout, 2, 2, generator=gen, dtype=torch.float64)
        b = torch.randn(Cout, generator=gen, dtype=torch.float64)
        dY, dX = Ho - 2 * H, Wo - 2 * W
        ref = F.pad(F.conv_transpose2d(x, w, b, stride=2), [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])
        assert torch.allclose(convt2x2_pad_ref(x, w, b, Ho, Wo), ref, rtol=1e-12, atol=1e-12)
    v = torch.tensor([1 + 2 ** -10, 1 + 2 ** -11, -(1 + 2 ** -11), 1 + 2 ** -11 + 2 ** -20, 3.0], dtype=torch.float32)
    assert tf32(v, "truncate").tolist() == [1 + 2 ** -10, 1.0, -1.0, 1.0, 3.0]
    assert tf32(v, "nearest").tolist() == [1 + 2 ** -10, 1 + 2 ** -10, -(1 + 2 ** -10), 1 + 2 ** -10, 3.0]


# ---------------------------------------------------------------------------------------------------------- layer shapes
# (C0, C1, Cout, H = W): the 3x3 convs of UNet(12, 1) at 288x288, Cin = [C0 | C1] (Up's virtual concat [skip | upsampled]).
# bilinear=True and bilinear=False share all of them but the 18x18 ones of down4 with bilinear=False (512 -> 1024 -> 1024).
LAYERS = [
    (12, 0, 64, 288), (64, 0, 64, 288), (64, 64, 64, 288),                            # inc, up4: N_TILE 64, PW 32
    (64, 0, 128, 144), (128, 0, 128, 144), (128, 128, 128, 144), (128, 0, 64, 144),   # down1, up3: PW 16
    (128, 0, 256, 72), (256, 0, 256, 72), (256, 256, 256, 72), (256, 0, 128, 72),     # down2, up2: ragged right patch
    (256, 0, 512, 36), (512, 0, 512, 36), (512, 512, 512, 36), (512, 0, 256, 36),     # down3, up1: ragged right and bottom
    (512, 0, 512, 18), (512, 0, 1024, 18), (1024, 0, 1024, 18),                       # down4: CUDA cores in every mode
]


def _lid(layer):
    C0, C1, Cout, H = layer
    return f"{C0}{'+' + str(C1) if C1 else ''}to{Cout}_S{H}"


def _batch(H):
    return {288: 1, 144: 2}.get(H, 4)


def _layer_data(layer):
    C0, C1, Cout, H = layer
    g = _gen(C0 * 131 + C1 * 17 + Cout * 7 + H)
    x = _randn((_batch(H), C0 + C1, H, H), g)
    w = _randn((Cout, C0 + C1, 3, 3), g, (9 * (C0 + C1)) ** -0.5)
    return g, x, w


def _split(x, C0, C1):
    return x[:, :C0].contiguous(), (x[:, C0:].contiguous() if C1 else None)


def _kernel(prof):
    names = list(prof.summary())
    assert len(names) == 1, names
    return names[0]


def _takes_tc(mode, W):
    return mode != "fp32" and W % 4 == 0


def _arith(mode, W):
    """The arithmetic a tensor-core mode request runs in: W % 4 != 0 takes the CUDA-core kernel (exact fp32 products)."""
    return mode if _takes_tc(mode, W) else "fp32"


# ============================================================================================================= A: forward
@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=_lid)
@pytest.mark.parametrize("mode", MODES)
def test_conv3x3_forward_at_network_shapes(layer, mode):
    """y = relu(scale * conv(x) + shift) (eval) and y = conv(x) + bias with the BatchNorm sums (train, as
    functional.dense_double_conv_fwd calls it) in every mode; the kernel that ran is the one the shape selects."""
    C0, C1, Cout, H = layer
    g, x, w = _layer_data(layer)
    x0, x1 = _split(x, C0, C1)
    scale = torch.rand(Cout, generator=g, device="cuda") + 0.5
    shift = _randn((Cout,), g)
    bias = _randn((Cout,), g, 0.3)
    wp = ops.conv3x3_pack_weight(w, C0, C1)
    ws = ops.split_tf32(wp) if mode == "tf32x3" else None
    am = _arith(mode, H)
    z = conv3x3_ref(*_operands(am, x, w))
    what = f"fwd {_lid(layer)} {mode}"
    tol = ERR_BOUND["fwd"][am]
    with ops.profile() as prof:
        y = ops.conv3x3(x0, wp, Cout, scale, shift, True, x1=x1, mode=mode, w_split=ws)
    assert _kernel(prof) == ("smaat_conv3x3_fwd" if _takes_tc(mode, H) else "smaat_conv3x3_fwd_simt")
    _check(y, torch.relu(z * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)), tol, f"{what} eval")
    stats = ops.new_stats(Cout, x.device)
    y = ops.conv3x3(x0, wp, Cout, None, bias, False, x1=x1, mode=mode, w_split=ws, stats=stats)
    zb = z + bias.double().view(1, -1, 1, 1)
    _check(y, zb, tol, f"{what} train")
    _check(stats[:Cout], zb.sum(dim=(0, 2, 3)), ERR_BOUND["stats"][am], f"{what} stats sum")
    _check(stats[Cout:], (zb * zb).sum(dim=(0, 2, 3)), ERR_BOUND["stats"][am], f"{what} stats sum of squares")


# ====================================================================================================== B: input gradient
@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=_lid)
@pytest.mark.parametrize("mode", MODES)
def test_conv3x3_input_gradient_at_network_shapes(layer, mode):
    """dx = the forward kernel on dz with the flipped, transposed weight (functional.conv3x3_bwd), split over the concat:
    up1.0 produces 1024 channels in 8 passes, inc.0 12 channels in one N tile with 52 dead columns."""
    C0, C1, Cout, H = layer
    g, x, w = _layer_data(layer)
    dz = _randn((x.shape[0], Cout, H, H), g)
    wt = ops.conv3x3_pack_weight(w, C0, C1, flip_transpose=True)
    ws = ops.split_tf32(wt) if mode == "tf32x3" else None
    am = _arith(mode, H)
    ref = conv3x3_input_grad_ref(*_operands(am, dz, w))
    with ops.profile() as prof:
        dx = ops.conv3x3(dz, wt, C0 + C1, None, None, False, mode=mode, w_split=ws)
    assert _kernel(prof) == ("smaat_conv3x3_fwd" if _takes_tc(mode, H) else "smaat_conv3x3_fwd_simt")
    what = f"dgrad {_lid(layer)} {mode}"
    _check(dx[:, :C0], ref[:, :C0], ERR_BOUND["dgrad"][am], f"{what} dx0")
    if C1:
        _check(dx[:, C0:], ref[:, C0:], ERR_BOUND["dgrad"][am], f"{what} dx1")


# ===================================================================================================== C: weight gradient
@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=_lid)
@pytest.mark.parametrize("mode", MODES)
def test_conv3x3_weight_gradient_at_network_shapes(layer, mode):
    """dW += dz . unfold([x0 | x1])^T: tensor cores in tf32x3 and tf32 (CUDA cores where W % 4 != 0), CUDA cores in fp32,
    accumulating into a non-zero dW.  B = 1 at 288 already reaches the production split-K count."""
    C0, C1, Cout, H = layer
    g, x, w = _layer_data(layer)
    x0, x1 = _split(x, C0, C1)
    dz = _randn((x.shape[0], Cout, H, H), g)
    am = _arith(mode, H)
    ref = conv3x3_weight_grad_ref(*_operands(am, dz, x))
    dW0 = _randn(ref.shape, g, 0.3 * ref.abs().max().item())
    dW = dW0.clone()
    with ops.profile() as prof:
        ops.conv3x3_bwd_weight(dz, x0, x1, dW, mode=mode)
    assert _kernel(prof) == ("smaat_conv3x3_bwd_weight" if _takes_tc(mode, H) else "smaat_conv3x3_bwd_weight_simt")
    _check(dW, dW0.double() + ref, ERR_BOUND["wgrad"][am], f"wgrad {_lid(layer)} {mode}")


# ========================================================================================== D: packing, transposed-conv up
def conv3x3_pack_ref(w, C0, C1, flip_transpose=False):
    """smaat_conv3x3_pack_weight restated: wp[o][3 dy + dx][k], k = c for x0's channels, C0p + c for x1's, zero padding; or
    (flip_transpose) wp[c][3 dy + dx][o] = w[o][c][2 - dy][2 - dx], o padded to 32."""
    Cout, Cin = w.shape[:2]
    if flip_transpose:
        out = torch.zeros((Cin, 9, _pad32(Cout)), device=w.device)
        out[:, :, :Cout] = w.flip(2, 3).permute(1, 2, 3, 0).reshape(Cin, 9, Cout)
        return out.view(Cin, -1)
    c0p = _pad32(C0)
    out = torch.zeros((Cout, 9, c0p + _pad32(C1)), device=w.device)
    out[:, :, :C0] = w[:, :C0].permute(0, 2, 3, 1).reshape(Cout, 9, C0)
    out[:, :, c0p:c0p + C1] = w[:, C0:].permute(0, 2, 3, 1).reshape(Cout, 9, C1)
    return out.view(Cout, -1)


@gpu
@pytest.mark.parametrize("Cout, C0, C1", [(64, 12, 0), (64, 12, 20), (40, 20, 12), (8, 3, 5), (1024, 512, 512), (512, 1024, 0),
                                          (1032, 64, 0)])
@pytest.mark.parametrize("flip", [False, True])
def test_conv3x3_pack_weight_is_exact(Cout, C0, C1, flip):
    w = _randn((Cout, C0 + C1, 3, 3), _gen(Cout + C0 * 3 + C1 * 5))
    ref = conv3x3_pack_ref(w, C0, C1, flip)
    wp = torch.full(ref.shape, float("nan"), device="cuda")      # the padding must be written, not inherited
    _lib.check(_lib.load().smaat_conv3x3_pack_weight(_p(w), _p(wp), Cout, C0, C1, int(flip), ops._stream()), "pack")
    assert torch.equal(wp, ref)
    assert torch.equal(ops.conv3x3_pack_weight(w, C0, C1, flip), ref)


@gpu
@pytest.mark.parametrize("Cin, Cout", [(1024, 512), (128, 64), (7, 5)])
def test_convt2x2_pack_weight_is_exact(Cin, Cout):
    w = _randn((Cin, Cout, 2, 2), _gen(Cin + Cout))
    assert torch.equal(ops.convt2x2_pack_weight(w), w.permute(2, 3, 1, 0).reshape(4 * Cout, Cin))


def pixel_shuffle2_pad_ref(t, bias, Cout, Ho, Wo):
    B, _, H, W = t.shape
    y = t.view(B, 2, 2, Cout, H, W).permute(0, 3, 4, 1, 5, 2).reshape(B, Cout, 2 * H, 2 * W)
    if bias is not None:
        y = y + bias.view(1, Cout, 1, 1)
    dY, dX = Ho - 2 * H, Wo - 2 * W
    return F.pad(y, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])


@gpu
@pytest.mark.parametrize("B, Cout, H, W, Ho, Wo", [(2, 64, 144, 144, 288, 288), (2, 5, 5, 7, 11, 17), (3, 4, 4, 6, 9, 15),
                                                   (1, 3, 3, 3, 8, 7)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_pixel_shuffle2_pad_is_exact(B, Cout, H, W, Ho, Wo, with_bias):
    """Bit for bit against view/permute + bias + F.pad (odd pads on either side, odd Wo); then into a channel slice of a
    wider NaN-filled buffer through the ABI: the channels outside the slice stay NaN."""
    g = _gen(B + Cout * 3 + H * 5 + Wo)
    t = _randn((B, 4 * Cout, H, W), g)
    bias = _randn((Cout,), g) if with_bias else None
    ref = pixel_shuffle2_pad_ref(t, bias, Cout, Ho, Wo)
    assert torch.equal(ops.pixel_shuffle2_pad(t, bias, Cout, Ho, Wo), ref)
    wide = torch.full((B, Cout + 5, Ho, Wo), float("nan"), device="cuda")
    sl = wide[:, 3:3 + Cout]
    _lib.check(_lib.load().smaat_pixel_shuffle2_pad_fwd(_p(t), _p(bias), _p(sl), wide.stride(0), B, Cout, H, W, Ho, Wo, ops._stream()),
               "pixel_shuffle2_pad_fwd")
    assert torch.equal(sl, ref)
    assert bool(wide[:, :3].isnan().all()) and bool(wide[:, 3 + Cout:].isnan().all())


# (Cin, H): the four ConvTranspose2d(Cin, Cin // 2, 2, stride=2) of UNet(12, 1, bilinear=False), H -> 2 H
CONVT_LAYERS = [(1024, 18), (512, 36), (256, 72), (128, 144)]


@gpu
@pytest.mark.parametrize("Cin, H", CONVT_LAYERS, ids=[f"{c}to{c // 2}_S{h}" for c, h in CONVT_LAYERS])
def test_transposed_up_forward_at_network_shapes(Cin, H):
    """Up(bilinear=False)._up_transposed: convt2x2_pack_weight -> pw1x1 GEMM to 4 Cout packed taps -> pixel_shuffle2_pad_fwd,
    against float64 ConvTranspose2d + pad, in every mode."""
    Cout = Cin // 2
    B = 2
    g = _gen(Cin + H)
    up = S.Up(Cin, Cin // 2, bilinear=False).cuda().eval()
    with torch.no_grad():
        up.up.weight.copy_(_randn(up.up.weight.shape, g, Cin ** -0.5))
        up.up.bias.copy_(_randn((Cout,), g, 0.3))
    x = _randn((B, Cin, H, H), g)
    w, b = up.up.weight.detach(), up.up.bias.detach()
    old = ops.get_pointwise_mode()
    for mode in MODES:
        ops.set_pointwise_mode(mode)
        try:
            with torch.no_grad():
                y = up._up_transposed(x, 2 * H, 2 * H)
        finally:
            ops.set_pointwise_mode(old)
        xr, wr = _operands(mode, x, w)
        _check(y, convt2x2_pad_ref(xr, wr, b.double(), 2 * H, 2 * H), ERR_BOUND["convt"][mode], f"convt {Cin}@{H} {mode}")


# ================================================================================================== E: edges and contracts
def _fwd_rc(x0, x1, wp, wlo, Cout, y, mode, scale=None, shift=None, stats=None):
    B, C0, H, W = x0.shape
    C1 = x1.shape[1] if x1 is not None else 0
    return _lib.load().smaat_conv3x3_fwd(_p(x0), C0, x0.stride(0), _p(x1), C1, x1.stride(0) if x1 is not None else 0, _p(wp), _p(wlo),
                                         _p(scale), _p(shift), _p(y), y.stride(0), _p(stats), B, H, W, Cout, 0, ops.PW_MODES[mode],
                                         ops._stream())


def _wgrad_rc(dz, x0, x1, dW, mode):
    B, C0, H, W = x0.shape
    C1 = x1.shape[1] if x1 is not None else 0
    return _lib.load().smaat_conv3x3_bwd_weight(_p(dz), _p(x0), C0, x0.stride(0), _p(x1), C1, x1.stride(0) if x1 is not None else 0,
                                                _p(dW), B, H, W, dz.shape[1], ops.PW_MODES[mode], ops._stream())


@gpu
@pytest.mark.parametrize("case", ["w_mod4", "cout_lt8", "x0_misaligned", "x1_misaligned"])
def test_conv3x3_forward_refusals(case):
    """The tensor-core modes return SMAAT_E_UNSUPPORTED (-3) and leave y untouched for each condition alone; ops.conv3x3
    takes the same data on the CUDA cores and gets it right."""
    g = _gen(len(case))
    B, H, W, C0, C1, Cout = 2, 8, 12 if case != "w_mod4" else 10, 16, 8, 24
    x = _randn((B, C0 + C1, H, W), g)
    w = _randn((Cout, C0 + C1, 3, 3), g, 0.2)
    x0, x1 = _split(x, C0, C1)
    if case == "x0_misaligned":
        x0 = _offset(x0)
    if case == "x1_misaligned":
        x1 = _offset(x1)
    if case == "cout_lt8":          # an input gradient into 4 channels: dz (24 channels) through the flipped weight of 4 -> 24
        w = _randn((24, 4, 3, 3), g, 0.2)
        x0, x1, C0, C1, Cout = _randn((B, 24, H, W), g), None, 24, 0, 4
        wp = ops.conv3x3_pack_weight(w, 4, 0, flip_transpose=True)
        ref = conv3x3_input_grad_ref(x0.double(), w.double())
    else:
        wp = ops.conv3x3_pack_weight(w, C0, C1)
        ref = conv3x3_ref(x.double(), w.double())
    hi, lo = ops.split_tf32(wp)
    for mode in ("tf32", "tf32x3"):
        y = torch.full((B, Cout, H, W), float("nan"), device="cuda")
        assert _fwd_rc(x0, x1, hi if mode == "tf32x3" else wp, lo if mode == "tf32x3" else None, Cout, y, mode) == -3
        torch.cuda.synchronize()
        assert bool(y.isnan().all())
        assert not ops.conv3x3_takes(x0, x1, wp, Cout, mode)
        with ops.profile() as prof:
            y = ops.conv3x3(x0, wp, Cout, None, None, False, x1=x1, mode=mode, w_split=(hi, lo) if mode == "tf32x3" else None)
        assert _kernel(prof) == "smaat_conv3x3_fwd_simt"
        _check(y, ref, ERR_BOUND["fwd"]["fp32"], f"refused fwd {case} {mode} -> simt")


@gpu
@pytest.mark.parametrize("case", ["w_mod4", "x0_misaligned", "x1_misaligned", "dz_misaligned"])
def test_conv3x3_weight_gradient_refusals(case):
    g = _gen(7 * len(case))
    B, H, W, C0, C1, Cout = 2, 8, 12 if case != "w_mod4" else 10, 16, 8, 24
    x = _randn((B, C0 + C1, H, W), g)
    dz = _randn((B, Cout, H, W), g)
    x0, x1 = _split(x, C0, C1)
    if case == "x0_misaligned":
        x0 = _offset(x0)
    if case == "x1_misaligned":
        x1 = _offset(x1)
    if case == "dz_misaligned":
        dz = _offset(dz)
    ref = conv3x3_weight_grad_ref(dz.double(), x.double())
    for mode in ("tf32", "tf32x3"):
        dW = torch.full((Cout, C0 + C1, 3, 3), float("nan"), device="cuda")
        assert _wgrad_rc(dz, x0, x1, dW, mode) == -3
        torch.cuda.synchronize()
        assert bool(dW.isnan().all())
        dW = torch.zeros_like(dW)
        with ops.profile() as prof:
            ops.conv3x3_bwd_weight(dz, x0, x1, dW, mode=mode)
        assert _kernel(prof) == "smaat_conv3x3_bwd_weight_simt"
        _check(dW, ref, ERR_BOUND["wgrad"]["fp32"], f"refused wgrad {case} {mode} -> simt")


@gpu
def test_conv3x3_more_than_1024_channels():
    """Cout > 1024 in the tensor-core modes: with an epilogue affine the request is refused (SMAAT_E_BADARG, y untouched);
    without one it runs: an input gradient into 1032 channels (9 channel passes) with its statistics."""
    g = _gen(1032)
    B, H, Cf, Cin = 2, 36, 64, 1032
    x = _randn((B, 64, H, H), g)
    wf = _randn((Cin, 64, 3, 3), g, 0.05)
    wp = ops.conv3x3_pack_weight(wf, 64)
    hi, lo = ops.split_tf32(wp)
    sc, sh = torch.ones(Cin, device="cuda"), torch.zeros(Cin, device="cuda")
    for mode in ("tf32", "tf32x3"):
        y = torch.full((B, Cin, H, H), float("nan"), device="cuda")
        assert _fwd_rc(x, None, hi if mode == "tf32x3" else wp, lo if mode == "tf32x3" else None, Cin, y, mode, scale=sc, shift=sh) == -1
        torch.cuda.synchronize()
        assert bool(y.isnan().all())
    w = _randn((Cf, Cin, 3, 3), g, (9 * Cf) ** -0.5)     # a Cin = 1032 -> Cf = 64 conv: its input gradient has 1032 channels
    dz = _randn((B, Cf, H, H), g)
    wt = ops.conv3x3_pack_weight(w, Cin, 0, flip_transpose=True)
    split = ops.split_tf32(wt)
    for mode in MODES:
        ref = conv3x3_input_grad_ref(*_operands(mode, dz, w))
        stats = ops.new_stats(Cin, dz.device)
        with ops.profile() as prof:
            dx = ops.conv3x3(dz, wt, Cin, None, None, False, mode=mode, w_split=split if mode == "tf32x3" else None, stats=stats)
        assert _kernel(prof) == ("smaat_conv3x3_fwd" if mode != "fp32" else "smaat_conv3x3_fwd_simt")
        _check(dx, ref, ERR_BOUND["dgrad"][mode], f"dgrad 64to1032 {mode}")
        _check(stats[:Cin], ref.sum(dim=(0, 2, 3)), ERR_BOUND["stats"][mode], f"dgrad 64to1032 {mode} stats sum")
        _check(stats[Cin:], (ref * ref).sum(dim=(0, 2, 3)), ERR_BOUND["stats"][mode], f"dgrad 64to1032 {mode} stats sum of squares")


@gpu
@pytest.mark.parametrize("layer", [(64, 64, 128, 36), (24, 40, 64, 288)], ids=_lid)
def test_conv3x3_strided_inputs(layer):
    """x0 and x1 as channel slices of wider tensors, read through their batch strides: the forward is bit-equal to the same
    call on contiguous copies (same kernel, same tiles), and the weight gradient matches float64."""
    C0, C1, Cout, H = layer
    g = _gen(C0 + C1 + H)
    B = 3 if H < 288 else 2
    big0, big1 = _randn((B, C0 + 6, H, H), g), _randn((B, C1 + 3, H, H), g)
    x0, x1 = big0[:, 4:4 + C0], big1[:, 1:1 + C1]
    assert x0.data_ptr() % 16 == 0 and x1.data_ptr() % 16 == 0 and not x0.is_contiguous()
    x = torch.cat([x0, x1], 1)
    w = _randn((Cout, C0 + C1, 3, 3), g, (9 * (C0 + C1)) ** -0.5)
    sc, sh = torch.rand(Cout, generator=g, device="cuda") + 0.5, _randn((Cout,), g)
    wp = ops.conv3x3_pack_weight(w, C0, C1)
    split = ops.split_tf32(wp)
    dz = _randn((B, Cout, H, H), g)
    for mode in MODES:
        ws = split if mode == "tf32x3" else None
        assert ops.conv3x3_takes(x0, x1, wp, Cout, mode) == (mode != "fp32")
        y = ops.conv3x3(x0, wp, Cout, sc, sh, True, x1=x1, mode=mode, w_split=ws)
        yc = ops.conv3x3(x0.contiguous(), wp, Cout, sc, sh, True, x1=x1.contiguous(), mode=mode, w_split=ws)
        assert torch.equal(y, yc), mode
        z = conv3x3_ref(*_operands(mode, x, w))
        _check(y, torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)), ERR_BOUND["fwd"][mode],
               f"strided fwd {mode}")
        dW = torch.zeros((Cout, C0 + C1, 3, 3), device="cuda")
        ops.conv3x3_bwd_weight(dz, x0, x1, dW, mode=mode)
        _check(dW, conv3x3_weight_grad_ref(*_operands(mode, dz, x)), ERR_BOUND["wgrad"][mode], f"strided wgrad {mode}")


# (Cin, Cout, H, W): PW 32 / 16 x N_TILE 64 / 128
BATCH_CASES = [(16, 64, 288, 288), (16, 128, 288, 288), (64, 64, 36, 36), (64, 128, 36, 36)]


@gpu
@pytest.mark.parametrize("Cin, Cout, H, W", BATCH_CASES, ids=["pw32_n64", "pw32_n128", "pw16_n64", "pw16_n128"])
def test_conv3x3_forward_is_batch_independent(Cin, Cout, H, W):
    """Tile shapes never depend on B: image b of a B = 4 forward is bit-equal to the same image run alone."""
    g = _gen(Cin * 5 + Cout + H)
    x = _randn((4, Cin, H, W), g)
    w = _randn((Cout, Cin, 3, 3), g, (9 * Cin) ** -0.5)
    sc, sh = torch.rand(Cout, generator=g, device="cuda") + 0.5, _randn((Cout,), g)
    wp = ops.conv3x3_pack_weight(w, Cin)
    split = ops.split_tf32(wp)
    for mode in ("tf32", "tf32x3"):
        ws = split if mode == "tf32x3" else None
        y4 = ops.conv3x3(x, wp, Cout, sc, sh, True, mode=mode, w_split=ws)
        for b in range(4):
            y1 = ops.conv3x3(x[b:b + 1].contiguous(), wp, Cout, sc, sh, True, mode=mode, w_split=ws)
            assert torch.equal(y4[b:b + 1], y1), (mode, b)


@gpu
@pytest.mark.parametrize("layer", [(64, 64, 64, 288), (512, 0, 512, 36)], ids=_lid)
def test_conv3x3_is_repeatable(layer):
    """Repeated forwards are bit-equal; the statistics and dW merge through atomics, so they are held to the bound only."""
    C0, C1, Cout, H = layer
    g, x, w = _layer_data(layer)
    x0, x1 = _split(x, C0, C1)
    bias = _randn((Cout,), g, 0.3)
    dz = _randn((x.shape[0], Cout, H, H), g)
    wp = ops.conv3x3_pack_weight(w, C0, C1)
    split = ops.split_tf32(wp)
    for mode in MODES:
        ws = split if mode == "tf32x3" else None
        zb = conv3x3_ref(*_operands(mode, x, w)) + bias.double().view(1, -1, 1, 1)
        dw_ref = conv3x3_weight_grad_ref(*_operands(mode, dz, x))
        first = None
        for rep in range(3):
            stats = ops.new_stats(Cout, x.device)
            y = ops.conv3x3(x0, wp, Cout, None, bias, False, x1=x1, mode=mode, w_split=ws, stats=stats)
            if first is None:
                first = y
            assert torch.equal(y, first), (mode, rep)
            _check(stats[:Cout], zb.sum(dim=(0, 2, 3)), ERR_BOUND["stats"][mode], f"repeat {rep} {mode} stats sum")
            dW = torch.zeros((Cout, C0 + C1, 3, 3), device="cuda")
            ops.conv3x3_bwd_weight(dz, x0, x1, dW, mode=mode)
            _check(dW, dw_ref, ERR_BOUND["wgrad"][mode], f"repeat {rep} {mode} wgrad")


# ================================================================================================== F: DoubleConv blocks
# (name, Cin split [C0, C1], mid, Cout, H, B)
BLOCKS = [("inc", (12, 0), 64, 64, 288, 1), ("up1.conv", (512, 512), 512, 256, 36, 4), ("down4", (512, 0), 512, 512, 18, 8)]


def _double_conv_ref(params, bufs, x, masks, eps, momentum):
    """float64 (Conv2d => BatchNorm2d(train) => ReLU) x 2 with the GEMM conv; the ReLUs route by the kernels' fp32 masks."""
    w0, b0, g0, be0, w1, b1, g1, be1 = params
    rm0, rv0, rm1, rv1 = bufs
    z0 = conv3x3_ref(x, w0) + b0.view(1, -1, 1, 1)
    n0 = F.batch_norm(z0, rm0, rv0, g0, be0, training=True, momentum=momentum, eps=eps)
    a0 = n0 * masks[0]
    z1 = conv3x3_ref(a0, w1) + b1.view(1, -1, 1, 1)
    n1 = F.batch_norm(z1, rm1, rv1, g1, be1, training=True, momentum=momentum, eps=eps)
    return n1 * masks[1], (n0, n1)


@gpu
@pytest.mark.parametrize("block", BLOCKS, ids=lambda b: b[0])
@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_double_conv_train_step_at_network_shapes(block, mode):
    """Train-mode DoubleConv forward + backward through autograd against float64 autograd of the same Conv2d / BatchNorm2d
    / ReLU stack (BatchNorm over >= 2 592 samples per channel): output, dx / dx1, every parameter gradient and the running
    statistics.  The reference takes its ReLU routing from the kernels' fp32 values (a pre-activation within rounding of 0
    may land on either side); the two routings may only differ where the reference is within the bound of 0."""
    name, (C0, C1), mid, Cout, H, B = block
    g = _gen(C0 + C1 + mid + H)
    old = ops.get_pointwise_mode()
    ops.set_pointwise_mode(mode)
    try:
        m = S.DoubleConv(C0 + C1, Cout, mid).cuda().train()
        with torch.no_grad():
            for idx in (0, 3):
                c, bn = m.double_conv[idx], m.double_conv[idx + 1]
                c.weight.copy_(_randn(c.weight.shape, g, (9 * c.in_channels) ** -0.5))
                c.bias.copy_(_randn(c.bias.shape, g, 0.3))
                bn.weight.copy_(torch.rand(bn.weight.shape, generator=g, device="cuda") + 0.5)
                bn.bias.copy_(_randn(bn.bias.shape, g, 0.3))
                bn.running_mean.copy_(_randn(bn.running_mean.shape, g, 0.1))
                bn.running_var.copy_(torch.rand(bn.running_var.shape, generator=g, device="cuda") + 0.5)
        ref_m = copy.deepcopy(m)
        x = _randn((B, C0 + C1, H, H), g)
        gout = _randn((B, Cout, H, H), g)
        x0 = x[:, :C0].contiguous().requires_grad_(True)
        x1 = x[:, C0:].contiguous().requires_grad_(True) if C1 else None
        y = m.run(x0, x1)
        saved = y.grad_fn.saved
        masks = ((saved["a0"] > 0).double(), (y.detach() > 0).double())
        y.backward(gout)
    finally:
        ops.set_pointwise_mode(old)

    names = ["conv0.weight", "conv0.bias", "bn0.weight", "bn0.bias", "conv1.weight", "conv1.bias", "bn1.weight", "bn1.bias"]
    mods = [ref_m.double_conv[i] for i in (0, 1, 3, 4)]
    params = [t.detach().double().requires_grad_(True) for mod in mods for t in (mod.weight, mod.bias)]
    bufs = [t.detach().double().clone() for mod in (mods[1], mods[3]) for t in (mod.running_mean, mod.running_var)]
    bn0 = mods[1]
    xr = x.double().requires_grad_(True)
    yr, pre = _double_conv_ref(params, bufs, xr, masks, bn0.eps, bn0.momentum)
    yr.backward(gout.double())
    what = f"block {name} {mode}"
    tol = ERR_BOUND["block"][mode]
    for mk, n, nm in zip(masks, pre, ("a0", "out")):   # the routings may differ only within the bound of 0
        n = n.detach()
        off = (mk > 0) != (n > 0)
        worst = float(n[off].abs().max()) / float(n.abs().max()) if bool(off.any()) else 0.0
        print(f"ERR {what} {nm} ReLU routing: {int(off.sum())} differ, at |pre| <= {worst:.3e} of max")
        assert worst <= tol, f"{what}: {nm} ReLU routing differs at |pre| = {worst:.3e} of its max"
    _check(y, yr, tol, f"{what} out")
    _check(x0.grad, xr.grad[:, :C0], tol, f"{what} dx0")
    if C1:
        _check(x1.grad, xr.grad[:, C0:], tol, f"{what} dx1")
    got = [t for i in (0, 1, 3, 4) for t in (m.double_conv[i].weight.grad, m.double_conv[i].bias.grad)]
    gmax = max(p.grad.abs().max().item() for p in params)
    for gk, p, nm in zip(got, params, names):
        if nm.startswith("conv") and nm.endswith("bias"):   # before a train-mode BatchNorm: mathematically zero
            e = gk.abs().max().item() / gmax
            print(f"ERR {what} d{nm} (vs largest gradient): {e:.3e} (bound {tol:.1e})")
            assert e <= tol, f"{what} d{nm}"
            continue
        _check(gk, p.grad, tol, f"{what} d{nm}")
    for i, (mod, nm) in enumerate(((m.double_conv[1], "bn0"), (m.double_conv[4], "bn1"))):
        _check(mod.running_mean, bufs[2 * i], tol, f"{what} {nm}.running_mean")
        _check(mod.running_var, bufs[2 * i + 1], tol, f"{what} {nm}.running_var")
