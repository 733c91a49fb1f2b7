"""SmaAt-UNet's serving forward from bf16 activations (the bf16 storage route) on the GPU.

  A  every new kernel instance against float64 on the same bf16 inputs, within one bf16 ulp of the once-rounded result
     (``_one_ulp``): the bf16-activation fused DS conv at the levels 1-3 layers of the 288 and 224 networks (k = 2, and k = 1
     on three of them; both halves of the virtual concat, the CBAM gate on and off, PW 32 and 16, partial tiles at 72 and 56),
     its one-class OutConv and K-class class map, the CBAM pools + MLP + max-pool (bf16 and fp32 max-pool) and the channel
     reduce, the upsample from fp32 and bf16 maps, and the unfused heads (OutConv, argmax, softmax)
  B  SmaAt_UNet(12, 1) (k = 2, B = 32, 288 x 288) logits and SmaAt_UNet(3, 21) (B = 8, 224 x 224) logits, probabilities and
     class map through InferenceSession(dtype=torch.bfloat16), against the float64 port with the route's roundings emulated
     (``_port_bf16``) and against the unrounded float64 port
  C  the session: forward equals the eager forward_serving bit for bit, submit / collect over several batches, partial
     batches equal the same rows of the full batch, refresh() after a weight change
  D  the requests the route does not take raise before anything is enqueued

One ulp in A: the kernels compute in fp32 what the float64 reference computes, then round once.  The fp32 accumulation adds
an error of at most the fp32 routes' kernel bounds (1.2e-5 of the largest value for the fused DS conv in bf16 mode,
tests/test_gpu_bf16.py), which ``_one_ulp`` allows on top of one ulp (``atol_rel``).
"""
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from smaat_unet_b200 import _lib, ops
from smaat_unet_b200.engine import InferenceSession
from tests.test_gpu_bf16 import _bn_randomise, _port, pw_ref_bf16
from tests.test_gpu_ds_forward_kernels import _check, _exact, _gen, _randn, dw_emul

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
# B: max |err| / max |ref| of the whole networks.  Measured on an H100 80GB HBM3 (700 W): 9.7e-3 / 1.2e-2 (SmaAt_UNet(12, 1)
# against the emulated / the unrounded port), 5.1e-3 / 6.1e-3 (SmaAt_UNet(3, 21) logits), 3.2e-3 (its probabilities against the
# emulated port); the bounds are about 3x those.  The emulation cannot follow a stored value that lands on the other side of
# a bf16 rounding boundary than in float64, so the rounded port is closer than the unrounded one, but not bit-close
NET_BOUND = {
    "smaat_12_1_emul": 3e-2, "smaat_12_1_port": 3.5e-2,
    "smaat_3_21_emul": 1.5e-2, "smaat_3_21_port": 2e-2,
    "smaat_3_21_probs_emul": 1e-2,
}
MIN_CLASS_AGREEMENT = 0.99      # B: share of pixels whose bf16 class map matches the emulated port's argmax


def r16(t):
    """The stored value: round to nearest even in bf16 (as float64)."""
    return t.to(BF).double()


DS_ATOL = 1.5e-5      # the fused DS conv's fp32 accumulation (bf16 mode's bound 1.2e-5)
HEAD_ATOL = 5e-5      # an OutConv over those activations: its logits cancel


def _one_ulp(got, ref, what, atol_rel=2e-6):
    """|got - ref| <= one bf16 ulp of ref + atol_rel * max |ref| at every element (got: bf16, ref: float64)."""
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    mag = ref.abs().clamp_min(1e-30)
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 7)
    err = (got - ref).abs()
    bound = ulp + atol_rel * ref.abs().max()
    worst = float((err / bound).max())
    print(f"ERR {what}: worst |err| / (1 ulp + atol) = {worst:.3f}")
    assert worst <= 1.0, f"{what}: off by more than one bf16 ulp ({worst:.3f})"


# ============================================================================================================ A: the kernels
# (name, C0, C1, Cout, H, gate): levels 1-3 of SmaAt_UNet(12, 1) at 288 and of SmaAt_UNet(3, 21) at 224
DS_LAYERS = [
    ("inc.0", 12, 0, 64, 288, False), ("inc.1", 64, 0, 64, 288, False), ("down1.0", 64, 0, 128, 144, False),
    ("down2.1", 256, 0, 256, 72, False), ("up2.0", 256, 256, 256, 72, True), ("up2.1", 256, 0, 128, 72, False),
    ("up3.0", 128, 128, 128, 144, True), ("up4.0", 64, 64, 64, 288, True),
    ("inc.0_224", 3, 0, 64, 224, False), ("down1.1_112", 128, 0, 128, 112, False), ("up2.0_56", 256, 256, 256, 56, True),
    ("up4.0_224", 64, 64, 64, 224, True),
]
DS_CASES = [(l, 2) for l in DS_LAYERS] + [(l, 1) for l in DS_LAYERS if l[0] in ("inc.1", "up3.0", "up2.0_56")]


def _ds_case(layer, k):
    name, C0, C1, Cout, H, gate = layer
    B = 2 if H >= 224 else 4
    g = _gen(C0 * 131 + C1 * 17 + Cout * 7 + H + k)
    Cin, K = C0 + C1, k * (C0 + C1)
    x = r16(_randn((B, Cin, H, H), g)).float()           # bf16 values, held in fp32 for the reference
    w, b = _randn((K, 1, 3, 3), g, 1.0 / 3.0), _randn((K,), g, 0.1)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = torch.rand((Cout,), generator=g, device="cuda") + 0.5, _randn((Cout,), g, 0.1)
    sc_g = sa_g = None
    if gate:
        sc_g = torch.rand((B, C0), generator=g, device="cuda") + 0.5
        sa_g = torch.rand((B, 1, H, H), generator=g, device="cuda")
    return g, x, w, b, pw, sc, sh, sc_g, sa_g


def _ds_ref(x, w, b, k, pw, sc, sh, C0, sc_g, sa_g, relu=True):
    """float64 of the kernel's arithmetic on the same bf16 x: the gate products and the depthwise in fp32 (dw_emul), bf16 GEMM
    operands, the affine."""
    if sc_g is not None:
        x = x.clone()
        x[:, :C0] = (x[:, :C0] * sc_g.view(*sc_g.shape, 1, 1)) * sa_g
    z = pw_ref_bf16(dw_emul(x, w, b, k), pw) * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)
    return torch.relu(z) if relu else z


@pytest.mark.parametrize("layer,k", DS_CASES, ids=[f"{l[0]}_k{k}" for l, k in DS_CASES])
def test_dsconv_bf16_within_one_ulp(layer, k):
    name, C0, C1, Cout, H, gate = layer
    g, x, w, b, pw, sc, sh, sc_g, sa_g = _ds_case(layer, k)
    x0, x1 = x[:, :C0].to(BF), (x[:, C0:].to(BF) if C1 else None)
    assert ops.dsconv_bf16_takes(x0, x1, pw, k)
    y = ops.dsconv_bf16(x0, w, b, k, pw, sc, sh, True, x1=x1, gate=(sc_g, sa_g) if gate else None)
    assert y.dtype == BF
    _one_ulp(y, _ds_ref(x, w, b, k, pw, sc, sh, C0, sc_g, sa_g), f"dsconv bf16 {name} k={k}", DS_ATOL)
    if gate:          # the same layer without the gate
        y = ops.dsconv_bf16(x0, w, b, k, pw, sc, sh, True, x1=x1)
        _one_ulp(y, _ds_ref(x, w, b, k, pw, sc, sh, C0, None, None), f"dsconv bf16 {name} k={k} no gate", DS_ATOL)


@pytest.mark.parametrize("H", [288, 224])
def test_dsconv_bf16_heads(H):
    """up4.1's heads: the one-class OutConv's bf16 logits, and the 21-class class map = the argmax of the fp32 logits (checked
    against float64 where the top two logits are apart by more than the fp32 accumulation can move them)."""
    layer = ("up4.1", 64, 0, 64, H, False)
    g, x, w, b, pw, sc, sh, _, _ = _ds_case(layer, 2)
    x0 = x.to(BF)
    act = _ds_ref(x, w, b, 2, pw, sc, sh, 64, None, None)
    ow, ob = _randn((1, 64), g, 64 ** -0.5), _randn((1,), g, 0.3)
    lg = ops.dsconv_head_bf16(x0, w, b, 2, pw, sc, sh, True, ow, ob, "logits")
    assert lg.dtype == BF and lg.shape == (x.shape[0], 1, H, H)
    _one_ulp(lg, torch.einsum("c,bchw->bhw", ow.double().view(-1), act).unsqueeze(1) + ob.double(), f"outconv head bf16 S{H}",
             HEAD_ATOL)
    ow21, ob21 = _randn((21, 64), g, 64 ** -0.5), _randn((21,), g, 0.3)
    cls = ops.dsconv_head_bf16(x0, w, b, 2, pw, sc, sh, True, ow21, ob21, "classes")
    ref = torch.einsum("kc,bchw->bkhw", ow21.double(), act) + ob21.double().view(1, -1, 1, 1)
    top2 = ref.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-5 * ref.abs().max()
    _exact(cls[clear], ref.argmax(dim=1)[clear], f"classify head bf16 S{H} (clear pixels)")
    assert float(clear.double().mean()) > 0.99


# (C, H, pooled dtype): the maps levels 1-3 pool, at 288 and 224
POOL_CASES = [(64, 288, BF), (128, 144, BF), (256, 72, torch.float32), (64, 224, BF), (128, 112, BF), (256, 56, torch.float32)]


@pytest.mark.parametrize("C,H,pdt", POOL_CASES, ids=[f"C{c}_S{h}_{str(p)[6:]}" for c, h, p in POOL_CASES])
def test_cbam_pools_maxpool_and_reduce_from_bf16(C, H, pdt):
    B = 4
    g = _gen(C + H)
    xf = r16(_randn((B, C, H, H), g, 1.0, 1.0)).float()     # mean 1: the pools' relative errors are those of their sums
    x = xf.to(BF)
    hid = C // 16
    w1, b1 = _randn((hid, C), g, C ** -0.5), _randn((hid,), g, 0.1)
    w2, b2 = _randn((C, hid), g, hid ** -0.5), _randn((C,), g, 0.1)
    sc, avg, mx, pooled = ops.cbam_pool_mlp(x, w1, b1, w2, b2, with_maxpool=True, pooled_dtype=pdt)
    xd = xf.double()
    _check(avg, xd.mean(dim=(2, 3)), 1e-5, f"pool_mlp bf16 avg C{C} S{H}")
    _exact(mx, xf.amax(dim=(2, 3)), f"pool_mlp bf16 max C{C} S{H}")
    assert pooled.dtype == pdt
    _exact(pooled.float(), F.max_pool2d(xf, 2), f"pool_mlp bf16 max-pool C{C} S{H}")
    mlp = lambda v: F.linear(F.relu(F.linear(v, w1.double(), b1.double())), w2.double(), b2.double())  # noqa: E731
    _check(sc, torch.sigmoid(mlp(avg.double()) + mlp(mx.double())), 1e-5, f"pool_mlp bf16 gate C{C} S{H}")
    avg2, mx2, pooled2 = ops.cbam_pool_maxpool(x, pooled_dtype=pdt)
    _exact(avg2, avg, f"pool_maxpool bf16 avg C{C} S{H}")
    _exact(pooled2, pooled, f"pool_maxpool bf16 max-pool C{C} S{H}")
    red = ops.cbam_reduce(x, sc)
    xs = xd * sc.double().view(B, C, 1, 1)
    _check(red[:, 0], xs.mean(dim=1), 1e-5, f"reduce bf16 mean C{C} S{H}")
    _check(red[:, 1], xs.amax(dim=1), 2e-7, f"reduce bf16 max C{C} S{H}")


@pytest.mark.parametrize("C,H,src", [(512, 36, torch.float32), (256, 72, BF), (128, 144, BF), (512, 28, torch.float32),
                                     (128, 112, BF)])
def test_upsample_to_bf16(C, H, src):
    B = 2
    g = _gen(C * 3 + H)
    xf = _randn((B, C, H, H), g)
    if src == BF:
        xf = r16(xf).float()
    y = ops.upsample2x_pad(xf.to(src), 2 * H, 2 * H, out_dtype=BF)
    assert y.dtype == BF
    # the fp32 kernel's values, rounded once: the same fp32 arithmetic on the same values
    _exact(y, ops.upsample2x_pad(xf, 2 * H, 2 * H).to(BF), f"upsample {str(src)[6:]} -> bf16 C{C} S{H} vs fp32 kernel rounded")
    # against float64: the kernels take the source coordinate dst * (H - 1) / (2 H - 1) in fp32 (as torch's fp32 kernel does),
    # off by up to ~2H * 6e-8 pixels, times a neighbour difference of up to 2 max |x|
    ref = F.interpolate(xf.double(), scale_factor=2, mode="bilinear", align_corners=True)
    _one_ulp(y, ref, f"upsample {str(src)[6:]} -> bf16 C{C} S{H}", atol_rel=4 * H * 6e-8)


@pytest.mark.parametrize("K", [1, 21, 40])
def test_unfused_heads_from_bf16(K):
    B, Cin, H = 2, 64, 224
    g = _gen(K)
    xf = r16(torch.relu(_randn((B, Cin, H, H), g))).float()
    w, b = _randn((K, Cin), g, Cin ** -0.5), _randn((K,), g, 0.3)
    lg = ops.outconv(xf.to(BF), w, b)
    ref = torch.einsum("kc,bchw->bkhw", w.double(), xf.double()) + b.double().view(1, -1, 1, 1)
    _one_ulp(lg, ref, f"outconv bf16 K={K}", HEAD_ATOL)
    _exact(ops.argmax_channels(lg), torch.argmax(lg, dim=1), f"argmax bf16 K={K}")
    pr = ops.softmax_channels(lg)
    assert pr.dtype == BF
    _one_ulp(pr, torch.softmax(lg.double(), dim=1), f"softmax bf16 K={K}")


# ======================================================================================================= B: whole networks
def _ds_port(x, sd, p, bf16_ops):
    """TP.ds_conv, with bf16 GEMM operands (the depthwise result and the pointwise weight) where ``bf16_ops``."""
    if not bf16_ops:
        return TP.ds_conv(x, sd, p)
    d = F.conv2d(x, sd[p + ".depthwise.weight"], sd[p + ".depthwise.bias"], padding=1, groups=x.shape[1])
    return F.conv2d(r16(d), r16(sd[p + ".pointwise.weight"]), sd[p + ".pointwise.bias"])


def _dc_port(x, sd, p, bf16, round_out=True):
    """TP.double_conv_ds with the bf16 route's roundings: bf16 operands, each output stored as bf16 (the last one too unless
    ``round_out`` is False: a head in the epilogue reads it unrounded)."""
    if not bf16:
        return TP.double_conv_ds(x, sd, p)
    y = r16(F.relu(TP._bn(_ds_port(x, sd, p + ".double_conv.0", True), sd, p + ".double_conv.1", False)))
    y = F.relu(TP._bn(_ds_port(y, sd, p + ".double_conv.3", True), sd, p + ".double_conv.4", False))
    return r16(y) if round_out else y


def _up(y, skip, dtype):
    up = F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=True)
    dY, dX = skip.shape[2] - up.shape[2], skip.shape[3] - up.shape[3]
    up = F.pad(up, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])
    return torch.cat([skip, r16(up) if dtype == BF else up], dim=1)


def _port_bf16(x, sd, fused_head):
    """TP.smaat_unet_forward in float64 with the bf16 route's roundings: input, level 1-3 maps and upsampled maps, level 1-3
    GEMM operands, logits.  ``fused_head``: up4's last conv feeds the OutConv unrounded (the epilogue head)."""
    enc = [_dc_port(r16(x), sd, "inc", True)]
    for i in range(1, 5):
        enc.append(_dc_port(F.max_pool2d(enc[-1], 2), sd, f"down{i}.maxpool_conv.1", i < 3))
    att = [TP.cbam(e, sd, f"cbam{i + 1}") for i, e in enumerate(enc)]
    y = TP.up_ds(att[4], att[3], sd, "up1")
    for i in range(2, 5):
        y = _dc_port(_up(y, att[4 - i], BF), sd, f"up{i}.conv", True, round_out=not (i == 4 and fused_head))
    return r16(F.conv2d(y, sd["outc.conv.weight"], sd["outc.conv.bias"]))


def _sd64(model):
    return {k: (v.detach() if v.dtype == torch.int64 else v.detach().double()) for k, v in model.state_dict().items()}


def _chunks(fn, x, n=4):
    with torch.no_grad():
        return torch.cat([fn(x[i:i + n]) for i in range(0, x.shape[0], n)])


def _model(n_ch, n_cls):
    torch.manual_seed(3)
    return _bn_randomise(S.SmaAt_UNet(n_ch, n_cls, kernels_per_layer=2), 4).cuda().eval()


def test_smaat_12_1_logits_against_the_emulated_port():
    B, shape = 32, (12, 288, 288)
    model = _model(12, 1)
    x = torch.rand((B,) + shape, generator=_gen(5), device="cuda").to(BF)
    sess = InferenceSession(model, B, shape, dtype=BF)
    y = sess.forward(x).clone()
    assert y.dtype == BF and sess.static_out.dtype == BF
    with torch.no_grad():
        _exact(y, model.forward_serving(x), "smaat_12_1 bf16 session vs eager serving forward")
    sd = _sd64(model)
    emul = _chunks(lambda v: _port_bf16(v.double(), sd, fused_head=True), x)
    _check(y, emul, NET_BOUND["smaat_12_1_emul"], "smaat_12_1 bf16 logits vs float64 port with the bf16 roundings")
    _check(y, _port(model, x.float()), NET_BOUND["smaat_12_1_port"], "smaat_12_1 bf16 logits vs the unrounded float64 port")


def test_smaat_3_21_logits_probs_and_classes_against_the_emulated_port():
    B, shape = 8, (3, 224, 224)
    model = _model(3, 21)
    x = torch.rand((B,) + shape, generator=_gen(6), device="cuda").to(BF)
    sd = _sd64(model)
    emul = _chunks(lambda v: _port_bf16(v.double(), sd, fused_head=False), x)
    lg = InferenceSession(model, B, shape, dtype=BF).forward(x).clone()
    with torch.no_grad():
        _exact(lg, model.forward_serving(x), "smaat_3_21 bf16 logits session vs eager")
    _check(lg, emul, NET_BOUND["smaat_3_21_emul"], "smaat_3_21 bf16 logits vs float64 port with the bf16 roundings")
    _check(lg, _port(model, x.float()), NET_BOUND["smaat_3_21_port"], "smaat_3_21 bf16 logits vs the unrounded float64 port")
    pr = InferenceSession(model, B, shape, output="probs", dtype=BF).forward(x).clone()
    assert pr.dtype == BF
    _exact(pr, ops.softmax_channels(lg), "smaat_3_21 bf16 probabilities = softmax of the served logits")
    _check(pr, torch.softmax(emul, dim=1), NET_BOUND["smaat_3_21_probs_emul"], "smaat_3_21 bf16 probabilities vs emulated port")
    cls = InferenceSession(model, B, shape, output="classes", dtype=BF).forward(x).clone()
    with torch.no_grad():
        _exact(cls, model.forward_classes(x), "smaat_3_21 bf16 class-map session vs eager")
    agree = float((cls == emul.argmax(dim=1)).double().mean())
    print(f"ERR smaat_3_21 bf16 class map agreement with the emulated port: {agree:.5f}")
    assert agree >= MIN_CLASS_AGREEMENT


# ============================================================================================================= C: the session
def test_session_submit_collect_partial_batches_and_refresh():
    B, shape = 8, (3, 224, 224)
    model = _model(3, 21)
    sess = InferenceSession(model, B, shape, output="probs", dtype=BF, batch_sizes=(3,))
    assert sess.static_in.dtype == BF and sess.h2d_bytes_per_step == B * 3 * 224 * 224 * 2
    assert sess.d2h_bytes_per_step == B * 21 * 224 * 224 * 2
    xs = [torch.rand((B,) + shape, generator=torch.Generator().manual_seed(10 + i)).to(BF).pin_memory() for i in range(3)]
    full = [sess.forward(x.cuda()).clone() for x in xs]
    sess.submit(xs[0])                   # two batches in flight (the session's two staging slots)
    sess.submit(xs[1])
    _exact(sess.collect().cuda(), full[0], "submit / collect batch 0")
    sess.submit(xs[2])
    for i in (1, 2):
        _exact(sess.collect().cuda(), full[i], f"submit / collect batch {i}")
    part = sess.forward(xs[0][:3].cuda()).clone()
    _exact(part, full[0][:3], "3-row request vs the same rows of the full batch")
    sess.submit(xs[1][:2])
    _exact(sess.collect().cuda(), full[1][:2], "2-row submit / collect")
    with pytest.raises(ValueError, match="bfloat16"):
        sess.forward(xs[0].float().cuda())
    with torch.no_grad():        # a cached weight (the bf16 pack) and one the kernels read in place
        model.inc.double_conv[0].pointwise.weight.mul_(1.5)
        model.outc.conv.bias.add_(0.5)
    sess.refresh()
    new = sess.forward(xs[0].cuda()).clone()
    with torch.no_grad():
        _exact(new, model.forward_probs(xs[0].cuda()), "after refresh(): the new weights")
    assert not torch.equal(new, full[0])


# ============================================================================================================ D: rejections
def _raises_before_launch(fn, match):
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match=match):
        fn()
    assert _lib.launch_count() == n0, "a rejected request enqueued kernels"


def test_rejections_raise_before_anything_is_enqueued():
    model = _model(12, 1)
    x = torch.rand((2, 12, 64, 64), device="cuda").to(BF)
    with torch.no_grad():
        _raises_before_launch(lambda: model(x), "forward_serving")
        _raises_before_launch(lambda: model.forward_serving(x[..., :48]), "multiples of 32")
        _raises_before_launch(lambda: S.SmaAt_UNet(12, 1, kernels_per_layer=4).cuda().eval().forward_serving(x), "kernels_per_layer")
        _raises_before_launch(lambda: S.UNet(12, 1).cuda().eval().forward_serving(x), "UNet has no bf16 route")
        _raises_before_launch(lambda: S.UNetAttention(12, 1).cuda().eval().forward_classes(x), "UNetAttention")
        model.train()
        _raises_before_launch(lambda: model.forward_serving(x), "train mode")
        model.eval()
    _raises_before_launch(lambda: model.forward_serving(x), "autograd")     # grad mode on, parameters require grad
    _raises_before_launch(lambda: InferenceSession(S.UNet(12, 1), 2, (12, 64, 64), dtype=BF), "UNet")


def test_a_declined_conv_raises_naming_the_layer():
    model = _model(12, 1)
    x = torch.rand((2, 12, 64, 64), device="cuda").to(BF)
    ops.set_dsconv_impl("smem")          # bf16 has the register A form only
    try:
        with torch.no_grad(), pytest.raises(ValueError, match=r"inc\.double_conv\.0"):
            model.forward_serving(x)
    finally:
        ops.set_dsconv_impl("auto")
    with torch.no_grad():
        assert model.forward_serving(x).dtype == BF
