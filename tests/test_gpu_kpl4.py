"""-m gpu: SmaAt-UNet with kernels_per_layer = 4 on the H100 path.

The fused DS conv's k = 4 instances (dsconv_kpl4_kernel: 8 input channels per chunk, two producer threads per task) at every
DS conv shape of SmaAt_UNet(12, 1, kernels_per_layer=4) at 288 x 288 and at the edges (a partly filled last chunk, partial
tiles, Cout from 8 to 512, batch statistics); their epilogues (1-class OutConv, K-class maps and logits, the CBAM gate on
load and the epilogue pools); the depthwise kernels at k = 4 (TMA, LDG and small-plane forward, TMA and tiled backward); the
whole network against the float64 port, InferenceSession against the eager serving forwards, the launch route against k = 2,
and training.  References are float64 on the CPU; tolerances are relative to max|reference| (PW_TOL / NET_TOL)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from smaat_unet_b200 import ops
from tests._util import NET_TOL, PW_TOL, assert_close, load_np_state_dict

pytestmark = pytest.mark.gpu

K4 = 4
MODES = ["tf32", "tf32x3"]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _conv_params(Cin, Cout, g, k=K4):
    K = k * Cin
    return dict(dw_w=torch.randn(K, 1, 3, 3, generator=g) / 3, dw_b=torch.randn(K, generator=g) * 0.1,
                pw=torch.randn(Cout, K, generator=g) * K ** -0.5, scale=torch.rand(Cout, generator=g) + 0.5,
                shift=torch.randn(Cout, generator=g) * 0.2)


def _cuda(prm):
    return {n: t.cuda() for n, t in prm.items()}


def _dw64(x, w, b, k=K4):
    x = x.double()
    return F.conv2d(x, w.double(), None if b is None else b.double(), padding=1, groups=x.shape[1])


def _ref64(x, prm, relu=True, affine=True, k=K4):
    """float64 DS conv (depthwise, pointwise) + affine (+ ReLU) on the CPU: (activation, raw pointwise output)."""
    z = torch.einsum("bkhw,ok->bohw", _dw64(x, prm["dw_w"], prm["dw_b"], k), prm["pw"].double())
    if not affine:
        return z, z
    y = z * prm["scale"].double().view(1, -1, 1, 1) + prm["shift"].double().view(1, -1, 1, 1)
    return (torch.relu(y) if relu else y), z


def _tol(mode, K):
    """PW_TOL, set for K = k Cin <= 2048 (k <= 2), grown like the fp32 rounding of a K-term sum beyond that (K = 4096: up1.0)"""
    return PW_TOL[mode] * max(1.0, (K / 2048) ** 0.5)


def _split(x, C0):
    return (x[:, :C0].contiguous().cuda(), x[:, C0:].contiguous().cuda() if x.shape[1] > C0 else None)


# ================================================================================================ every DS conv of the network
# (name, C0, C1, Cout, S) of SmaAt_UNet(12, 1, kernels_per_layer=4) at 288 x 288; Up's first conv reads [skip | upsampled]
NET_LAYERS = [
    ("inc.0", 12, 0, 64, 288), ("inc.1", 64, 0, 64, 288),
    ("down1.0", 64, 0, 128, 144), ("down1.1", 128, 0, 128, 144),
    ("down2.0", 128, 0, 256, 72), ("down2.1", 256, 0, 256, 72),
    ("down3.0", 256, 0, 512, 36), ("down3.1", 512, 0, 512, 36),
    ("down4.0", 512, 0, 512, 18), ("down4.1", 512, 0, 512, 18),
    ("up1.0", 512, 512, 512, 36), ("up1.1", 512, 0, 256, 36),
    ("up2.0", 256, 256, 256, 72), ("up2.1", 256, 0, 128, 72),
    ("up3.0", 128, 128, 128, 144), ("up3.1", 128, 0, 64, 144),
    ("up4.0", 64, 64, 64, 288), ("up4.1", 64, 0, 64, 288),
]


def _run_layer(x, C0, prm, mode, Cout, stats=False, like_k2=False):
    """The fused conv where it takes the shape (``like_k2``: with the same decision as k = 2), else dw3x3 + pw1x1.
    (y, stats or None, fused)"""
    x0, x1 = _split(x, C0)
    p = _cuda(prm)
    fused = ops.dsconv_takes(x0, x1, p["pw"], K4, mode=mode, stats=stats)
    if like_k2:
        pw2 = torch.empty(Cout, 2 * (x.shape[1]), device="cuda")
        assert fused == ops.dsconv_takes(x0, x1, pw2, 2, mode=mode, stats=stats), "k = 4 and k = 2 are routed alike"
    if fused:
        st = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda") if stats else None
        y = ops.dsconv(x0, p["dw_w"], p["dw_b"], K4, p["pw"], None if stats else p["scale"], None if stats else p["shift"], not stats,
                       x1=x1, mode=mode, stats=st)
        assert y is not None
        return y, st, True
    d = ops.dw3x3(x0, p["dw_w"], p["dw_b"], K4, x1=x1)
    return ops.pw1x1(d, p["pw"], p["scale"], p["shift"], True, mode=mode), None, False


@pytest.mark.parametrize("layer", NET_LAYERS, ids=[n for n, *_ in NET_LAYERS])
def test_every_network_conv_against_float64(layer):
    name, C0, C1, Cout, S_ = layer
    g = _gen(sum(map(ord, name)))
    x = torch.randn(2, C0 + C1, S_, S_, generator=g)
    if name != "inc.0":
        x = torch.relu(x)
    prm = _conv_params(C0 + C1, Cout, g)
    ref, _ = _ref64(x, prm)
    for mode in MODES:
        y, _, fused = _run_layer(x, C0, prm, mode, Cout, like_k2=True)
        assert fused == (S_ % 4 == 0 and S_ not in (36,)), f"{name}: fused = {fused}"
        assert_close(y, ref.numpy(), _tol(mode, 4 * (C0 + C1)), f"{name} k=4 {mode} ({'fused' if fused else 'dw3x3 + pw1x1'})")


# (name, B, C0, C1, H, W, Cout)
EDGES = [
    ("Cin3", 2, 3, 0, 64, 64, 64),           # one chunk, 3 of its 8 channels real
    ("Cin12", 2, 12, 0, 96, 96, 64),         # two chunks, the second half filled
    ("concat8_8", 2, 8, 8, 64, 64, 64),      # smallest concat: C0 % 8 == 0
    ("H20_W44", 2, 16, 0, 20, 44, 64),       # PW 16, partial tiles in both directions
    ("H99_W96", 2, 16, 8, 99, 96, 64),       # PW 32, odd H
    ("H70_W100", 1, 24, 0, 70, 100, 96),     # PW 16, partial tiles, N_TILE 128
    ("Cout8", 2, 16, 0, 64, 64, 8),
    ("Cout65", 2, 16, 0, 64, 64, 65),
    ("Cout128", 2, 16, 16, 64, 64, 128),
    ("Cout256", 1, 32, 0, 64, 64, 256),
    ("Cout512", 1, 32, 32, 32, 32, 512),
]


@pytest.mark.parametrize("case", EDGES, ids=[c[0] for c in EDGES])
def test_fused_edges_against_float64(case):
    name, B, C0, C1, H, W, Cout = case
    g = _gen(sum(map(ord, name)) + 1)
    x = torch.randn(B, C0 + C1, H, W, generator=g)
    prm = _conv_params(C0 + C1, Cout, g)
    ref, z = _ref64(x, prm)
    for mode in MODES:
        y, _, fused = _run_layer(x, C0, prm, mode, Cout)
        assert fused, f"{name}: not fused"
        assert_close(y, ref.numpy(), PW_TOL[mode], f"{name} {mode}")
        if Cout <= 128:
            y2, st, fused = _run_layer(x, C0, prm, mode, Cout, stats=True)
            assert fused
            assert_close(y2, z.numpy(), PW_TOL[mode], f"{name} {mode} (raw output with statistics)")
            s1, s2 = z.sum((0, 2, 3)), (z * z).sum((0, 2, 3))
            tol = 10 * PW_TOL[mode]
            assert float((st[:Cout].cpu() - s1).abs().max()) <= tol * float(z.abs().sum((0, 2, 3)).max()), f"{name} {mode}: sums"
            assert float((st[Cout:].cpu() - s2).abs().max()) <= tol * float(s2.max()), f"{name} {mode}: sums of squares"


def test_k4_routes_like_k2_and_the_smem_form_keeps_k4_unfused():
    x = torch.zeros(2, 64, 64, 64, device="cuda")
    pw4, pw2 = torch.zeros(64, 4 * 64, device="cuda"), torch.zeros(64, 2 * 64, device="cuda")
    assert ops.dsconv_takes(x, None, pw4, 4) and ops.dsconv_takes(x, None, pw2, 2)
    assert not ops.dsconv_takes(x, None, torch.zeros(64, 3 * 64, device="cuda"), 3)
    ops.set_dsconv_impl("smem")
    try:
        assert not ops.dsconv_takes(x, None, pw4, 4) and ops.dsconv_takes(x, None, pw2, 2)
    finally:
        ops.set_dsconv_impl("auto")
    ops.set_dsconv_impl("regs")
    try:
        assert ops.dsconv_takes(x, None, pw4, 4)
    finally:
        ops.set_dsconv_impl("auto")


# ============================================================================================================== epilogues
def _head_layer(seed, B=2, C0=64, C1=0, H=96, W=96, Cout=64):
    g = _gen(seed)
    x = torch.relu(torch.randn(B, C0 + C1, H, W, generator=g))
    return x, _conv_params(C0 + C1, Cout, g), g


@pytest.mark.parametrize("mode", MODES)
def test_outconv_epilogue_against_float64(mode):
    x, prm, g = _head_layer(11)
    ow, ob = torch.randn(1, 64, generator=g) * 0.2, torch.randn(1, generator=g)
    ref = torch.einsum("bchw,c->bhw", _ref64(x, prm)[0], ow[0].double())[:, None] + float(ob)
    p = _cuda(prm)
    y = ops.dsconv(x.cuda(), p["dw_w"], p["dw_b"], K4, p["pw"], p["scale"], p["shift"], True, mode=mode,
                   outconv=(ow.cuda(), ob.cuda()))
    assert y is not None and y.shape == (2, 1, 96, 96)
    assert_close(y, ref.numpy(), PW_TOL[mode], f"outconv {mode}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("K", [8, 21])
@pytest.mark.parametrize("cout", [64, 128])
def test_class_maps_and_probabilities_against_float64(cout, K, mode):
    x, prm, g = _head_layer(20 + K + cout, C0=32, C1=32, H=70, W=100, Cout=cout)
    ow, ob = torch.randn(K, cout, generator=g) * (4.0 / cout ** 0.5), torch.randn(K, generator=g) * 0.1
    lg64 = torch.einsum("bchw,kc->bkhw", _ref64(x, prm)[0], ow.double()) + ob.double().view(1, -1, 1, 1)
    p = _cuda(prm)
    x0, x1 = _split(x, 32)
    args = (x0, p["dw_w"], p["dw_b"], K4, p["pw"], p["scale"], p["shift"], True, ow.cuda(), ob.cuda())
    assert ops.dsconv_classify_takes(x0, x1, p["pw"], K4, K, mode)
    cls, lg = ops.dsconv_classify(*args, x1=x1, mode=mode, want_logits=True)
    assert_close(lg, lg64.numpy(), PW_TOL[mode], f"logits K={K} Cout={cout} {mode}")
    top2 = lg64.topk(2, dim=1).values
    near = (top2[:, 0] - top2[:, 1]) <= 4 * PW_TOL[mode] * float(lg64.abs().max())
    diff = cls.cpu() != lg64.argmax(1)
    assert int((diff & ~near).sum()) == 0, f"{int((diff & ~near).sum())} classes differ away from a tie"


# (name, B, C0, C1, H, W, Cout)
GATE_CASES = [("up4.0", 2, 64, 64, 288, 288, 64), ("up3.0", 2, 128, 128, 144, 144, 128), ("up2.0", 2, 256, 256, 72, 72, 256),
              ("H70_W100", 2, 32, 16, 70, 100, 96)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", GATE_CASES, ids=[c[0] for c in GATE_CASES])
def test_cbam_gate_on_load_is_the_conv_on_the_materialised_output_bit_for_bit(case, mode):
    name, B, C0, C1, H, W, Cout = case
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    x0 = torch.relu(torch.randn(B, C0, H, W, generator=g, device="cuda"))
    x1 = torch.randn(B, C1, H, W, generator=g, device="cuda") if C1 else None
    sc = torch.rand(B, C0, generator=g, device="cuda")
    sa = torch.rand(B, 1, H, W, generator=g, device="cuda")
    p = _cuda(_conv_params(C0 + C1, Cout, _gen(3)))
    args = (p["dw_w"], p["dw_b"], K4, p["pw"], p["scale"], p["shift"], True)
    assert ops.dsconv_cbam_takes(x0, x1, p["pw"], K4, gate=True, mode=mode)
    y = ops.dsconv_cbam(x0, *args, x1=x1, mode=mode, gate=(sc, sa))
    mat = ops.dsconv(ops.cbam_scale(x0, sc, sa), *args, x1=x1, mode=mode)
    assert torch.equal(y, mat), f"gate {name} {mode}"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", [(64, 64, 288), (128, 128, 144), (256, 256, 72)])
def test_epilogue_pools_are_the_pools_of_the_output(shape, mode):
    Cin, Cout, S_ = shape
    x = torch.relu(torch.randn(2, Cin, S_, S_, device="cuda"))
    p = _cuda(_conv_params(Cin, Cout, _gen(Cin)))
    args = (p["dw_w"], p["dw_b"], K4, p["pw"], p["scale"], p["shift"], True)
    if not ops.dsconv_cbam_takes(x, None, p["pw"], K4, pools=True, mode=mode):
        pytest.skip("this instance keeps the direct-store epilogue")
    y, psum, pmax, pooled = ops.dsconv_cbam(x, *args, mode=mode, pools=True)
    assert torch.equal(y, ops.dsconv(x, *args, mode=mode))
    assert torch.equal(pooled, F.max_pool2d(y, 2))
    assert torch.equal(pmax.amax(1), y.amax((2, 3)))
    assert_close(psum.double().sum(1), y.double().sum((2, 3)).cpu().numpy(), 1e-5, "channel sums")


# ======================================================================================================= depthwise kernels
# (B, C0, C1, H, W): the network's depthwise planes and a small-plane / odd case
DW_CASES = [(2, 12, 0, 288, 288), (2, 64, 64, 288, 288), (2, 128, 0, 144, 144), (2, 256, 256, 72, 72), (2, 512, 0, 36, 36),
            (2, 512, 0, 18, 18), (2, 5, 3, 20, 17)]


@pytest.mark.parametrize("pro", [False, True])
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: f"C{c[1]}+{c[2]}_{c[3]}x{c[4]}")
def test_dw3x3_k4_loaders_against_float64(case, pro):
    B, C0, C1, H, W = case
    g = _gen(H * 7 + C0 + C1)
    Cin = C0 + C1
    x = torch.randn(B, Cin, H, W, generator=g)
    w, b = torch.randn(4 * Cin, 1, 3, 3, generator=g), torch.randn(4 * Cin, generator=g)
    sc, sh = torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3
    xin = torch.relu(x.double() * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)) if pro else x
    ref = _dw64(xin, w, b).numpy()
    x0, x1 = _split(x, C0)
    loaders = [1, 2] if W % 4 == 0 else [0, 1]      # W % 4 != 0: auto = the small-plane kernel (18 x 18) or LDG
    for loader in loaders:
        y = ops.dw3x3(x0, w.cuda(), b.cuda(), 4, x1=x1, in_scale=sc.cuda() if pro else None, in_shift=sh.cuda() if pro else None,
                      loader=loader)
        assert_close(y, ref, 2e-6, f"dw3x3 k=4 {case} loader={loader} pro={pro}")


@pytest.mark.parametrize("case", [(1, 64, 0, 288, 288), (1, 64, 64, 288, 288), (2, 128, 0, 144, 144), (2, 256, 0, 72, 72),
                                  (2, 512, 0, 36, 36), (2, 512, 0, 18, 18), (2, 4, 4, 20, 44), (2, 3, 0, 20, 17),
                                  (2, 64, 0, 32, 32)],     # 32 x 32: the weight kernel runs one warp for 40 sums
                         ids=lambda c: f"C{c[1]}+{c[2]}_{c[3]}x{c[4]}")
@pytest.mark.parametrize("pro", [False, True])
def test_dw3x3_backward_k4_against_float64_autograd(case, pro):
    from smaat_unet_b200 import functional as Fn
    B, C0, C1, H, W = case
    g = _gen(B * 1000 + H * 10 + W + C1)
    Cin = C0 + C1
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(4 * Cin, 1, 3, 3, generator=g, dtype=torch.float64)
    dd = torch.randn(B, 4 * Cin, H, W, generator=g, dtype=torch.float64)
    sc = torch.rand(Cin, generator=g, dtype=torch.float64) + 0.5
    sh = torch.randn(Cin, generator=g, dtype=torch.float64) * 0.3
    inp = (torch.relu(x * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)) if pro else x).requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    bb = torch.zeros(4 * Cin, dtype=torch.float64, requires_grad=True)
    F.conv2d(inp, wr, bb, padding=1, groups=Cin).backward(dd)
    f32 = lambda t: t.to(torch.float32).cuda().contiguous()
    x0 = f32(x[:, :C0])
    x1 = f32(x[:, C0:]) if C1 else None
    dW = torch.zeros(4 * Cin, 1, 3, 3, device="cuda")
    db = torch.zeros(4 * Cin, device="cuda")
    dx0, dx1 = Fn.dw_bwd(f32(dd), f32(w), x0, x1, f32(sc) if pro else None, f32(sh) if pro else None, 4, dW, db)
    assert_close(torch.cat([dx0, dx1], 1) if C1 else dx0, inp.grad.numpy(), 2e-5, f"dw3x3_bwd_input k=4 {case}")
    assert_close(dW, wr.grad.numpy(), 1e-4, f"dw3x3_bwd_weight k=4 {case}")
    assert_close(db, bb.grad.numpy(), 1e-4, f"dw3x3_bwd_bias k=4 {case}")


# ========================================================================================================== whole network
def _net(n_ch=12, K=1, k=K4, seed=5):
    sd = cast_sd(fill_schema(smaat_unet_schema(n_ch, K, k), seed), np.float32)
    m = load_np_state_dict(S.SmaAt_UNet(n_ch, K, kernels_per_layer=k), sd).cuda().eval()
    return m, sd


@pytest.mark.parametrize("mode", MODES)
def test_network_eval_against_float64_port(mode):
    m, sd = _net()
    x = torch.from_numpy(np.random.default_rng(9).uniform(0, 1, (2, 12, 288, 288)).astype(np.float32))
    with torch.no_grad():
        ref = TP.smaat_unet_forward(x.double(), TP.to_torch_sd(sd, torch.float64))
        S.set_pointwise_mode(mode)
        try:
            y = m(x.cuda())
            ys = m.forward_serving(x.cuda())
        finally:
            S.set_pointwise_mode("tf32x3")
    assert_close(y, ref.numpy(), NET_TOL[mode], f"SmaAt_UNet k=4 {mode}")
    assert_close(ys, ref.numpy(), NET_TOL[mode], f"SmaAt_UNet k=4 forward_serving {mode}")


def _launches(m, x, fn):
    with ops.profile() as prof, torch.no_grad():
        getattr(m, fn)(x)
    return {n: a["launches"] for n, a in prof.summary().items()}


@pytest.mark.parametrize("fn", ["forward", "forward_serving", "forward_classes", "forward_probs"])
def test_k4_launches_are_k2s(fn):
    K = 1 if fn in ("forward", "forward_serving") else 8
    x = torch.rand(2, 12, 288, 288, device="cuda")
    got = {k: _launches(_net(12, K, k)[0], x, fn) for k in (2, 4)}
    assert got[4] == got[2], f"{fn}: k = 4 {got[4]} vs k = 2 {got[2]}"
    for name in ("smaat_cbam_scale_fwd", "smaat_dw3x3_fwd", "smaat_outconv_fwd"):
        assert got[4].get(name, 0) == got[2].get(name, 0)
    if fn == "forward_serving":
        assert "smaat_dsconv_cbam_fwd" in str(got[4]) or got[4].get("smaat_dsconv_fwd", 0) > 0
        assert "smaat_dsconv_outconv_fwd" in got[4] and "smaat_outconv_fwd" not in got[4]


@pytest.mark.parametrize("output", ["logits", "classes", "probs"])
def test_inference_session_is_the_eager_serving_forward_bit_for_bit(output):
    from smaat_unet_b200.engine import InferenceSession
    K = 1 if output == "logits" else 8
    m, _ = _net(12, K)
    with torch.no_grad():
        m.outc.conv.weight.mul_(20.0)
    sess = InferenceSession(m, 2, (12, 288, 288), output=output)
    eager = {"logits": m.forward_serving, "classes": m.forward_classes, "probs": m.forward_probs}[output]
    for seed in range(2):
        x = torch.rand(2, 12, 288, 288, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
        got = sess.forward(x).clone()
        with torch.no_grad():
            assert torch.equal(got, eager(x)), f"InferenceSession({output}) vs eager, batch {seed}"


# ================================================================================================================ training
def test_train_session_step_against_float64_autograd():
    """One cross-entropy TrainSession step of SmaAt_UNet(3, 21, kernels_per_layer=4): its loss is the float64 port's, and the
    parameters move as one Adam step on the port's float64 gradients moves them: by lr times the gradient's sign.  At B = 2
    the deep BatchNorms normalise over 32 values, so fp32 rounding flips some gradient signs; per parameter, over the entries
    at least 1 % of the largest gradient (biases that feed a train-mode BatchNorm have a zero gradient), the step must agree
    with the float64 signs as often as the port's own float32 gradients do, less 5 %."""
    from smaat_unet_b200.train import TrainSession
    B, K, HW, lr = 2, 21, 64, 1e-3
    m, sd = _net(3, K, seed=7)
    m.train()
    g = torch.Generator().manual_seed(4)
    x = torch.rand(B, 3, HW, HW, generator=g)
    y = torch.randint(0, K, (B, HW, HW), generator=g)
    names = dict(m.named_parameters())
    sd64 = {k: v.clone().requires_grad_(k in names) for k, v in TP.to_torch_sd(sd, torch.float64).items()}
    loss64 = F.cross_entropy(TP.smaat_unet_forward(x.double(), sd64, True), y)
    loss64.backward()
    sd32 = {k: (v.detach().float().requires_grad_(k in names) if v.is_floating_point() else v) for k, v in sd64.items()}
    F.cross_entropy(TP.smaat_unet_forward(x, sd32, True), y).backward()
    before = {k: v.detach().clone() for k, v in m.state_dict().items()}
    sess = TrainSession(m, B, (3, HW, HW), lr=lr, use_graph=False, loss="cross_entropy")
    loss = float(sess.step(x.cuda(), y.cuda()).detach())
    assert abs(loss - float(loss64)) <= 1e-4 * abs(float(loss64)), (loss, float(loss64))
    after = m.state_dict()
    gmax = max(float(p.grad.abs().max()) for p in sd64.values() if p.grad is not None)
    checked = 0
    for k, p in sd64.items():
        if p.grad is None:
            continue
        strong = p.grad.abs() >= 1e-2 * gmax
        if not bool(strong.any()):
            continue
        step = (before[k].double().cpu() - after[k].double().cpu()).view_as(p.grad)
        sign64 = torch.sign(p.grad[strong])
        agree = float((torch.sign(step[strong]) == sign64).double().mean())
        agree32 = float((torch.sign(sd32[k].grad.double()[strong]) == sign64).double().mean())
        assert agree >= agree32 - 0.05, f"{k}: the Adam step has the float64 gradient's sign at {agree:.3f} of its strong entries " \
                                        f"(the float32 port {agree32:.3f})"
        checked += 1
    assert checked >= 20, checked


def _port_grads(sd, x, t, dtype, names):
    sd_t = {k: v.clone().to(dtype).requires_grad_(k in names) if v.is_floating_point() else v.clone()
            for k, v in TP.to_torch_sd(sd, torch.float64).items()}
    (F.mse_loss(TP.smaat_unet_forward(x.to(dtype), sd_t, True).squeeze(1), t.to(dtype), reduction="sum") / x.shape[0]).backward()
    return {k: v.grad.double().numpy() for k, v in sd_t.items() if k in names}


def test_full_size_gradients_against_float64_autograd():
    """B = 2, 12 x 288 x 288, train mode, mse: every parameter's gradient against float64 autograd of the port, within a small
    multiple of the port's own fp32-vs-fp64 movement (as the k = 2 check in test_gpu_api_paths); gradients that are
    mathematically zero (a bias cancelled by BatchNorm's mean subtraction) only within 1e-3 of the largest gradient."""
    m, sd = _net(12, 1, seed=8)
    m.train()
    g = torch.Generator().manual_seed(6)
    x = torch.rand(2, 12, 288, 288, generator=g)
    t = torch.rand(2, 288, 288, generator=g)
    loss = F.mse_loss(m(x.cuda()).squeeze(1), t.cuda(), reduction="sum") / 2
    loss.backward()
    names = dict(m.named_parameters())
    g64 = _port_grads(sd, x, t, torch.float64, names)
    g32 = _port_grads(sd, x, t, torch.float32, names)

    def rel_max(a, b):
        return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))

    def rel_l2(a, b):
        return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    gmax = max(float(np.abs(v).max()) for v in g64.values())
    live = [k for k, v in g64.items() if np.abs(v).max() >= 1e-6 * gmax]
    tol_max = max(2e-3, 5.0 * max(rel_max(g32[k], g64[k]) for k in live))
    tol_l2 = max(1e-3, 5.0 * max(rel_l2(g32[k], g64[k]) for k in live))
    for k, p in names.items():
        got = p.grad.double().cpu().numpy()
        if k not in live:
            assert float(np.abs(got).max()) <= 1e-3 * gmax, k
            continue
        e_max, e_l2 = rel_max(got, g64[k]), rel_l2(got, g64[k])
        assert e_max <= tol_max and e_l2 <= tol_l2, f"grad {k}: rel max {e_max:.3e} (tol {tol_max:.1e}), rel L2 {e_l2:.3e} (tol {tol_l2:.1e})"
    assert len(live) > 50, len(live)
