"""-m gpu: the dense networks' serving outputs from the last 3x3 conv's epilogue.  smaat_conv3x3_classify_fwd /
smaat_conv3x3_probs_fwd bit for bit against the unfused route they replace (smaat_conv3x3_fwd -> smaat_outconv_fwd [->
smaat_argmax_channels_fwd / smaat_softmax_channels_fwd]) at up4's last conv of UNet(12, 1) and UNet(3, 21), partial tiles in
both patch widths, a concat input, Cout < 64, K from 1 to 32 with and without bias, in tf32 and tf32x3; NaN rows and ties;
UNet / UNetAttention (bilinear and transposed) forward_serving / forward_classes / forward_probs against forward; the float64
port; the fallbacks; and InferenceSession end to end."""
import pytest
import torch

import smaat_unet_b200 as S
from oracle import dense_oracle as D
from smaat_unet_b200 import ops
from smaat_unet_b200.engine import InferenceSession
from tests._util import NET_TOL, assert_close

pytestmark = pytest.mark.gpu

FUSED = ("smaat_conv3x3_classify_fwd", "smaat_conv3x3_probs_fwd")


def _bits_equal(a, b):
    """Bitwise equality (NaN payloads and the sign of zero included)."""
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


@pytest.fixture
def mode_guard():
    """The dense serving fusion switched on (it is off by default: slower on an H100, same bits), the mode restored after."""
    old = ops.get_pointwise_mode()
    ops.set_fused_dense_head(True)
    yield
    ops.set_pointwise_mode(old)
    ops.set_fused_classify(True)
    ops.set_fused_dense_head(False)


def _layer(C0, C1, Cout, K, H, W, B, bias, seed, oc_scale=0.3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C0, H, W, generator=g).cuda()
    x1 = torch.randn(B, C1, H, W, generator=g).cuda() if C1 else None
    w = (torch.randn(Cout, C0 + C1, 3, 3, generator=g) * (2.0 / (9 * (C0 + C1))) ** 0.5).cuda()
    sc = (torch.rand(Cout, generator=g) + 0.5).cuda()
    sh = (torch.randn(Cout, generator=g) * 0.1).cuda()
    ow = (torch.randn(K, Cout, generator=g) * oc_scale).cuda()
    ob = (torch.randn(K, generator=g) * 0.1).cuda() if bias else None
    return x, x1, w, sc, sh, ow, ob


def _routes(x, x1, w, sc, sh, ow, ob, mode):
    """(unfused logits, class map, probabilities), (fused logits-only, classes-only, (classes, logits), probabilities)."""
    C0, C1, Cout = x.shape[1], (x1.shape[1] if x1 is not None else 0), w.shape[0]
    wp = ops.conv3x3_pack_weight(w, C0, C1)
    split = ops.split_tf32(wp) if mode == "tf32x3" else None
    y = ops.conv3x3(x, wp, Cout, sc, sh, True, x1=x1, mode=mode, w_split=split)
    lg = ops.outconv(y, ow, ob)
    ref = (lg, ops.argmax_channels(lg), ops.softmax_channels(lg))
    args = (x, wp, Cout, sc, sh, True, ow, ob)
    kw = dict(x1=x1, mode=mode, w_split=split)
    got = (ops.conv3x3_classify(*args, **kw, want_logits=True, want_classes=False), ops.conv3x3_classify(*args, **kw),
           ops.conv3x3_classify(*args, **kw, want_logits=True), ops.conv3x3_probs(*args, **kw))
    return ref, got


def _check_routes(ref, got, what):
    lg, cls, pr = ref
    lo, co, (cb, lb), po = got
    assert _bits_equal(lo, lg), f"{what}: logits"
    assert _bits_equal(lb, lg), f"{what}: logits written beside the class map"
    assert co.dtype == torch.int64 and torch.equal(co, cls) and torch.equal(cb, cls), f"{what}: class map"
    assert _bits_equal(po, pr), f"{what}: probabilities"


# (name, C0, C1, Cout, K, H, W, B)
LAYERS = [
    ("UNet(12,1) up4.1 288", 64, 0, 64, 1, 288, 288, 2),
    ("UNet(3,21) up4.1 224", 64, 0, 64, 21, 224, 224, 2),
    ("PW16 partial 40x36", 64, 0, 64, 8, 40, 36, 3),          # c3_pick_pw: 16; the last column of patches is partial
    ("PW32 partial 38x52", 64, 0, 64, 2, 38, 52, 2),          # PW 32, partial in both directions
    ("concat [64|64] 40x36", 64, 64, 64, 32, 40, 36, 2),      # up4's first conv's input form, Cout 64
    ("Cout 40 20x20", 48, 0, 40, 8, 20, 20, 2),               # channels past Cout in the staged tile
]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("layer", LAYERS, ids=[c[0] for c in LAYERS])
def test_fused_outputs_equal_the_unfused_route_bit_for_bit(layer, bias, mode):
    name, C0, C1, Cout, K, H, W, B = layer
    t = _layer(C0, C1, Cout, K, H, W, B, bias, seed=K + H + C1)
    assert ops.conv3x3_classify_takes(t[0], t[1], ops.conv3x3_pack_weight(t[2], C0, C1), Cout, K, mode)
    ref, got = _routes(*t, mode)
    _check_routes(ref, got, f"{name} {mode} bias={bias}")
    if K > 1:
        assert int(torch.unique(ref[1]).numel()) > 1, "the class map should not be constant"


def test_nan_row_wins_everywhere_and_ties_go_to_the_first_index():
    x, x1, w, sc, sh, ow, ob = _layer(64, 0, 64, 8, 40, 36, 2, True, seed=3)
    ow_nan = ow.clone()
    ow_nan[5, 7] = float("nan")
    ref, got = _routes(x, x1, w, sc, sh, ow_nan, ob, "tf32x3")
    _check_routes(ref, got, "NaN weight row")
    assert bool((got[1] == 5).all()), "a NaN logit must win at every pixel"
    p = got[3]
    assert bool(torch.isnan(p).all()), "every probability of a pixel with a NaN logit is NaN"
    assert torch.equal(torch.isnan(p), torch.isnan(torch.softmax(ref[0], 1)))
    # classes 2 and 6 share a row and a bias that dominate the others: equal logits, the first index wins
    ow_tie, ob_tie = ow.clone(), ob.clone()
    ow_tie[2] = ow[2].abs() + 1.0
    ow_tie[6] = ow_tie[2]
    ob_tie[6] = ob_tie[2]
    ref, got = _routes(x, x1, w, sc, sh, ow_tie, ob_tie, "tf32")
    _check_routes(ref, got, "tied rows")
    assert _bits_equal(got[0][:, 2], got[0][:, 6])
    assert bool((got[1] != 6).all()) and int((got[1] == 2).sum()) > 0


def _spread(m):
    with torch.no_grad():                 # a freshly initialised OutConv lets its bias pick one class everywhere
        m.outc.conv.weight.mul_(50.0)
    return m


MODELS = [(S.UNet, True), (S.UNet, False), (S.UNetAttention, True), (S.UNetAttention, False)]


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("arch", MODELS, ids=[f"{c.__name__}-{'bilinear' if b else 'transposed'}" for c, b in MODELS])
def test_model_serving_outputs_equal_forward(arch, mode, mode_guard):
    ops.set_pointwise_mode(mode)
    cls, bilinear = arch
    torch.manual_seed(11)
    m = _spread(cls(3, 21, bilinear)).cuda().eval()
    x = torch.rand(2, 3, 64, 64, device="cuda")
    with torch.no_grad():
        lg = m(x)
        with ops.profile() as prof:
            ys, cs, ps = m.forward_serving(x), m.forward_classes(x), m.forward_probs(x)
    names = prof.summary()
    assert names["smaat_conv3x3_classify_fwd"]["launches"] == 2 and names["smaat_conv3x3_probs_fwd"]["launches"] == 1
    assert not any(k in names for k in ("smaat_outconv_fwd", "smaat_argmax_channels_fwd", "smaat_softmax_channels_fwd"))
    assert _bits_equal(ys, lg)
    assert torch.equal(cs, ops.argmax_channels(lg)) and torch.equal(cs, torch.argmax(lg, 1))
    assert _bits_equal(ps, ops.softmax_channels(lg))
    assert int(torch.unique(cs).numel()) > 1


def test_model_serving_against_the_float64_port(mode_guard):
    ops.set_pointwise_mode("tf32x3")
    torch.manual_seed(2)
    m = S.UNet(12, 1).cuda().eval()
    x = torch.rand(2, 12, 96, 96, device="cuda")
    with torch.no_grad():
        y = m.forward_serving(x)
        sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
        yr = D.port_unet_forward(x.cpu().double(), sd)
    assert_close(y, yr.numpy(), NET_TOL["tf32x3"], "UNet(12, 1).forward_serving 96")


def _launches(fn, *a):
    with ops.profile() as prof:
        out = fn(*a)
    return out, prof.summary()


def test_fallbacks_give_todays_results(mode_guard):
    torch.manual_seed(5)
    x = torch.rand(2, 3, 64, 64, device="cuda")
    # fp32: the exact CUDA-core conv, then OutConv and the argmax / softmax kernels
    ops.set_pointwise_mode("fp32")
    m = _spread(S.UNet(3, 21)).cuda().eval()
    with torch.no_grad():
        lg = m(x)
        for fn, want in ((m.forward_serving, lg), (m.forward_classes, ops.argmax_channels(lg)), (m.forward_probs, ops.softmax_channels(lg))):
            got, names = _launches(fn, x)
            assert _bits_equal(got, want) and not any(k in names for k in FUSED)
    ops.set_pointwise_mode("tf32x3")
    # 33 classes: more than the epilogue keeps
    m33 = _spread(S.UNet(3, 33)).cuda().eval()
    with torch.no_grad():
        lg = m33(x)
        got, names = _launches(m33.forward_classes, x)
        assert torch.equal(got, ops.argmax_channels(lg)) and not any(k in names for k in FUSED)
        got, names = _launches(m33.forward_probs, x)
        assert _bits_equal(got, ops.softmax_channels(lg)) and not any(k in names for k in FUSED)
    # an 18-wide layer (W % 4 != 0): the CUDA-core conv, OutConv apart
    dc, oc = S.DoubleConv(64, 64).cuda().eval(), S.OutConv(64, 8).cuda().eval()
    z = torch.rand(2, 64, 18, 18, device="cuda")
    with torch.no_grad():
        want = oc(dc.run(z))
        got, names = _launches(dc.run, z, None, oc)
        assert _bits_equal(got, want) and not any(k in names for k in FUSED)
        got, names = _launches(lambda: dc.run(z, outconv=oc, head="classes"))
        assert torch.equal(got, ops.argmax_channels(want)) and not any(k in names for k in FUSED)
    # set_fused_classify(False): the separate launches, the same bits
    ops.set_fused_classify(False)
    with torch.no_grad():
        lg = m(x)
        got, names = _launches(m.forward_probs, x)
        assert _bits_equal(got, ops.softmax_channels(lg)) and not any(k in names for k in FUSED)
    ops.set_fused_classify(True)
    # autograd: the plain, differentiable calls
    xg = x.clone().requires_grad_()
    y, names = _launches(m.forward_serving, xg)
    assert y.requires_grad and not any(k in names for k in FUSED)
    y.sum().backward()
    assert xg.grad is not None and torch.isfinite(xg.grad).all()
    with torch.no_grad():
        assert_close(y.detach(), m(x).double().cpu().numpy(), NET_TOL["tf32x3"], "forward_serving under autograd")
    # train mode: batch statistics, no fused epilogue
    m.train()
    with torch.no_grad():
        got, names = _launches(m.forward_classes, x)
    assert got.dtype == torch.int64 and got.shape == (2, 64, 64) and not any(k in names for k in FUSED)


@pytest.mark.parametrize("output", ["logits", "classes", "probs"])
def test_inference_session_serves_the_fused_route(output, mode_guard):
    torch.manual_seed(7)
    m = _spread(S.UNet(3, 21)).cuda().eval()
    B, HW = 2, 64
    fused = InferenceSession(m, B, (3, HW, HW), output=output)
    plain = InferenceSession(m, B, (3, HW, HW), output=output, serving_fusions=False)
    assert plain.launches_per_forward - fused.launches_per_forward == (1 if output == "logits" else 2)
    fwd = {"logits": m.forward_serving, "classes": m.forward_classes, "probs": m.forward_probs}[output]
    for i in range(2):
        x = torch.rand(B, 3, HW, HW, device="cuda")
        got = fused.forward(x).clone()
        want = plain.forward(x).clone()
        with torch.no_grad():
            eager = fwd(x)
        assert _bits_equal(got, eager), f"{output}: the graph replay differs from the eager forward"
        assert _bits_equal(got, want), f"{output}: the fused session differs from the unfused one"
    host = x.cpu().pin_memory()
    fused.submit(host)
    assert _bits_equal(fused.collect().clone(), got.cpu())


def test_the_separate_launches_are_the_default_route():
    assert not ops.fused_dense_head()
    torch.manual_seed(9)
    m = _spread(S.UNetAttention(3, 21)).cuda().eval()
    x = torch.rand(2, 3, 64, 64, device="cuda")
    with torch.no_grad():
        lg = m(x)
        got, names = _launches(m.forward_classes, x)
    assert torch.equal(got, ops.argmax_channels(lg)) and not any(k in names for k in FUSED)
    s_default = InferenceSession(m, 2, (3, 64, 64), output="probs")
    s_plain = InferenceSession(m, 2, (3, 64, 64), output="probs", serving_fusions=False)
    assert s_default.launches_per_forward == s_plain.launches_per_forward
