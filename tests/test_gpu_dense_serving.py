"""-m gpu: the dense networks' serving outputs.  UNet / UNetAttention (bilinear and transposed) forward_serving /
forward_classes / forward_probs bit for bit against forward and the argmax / softmax kernels applied to its logits; the
float64 port; the fallbacks; and InferenceSession end to end."""
import pytest
import torch

import smaat_unet_b200 as S
from oracle import dense_oracle as D
from smaat_unet_b200 import ops
from smaat_unet_b200.engine import InferenceSession
from tests._util import NET_TOL, assert_close

pytestmark = pytest.mark.gpu


def _bits_equal(a, b):
    """Bitwise equality (NaN payloads and the sign of zero included)."""
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


@pytest.fixture
def mode_guard():
    """The pointwise mode and the class-map fusion restored after the test."""
    old = ops.get_pointwise_mode()
    yield
    ops.set_pointwise_mode(old)
    ops.set_fused_classify(True)


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
    assert names["smaat_outconv_fwd"]["launches"] == 3
    assert names["smaat_argmax_channels_fwd"]["launches"] == 1 and names["smaat_softmax_channels_fwd"]["launches"] == 1
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
            assert _bits_equal(got, want) and "smaat_outconv_fwd" in names
    ops.set_pointwise_mode("tf32x3")
    # 33 classes
    m33 = _spread(S.UNet(3, 33)).cuda().eval()
    with torch.no_grad():
        lg = m33(x)
        got, names = _launches(m33.forward_classes, x)
        assert torch.equal(got, ops.argmax_channels(lg)) and "smaat_outconv_fwd" in names
        got, names = _launches(m33.forward_probs, x)
        assert _bits_equal(got, ops.softmax_channels(lg)) and "smaat_outconv_fwd" in names
    # an 18-wide layer (W % 4 != 0): the CUDA-core conv, OutConv apart
    dc, oc = S.DoubleConv(64, 64).cuda().eval(), S.OutConv(64, 8).cuda().eval()
    z = torch.rand(2, 64, 18, 18, device="cuda")
    with torch.no_grad():
        want = oc(dc.run(z))
        got, names = _launches(dc.run, z, None, oc)
        assert _bits_equal(got, want) and "smaat_outconv_fwd" in names
        got, names = _launches(lambda: dc.run(z, outconv=oc, head="classes"))
        assert torch.equal(got, ops.argmax_channels(want)) and "smaat_outconv_fwd" in names
    # set_fused_classify(False): the separate launches, the same bits
    ops.set_fused_classify(False)
    with torch.no_grad():
        lg = m(x)
        got, names = _launches(m.forward_probs, x)
        assert _bits_equal(got, ops.softmax_channels(lg)) and "smaat_outconv_fwd" in names
    ops.set_fused_classify(True)
    # autograd: the plain, differentiable calls
    xg = x.clone().requires_grad_()
    y, names = _launches(m.forward_serving, xg)
    assert y.requires_grad and "smaat_outconv_fwd" in names
    y.sum().backward()
    assert xg.grad is not None and torch.isfinite(xg.grad).all()
    with torch.no_grad():
        assert_close(y.detach(), m(x).double().cpu().numpy(), NET_TOL["tf32x3"], "forward_serving under autograd")
    # train mode: batch statistics
    m.train()
    with torch.no_grad():
        got, names = _launches(m.forward_classes, x)
    assert got.dtype == torch.int64 and got.shape == (2, 64, 64) and "smaat_outconv_fwd" in names


@pytest.mark.parametrize("output", ["logits", "classes", "probs"])
def test_inference_session_equals_the_eager_serving_forward(output, mode_guard):
    torch.manual_seed(7)
    m = _spread(S.UNet(3, 21)).cuda().eval()
    B, HW = 2, 64
    fused = InferenceSession(m, B, (3, HW, HW), output=output)
    plain = InferenceSession(m, B, (3, HW, HW), output=output, serving_fusions=False)
    assert plain.launches_per_forward == fused.launches_per_forward
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
