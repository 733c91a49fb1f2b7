"""-m gpu: class maps from multi-class SmaAt-UNet.  smaat_dsconv_classify_fwd (K-class OutConv + argmax in the last DS conv's
epilogue) against smaat_dsconv_outconv_fwd row by row, bit for bit, at up4's last conv shapes (224 x 224, B = 8; 288 x 288),
its class map against torch.argmax and against a float64 port of the layer; smaat_argmax_channels_fwd against torch.argmax
with ties and NaNs; InferenceSession(output="classes") end to end (forward vs submit / collect, other models, IoU, refresh)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

import smaat_unet_b200 as S
from smaat_unet_b200 import ops
from smaat_unet_b200.engine import InferenceSession
from tests._util import NET_TOL

pytestmark = pytest.mark.gpu

C = 64                                    # up4's last conv: 64 -> 64 channels (UpDS(128, 64): DoubleConvDS(128, 64, 64))
SHAPES = [(8, 224, 224), (2, 288, 288)]   # B, H, W


@pytest.fixture(params=["smem", "regs"])
def ds_impl(request):
    ops.set_dsconv_impl(request.param)
    yield request.param
    ops.set_dsconv_impl("auto")


def _layer(B, H, W, k, seed, cout=C):
    g = torch.Generator().manual_seed(seed)

    def u(*shape, lo=-1.0, hi=1.0):
        return (torch.rand(shape, generator=g) * (hi - lo) + lo).cuda()

    return dict(x=u(B, C, H, W, lo=0.0), dw_w=u(k * C, 1, 3, 3, lo=-0.5, hi=0.5), dw_b=u(k * C, lo=-0.1, hi=0.1),
                pw_w=u(cout, k * C, 1, 1, lo=-0.15, hi=0.15), scale=u(cout, lo=0.5, hi=1.5), shift=u(cout, lo=-0.2, hi=0.2), k=k, g=g,
                cout=cout)


def _classify(L, ow, ob, mode, want_logits=True):
    r = ops.dsconv_classify(L["x"], L["dw_w"], L["dw_b"], L["k"], L["pw_w"], L["scale"], L["shift"], True, ow, ob, mode=mode,
                            want_logits=want_logits)
    assert r is not None, "the fused class epilogue refused up4's last conv"
    return r


def _one_class(L, w_row, b_row, mode):
    return ops.dsconv(L["x"], L["dw_w"], L["dw_b"], L["k"], L["pw_w"], L["scale"], L["shift"], True, mode=mode,
                      outconv=(w_row.contiguous(), b_row))


def _oc(L, K):
    g = L["g"]
    return (torch.rand(K, L["cout"], generator=g) * 0.4 - 0.2).cuda(), (torch.rand(K, generator=g) * 0.2 - 0.1).cuda()


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("shape", SHAPES)
def test_classify_logits_are_the_one_class_kernels_bit_for_bit(shape, k, mode, ds_impl):
    B, H, W = shape
    L = _layer(B, H, W, k, seed=H + 10 * k)
    for K in (2, 8, 21, 32):
        ow, ob = _oc(L, K)
        for bias in (ob, None) if K == 8 else (ob,):
            cls, lg = _classify(L, ow, bias, mode)
            assert cls.dtype == torch.int64 and tuple(cls.shape) == (B, H, W) and tuple(lg.shape) == (B, K, H, W)
            for j in range(K):
                one = _one_class(L, ow[j], None if bias is None else bias[j:j + 1], mode)
                assert torch.equal(lg[:, j], one[:, 0]), f"K={K} class {j}: logits differ from smaat_dsconv_outconv_fwd"
            assert torch.equal(cls, lg.argmax(1)), f"K={K}: class map is not torch.argmax of the logits"
            alone = _classify(L, ow, bias, mode, want_logits=False)
            again = _classify(L, ow, bias, mode, want_logits=False)
            assert torch.equal(alone, cls) and torch.equal(again, cls), f"K={K}: class map depends on the logits output / launch"


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("cout", [96, 128])
def test_classify_at_n_tile_128_is_the_one_class_kernel_bit_for_bit(cout, k, mode, ds_impl):
    """Cout in (64, 128]: the N_TILE 128 instances, with the zero-padded class weights past Cout at 96.  They keep the weights of
    at most 22 classes beside their rings; 32 classes are declined (the caller then runs the layers apart)."""
    L = _layer(2, 224, 224, k, seed=cout + k, cout=cout)
    for K in (2, 21, 22):
        ow, ob = _oc(L, K)
        cls, lg = _classify(L, ow, ob, mode)
        for j in range(K):
            one = _one_class(L, ow[j], ob[j:j + 1], mode)
            assert torch.equal(lg[:, j], one[:, 0]), f"Cout={cout} K={K} class {j}: logits differ from smaat_dsconv_outconv_fwd"
        assert torch.equal(cls, lg.argmax(1))
        assert torch.equal(_classify(L, ow, ob, mode, want_logits=False), cls)
    ow, ob = _oc(L, 32)
    assert not ops.dsconv_classify_takes(L["x"], None, L["pw_w"], k, 32, mode)
    assert ops.dsconv_classify(L["x"], L["dw_w"], L["dw_b"], k, L["pw_w"], L["scale"], L["shift"], True, ow, ob, mode=mode) is None


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_classify_ties_go_to_the_first_index_and_nan_wins(mode, ds_impl):
    B, H, W = SHAPES[0]
    L = _layer(2, H, W, 2, seed=5)
    ow, ob = _oc(L, 8)
    ow[1] *= 4.0                                          # class 1 wins often ...
    ow[3], ob[3] = ow[1], ob[1]                           # ... and so would its duplicates 3 and 6
    ow[6], ob[6] = ow[1], ob[1]
    cls, lg = _classify(L, ow, ob, mode)
    assert torch.equal(lg[:, 1], lg[:, 3]) and torch.equal(lg[:, 1], lg[:, 6])
    assert int((cls == 1).sum()) > 0 and int(((cls == 3) | (cls == 6)).sum()) == 0
    assert torch.equal(cls, lg.argmax(1))
    same = ow[:1].expand(8, C).contiguous()              # every class the same: all pixels to class 0
    assert int(_classify(L, same, ob[:1].expand(8).contiguous(), mode, want_logits=False).abs().sum()) == 0
    ob_nan = ob.clone()
    ob_nan[5] = float("nan")
    ob_nan[7] = float("nan")
    cls, lg = _classify(L, ow, ob_nan, mode)
    assert bool(torch.isnan(lg[:, 5]).all()) and bool((cls == 5).all())


def _port_logits64(L, ow, ob):
    """The layer in float64 on the CPU: depthwise 3x3 (groups = Cin, k per channel), pointwise, BatchNorm affine, ReLU, OutConv."""
    x = L["x"].double().cpu()
    d = F.conv2d(x, L["dw_w"].double().cpu(), L["dw_b"].double().cpu(), padding=1, groups=C)
    z = F.conv2d(d, L["pw_w"].double().cpu())
    a = torch.relu(z * L["scale"].double().cpu()[None, :, None, None] + L["shift"].double().cpu()[None, :, None, None])
    return F.conv2d(a, ow.double().cpu()[:, :, None, None], ob.double().cpu())


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("K", [8, 21])
def test_classify_against_float64(K, mode):
    L = _layer(2, 224, 224, 2, seed=77 + K)
    ow, ob = _oc(L, K)
    cls, lg = _classify(L, ow, ob, mode)
    ref = _port_logits64(L, ow, ob)
    scale = float(ref.abs().max())
    err = float((lg.double().cpu() - ref).abs().max()) / scale
    tol = NET_TOL[mode]
    assert err <= tol, f"logits: max rel err {err:.3e} > {tol:.1e}"
    top2 = ref.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 2 * tol * scale
    want = ref.argmax(1)
    bad = int(((cls.cpu() != want) & clear).sum())
    print(f"ERR classify K={K} {mode}: logits {err:.3e} (bound {tol:.1e}); {int((~clear).sum())} of {clear.numel()} pixels "
          f"within the bound of a tie, {int((cls.cpu() != want).sum())} classes differ from float64")
    assert bad == 0


def _planted(B, K, P, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, K, P, generator=g)
    n = max(1, P // 8)
    px = torch.randint(0, P, (B, n), generator=g)
    for b in range(B):                                   # ties: copy each chosen pixel's max into another channel
        for p in px[b].tolist():
            c = int(torch.randint(0, K, (1,), generator=g))
            x[b, c, p] = x[b, :, p].max()
    x[0, K - 1, 0] = float("nan")                        # a lone NaN in the last channel
    if P > 3:
        x[B - 1, K // 2, 3] = float("nan")               # two NaNs: the first wins
        x[B - 1, K - 1, 3] = float("nan")
        x[0, :, 2] = 0.25                                # every channel equal: class 0
    return x


@pytest.mark.parametrize("K", [2, 8, 21, 32, 100, 1024])
@pytest.mark.parametrize("P", [(16, 20), (15, 13)])
@pytest.mark.parametrize("misaligned", [False, True])
def test_argmax_channels_equals_torch_argmax(K, P, misaligned):
    H, W = P
    x = _planted(3, K, H * W, seed=K + H).view(3, K, H, W)
    if misaligned:
        base = torch.empty(x.numel() + 1, device="cuda")
        xd = base[1:].view(x.shape)                      # 4-byte aligned only: the scalar kernel
        xd.copy_(x.cuda())
    else:
        xd = x.cuda()
    got = ops.argmax_channels(xd)
    want = x.argmax(1)
    assert got.dtype == torch.int64 and torch.equal(got.cpu(), want)
    assert torch.equal(got, xd.argmax(1))


class _PlainWrapper(nn.Module):
    """A model with neither forward_serving nor forward_classes (as a reference class used through patch_reference())."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x)


def _conf(pred, y, K):
    m = S.IoU(K)
    m.add(pred, y)
    return m.conf_metric.counts()[0]


@pytest.mark.parametrize("cfg", [(3, 21, 8, 224), (12, 8, 4, 288)])
def test_inference_session_classes_end_to_end(cfg):
    n_ch, K, B, HW = cfg
    torch.manual_seed(K)
    m = S.SmaAt_UNet(n_ch, K).cuda().eval()
    with torch.no_grad():             # a freshly initialised OutConv lets its bias pick one class everywhere: spread the logits
        m.outc.conv.weight.mul_(50.0)
        m.outc.conv.bias.zero_()
    sc = InferenceSession(m, B, (n_ch, HW, HW), output="classes")
    sl = InferenceSession(m, B, (n_ch, HW, HW))
    assert sc.static_out.dtype == torch.int64 and sc.out_shape == (B, HW, HW)
    assert sc.d2h_bytes_per_step == B * HW * HW * 8 and sl.d2h_bytes_per_step == B * K * HW * HW * 4
    with ops.profile() as prof:
        with torch.no_grad():
            m.forward_classes(torch.rand(B, n_ch, HW, HW, device="cuda"))
    names = prof.summary()
    assert "smaat_dsconv_classify_fwd" in names and "smaat_outconv_fwd" not in names and "smaat_argmax_channels_fwd" not in names
    xs = [torch.rand(B, n_ch, HW, HW, device="cuda") for _ in range(3)]
    dev_maps = [sc.forward(x).clone() for x in xs]
    print(f"ERR session classes K={K}: distinct classes per batch {[int(torch.unique(c).numel()) for c in dev_maps]}")
    host = [x.cpu().pin_memory() for x in xs]
    sc.submit(host[0])
    sc.submit(host[1])
    got = [sc.collect().clone()]
    sc.submit(host[2])
    got += [sc.collect().clone(), sc.collect().clone()]
    for i in range(3):
        assert got[i].dtype == torch.int64 and torch.equal(got[i], dev_maps[i].cpu()), f"batch {i}: submit/collect differs"
    y = torch.randint(0, K, (B, HW, HW), device="cuda")
    tol = NET_TOL[S.get_pointwise_mode()]
    for x, cls in zip(xs, dev_maps):
        lg = sl.forward(x).clone()
        with torch.no_grad():
            assert torch.equal(cls, m.forward_classes(x))           # the graph replays the eager class map
        top2 = lg.topk(2, dim=1).values
        near = (top2[:, 0] - top2[:, 1]) <= 2 * tol * float(lg.abs().max())
        diff = cls != lg.argmax(1)
        print(f"ERR session classes K={K}: {int(near.sum())} pixels near a tie, {int(diff.sum())} differ from argmax(logits)")
        assert int((diff & ~near).sum()) == 0
        c_cls, c_lg = _conf(cls, y, K), _conf(lg, y, K)
        assert int(np.abs(c_cls - c_lg).sum()) <= 2 * int(diff.sum())
        if int(diff.sum()) == 0:
            assert np.array_equal(c_cls, c_lg)


def test_inference_session_classes_without_forward_classes_and_for_the_dense_unet():
    torch.manual_seed(4)
    x = torch.rand(2, 3, 64, 64, device="cuda")
    for m in (S.UNet(3, 21).cuda().eval(), _PlainWrapper(S.SmaAt_UNet(3, 21)).cuda().eval(), S.SmaAt_UNet(3, 40).cuda().eval()):
        sess = InferenceSession(m, 2, (3, 64, 64), output="classes")
        got = sess.forward(x).clone()
        with torch.no_grad():
            want = torch.argmax(m(x), 1)
        assert torch.equal(got, want), type(m).__name__


def test_inference_session_classes_refresh_follows_new_weights():
    torch.manual_seed(6)
    m = S.SmaAt_UNet(3, 21).cuda().eval()
    with torch.no_grad():
        m.outc.conv.weight.mul_(50.0)
        m.outc.conv.bias.zero_()
    x = torch.rand(2, 3, 96, 96, device="cuda")
    sess = InferenceSession(m, 2, (3, 96, 96), output="classes")
    before = sess.forward(x).clone()
    with torch.no_grad():
        m.outc.conv.weight.mul_(-1.0)
        m.up4.conv.double_conv[4].running_mean.add_(0.3)
    sess.refresh()
    after = sess.forward(x).clone()
    with torch.no_grad():
        want = m.forward_classes(x)
    assert torch.equal(after, want) and not torch.equal(after, before)
