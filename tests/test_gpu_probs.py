"""-m gpu: class probabilities from multi-class models.  smaat_softmax_channels_fwd against float64 softmax and torch.softmax,
with torch's NaN / 0 / 1 pattern on non-finite logits; SmaAt_UNet.forward_probs bit for bit the softmax kernel applied to
forward_serving's logits, and against float64 softmax of the float64 port's logits; InferenceSession(output="probs") end to
end."""
import numpy as np
import pytest
import torch
from torch import nn

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from smaat_unet_b200 import ops
from smaat_unet_b200.engine import InferenceSession
from tests._util import NET_TOL, load_np_state_dict

pytestmark = pytest.mark.gpu

ABS_TOL, REL_TOL = 1e-6, 1e-5             # softmax rounding: absolute, and relative where the float64 probability > 1e-30


def _mx(t):
    return float(t.max()) if t.numel() else 0.0


def _check_softmax(p, x, what):
    """p: fp32 probabilities of the fp32 logits x (B, K, ...), against float64 softmax of the same logits."""
    p64 = torch.softmax(x.double().cpu(), 1)
    got = p.double().cpu()
    err = (got - p64).abs()
    # Relative where the probability is representable, absolute below.  An absolute 1e-6 cannot hold near p = 1 at large K:
    # each change of the running max rescales s by one more rounded exp, and at K = 1024 a pixel with p = 0.957 is off by
    # 4.1e-6 (4.3e-6 relative) -- exactly what a float32 emulation of the recurrence on the CPU gives
    big = p64 > 1e-30
    assert _mx(err[~big]) <= ABS_TOL, f"{what}: max abs err {_mx(err[~big]):.3e} where p64 <= 1e-30"
    rel = float((err[big] / p64[big]).max())
    assert rel <= REL_TOL, f"{what}: max rel err {rel:.3e}"
    K = x.shape[1]
    drift = float((got.sum(1) - 1.0).abs().max())
    assert drift <= K * 2.0 ** -23, f"{what}: a row sums to 1 +- {drift:.3e} (K = {K})"
    return float(err.max()), rel


def _logits(B, K, P, seed):
    """randn * 4 logits, a quarter of the pixels scaled by 10^u, u in [0, 30): magnitudes up to 1e30."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, K, P, generator=g) * 4.0
    big = torch.rand(B, 1, P, generator=g) < 0.25
    scale = torch.pow(10.0, torch.rand(B, 1, P, generator=g) * 30.0)
    return torch.where(big, x * scale, x)


@pytest.mark.parametrize("K", [1, 2, 8, 21, 32, 33, 1024])
@pytest.mark.parametrize("HW", [(16, 20), (15, 13)])      # P = 320: 128-bit loads; P = 195: the scalar kernel
@pytest.mark.parametrize("misaligned", [False, True])
def test_softmax_channels_against_float64_and_torch(K, HW, misaligned):
    H, W = HW
    x = _logits(3, K, H * W, seed=K + H).view(3, K, H, W)
    if misaligned:
        base = torch.empty(x.numel() + 1, device="cuda")
        xd = base[1:].view(x.shape)                      # 4-byte aligned only: the scalar kernel
        xd.copy_(x.cuda())
    else:
        xd = x.cuda()
    p = ops.softmax_channels(xd)
    assert p.dtype == torch.float32 and p.shape == x.shape
    e_abs, e_rel = _check_softmax(p, x, f"K={K} P={H * W}")
    pt = torch.softmax(xd, 1)
    d = (p - pt).abs()
    big = pt > 1e-30
    assert _mx(d[~big]) <= ABS_TOL and float((d[big] / pt[big]).max()) <= REL_TOL, f"K={K}: differs from torch.softmax"
    print(f"ERR softmax_channels K={K} P={H * W} misaligned={misaligned}: abs {e_abs:.2e} rel {e_rel:.2e}")


def _nonfinite_cases():
    """(K, pixel columns): each column a logit vector with a non-finite pattern, in the order torch's results are pinned."""
    inf, nan = float("inf"), float("nan")
    cols = {
        4: [[0.5, nan, -1.0, 2.0],             # a NaN logit: NaN everywhere
            [nan, 0.5, -1.0, 2.0],             # ... also as the first class
            [0.5, inf, -1.0, 2.0],             # a +inf logit: NaN everywhere
            [inf, inf, 0.0, 1.0],              # two +inf logits
            [-inf, -inf, -inf, -inf],          # all -inf: NaN everywhere
            [0.5, -inf, -1.0, 2.0],            # a -inf logit among finite ones: 0 there
            [-inf, 0.5, -1.0, 2.0],            # ... also as the first class
            [-inf, -inf, 3.0, -inf],           # one finite logit: 1 there, 0 elsewhere
            [-inf, nan, 3.0, 1.0],             # -inf then NaN
            [inf, -inf, 0.0, 1.0],             # +inf and -inf
            [1e30, -1e30, 3.0, 1e30]],         # huge finite logits
        1: [[0.5], [-3e30], [nan], [inf], [-inf]],
    }
    return cols


@pytest.mark.parametrize("vector", [False, True])      # the columns alone (scalar kernel) or zero-padded to a multiple of 4
def test_softmax_channels_nonfinite_is_torchs_pattern(vector):
    for K, cols in _nonfinite_cases().items():
        x = torch.tensor(cols, dtype=torch.float32).t().contiguous()        # (K, n)
        n = (x.shape[1] + 3) // 4 * 4 if vector else x.shape[1]
        assert (n % 4 == 0) == vector
        xp = torch.zeros(K, n)
        xp[:, :x.shape[1]] = x
        xb = xp[None].expand(2, K, n).contiguous()
        p = ops.softmax_channels(xb.cuda()).cpu()
        want = torch.softmax(xb, 1)
        nan_w, nan_p = torch.isnan(want), torch.isnan(p)
        assert torch.equal(nan_w, nan_p), f"K={K}: NaN pattern {nan_p[0].t().tolist()} != torch's {nan_w[0].t().tolist()}"
        for v in (0.0, 1.0):
            assert torch.equal(want == v, p == v), f"K={K}: pattern of {v} differs from torch's"
        fin = ~nan_w
        assert float((p[fin] - want[fin]).abs().max()) <= ABS_TOL
    # K = 1 on finite logits is exactly 1 everywhere
    x = torch.randn(2, 1, 7, 9, device="cuda") * 1e3
    assert bool((ops.softmax_channels(x) == 1.0).all())


# ---- the network ---------------------------------------------------------------------------------------------------------------
def test_forward_probs_is_the_softmax_of_the_serving_logits():
    # K = 8 and 21 have a fused class-map epilogue, K = 33 does not: the probabilities take the logits route either way
    for K in (8, 21, 33):
        torch.manual_seed(K)
        m = S.SmaAt_UNet(3, K).cuda().eval()
        x = torch.rand(2, 3, 64, 64, device="cuda")
        with ops.profile() as prof, torch.no_grad():
            p = m.forward_probs(x)
        names = prof.summary()
        assert "smaat_softmax_channels_fwd" in names and "smaat_outconv_fwd" in names, f"K={K}"
        with torch.no_grad():
            lg = m.forward_serving(x)            # the same convs and OutConv, ending in the logits
        assert torch.equal(p, ops.softmax_channels(lg)), f"K={K}"
        _check_softmax(p, lg.cpu(), f"SmaAt_UNet(3, {K}).forward_probs")


def _net(n_ch, K, seed):
    sd = cast_sd(fill_schema(smaat_unet_schema(n_ch, K, 2), seed), np.float32)
    m = load_np_state_dict(S.SmaAt_UNet(n_ch, K, kernels_per_layer=2), sd).cuda().eval()
    return m, TP.to_torch_sd(sd, dtype=torch.float64)


@pytest.mark.parametrize("cfg", [(3, 21, 224), (12, 8, 288)])
def test_forward_probs_against_float64_port(cfg):
    n_ch, K, HW = cfg
    m, sd64 = _net(n_ch, K, seed=K)
    x = torch.from_numpy(np.random.default_rng(K).uniform(0, 1, (2, n_ch, HW, HW)).astype(np.float32))
    with torch.no_grad():
        l64 = TP.smaat_unet_forward(x.double(), sd64)
    p64 = torch.softmax(l64, 1)
    for mode in ("tf32x3", "tf32"):
        S.set_pointwise_mode(mode)
        try:
            with ops.profile() as prof, torch.no_grad():
                p = m.forward_probs(x.cuda())
            names = prof.summary()
        finally:
            S.set_pointwise_mode("tf32x3")
        assert "smaat_outconv_fwd" in names and "smaat_softmax_channels_fwd" in names
        err = (p.double().cpu() - p64).abs()
        # the softmax Jacobian's infinity norm is at most 1/2: a logit error of e moves a probability by at most e / 2
        bound = 0.5 * NET_TOL[mode] * float(l64.abs().max()) + ABS_TOL + REL_TOL * p64
        worst = float((err / bound).max())
        print(f"ERR forward_probs {cfg} [{mode}]: max abs err {float(err.max()):.3e}, max|logit| {float(l64.abs().max()):.3f}, "
              f"worst err / bound {worst:.3f}")
        assert worst <= 1.0, f"{cfg} [{mode}]"


class _PlainWrapper(nn.Module):
    """A model with neither forward_serving nor forward_probs (as a reference class used through patch_reference())."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x)


@pytest.mark.parametrize("cfg", [(3, 21, 8, 224), (12, 8, 4, 288)])
def test_inference_session_probs_end_to_end(cfg):
    n_ch, K, B, HW = cfg
    m, _ = _net(n_ch, K, seed=K + 1)
    sp = InferenceSession(m, B, (n_ch, HW, HW), output="probs")
    assert sp.static_out.dtype == torch.float32 and sp.out_shape == (B, K, HW, HW)
    assert sp.d2h_bytes_per_step == B * K * HW * HW * 4
    xs = [torch.rand(B, n_ch, HW, HW, device="cuda") for _ in range(5)]
    dev = [sp.forward(x).clone() for x in xs]
    for x, p in zip(xs, dev):
        with torch.no_grad():
            assert torch.equal(p, m.forward_probs(x)), "the graph does not replay the eager forward_probs"
    assert not torch.equal(dev[0], dev[1])
    host = [x.cpu().pin_memory() for x in xs]
    got = []
    sp.submit(host[0])
    sp.submit(host[1])
    for i in range(2, 5):
        got.append(sp.collect().clone())
        sp.submit(host[i])
    got += [sp.collect().clone(), sp.collect().clone()]
    for i in range(5):
        assert got[i].dtype == torch.float32 and torch.equal(got[i], dev[i].cpu()), f"batch {i}: submit/collect differs"


def test_inference_session_probs_other_routes_are_the_softmax_kernel_on_the_logits():
    torch.manual_seed(4)
    x = torch.rand(2, 3, 64, 64, device="cuda")
    cases = [(S.UNet(3, 21), True), (S.UNetAttention(3, 21), True), (_PlainWrapper(S.SmaAt_UNet(3, 21)), True),
             (S.SmaAt_UNet(3, 21), False)]
    for m, fusions in cases:
        m = m.cuda().eval()
        sess = InferenceSession(m, 2, (3, 64, 64), output="probs", serving_fusions=fusions)
        got = sess.forward(x).clone()
        with torch.no_grad():
            lg = m(x)
        assert torch.equal(got, ops.softmax_channels(lg)), f"{type(m).__name__} serving_fusions={fusions}"
        _check_softmax(got, lg.cpu(), type(m).__name__)


def test_inference_session_probs_refresh_follows_new_weights():
    m, _ = _net(3, 21, seed=6)
    x = torch.rand(2, 3, 96, 96, device="cuda")
    sess = InferenceSession(m, 2, (3, 96, 96), output="probs")
    before = sess.forward(x).clone()
    with torch.no_grad():
        m.outc.conv.weight.mul_(-1.0)
        m.up4.conv.double_conv[4].running_mean.add_(0.3)
    sess.refresh()
    after = sess.forward(x).clone()
    with torch.no_grad():
        want = m.forward_probs(x)
    assert torch.equal(after, want) and not torch.equal(after, before)


def test_inference_session_probs_rejects_a_one_class_model():
    m = S.SmaAt_UNet(12, 1).cuda().eval()
    with pytest.raises(ValueError, match="one output channel"):
        InferenceSession(m, 1, (12, 64, 64), output="probs")


def test_forward_probs_in_train_mode_and_under_autograd_is_the_plain_forward_then_the_kernel():
    torch.manual_seed(8)
    m = S.SmaAt_UNet(3, 8).cuda().eval()
    x = torch.rand(2, 3, 64, 64, device="cuda", requires_grad=True)
    p = m.forward_probs(x)
    assert not p.requires_grad
    with torch.no_grad():
        assert torch.equal(p, ops.softmax_channels(m(x)))
