"""-m gpu: the dense UNet path (3x3 conv kernels, DoubleConv / Down / Up, UNet / UNetAttention, sessions) vs the oracles."""
import json
import os

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle import dense_oracle as D
from oracle.cases_dense import DENSE_CASES, case_tensors, run_port
from oracle.torch_port import to_torch_sd
from smaat_unet_b200 import ops
from tests._util import NET_TOL, PW_TOL, assert_close, dev, load_np_state_dict

pytestmark = pytest.mark.gpu
RNG = np.random.default_rng(4321)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODES = ("fp32", "tf32x3", "tf32")
# The dense convs sum K = 9 Cin products (up to 9 216): fp32 accumulation noise grows with K, so the per-conv bounds of
# tests/_util.py (set for the pointwise K <= 1 024) get a factor of 3 here.
CONV_TOL = {m: 3 * t for m, t in PW_TOL.items()}


def rnd(*shape, lo=-1.0, hi=1.0):
    return RNG.uniform(lo, hi, shape).astype(np.float32)


@pytest.fixture(autouse=True)
def _restore_mode():
    old = ops.get_pointwise_mode()
    yield
    ops.set_pointwise_mode(old)


# ------------------------------------------------------------------------------ kernel level
CONV_CASES = [
    # B, C0, C1, H, W, Cout
    (2, 12, 0, 16, 20, 64),        # inc.0: Cin = 12 (one zero-padded chunk)
    (1, 64, 0, 12, 16, 8),
    (2, 96, 0, 9, 12, 128),        # ragged patch rows
    (1, 64, 64, 10, 8, 64),        # Up's virtual concat
    (1, 12, 20, 6, 8, 256),        # concat of two partial chunks, two channel passes
    (1, 128, 0, 5, 4, 512),
    (1, 16, 0, 7, 10, 16),         # W % 4 != 0: CUDA-core kernel in every mode
    (1, 8, 0, 6, 288, 64),         # a 288-wide slice
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv3x3_matches_oracle(case, mode):
    B, C0, C1, H, W, Cout = case
    x = rnd(B, C0 + C1, H, W)
    w = rnd(Cout, C0 + C1, 3, 3, lo=-0.2, hi=0.2)
    sc, sh = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    z = D.conv3x3(x.astype(np.float64), w, None) * sc[None, :, None, None] + sh[None, :, None, None]
    x0 = dev(x[:, :C0])
    x1 = dev(x[:, C0:]) if C1 else None
    wp = ops.conv3x3_pack_weight(dev(w), C0, C1)
    split = ops.split_tf32(wp) if mode == "tf32x3" else None
    for relu in (False, True):
        stats = ops.new_stats(Cout, x0.device)
        y = ops.conv3x3(x0, wp, Cout, dev(sc), dev(sh), relu, x1=x1, mode=mode, w_split=split, stats=stats)
        assert_close(y, np.maximum(z, 0) if relu else z, CONV_TOL[mode], f"conv3x3 {case} {mode} relu={relu}")
        s = stats.cpu().numpy()
        n = B * H * W
        assert_close(s[:Cout] / n, z.mean(axis=(0, 2, 3)), CONV_TOL[mode], "stats: mean")
        assert_close(s[Cout:] / n, (z * z).mean(axis=(0, 2, 3)), CONV_TOL[mode], "stats: mean of squares")
    assert ops.conv3x3_takes(x0, x1, wp, Cout, mode) == (mode != "fp32" and W % 4 == 0)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [(2, 12, 0, 8, 12, 16), (1, 16, 8, 6, 8, 24), (2, 8, 0, 5, 7, 8)])
def test_conv3x3_gradients_match_autograd(case, mode):
    """dX (forward kernel on the flipped, transposed weight, split over the concat) and dW vs float64 CPU autograd."""
    ops.set_pointwise_mode(mode)
    B, C0, C1, H, W, Cout = case
    x, w, g = rnd(B, C0 + C1, H, W), rnd(Cout, C0 + C1, 3, 3, lo=-0.3, hi=0.3), rnd(B, Cout, H, W)
    xr = torch.from_numpy(x).double().requires_grad_()
    wr = torch.from_numpy(w).double().requires_grad_()
    torch.nn.functional.conv2d(xr, wr, padding=1).backward(torch.from_numpy(g).double())
    m = S.DoubleConv(C0 + C1, Cout).cuda()
    with torch.no_grad():
        m.double_conv[0].weight.copy_(dev(w))
    x0, x1 = dev(x[:, :C0]), (dev(x[:, C0:]) if C1 else None)
    dW = torch.zeros((Cout, C0 + C1, 3, 3), device="cuda")
    from smaat_unet_b200 import functional as Fn
    dx0, dx1 = Fn.conv3x3_bwd(m, 0, dev(g), x0, x1, dW)
    tol = 5 * CONV_TOL[mode]
    assert_close(dW, wr.grad.numpy(), tol, f"dW {case}")
    assert_close(dx0, xr.grad[:, :C0].numpy(), tol, f"dx0 {case}")
    if C1:
        assert_close(dx1, xr.grad[:, C0:].numpy(), tol, f"dx1 {case}")


WGRAD_CASES = [
    # B, C0, C1, H, W, Cout
    (2, 12, 0, 7, 12, 64),          # inc.0: 12 input channels in one 64-channel tile
    (1, 96, 80, 5, 40, 136),        # concat, two channel tiles per source, two output tiles, a ragged 32-pixel segment
    (2, 64, 0, 4, 288, 8),          # a 288-wide slice, Cout < 128 (zero-filled dz rows)
]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
@pytest.mark.parametrize("case", WGRAD_CASES)
def test_conv3x3_wgrad_tensor_core_matches_autograd(case, mode):
    """The wgmma weight gradient (conv3x3_wgrad_tc.cu) vs float64 CPU autograd, accumulating into a non-zero dW."""
    B, C0, C1, H, W, Cout = case
    x, g = rnd(B, C0 + C1, H, W), rnd(B, Cout, H, W)
    xr = torch.from_numpy(x).double()
    wr = torch.zeros((Cout, C0 + C1, 3, 3), dtype=torch.float64, requires_grad=True)
    torch.nn.functional.conv2d(xr, wr, padding=1).backward(torch.from_numpy(g).double())
    base = rnd(Cout, C0 + C1, 3, 3)
    dW = dev(base)
    with ops.profile() as prof:
        ops.conv3x3_bwd_weight(dev(g), dev(x[:, :C0]), dev(x[:, C0:]) if C1 else None, dW, mode=mode)
    assert [k for k in prof.summary()] == ["smaat_conv3x3_bwd_weight"]
    ref = wr.grad.numpy()
    got = dW.double().cpu().numpy() - base
    assert_close(got, ref, 5 * CONV_TOL[mode], f"wgrad(tc) {case} {mode}")


def test_conv3x3_refuses_tensor_core_requests_it_cannot_take():
    x = torch.zeros(1, 8, 5, 6, device="cuda")                       # W % 4 != 0
    wp = ops.conv3x3_pack_weight(torch.zeros(16, 8, 3, 3, device="cuda"), 8)
    y = torch.empty(1, 16, 5, 6, device="cuda")
    lib = S._lib.load()
    rc = lib.smaat_conv3x3_fwd(x.data_ptr(), 8, 8 * 30, None, 0, 0, wp.data_ptr(), None, None, None, y.data_ptr(), 16 * 30, None,
                               1, 5, 6, 16, 0, 1, ops._stream())
    assert rc == -3       # SMAAT_E_UNSUPPORTED
    with pytest.raises(NotImplementedError):
        m = S.DoubleConv(4, 8).cuda().eval()
        m.double_conv[0] = torch.nn.Conv2d(4, 8, 5, padding=2).cuda()
        with torch.no_grad():
            m(torch.zeros(1, 4, 8, 8, device="cuda"))


# ------------------------------------------------------------------------------ modules / networks vs the goldens
def _golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def _build(name):
    c = DENSE_CASES[name]
    kind = c["kind"]
    if kind == "doubleconv":
        m = S.DoubleConv(c["cin"], c["cout"], c["mid"])
    elif kind == "down":
        m = S.Down(c["cin"], c["cout"])
    elif kind == "up":
        m = S.Up(c["cin"], c["cout"], c.get("bilinear", True))
    elif kind == "unet":
        return S.UNet(c["n_channels"], c["n_classes"], c.get("bilinear", True))
    else:
        return S.UNetAttention(c["n_channels"], c["n_classes"], c.get("bilinear", True))

    class Wrap(torch.nn.Module):      # reference-keyed "m." prefix
        def __init__(self, mod):
            super().__init__()
            self.m = mod

        def forward(self, *a):
            return self.m(*a)
    return Wrap(m)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_dense_modules_match_goldens(name, mode):
    ops.set_pointwise_mode(mode)
    c = DENSE_CASES[name]
    sd, xs = case_tensors(name, np.float32)
    m = load_np_state_dict(_build(name), sd).cuda()
    train = c.get("train", False)
    m.train(train)
    with torch.no_grad():
        y = m(*[dev(x) for x in xs])
    g = _golden(name)
    tol = (NET_TOL if c["kind"] in ("unet", "unetatt") else CONV_TOL)[mode]
    if train:
        tol *= 10       # batch statistics over a handful of pixels amplify the conv noise (cf. test_gpu_modules)
    assert_close(y, g["output"], tol, f"{name} {mode}")
    if train:
        msd = m.state_dict()
        for k in g.files:
            if k.startswith("buf:"):
                assert_close(msd[k[4:]], g[k], 10 * CONV_TOL[mode] + 1e-6, f"{name} {k}")


def _rel_max(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_dense_gradients_match_cpu_autograd():
    """Train-mode UNetAttention (dense blocks + CBAMs, B = 2, 64 x 64) gradients vs float64 CPU autograd of the port, in
    fp32 mode.  Noise-calibrated as in test_gpu_api_paths: BatchNorm over the 4 x 4 bottleneck amplifies rounding, so the
    bound is a small multiple of how far the port itself moves between fp32 and fp64 on the same case."""
    ops.set_pointwise_mode("fp32")
    sd, _ = case_tensors("dense_unetatt_32", np.float64)
    x64 = RNG.uniform(0, 1, (2, 12, 64, 64))
    g = RNG.uniform(-1, 1, (2, 1, 64, 64))
    m = load_np_state_dict(S.UNetAttention(12, 1), sd).cuda().train()
    y = m(dev(x64))
    y.backward(dev(g))
    grads = {}
    for dt in (torch.float64, torch.float32):
        tsd = to_torch_sd(sd, dt)
        names = [k for k, _ in m.named_parameters()]
        for k in names:
            tsd[k].requires_grad_()
        yr = D.port_unet_forward(torch.from_numpy(x64).to(dt), tsd, training=True, attention=True)
        yr.backward(torch.from_numpy(g).to(dt))
        grads[dt] = {k: tsd[k].grad.double().numpy() for k in names}
        if dt == torch.float64:
            assert_close(y, yr.detach().numpy(), 1e-4, "train forward")
    g64, g32 = grads[torch.float64], grads[torch.float32]
    gmax = max(float(np.abs(v).max()) for v in g64.values())
    live = [k for k, v in g64.items() if np.abs(v).max() >= 1e-6 * gmax]
    noise = max(_rel_max(g32[k], g64[k]) for k in live)
    tol = max(2e-3, 5.0 * noise)
    for k, p in m.named_parameters():
        got = p.grad.double().cpu().numpy()
        if k not in live:        # conv bias before a train-mode BatchNorm: mathematically zero
            assert float(np.abs(got).max()) <= 1e-3 * gmax, k
            continue
        e = _rel_max(got, g64[k])
        assert np.isfinite(e) and e <= tol, f"grad {k}: rel max {e:.3e} (tol {tol:.1e}; port fp32 noise {noise:.1e})"


def test_unet_288_uses_the_tensor_core_kernel_and_matches_the_port():
    ops.set_pointwise_mode("tf32x3")
    torch.manual_seed(0)
    m = S.UNet(12, 1).cuda().eval()
    x = torch.rand(2, 12, 288, 288, device="cuda")
    with torch.no_grad(), ops.profile() as prof:
        y = m(x)
    s = prof.summary(by_shape=True)
    tc = {k for k in s if k.startswith("smaat_conv3x3_fwd[")}
    simt = {k for k in s if k.startswith("smaat_conv3x3_fwd_simt")}
    assert sum(s[k]["launches"] for k in tc) + sum(s[k]["launches"] for k in simt) == 18
    # every layer with W % 4 == 0 runs on the tensor cores; only the 18 x 18 bottleneck (W % 4 == 2) takes the CUDA cores
    assert all("S18x18" in k for k in simt), simt
    assert sum(s[k]["launches"] for k in tc) == 16
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    with torch.no_grad():
        yr = D.port_unet_forward(x.cpu().double(), sd)
    assert_close(y, yr.numpy(), NET_TOL["tf32x3"], "UNet 288")


# ------------------------------------------------------------------------------ sessions
def test_inference_session_replays_unet_bit_exactly():
    from smaat_unet_b200.engine import InferenceSession
    torch.manual_seed(1)
    m = S.UNet(12, 1).cuda().eval()
    x = torch.rand(2, 12, 64, 64, device="cuda")
    with torch.no_grad():
        ref = m(x).clone()
    sess = InferenceSession(m, 2, (12, 64, 64))
    y = sess.forward(x)
    torch.cuda.synchronize()
    assert torch.equal(y, ref)


def _port_grads(sd, names, x, y, dtype):
    """Parameter gradients of the port's train-mode UNetAttention under the sessions' loss (sum of squares / B)."""
    tsd = to_torch_sd(sd, dtype)
    for k in names:
        tsd[k].requires_grad_()
    pred = D.port_unet_forward(torch.from_numpy(x).to(dtype), tsd, training=True, attention=True)
    loss = torch.nn.functional.mse_loss(pred.squeeze(1), torch.from_numpy(y).to(dtype), reduction="sum") / x.shape[0]
    loss.backward()
    return float(loss.detach()), {k: tsd[k].grad.double().numpy() for k in names}


def _rel_l2(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_train_session_unet_attention_gradients(mode):
    """One TrainSession step of UNetAttention (CUDA graphs, two-phase backward, flat gradient bucket, weight caches re-derived
    inside the capture) with lr = 0, B = 2, 128 x 128.  The bucket must hold
      * the gradients of a plain eager forward + backward of the same model on the same GPU, per parameter to 1e-4 of its
        maximum (the two differ only in the order of atomically merged sums: measured <= 1e-6), in both modes, and
      * in fp32 mode, the gradients of CPU float64 autograd through the port, to a small multiple of the port's own
        fp32-vs-fp64 movement on the same case (max and L2 norms, as test_gpu_api_paths).  3xTF32 carries ~8x the product
        error of fp32, which train-mode BatchNorm over small deep maps amplifies beyond an fp32-calibrated bound: its
        arithmetic is checked per kernel (test_conv3x3_*), the session path by the first comparison."""
    import copy

    from smaat_unet_b200.train import TrainSession
    ops.set_pointwise_mode(mode)
    torch.manual_seed(5)
    B, S_ = 2, 128
    m = S.UNetAttention(12, 1).cuda().train()
    m_eager = copy.deepcopy(m)
    sd = {k: v.detach().cpu().double().numpy().copy() for k, v in m.state_dict().items()}
    names = [k for k, _ in m.named_parameters()]
    x = RNG.uniform(0, 1, (B, 12, S_, S_))
    y = RNG.uniform(0, 1, (B, S_, S_))
    sess = TrainSession(m, B, (12, S_, S_), lr=0.0, use_graph=True)
    loss = float(sess.step(dev(x), dev(y)))
    torch.cuda.synchronize()
    bucket = {k: v.double().cpu().numpy() for k, v in zip(names, sess._views)}
    for k, p in m.named_parameters():
        assert p.grad.data_ptr() == sess._views[names.index(k)].data_ptr(), k      # the parameter's grad is its bucket slot
    sess.close()
    pred = m_eager(dev(x))
    l_eager = torch.nn.functional.mse_loss(pred.squeeze(1), dev(y), reduction="sum") / B
    l_eager.backward()
    assert abs(loss - float(l_eager)) <= 1e-5 * abs(float(l_eager)), (loss, float(l_eager))
    for k, p in m_eager.named_parameters():
        ref = p.grad.double().cpu().numpy()
        assert np.abs(bucket[k] - ref).max() <= 1e-4 * max(np.abs(ref).max(), 1e-30), f"{mode}: bucket vs eager, {k}"
    if mode != "fp32":
        return
    l64, g64 = _port_grads(sd, names, x, y, torch.float64)
    _, g32 = _port_grads(sd, names, x, y, torch.float32)
    assert abs(loss - l64) <= 1e-4 * abs(l64), (loss, l64)
    gmax = max(float(np.abs(v).max()) for v in g64.values())
    live = [k for k, v in g64.items() if np.abs(v).max() >= 1e-6 * gmax]
    noise_max = max(_rel_max(g32[k], g64[k]) for k in live)
    noise_l2 = max(_rel_l2(g32[k], g64[k]) for k in live)
    tol_max, tol_l2 = max(2e-3, 5.0 * noise_max), max(1e-3, 5.0 * noise_l2)
    for k in names:
        if k not in live:         # conv bias before a train-mode BatchNorm: mathematically zero
            assert float(np.abs(bucket[k]).max()) <= 1e-3 * gmax, k
            continue
        e_max, e_l2 = _rel_max(bucket[k], g64[k]), _rel_l2(bucket[k], g64[k])
        assert np.isfinite(e_max) and e_max <= tol_max and e_l2 <= tol_l2, \
            f"bucket grad {k}: rel max {e_max:.3e} (tol {tol_max:.1e}), rel L2 {e_l2:.3e} (tol {tol_l2:.1e})"


def test_dense_index_shapes():
    with open(os.path.join(GOLDEN, "dense_index.json")) as f:
        idx = json.load(f)["cases"]
    for name in DENSE_CASES:
        assert tuple(_golden(name)["output"].shape) == tuple(idx[name]["output_shape"])
