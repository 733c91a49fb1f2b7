"""-m gpu: train-mode forward (batch-statistics BatchNorm, running-stat updates) vs the reference's golden
outputs, and every gradient of the differentiable blocks vs torch autograd over the CPU port (float64)."""
import os

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import CASES, case_tensors
from tests._util import assert_close, dev, load_np_state_dict
from tests.test_gpu_modules import build

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TRAIN_CASES = sorted(n for n, c in CASES.items() if c.get("train", False))
# train-mode BatchNorm divides by the batch std: fp32 noise is amplified (SURVEY 6: reference self-noise 2e-5)
FWD_TOL = {"fp32": 2e-4, "tf32x3": 2e-4}
GRAD_TOL = 5e-4


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", TRAIN_CASES)
def test_train_forward_matches_reference_golden(name, mode):
    c = CASES[name]
    sd, xs = case_tensors(name, np.float32)
    mod, prefix = build(c)
    load_np_state_dict(mod, sd, prefix)
    mod = mod.cuda().train()
    S.set_pointwise_mode(mode)
    try:
        with torch.no_grad():
            y = mod(*[dev(x) for x in xs])
        torch.cuda.synchronize()
    finally:
        S.set_pointwise_mode("tf32x3")
    g = np.load(os.path.join(GOLD, name + ".npz"))
    assert_close(y, g["output"], FWD_TOL[mode], f"{name} train fwd [{mode}]")
    after = mod.state_dict()
    for key in g.files:                      # running_mean / running_var / num_batches_tracked after one step
        if key.startswith("buf:"):
            k2 = key[4:][len(prefix):] if prefix else key[4:]
            got = after[k2].double().cpu().numpy()
            ref = g[key].astype(np.float64)
            assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), key


def _cpu_reference(kind, c, sd_np, xs_np, train, R, dtype=torch.float64):
    """torch autograd over the CPU port (float64 = ground truth): returns (output, dict name -> grad, [input grads])."""
    sd = {}
    for k, v in sd_np.items():
        t = torch.as_tensor(np.asarray(v))
        sd[k] = t.to(dtype).requires_grad_(True) if t.dtype != torch.int64 and not k.endswith(("running_mean", "running_var")) \
            else (t.to(dtype) if t.dtype != torch.int64 else t)
    xs = [torch.from_numpy(x).to(dtype).requires_grad_(True) for x in xs_np]
    if kind == "dsconv":
        y = TP.ds_conv(xs[0], sd, "m")
    elif kind == "doubleconv":
        y = TP.double_conv_ds(xs[0], sd, "m", train)
    elif kind == "down":
        y = TP.down_ds(xs[0], sd, "m", train)
    elif kind == "up":
        y = TP.up_ds(xs[0], xs[1], sd, "m", train)
    elif kind == "cbam":
        y = TP.cbam(xs[0], sd, "m", train)
    elif kind == "outconv":
        y = torch.nn.functional.conv2d(xs[0], sd["m.conv.weight"], sd["m.conv.bias"])
    elif kind == "unet":
        y = TP.smaat_unet_forward(xs[0], sd, train)
    else:
        raise KeyError(kind)
    (y * torch.from_numpy(R).to(dtype)).sum().backward()
    grads = {k: v.grad.double().numpy() for k, v in sd.items() if isinstance(v, torch.Tensor) and v.requires_grad and v.grad is not None}
    return y.detach().double().numpy(), grads, [x.grad.double().numpy() for x in xs]


GRAD_CASES = ["dsconv_k1", "dsconv_k2", "dsconv_k3", "doubleconv_eval", "doubleconv_mid_eval", "doubleconv_train", "down_eval", "up_eval_even", "up_eval_pad",
              "up_convt_even", "up_convt_pad", "up_convt_train",
              "cbam_k7_eval", "cbam_k3_eval", "cbam_k7_train", "outconv", "unet_12_1_k2_32", "unet_12_1_k2_train", "unet_3_5_k1_48"]


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("name", GRAD_CASES)
def test_gradients_match_cpu_autograd(name, train):
    c = CASES[name]
    kind = c["kind"]
    if kind in ("outconv", "dsconv") and train:
        pytest.skip("no mode dependence")
    sd_np, xs_np = case_tensors(name, np.float64)
    mod, prefix = build(c)
    load_np_state_dict(mod, {k: np.asarray(v, dtype=np.float32) if np.asarray(v).dtype != np.int64 else v for k, v in sd_np.items()}, prefix)
    mod = mod.cuda().train(train)
    xs = [dev(x).requires_grad_(True) for x in xs_np]
    y = mod(*xs)
    assert y.requires_grad, "output is not attached to the autograd tape"
    R = np.random.default_rng(77).uniform(-1, 1, tuple(y.shape))
    (y * dev(R)).sum().backward()
    torch.cuda.synchronize()
    y_ref, g_ref, gx_ref = _cpu_reference(kind, c, sd_np, xs_np, train, R)
    assert_close(y, y_ref, 3e-4, f"{name} forward (train={train})")
    # Full networks in train mode on these tiny frames normalise the bottleneck with batch statistics over
    # n = B*2*2 = 8 values: ill-conditioned -- the reference itself moves by ~1e-2 between fp32 and fp64
    # (measured on the CPU port: dx 1.2e-2, dW 9e-3 for unet_12_1_k2_32).  There the max-norm bound is
    # loosened and a relative L2 bound added; every per-block case keeps the tight bound.
    loose = kind == "unet" and train
    if loose:   # conditioning probe: how far does the reference algorithm itself move when run in fp32?
        _, g32, gx32 = _cpu_reference(kind, c, sd_np, xs_np, train, R, torch.float32)

        def _rel(a, b):
            return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))
        # one noise level for the whole case (per-tensor estimates of single-element tensors are a coin flip)
        noise = max([_rel(g32[k], g_ref[k]) for k in g_ref if np.abs(g_ref[k]).max() > 0] + [_rel(a, b) for a, b in zip(gx32, gx_ref)])

    def tol_for(ref, ref32):
        if not loose:
            return GRAD_TOL
        return max(GRAD_TOL, 10.0 * noise)      # within an order of magnitude of the reference's own fp32 noise

    def rel_l2(got, ref):
        got = got.detach().double().cpu().numpy()
        return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))

    for i, (x, gr) in enumerate(zip(xs, gx_ref)):
        assert x.grad is not None
        assert_close(x.grad, gr, tol_for(gr, gx32[i] if loose else None), f"{name} d/d(input) (train={train})")
        assert rel_l2(x.grad, gr) <= (5e-2 if loose else 1e-3)
    named = dict(mod.named_parameters())
    checked = 0
    gmax_all = max(float(np.abs(gr).max()) for gr in g_ref.values())
    for k, gr in g_ref.items():
        pk = k[len(prefix):] if prefix else k
        p = named[pk]
        assert p.grad is not None, f"no gradient for {pk}"
        if np.abs(gr).max() < 1e-6 * gmax_all:
            # mathematically zero gradients (a conv bias feeding a train-mode BatchNorm is cancelled by the mean
            # subtraction): both sides hold only summation noise -- bound it relative to the real gradients
            assert float(p.grad.abs().max()) <= (5e-3 if loose else 1e-3) * gmax_all, pk
        else:
            assert_close(p.grad, gr, tol_for(gr, g32[k] if loose else None), f"{name} d/d({pk}) (train={train})")
        checked += 1
    assert checked == len(named)


def test_training_step_reduces_loss_and_matches_cpu_one_step():
    """One Adam step on the reference's loss (regression_lightning.py:57-65: mse(sum)/B) moves the parameters the same
    way on the GPU path and on the CPU port."""
    name = "unet_12_1_k2_train"
    sd_np, xs_np = case_tensors(name, np.float64)
    tgt = np.random.default_rng(5).uniform(0, 1, (xs_np[0].shape[0], 32, 32))
    model = load_np_state_dict(S.SmaAt_UNet(12, 1, kernels_per_layer=2), {k: (np.asarray(v, np.float32) if np.asarray(v).dtype != np.int64 else v)
                                                                          for k, v in sd_np.items()}).cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    x, t = dev(xs_np[0]), dev(tgt)
    losses = []
    for _ in range(3):
        opt.zero_grad()
        pred = model(x)
        loss = torch.nn.functional.mse_loss(pred.squeeze(1), t, reduction="sum") / x.shape[0]
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[2] < losses[0]
    # CPU port, same 1st-step loss
    sd = TP.to_torch_sd(sd_np, torch.float64)
    with torch.no_grad():
        p0 = TP.smaat_unet_forward(torch.from_numpy(xs_np[0]), sd, True)
    l0 = float(torch.nn.functional.mse_loss(p0.squeeze(1), torch.from_numpy(tgt), reduction="sum") / x.shape[0])
    assert abs(losses[0] - l0) <= 1e-3 * abs(l0)


# B, C0, C1, H, W, k, prologue  (W % 4 == 0 and k <= 2 take the TMA kernels, the rest the LDS-tiled ones)
DW_BWD_CASES = [
    (2, 5, 0, 9, 11, 1, False),
    (2, 6, 0, 12, 8, 2, True),
    (1, 4, 0, 7, 5, 3, False),
    (2, 3, 5, 16, 20, 2, False),
    (1, 8, 0, 18, 18, 2, True),
    (2, 4, 0, 36, 36, 2, True),
    (1, 3, 2, 72, 72, 1, False),
    (1, 2, 2, 144, 144, 2, True),
    (1, 3, 0, 288, 288, 2, False),
    (1, 2, 0, 100, 148, 2, True),
]


@pytest.mark.parametrize("case", DW_BWD_CASES)
def test_dw3x3_backward_kernels_match_cpu_autograd(case):
    """smaat_dw3x3_bwd_input / _bwd_weight vs float64 autograd of conv2d(groups=Cin) (reference layers.py:38-44)."""
    from smaat_unet_b200 import functional as Fn
    B, C0, C1, H, W, k, pro = case
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + k)
    Cin = C0 + C1
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Cin * k, 1, 3, 3, generator=g, dtype=torch.float64)
    dd = torch.randn(B, Cin * k, H, W, generator=g, dtype=torch.float64)
    sc = torch.rand(Cin, generator=g, dtype=torch.float64) + 0.5
    sh = torch.randn(Cin, generator=g, dtype=torch.float64) * 0.3
    a = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    b = torch.zeros(Cin * k, dtype=torch.float64, requires_grad=True)
    inp = torch.relu(a * sc[None, :, None, None] + sh[None, :, None, None]) if pro else a
    y = torch.nn.functional.conv2d(inp, wr, b, padding=1, groups=Cin)
    y.backward(dd)
    # the kernels return d(loss)/d(conv input); with the prologue that is the gradient w.r.t. relu(BN(x))
    if pro:
        a2 = inp.detach().clone().requires_grad_(True)
        torch.nn.functional.conv2d(a2, w, None, padding=1, groups=Cin).backward(dd)
        want_dx = a2.grad
    else:
        want_dx = a.grad
    f32 = lambda t: t.to(torch.float32).cuda().contiguous()
    x0 = f32(x[:, :C0])
    x1 = f32(x[:, C0:]) if C1 else None
    dW = torch.zeros(Cin * k, 1, 3, 3, device="cuda")
    db = torch.zeros(Cin * k, device="cuda")
    dx0, dx1 = Fn.dw_bwd(f32(dd), f32(w), x0, x1, f32(sc) if pro else None, f32(sh) if pro else None, k, dW, db)
    got_dx = torch.cat([dx0, dx1], 1) if C1 else dx0
    assert_close(got_dx, want_dx.numpy(), 2e-5, f"dw3x3_bwd_input {case}")
    assert_close(dW, wr.grad.numpy(), 1e-4, f"dw3x3_bwd_weight {case}")
    assert_close(db, b.grad.numpy(), 1e-4, f"dw3x3_bwd_bias {case}")


@pytest.mark.parametrize("use_graph", [False, True])
def test_train_session_matches_eager_steps(use_graph):
    """TrainSession (flat gradient bucket, fused loss+metrics, optional CUDA graphs) reproduces plain eager steps of
    the same modules with torch's mse_loss + Adam, and leaves the caller's model untouched by its warm-up.
    Training this net on a tiny batch is chaotic (BatchNorm over a handful of samples in the deep layers, Adam turning
    rounding-noise gradients into +-lr moves: measured eager-vs-graph loss drift 1e-7, 1e-4, 1e-3 over steps 2..4), so the
    first step is compared tightly and the following ones on the scale that still separates "updated" from "not"."""
    from smaat_unet_b200.train import TrainSession
    torch.manual_seed(3)
    B, S_ = 2, 64
    m1 = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
    m2 = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
    m2.load_state_dict(m1.state_dict())
    xs = [torch.rand(B, 12, S_, S_, device="cuda") for _ in range(3)]
    ys = [torch.rand(B, S_, S_, device="cuda") for _ in range(3)]
    sess = TrainSession(m1, B, (12, S_, S_), lr=1e-3, use_graph=use_graph)
    for k, v in m2.state_dict().items():                      # warm-up steps were rolled back
        assert torch.equal(v, m1.state_dict()[k]), k
    opt = torch.optim.Adam(m2.parameters(), lr=1e-3)
    tols = [1e-5, 2e-3, 2e-2]
    for i, (x, y) in enumerate(zip(xs, ys)):
        l1 = float(sess.step(x, y))
        opt.zero_grad(set_to_none=True)
        l2 = torch.nn.functional.mse_loss(m2(x).squeeze(1), y, reduction="sum") / B
        l2.backward()
        opt.step()
        assert abs(l1 - float(l2)) <= tols[i] * abs(float(l2)), (i, l1, float(l2))
        if i == 0:   # after ONE Adam step every parameter has moved by at most lr (twice that apart, for noise-sign gradients)
            for (k, a), b in zip(m1.state_dict().items(), m2.state_dict().values()):
                if a.dtype == torch.int64:
                    assert torch.equal(a, b), k
                else:
                    assert (a - b).abs().max().item() <= 2.5e-3, k
    assert int(sess.metrics.total_samples) == 3 * B
    assert int(m1.state_dict()["inc.double_conv.1.num_batches_tracked"]) == 3



def test_train_session_fed_by_pinned_loader_matches_direct_batches():
    """PinnedBatchLoader (pinned ring, background fill, guard events) -> TrainSession gives the same losses as feeding the
    same samples as device tensors."""
    from smaat_unet_b200 import data as D
    from smaat_unet_b200.train import TrainSession
    rng = np.random.default_rng(7)
    arr = rng.random((12, 13, 32, 32), dtype=np.float32)            # 12 samples, 12 inputs + target
    ds = D.precipitation_maps_oversampled_shard(arr, 12, 1)
    torch.manual_seed(5)
    m1 = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
    m2 = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
    m2.load_state_dict(m1.state_dict())
    s1 = TrainSession(m1, 4, (12, 32, 32), use_graph=True)
    s2 = TrainSession(m2, 4, (12, 32, 32), use_graph=True)
    loader = D.PinnedBatchLoader(ds, batch_size=4, ring=2)
    l1, l2 = [], []
    for bi, (x, y) in enumerate(loader):
        assert x.is_pinned() and y.is_pinned()
        l1.append(s1.step(x, y).clone())
        loader.guard(s1.last_h2d_event())
        xb = torch.from_numpy(arr[bi * 4:(bi + 1) * 4, :12]).cuda()
        yb = torch.from_numpy(arr[bi * 4:(bi + 1) * 4, -1]).cuda()
        l2.append(s2.step(xb, yb).clone())
    torch.cuda.synchronize()
    assert len(l1) == 3
    assert abs(float(l1[0]) - float(l2[0])) <= 1e-5 * abs(float(l2[0]))      # same batch, same weights
    for a, b in zip(l1[1:], l2[1:]):                                           # later steps: chaotic drift bound (see above)
        assert abs(float(a) - float(b)) <= 2e-2 * abs(float(b))


def test_flat_adam_kernel_matches_torch_adam():
    """smaat_adam_step (one kernel over a flat bucket, device-side lr and step count) vs torch.optim.Adam over 6 steps,
    with a learning-rate change in the middle (ReduceLROnPlateau factor 0.1, regression_lightning.py:49-55)."""
    from smaat_unet_b200 import _lib
    from smaat_unet_b200.ops import _stream
    torch.manual_seed(11)
    n = 4096 + 64
    p0 = torch.randn(n, device="cuda")
    p_ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([p_ref], lr=1e-3)
    p, m, v = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    lr, step = torch.full((), 1e-3, device="cuda"), torch.zeros((), device="cuda")
    lib = _lib.load()
    for it in range(6):
        g = torch.randn(n, device="cuda") * (10.0 ** (it - 3))          # a few orders of magnitude
        if it == 3:
            opt.param_groups[0]["lr"] = 1e-4
            lr.fill_(1e-4)
        p_ref.grad = g.clone()
        opt.step()
        _lib.check(lib.smaat_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, lr.data_ptr(), step.data_ptr(),
                                       0.9, 0.999, 1e-8, _stream()), "smaat_adam_step")
        torch.cuda.synchronize()
        assert float(step) == it + 1
        assert (p - p_ref.detach()).abs().max().item() <= 2e-7 * max(1.0, p_ref.detach().abs().max().item()), it
    st = opt.state[p_ref]
    assert_close(m, st["exp_avg"].double().cpu().numpy(), 1e-6, "exp_avg")
    assert_close(v, st["exp_avg_sq"].double().cpu().numpy(), 1e-6, "exp_avg_sq")


def test_train_session_lr_lives_on_the_device_and_state_dict_round_trips():
    """ADVICE r1: a captured step must follow learning-rate changes; the optimizer state must be exportable in
    torch.optim.Adam's schema (train_SmaAtUNet.py:85-96 checkpoints it)."""
    from smaat_unet_b200.train import TrainSession
    torch.manual_seed(5)
    m = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda()
    sess = TrainSession(m, 2, (12, 32, 32), lr=1e-3, use_graph=True)
    x, y = torch.rand(2, 12, 32, 32, device="cuda"), torch.rand(2, 32, 32, device="cuda")
    w = m.outc.conv.weight
    assert w.data_ptr() >= sess.flat_param.data_ptr() and w.grad.data_ptr() >= sess.flat_grad.data_ptr()
    before = w.detach().clone()
    sess.step(x, y)
    d1 = (w.detach() - before).abs().max().item()
    assert 0 < d1 <= 1.01e-3                       # first Adam step moves every weight by ~lr
    sess.set_lr(0.0)
    mid = w.detach().clone()
    sess.step(x, y)                                # same captured graph, lr = 0: nothing may move
    assert torch.equal(w.detach(), mid)
    sess.set_lr(1e-5)
    sess.step(x, y)
    d3 = (w.detach() - mid).abs().max().item()
    assert 0 < d3 <= 1.5e-5
    sd = sess.optimizer_state_dict()
    assert len(sd["state"]) == len(list(m.parameters())) and float(sd["state"][0]["step"]) == 3
    ref = torch.optim.Adam(m.parameters(), lr=1e-3)
    ref.load_state_dict(sd)                        # torch accepts the schema
    assert abs(ref.param_groups[0]["lr"] - 1e-5) < 1e-12
    m2 = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda()
    m2.load_state_dict(m.state_dict())
    sess2 = TrainSession(m2, 2, (12, 32, 32), lr=1e-3, use_graph=False)
    sess2.load_optimizer_state_dict(sd)
    assert torch.equal(sess2.exp_avg_sq, sess.exp_avg_sq) and float(sess2.opt_step) == 3 and abs(sess2.get_lr() - 1e-5) < 1e-12
    sess.close()
    sess2.close()


def test_two_phase_backward_is_verified_not_assumed():
    """The decoder-first gradient split (train.py) is taken for SmaAt-UNet and refused -- by measurement -- for a net whose
    decoder also reads an un-attended encoder map (UNetDSAttention4CBAMs, unet_precip_regression_lightning.py:193-208);
    both must produce the gradients of a plain backward."""
    from smaat_unet_b200.train import TrainSession
    from tests.test_gpu_api_paths import RefOrderNet
    for n_cbams, expect_split in ((5, True), (4, False)):
        torch.manual_seed(7)
        m = RefOrderNet(12, 1, 2, n_cbams).cuda()
        m_ref = RefOrderNet(12, 1, 2, n_cbams).cuda().train()
        m_ref.load_state_dict(m.state_dict())
        sess = TrainSession(m, 2, (12, 32, 32), lr=0.0, use_graph=True)       # lr 0: weights stay comparable
        assert (sess._split is not None) == expect_split, n_cbams
        x, y = torch.rand(2, 12, 32, 32, device="cuda"), torch.rand(2, 32, 32, device="cuda")
        sess.step(x, y)
        loss = torch.nn.functional.mse_loss(m_ref(x).squeeze(1), y, reduction="sum") / 2
        loss.backward()
        torch.cuda.synchronize()
        gmax = max(float(p.grad.abs().max()) for p in m_ref.parameters())
        for (k, p), q in zip(m.named_parameters(), m_ref.parameters()):
            assert (p.grad - q.grad).abs().max().item() <= 2e-3 * gmax, (n_cbams, k)
        sess.close()


def test_recompute_depthwise_matches_and_saves_memory():
    """functional.set_recompute_depthwise drops the depthwise results after the forward and re-runs the same kernel in the
    backward: gradients agree to the run-to-run noise of the atomically merged reductions (same kernel, same inputs), peak memory of a forward+backward goes down."""
    from smaat_unet_b200 import functional as Fn
    torch.manual_seed(5)
    m = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
    x = torch.rand(4, 12, 96, 96, device="cuda")

    def run(flag):
        old = Fn.set_recompute_depthwise(flag)
        try:
            for p in m.parameters():
                p.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            y = m(x)
            held = torch.cuda.memory_allocated() - base      # activations the backward keeps alive
            y.square().sum().backward()
            torch.cuda.synchronize()
            return [p.grad.clone() for p in m.parameters()], held
        finally:
            Fn.set_recompute_depthwise(old)

    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g0, held0 = run(False)
    m.load_state_dict(sd)                                     # same running statistics for every pass
    g0b, _ = run(False)                                       # run-to-run noise of the fp32-atomic reductions (split-K merges, dw wgrad)
    m.load_state_dict(sd)
    g1, held1 = run(True)
    gmax = max(a.abs().max().item() for a in g0)
    for a, a2, b, (n, _) in zip(g0, g0b, g1, m.named_parameters()):
        noise = (a - a2).abs().max().item()
        assert (a - b).abs().max().item() <= 10 * noise + 1e-6 * gmax, (n, noise, gmax)
    assert held1 < 0.75 * held0, (held0, held1)
    assert not Fn.get_recompute_depthwise()
