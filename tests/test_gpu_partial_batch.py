"""-m gpu: requests and training steps with fewer rows than a session's batch.  InferenceSession runs the smallest captured
size that holds a request (``batch_sizes``) and returns only its rows; TrainSession steps exactly the rows it is given,
from a captured graph of that size or eagerly."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import smaat_unet_b200 as S
from smaat_unet_b200 import data as D
from smaat_unet_b200.engine import InferenceSession
from smaat_unet_b200.segmentation import IoU
from smaat_unet_b200.train import TrainSession
from tests._util import NET_TOL

pytestmark = pytest.mark.gpu

B, HW = 8, 32
MODELS = {
    "smaat_12_1": (lambda: S.SmaAt_UNet(12, 1), 12),
    "smaat_3_21": (lambda: S.SmaAt_UNet(3, 21), 3),
    "unet_12_1": (lambda: S.UNet(12, 1), 12),
}


def make(name, seed=0):
    """Default initialisation with random BatchNorm statistics and affines, on the GPU in eval mode."""
    torch.manual_seed(seed)
    m = MODELS[name][0]()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.running_mean.uniform_(-0.2, 0.2, generator=g)
                mod.running_var.uniform_(0.5, 1.5, generator=g)
                mod.weight.uniform_(0.8, 1.2, generator=g)
                mod.bias.uniform_(-0.1, 0.1, generator=g)
    return m.cuda().eval()


def inputs(n, c, seed, hw=HW):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(n, c, hw, hw, device="cuda", generator=g)


def test_one_sample_is_not_broadcast_and_bad_requests_raise():
    m = make("smaat_12_1")
    sess = InferenceSession(m, B, (12, HW, HW))
    x = inputs(B, 12, 1)
    full = sess.forward(x).clone()
    one = sess.forward(x[:1].clone()).clone()
    assert tuple(one.shape) == (1, 1, HW, HW)
    assert torch.equal(one, full[:1])
    other = inputs(B, 12, 2)
    other[0] = x[0]                                    # the same sample among different ones
    assert torch.equal(sess.forward(other)[:1], one)
    for bad in (torch.zeros(0, 12, HW, HW, device="cuda"), torch.zeros(B + 1, 12, HW, HW, device="cuda"),
                torch.zeros(1, 12, HW, HW // 2, device="cuda"), torch.zeros(12, HW, HW, device="cuda")):
        with pytest.raises(ValueError):
            sess.forward(bad)
        with pytest.raises(ValueError):
            sess.submit(bad.cpu().pin_memory())
    assert not sess._pending


CASES = [("smaat_12_1", "logits", True), ("smaat_12_1", "logits", False), ("smaat_3_21", "classes", True),
         ("smaat_3_21", "probs", True), ("smaat_3_21", "probs", False), ("unet_12_1", "logits", True)]


@pytest.mark.parametrize("name,output,fusions", CASES)
def test_every_size_returns_the_full_batch_rows_bitwise(name, output, fusions):
    m = make(name)
    C = MODELS[name][1]
    plain = InferenceSession(m, B, (C, HW, HW), output=output, serving_fusions=fusions)
    sess = InferenceSession(m, B, (C, HW, HW), output=output, serving_fusions=fusions, batch_sizes=(1, 3))
    assert sess.sizes == (1, 3, B) and plain.sizes == (B,)
    assert sess.out_shape == plain.out_shape and sess.launches_per_forward == plain.launches_per_forward
    assert sess.h2d_bytes_per_step == plain.h2d_bytes_per_step and sess.d2h_bytes_per_step == plain.d2h_bytes_per_step
    x = inputs(B, C, 3)
    ref = plain.forward(x).clone()
    assert torch.equal(sess.forward(x), ref)
    for n in range(1, B + 1):
        assert sess.size_for(n) == (1 if n == 1 else 3 if n <= 3 else B)
        # the last n samples: each lands on another row than in the reference batch
        got = sess.forward(x[B - n:].clone())
        assert got.shape[0] == n
        assert torch.equal(got, ref[B - n:]), n
        sess.submit(x[B - n:].cpu().pin_memory())
        host = sess.collect()
        assert host.shape[0] == n and host.is_pinned()
        assert torch.equal(host, ref[B - n:].cpu()), n


def test_interleaved_sizes_match_each_size_alone():
    m = make("smaat_12_1")
    sess = InferenceSession(m, B, (12, HW, HW), batch_sizes=(1, 3))
    order = [8, 1, 3, 8, 3, 1]
    xs = [inputs(n, 12, 10 + i) for i, n in enumerate(order)]
    live, got = {}, []
    for n, x in zip(order, xs):
        live[n] = sess.forward(x)                       # views of each size's static output
        got.append(live[n].clone())
    torch.cuda.synchronize()
    for n in (8, 3, 1):                                 # a size's output survives the other sizes' replays
        last = max(i for i, k in enumerate(order) if k == n)
        assert torch.equal(live[n], got[last]), n
    solo = InferenceSession(m, B, (12, HW, HW), batch_sizes=(1, 3))
    for n in (8, 3, 1):                                 # each size replayed alone, one size after the other
        for i, k in enumerate(order):
            if k == n:
                assert torch.equal(solo.forward(xs[i]), got[i]), (i, n)


@pytest.mark.parametrize("first", [1, 3, 8])
def test_a_live_output_survives_every_other_size(first):
    """A size's returned view is left alone by requests of every other size, whichever of them was captured first."""
    m = make("smaat_12_1")
    sess = InferenceSession(m, B, (12, HW, HW), batch_sizes=(1, 3))
    view = sess.forward(inputs(first, 12, 20))
    kept = view.clone()
    for i, n in enumerate(k for k in (8, 3, 1, 8, 1, 3) if k != first):
        sess.forward(inputs(n, 12, 30 + i))               # different inputs, so a clobbered view would change
        torch.cuda.synchronize()
        assert torch.equal(view, kept), (first, n)


def test_sessions_build_while_unreachable_cuda_objects_await_collection():
    """Python's cyclic collector may run at any allocation.  Unreachable cycles that own pinned host memory and CUDA events
    (as earlier sessions may) must not be collected inside a capture, where releasing them would invalidate it."""
    import gc

    class Cycle:
        def __init__(self):
            self.me, self.pinned, self.event = self, torch.empty(1 << 16).pin_memory(), torch.cuda.Event()
            self.event.record()

    m = make("smaat_12_1")
    x = inputs(B, 12, 5)
    want = InferenceSession(m, B, (12, HW, HW)).forward(x).clone()
    old = gc.get_threshold()
    try:
        for _ in range(8):
            Cycle()
        gc.set_threshold(1)                           # a collection at nearly every allocation
        sess = InferenceSession(m, B, (12, HW, HW), batch_sizes=(3,))
        ts = TrainSession(S.SmaAt_UNet(12, 1).cuda(), 2, (12, HW, HW), batch_sizes=(1,), warmup=1)
        for _ in range(8):
            Cycle()
    finally:
        gc.set_threshold(*old)
    assert torch.equal(sess.forward(x), want) and torch.equal(sess.forward(x[:3]), want[:3])
    ts.step(x[:1], torch.rand(1, HW, HW, device="cuda"))
    torch.cuda.synchronize()
    ts.close()


def test_partial_request_at_the_benchmark_shape():
    """SmaAt_UNet(12, 1), k = 2, B = 32, 12x288x288 (bench.py's workload) with a 5-sample size: bitwise the full session's
    rows, and within the full-network tolerance of the float64 CPU port."""
    from oracle import torch_port as TP
    torch.manual_seed(0)
    m = S.SmaAt_UNet(12, 1, kernels_per_layer=2)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
                mod.weight.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
    m = m.cuda().eval()
    sess = InferenceSession(m, 32, (12, 288, 288), batch_sizes=(5,))
    x = inputs(32, 12, 4, hw=288)
    full = sess.forward(x).clone()
    part = sess.forward(x[:5].clone()).clone()
    assert tuple(part.shape) == (5, 1, 288, 288)
    assert torch.equal(part, full[:5])
    sd = {k: (v.detach().cpu().double() if v.is_floating_point() else v.detach().cpu()) for k, v in m.state_dict().items()}
    fr = [0, 4]
    with torch.no_grad():
        ref = TP.smaat_unet_forward(x[fr].cpu().double(), sd).numpy()
    got = part[fr].double().cpu().numpy()
    err = float(np.abs(got - ref).max() / np.abs(ref).max())
    assert err <= NET_TOL[S.get_pointwise_mode()], err


# ---------------------------------------------------------------------------------------------------------- training
TB, THW = 4, 64


def _flat(ts):
    return torch.cat([t.detach().reshape(-1).double() for t in ts])


def _rel_l2(a, b):
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


@pytest.mark.parametrize("loss", ["mse", "cross_entropy"])
def test_train_tail_steps_match_eager_adam(loss):
    """Full step, 2-sample step (not declared: eager), 3-sample step (captured), full step against the eager modules and
    torch.optim.Adam; the captured steps after the eager one show that it leaves the graphs intact.  Training this net on a
    handful of samples is chaotic (test_gpu_train.py), so before every step the reference takes the session's parameters,
    buffers and Adam state, and each step is compared as a first step: the loss tightly, gradients and Adam moments within
    the full network's train-mode relative L2 bound, running statistics within forward noise.  The parameters must have
    moved by exactly one Adam update from the session's own moments and step count.  The metric totals of the whole
    sequence agree as well."""
    K = 1 if loss == "mse" else 4
    torch.manual_seed(3)
    m1 = S.SmaAt_UNet(12, K, kernels_per_layer=2).cuda().train()
    m2 = S.SmaAt_UNet(12, K, kernels_per_layer=2).cuda().train()
    m2.load_state_dict(m1.state_dict())
    before = {k: v.clone() for k, v in m1.state_dict().items()}
    sess = TrainSession(m1, TB, (12, THW, THW), lr=1e-3, loss=loss, batch_sizes=(3,))
    for k, v in m1.state_dict().items():                  # building the session leaves the model as it was
        assert torch.equal(v, before[k]), k
    assert sess.sizes == (3, TB) and set(sess._size_graphs) == {3, TB}      # 2 has no graph: its step runs eagerly
    ref_metric = S.PrecipitationMetrics() if K == 1 else IoU(K)
    g = torch.Generator(device="cuda").manual_seed(9)
    lr, (b1, b2), eps = 1e-3, sess.betas, sess.eps
    for i, n in enumerate([TB, 2, 3, TB]):
        x = torch.rand(n, 12, THW, THW, device="cuda", generator=g)
        y = torch.rand(n, THW, THW, device="cuda", generator=g) if K == 1 else \
            torch.randint(K, (n, THW, THW), device="cuda", generator=g)
        m2.load_state_dict(m1.state_dict())
        opt = torch.optim.Adam(m2.parameters(), lr=1e-3)
        if i:
            sd = sess.optimizer_state_dict()
            for st in sd["state"].values():
                st["step"] = st["step"].cpu()          # torch.optim.Adam keeps a non-capturable step count on the host
            opt.load_state_dict(sd)
        p_before = _flat(m1.parameters())
        l1 = float(sess.step(x, y))
        opt.zero_grad(set_to_none=True)
        pred = m2(x)
        if K == 1:
            l2 = nn.functional.mse_loss(pred.squeeze(1), y, reduction="sum") / n
            ref_metric.update(pred.detach(), y)
        else:
            l2 = nn.functional.cross_entropy(pred, y)
            ref_metric.add(pred.detach(), y)
        l2.backward()
        opt.step()
        torch.cuda.synchronize()
        assert abs(l1 - float(l2)) <= 1e-5 * abs(float(l2)), (i, n, l1, float(l2))
        ps1, ps2 = list(m1.parameters()), list(m2.parameters())
        assert _rel_l2(_flat(p.grad for p in ps1), _flat(p.grad for p in ps2)) <= 5e-2, (i, n)
        st = [opt.state[p] for p in ps2]
        mine = list(sess.optimizer_state_dict()["state"].values())
        for key in ("exp_avg", "exp_avg_sq"):
            assert _rel_l2(_flat(s[key] for s in mine), _flat(s[key] for s in st)) <= 5e-2, (i, n, key)
        t = i + 1
        assert float(sess.opt_step) == t == float(st[0]["step"])
        m_hat = _flat(s["exp_avg"] for s in mine) / (1 - b1 ** t)
        v_hat = _flat(s["exp_avg_sq"] for s in mine) / (1 - b2 ** t)
        want_p = p_before - lr * m_hat / (v_hat.sqrt() + eps)
        assert (_flat(m1.parameters()) - want_p).abs().max().item() <= 1e-6, (i, n)
        for (k, a), b in zip(m1.state_dict().items(), m2.state_dict().values()):
            if a.dtype == torch.int64:
                assert torch.equal(a, b), (i, k)
            elif k.endswith(("running_mean", "running_var")):
                assert (a - b).abs().max().item() <= 1e-4 * max(1.0, b.abs().max().item()), (i, k)
    assert int(m1.state_dict()["inc.double_conv.1.num_batches_tracked"]) == 4
    got, want = sess.metrics.totals_snapshot().double(), ref_metric.totals_snapshot().double()
    if K == 1:       # total_loss, total_loss_denorm, total_samples, total_pixels, tn, fp, fn, tp, skipped_batches
        assert int(got[2]) == int(want[2]) == 13 and int(got[3]) == int(want[3]) and int(got[8]) == int(want[8]) == 0
        assert torch.allclose(got[:2], want[:2], rtol=1e-5, atol=0)
        assert (got[4:8] - want[4:8]).abs().max().item() <= 1e-3 * float(want[3])
    else:            # confusion matrix
        assert float(got.sum()) == float(want.sum()) == 13 * THW * THW
        assert (got - want).abs().max().item() <= 1e-3 * float(want.sum())
    sess.close()


def test_epoch_with_tail_matches_eager_metrics():
    """N = 2B + 3 samples through PinnedBatchLoader(drop_last=False) into a session with the tail size: the threshold
    counts are exactly those of the eager forward over all N samples at once.  The MSE totals add one mean per batch
    (precipitation_metrics.py:61-64), so they are compared with eager forwards over the same batches."""
    Bt, N = 4, 11
    rng = np.random.default_rng(7)
    arr = rng.random((N, 13, HW, HW), dtype=np.float32)            # 12 inputs + target per sample
    ds = D.precipitation_maps_oversampled_shard(arr, 12, 1)
    m = make("smaat_12_1")
    want, want_mse = S.PrecipitationMetrics(), S.PrecipitationMetrics()
    with torch.no_grad():
        want.update(m(torch.from_numpy(arr[:, :12]).cuda()), torch.from_numpy(arr[:, -1]).cuda())
        for lo in range(0, N, Bt):
            want_mse.update(m(torch.from_numpy(arr[lo:lo + Bt, :12]).cuda()), torch.from_numpy(arr[lo:lo + Bt, -1]).cuda())
    sess = InferenceSession(m, Bt, (12, HW, HW), batch_sizes=(N % Bt,))
    got = S.PrecipitationMetrics()
    loader = D.PinnedBatchLoader(ds, batch_size=Bt, drop_last=False, ring=2)
    sizes = []
    for x, y in loader:
        sizes.append(x.shape[0])
        got.update(sess.forward(x.cuda()), y.cuda())
    assert sizes == [Bt, Bt, N % Bt]
    a, b = got.totals_snapshot().cpu(), want.totals_snapshot().cpu()
    assert torch.equal(a[2:], b[2:]), (a, b)          # samples, pixels, TN, FP, FN, TP, skipped batches
    assert torch.allclose(a[:2], want_mse.totals_snapshot().cpu()[:2], rtol=1e-6, atol=0)
    assert abs(float(got.compute()["mse"]) - float(want_mse.compute()["mse"])) <= 1e-6 * abs(float(want_mse.compute()["mse"]))
