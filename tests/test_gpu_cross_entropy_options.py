"""-m gpu: cross-entropy with class weights, label smoothing, probability / one-hot targets and reduction="none"
(smaat_cross_entropy_fwd), and one-hot targets in IoU / ConfusionMatrix (smaat_onehot_classes).  Loss, per-pixel loss and
gradient against float64 F.cross_entropy + autograd at the shapes of test_gpu_segmentation.py's CE_CASES and at the training
shape; bitwise agreement with smaat_ce_fwd when no option is set; the edge cases of include/smaat_b200.h; IoU against the
reference's own outputs on one-hot targets (tests/golden/seg_onehot.npz); TrainSession with a weighted, smoothed loss
against eager nn.CrossEntropyLoss + Adam steps."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle.make_golden_seg import CONFIGS, K as GK, N_BATCHES
from smaat_unet_b200 import _lib
from smaat_unet_b200.segmentation import ce_forward, ce_forward_opts
from tests.test_gpu_segmentation import CE_CASES, _case, _place

pytestmark = pytest.mark.gpu
SEG = np.load(os.path.join(os.path.dirname(__file__), "golden", "seg_metrics.npz"))
ONEHOT = np.load(os.path.join(os.path.dirname(__file__), "golden", "seg_onehot.npz"))

TRAIN_CASE = (32, 8, 288, 288, 6.0, False, -100)


def _weight(kind, K, seed):
    if kind == "none":
        return None
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(K, generator=g) * 2 + 0.25
    if kind == "zeros":
        w[torch.randperm(K, generator=g)[: max(1, K // 4)]] = 0.0
    return w


def _prob_target(lg, t, seed):
    """float32 probabilities shaped like the logits: softmax rows, a third of them exact one-hot rows of `t`."""
    g = torch.Generator().manual_seed(seed)
    K = lg.shape[1]
    q = torch.softmax(torch.randn(lg.shape, generator=g) * 2, dim=1)
    hot = F.one_hot(t.clamp(0, K - 1), K).movedim(-1, 1).float()
    pick = (torch.rand((lg.shape[0], 1) + tuple(lg.shape[2:]), generator=g) < 0.33).float()
    return q * (1 - pick) + hot * pick


def _row_checks(q):
    """(valid, argmax) of each target row as the kernels decide: values in [0, 1] and an fp32 sum in class order == 1."""
    s = torch.zeros_like(q[:, 0])
    for c in range(q.shape[1]):
        s = s + q[:, c]
    valid = ((q >= 0) & (q <= 1)).all(1) & (s == 1.0)
    return valid, q.argmax(1)


def _targets(kind, lg, t, ig):
    """(device target, float64 reference target, ignore_index for both, mask of counted pixels, confusion rows, valid rows)."""
    K = lg.shape[1]
    if kind == "index":
        keep = t != ig
        return t.cuda(), t, ig, keep, t, keep
    fill = torch.where(t == ig, torch.zeros_like(t), t)
    q = _prob_target(lg, fill, seed=int(t.numel()) % 1000) if kind == "prob" else F.one_hot(fill, K).movedim(-1, 1).float()
    valid, rows = _row_checks(q)
    return q.cuda(), q.double(), -100, torch.ones_like(valid), rows, valid


def _check_case(case, wkind, eps, reduction, tkind):
    B, K, H, W, spread, mis, ig = case
    lg, t = _case(B, K, H, W, spread, seed=K * 100 + H, ignore=(ig,))
    tgt, tref, ign, keep, rows, valid = _targets(tkind, lg, t, ig)
    w = _weight(wkind, K, seed=K + H)
    x = _place(lg, mis).detach().requires_grad_(True)          # detach keeps the (mis)aligned storage offset
    iou = S.IoU(K)
    loss = S.ce_step(x, tgt, iou, ign, reduction, weight=None if w is None else w.cuda(), label_smoothing=eps)
    up = torch.rand((B, H, W), generator=torch.Generator().manual_seed(5)) + 0.5 if reduction == "none" else torch.tensor(1.7)
    l64 = lg.double().requires_grad_(True)
    ref = F.cross_entropy(l64, tref, weight=None if w is None else w.double(), ignore_index=ign, reduction=reduction,
                          label_smoothing=eps)
    if reduction == "none":
        loss.backward(up.cuda())
        ref.backward(up.double())
    else:
        (loss * 1.7).backward()
        (ref * 1.7).backward()
    torch.cuda.synchronize()
    tag = (case, wkind, eps, reduction, tkind)
    if reduction == "none":
        got = loss.detach().cpu().double()
        assert got.shape == ref.shape, tag
        assert (got - ref.detach()).abs().max().item() <= 2e-6 * ref.detach().abs().max().item(), tag
        assert torch.all(got[~keep] == 0), tag
    else:
        assert loss.dtype == torch.float32 and loss.dim() == 0
        assert abs(float(loss) - float(ref)) <= 2e-6 * abs(float(ref)), (tag, float(loss), float(ref))
    gref, got_g = l64.grad, x.grad.cpu().double()
    assert (got_g - gref).abs().max().item() <= 2e-6 * gref.abs().max().item(), tag
    assert torch.all(got_g.movedim(1, -1)[~keep] == 0), tag          # exactly 0 on ignored pixels
    am = lg.argmax(1)
    ok = keep & valid
    want = torch.bincount(rows[ok] * K + am[ok], minlength=K * K).view(K, K).numpy()
    counts, invalid = iou.conf_metric.counts()
    assert np.array_equal(counts, want) and invalid == int((keep & ~valid).sum()), tag


@pytest.mark.parametrize("tkind", ["index", "prob", "onehot"])
@pytest.mark.parametrize("reduction", ["mean", "sum", "none"])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("wkind", ["none", "positive", "zeros"])
@pytest.mark.parametrize("case", CE_CASES)
def test_cross_entropy_options_match_float64(case, wkind, eps, reduction, tkind):
    _check_case(case, wkind, eps, reduction, tkind)


@pytest.mark.parametrize("wkind, eps, reduction, tkind", [
    ("positive", 0.1, "mean", "index"), ("zeros", 0.0, "sum", "index"), ("zeros", 0.1, "none", "index"),
    ("positive", 0.1, "mean", "prob"), ("none", 0.0, "none", "onehot")])
def test_cross_entropy_options_at_training_shape(wkind, eps, reduction, tkind):
    _check_case(TRAIN_CASE, wkind, eps, reduction, tkind)


@pytest.mark.parametrize("case", CE_CASES + [TRAIN_CASE])
def test_no_options_is_bitwise_the_plain_kernel(case):
    B, K, H, W, spread, mis, ig = case
    lg, t = _case(B, K, H, W, spread, seed=K * 100 + H, ignore=(ig,))
    x, tc = _place(lg, mis), t.cuda()
    c1 = torch.zeros(K, K, dtype=torch.int64, device="cuda")
    c2 = torch.zeros_like(c1)
    a1, d1 = ce_forward(x, tc, ig, True, want_grad=True, conf=c1)
    a2, _, d2 = ce_forward_opts(x, tc, torch.ones(K, device="cuda"), 0.0, ig, True, want_grad=True, conf=c2)
    torch.cuda.synchronize()
    assert torch.equal(d1, d2) and torch.equal(c1, c2)
    assert abs(float(a1[0]) - float(a2[0])) <= 1e-12 * abs(float(a1[0]))
    assert float(a1[1]) == float(a2[1]) == float(a2[3]) and float(a1[2]) == float(a2[2]) == 0


def test_invalid_labels_with_options():
    K = 8
    lg, t = _case(2, K, 12, 16, 4.0, seed=3, ignore=(-100,), invalid=(K, -7, 1000))
    w = _weight("positive", K, 1).cuda()
    bad = (t != -100) & ((t < 0) | (t >= K))
    ok = ~bad & (t != -100)
    x = lg.cuda().requires_grad_(True)
    iou = S.IoU(K)
    loss = S.ce_step(x, t.cuda(), iou, weight=w, label_smoothing=0.1)
    loss.backward()
    torch.cuda.synchronize()
    assert bad.any() and math.isnan(float(loss))
    g = x.grad.cpu().movedim(1, -1)
    assert torch.all(g[bad] == 0) and torch.all(g[t == -100] == 0) and torch.isfinite(g).all()
    ref_l = lg.double().requires_grad_(True)
    F.cross_entropy(ref_l, torch.where(ok, t, torch.full_like(t, -100)), weight=w.double().cpu(), label_smoothing=0.1).backward()
    assert (x.grad.cpu().double() - ref_l.grad).abs().max().item() <= 2e-6 * ref_l.grad.abs().max().item()
    counts, invalid = iou.conf_metric.counts()
    assert invalid == int(bad.sum()) and counts.sum() == int(ok.sum())
    with pytest.raises(AssertionError):
        iou.value()
    per_px = S.CrossEntropyLossWithOptions(weight=w, label_smoothing=0.1, reduction="none")(lg.cuda(), t.cuda()).cpu()
    assert torch.isnan(per_px[bad]).all() and torch.all(per_px[t == -100] == 0) and torch.isfinite(per_px[ok]).all()


def test_nan_logit_poisons_its_own_pixel():
    K = 8
    lg, t = _case(1, K, 8, 8, 4.0, seed=4)
    lg[0, 5, 2, 3] = float("nan")
    w = _weight("positive", K, 2).cuda()
    for target in (t.cuda(), F.one_hot(t, K).movedim(-1, 1).float().cuda()):
        x = lg.cuda().requires_grad_(True)
        per_px = S.cross_entropy(x, target, reduction="none", weight=w, label_smoothing=0.1)
        per_px.sum().backward()
        torch.cuda.synchronize()
        m = per_px.detach().cpu()
        assert math.isnan(float(m[0, 2, 3]))
        m[0, 2, 3] = 0
        assert torch.isfinite(m).all()
        g = x.grad.cpu()
        assert torch.isnan(g[0, :, 2, 3]).all()
        g[0, :, 2, 3] = 0
        assert torch.isfinite(g).all()
        assert math.isnan(float(S.cross_entropy(lg.cuda(), target, weight=w)))


@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_zero_total_weight_gives_nan_like_torch(eps):
    """Pixels are counted but all their weights are 0 (D = 0): torch's mean is NaN and so is the gradient of every counted
    pixel.  Nothing counted at all: NaN loss, zero gradient (as the plain path)."""
    K = 6
    lg, t = _case(2, K, 8, 8, 4.0, seed=6, ignore=(-100,))
    t = torch.where(t == -100, t, t % 2)                       # labels only in classes 0 and 1 ...
    w = torch.tensor([0.0, 0.0, 1.0, 2.0, 0.5, 1.0])           # ... which weigh nothing
    x = lg.cuda().requires_grad_(True)
    loss = S.CrossEntropyLossWithOptions(weight=w.cuda(), label_smoothing=eps)(x, t.cuda())
    loss.backward()
    l64 = lg.double().requires_grad_(True)
    ref = F.cross_entropy(l64, t, weight=w.double(), label_smoothing=eps)
    ref.backward()
    torch.cuda.synchronize()
    counted = t != -100
    assert math.isnan(float(ref)) and math.isnan(float(loss))
    assert torch.isnan(l64.grad.movedim(1, -1)[counted]).all()
    assert torch.isnan(x.grad.cpu().movedim(1, -1)[counted]).all()
    x.grad = None
    none = torch.full_like(t, -100)
    loss = S.CrossEntropyLossWithOptions(weight=w.cuda(), label_smoothing=eps)(x, none.cuda())
    loss.backward()
    assert math.isnan(float(loss)) and torch.all(x.grad == 0)


@pytest.mark.parametrize("form", ["int", "scores"])
@pytest.mark.parametrize("tag", sorted(CONFIGS))
def test_iou_with_onehot_targets_matches_reference(tag, form):
    normalized, ignore = CONFIGS[tag]
    m = S.IoU(GK, normalized=normalized, ignore_index=ignore)
    for i in range(N_BATCHES):
        p, s = (torch.from_numpy(SEG[f"batch{i}/{k}"]) for k in ("pred", "scores"))
        m.add((s if form == "scores" else p).cuda(), torch.from_numpy(ONEHOT[f"batch{i}/onehot"]).cuda())
    iou, miou = m.value()
    want = ONEHOT[f"{tag}/{form}/iou"]
    assert iou.dtype == want.dtype and np.array_equal(iou, want, equal_nan=True)
    assert miou == ONEHOT[f"{tag}/{form}/miou"]
    assert np.array_equal(m.conf_metric.value(), ONEHOT[f"{tag}/{form}/conf"])


def test_confusion_matrix_with_onehot_rows_and_the_reference_checks():
    cm = S.ConfusionMatrix(GK)
    eye = np.eye(GK, dtype=np.float32)
    for i in range(N_BATCHES):
        p, t = SEG[f"batch{i}/pred"], SEG[f"batch{i}/target"]
        cm.add(torch.from_numpy(p).reshape(-1).cuda(), torch.from_numpy(eye[t.reshape(-1)]))     # host one-hot rows
    assert np.array_equal(cm.counts()[0], ONEHOT["cm/conf"]) and np.array_equal(cm.value(), ONEHOT["cm/conf"])
    pred = torch.from_numpy(ONEHOT["bad/pred"])
    for bad in ("sum09", "range"):
        assert bool(ONEHOT[f"bad/{bad}/raised"])               # the reference asserts on this row ...
        tgt = torch.from_numpy(ONEHOT[f"bad/{bad}/target"])
        cm = S.ConfusionMatrix(GK)
        cm.add(pred.cuda(), tgt.cuda())
        counts, invalid = cm.counts()
        assert invalid == 1 and counts.sum() == len(pred) - 1
        with pytest.raises(AssertionError):                    # ... and value() raises here
            cm.value()
        scores = F.one_hot(pred, GK).float()[:, :, None, None].cuda()     # score predictions, (N, K, 1, 1) targets
        iou = S.IoU(GK)
        iou.add(scores, tgt[:, :, None, None].cuda())
        with pytest.raises(AssertionError):
            iou.value()


def test_ce_step_with_probability_targets_updates_iou_in_the_same_pass():
    K = 8
    lg, t = _case(2, K, 16, 20, 4.0, seed=8)
    q = _prob_target(lg, t, seed=2).cuda()
    valid, rows = _row_checks(q.cpu())
    a, b = S.IoU(K), S.IoU(K)
    n0 = _lib.launch_count()
    loss = S.ce_step(lg.cuda(), q, a, weight=_weight("positive", K, 3).cuda())
    assert _lib.launch_count() - n0 == 1                       # loss, gradient-free here, and the IoU update: one kernel
    b.add(lg.cuda(), q)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss))                          # probability rows are not validated by the loss
    ca, ia = a.conf_metric.counts()
    cb, ib = b.conf_metric.counts()
    am = lg.argmax(1)
    want = torch.bincount(rows[valid] * K + am[valid], minlength=K * K).view(K, K).numpy()
    assert np.array_equal(ca, want) and np.array_equal(cb, want)
    assert ia == ib == int((~valid).sum()) > 0


def test_session_with_loss_instance_rejects_float_targets():
    from smaat_unet_b200.train import TrainSession
    K = 4
    sess = TrainSession(S.SmaAt_UNet(3, K, kernels_per_layer=2).cuda(), 2, (3, 32, 32), use_graph=False, warmup=1,
                        loss=S.CrossEntropyLossWithOptions(weight=torch.ones(K), label_smoothing=0.1))
    x = torch.rand(2, 3, 32, 32, device="cuda")
    y = torch.randint(0, K, (2, 32, 32), device="cuda")
    with pytest.raises(TypeError, match="class-index targets"):
        sess.step(x, y.float())
    sess.step(x, y)
    sess.close()


@pytest.mark.parametrize("use_graph", [False, True])
def test_train_session_weighted_smoothed_loss_matches_eager_steps(use_graph):
    """TrainSession(loss=CrossEntropyLossWithOptions(weight=w, label_smoothing=0.1)) reproduces eager steps of the same modules with
    torch.nn.CrossEntropyLoss(weight=w, label_smoothing=0.1) + Adam; the warm-up leaves the model and the IoU totals
    untouched.  Scheme and bounds of test_gpu_segmentation.py::test_train_session_cross_entropy_matches_eager_steps."""
    from smaat_unet_b200.train import TrainSession
    torch.manual_seed(3)
    B, S_, K = 2, 64, 21
    w = torch.rand(K) * 2 + 0.25
    m1 = S.SmaAt_UNet(3, K, kernels_per_layer=2).cuda().train()
    m2 = S.SmaAt_UNet(3, K, kernels_per_layer=2).cuda().train()
    m2.load_state_dict(m1.state_dict())
    xs = [torch.rand(B, 3, S_, S_, device="cuda") for _ in range(3)]
    ys = [torch.randint(0, K, (B, S_, S_), device="cuda") for _ in range(3)]
    held = S.IoU(K)
    pre = torch.arange(K * K + 1, device="cuda", dtype=torch.int64) % 7
    pre[-1] = 0
    held.load_totals(pre)
    loss = S.CrossEntropyLossWithOptions(weight=w, label_smoothing=0.1).cuda()
    sess = TrainSession(m1, B, (3, S_, S_), lr=1e-3, use_graph=use_graph, loss=loss, metrics=held)
    loss.weight.fill_(1.0)                                    # the session holds a snapshot taken at construction
    for k, v in m2.state_dict().items():                      # warm-up steps were rolled back
        assert torch.equal(v, m1.state_dict()[k]), k
    assert torch.equal(held.totals_snapshot(), pre)           # ... and so were the metric totals
    assert sess.y.dtype == torch.int64
    opt = torch.optim.Adam(m2.parameters(), lr=1e-3)
    crit = torch.nn.CrossEntropyLoss(weight=w.cuda(), label_smoothing=0.1)
    tols = [1e-5, 2e-3, 2e-2]
    for i, (x, y) in enumerate(zip(xs, ys)):
        l1 = float(sess.step(x, y))
        opt.zero_grad(set_to_none=True)
        l2 = crit(m2(x), y)
        l2.backward()
        opt.step()
        assert abs(l1 - float(l2)) <= tols[i] * abs(float(l2)), (i, l1, float(l2))
        if i == 0:
            for (k, a), b in zip(m1.state_dict().items(), m2.state_dict().values()):
                if a.dtype == torch.int64:
                    assert torch.equal(a, b), k
                else:
                    assert (a - b).abs().max().item() <= 2.5e-3, k
    counts, invalid = held.conf_metric.counts()
    assert invalid == 0 and int(counts.sum()) == int(pre[:-1].sum()) + 3 * B * S_ * S_
    sess.close()
