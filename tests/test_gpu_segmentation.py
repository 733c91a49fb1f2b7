"""-m gpu: the segmentation workflow (train_SmaAtUNet.py:139-199) on the device.  smaat_ce_fwd against float64
F.cross_entropy + autograd, CrossEntropyLoss / IoU / ConfusionMatrix against torch and against the reference's own outputs
(tests/golden/seg_metrics.npz), TrainSession(loss="cross_entropy") against eager steps with nn.CrossEntropyLoss + Adam,
one full-size gradient check, and the InferenceSession + ce_step validation path."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from oracle.make_golden_seg import CONFIGS, K as GK, N_BATCHES
from smaat_unet_b200.segmentation import ce_forward
from tests._util import dev, load_np_state_dict

pytestmark = pytest.mark.gpu
SEG = np.load(os.path.join(os.path.dirname(__file__), "golden", "seg_metrics.npz"))


def _case(B, K, H, W, spread, seed, ignore=(), invalid=()):
    """float32 logits whose top class leads the runner-up by >= 0.25 (so every argmax agrees), int64 labels with a share of
    each value in `ignore` / `invalid`."""
    g = torch.Generator().manual_seed(seed)
    lg = (torch.rand(B, K, H, W, generator=g) * 2 - 1) * spread
    top = torch.randint(0, K, (B, H, W), generator=g)
    lead = lg.max(1, keepdim=True).values + 0.25 + torch.rand(B, 1, H, W, generator=g)
    lg.scatter_(1, top[:, None], lead)
    t = torch.randint(0, K, (B, H, W), generator=g)
    for v in tuple(ignore) + tuple(invalid):
        t[torch.rand(B, H, W, generator=g) < 0.08] = v
    return lg, t


def _place(lg, misaligned):
    if not misaligned:
        return lg.cuda()
    base = torch.empty(lg.numel() + 1, device="cuda")
    x = base[1:].view(lg.shape)                 # 4-byte aligned only: the scalar kernel
    x.copy_(lg.cuda())
    return x


# B, K, H, W, spread, misaligned, ignore_index
CE_CASES = [
    (2, 2, 16, 16, 4.0, False, -100),
    (2, 8, 17, 19, 4.0, False, 255),           # P % 4 != 0: scalar path
    (2, 8, 32, 32, 80.0, False, -100),         # logits in +-80
    (3, 21, 24, 24, 6.0, True, 255),           # misaligned view: scalar path
    (2, 21, 28, 36, 80.0, False, 255),
    (1, 150, 20, 24, 10.0, False, -100),       # K above the shared-memory histogram: global-atomic histogram
]


@pytest.mark.parametrize("case", CE_CASES)
def test_ce_fwd_matches_float64_cross_entropy(case):
    B, K, H, W, spread, mis, ig = case
    lg, t = _case(B, K, H, W, spread, seed=K * 100 + H, ignore=(ig,))
    x, tc = _place(lg, mis), t.cuda()
    g = torch.Generator().manual_seed(9)
    conf0 = torch.randint(0, 50, (K, K), generator=g).cuda()
    conf = conf0.clone()
    acc, dl = ce_forward(x, tc, ig, True, want_grad=True, conf=conf)
    l64 = lg.double().requires_grad_(True)
    ref = F.cross_entropy(l64, t, ignore_index=ig, reduction="sum")
    ref.backward()
    torch.cuda.synchronize()
    keep = t != ig
    assert abs(float(acc[0]) - float(ref)) <= 2e-6 * abs(float(ref))
    assert int(acc[1]) == int(keep.sum()) and int(acc[2]) == 0
    gref = l64.grad
    d = dl.cpu().double()
    assert (d - gref).abs().max().item() <= 2e-6 * gref.abs().max().item()
    assert torch.all(d.permute(0, 2, 3, 1)[~keep] == 0)              # exactly 0 on ignored pixels
    am = lg.argmax(1)
    want = torch.bincount((t[keep] * K + am[keep]), minlength=K * K).view(K, K)
    assert torch.equal((conf - conf0).cpu(), want)
    conf2 = conf0.clone()
    acc2, dl2 = ce_forward(x, tc, ig, True, want_grad=True, conf=conf2)
    assert torch.equal(conf2, conf) and torch.equal(dl2, dl) and float(acc2[1]) == float(acc[1])


@pytest.mark.parametrize("reduction", ["mean", "sum"])
@pytest.mark.parametrize("ig", [-100, 255])
def test_cross_entropy_loss_forward_backward_match_torch_float64(reduction, ig):
    lg, t = _case(2, 21, 20, 24, 8.0, seed=31, ignore=(ig,))
    x = lg.cuda().requires_grad_(True)
    loss = S.CrossEntropyLoss(ignore_index=ig, reduction=reduction)(x, t.cuda())
    (loss * 1.7).backward()
    l64 = lg.double().requires_grad_(True)
    ref = F.cross_entropy(l64, t, ignore_index=ig, reduction=reduction)
    (ref * 1.7).backward()
    assert loss.dtype == torch.float32 and loss.dim() == 0
    assert abs(float(loss) - float(ref)) <= 2e-6 * abs(float(ref))
    assert (x.grad.cpu().double() - l64.grad).abs().max().item() <= 2e-6 * l64.grad.abs().max().item()


def test_all_equal_logits_go_to_class_zero():
    K = 8
    x = torch.full((2, K, 8, 12), 0.3, device="cuda")
    t = torch.randint(0, K, (2, 8, 12), device="cuda")
    conf = torch.zeros(K, K, dtype=torch.int64, device="cuda")
    acc, _ = ce_forward(x, t, -100, True, conf=conf)
    want = torch.bincount(t.flatten().cpu() * K, minlength=K * K).view(K, K)
    assert torch.equal(conf.cpu(), want) and int(conf[:, 1:].sum()) == 0
    assert abs(float(acc[0]) / float(acc[1]) - math.log(K)) <= 1e-6 * math.log(K)


def test_invalid_labels_are_counted_not_indexed():
    K = 8
    lg, t = _case(2, K, 12, 16, 4.0, seed=3, ignore=(-100,), invalid=(K, -7, 1000))
    x = lg.cuda().requires_grad_(True)
    iou = S.IoU(K)
    loss = S.ce_step(x, t.cuda(), iou)
    loss.backward()
    torch.cuda.synchronize()
    bad = (t != -100) & ((t < 0) | (t >= K))
    assert bad.any() and math.isnan(float(loss))
    g = x.grad.cpu().permute(0, 2, 3, 1)
    assert torch.all(g[bad] == 0) and torch.all(g[t == -100] == 0) and torch.isfinite(g).all()
    ok = ~bad & (t != -100)
    ref_l = lg.double().requires_grad_(True)
    F.cross_entropy(ref_l, torch.where(ok, t, torch.full_like(t, -100)), ignore_index=-100).backward()
    assert (x.grad.cpu().double() - ref_l.grad).abs().max().item() <= 2e-6 * ref_l.grad.abs().max().item()
    counts, invalid = iou.conf_metric.counts()
    assert invalid == int(bad.sum()) and counts.sum() == int(ok.sum())
    with pytest.raises(AssertionError):
        iou.value()
    acc, _ = ce_forward(lg.cuda(), t.cuda(), -100, True)
    assert int(acc[2]) == int(bad.sum())


def test_nan_logits_give_nan_loss_and_count_under_the_first_nan_channel():
    """Documented in include/smaat_b200.h: the pixel's loss and gradient are NaN; its argmax is the first NaN channel
    (torch.argmax's answer) and the pixel is counted under that column."""
    K = 8
    lg, t = _case(1, K, 8, 8, 4.0, seed=4)
    lg[0, 5, 2, 3] = float("nan")
    lg[0, 6, 2, 3] = float("nan")
    assert int(lg.argmax(1)[0, 2, 3]) == 5
    x = lg.cuda().requires_grad_(True)
    iou = S.IoU(K)
    loss = S.ce_step(x, t.cuda(), iou)
    loss.backward()
    assert math.isnan(float(loss)) and math.isnan(float(F.cross_entropy(lg, t)))
    g = x.grad.cpu()
    assert torch.isnan(g[0, :, 2, 3]).all()
    g[0, :, 2, 3] = 0
    assert torch.isfinite(g).all()
    counts, invalid = iou.conf_metric.counts()
    want = torch.bincount(t.flatten() * K + lg.argmax(1).flatten(), minlength=K * K).view(K, K).numpy()
    assert invalid == 0 and np.array_equal(counts, want) and counts[int(t[0, 2, 3]), 5] >= 1


@pytest.mark.parametrize("cpu_target", [False, True])
@pytest.mark.parametrize("form", ["int", "scores"])
@pytest.mark.parametrize("tag", sorted(CONFIGS))
def test_iou_and_confusion_matrix_drop_ins_match_reference(tag, form, cpu_target):
    normalized, ignore = CONFIGS[tag]
    m = S.IoU(GK, normalized=normalized, ignore_index=ignore)
    cm = S.ConfusionMatrix(GK, normalized=normalized)
    for i in range(N_BATCHES):
        p, t, s = (torch.from_numpy(SEG[f"batch{i}/{k}"]) for k in ("pred", "target", "scores"))
        pred = (s if form == "scores" else p).cuda()
        tgt = t if cpu_target else t.cuda()
        m.add(pred, tgt)
        cm.add(pred.reshape(-1) if form == "int" else pred.permute(0, 2, 3, 1).reshape(-1, GK), tgt.reshape(-1))
    iou, miou = m.value()
    want = SEG[f"{tag}/{form}/iou"]
    assert iou.dtype == want.dtype and np.array_equal(iou, want, equal_nan=True)
    assert miou == SEG[f"{tag}/{form}/miou"]
    assert np.array_equal(m.conf_metric.value(), SEG[f"{tag}/{form}/conf"])
    assert np.array_equal(cm.value(), SEG[f"{tag}/{form}/conf"])
    assert np.array_equal(m.conf_metric.counts()[0], SEG["counts"])          # counts exact


def test_ce_step_with_iou_equals_separate_loss_and_add():
    lg, t = _case(4, 21, 24, 32, 6.0, seed=12)
    x, tc = lg.cuda(), t.cuda()
    a, b = S.IoU(21), S.IoU(21)
    l1 = S.ce_step(x, tc, a)
    l2 = S.CrossEntropyLoss()(x, tc)
    b.add(x, tc)
    assert abs(float(l1) - float(l2)) <= 1e-12 * abs(float(l2)) + 1e-7 * abs(float(l2))
    assert np.array_equal(a.conf_metric.counts()[0], b.conf_metric.counts()[0])
    ia, ma = a.value()
    ib, mb = b.value()
    assert np.array_equal(ia, ib, equal_nan=True) and ma == mb


@pytest.mark.parametrize("use_graph", [False, True])
def test_train_session_cross_entropy_matches_eager_steps(use_graph):
    """TrainSession(loss="cross_entropy") reproduces eager steps of the same modules with nn.CrossEntropyLoss + Adam
    (train_SmaAtUNet.py:54-57,181-182); the warm-up leaves the model and the IoU totals untouched.  Same scheme and bounds
    as test_gpu_train.py::test_train_session_matches_eager_steps (chaotic drift after the first step)."""
    from smaat_unet_b200.train import TrainSession
    torch.manual_seed(3)
    B, S_, K = 2, 64, 21
    m1 = S.SmaAt_UNet(3, K, kernels_per_layer=2).cuda().train()
    m2 = S.SmaAt_UNet(3, K, kernels_per_layer=2).cuda().train()
    m2.load_state_dict(m1.state_dict())
    xs = [torch.rand(B, 3, S_, S_, device="cuda") for _ in range(3)]
    ys = [torch.randint(0, K, (B, S_, S_), device="cuda") for _ in range(3)]
    held = S.IoU(K)
    pre = torch.arange(K * K + 1, device="cuda", dtype=torch.int64) % 7
    pre[-1] = 0
    held.load_totals(pre)
    sess = TrainSession(m1, B, (3, S_, S_), lr=1e-3, use_graph=use_graph, loss="cross_entropy", metrics=held)
    for k, v in m2.state_dict().items():                      # warm-up steps were rolled back
        assert torch.equal(v, m1.state_dict()[k]), k
    assert torch.equal(held.totals_snapshot(), pre)           # ... and so were the metric totals
    assert sess.y.dtype == torch.int64
    opt = torch.optim.Adam(m2.parameters(), lr=1e-3)
    crit = torch.nn.CrossEntropyLoss()
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
    assert int(m1.state_dict()["inc.double_conv.1.num_batches_tracked"]) == 3
    sess.close()
    # the default metric is an IoU over the logits' channel count, fresh
    sess2 = TrainSession(S.SmaAt_UNet(3, K, kernels_per_layer=2).cuda(), B, (3, S_, S_), use_graph=use_graph, loss="cross_entropy")
    assert isinstance(sess2.metrics, S.IoU) and sess2.metrics.num_classes == K
    assert int(sess2.metrics.conf_metric.counts()[0].sum()) == 0
    sess2.step(xs[0], ys[0])
    assert int(sess2.metrics.conf_metric.counts()[0].sum()) == B * S_ * S_
    sess2.close()


def _port_ce_step(sd_np, x_np, t_np, dtype):
    sd = {}
    for k, v in sd_np.items():
        t = torch.as_tensor(np.asarray(v))
        if t.dtype == torch.int64:
            sd[k] = t
        elif k.endswith(("running_mean", "running_var")):
            sd[k] = t.float().to(dtype)
        else:
            sd[k] = t.float().to(dtype).requires_grad_(True)
    y = TP.smaat_unet_forward(torch.from_numpy(x_np).float().to(dtype), sd, True)
    loss = F.cross_entropy(y, torch.from_numpy(t_np))
    loss.backward()
    return float(loss.detach()), {k: v.grad.double().numpy() for k, v in sd.items() if v.dtype != torch.int64 and v.requires_grad}


def test_cross_entropy_gradient_at_voc_shape_matches_cpu_autograd_fp64():
    """SmaAt_UNet(3, 21) at the VOC training shape (B = 2, 3x224x224, train mode): CE gradient vs float64 autograd over the
    CPU port, held to a small multiple of the reference algorithm's own fp32-vs-fp64 movement (as test_gpu_api_paths.py's
    full-size gradient check)."""
    sd_np = fill_schema(smaat_unet_schema(3, 21, 2), 21)
    m = load_np_state_dict(S.SmaAt_UNet(3, 21), cast_sd(sd_np, np.float32)).cuda().train()
    rng = np.random.default_rng(8)
    x_np = rng.uniform(0, 1, (2, 3, 224, 224))
    t_np = rng.integers(0, 21, (2, 224, 224))
    loss = S.CrossEntropyLoss()(m(dev(x_np)), torch.from_numpy(t_np).cuda())
    loss.backward()
    torch.cuda.synchronize()
    l64, g64 = _port_ce_step(sd_np, x_np, t_np, torch.float64)
    _, g32 = _port_ce_step(sd_np, x_np, t_np, torch.float32)
    assert abs(float(loss) - l64) <= 2e-4 * abs(l64)

    def rel_max(a, b):
        return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))

    def rel_l2(a, b):
        return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    gmax = max(float(np.abs(g).max()) for g in g64.values())
    live = [k for k, g in g64.items() if np.abs(g).max() >= 1e-6 * gmax]
    noise_max = max(rel_max(g32[k], g64[k]) for k in live)
    noise_l2 = max(rel_l2(g32[k], g64[k]) for k in live)
    tol_max, tol_l2 = max(2e-3, 5.0 * noise_max), max(1e-3, 5.0 * noise_l2)
    for name, p in m.named_parameters():
        got = p.grad.double().cpu().numpy()
        if name not in live:
            assert float(np.abs(got).max()) <= 1e-3 * gmax, name
            continue
        e_max, e_l2 = rel_max(got, g64[name]), rel_l2(got, g64[name])
        assert np.isfinite(e_max) and e_max <= tol_max and e_l2 <= tol_l2, \
            f"grad {name}: rel max {e_max:.3e} (tol {tol_max:.1e}), rel L2 {e_l2:.3e} (tol {tol_l2:.1e})"


def test_validation_path_inference_session_and_ce_step():
    """The validation loop of train_SmaAtUNet.py:67-77 on the serving path: InferenceSession logits are bitwise the eager
    no_grad forward's, and ce_step on them equals CrossEntropyLoss + IoU.add on the same logits."""
    from smaat_unet_b200.engine import InferenceSession
    torch.manual_seed(2)
    m = S.SmaAt_UNet(3, 21).cuda().eval()
    x = torch.rand(8, 3, 224, 224, device="cuda")
    y = torch.randint(0, 21, (8, 224, 224))
    with torch.no_grad():
        want = m(x).clone()
    sess = InferenceSession(m, 8, (3, 224, 224))
    got = sess.forward(x).clone()
    assert torch.equal(got, want)
    a, b = S.IoU(21), S.IoU(21)
    with torch.no_grad():
        l1 = S.ce_step(got, y, a)                               # host target, as train_SmaAtUNet.py:77 passes it
        l2 = S.CrossEntropyLoss()(got, y.cuda())
        b.add(got, y)
    assert abs(float(l1) - float(l2)) <= 1e-7 * abs(float(l2))
    assert np.array_equal(a.conf_metric.counts()[0], b.conf_metric.counts()[0])
    ref = F.cross_entropy(want.double().cpu(), y)
    assert abs(float(l1) - float(ref)) <= 2e-6 * abs(float(ref))
