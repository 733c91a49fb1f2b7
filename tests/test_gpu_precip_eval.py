"""The threshold sweep and the test-set evaluator on the GPU: the kernel against the reference's batch-1 golden numbers and
against PrecipitationMetrics image by image, the per-image NaN rule, the strided persistence read, the kernel's edges
through poisoned over-allocated buffers, graph capture, and evaluate_precipitation end to end."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import sweep_oracle as SO

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "precip_eval.npz"))
TH = SO.GOLDEN_THRESHOLDS
KEYS = ("mse", "mse_denorm", "mse_pixel", "precision", "recall", "accuracy", "f1", "csi", "far", "hss")
MSE_KEYS = ("mse", "mse_denorm", "mse_pixel")
COUNT_IDX = {"total_tn": 4, "total_fp": 5, "total_fn": 6, "total_tp": 7, "total_samples": 2, "total_pixels": 3}


def _same(a, b, tol, what):
    a, b = float(a), float(b)
    if math.isnan(b):
        assert math.isnan(a), what
    else:
        assert abs(a - b) <= tol * max(abs(b), 1e-30), f"{what}: {a} vs {b}"


def _rain(shape, seed, scale=0.06):
    g = torch.Generator().manual_seed(seed)
    v = torch.rand(shape, generator=g) ** 3 * scale
    return torch.where(torch.rand(shape, generator=g) < 0.3, torch.zeros(()), v)


@pytest.mark.parametrize("denorm", [True, False])
def test_sweep_matches_reference_golden(denorm):
    import smaat_unet_b200 as S
    tag = "denorm" if denorm else "norm"
    x, y = torch.from_numpy(GOLD["x"]).cuda(), torch.from_numpy(GOLD["y"]).cuda()
    m = S.PrecipitationMetricsSweep(TH, denormalize=denorm)
    m.update_persistence(x[:6], y[:6])          # two batches: the split changes nothing
    m.update_persistence(x[6:], y[6:])
    assert int(m.skipped_images) == 2 and int(m.total_samples) == len(x) - 2
    tot = m.threshold_totals()
    out = m.compute()
    for t in TH:
        for k, i in COUNT_IDX.items():
            assert int(tot[t][i]) == int(GOLD[f"{tag}/{t}/{k}"]), (t, k)
        for k in KEYS:
            _same(out[t][k], GOLD[f"{tag}/{t}/{k}"], 2e-6, f"{tag}/{t}/{k}")


def _per_image_reference(preds, target, thresholds, denorm):
    """PrecipitationMetrics(threshold=t) for every t, updated with one image at a time."""
    import smaat_unet_b200 as S
    ms = {t: S.PrecipitationMetrics(threshold=t, denormalize=denorm) for t in thresholds}
    for i in range(target.size(0)):
        for m in ms.values():
            m.update(preds[i:i + 1], target[i:i + 1])
    return ms


def _check_against(sweep, ms, rtol=1e-6):
    tot, out = sweep.threshold_totals(), sweep.compute()
    for t, m in ms.items():
        ref = m._totals.cpu()
        assert torch.equal(tot[t][2:8], ref[2:8]), (t, tot[t], ref)          # samples, pixels and counts: exact
        want = m.compute()
        for k in KEYS:
            _same(out[t][k], want[k], rtol if k in MSE_KEYS else 0.0, f"{t}/{k}")


@pytest.mark.parametrize("denorm", [True, False])
@pytest.mark.parametrize("shape", [(4, 288, 288), (3, 37, 53)])
def test_sweep_equals_per_image_precipitation_metrics(denorm, shape):
    import smaat_unet_b200 as S
    y = _rain(shape, 1).cuda()
    p = (y + 0.01 * torch.randn(shape, generator=torch.Generator().manual_seed(2)).cuda()).abs().unsqueeze(1)
    th = TH if denorm else (0.05, 0.1, 0.2, 0.4)
    sweep = S.PrecipitationMetricsSweep(th, denormalize=denorm)
    sweep.update(p, y)
    _check_against(sweep, _per_image_reference(p, y, th, denorm))


def test_nan_image_is_skipped_alone():
    import smaat_unet_b200 as S
    y = _rain((8, 64, 72), 3).cuda()
    p = _rain((8, 1, 64, 72), 4).cuda()
    p[5, 0, 10, 11] = float("nan")
    sweep = S.PrecipitationMetricsSweep(TH)
    sweep.update(p, y)
    assert int(sweep.skipped_images) == 1 and int(sweep.total_samples) == 7 and int(sweep.total_pixels) == 7 * 64 * 72
    ms = _per_image_reference(p, y, TH, True)
    assert all(int(m.skipped_batches) == 1 for m in ms.values())
    _check_against(sweep, ms)
    # the reference's batch update would have dropped all eight
    m8 = S.PrecipitationMetrics(threshold=0.5)
    m8.update(p, y)
    assert int(m8.total_samples) == 0


def test_persistence_read_in_place_equals_contiguous_copy():
    import smaat_unet_b200 as S
    from smaat_unet_b200.engine import InferenceSession
    x = _rain((5, 12, 96, 80), 5).cuda()
    y = _rain((5, 96, 80), 6).cuda()
    a, b = S.PrecipitationMetricsSweep(TH), S.PrecipitationMetricsSweep(TH)
    a.update_persistence(x, y)
    b.update(x[:, -1:].contiguous(), y)
    assert torch.equal(a.totals_snapshot(), b.totals_snapshot())
    out = InferenceSession(S.PersistenceModel(), 5, (12, 96, 80)).forward(x)
    assert torch.equal(out, x[:, -1:])


# ----------------------------------------------------------------------------------------------- the C ABI at its edges
def _raw_sweep(pred, bstride, target, B, P, thresholds, denorm, stream=None):
    """smaat_precip_sweep_fwd into over-allocated, poisoned buffers; returns (per_image, hist) and checks the tails."""
    import smaat_unet_b200 as S
    T = len(thresholds)
    cells = (T + 1) ** 2
    per = torch.full((B * 3 + 7,), float("nan"), dtype=torch.float64, device="cuda")
    hist = torch.full((B * cells + 9,), -1, dtype=torch.int32, device="cuda")
    thr = (ctypes.c_float * T)(*thresholds)
    lib = S._lib.load()
    st = torch.cuda.current_stream().cuda_stream if stream is None else stream
    S._lib.check(lib.smaat_precip_sweep_fwd(pred, bstride, target.data_ptr(), B, P, 47.83, thr, T, int(denorm), per.data_ptr(),
                                            hist.data_ptr(), st), "sweep")
    torch.cuda.synchronize()
    assert torch.isnan(per[B * 3:]).all(), "per_image written past its end"
    assert (hist[B * cells:] == -1).all(), "hist written past its end"
    return per[:B * 3].view(B, 3).cpu(), hist[:B * cells].view(B, T + 1, T + 1).cpu()


def _check_raw(per, hist, pn, yn, thresholds, denorm):
    T1 = len(thresholds) + 1
    for b in range(len(pn)):
        want = np.zeros((T1, T1), np.int64)        # the fwd pass histograms every image; a NaN value is in bin 0
        np.add.at(want, (SO.bins(yn[b], thresholds, denorm), SO.bins(pn[b], thresholds, denorm)), 1)
        assert torch.equal(hist[b].to(torch.int64), torch.from_numpy(want)), b
        d = pn[b].astype(np.float64) - yn[b]
        assert float(per[b, 0]) == pytest.approx(float((d ** 2).sum()), rel=1e-6, abs=1e-30, nan_ok=True)
        f = SO.MO.FACTOR if denorm else np.float32(1)
        dd = (pn[b] * f).astype(np.float64) - (yn[b] * f)
        assert float(per[b, 1]) == pytest.approx(float((dd ** 2).sum()), rel=1e-6, abs=1e-30, nan_ok=True)
        assert float(per[b, 2]) == float(np.isnan(pn[b]).sum() + np.isnan(yn[b]).sum() - (np.isnan(pn[b]) & np.isnan(yn[b])).sum())


@pytest.mark.parametrize("B,H,W,offset,T", [
    (3, 33, 35, 0, 6),      # P % 4 != 0: scalar kernel
    (2, 64, 64, 1, 6),      # unaligned pointers: scalar kernel
    (1, 64, 64, 0, 1),      # B = 1, T = 1, vector kernel
    (4, 40, 48, 0, 32),     # T = 32
    (2, 17, 19, 3, 32),
    (5, 288, 288, 0, 6),    # several slices per image
])
def test_sweep_kernel_edges_in_poisoned_buffers(B, H, W, offset, T):
    P = H * W
    thresholds = TH if T == 6 else ((0.5,) if T == 1 else tuple(0.25 * (i + 1) for i in range(T)))
    y = _rain((B, P), 7 + B).cuda()
    p = _rain((B, P), 9 + B).cuda()
    p[0, 3] = float("nan")
    yb = torch.empty(B * P + offset, device="cuda")
    yb[offset:] = y.reshape(-1)
    pb = torch.empty(B * P + offset, device="cuda")
    pb[offset:] = p.reshape(-1)
    target = yb[offset:]
    for denorm in (True, False):
        per, hist = _raw_sweep(pb.data_ptr() + 4 * offset, P, target, B, P, thresholds, denorm)
        _check_raw(per, hist, p.cpu().numpy(), y.cpu().numpy(), thresholds, denorm)


def test_sweep_kernel_reads_the_strided_last_frame():
    B, C, H, W = 3, 4, 24, 28
    x = _rain((B, C, H, W), 11).cuda()
    y = _rain((B, H, W), 12).cuda()
    per, hist = _raw_sweep(x.data_ptr() + (C - 1) * H * W * 4, C * H * W, y, B, H * W, TH, True)
    _check_raw(per, hist, x[:, -1].reshape(B, -1).cpu().numpy(), y.reshape(B, -1).cpu().numpy(), TH, True)


def test_commit_in_cuda_graph_equals_eager():
    import smaat_unet_b200 as S
    y = _rain((6, 72, 80), 13).cuda()
    x = _rain((6, 12, 72, 80), 14).cuda()
    x[2, -1, 0, 0] = float("nan")
    eager, graphed = S.PrecipitationMetricsSweep(TH), S.PrecipitationMetricsSweep(TH)
    for _ in range(3):
        eager.update_persistence(x, y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        graphed.update_persistence(x, y)     # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graphed.reset()
    with torch.cuda.graph(g):
        graphed.update_persistence(x, y)
    graphed.reset()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(graphed.totals_snapshot(), eager.totals_snapshot())
    assert int(graphed.skipped_images) == 3 and int(graphed.total_samples) == 15


# ----------------------------------------------------------------------------------------------- end to end
def test_evaluate_precipitation_counts_every_sample_once(monkeypatch):
    import smaat_unet_b200 as S
    from smaat_unet_b200 import evaluate as E
    from smaat_unet_b200.engine import InferenceSession
    n, H, W = 37, 64, 64
    frames = _rain((n, 18, H, W), 21).numpy()
    ds = S.precipitation_maps_oversampled_shard(frames, 12, 6, train=False)
    torch.manual_seed(0)
    models = {"PersistenceModel": S.PersistenceModel(), "SmaAt-UNet": S.SmaAt_UNet(12, 1, kernels_per_layer=2),
              "UNetDS": S.UNetDS(12, 1, kernels_per_layer=2), "UNet": S.UNet(12, 1)}
    for m in models.values():
        for mod in m.modules():          # small outputs, so they spread across the thresholds in mm/h
            if isinstance(mod, S.OutConv):
                torch.nn.init.normal_(mod.conv.weight, 0, 0.002)
                torch.nn.init.constant_(mod.conv.bias, 0.005)
    made = []

    class Recorded(S.PrecipitationMetricsSweep):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            made.append(self)

    monkeypatch.setattr(E, "PrecipitationMetricsSweep", Recorded)
    res = E.evaluate_precipitation(models, ds, batch=8, thresholds=TH)
    assert list(res) == list(models)
    assert [int(a.total_samples) for a in made] == [n] * len(models)
    assert [int(a.skipped_images) for a in made] == [0] * len(models)
    xs = torch.from_numpy(frames[:, :12]).cuda()
    ys = torch.from_numpy(frames[:, -1]).cuda()
    failed = []
    for name, m in models.items():
        if name == "PersistenceModel":
            preds = xs[:, -1:]
        else:
            sess = InferenceSession(m, 1, (12, H, W))
            preds = torch.cat([sess.forward(xs[i:i + 1]).clone() for i in range(n)])
        ms = _per_image_reference(preds, ys, TH, True)
        for t, metric in ms.items():
            want, got = metric.compute(), res[name][t]
            assert int(metric.total_samples) == n
            for k in KEYS:
                w, g = float(want[k]), float(got[k])
                tol = 1e-6 if k in MSE_KEYS else 0.0
                if not ((math.isnan(w) and math.isnan(g)) or abs(g - w) <= tol * max(abs(w), 1e-30)):
                    failed.append(f"{name} {t} {k}: {g} vs {w}")
    assert not failed, failed
