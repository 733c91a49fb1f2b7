"""CPU restatement of the threshold sweep (smaat_precip_sweep_fwd / _commit) -- TEST INFRASTRUCTURE ONLY.

Every image is a batch of one of the reference's ``PrecipitationMetrics.update`` (metric/precipitation_metrics.py:37-95),
for several thresholds at once: an image with a NaN is skipped; the others add sum((p-y)^2), sum((p*f-y*f)^2), one sample,
their pixels, and a joint (target bin, pred bin) histogram, where a value's bin is the number of thresholds its
``(v * f) * 12`` exceeds in float32.  For strictly increasing thresholds the histogram holds every threshold's confusion
matrix.  Pinned against the unmodified reference class, run at batch size 1 per threshold, by oracle/make_golden_eval.py
-> tests/golden/precip_eval.npz.
"""
from __future__ import annotations

import numpy as np

from oracle import metrics_oracle as MO

GOLDEN_THRESHOLDS = (0.5, 1.0, 2.0, 5.0, 10.0, 30.0)


def bins(v, thresholds, denormalize=True):
    """#{i : (v * 47.83) * 12 > thresholds[i]} in float32 (v * 12 without denormalize), precipitation_metrics.py:80-85."""
    v = np.asarray(v, np.float32)
    h = (v * MO.FACTOR if denormalize else v) * np.float32(12)
    thr = np.asarray(thresholds, np.float32)
    return (h[..., None] > thr).sum(-1).astype(np.int64)


def sweep(preds, targets, thresholds, denormalize=True):
    """preds, targets: (N, P) float32, image by image.  Returns the totals (``metrics_oracle`` state names, plus
    ``skipped`` and ``hist`` (T+1, T+1) [target bin][pred bin])."""
    T1 = len(thresholds) + 1
    st = dict(total_loss=0.0, total_loss_denorm=0.0, total_samples=0, total_pixels=0, skipped=0,
              hist=np.zeros((T1, T1), np.int64))
    for p, y in zip(np.asarray(preds, np.float32), np.asarray(targets, np.float32)):
        if np.isnan(p).any() or np.isnan(y).any():
            st["skipped"] += 1
            continue
        st["total_loss"] += float(np.sum((p - y).astype(np.float64) ** 2))
        if denormalize:
            st["total_loss_denorm"] += float(np.sum((p * MO.FACTOR - y * MO.FACTOR).astype(np.float64) ** 2))
        st["total_samples"] += 1
        st["total_pixels"] += p.size
        np.add.at(st["hist"], (bins(y, thresholds, denormalize), bins(p, thresholds, denormalize)), 1)
    return st


def threshold_state(st, i):
    """The ``metrics_oracle`` state of threshold number i (0-based) from the sweep totals."""
    h, k = st["hist"], i + 1
    out = {key: st[key] for key in ("total_loss", "total_loss_denorm", "total_samples", "total_pixels")}
    out.update(total_tp=int(h[k:, k:].sum()), total_fn=int(h[k:, :k].sum()), total_fp=int(h[:k, k:].sum()),
               total_tn=int(h[:k, :k].sum()))
    return out


def compute(st, thresholds, denormalize=True):
    """{threshold: the reference's compute() dict}."""
    return {t: MO.compute(threshold_state(st, i), denormalize) for i, t in enumerate(thresholds)}


def _boundary_values(threshold, denormalize):
    """Normalised float32 values whose (v * 47.83) * 12 (v * 12) lands next to ``threshold``: every value within one
    float32 ulp of it, and the nearest value on each side."""
    t = np.float32(threshold)
    v = np.float32(t / (12 * MO.FACTOR if denormalize else 12))
    for _ in range(16):
        v = np.nextafter(v, np.float32(0))
    cand = []
    for _ in range(33):
        cand.append((v, (v * MO.FACTOR if denormalize else v) * np.float32(12)))
        v = np.nextafter(v, np.float32(np.inf))
    below = max((c for c in cand if c[1] < t), key=lambda c: c[1])
    above = min((c for c in cand if c[1] > t), key=lambda c: c[1])
    near = {float(c[0]) for c in cand if abs(float(c[1]) - float(t)) <= float(np.spacing(t))}
    return sorted(near | {float(below[0]), float(above[0])})


def eval_samples(seed=0, n=13, C=3, H=16, W=20):
    """Deterministic (x (n, C, H, W), y (n, H, W)) float32 test samples for the golden file and the tests.
    Sample 0 is all dry, sample 1 has a NaN in its last input frame (the persistence prediction), sample 2 has a NaN in its
    target, and samples 3 and 4 carry values within one float32 ulp of every golden threshold, on either side, in the
    prediction and the target (sample 3 for ``denormalize=True``, sample 4 for ``False``); the rest are rain fields that
    spread over all the golden thresholds."""
    rng = np.random.default_rng(seed)
    x = (rng.random((n, C, H, W)) ** 3 * 0.06).astype(np.float32)
    x[rng.random((n, C, H, W)) < 0.3] = 0
    y = (rng.random((n, H, W)) ** 3 * 0.06).astype(np.float32)
    y[rng.random((n, H, W)) < 0.3] = 0
    x[0], y[0] = 0, 0
    x[1, C - 1, 3, 7] = np.nan
    y[2, 5, 2] = np.nan
    for s, denorm in ((3, True), (4, False)):
        vals = np.concatenate([_boundary_values(t, denorm) for t in GOLDEN_THRESHOLDS]).astype(np.float32)
        k = len(vals)
        assert 3 * k <= H * W
        fx, fy = x[s, C - 1].reshape(-1), y[s].reshape(-1)
        fx[:k] = vals                          # boundary predictions against random targets
        fy[k:2 * k] = vals                     # and boundary targets against random predictions
        fy[2 * k:3 * k] = vals[::-1]
    return x, y
