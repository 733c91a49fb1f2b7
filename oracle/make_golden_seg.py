"""Generate tests/golden/seg_metrics.npz and tests/golden/dataset_classification.npz from the UNMODIFIED reference classes
-- TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_seg

seg_metrics.npz: the reference's ``metric.iou.IoU`` / ``metric.confusionmatrix.ConfusionMatrix`` (numpy + torch only) fed
seeded batches in both of IoU.add's forms -- (N, H, W) integer predictions and (N, K, H, W) scores -- for normalized
True / False and ignore_index None / an int / a tuple.  Class ``ABSENT`` occurs in no prediction and no label, so its IoU
is NaN.  The inputs are stored next to the results so the GPU tests replay the same batches.

dataset_classification.npz: ``precipitation_maps_classification_h5`` (utils/dataset_precip.py:83-127) run unmodified under
the h5py stand-in of oracle/make_golden_data.py, over ``classification_array()``.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get("SMAAT_REFERENCE", "/root/reference")
GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
K = 6
ABSENT = 4
N_BATCHES = 3
CONFIGS = {"plain": (False, None), "norm": (True, None), "ign_int": (False, 1), "ign_tuple": (False, (0, 2)),
           "norm_ign_tuple": (True, (0, 2))}
INDICES = (0, 1, 7, 13)
EDGES_MM_H = (0.0, 0.5, 1.0, 2.0, 5.0, 10.0, 30.0)


def seg_batches():
    """[(pred int64 (N, H, W), target int64 (N, H, W), scores float32 (N, K, H, W) with argmax == pred)] -- the top score
    leads the runner-up by at least 0.5, so any argmax agrees."""
    rng = np.random.default_rng(20261015)
    present = np.array([c for c in range(K) if c != ABSENT])
    out = []
    for i in range(N_BATCHES):
        shape = (2, 9 + i, 12)
        target = present[rng.integers(0, len(present), shape)]
        pred = np.where(rng.random(shape) < 0.6, target, present[rng.integers(0, len(present), shape)])
        scores = rng.uniform(-3.0, 3.0, (shape[0], K) + shape[1:]).astype(np.float32)
        top = scores.max(axis=1)
        np.put_along_axis(scores, pred[:, None], (top + 0.5 + rng.random(top.shape))[:, None].astype(np.float32), axis=1)
        out.append((pred.astype(np.int64), target.astype(np.int64), scores))
    return out


def classification_array():
    """(n_images, H, W) float32 frames in [0, 1) with exact zeros and values on the bin edges (in mm/h after * 47.83 * 12)."""
    rng = np.random.default_rng(20261016)
    a = rng.random((40, 6, 5), dtype=np.float32) * np.float32(0.08)
    a[rng.random(a.shape) < 0.2] = 0.0
    edges = np.asarray([e / (47.83 * 12) for e in EDGES_MM_H], np.float32)
    m = rng.random(a.shape) < 0.2
    a[m] = edges[rng.integers(0, len(edges), int(m.sum()))]
    return a


def _metrics_golden():
    sys.path.insert(0, REF)
    from metric.confusionmatrix import ConfusionMatrix  # noqa: E402
    from metric.iou import IoU  # noqa: E402
    res = {"K": np.int64(K), "absent": np.int64(ABSENT)}
    batches = seg_batches()
    for i, (p, t, s) in enumerate(batches):
        res[f"batch{i}/pred"], res[f"batch{i}/target"], res[f"batch{i}/scores"] = p, t, s
    counts = ConfusionMatrix(K)
    for p, t, _ in batches:
        counts.add(torch.from_numpy(p).view(-1), torch.from_numpy(t).view(-1))
    res["counts"] = counts.value().astype(np.int64)
    for tag, (normalized, ignore) in CONFIGS.items():
        for form in ("int", "scores"):
            m = IoU(K, normalized=normalized, ignore_index=ignore)
            for p, t, s in batches:
                m.add(torch.from_numpy(s if form == "scores" else p), torch.from_numpy(t))
            conf = np.array(m.conf_metric.value(), copy=True)
            iou, miou = m.value()
            res[f"{tag}/{form}/conf"], res[f"{tag}/{form}/iou"], res[f"{tag}/{form}/miou"] = conf, iou, np.float64(miou)
        assert np.array_equal(res[f"{tag}/int/iou"], res[f"{tag}/scores/iou"], equal_nan=True)
        assert np.isnan(res[f"{tag}/int/iou"][ABSENT])
    np.savez(os.path.join(GOLD, "seg_metrics.npz"), **res)
    print("wrote seg_metrics.npz", {k: res[f"{k}/int/miou"] for k in CONFIGS})


def _dataset_golden():
    seq = classification_array()
    files = {"seq.h5": {"train": {"images": seq}, "test": {"images": seq[::-1].copy()}}}
    h5 = types.ModuleType("h5py")
    h5.File = lambda name, mode="r", **kw: files[name]
    sys.modules["h5py"] = h5
    sys.path.insert(0, REF)
    from utils import dataset_precip as D  # noqa: E402
    res = {}
    for train in (True, False):
        tag = "train" if train else "test"
        ds = D.precipitation_maps_classification_h5("seq.h5", 12, 6, train=train)
        res[f"{tag}/len"] = np.int64(len(ds))
        for i in INDICES:
            x, y = ds[i]
            res[f"{tag}/{i}/x"], res[f"{tag}/{i}/y"] = x, y
    np.savez(os.path.join(GOLD, "dataset_classification.npz"), **res)
    ys = np.concatenate([res[f"train/{i}/y"].ravel() for i in INDICES])
    print("wrote dataset_classification.npz; classes seen:", np.unique(ys).tolist(), "dtype", ys.dtype)


def main():
    _metrics_golden()
    _dataset_golden()


if __name__ == "__main__":
    main()
