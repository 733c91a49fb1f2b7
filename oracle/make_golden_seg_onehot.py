"""Generate tests/golden/seg_onehot.npz from the UNMODIFIED reference metric classes -- TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_seg_onehot

The reference's ``metric.iou.IoU`` fed the batches of oracle/make_golden_seg.py with ONE-HOT (N, K, H, W) float32 targets,
in both of IoU.add's prediction forms, for every configuration of make_golden_seg.CONFIGS; and its
``metric.confusionmatrix.ConfusionMatrix`` fed (N,) predictions with (N, K) one-hot targets.  Two malformed target rows
record what the reference's one-hot checks (metric/confusionmatrix.py:57-61) do with them: a row summing to 0.9 and a row
[1.5, -0.5, 0, ...] that sums to 1 with values outside [0, 1].  The reference asserts on both.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

from oracle.make_golden_seg import CONFIGS, GOLD, K, REF, seg_batches


def onehot(t):
    """(N, H, W) int64 -> (N, K, H, W) float32 one-hot."""
    return np.moveaxis(np.eye(K, dtype=np.float32)[t], -1, 1).copy()


def bad_rows():
    """{tag: (N, K) float32 targets with one malformed row} for the ConfusionMatrix checks."""
    base = np.eye(K, dtype=np.float32)[np.arange(8) % K]
    sum09 = base.copy()
    sum09[3] = 0.0
    sum09[3, 2], sum09[3, 5] = np.float32(0.5), np.float32(0.4)
    rng = base.copy()
    rng[5] = 0.0
    rng[5, 0], rng[5, 1] = np.float32(1.5), np.float32(-0.5)
    return {"sum09": sum09, "range": rng}


def main():
    sys.path.insert(0, REF)
    from metric.confusionmatrix import ConfusionMatrix  # noqa: E402
    from metric.iou import IoU  # noqa: E402
    res = {}
    batches = seg_batches()
    for i, (_, t, _) in enumerate(batches):
        res[f"batch{i}/onehot"] = onehot(t)
    for tag, (normalized, ignore) in CONFIGS.items():
        for form in ("int", "scores"):
            m = IoU(K, normalized=normalized, ignore_index=ignore)
            for p, t, s in batches:
                m.add(torch.from_numpy(s if form == "scores" else p), torch.from_numpy(onehot(t)))
            conf = np.array(m.conf_metric.value(), copy=True)
            iou, miou = m.value()
            res[f"{tag}/{form}/conf"], res[f"{tag}/{form}/iou"], res[f"{tag}/{form}/miou"] = conf, iou, np.float64(miou)
    cm = ConfusionMatrix(K)
    for p, t, _ in batches:
        cm.add(torch.from_numpy(p).view(-1), torch.from_numpy(np.eye(K, dtype=np.float32)[t.reshape(-1)]))
    res["cm/conf"] = cm.value().astype(np.int64)
    pred8 = np.arange(8, dtype=np.int64)[::-1] % K
    res["bad/pred"] = pred8.copy()
    for tag, tgt in bad_rows().items():
        res[f"bad/{tag}/target"] = tgt
        try:
            ConfusionMatrix(K).add(torch.from_numpy(pred8.copy()), torch.from_numpy(tgt))
            raised = False
        except AssertionError:
            raised = True
        res[f"bad/{tag}/raised"] = np.bool_(raised)
        assert raised, tag
    np.savez(os.path.join(GOLD, "seg_onehot.npz"), **res)
    print("wrote seg_onehot.npz", {k: res[f"{k}/int/miou"] for k in CONFIGS})


if __name__ == "__main__":
    main()
