"""Generate tests/golden/precip_eval.npz from the UNMODIFIED reference classes -- TEST INFRASTRUCTURE ONLY.

    python -m oracle.make_golden_eval

What calc_metrics_test_set.py computes for the persistence baseline, at its batch size of 1: the reference's
``PersistenceModel.forward`` (models/regression_lightning.py:202-204, built under the stand-ins of oracle/ref_stubs.py) on
each sample of ``sweep_oracle.eval_samples()``, and one unmodified ``PrecipitationMetrics`` per threshold
(metric/precipitation_metrics.py, under the torchmetrics stand-in) updated one sample at a time, for thresholds
0.5 / 1 / 2 / 5 / 10 / 30 and both ``denormalize`` settings.  Stores the samples, ``compute()`` and the integer states.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

from oracle import ref_stubs
from oracle.sweep_oracle import GOLDEN_THRESHOLDS, eval_samples

REF = os.environ.get("SMAAT_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "precip_eval.npz")
COUNTS = ("total_tp", "total_fp", "total_tn", "total_fn", "total_samples", "total_pixels")


def main():
    ref_stubs.install()
    sys.path.insert(0, REF)
    from metric.precipitation_metrics import PrecipitationMetrics  # noqa: E402
    from models.regression_lightning import PersistenceModel  # noqa: E402

    x, y = eval_samples()
    model = PersistenceModel(argparse.Namespace())
    res = {"x": x, "y": y, "thresholds": np.asarray(GOLDEN_THRESHOLDS, np.float64)}
    for denorm in (True, False):
        tag = "denorm" if denorm else "norm"
        for t in GOLDEN_THRESHOLDS:
            m = PrecipitationMetrics(threshold=t, denormalize=denorm)
            for i in range(len(x)):                      # DataLoader(batch_size=1): one sample per test_step
                xb, yb = torch.from_numpy(x[i:i + 1]), torch.from_numpy(y[i:i + 1])
                m.update(model(xb).detach(), yb.detach())
            for k, v in m.compute().items():
                res[f"{tag}/{t}/{k}"] = np.float64(float(v))
            for k in COUNTS:
                res[f"{tag}/{t}/{k}"] = np.int64(int(getattr(m, k)))
    np.savez(OUT, **res)
    print("wrote", OUT, {k: v.tolist() for k, v in res.items() if k.startswith("denorm/0.5/")})


if __name__ == "__main__":
    main()
