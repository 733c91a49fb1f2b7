"""Generate tests/golden/dense_*.npz by running the UNMODIFIED reference's dense blocks -- TEST INFRASTRUCTURE ONLY.

Run where the reference checkout exists (``SMAAT_REFERENCE``, default /root/reference):

    python -m oracle.make_golden_dense

For every case in ``oracle/cases_dense.py`` this builds the reference's own DoubleConv / Down / Up
(models/unet_parts.py) or its Lightning UNet / UNetAttention (models/unet_precip_regression_lightning.py, under the import
stand-ins of oracle/ref_stubs.py), checks its ``state_dict()`` keys and shapes against the restated schema, loads the
deterministic float64 parameters, runs the reference forward in float64, and stores the output (and, for train-mode
cases, the BatchNorm buffers after the step) plus ``dense_index.json``.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

REF = os.environ.get("SMAAT_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def build_reference_module(c):
    sys.path.insert(0, REF)
    from models.unet_parts import DoubleConv, Down, Up          # noqa: E402

    class Wrap(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, *a):
            return self.m(*a)

    kind = c["kind"]
    if kind == "doubleconv":
        return Wrap(DoubleConv(c["cin"], c["cout"], c["mid"]))
    if kind == "down":
        return Wrap(Down(c["cin"], c["cout"]))
    if kind == "up":
        return Wrap(Up(c["cin"], c["cout"], c.get("bilinear", True)))
    if kind in ("unet", "unetatt"):
        from oracle import ref_stubs
        ref_stubs.install()
        import models.unet_precip_regression_lightning as L      # noqa: E402
        cls = L.UNet if kind == "unet" else L.UNetAttention
        return cls(hparams=ref_stubs.hparams(c["n_channels"], c["n_classes"], 1, bilinear=c.get("bilinear", True)))
    raise KeyError(kind)


def main():
    from oracle.cases_dense import DENSE_CASES, case_schema, case_tensors
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    index = {}
    for name, c in DENSE_CASES.items():
        mod = build_reference_module(c).double()
        ref_sd = mod.state_dict()
        schema = case_schema(c)
        assert set(ref_sd) == set(schema), (name, set(ref_sd) ^ set(schema))
        for k, v in ref_sd.items():
            assert tuple(v.shape) == tuple(schema[k]), (name, k, tuple(v.shape), schema[k])
        sd, xs = case_tensors(name, np.float64)
        mod.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
        train = c.get("train", False)
        mod.train(train)
        with torch.no_grad():
            y = mod(*[torch.from_numpy(x) for x in xs])
        index[name] = {"output_shape": list(y.shape), "train": train, "abs_max": float(y.abs().max()),
                       "n_state": len(schema)}
        arrays = {"output": y.numpy()}
        if train:
            for k, v in mod.state_dict().items():
                if k.endswith(("running_mean", "running_var", "num_batches_tracked")):
                    arrays["buf:" + k] = v.numpy()
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **arrays)
        print(f"{name:28s} out={tuple(y.shape)} absmax={index[name]['abs_max']:.4f}")
    meta = {"reference": "HansBambel/SmaAt-UNet (models/unet_parts.py, models/unet_precip_regression_lightning.py)",
            "torch": torch.__version__, "reference_pins_torch": "2.6.0", "dtype": "float64", "cases": index}
    with open(os.path.join(OUT, "dense_index.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
