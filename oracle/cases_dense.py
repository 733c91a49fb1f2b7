"""Golden cases of the dense UNet blocks and networks -- TEST INFRASTRUCTURE ONLY.

The dense counterparts of ``oracle/cases.py``: DoubleConv / Down / Up (``models/unet_parts.py:8-64``) and the Lightning
classes UNet / UNetAttention (``models/unet_precip_regression_lightning.py:7-83``).  Kept apart from ``cases.CASES`` (whose
kinds the DS-path tests enumerate); fixtures live in ``tests/golden/dense_*.npz`` with ``tests/golden/dense_index.json``.
Deterministic values come from ``cases.fill_schema`` / ``cases.rand_input``.
"""
from __future__ import annotations

import numpy as np

from .cases import bn_schema, cast_sd, cbam_schema, fill_schema, rand_input


def conv3x3_schema(prefix, cin, cout):
    # nn.Conv2d(cin, cout, kernel_size=3, padding=1) (unet_parts.py:16,19)
    return {f"{prefix}.weight": (cout, cin, 3, 3), f"{prefix}.bias": (cout,)}


def double_conv_schema(prefix, cin, cout, mid=None):
    # models/unet_parts.py:11-22
    mid = mid or cout
    s = {}
    s.update(conv3x3_schema(f"{prefix}.double_conv.0", cin, mid))
    s.update(bn_schema(f"{prefix}.double_conv.1", mid))
    s.update(conv3x3_schema(f"{prefix}.double_conv.3", mid, cout))
    s.update(bn_schema(f"{prefix}.double_conv.4", cout))
    return s


def up_schema(prefix, cin, cout, bilinear=True):
    # models/unet_parts.py:42-51
    if bilinear:
        return double_conv_schema(f"{prefix}.conv", cin, cout, cin // 2)
    s = {f"{prefix}.up.weight": (cin, cin // 2, 2, 2), f"{prefix}.up.bias": (cin // 2,)}
    s.update(double_conv_schema(f"{prefix}.conv", cin, cout))
    return s


def unet_schema(n_channels, n_classes, bilinear=True, attention=False, r=16):
    # models/unet_precip_regression_lightning.py:14-25 (UNet), :49-65 (UNetAttention)
    factor = 2 if bilinear else 1
    chans = [64, 128, 256, 512, 1024 // factor]
    s = {}
    s.update(double_conv_schema("inc", n_channels, 64))
    for i in range(1, 5):
        s.update(double_conv_schema(f"down{i}.maxpool_conv.1", chans[i - 1], chans[i]))
    if attention:
        for i in range(5):
            s.update(cbam_schema(f"cbam{i + 1}", chans[i], r))
    for i, (cin, cout) in enumerate([(1024, 512 // factor), (512, 256 // factor), (256, 128 // factor), (128, 64)], start=1):
        s.update(up_schema(f"up{i}", cin, cout, bilinear))
    s.update({"outc.conv.weight": (n_classes, 64, 1, 1), "outc.conv.bias": (n_classes,)})
    return s


DENSE_CASES = {
    "dense_doubleconv_eval": dict(kind="doubleconv", cin=12, cout=16, mid=None, x=(2, 12, 16, 20), seed=121, train=False),
    "dense_doubleconv_mid_eval": dict(kind="doubleconv", cin=12, cout=8, mid=24, x=(2, 12, 10, 12), seed=122, train=False),
    "dense_doubleconv_train": dict(kind="doubleconv", cin=12, cout=16, mid=None, x=(3, 12, 12, 12), seed=123, train=True),
    "dense_down_odd": dict(kind="down", cin=8, cout=16, x=(2, 8, 13, 18), seed=131, train=False),
    "dense_up_even": dict(kind="up", cin=32, cout=8, x=(2, 16, 6, 8), skip=(2, 16, 12, 16), seed=141, train=False),
    "dense_up_pad": dict(kind="up", cin=32, cout=8, x=(1, 16, 4, 6), skip=(1, 16, 9, 13), seed=142, train=False),
    # Up(bilinear=False): ConvTranspose2d(in, in // 2, 2, 2) (unet_parts.py:50-51); x has `cin` channels, the skip cin // 2
    "dense_up_convt_even": dict(kind="up", cin=32, cout=8, x=(2, 32, 6, 8), skip=(2, 16, 12, 16), seed=143, train=False, bilinear=False),
    "dense_up_convt_train": dict(kind="up", cin=16, cout=8, x=(2, 16, 4, 4), skip=(2, 8, 8, 8), seed=144, train=True, bilinear=False),
    "dense_unet_32": dict(kind="unet", n_channels=12, n_classes=1, x=(2, 12, 32, 32), seed=151, train=False),
    "dense_unet_odd": dict(kind="unet", n_channels=12, n_classes=1, x=(1, 12, 36, 52), seed=152, train=False),
    "dense_unet_train": dict(kind="unet", n_channels=12, n_classes=1, x=(2, 12, 32, 32), seed=153, train=True),
    "dense_unet_convt": dict(kind="unet", n_channels=12, n_classes=1, x=(1, 12, 32, 32), seed=154, train=False, bilinear=False),
    "dense_unetatt_32": dict(kind="unetatt", n_channels=12, n_classes=1, x=(2, 12, 32, 32), seed=161, train=False),
    "dense_unetatt_48": dict(kind="unetatt", n_channels=12, n_classes=1, x=(1, 12, 48, 48), seed=162, train=False),
}


def case_schema(c):
    kind = c["kind"]
    if kind == "doubleconv":
        return double_conv_schema("m", c["cin"], c["cout"], c["mid"])
    if kind == "down":
        return double_conv_schema("m.maxpool_conv.1", c["cin"], c["cout"])
    if kind == "up":
        return up_schema("m", c["cin"], c["cout"], c.get("bilinear", True))
    if kind in ("unet", "unetatt"):
        return unet_schema(c["n_channels"], c["n_classes"], c.get("bilinear", True), attention=kind == "unetatt")
    raise KeyError(kind)


def case_tensors(name, dtype=np.float64):
    """(state_dict, inputs) for a dense case, as numpy arrays of ``dtype``."""
    c = DENSE_CASES[name]
    sd = cast_sd(fill_schema(case_schema(c), c["seed"]), dtype)
    lo = 0.0 if c["kind"] in ("unet", "unetatt") else -1.0
    xs = [rand_input(c["x"], c["seed"] + 1000, lo, 1.0).astype(dtype)]
    if "skip" in c:
        xs.append(rand_input(c["skip"], c["seed"] + 2000, -1.0, 1.0).astype(dtype))
    return sd, xs


def run_oracle(name, dtype=np.float64):
    """Run the numpy dense oracle on a case; returns (output, running-stat updates)."""
    from . import dense_oracle as D
    c = DENSE_CASES[name]
    sd, xs = case_tensors(name, dtype)
    kind, train = c["kind"], c.get("train", False)
    if kind == "doubleconv":
        return D.double_conv(xs[0], sd, "m", train)
    if kind == "down":
        return D.down(xs[0], sd, "m", train)
    if kind == "up":
        return D.up(xs[0], xs[1], sd, "m", train)
    if kind in ("unet", "unetatt"):
        return D.unet_forward(xs[0], sd, train, attention=kind == "unetatt")
    raise KeyError(kind)


def run_port(name, dtype=None):
    """Run the torch-functional dense port on a case (CPU, float64 by default); returns the output tensor."""
    import torch

    from . import dense_oracle as D
    from .torch_port import to_torch_sd
    dtype = dtype or torch.float64
    c = DENSE_CASES[name]
    sd, xs = case_tensors(name, np.float64)
    sd = to_torch_sd(sd, dtype)
    xs = [torch.from_numpy(x).to(dtype) for x in xs]
    kind, train = c["kind"], c.get("train", False)
    if kind == "doubleconv":
        return D.port_double_conv(xs[0], sd, "m", train)
    if kind == "down":
        return D.port_down(xs[0], sd, "m", train)
    if kind == "up":
        return D.port_up(xs[0], xs[1], sd, "m", train)
    return D.port_unet_forward(xs[0], sd, train, attention=kind == "unetatt")
