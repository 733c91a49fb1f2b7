"""Deterministic, machine-portable parity cases -- TEST INFRASTRUCTURE ONLY.

Parameters and inputs are drawn from ``numpy.random.default_rng(seed)`` (PCG64:
bit-identical on every machine), so the GPU box can rebuild the exact tensors
the golden outputs under ``tests/golden/`` were produced from without having
/root/reference.  The state_dict schemas below restate the reference's key
names and shapes (SURVEY 8b); ``oracle/make_golden.py`` asserts they equal the
live reference modules' ``state_dict()`` before writing any fixture.
"""
from __future__ import annotations

import numpy as np


# ----------------------------------------------------------------------------
# state_dict schemas (key -> shape), reference naming
# ----------------------------------------------------------------------------
def ds_conv_schema(prefix, cin, cout, k):
    # models/layers.py:38-45
    return {
        f"{prefix}.depthwise.weight": (k * cin, 1, 3, 3),
        f"{prefix}.depthwise.bias": (k * cin,),
        f"{prefix}.pointwise.weight": (cout, k * cin, 1, 1),
        f"{prefix}.pointwise.bias": (cout,),
    }


def bn_schema(prefix, c):
    return {
        f"{prefix}.weight": (c,), f"{prefix}.bias": (c,),
        f"{prefix}.running_mean": (c,), f"{prefix}.running_var": (c,),
        f"{prefix}.num_batches_tracked": (),
    }


def double_conv_ds_schema(prefix, cin, cout, mid=None, k=1):
    # models/unet_parts_depthwise_separable.py:13-36
    mid = mid or cout
    s = {}
    s.update(ds_conv_schema(f"{prefix}.double_conv.0", cin, mid, k))
    s.update(bn_schema(f"{prefix}.double_conv.1", mid))
    s.update(ds_conv_schema(f"{prefix}.double_conv.3", mid, cout, k))
    s.update(bn_schema(f"{prefix}.double_conv.4", cout))
    return s


def cbam_schema(prefix, c, r=16, ks=7):
    # models/layers.py:94-103,119-120
    s = {
        f"{prefix}.channel_att.MLP.1.weight": (c // r, c), f"{prefix}.channel_att.MLP.1.bias": (c // r,),
        f"{prefix}.channel_att.MLP.3.weight": (c, c // r), f"{prefix}.channel_att.MLP.3.bias": (c,),
        f"{prefix}.spatial_att.conv.weight": (1, 2, ks, ks),
    }
    s.update(bn_schema(f"{prefix}.spatial_att.bn", 1))
    return s


def smaat_unet_schema(n_channels, n_classes, k=2, r=16, n_cbams=5, bilinear=True):
    # models/SmaAt_UNet.py:23-39 (bilinear=True -> factor 2); n_cbams = 4 / 0: the Lightning variants
    # UNetDSAttention4CBAMs / UNetDS (models/unet_precip_regression_lightning.py:167-208, 86-117).  bilinear=False: factor 1
    # (x5 is 1024 channels wide) and each UpDS upsamples with ConvTranspose2d(in, in // 2, 2, 2) (parts_ds.py:72-73)
    factor = 2 if bilinear else 1
    s = {}
    s.update(double_conv_ds_schema("inc", n_channels, 64, None, k))
    chans = [64, 128, 256, 512, 1024 // factor]
    for i in range(n_cbams):
        s.update(cbam_schema(f"cbam{i + 1}", chans[i], r))
    for i in range(1, 5):
        s.update(double_conv_ds_schema(f"down{i}.maxpool_conv.1", chans[i - 1], chans[i], None, k))
    ups = [(1024, 512 // factor), (512, 256 // factor), (256, 128 // factor), (128, 64)]
    for i, (cin, cout) in enumerate(ups, start=1):
        if not bilinear:
            s.update({f"up{i}.up.weight": (cin, cin // 2, 2, 2), f"up{i}.up.bias": (cin // 2,)})
        s.update(double_conv_ds_schema(f"up{i}.conv", cin, cout, cin // 2 if bilinear else None, k))
    s.update({"outc.conv.weight": (n_classes, 64, 1, 1), "outc.conv.bias": (n_classes,)})
    return s


# ----------------------------------------------------------------------------
# deterministic values
# ----------------------------------------------------------------------------
def fill_schema(schema, seed):
    """float64 numpy state_dict: conv/linear ~ U(-1/sqrt(fan_in), +), BN randomised so
    eval-mode BN is not the identity (SURVEY 8d)."""
    rng = np.random.default_rng(seed)
    sd = {}
    for key, shape in schema.items():
        leaf = key.rsplit(".", 1)[-1]
        is_bn = (key.rsplit(".", 1)[0] + ".running_mean") in schema
        if leaf == "num_batches_tracked":
            sd[key] = np.zeros((), dtype=np.int64)
        elif leaf == "running_mean":
            sd[key] = rng.normal(0.0, 0.1, shape)
        elif leaf == "running_var":
            sd[key] = rng.uniform(0.5, 1.5, shape)
        elif is_bn and leaf == "weight":
            sd[key] = rng.uniform(0.5, 1.5, shape)
        elif is_bn and leaf == "bias":
            sd[key] = rng.normal(0.0, 0.1, shape)
        elif leaf == "weight":
            fan_in = int(np.prod(shape[1:])) if len(shape) > 1 else shape[0]
            a = 1.0 / np.sqrt(fan_in)
            sd[key] = rng.uniform(-a, a, shape)
        else:  # conv / linear bias
            sd[key] = rng.uniform(-0.2, 0.2, shape)
    return sd


def rand_input(shape, seed, lo=0.0, hi=1.0):
    """Radar maps are min-max normalised to [0,1] (README.md:102); signed range used for mid-network ops."""
    return np.random.default_rng(seed).uniform(lo, hi, shape)


def cast_sd(sd, dtype):
    return {k: (v if v.dtype == np.int64 else v.astype(dtype)) for k, v in sd.items()}


# ----------------------------------------------------------------------------
# the cases.  kind selects the reference module built by make_golden.py and the
# oracle function called by the tests.
# ----------------------------------------------------------------------------
CASES = {
    # --- leaf / block level ---------------------------------------------------
    "dsconv_k1": dict(kind="dsconv", cin=5, cout=7, k=1, x=(2, 5, 9, 11), seed=11),
    "dsconv_k2": dict(kind="dsconv", cin=6, cout=8, k=2, x=(2, 6, 12, 8), seed=12),
    "dsconv_k3": dict(kind="dsconv", cin=4, cout=16, k=3, x=(1, 4, 7, 5), seed=13),
    "doubleconv_eval": dict(kind="doubleconv", cin=12, cout=16, mid=None, k=2, x=(2, 12, 16, 20), seed=21, train=False),
    "doubleconv_mid_eval": dict(kind="doubleconv", cin=16, cout=8, mid=8, k=2, x=(2, 16, 10, 10), seed=22, train=False),
    "doubleconv_train": dict(kind="doubleconv", cin=8, cout=16, mid=None, k=2, x=(3, 8, 12, 12), seed=23, train=True),
    "down_eval": dict(kind="down", cin=8, cout=16, k=2, x=(2, 8, 13, 18), seed=31, train=False),
    "up_eval_even": dict(kind="up", cin=32, cout=8, k=2, x=(2, 16, 6, 8), skip=(2, 16, 12, 16), seed=41, train=False),
    "up_eval_pad": dict(kind="up", cin=32, cout=8, k=1, x=(1, 16, 4, 6), skip=(1, 16, 9, 13), seed=42, train=False),
    # UpDS(bilinear=False): ConvTranspose2d(in, in // 2, 2, 2) upsampling (parts_ds.py:72-73); x has `cin` channels, the skip cin // 2
    "up_convt_even": dict(kind="up", cin=32, cout=8, k=2, x=(2, 32, 6, 8), skip=(2, 16, 12, 16), seed=43, train=False, bilinear=False),
    "up_convt_pad": dict(kind="up", cin=16, cout=8, k=1, x=(1, 16, 4, 6), skip=(1, 8, 9, 13), seed=44, train=False, bilinear=False),
    "up_convt_train": dict(kind="up", cin=16, cout=8, k=2, x=(2, 16, 4, 4), skip=(2, 8, 8, 8), seed=45, train=True, bilinear=False),
    "cbam_k7_eval": dict(kind="cbam", c=32, r=16, ks=7, x=(2, 32, 14, 10), seed=51, train=False),
    "cbam_k3_eval": dict(kind="cbam", c=64, r=8, ks=3, x=(1, 64, 9, 9), seed=52, train=False),
    "cbam_k7_train": dict(kind="cbam", c=32, r=16, ks=7, x=(3, 32, 12, 12), seed=53, train=True),
    "outconv": dict(kind="outconv", cin=64, cout=3, x=(2, 64, 8, 8), seed=61),
    # --- BASELINE.json configs[0]: DoubleConvDS+CBAM, B=1, 64ch, 64x64 -------------
    "config1_block": dict(kind="config1", c=64, k=2, x=(1, 64, 64, 64), seed=71, train=False, store="f4"),
    # --- full model (SmaAt_UNet.py:41-57) ------------------------------------------
    "unet_12_1_k2_32": dict(kind="unet", n_channels=12, n_classes=1, k=2, x=(2, 12, 32, 32), seed=81, train=False),
    "unet_12_1_k2_odd": dict(kind="unet", n_channels=12, n_classes=1, k=2, x=(1, 12, 36, 52), seed=82, train=False),
    "unet_3_5_k1_48": dict(kind="unet", n_channels=3, n_classes=5, k=1, x=(2, 3, 48, 48), seed=83, train=False),
    "unet_12_1_k2_train": dict(kind="unet", n_channels=12, n_classes=1, k=2, x=(2, 12, 32, 32), seed=84, train=True),
    # the Lightning wrappers' own forward bodies (models/unet_precip_regression_lightning.py): UNetDSAttention (:148-164),
    # UNetDSAttention4CBAMs (:193-208, x5 goes to the decoder un-attended), UNetDS (:104-117, no CBAM)
    "lit_dsatt_k2_32": dict(kind="lit", cls="UNetDSAttention", n_cbams=5, n_channels=12, n_classes=1, k=2, x=(2, 12, 32, 32), seed=91, train=False),
    "lit_dsatt4_k2_48": dict(kind="lit", cls="UNetDSAttention4CBAMs", n_cbams=4, n_channels=12, n_classes=1, k=2, x=(1, 12, 48, 48), seed=92, train=False),
    "lit_ds_k1_32": dict(kind="lit", cls="UNetDS", n_cbams=0, n_channels=12, n_classes=1, k=1, x=(2, 12, 32, 32), seed=93, train=False),
}


def case_schema(c):
    kind = c["kind"]
    if kind == "dsconv":
        return ds_conv_schema("m", c["cin"], c["cout"], c["k"])
    if kind == "doubleconv":
        return double_conv_ds_schema("m", c["cin"], c["cout"], c["mid"], c["k"])
    if kind == "down":
        return double_conv_ds_schema("m.maxpool_conv.1", c["cin"], c["cout"], None, c["k"])
    if kind == "up":
        if not c.get("bilinear", True):      # parts_ds.py:72-73: ConvTranspose2d(in, in // 2, 2, 2) + DoubleConvDS(in, out)
            s = {"m.up.weight": (c["cin"], c["cin"] // 2, 2, 2), "m.up.bias": (c["cin"] // 2,)}
            s.update(double_conv_ds_schema("m.conv", c["cin"], c["cout"], None, c["k"]))
            return s
        return double_conv_ds_schema("m.conv", c["cin"], c["cout"], c["cin"] // 2, c["k"])
    if kind == "cbam":
        return cbam_schema("m", c["c"], c["r"], c["ks"])
    if kind == "outconv":
        return {"m.conv.weight": (c["cout"], c["cin"], 1, 1), "m.conv.bias": (c["cout"],)}
    if kind == "config1":
        s = double_conv_ds_schema("conv", c["c"], c["c"], None, c["k"])
        s.update(cbam_schema("cbam", c["c"]))
        return s
    if kind == "unet":
        return smaat_unet_schema(c["n_channels"], c["n_classes"], c["k"])
    if kind == "lit":
        return smaat_unet_schema(c["n_channels"], c["n_classes"], c["k"], n_cbams=c["n_cbams"])
    raise KeyError(kind)


def case_tensors(name, dtype=np.float64):
    """(state_dict, inputs) for a case, as numpy arrays of ``dtype``."""
    c = CASES[name]
    sd = cast_sd(fill_schema(case_schema(c), c["seed"]), dtype)
    lo = 0.0 if c["kind"] in ("unet", "lit") else -1.0
    xs = [rand_input(c["x"], c["seed"] + 1000, lo, 1.0).astype(dtype)]
    if "skip" in c:
        xs.append(rand_input(c["skip"], c["seed"] + 2000, -1.0, 1.0).astype(dtype))
    return sd, xs


def run_oracle(name, dtype=np.float64):
    """Run the numpy oracle on a case; returns (output, running-stat updates)."""
    from . import smaat_oracle as O
    c = CASES[name]
    sd, xs = case_tensors(name, dtype)
    kind, train = c["kind"], c.get("train", False)
    if kind == "dsconv":
        return O.ds_conv(xs[0], sd, "m", c["k"]), {}
    if kind == "doubleconv":
        return O.double_conv_ds(xs[0], sd, "m", c["k"], train)
    if kind == "down":
        return O.down_ds(xs[0], sd, "m", c["k"], train)
    if kind == "up":
        return O.up_ds(xs[0], xs[1], sd, "m", c["k"], train)
    if kind == "cbam":
        return O.cbam(xs[0], sd, "m", train)
    if kind == "outconv":
        return O.out_conv(xs[0], sd, "m"), {}
    if kind == "config1":
        y, u = O.double_conv_ds(xs[0], sd, "conv", c["k"], train)
        y, u2 = O.cbam(y, sd, "cbam", train)
        u.update(u2)
        return y, u
    if kind == "unet":
        return O.smaat_unet_forward(xs[0], sd, c["k"], train, return_updates=True)
    if kind == "lit":
        return O.smaat_unet_forward(xs[0], sd, c["k"], train, return_updates=True, n_cbams=c["n_cbams"])
    raise KeyError(kind)
