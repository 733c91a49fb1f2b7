"""The oracle is only trustworthy once pinned: numpy oracle and torch port vs the
golden outputs produced by the UNMODIFIED reference (oracle/make_golden.py)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import torch_port as TP
from oracle.cases import CASES, case_schema, case_tensors, run_oracle

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def test_index_lists_every_case():
    with open(os.path.join(GOLD, "index.json")) as f:
        idx = json.load(f)
    assert set(idx["cases"]) == set(CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_numpy_oracle_fp64_matches_reference(name):
    y, upd = run_oracle(name, np.float64)
    g = _gold(name)
    ref = g["output"].astype(np.float64)
    tol = 2e-7 if CASES[name].get("store") == "f4" else 1e-11   # f4 fixture: rounding of the stored value
    assert y.shape == ref.shape
    assert np.abs(y - ref).max() <= tol * max(1.0, np.abs(ref).max())
    for k in g.files:
        if k.startswith("buf:"):
            got = np.asarray(upd[k[4:]], dtype=np.float64)
            assert np.abs(got - g[k]).max() <= 1e-12, k


@pytest.mark.parametrize("name", sorted(CASES))
def test_numpy_oracle_fp32_within_fp32_noise(name):
    """fp32 evaluation of the same algorithm: sets the noise floor the CUDA path is held to."""
    y, _ = run_oracle(name, np.float32)
    ref = _gold(name)["output"].astype(np.float64)
    tol = 2e-4 if CASES[name].get("train") else 2e-5
    assert np.abs(y - ref).max() <= tol * max(1.0, np.abs(ref).max())


_RUN = {
    "dsconv": lambda c, sd, xs: TP.ds_conv(xs[0], sd, "m"),
    "doubleconv": lambda c, sd, xs: TP.double_conv_ds(xs[0], sd, "m", c.get("train", False)),
    "down": lambda c, sd, xs: TP.down_ds(xs[0], sd, "m", c.get("train", False)),
    "up": lambda c, sd, xs: TP.up_ds(xs[0], xs[1], sd, "m", c.get("train", False)),
    "cbam": lambda c, sd, xs: TP.cbam(xs[0], sd, "m", c.get("train", False)),
    "outconv": lambda c, sd, xs: torch.nn.functional.conv2d(xs[0], sd["m.conv.weight"], sd["m.conv.bias"]),
    "config1": lambda c, sd, xs: TP.cbam(TP.double_conv_ds(xs[0], sd, "conv"), sd, "cbam"),
    "unet": lambda c, sd, xs: TP.smaat_unet_forward(xs[0], sd, c.get("train", False)),
    "lit": lambda c, sd, xs: TP.smaat_unet_forward(xs[0], sd, c.get("train", False), n_cbams=c["n_cbams"]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_torch_port_fp64_matches_reference(name):
    c = CASES[name]
    sd_np, xs_np = case_tensors(name, np.float64)
    sd = TP.to_torch_sd(sd_np, torch.float64)
    xs = [torch.from_numpy(x) for x in xs_np]
    with torch.no_grad():
        y = _RUN[c["kind"]](c, sd, xs).numpy()
    g = _gold(name)
    ref = g["output"].astype(np.float64)
    tol = 2e-7 if c.get("store") == "f4" else 1e-11
    assert np.abs(y - ref).max() <= tol * max(1.0, np.abs(ref).max())
    for k in g.files:                       # F.batch_norm updates running stats in place
        if k.startswith("buf:") and not k.endswith("num_batches_tracked"):
            assert np.abs(sd[k[4:]].numpy() - g[k]).max() <= 1e-12, k


def _cbam_with_reference_pools(x, sd, p, training, split_ties=False):
    """CBAM (reference models/layers.py:105-141) restated with the reference's own pooling modules / calls:
    nn.AdaptiveAvgPool2d(1), nn.AdaptiveMaxPool2d(1) + Flatten, torch.mean / torch.max(dim=1).
    ``split_ties`` swaps both max pools for Tensor.amax (same values, tied gradients split evenly)."""
    F = torch.nn.functional
    ca = p + ".channel_att.MLP"

    def mlp(v):
        v = torch.flatten(v, 1)
        return F.linear(F.relu(F.linear(v, sd[ca + ".1.weight"], sd[ca + ".1.bias"])), sd[ca + ".3.weight"], sd[ca + ".3.bias"])

    mx = x.amax(dim=(2, 3)) if split_ties else torch.nn.AdaptiveMaxPool2d(1)(x)
    out = mlp(torch.nn.AdaptiveAvgPool2d(1)(x)) + mlp(mx)
    x = x * torch.sigmoid(out).unsqueeze(2).unsqueeze(3).expand_as(x)
    avg_out = torch.mean(x, dim=1, keepdim=True)
    max_out = x.amax(dim=1, keepdim=True) if split_ties else torch.max(x, dim=1, keepdim=True)[0]
    w = sd[p + ".spatial_att.conv.weight"]
    a = F.conv2d(torch.cat([avg_out, max_out], dim=1), w, None, padding=w.shape[-1] // 2)
    a = F.batch_norm(a, sd[p + ".spatial_att.bn.running_mean"], sd[p + ".spatial_att.bn.running_var"],
                     sd[p + ".spatial_att.bn.weight"], sd[p + ".spatial_att.bn.bias"], training=training, momentum=0.1, eps=1e-5)
    return x * torch.sigmoid(a)


def _cbam_tie_case():
    """A CBAM input full of tied maxima: relu(N(0,1)) (about half exact zeros), two dead pixels (all channels 0), a dead
    plane (one channel 0 everywhere) and a plane whose maximum sits at two positions."""
    g = torch.Generator().manual_seed(2024)
    B, C, H, W, hidden = 2, 32, 6, 7, 2
    x = torch.relu(torch.randn(B, C, H, W, generator=g, dtype=torch.float64))
    x[0, :, 1, 2] = 0.0
    x[1, :, 4, 6] = 0.0
    x[1, 5] = 0.0
    x[0, 9, 2, 3] = x[0, 9, 5, 0] = x[0, 9].max() + 1.0
    sd = {
        "m.channel_att.MLP.1.weight": torch.randn(hidden, C, generator=g, dtype=torch.float64) * 0.3,
        "m.channel_att.MLP.1.bias": torch.randn(hidden, generator=g, dtype=torch.float64) * 0.1 + 0.5,
        "m.channel_att.MLP.3.weight": torch.randn(C, hidden, generator=g, dtype=torch.float64) * 0.3,
        "m.channel_att.MLP.3.bias": torch.randn(C, generator=g, dtype=torch.float64) * 0.1,
        "m.spatial_att.conv.weight": torch.randn(1, 2, 7, 7, generator=g, dtype=torch.float64) * 0.2,
        "m.spatial_att.bn.weight": torch.tensor([1.3], dtype=torch.float64),
        "m.spatial_att.bn.bias": torch.tensor([-0.2], dtype=torch.float64),
        "m.spatial_att.bn.running_mean": torch.zeros(1, dtype=torch.float64),
        "m.spatial_att.bn.running_var": torch.ones(1, dtype=torch.float64),
    }
    gout = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    return x, sd, gout


def _cbam_grads(fn, x, sd, gout, training, **kw):
    sd = {k: v.clone() for k, v in sd.items()}
    names = ["m.channel_att.MLP.1.weight", "m.channel_att.MLP.1.bias", "m.channel_att.MLP.3.weight", "m.channel_att.MLP.3.bias",
             "m.spatial_att.conv.weight", "m.spatial_att.bn.weight", "m.spatial_att.bn.bias"]
    for k in names:
        sd[k].requires_grad_(True)
    xi = x.clone().requires_grad_(True)
    y = fn(xi, sd, "m", training, **kw)
    y.backward(gout)
    return y.detach(), [xi.grad] + [sd[k].grad for k in names]


@pytest.mark.parametrize("training", [False, True])
def test_torch_port_cbam_routes_max_ties_like_reference(training):
    """The port is the gradient oracle of the CBAM backward kernels, so its max pools must route ties the reference's way:
    all of the gradient to one index (nn.AdaptiveMaxPool2d(1), torch.max(dim=1)), not split evenly as Tensor.amax does."""
    x, sd, gout = _cbam_tie_case()
    y_ref, g_ref = _cbam_grads(_cbam_with_reference_pools, x, sd, gout, training)
    y, g = _cbam_grads(TP.cbam, x, sd, gout, training)
    assert torch.equal(y, y_ref)
    for i, (a, b) in enumerate(zip(g, g_ref)):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-12), i

    # the case is discriminating: splitting the tied gradients (Tensor.amax) changes the input gradient
    _, g_split = _cbam_grads(_cbam_with_reference_pools, x, sd, gout, training, split_ties=True)
    assert not torch.allclose(g_split[0], g_ref[0], rtol=1e-6, atol=1e-9)


def test_schema_param_count_matches_survey():
    # SURVEY section 6: SmaAt_UNet(12,1,kpl=2) has 4 033 537 trainable parameters, 214 state_dict entries
    s = case_schema(CASES["unet_12_1_k2_32"])
    assert len(s) == 214
    n = sum(int(np.prod(v)) for k, v in s.items()
            if not k.endswith(("running_mean", "running_var", "num_batches_tracked")))
    assert n == 4_033_537
