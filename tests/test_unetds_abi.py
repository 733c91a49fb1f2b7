"""CPU-side checks of UNetDS and UNetDSAttention4CBAMs and of the fused DS conv's max-pool epilogue: the models' state_dict keys
and parameter order against the reference's, their bf16 refusals (raised before any device work), the new entry points'
argument checks (fake aligned addresses that are never dereferenced), and the bf16 shape rule against the epilogue's
eligibility."""
import json
import os

import pytest
import torch

import smaat_unet_b200 as S
from oracle.cases import CASES, case_schema
from smaat_unet_b200.model import bf16_shape_refusal

A = 1 << 20      # fake, 16-byte aligned address
BADARG, UNSUPPORTED = -1, -3
BF = torch.bfloat16
GOLD = os.path.join(os.path.dirname(__file__), "golden")
MODELS = {"lit_ds_k1_32": S.UNetDS, "lit_dsatt4_k2_48": S.UNetDSAttention4CBAMs}


def _reference_order(n_cbams):
    """Block names in the reference classes' registration order (unet_precip_regression_lightning.py:95-104 / :175-190):
    inc, [cbam1], down1, [cbam2], ..., down4, up1-up4, outc."""
    blocks = ["inc"]
    for i in range(1, 5):
        if i <= n_cbams:
            blocks.append(f"cbam{i}")
        blocks.append(f"down{i}")
    blocks += ["up1", "up2", "up3", "up4", "outc"]
    return blocks


@pytest.mark.parametrize("name", sorted(MODELS))
def test_state_dict_and_parameter_order_are_the_references(name):
    c = CASES[name]
    model = MODELS[name](c["n_channels"], c["n_classes"], kernels_per_layer=c["k"])
    sd = model.state_dict()
    schema = case_schema(c)
    assert set(sd) == set(schema)
    assert all(tuple(sd[k].shape) == tuple(schema[k]) for k in schema)
    with open(os.path.join(GOLD, "index.json")) as f:
        assert sum(v.numel() for v in sd.values()) == json.load(f)["cases"][name]["n_params"]
    # the golden's checkpoint loads strictly
    model.load_state_dict({k: torch.zeros(tuple(s)) for k, s in schema.items()}, strict=True)
    # registration order: block by block as the reference registers them, each block's parameters in the schema's order
    blocks = _reference_order(c["n_cbams"])
    assert [n for n, _ in model.named_children()] == blocks
    names = [n for n, _ in model.named_parameters()]
    expect = [k for b in blocks for k in schema if k.split(".")[0] == b and "running_" not in k and "num_batches" not in k]
    assert names == expect


def test_smaat_unet_keeps_its_state_dict():
    """SmaAt_UNet is the same body with a CBAM on every level: its keys and their order are the 5-CBAM schema's, cbam5 after
    down4."""
    c = dict(CASES["lit_dsatt_k2_32"])
    m = S.SmaAt_UNet(c["n_channels"], c["n_classes"], kernels_per_layer=c["k"])
    assert set(m.state_dict()) == set(case_schema(c))
    assert [n for n, _ in m.named_children()] == ["inc", "cbam1", "down1", "cbam2", "down2", "cbam3", "down3", "cbam4", "down4",
                                                  "cbam5", "up1", "up2", "up3", "up4", "outc"]


def _x(shape=(2, 12, 64, 64)):
    return torch.zeros(shape, dtype=BF)


@pytest.mark.parametrize("cls", [S.UNetDS, S.UNetDSAttention4CBAMs])
def test_bf16_requests_without_a_route_raise_before_any_device_work(cls):
    model = cls(12, 1).eval()
    with torch.no_grad():
        for call in (lambda: model(_x()), lambda: model.forward_serving(_x((2, 12, 64, 48))),
                     lambda: cls(12, 1, kernels_per_layer=4).eval().forward_serving(_x()),
                     lambda: cls(12, 1, bilinear=False).eval().forward_classes(_x())):
            with pytest.raises(ValueError, match="forward_serving / forward_classes / forward_probs"):
                call()
        with pytest.raises(ValueError, match="level-3 maps are 8 wide"):
            model.forward_probs(_x((2, 12, 64, 32)))
        model.train()
        with pytest.raises(ValueError, match="train mode"):
            model.forward_serving(_x())
    model.eval()
    with pytest.raises(ValueError, match="autograd"):
        model.forward_serving(_x())
    # an admitted request goes on to the first kernel, which refuses the CPU tensor
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        model.forward_serving(_x())


def test_maxpool_entry_points_validate_their_arguments():
    lib = S._lib.load()
    mp = lambda y=A, pooled=A, W=64, k=2, mode=2, lo=A: lib.smaat_dsconv_maxpool_fwd(  # noqa: E731
        A, 64, 64 * 8 * W, None, 0, 0, A, None, A, lo, A, A, y, 64 * 8 * W, pooled, 2, 8, W, k, 64, 1, mode, None)
    assert mp(y=None) == BADARG and mp(pooled=None) == BADARG
    assert mp(pooled=A + 4) == BADARG                       # fp32 max-pool: 8-byte stores
    assert mp(mode=0) == BADARG and mp(lo=None) == BADARG   # no fp32 SIMT form; tf32x3 needs the lo parts
    assert mp(W=62) == UNSUPPORTED
    mb = lambda y=A, pooled=A, pb=1, W=64, k=2: lib.smaat_dsconv_maxpool_bf16_fwd(  # noqa: E731
        A, 64, 64 * 8 * W, None, 0, 0, A, None, A, A, A, y, 64 * 8 * W, pooled, pb, 2, 8, W, k, 64, 1, None)
    assert mb(y=None) == BADARG and mb(pooled=None) == BADARG and mb(pb=2) == BADARG
    assert mb(pooled=A + 2) == BADARG                       # bf16 max-pool: 4-byte stores
    assert mb(pooled=A + 4, pb=0) == BADARG                 # fp32 max-pool: 8-byte stores
    assert mb(W=60) == UNSUPPORTED and mb(k=4) == UNSUPPORTED
    assert b"dsconv" in lib.smaat_last_error()
    el = lambda H, W, k=2, Cout=64, mode=2: lib.smaat_dsconv_maxpool_eligible(A, 64, 64 * H * W, None, 0, 0, A, H, W, k, Cout, mode)  # noqa: E731
    assert el(288, 288) == 1 and el(36, 36, Cout=512) == 0 and el(288, 288, mode=0) == 0 and el(64, 62) == 0
    eb = lambda H, W, k=2: lib.smaat_dsconv_maxpool_bf16_eligible(A, 64, 64 * H * W, None, 0, 0, A, H, W, k, 64)  # noqa: E731
    assert eb(288, 288) == 1 and eb(288, 288, k=4) == 0 and eb(64, 60) == 0


def test_the_bf16_shape_check_admits_only_what_every_pooling_conv_takes():
    """For H, W multiples of 32 up to 640 and k = 1, 2: an input UNetDS's bf16 route admits has each of its level 1-3 producing
    convs (inc.1, down1.1, down2.1) taken by the bf16 max-pool epilogue, the only max-pool the route has for bf16 maps."""
    lib = S._lib.load()
    sizes = range(32, 641, 32)
    for k in (1, 2):
        for H in sizes:
            for W in sizes:
                if bf16_shape_refusal((2, 12, H, W)) is not None:
                    continue
                for s, C in ((1, 64), (2, 128), (4, 256)):
                    h, w = H // s, W // s
                    assert lib.smaat_dsconv_maxpool_bf16_eligible(A, C, C * h * w, None, 0, 0, A, h, w, k, C) == 1, (k, H, W, s)
