"""CPU: the dense oracles (numpy + torch port) vs the goldens of the reference's dense blocks, schemas, patching, no CPU path."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle.cases_dense import DENSE_CASES, case_schema, run_oracle, run_port, unet_schema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_dense_index_lists_every_case():
    with open(os.path.join(GOLDEN, "dense_index.json")) as f:
        assert set(json.load(f)["cases"]) == set(DENSE_CASES)
    for name in DENSE_CASES:
        assert os.path.exists(os.path.join(GOLDEN, name + ".npz")), name


@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_numpy_oracle_matches_golden_fp64(name):
    y, upd = run_oracle(name, np.float64)
    g = _golden(name)
    assert _rel(y, g["output"]) < 1e-10, name
    for k in g.files:
        if k.startswith("buf:"):
            assert np.allclose(upd[k[4:]], g[k], rtol=1e-10, atol=1e-12), (name, k)


@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_torch_port_matches_golden_fp64(name):
    assert _rel(run_port(name).numpy(), _golden(name)["output"]) < 1e-10, name


@pytest.mark.parametrize("name", ["dense_doubleconv_eval", "dense_up_pad", "dense_unet_odd", "dense_unetatt_48"])
def test_fp32_noise_of_the_oracle_is_small(name):
    """An fp32 evaluation of the same algorithm stays well inside the GPU tolerances (tests/_util.py)."""
    y, _ = run_oracle(name, np.float32)
    assert _rel(y, _golden(name)["output"]) < 1e-4, name


@pytest.mark.parametrize("name", list(DENSE_CASES))
def test_drop_in_schema_equals_reference_schema(name):
    c = DENSE_CASES[name]
    kind = c["kind"]
    if kind == "doubleconv":
        m = torch.nn.ModuleDict({"m": S.DoubleConv(c["cin"], c["cout"], c["mid"])})
    elif kind == "down":
        m = torch.nn.ModuleDict({"m": S.Down(c["cin"], c["cout"])})
    elif kind == "up":
        m = torch.nn.ModuleDict({"m": S.Up(c["cin"], c["cout"], c.get("bilinear", True))})
    elif kind == "unet":
        m = S.UNet(c["n_channels"], c["n_classes"], c.get("bilinear", True))
    else:
        m = S.UNetAttention(c["n_channels"], c["n_classes"], c.get("bilinear", True))
    sd = m.state_dict()
    schema = case_schema(c)
    assert set(sd) == set(schema)
    assert all(tuple(sd[k].shape) == tuple(schema[k]) for k in schema)


def test_network_state_dict_sizes():
    assert len(S.UNet(12, 1).state_dict()) == len(unet_schema(12, 1)) == 128
    assert len(S.UNetAttention(12, 1).state_dict()) == len(unet_schema(12, 1, attention=True)) == 178
    assert list(S.UNet(12, 1).state_dict()) == list(unet_schema(12, 1))            # registration order too


# A stand-in `models` package with the reference's import-by-name structure; its placeholder blocks refuse construction,
# so a network built after patch_reference() proves the dense names were rebound.
_PLACEHOLDER = """from torch import nn


def _placeholder(name):
    def __init__(self, *args, **kwargs):
        raise AssertionError(f"{name}: the unpatched block was constructed")
    return type(name, (nn.Module,), {"__init__": __init__})


"""
_STANDIN = {
    "__init__.py": "",
    "layers.py": _PLACEHOLDER + "\n".join(f'{n} = _placeholder("{n}")' for n in ("DepthwiseSeparableConv", "ChannelAttention", "SpatialAttention", "CBAM")),
    "unet_parts.py": _PLACEHOLDER + "\n".join(f'{n} = _placeholder("{n}")' for n in ("DoubleConv", "Down", "Up", "OutConv")),
    "unet_parts_depthwise_separable.py": _PLACEHOLDER + "\n".join(f'{n} = _placeholder("{n}")' for n in ("DepthwiseSeparableConv", "DoubleConvDS", "DownDS", "UpDS")),
    "unet_precip_regression_lightning.py": """from torch import nn
from models.unet_parts import Down, DoubleConv, Up, OutConv  # noqa: F401
from models.unet_parts_depthwise_separable import DoubleConvDS, UpDS, DownDS  # noqa: F401
from models.layers import CBAM  # noqa: F401


class UNetAttention(nn.Module):
    def __init__(self, hparams):
        super().__init__()
        h = hparams
        factor = 2 if h.bilinear else 1
        self.inc = DoubleConv(h.n_channels, 64)
        self.cbam1 = CBAM(64, reduction_ratio=h.reduction_ratio)
        self.down1 = Down(64, 128)
        self.cbam2 = CBAM(128, reduction_ratio=h.reduction_ratio)
        self.down2 = Down(128, 256)
        self.cbam3 = CBAM(256, reduction_ratio=h.reduction_ratio)
        self.down3 = Down(256, 512)
        self.cbam4 = CBAM(512, reduction_ratio=h.reduction_ratio)
        self.down4 = Down(512, 1024 // factor)
        self.cbam5 = CBAM(1024 // factor, reduction_ratio=h.reduction_ratio)
        self.up1 = Up(1024, 512 // factor, h.bilinear)
        self.up2 = Up(512, 256 // factor, h.bilinear)
        self.up3 = Up(256, 128 // factor, h.bilinear)
        self.up4 = Up(128, 64, h.bilinear)
        self.outc = OutConv(64, h.n_classes)
""",
}


@pytest.fixture
def standin_reference(tmp_path):
    root = tmp_path / "reference"
    (root / "models").mkdir(parents=True)
    for name, src in _STANDIN.items():
        (root / "models" / name).write_text(src)
    saved = {k: v for k, v in sys.modules.items() if k == "models" or k.startswith("models.")}
    for k in saved:
        del sys.modules[k]
    yield str(root)
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    if str(root) in sys.path:
        sys.path.remove(str(root))


def test_patch_reference_rebinds_the_dense_blocks(standin_reference):
    from oracle import ref_stubs
    done = S.patch_reference(standin_reference)
    assert {"DoubleConv", "Down", "Up"} <= set(done["models.unet_parts"])
    assert {"DoubleConv", "Down", "Up"} <= set(done["models.unet_precip_regression_lightning"])
    import models.unet_precip_regression_lightning as L
    m = L.UNetAttention(hparams=ref_stubs.hparams(12, 1, 1))
    assert type(m.inc) is S.DoubleConv and type(m.down4) is S.Down and type(m.up1) is S.Up
    assert len(m.state_dict()) == 178
    m.load_state_dict(S.UNetAttention(12, 1).state_dict(), strict=True)


def test_cpu_input_raises():
    m = S.DoubleConv(4, 8).eval()
    with pytest.raises(RuntimeError, match="no CPU fallback"), torch.no_grad():
        m(torch.zeros(1, 4, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"), torch.no_grad():
        S.Up(16, 8)(torch.zeros(1, 8, 4, 4), torch.zeros(1, 8, 8, 8))
