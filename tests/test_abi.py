"""CPU-side checks of the boundary: the C-ABI library loads and exports every symbol the
header declares; host-side module logic (constructors, state_dict schema, loud failure)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle.cases import CASES, case_schema

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "smaat_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(smaat_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(S._lib.LIB_PATH)
    syms = _header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/smaat_b200.h but not exported"


def test_binding_table_matches_header():
    assert _header_symbols() == S._lib.EXPORTED


def test_abi_version_and_error_string():
    lib = S._lib.load()
    assert lib.smaat_abi_version() == 3
    # argument validation happens on the host before any CUDA call: usable without a GPU
    rc = lib.smaat_maxpool2_fwd(None, None, 1, 4, 4, None)
    assert rc == -1 and b"maxpool2" in lib.smaat_last_error()
    rc = lib.smaat_cbam_gate_fwd(1, 1, None, 1, None, 1, 8, 8, 5, None)
    assert rc == -1 and b"kernel size must be 3 or 7" in lib.smaat_last_error()


@pytest.mark.parametrize("args", [(12, 1, 2, 16), (3, 21, 1, 8)])
def test_model_state_dict_schema_matches_reference_schema(args):
    n_ch, n_cls, k, r = args
    from oracle.cases import smaat_unet_schema
    m = S.SmaAt_UNet(n_ch, n_cls, kernels_per_layer=k, reduction_ratio=r)
    sd = m.state_dict()
    schema = smaat_unet_schema(n_ch, n_cls, k, r)
    assert set(sd) == set(schema)
    for key, shape in schema.items():
        assert tuple(sd[key].shape) == tuple(shape), key


def test_block_schemas_match():
    for name, c in CASES.items():
        schema = case_schema(c)
        kind = c["kind"]
        if kind == "dsconv":
            m = S.DepthwiseSeparableConv(c["cin"], c["cout"], 3, padding=1, kernels_per_layer=c["k"])
        elif kind == "doubleconv":
            m = S.DoubleConvDS(c["cin"], c["cout"], c["mid"], kernels_per_layer=c["k"])
        elif kind == "down":
            m = S.DownDS(c["cin"], c["cout"], kernels_per_layer=c["k"])
        elif kind == "up":
            m = S.UpDS(c["cin"], c["cout"], c.get("bilinear", True), kernels_per_layer=c["k"])
        elif kind == "cbam":
            m = S.CBAM(c["c"], reduction_ratio=c["r"], kernel_size=c["ks"])
        elif kind == "outconv":
            m = S.OutConv(c["cin"], c["cout"])
        else:
            continue
        got = {"m." + k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert got == {k: tuple(v) for k, v in schema.items()}, name


def test_no_cpu_fallback_fails_loudly():
    m = S.SmaAt_UNet(12, 1).eval()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.zeros(1, 12, 32, 32))
    with pytest.raises(RuntimeError, match="no CPU fallback"), torch.no_grad():      # the ConvTranspose2d branch too
        S.UpDS(8, 4, bilinear=False).eval()(torch.zeros(1, 8, 4, 4), torch.zeros(1, 4, 8, 8))


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "smaat_unet_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("# oracle", ""), f"{fn} references the oracle"


# A stand-in for the reference's `models` package with its import structure: every module imports the block classes BY NAME
# (models/SmaAt_UNet.py:2-4, unet_precip_regression_lightning.py:1-3), and the placeholder blocks refuse to be constructed,
# so a model built after patch_reference() proves that each module's names were rebound.  The assemblies restate the
# constructors the repository already restates in smaat_unet_b200/model.py.
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
    "unet_parts_depthwise_separable.py": "from models.layers import DepthwiseSeparableConv  # noqa: F401\n" + _PLACEHOLDER
    + "\n".join(f'{n} = _placeholder("{n}")' for n in ("DoubleConvDS", "DownDS", "UpDS")),
    "_assemble.py": """def assemble(m, g, n_channels, n_classes, k, bilinear, r, n_cbams):
    # g: the globals of the calling module, i.e. the block names as that module sees them
    factor = 2 if bilinear else 1
    widths = (64, 128, 256, 512, 1024 // factor)
    m.inc = g["DoubleConvDS"](n_channels, 64, kernels_per_layer=k)
    for lvl in range(5):
        if lvl > 0:
            setattr(m, f"down{lvl}", g["DownDS"](widths[lvl - 1], widths[lvl], kernels_per_layer=k))
        if lvl < n_cbams:
            setattr(m, f"cbam{lvl + 1}", g["CBAM"](widths[lvl], reduction_ratio=r))
    for i, (cin, cout) in enumerate(zip((1024, 512, 256, 128), (512 // factor, 256 // factor, 128 // factor, 64))):
        setattr(m, f"up{i + 1}", g["UpDS"](cin, cout, bilinear, kernels_per_layer=k))
    m.outc = g["OutConv"](64, n_classes)
""",
    "SmaAt_UNet.py": """from torch import nn
from models.unet_parts import OutConv  # noqa: F401
from models.unet_parts_depthwise_separable import DoubleConvDS, UpDS, DownDS  # noqa: F401
from models.layers import CBAM  # noqa: F401
from models._assemble import assemble


class SmaAt_UNet(nn.Module):
    def __init__(self, n_channels, n_classes, kernels_per_layer=2, bilinear=True, reduction_ratio=16):
        super().__init__()
        assemble(self, globals(), n_channels, n_classes, kernels_per_layer, bilinear, reduction_ratio, 5)
""",
    "unet_precip_regression_lightning.py": """from torch import nn
from models.unet_parts import Down, DoubleConv, Up, OutConv  # noqa: F401
from models.unet_parts_depthwise_separable import DoubleConvDS, UpDS, DownDS  # noqa: F401
from models.layers import CBAM  # noqa: F401
from models._assemble import assemble


def _wrapper(n_cbams):
    def __init__(self, hparams):
        nn.Module.__init__(self)
        h = hparams
        assemble(self, globals(), h.n_channels, h.n_classes, h.kernels_per_layer, h.bilinear, h.reduction_ratio, n_cbams)
    return __init__


UNetDS = type("UNetDS", (nn.Module,), {"__init__": _wrapper(0)})
UNetDSAttention = type("UNetDSAttention", (nn.Module,), {"__init__": _wrapper(5)})
UNetDSAttention4CBAMs = type("UNetDSAttention4CBAMs", (nn.Module,), {"__init__": _wrapper(4)})
""",
}


@pytest.fixture
def standin_reference(tmp_path):
    import sys
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


def test_patch_reference_rebinds_names(standin_reference):
    done = S.patch_reference(standin_reference)
    assert "models.SmaAt_UNet" in done
    import models.SmaAt_UNet as msu
    m = msu.SmaAt_UNet(12, 1)
    assert type(m.inc) is S.DoubleConvDS and type(m.cbam3) is S.CBAM and type(m.up2) is S.UpDS and type(m.outc) is S.OutConv
    assert len(m.state_dict()) == 214


def test_patch_reference_reaches_the_lightning_wrappers(standin_reference):
    """The Lightning wrapper classes (models/unet_precip_regression_lightning.py:86-208) import the block classes by name;
    after patch_reference() their constructors build H100 blocks and keep the reference's state_dict schema."""
    from oracle import ref_stubs
    from oracle.cases import smaat_unet_schema
    done = S.patch_reference(standin_reference, strict=True)
    assert "models.unet_precip_regression_lightning" in done
    import models.unet_precip_regression_lightning as L
    for cls, n_cbams in (("UNetDSAttention", 5), ("UNetDSAttention4CBAMs", 4), ("UNetDS", 0)):
        m = getattr(L, cls)(hparams=ref_stubs.hparams(12, 1, 2))
        assert type(m.inc) is S.DoubleConvDS and type(m.down4) is S.DownDS and type(m.up1) is S.UpDS and type(m.outc) is S.OutConv
        if n_cbams:
            assert type(m.cbam1) is S.CBAM
        sd = m.state_dict()
        schema = smaat_unet_schema(12, 1, 2, n_cbams=n_cbams)
        assert set(sd) == set(schema)
        assert all(tuple(sd[k].shape) == tuple(schema[k]) for k in schema)
