"""Rebind the reference's block classes to the H100 drop-ins, in place.

The reference has no plugin registry: ``models/SmaAt_UNet.py:2-4`` and
``models/unet_precip_regression_lightning.py:1-3`` import the block classes by name.
``patch_reference()`` swaps those names in the already-importable reference modules so that
``SmaAt_UNet`` and the Lightning variants (UNet, UNetAttention, UNetDS, UNetDSAttention,
UNetDSAttention4CBAMs) are constructed from H100 blocks with no change to reference code.
"""
from __future__ import annotations

import importlib
import sys

from . import modules as M

_TARGETS = {
    "models.layers": ("DepthwiseSeparableConv", "ChannelAttention", "SpatialAttention", "CBAM"),
    "models.unet_parts_depthwise_separable": ("DepthwiseSeparableConv", "DoubleConvDS", "DownDS", "UpDS"),
    "models.unet_parts": ("DoubleConv", "Down", "Up", "OutConv"),
    "models.SmaAt_UNet": ("OutConv", "DoubleConvDS", "UpDS", "DownDS", "CBAM"),
    # needs `lightning`; patched only if it imports
    "models.unet_precip_regression_lightning": ("Down", "DoubleConv", "Up", "OutConv", "DoubleConvDS", "UpDS", "DownDS", "CBAM"),
}


def patch_reference(reference_root: str | None = None, strict: bool = False):
    """Returns {module name: [rebound names]}.  ``reference_root`` is prepended to sys.path if given."""
    if reference_root and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    done = {}
    for modname, names in _TARGETS.items():
        try:
            mod = importlib.import_module(modname)
        except Exception:
            if strict:
                raise
            continue
        for n in names:
            if hasattr(mod, n):
                setattr(mod, n, getattr(M, n))
                done.setdefault(modname, []).append(n)
    return done
