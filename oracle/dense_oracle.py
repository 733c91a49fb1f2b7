"""CPU oracles of the dense UNet blocks -- TEST INFRASTRUCTURE ONLY.

Numpy restatement (``double_conv`` ... ``unet_forward``) and torch-functional port (``port_*``) of DoubleConv / Down / Up
(``models/unet_parts.py:8-64``) and the Lightning UNet / UNetAttention forward bodies
(``models/unet_precip_regression_lightning.py:27-38, 67-83``), built on the leaf functions of ``oracle/smaat_oracle.py`` and
``oracle/torch_port.py``.  Pinned against the reference by ``oracle/make_golden_dense.py`` / ``tests/golden/dense_*.npz``.
Never imported by the product package.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import smaat_oracle as O
from . import torch_port as T


# ---------------------------------------------------------------------------- numpy
def conv3x3(x, weight, bias):
    """nn.Conv2d(Cin, Cout, 3, padding=1) (unet_parts.py:16,19): cross-correlation, zero padding 1."""
    B, Cin, H, W = x.shape
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    w = weight.astype(x.dtype)
    y = np.zeros((B, w.shape[0], H, W), dtype=x.dtype)
    for dy in range(3):
        for dx in range(3):
            y += np.einsum("oc,bchw->bohw", w[:, :, dy, dx], xp[:, :, dy:dy + H, dx:dx + W], optimize=True)
    if bias is not None:
        y += bias.astype(x.dtype)[None, :, None, None]
    return y


def double_conv(x, sd, prefix, training=False):
    """DoubleConv (unet_parts.py:8-25): [Conv3x3, BN, ReLU] x 2 as double_conv.{0,1,2,3,4,5}."""
    upd = {}
    y = conv3x3(x, sd[prefix + ".double_conv.0.weight"], sd[prefix + ".double_conv.0.bias"])
    y, u = O._bn(y, sd, prefix + ".double_conv.1", training); upd.update(u)
    y = conv3x3(O.relu(y), sd[prefix + ".double_conv.3.weight"], sd[prefix + ".double_conv.3.bias"])
    y, u = O._bn(y, sd, prefix + ".double_conv.4", training); upd.update(u)
    return O.relu(y), upd


def down(x, sd, prefix, training=False):
    """Down (unet_parts.py:28-36): MaxPool2d(2) then DoubleConv under maxpool_conv.1."""
    return double_conv(O.maxpool2(x), sd, prefix + ".maxpool_conv.1", training)


def up(x_low, x_skip, sd, prefix, training=False):
    """Up (unet_parts.py:39-64): upsample x2 (bilinear, or ConvTranspose2d when the state_dict holds `up.weight`), pad to
    the skip, cat([skip, up]), DoubleConv."""
    if prefix + ".up.weight" in sd:
        u = O.conv_transpose2x2(x_low, sd[prefix + ".up.weight"], sd[prefix + ".up.bias"])
    else:
        u = O.upsample_bilinear2x(x_low)
    u = O.pad_to(u, x_skip.shape[2], x_skip.shape[3])
    return double_conv(np.concatenate([x_skip, u], axis=1), sd, prefix + ".conv", training)


def unet_forward(x, sd, training=False, attention=False):
    """UNet.forward (unet_precip_regression_lightning.py:27-38); ``attention``: UNetAttention.forward (:67-83), whose
    decoder reads the CBAM-attended skips while the encoder continues from the un-attended maps."""
    upd = {}
    enc = []
    y, u = double_conv(x, sd, "inc", training); upd.update(u)
    enc.append(y)
    for i in range(1, 5):
        y, u = down(enc[-1], sd, f"down{i}", training); upd.update(u)
        enc.append(y)
    skips = enc
    if attention:
        skips = []
        for i, e in enumerate(enc):
            a, u = O.cbam(e, sd, f"cbam{i + 1}", training); upd.update(u)
            skips.append(a)
    y = skips[4]
    for i in range(1, 5):
        y, u = up(y, skips[4 - i], sd, f"up{i}", training); upd.update(u)
    return O.out_conv(y, sd, "outc"), upd


# ---------------------------------------------------------------------------- torch port
def port_double_conv(x, sd, p, training=False):
    # unet_parts.py:15-22
    y = F.relu(T._bn(F.conv2d(x, sd[p + ".double_conv.0.weight"], sd[p + ".double_conv.0.bias"], padding=1), sd, p + ".double_conv.1", training))
    return F.relu(T._bn(F.conv2d(y, sd[p + ".double_conv.3.weight"], sd[p + ".double_conv.3.bias"], padding=1), sd, p + ".double_conv.4", training))


def port_down(x, sd, p, training=False):
    # unet_parts.py:33-36
    return port_double_conv(F.max_pool2d(x, 2), sd, p + ".maxpool_conv.1", training)


def port_up(x_low, x_skip, sd, p, training=False):
    # unet_parts.py:53-64
    if p + ".up.weight" in sd:
        u = F.conv_transpose2d(x_low, sd[p + ".up.weight"], sd[p + ".up.bias"], stride=2)
    else:
        u = F.interpolate(x_low, scale_factor=2, mode="bilinear", align_corners=True)
    dY, dX = x_skip.shape[2] - u.shape[2], x_skip.shape[3] - u.shape[3]
    u = F.pad(u, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])
    return port_double_conv(torch.cat([x_skip, u], dim=1), sd, p + ".conv", training)


def port_unet_forward(x, sd, training=False, attention=False):
    # unet_precip_regression_lightning.py:27-38 / :67-83
    enc = [port_double_conv(x, sd, "inc", training)]
    for i in range(1, 5):
        enc.append(port_down(enc[-1], sd, f"down{i}", training))
    skips = [T.cbam(e, sd, f"cbam{i + 1}", training) for i, e in enumerate(enc)] if attention else enc
    y = skips[4]
    for i in range(1, 5):
        y = port_up(y, skips[4 - i], sd, f"up{i}", training)
    return F.conv2d(y, sd["outc.conv.weight"], sd["outc.conv.bias"])
