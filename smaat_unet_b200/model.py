"""SmaAt-UNet, its ablations (UNetDS, UNetDSAttention4CBAMs) and the paper's dense baselines (UNet, UNetAttention) assembled
from the H100 drop-in blocks.

Same constructor, attribute names (hence state_dict keys) and forward graph as the
reference's ``models/SmaAt_UNet.py:7-57`` and the Lightning classes of ``models/unet_precip_regression_lightning.py``; provided so
the full models can be built where the reference checkout is not importable (e.g. the GPU box).  With the reference on
``sys.path`` prefer ``smaat_unet_b200.patch_reference()`` and use its own ``SmaAt_UNet``
(and the Lightning wrappers) unchanged.
"""
from __future__ import annotations

import torch
from torch import nn

from .modules import (CBAM, Bf16Declined, DoubleConv, DoubleConvDS, Down, DownDS, OutConv, Up, UpDS, _needs_grad,
                      apply_head)

_ENC = (64, 128, 256, 512)

BF16_ROUTE = ("bf16 input is taken by the serving forward of SmaAt_UNet, UNetDSAttention4CBAMs and UNetDS only: forward_serving / "
              "forward_classes / forward_probs in eval mode under torch.no_grad(), or InferenceSession(model, ..., "
              "dtype=torch.bfloat16)")


def _refuse_bf16(x, why):
    if isinstance(x, torch.Tensor) and x.dtype == torch.bfloat16:
        raise ValueError(f"{BF16_ROUTE}; {why}")


def bf16_shape_refusal(shape):
    """Why the bf16 route of SmaAt_UNet, UNetDSAttention4CBAMs and UNetDS does not take an input of this shape, or None.
    Levels 1-3 are H x W, H / 2 x W / 2 and H / 4 x W / 4; the bf16 DS conv (and its max-pool epilogue) needs rows of a multiple
    of 8 bf16 (16 bytes, for TMA) at each, and tiles a map in patches 16 or 32 pixels wide: an 8-wide level-3 map (W = 32)
    wastes half of either patch and is declined."""
    shape = tuple(shape)
    if len(shape) != 4 or shape[2] % 32 or shape[3] % 32:
        return f"H and W must be multiples of 32 (16-byte bf16 rows at levels 1-3), got shape {shape}"
    if shape[3] < 64:
        return (f"W must be at least 64: at W = {shape[3]} the level-3 maps are {shape[3] // 4} wide, which the fused bf16 DS conv "
                f"does not tile, got shape {shape}")
    return None


class _ServingForward(nn.Module):
    """The serving forwards ``engine.InferenceSession`` captures, for the five networks.  Each network provides
    ``_serving(x, head)``: its eval forward, ending in up4 with the OutConv and the head (modules.HEADS); its class docstring
    says what that fuses.  In train mode or under autograd they run the plain forward, then ``modules.apply_head``."""

    def forward_serving(self, x):
        """``forward``'s logits, through the serving forward's fusions."""
        return self._serve(x, "logits")

    def forward_classes(self, x):
        """The (B, H, W) int64 class map of the logits, argmax over their channels (the reference's
        ``torch.argmax(softmax(y_pred), dim=1)``, train_SmaAtUNet.py:76).  Inference only."""
        return self._serve(x, "classes")

    def forward_probs(self, x):
        """The (B, n_classes, H, W) fp32 class probabilities, ``softmax_channels`` of ``forward_serving``'s logits (the
        reference's ``softmax(y_pred)``, train_SmaAtUNet.py:76).  Inference only, with no gradient."""
        return self._serve(x, "probs")

    def _serve(self, x, head):
        if isinstance(x, torch.Tensor) and x.dtype == torch.bfloat16:
            return self._serve_bf16(x, head)
        if self.training or _needs_grad(self, x):
            return apply_head(self, x, head)
        return self._serving(x, head)

    def _serve_bf16(self, x, head):
        _refuse_bf16(x, f"{type(self).__name__} has no bf16 route")


class _DSUNet(_ServingForward):
    """The depthwise-separable networks of the paper: SmaAt_UNet, UNetDSAttention4CBAMs and UNetDS, one body parameterised by
    ``CBAM_LEVELS``, the levels (1-5) whose encoder map carries a CBAM.  Attribute names and parameter registration order are
    the reference's (models/SmaAt_UNet.py:22-38, unet_precip_regression_lightning.py:87-104 and :173-190): inc, [cbam1], down1,
    [cbam2], ..., down4, [cbam5], up1-up4, outc.

    Serving forward (``forward_serving`` / ``forward_classes`` / ``forward_probs``):
    * up4's last DS conv applies the OutConv in its epilogue (SmaAt_UNet.py:55-56), so the 64-channel activation never reaches
      HBM: the 1-class OutConv for the logits, the n_classes-class OutConv and the argmax for class maps (n_classes <= 32;
      more classes take the unfused convs, OutConv and the argmax kernel).  Each class's logit there is the one-class fused
      OutConv's arithmetic, which sums in another order than the unfused OutConv of the logits route: pixels whose top two
      logits lie within rounding of each other may pick the other class.  The probabilities are the channel softmax of the
      logits route's output;
    * a CBAM at level 1-3 never writes its output: it computes only its two gates, and the first DS conv of up2 / up3 / up4
      applies them as it loads the skip, with the products the CBAM's own kernel would have used (bit for bit the same
      logits).  A CBAM at level 4-5 runs the plain call, which hands its max-pool to the DownDS that follows;
    * a level 1-4 map without a CBAM (UNetDS) gets its 2x2 max-pool from the epilogue of the DS conv that produced it, bit for
      bit the max-pool of the stored map, so the next DownDS does not read the map again (``smaat_maxpool2_fwd`` where that
      kernel declines the shape)."""

    CBAM_LEVELS = ()

    def __init__(self, n_channels, n_classes, kernels_per_layer=2, bilinear=True, reduction_ratio=16):
        super().__init__()
        self.n_channels, self.n_classes, self.bilinear = n_channels, n_classes, bilinear
        k, r = kernels_per_layer, reduction_ratio
        factor = 2 if bilinear else 1
        widths = list(_ENC) + [1024 // factor]            # channels of x1..x5
        self.inc = DoubleConvDS(n_channels, widths[0], kernels_per_layer=k)
        for lvl in range(5):                                # [down_l,] [cbam_{l+1}] -- registration order = reference's
            if lvl > 0:
                setattr(self, f"down{lvl}", DownDS(widths[lvl - 1], widths[lvl], kernels_per_layer=k))
            if lvl + 1 in self.CBAM_LEVELS:
                setattr(self, f"cbam{lvl + 1}", CBAM(widths[lvl], reduction_ratio=r))
        dec_in = (1024, 512, 256, 128)
        dec_out = (512 // factor, 256 // factor, 128 // factor, 64)
        for i in range(4):                                  # up1..up4
            setattr(self, f"up{i + 1}", UpDS(dec_in[i], dec_out[i], bilinear, kernels_per_layer=k))
        self.outc = OutConv(64, n_classes)

    def _cbam(self, lvl):
        return getattr(self, f"cbam{lvl + 1}", None)

    def forward(self, x):
        """The reference's graph, block for block and in its call order (models/SmaAt_UNet.py:41-57,
        unet_precip_regression_lightning.py:107-118 and :193-208): plain calls only -- exactly what a ``patch_reference()`` user
        of the unchanged reference class executes.  Where a CBAM precedes a DownDS the max-pool fusion still happens:
        ``cbamN(f)`` leaves MaxPool2d(2)(f) behind for the ``downN(f)`` that follows (modules.CBAM.forward)."""
        _refuse_bf16(x, "model(x) runs the fp32 plain-call graph")
        f = self.inc(x)
        att = []
        for lvl in range(5):
            if lvl > 0:
                f = getattr(self, f"down{lvl}")(f)
            cbam = self._cbam(lvl)
            att.append(cbam(f) if cbam is not None else f)
        y = att[4]                                                  # x5 (x5Att) is the decoder input
        for i in range(4):
            y = getattr(self, f"up{i + 1}")(y, att[3 - i])          # attended maps, where there is a CBAM, are the skips
        return self.outc(y)

    def _serve_bf16(self, x, head):
        """The bf16 storage route (opt-in by the input's dtype): the input and the level 1-3 maps are bf16 in HBM, levels 4-5
        fp32 with the fp32 route's kernels; the level 1-3 GEMMs take bf16 operands whatever ``set_pointwise_mode`` says.  Every
        request it does not take raises ``ValueError`` before any launch; a level 1-3 conv its kernel declines raises naming
        the layer."""
        if self.training or _needs_grad(self, x):
            _refuse_bf16(x, "train mode and autograd have no bf16 route")
        if self.inc.double_conv[0].kernels_per_layer not in (1, 2):
            _refuse_bf16(x, f"kernels_per_layer={self.inc.double_conv[0].kernels_per_layer} has no bf16 kernel (1 or 2 only)")
        if not self.bilinear:
            _refuse_bf16(x, "bilinear=False (the transposed-conv upsample) has no bf16 route")
        why = bf16_shape_refusal(x.shape)
        if why:
            _refuse_bf16(x, why)
        try:
            return self._serving(x, head)
        except Bf16Declined as e:
            name = next((n for n, m in self.named_modules() if m is e.module), type(e.module).__name__)
            raise ValueError(f"{type(self).__name__} bf16 serving forward: {name}: {e}") from None

    def _serving(self, x, head):
        skips, pooled = [], None
        for lvl in range(5):
            cbam = self._cbam(lvl)
            # no CBAM to hand the max-pool over: the conv that makes the map writes it for the next DownDS.  The bf16 route's
            # max-pool is bf16 into levels 2-3, fp32 into level 4
            kw = {} if cbam is not None or lvl == 4 else {
                "with_maxpool": True, "pooled_dtype": torch.float32 if lvl >= 2 else x.dtype}
            f = self.inc.run(x, **kw) if lvl == 0 else getattr(self, f"down{lvl}")(f, pooled=pooled, **kw)
            if kw:
                f, pooled = f
            if cbam is None:
                skips.append((f, None))
                continue
            bn = cbam.spatial_att.bn
            if lvl < 3 and not bn.training and bn.track_running_stats:
                sc, sa, pooled = cbam.serving_gates(f, pooled_dtype=torch.float32 if lvl == 2 else f.dtype)
                skips.append((f, (sc, sa)))
            else:
                skips.append((cbam(f), None))       # a plain call leaves its max-pool for the DownDS that follows
                pooled = None
        y = skips[4][0]
        for i in range(3):
            skip, gate = skips[3 - i]
            y = getattr(self, f"up{i + 1}")(y, skip, gate=gate)
        skip, gate = skips[0]
        return self.up4(y, skip, outconv=self.outc, gate=gate, head=head)


class SmaAt_UNet(_DSUNet):
    """models/SmaAt_UNet.py:7-57: a CBAM on every level.  Serving forward: ``_DSUNet``'s, with the three large CBAMs (levels
    1-3) as gates applied on load and levels 4-5 as plain calls."""

    CBAM_LEVELS = (1, 2, 3, 4, 5)


class UNetDSAttention4CBAMs(_DSUNet):
    """``models/unet_precip_regression_lightning.py:173-208`` (the Lightning class without its training plumbing): SmaAt-UNet
    without the bottleneck's CBAM, so x5 goes to up1 un-attended.  Serving forward: ``_DSUNet``'s -- levels 1-3 gated on load,
    level 4 a plain ``cbam4`` call that hands its max-pool to ``down4``."""

    CBAM_LEVELS = (1, 2, 3, 4)


class UNetDS(_DSUNet):
    """``models/unet_precip_regression_lightning.py:86-118``: SmaAt-UNet without attention, the DS convs' ablation.  Serving
    forward: ``_DSUNet``'s -- the un-attended maps are the skips, and the max-pools feeding down1-down4 come from the epilogues
    of the convs that produced the maps."""

    CBAM_LEVELS = ()

    def __init__(self, n_channels, n_classes, kernels_per_layer=2, bilinear=True):
        super().__init__(n_channels, n_classes, kernels_per_layer=kernels_per_layer, bilinear=bilinear)


class UNet(_ServingForward):
    """The dense baseline of ``models/unet_precip_regression_lightning.py:7-38`` (the Lightning class without its training
    plumbing): same attribute names (hence the reference's 128 state_dict keys with ``bilinear=True``) and forward order.

    Its serving forward runs the plain calls: bit for bit ``forward``'s logits and ``argmax_channels`` / ``softmax_channels``
    of them (an OutConv epilogue in up4's last 3x3 conv measured slower on an H100: DESIGN section 6)."""

    def __init__(self, n_channels, n_classes, bilinear=True):
        super().__init__()
        self.n_channels, self.n_classes, self.bilinear = n_channels, n_classes, bilinear
        self.inc = DoubleConv(n_channels, 64)
        self.down1 = Down(64, 128)
        self.down2 = Down(128, 256)
        self.down3 = Down(256, 512)
        factor = 2 if bilinear else 1
        self.down4 = Down(512, 1024 // factor)
        self.up1 = Up(1024, 512 // factor, bilinear)
        self.up2 = Up(512, 256 // factor, bilinear)
        self.up3 = Up(256, 128 // factor, bilinear)
        self.up4 = Up(128, 64, bilinear)
        self.outc = OutConv(64, n_classes)

    def _to_up4(self, x):
        """The encoder and up1-up3: up4's two inputs."""
        x1 = self.inc(x)
        x2 = self.down1(x1)
        x3 = self.down2(x2)
        x4 = self.down3(x3)
        x5 = self.down4(x4)
        x = self.up1(x5, x4)
        x = self.up2(x, x3)
        x = self.up3(x, x2)
        return x, x1

    def forward(self, x):
        _refuse_bf16(x, "UNet has no bf16 route")
        return self.outc(self.up4(*self._to_up4(x)))

    def _serving(self, x, head):
        return self.up4(*self._to_up4(x), outconv=self.outc, head=head)


class UNetAttention(_ServingForward):
    """``models/unet_precip_regression_lightning.py:41-83``: UNet with a CBAM on every skip (178 state_dict keys with
    ``bilinear=True``).  ``downN`` runs on the un-attended map right after ``cbamN`` did, so the CBAM hands it its 2x2 max-pool.

    Its serving forward runs the plain calls: bit for bit ``forward``'s logits and ``argmax_channels`` / ``softmax_channels``
    of them (an OutConv epilogue in up4's last 3x3 conv measured slower on an H100: DESIGN section 6)."""

    def __init__(self, n_channels, n_classes, bilinear=True, reduction_ratio=16):
        super().__init__()
        self.n_channels, self.n_classes, self.bilinear = n_channels, n_classes, bilinear
        r = reduction_ratio
        self.inc = DoubleConv(n_channels, 64)
        self.cbam1 = CBAM(64, reduction_ratio=r)
        self.down1 = Down(64, 128)
        self.cbam2 = CBAM(128, reduction_ratio=r)
        self.down2 = Down(128, 256)
        self.cbam3 = CBAM(256, reduction_ratio=r)
        self.down3 = Down(256, 512)
        self.cbam4 = CBAM(512, reduction_ratio=r)
        factor = 2 if bilinear else 1
        self.down4 = Down(512, 1024 // factor)
        self.cbam5 = CBAM(1024 // factor, reduction_ratio=r)
        self.up1 = Up(1024, 512 // factor, bilinear)
        self.up2 = Up(512, 256 // factor, bilinear)
        self.up3 = Up(256, 128 // factor, bilinear)
        self.up4 = Up(128, 64, bilinear)
        self.outc = OutConv(64, n_classes)

    def _to_up4(self, x):
        """The encoder and up1-up3, in the reference's call order: up4's two inputs."""
        x1 = self.inc(x)
        x1Att = self.cbam1(x1)
        x2 = self.down1(x1)
        x2Att = self.cbam2(x2)
        x3 = self.down2(x2)
        x3Att = self.cbam3(x3)
        x4 = self.down3(x3)
        x4Att = self.cbam4(x4)
        x5 = self.down4(x4)
        x5Att = self.cbam5(x5)
        x = self.up1(x5Att, x4Att)
        x = self.up2(x, x3Att)
        x = self.up3(x, x2Att)
        return x, x1Att

    def forward(self, x):
        _refuse_bf16(x, "UNetAttention has no bf16 route")
        return self.outc(self.up4(*self._to_up4(x)))

    def _serving(self, x, head):
        return self.up4(*self._to_up4(x), outconv=self.outc, head=head)
