"""SmaAt-UNet and the paper's dense baselines (UNet, UNetAttention) assembled from the H100 drop-in blocks.

Same constructor, attribute names (hence state_dict keys) and forward graph as the
reference's ``models/SmaAt_UNet.py:7-57``; provided so the full model can be built where the
reference checkout is not importable (e.g. the GPU box).  With the reference on
``sys.path`` prefer ``smaat_unet_b200.patch_reference()`` and use its own ``SmaAt_UNet``
(and the Lightning wrappers) unchanged.
"""
from __future__ import annotations

import torch
from torch import nn

from . import ops
from .modules import CBAM, DoubleConv, DoubleConvDS, Down, DownDS, OutConv, Up, UpDS, _needs_grad

_ENC = (64, 128, 256, 512)


def _classes_of(model, x):
    """The class map of ``model(x)``'s logits: the plain forward, then the channel argmax kernel (ops.argmax_channels)."""
    with torch.no_grad():
        return ops.argmax_channels(model(x))


def _probs_of(model, x):
    """The class probabilities of ``model(x)``'s logits: the plain forward, then the channel softmax kernel
    (ops.softmax_channels), with no gradient."""
    with torch.no_grad():
        return ops.softmax_channels(model(x))


class SmaAt_UNet(nn.Module):
    def __init__(self, n_channels, n_classes, kernels_per_layer=2, bilinear=True, reduction_ratio=16):
        super().__init__()
        self.n_channels, self.n_classes, self.bilinear = n_channels, n_classes, bilinear
        k, r = kernels_per_layer, reduction_ratio
        factor = 2 if bilinear else 1
        widths = list(_ENC) + [1024 // factor]            # channels of x1..x5
        self.inc = DoubleConvDS(n_channels, widths[0], kernels_per_layer=k)
        for lvl in range(5):                                # [down_l,] cbam_{l+1} -- registration order = reference's
            if lvl > 0:
                setattr(self, f"down{lvl}", DownDS(widths[lvl - 1], widths[lvl], kernels_per_layer=k))
            setattr(self, f"cbam{lvl + 1}", CBAM(widths[lvl], reduction_ratio=r))
        dec_in = (1024, 512, 256, 128)
        dec_out = (512 // factor, 256 // factor, 128 // factor, 64)
        for i in range(4):                                  # up1..up4
            setattr(self, f"up{i + 1}", UpDS(dec_in[i], dec_out[i], bilinear, kernels_per_layer=k))
        self.outc = OutConv(64, n_classes)

    def forward(self, x):
        """The reference's graph, block for block and in its call order (models/SmaAt_UNet.py:41-57): plain calls only --
        exactly what a ``patch_reference()`` user of the unchanged reference class executes.  The max-pool fusion still
        happens: ``cbamN(f)`` leaves MaxPool2d(2)(f) behind for the ``downN(f)`` that follows (modules.CBAM.forward)."""
        f = self.inc(x)
        att = [self.cbam1(f)]
        for lvl in range(1, 5):
            f = getattr(self, f"down{lvl}")(f)
            att.append(getattr(self, f"cbam{lvl + 1}")(f))
        y = att[4]                                                  # x5Att is the decoder input
        for i in range(4):
            y = getattr(self, f"up{i + 1}")(y, att[3 - i])          # attended maps are the skips
        return self.outc(y)

    def forward_serving(self, x):
        """Same graph with the fusions the plain-call API cannot express (``engine.InferenceSession``; inference only, the
        plain calls under autograd / train mode):
        * up4's last DS conv applies the 1-class OutConv in its epilogue (SmaAt_UNet.py:55-56), so the 64-channel activation
          never reaches HBM;
        * the three large CBAMs (levels 1-3) never write their output: they compute only their two gates, and the first DS
          conv of up2 / up3 / up4 applies them as it loads the skip, with the products the CBAM's own kernel would have used
          (bit for bit the same logits).  Levels 4-5 run the plain calls."""
        return self._serving(x, classes=False)

    def forward_classes(self, x):
        """``forward_serving``'s graph ending in the (B, H, W) int64 class map the reference predicts from the logits
        (``torch.argmax(softmax(y_pred), dim=1)``, train_SmaAtUNet.py:76): up4's last DS conv applies the n_classes-class
        OutConv and the argmax in its epilogue (n_classes <= 32), so neither its 64-channel activation nor the logits reach
        HBM.  Each class's logit there is the one-class fused OutConv's arithmetic, which sums in another order than the
        unfused OutConv of the logits route: pixels whose top two logits lie within rounding of each other may pick the other
        class.  Inference only; in train mode or under autograd the plain forward followed by the argmax kernel."""
        if self.training or _needs_grad(self, x):
            return _classes_of(self, x)
        return self._serving(x, classes=True)

    def forward_probs(self, x):
        """``forward_serving``'s graph ending in the (B, n_classes, H, W) fp32 class probabilities, softmax over the logits'
        channels (the reference's ``softmax(y_pred)``, train_SmaAtUNet.py:76): up4's last DS conv applies the n_classes-class
        OutConv and the softmax in its epilogue (n_classes <= 32), so only the probabilities reach HBM; more classes take the
        unfused convs, OutConv and the softmax kernel.  Inference only, with no gradient: in train mode or under autograd
        the plain forward followed by the softmax kernel, under no_grad."""
        if self.training or _needs_grad(self, x):
            return _probs_of(self, x)
        return self._serving(x, probs=True)

    def _serving(self, x, classes=False, probs=False):
        if self.training or _needs_grad(self, x):
            return self.forward(x)
        skips, f = [], self.inc(x)
        for lvl in range(5):
            if lvl > 0:
                f = getattr(self, f"down{lvl}")(f, pooled=pooled)
            cbam = getattr(self, f"cbam{lvl + 1}")
            bn = cbam.spatial_att.bn
            if lvl < 3 and not bn.training and bn.track_running_stats:
                sc, sa, pooled = cbam.serving_gates(f)
                skips.append((f, (sc, sa)))
            else:
                skips.append((cbam(f), None))       # a plain call leaves its max-pool for the DownDS that follows
                pooled = None
        y = skips[4][0]
        for i in range(3):
            skip, gate = skips[3 - i]
            y = getattr(self, f"up{i + 1}")(y, skip, gate=gate)
        skip, gate = skips[0]
        return self.up4(y, skip, outconv=self.outc, gate=gate, classes=classes, probs=probs)


class UNet(nn.Module):
    """The dense baseline of ``models/unet_precip_regression_lightning.py:7-38`` (the Lightning class without its training
    plumbing): same attribute names (hence the reference's 128 state_dict keys with ``bilinear=True``) and forward order."""

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

    def forward(self, x):
        x1 = self.inc(x)
        x2 = self.down1(x1)
        x3 = self.down2(x2)
        x4 = self.down3(x3)
        x5 = self.down4(x4)
        x = self.up1(x5, x4)
        x = self.up2(x, x3)
        x = self.up3(x, x2)
        x = self.up4(x, x1)
        return self.outc(x)

    def forward_serving(self, x):
        """``forward`` for ``engine.InferenceSession``, bit for bit ``forward``'s logits.  With ``ops.set_fused_dense_head(True)``
        up4's last 3x3 conv applies the OutConv in its epilogue, so the 64-channel activation never reaches HBM; by default (the
        faster route on an H100) and in train mode, under autograd, or where the epilogue does not take the shape ('fp32'
        mode, W % 4 != 0, more than 32 classes), the plain calls."""
        return self._serving(x)

    def forward_classes(self, x):
        """The (B, H, W) int64 class map of ``forward``'s logits (train_SmaAtUNet.py:76), bit for bit ``argmax_channels(forward(x))``:
        with ``ops.set_fused_dense_head(True)`` up4's last conv applies the OutConv and the argmax in its epilogue, so neither its
        activation nor the logits reach HBM.  Otherwise (see ``forward_serving``): the forward, then the argmax kernel."""
        if self.training or _needs_grad(self, x):
            return _classes_of(self, x)
        return self._serving(x, classes=True)

    def forward_probs(self, x):
        """The class probabilities of ``forward``'s logits (train_SmaAtUNet.py:76), bit for bit ``softmax_channels(forward(x))``:
        with ``ops.set_fused_dense_head(True)`` up4's last conv applies the OutConv and the softmax in its epilogue.  Otherwise:
        the forward, then the softmax kernel.  Inference only, with no gradient."""
        if self.training or _needs_grad(self, x):
            return _probs_of(self, x)
        return self._serving(x, probs=True)

    def _serving(self, x, classes=False, probs=False):
        if self.training or _needs_grad(self, x):
            return self.forward(x)
        x1 = self.inc(x)
        x2 = self.down1(x1)
        x3 = self.down2(x2)
        x4 = self.down3(x3)
        x5 = self.down4(x4)
        x = self.up1(x5, x4)
        x = self.up2(x, x3)
        x = self.up3(x, x2)
        return self.up4(x, x1, outconv=self.outc, classes=classes, probs=probs)


class UNetAttention(nn.Module):
    """``models/unet_precip_regression_lightning.py:41-83``: UNet with a CBAM on every skip (178 state_dict keys with
    ``bilinear=True``).  ``downN`` runs on the un-attended map right after ``cbamN`` did, so the CBAM hands it its 2x2 max-pool."""

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

    def forward(self, x):
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
        x = self.up4(x, x1Att)
        return self.outc(x)

    def forward_serving(self, x):
        """``forward`` for ``engine.InferenceSession``, bit for bit ``forward``'s logits.  With ``ops.set_fused_dense_head(True)``
        up4's last 3x3 conv applies the OutConv in its epilogue, so the 64-channel activation never reaches HBM; by default (the
        faster route on an H100) and in train mode, under autograd, or where the epilogue does not take the shape ('fp32'
        mode, W % 4 != 0, more than 32 classes), the plain calls."""
        return self._serving(x)

    def forward_classes(self, x):
        """The (B, H, W) int64 class map of ``forward``'s logits (train_SmaAtUNet.py:76), bit for bit ``argmax_channels(forward(x))``:
        with ``ops.set_fused_dense_head(True)`` up4's last conv applies the OutConv and the argmax in its epilogue, so neither its
        activation nor the logits reach HBM.  Otherwise (see ``forward_serving``): the forward, then the argmax kernel."""
        if self.training or _needs_grad(self, x):
            return _classes_of(self, x)
        return self._serving(x, classes=True)

    def forward_probs(self, x):
        """The class probabilities of ``forward``'s logits (train_SmaAtUNet.py:76), bit for bit ``softmax_channels(forward(x))``:
        with ``ops.set_fused_dense_head(True)`` up4's last conv applies the OutConv and the softmax in its epilogue.  Otherwise:
        the forward, then the softmax kernel.  Inference only, with no gradient."""
        if self.training or _needs_grad(self, x):
            return _probs_of(self, x)
        return self._serving(x, probs=True)

    def _serving(self, x, classes=False, probs=False):
        if self.training or _needs_grad(self, x):
            return self.forward(x)
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
        return self.up4(x, x1Att, outconv=self.outc, classes=classes, probs=probs)
