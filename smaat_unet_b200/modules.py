"""Drop-in nn.Module replacements for the SmaAt-UNet hot-path blocks.

Host-side mirror of the reference's class interface (SURVEY.md 8b): same class names,
constructor signatures, forward signatures and ``state_dict`` keys as

* ``models/layers.py``: DepthwiseSeparableConv (:34-50), ChannelAttention (:90-111),
  SpatialAttention (:114-129), CBAM (:132-141)
* ``models/unet_parts_depthwise_separable.py``: DoubleConvDS (:10-39), DownDS (:42-53), UpDS (:56-86)
* ``models/unet_parts.py``: DoubleConv (:8-25), Down (:28-36), Up (:39-64), OutConv (:67-73)

so checkpoints trained with the reference load unchanged (``calc_metrics_test_set.py:114``).
The parameter containers are ordinary torch modules (``nn.Conv2d`` / ``nn.BatchNorm2d`` /
``nn.Linear`` -> identical default initialisation and key names) but their ``forward`` is
never called: all arithmetic runs in libsmaat_b200.so (sm_90a kernels) through ``ops``.
There is no PyTorch / CPU fallback; unsupported requests raise.
"""
from __future__ import annotations

import weakref

import torch
from torch import nn

from . import ops


def _versions(*tensors):
    """Cache key for tensors derived from parameters / buffers.  ``_version`` only sees writes that go through torch
    dispatch; our kernels (BatchNorm running statistics in smaat_bn_finalize, anything replayed from a CUDA graph)
    write through raw pointers, so the key also carries ``ops.weights_generation()`` -- bumped by every such write
    (ops.bn_finalize, TrainSession.step) and by every train()/eval() switch of a caching module."""
    return (ops.weights_generation(),) + tuple((t.data_ptr(), t._version) for t in tensors if t is not None)


def _held(*tensors):
    """Aliases of the tensors a cache entry was derived from, stored with the entry.  A ``_versions`` key names addresses:
    while the entry holds their blocks, no tensor that replaces a source (``load_state_dict(..., assign=True)``,
    ``p.data = ...``) can be allocated on a cached address at the cached version and hit the stale entry."""
    return tuple(t.detach() for t in tensors if t is not None)


class _CachingModule(nn.Module):
    """Modules that cache tensors derived from their parameters drop those caches on every mode switch."""

    def _drop_caches(self):
        pass

    def train(self, mode=True):
        self._drop_caches()
        ops.bump_weights_generation()
        return super().train(mode)


def _needs_grad(mod, *inputs):
    """True when the call must be recorded on the autograd tape (grad mode on and a parameter or input requires grad)."""
    if not torch.is_grad_enabled():
        return False
    if any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs):
        return True
    return any(p.requires_grad for p in mod.parameters())


class Bf16Declined(RuntimeError):
    """A bf16 request the bf16 route's fused kernel does not take, raised by the module (``module``) that declined it: the bf16
    route has no unfused fallback.  SmaAt_UNet names the layer (model.py)."""

    def __init__(self, module, msg):
        super().__init__(msg)
        self.module = module


def _no_autograd(mod, *inputs):
    if _needs_grad(mod, *inputs):
        raise NotImplementedError(
            f"{type(mod).__name__}: autograd through this standalone module is not implemented in smaat_unet_b200 "
            "(DoubleConvDS / DownDS / UpDS / CBAM / OutConv are differentiable). Use torch.no_grad(); no PyTorch fallback is provided.")


class DepthwiseSeparableConv(_CachingModule):
    """models/layers.py:34-50 -- depthwise(k x k, groups=Cin, kpl outputs per channel) then pointwise 1x1."""

    def __init__(self, in_channels, output_channels, kernel_size, padding=0, kernels_per_layer=1):
        super().__init__()
        self.depthwise = nn.Conv2d(in_channels, in_channels * kernels_per_layer, kernel_size=kernel_size,
                                   padding=padding, groups=in_channels)
        self.pointwise = nn.Conv2d(in_channels * kernels_per_layer, output_channels, kernel_size=1)
        self.kernels_per_layer = kernels_per_layer
        self._wsplit = None
        self._wsplit_key = None
        self._wsplit_src = None

    def _drop_caches(self):
        self._wsplit = self._wsplit_key = self._wsplit_src = None

    def _check(self):
        if self.depthwise.kernel_size != (3, 3) or self.depthwise.padding != (1, 1):
            raise NotImplementedError("smaat_unet_b200 implements the depthwise conv the reference uses: 3x3, padding=1 "
                                      "(parts_ds.py:18-33)")

    def pw_operands(self, mode=None):
        """The pointwise weight's operands in the current mode (or ``mode``: the bf16 route always takes 'bf16') --
        ``ops.derived_operands``: the tf32 (hi, lo) split in 'tf32x3', (bf16 pack, None) in 'bf16', None in the modes that take
        the weight as it is -- cached on the parameter's version counter and the mode."""
        mode = ops.PW_MODES[mode or ops.get_pointwise_mode()]
        w = self.pointwise.weight
        key = (_versions(w), mode)
        # while a training step is being captured into a CUDA graph the operands must be part of the graph: replays see new
        # weights
        in_train_capture = self.training and torch.cuda.is_current_stream_capturing()
        if in_train_capture or self._wsplit_key != key:
            with torch.no_grad():
                self._wsplit = ops.derived_operands(w.detach().view(w.shape[0], -1), mode)
            self._wsplit_key = None if in_train_capture else key
            self._wsplit_src = _held(w)
        return self._wsplit

    def fused_takes(self, x, x1=None, stats=False) -> bool:
        """Whether the one-kernel depthwise->pointwise path takes this input (shape, alignment, arithmetic mode)."""
        return ops.dsconv_takes(x, x1, self.pointwise.weight.detach(), self.kernels_per_layer, stats=stats)

    def _operands(self, shift):
        """What ``run``, ``run_head`` and ``run_cbam`` hand the kernels besides the input and the epilogue scale: the depthwise
        bias, the epilogue shift (the pointwise bias where the caller gives none), the arithmetic mode and the pointwise
        weight's cached operands in that mode (``pw_operands``)."""
        self._check()
        dw_b = self.depthwise.bias.detach() if self.depthwise.bias is not None else None
        if shift is None:
            shift = self.pointwise.bias.detach() if self.pointwise.bias is not None else None
        mode = ops.get_pointwise_mode()
        return dw_b, shift, mode, self.pw_operands()

    def _bf16(self, x, x1, scale, shift, relu, gate=None):
        """The bf16 route (bf16 x [, x1] -> bf16 y, bf16 GEMM operands whatever the pointwise mode): the fused kernel or
        ``Bf16Declined``."""
        self._check()
        if not ops.dsconv_bf16_takes(x, x1, self.pointwise.weight.detach(), self.kernels_per_layer):
            raise Bf16Declined(self, f"the bf16 DS conv does not take input {tuple(x.shape)}"
                                     f"{'' if x1 is None else f' + {tuple(x1.shape)}'}, kernels_per_layer={self.kernels_per_layer} "
                                     "(needs k = 1 or 2, W a multiple of 8, set_dsconv_impl other than 'smem' and "
                                     "set_fused_dsconv(True))")
        dw_b = self.depthwise.bias.detach() if self.depthwise.bias is not None else None
        if shift is None:
            shift = self.pointwise.bias.detach() if self.pointwise.bias is not None else None
        return ops.dsconv_bf16(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, self.pointwise.weight.detach(), scale,
                               shift, relu, x1=x1, w_split=self.pw_operands("bf16"), gate=gate)

    def run(self, x, x1=None, scale=None, shift=None, relu=False, in_scale=None, in_shift=None, stats=None):
        """dw -> pw with the pw epilogue y = act(scale * acc + shift).  scale/shift None => (1, pointwise.bias).  A bf16 x is the
        bf16 route: bf16 output from the fused kernel (no input affine, no statistics)."""
        if ops.is_bf16(x) and in_scale is None and stats is None:
            return self._bf16(x, x1, scale, shift, relu)
        dw_b, shift, mode, split = self._operands(shift)
        if in_scale is None:
            # one kernel: the k*Cin-channel depthwise result never reaches HBM (where the shape allows)
            y = ops.dsconv(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, self.pointwise.weight.detach(),
                           scale, shift, relu, x1=x1, mode=mode, w_split=split, stats=stats)
            if y is not None:
                return y
        d = ops.dw3x3(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, x1=x1, in_scale=in_scale, in_shift=in_shift)
        return ops.pw1x1(d, self.pointwise.weight.detach(), scale, shift, relu, mode=mode, w_split=split, stats=stats)

    def run_head(self, x, scale, shift, relu, outconv, head):
        """``run`` followed by the OutConv ``outconv=(weight (K, Cout[,1,1]), bias or None)`` in the fused kernel's epilogue, ending
        in ``head``: "logits" (one class: the (B, 1, H, W) logits, ``ops.dsconv``) or "classes" (the (B, H, W) int64 class map
        of the K-class logits, ``ops.dsconv_classify``).  None where that kernel does not take the request: the caller then runs
        this conv and the OutConv separately."""
        if head not in ("logits", "classes"):
            raise ValueError(f"run_head: head must be 'logits' or 'classes', got {head!r}")
        if ops.is_bf16(x):          # the bf16 route: bf16 logits / the class map from bf16 activations
            self._check()
            dw_b = self.depthwise.bias.detach() if self.depthwise.bias is not None else None
            if shift is None:
                shift = self.pointwise.bias.detach() if self.pointwise.bias is not None else None
            return ops.dsconv_head_bf16(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer,
                                        self.pointwise.weight.detach(), scale, shift, relu, *outconv, head,
                                        w_split=self.pw_operands("bf16"))
        dw_b, shift, mode, split = self._operands(shift)
        args = (x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, self.pointwise.weight.detach(), scale, shift, relu)
        if head == "logits":
            return ops.dsconv(*args, mode=mode, w_split=split, outconv=outconv)
        return ops.dsconv_classify(*args, *outconv, mode=mode, w_split=split)

    def run_maxpool(self, x, scale, shift, relu, pooled_dtype=torch.float32):
        """``run`` that also returns MaxPool2d(2) of its output, written by the fused kernel's epilogue: (y, pooled), pooled None
        where that kernel does not take the shape (the caller then runs ``ops.maxpool2``).  A bf16 x: the bf16 route, pooled in
        ``pooled_dtype`` (bf16 or fp32), or ``Bf16Declined``."""
        if ops.is_bf16(x):
            self._check()
            if not ops.dsconv_maxpool_bf16_takes(x, None, self.pointwise.weight.detach(), self.kernels_per_layer):
                raise Bf16Declined(self, f"the bf16 DS conv with the max-pool epilogue does not take input {tuple(x.shape)}, "
                                         f"kernels_per_layer={self.kernels_per_layer} (needs k = 1 or 2, W a multiple of 8, "
                                         "set_dsconv_impl other than 'smem' and set_fused_dsconv(True))")
            dw_b = self.depthwise.bias.detach() if self.depthwise.bias is not None else None
            if shift is None:
                shift = self.pointwise.bias.detach() if self.pointwise.bias is not None else None
            return ops.dsconv_maxpool_bf16(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, self.pointwise.weight.detach(),
                                           scale, shift, relu, w_split=self.pw_operands("bf16"), pooled_dtype=pooled_dtype)
        dw_b, shift, mode, split = self._operands(shift)
        out = ops.dsconv_maxpool(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, self.pointwise.weight.detach(),
                                 scale, shift, relu, mode=mode, w_split=split)
        return out if out is not None else (self.run(x, scale=scale, shift=shift, relu=relu), None)

    def cbam_takes(self, x, x1=None, gate=False, pools=False) -> bool:
        """Whether ``run_cbam`` takes this input: the fused kernel with the serving forward's CBAM fusions.  For a bf16 x (the bf16
        route, gate only) always: that kernel is its only form, and ``run_cbam`` raises ``Bf16Declined`` where it declines."""
        if ops.is_bf16(x) and not pools:
            return True
        return ops.dsconv_cbam_takes(x, x1, self.pointwise.weight.detach(), self.kernels_per_layer, gate=gate, pools=pools)

    def run_cbam(self, x, x1=None, scale=None, shift=None, relu=False, gate=None, pools=False):
        """``run`` in one fused kernel that reads x as the CBAM output (x * sc) * sa (``gate=(sc, sa)``) and / or also returns
        the channel gate's partial pools and the 2x2 max-pool of its output (``pools``): see ``ops.dsconv_cbam``.  A bf16 x: the
        bf16 route, gate only."""
        if ops.is_bf16(x) and not pools:
            return self._bf16(x, x1, scale, shift, relu, gate=gate)
        dw_b, shift, mode, split = self._operands(shift)
        return ops.dsconv_cbam(x, self.depthwise.weight.detach(), dw_b, self.kernels_per_layer, self.pointwise.weight.detach(),
                               scale, shift, relu, x1=x1, mode=mode, w_split=split, gate=gate, pools=pools)

    def forward(self, x):
        if _needs_grad(self, x):
            from .autograd import DSConvFn
            self._check()
            return DSConvFn.run(self, x)
        return self.run(x)


# What a block call with an OutConv ends in: the OutConv's logits, their (B, H, W) int64 class map (the reference's
# ``torch.argmax(softmax(y_pred), dim=1)``, train_SmaAtUNet.py:76) or their (B, K, H, W) softmax probabilities.
HEADS = ("logits", "classes", "probs")


def _check_head(head, outconv):
    if head not in HEADS:
        raise ValueError(f"smaat_unet_b200: head must be one of {HEADS}, got {head!r}")
    if head != "logits" and outconv is None:
        raise ValueError(f"smaat_unet_b200: head={head!r} needs the OutConv that produces the logits")


def apply_head(module, x, head):
    """``module(x)``'s logits (``head="logits"``), or their class map / probabilities from the channel argmax / softmax kernel,
    with ``module`` run under no_grad: neither has a gradient.  The unfused end of every serving head (``OutConv.classes`` /
    ``probs``, the blocks' and models' routes that do not fuse it, ``engine.InferenceSession`` for models without ``forward_*``)."""
    if head == "logits":
        return module(x)
    with torch.no_grad():
        logits = module(x)
        return ops.argmax_channels(logits) if head == "classes" else ops.softmax_channels(logits)


class _DoubleConvBase(_CachingModule):
    """What DoubleConvDS and DoubleConv share: ``double_conv`` = (conv => BN => ReLU) * 2, its folded BatchNorm, and the routing
    of a call to its eval fast path, to autograd / batch statistics, and to an OutConv head.  A subclass provides
    ``_folded_conv`` (conv 0 or 3 with its folded BatchNorm and the ReLU) and ``_unfolded`` (the block under autograd or batch
    statistics), and may override ``_fused_last`` (the last conv with the OutConv and the head in its epilogue)."""

    def __init__(self, double_conv):
        super().__init__()
        self.double_conv = double_conv
        self._drop_caches()

    def _drop_caches(self):
        self._fold = {}

    def _folded(self, idx):
        """(scale, shift) of eval BatchNorm idx+1 folded with the bias of conv idx (a DS conv's pointwise bias); cached."""
        conv, bn = self.double_conv[idx], self.double_conv[idx + 1]
        cb = getattr(conv, "pointwise", conv).bias
        src = (bn.weight, bn.bias, bn.running_mean, bn.running_var, cb)
        key = _versions(*src)
        hit = self._fold.get(idx)
        if hit is None or hit[0] != key:
            with torch.no_grad():
                sc_sh = ops.bn_fold(bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var,
                                    cb.detach() if cb is not None else None, bn.eps)
            self._fold[idx] = (key, sc_sh, _held(*src))
            hit = self._fold[idx]
        return hit[1]

    def _eval_folded(self, *inputs):
        """True when this call runs the eval fast path: folded BatchNorm, no batch statistics, no autograd tape."""
        bns = (self.double_conv[1], self.double_conv[4])
        return not (_needs_grad(self, *inputs) or self.training
                    or any(not bn.track_running_stats or bn.running_mean is None for bn in bns))

    def _plain(self, x, x1, gate=None):
        """The block's own output."""
        if self._eval_folded(x, x1):
            return self._folded_conv(3, self._folded_conv(0, x, x1, gate))
        return self._unfolded(x, x1)

    def _run_head(self, x, x1, outconv, head, gate=None):
        """OutConv(block(x)) ending in ``head``.  Eval fast path: the first conv, then the last conv with the OutConv and the head
        in its epilogue where ``_fused_last`` takes it, else the last conv and ``apply_head``.  Under autograd or batch
        statistics: the plain block, then ``apply_head``."""
        if not (self._eval_folded(x, x1) and not _needs_grad(outconv, x)):
            return apply_head(outconv, self._plain(x, x1, gate), head)
        y = self._folded_conv(0, x, x1, gate)
        out = self._fused_last(y, outconv, head)
        return out if out is not None else apply_head(outconv, self._folded_conv(3, y), head)

    def _fused_last(self, y, outconv, head):
        """The last conv with the OutConv and the head in its epilogue, or None: then the last conv and ``apply_head`` run."""
        return None

    def forward(self, x):
        return self.run(x)


class DoubleConvDS(_DoubleConvBase):
    """models/unet_parts_depthwise_separable.py:10-39 -- (DS conv => BN => ReLU) * 2.

    Eval mode runs 4 kernels: dw, pw(+folded BN +ReLU), dw, pw(+folded BN +ReLU).
    """

    def __init__(self, in_channels, out_channels, mid_channels=None, kernels_per_layer=1):
        if not mid_channels:
            mid_channels = out_channels
        super().__init__(nn.Sequential(
            DepthwiseSeparableConv(in_channels, mid_channels, kernel_size=3, kernels_per_layer=kernels_per_layer, padding=1),
            nn.BatchNorm2d(mid_channels),
            nn.ReLU(inplace=True),
            DepthwiseSeparableConv(mid_channels, out_channels, kernel_size=3, kernels_per_layer=kernels_per_layer, padding=1),
            nn.BatchNorm2d(out_channels),
            nn.ReLU(inplace=True),
        ))

    def run(self, x, x1=None, outconv=None, gate=None, head="logits", with_maxpool=False, pooled_dtype=torch.float32):
        """``outconv`` (an OutConv module, inference only): return OutConv(block(x)) ending in ``head`` (``HEADS``) -- its logits,
        their (B, H, W) int64 class map or their (B, K, H, W) softmax probabilities (no gradient).  In the eval fast path the
        last kernel applies the OutConv and the head in its epilogue where it takes the shape (``_fused_last``), and the
        block's own output is then never materialised (models/SmaAt_UNet.py:55-56).
        ``gate=(sc, sa)``: x is the un-attended skip and the block's input is the CBAM output (x * sc) * sa, which the first
        DS conv computes as it loads x (inference only; materialised first where that kernel does not take it).
        ``with_maxpool`` (no ``outconv``): return (block(x), MaxPool2d(2) of it or None).  In the eval fast path the last DS conv
        writes the max-pool in its epilogue where it takes the shape (``DepthwiseSeparableConv.run_maxpool``; a bf16 x writes it in
        ``pooled_dtype``); elsewhere it is None and the DownDS that reads the block's output pools it itself."""
        _check_head(head, outconv)
        ops._req(x, "input", 4, bf16=True)
        if gate is not None and not (self._eval_folded(x, x1) and self.double_conv[0].cbam_takes(x, x1, gate=True)):
            x, gate = ops.cbam_scale(x, gate[0], gate[1]), None
        if outconv is not None:
            return self._run_head(x, x1, outconv, head, gate)
        if with_maxpool:
            if not self._eval_folded(x, x1):
                return self._plain(x, x1, gate), None
            s1, t1 = self._folded(3)
            return self.double_conv[3].run_maxpool(self._folded_conv(0, x, x1, gate), s1, t1, True, pooled_dtype=pooled_dtype)
        return self._plain(x, x1, gate)

    def _folded_conv(self, idx, x, x1=None, gate=None):
        s, t = self._folded(idx)
        if gate is not None:
            return self.double_conv[idx].run_cbam(x, x1=x1, scale=s, shift=t, relu=True, gate=gate)
        return self.double_conv[idx].run(x, x1=x1, scale=s, shift=t, relu=True)

    def _unfolded(self, x, x1):
        if _needs_grad(self, x, x1):
            from .autograd import DoubleConvDSFn
            return DoubleConvDSFn.run(self, x, x1)
        from . import functional as Fn       # batch statistics (and running-stat update), no tape
        return Fn.double_conv_fwd(self, x, x1)[0]

    def _fused_last(self, y, outconv, head):
        """The last DS conv with the OutConv and the head in its epilogue (smaat_dsconv_outconv_fwd, smaat_dsconv_classify_fwd),
        or None where that kernel does not take the shape (K > 32, Cout > 128, ...).  Logits only for a one-class OutConv: the
        K-class epilogue sums each logit in another order than the OutConv kernel, which would change the logits
        ``InferenceSession`` serves (DESIGN section 9).  Never probabilities: they are the channel softmax of the served logits,
        and a softmax epilogue measured slower than that kernel (DESIGN section 6)."""
        oc = outconv.conv
        if head == "probs" or (head == "logits" and oc.out_channels != 1):
            return None
        s1, t1 = self._folded(3)
        ob = oc.bias.detach() if oc.bias is not None else None
        return self.double_conv[3].run_head(y, s1, t1, True, (oc.weight.detach(), ob), head)


# The reference calls ``cbamN(x)`` and then ``downN(x)`` on the same un-attended map (models/SmaAt_UNet.py:42-50,
# unet_precip_regression_lightning.py:148-157): the channel gate's global pools and the 2x2 max-pool are produced by ONE
# read of x.  The plain-call API has no way to hand the pooled map over, so the CBAM leaves it in this one-slot stash,
# keyed on the identity of x; DownDS takes it when (and only when) it is called on the very same tensor.
_maxpool_stash = None


def _tensor_key(x):
    return (x.data_ptr(), x._version, tuple(x.shape), tuple(x.stride()), x.device.index)


def _stash_maxpool(x, pooled):
    """The entry names x by a weak reference (checked with ``is``) as well as by address and version: a tensor that is
    allocated on x's block after x is freed has the same address and, fresh from a kernel, the same version 0."""
    global _maxpool_stash
    _maxpool_stash = (weakref.ref(x), _tensor_key(x), pooled)


def _take_stashed_maxpool(x):
    """The stashed MaxPool2d(2)(x), or None.  Never under autograd: the stashed map was produced without a tape, so taking
    it for an ``x`` that requires grad would cut the max-pool's gradient path to ``x``."""
    global _maxpool_stash
    hit = _maxpool_stash
    if hit is None or not isinstance(x, torch.Tensor) or not x.is_cuda:
        return None
    if torch.is_grad_enabled() and x.requires_grad:
        return None
    if hit[0]() is not x or hit[1] != _tensor_key(x):
        return None
    _maxpool_stash = None
    return hit[2]


class _Down(nn.Module):
    """MaxPool2d(2) then the double conv ``maxpool_conv[1]``: DownDS and Down."""

    def forward(self, x, pooled=None, **run_kw):
        """``pooled``: MaxPool2d(2)(x) when the caller already has it.  Called plainly (``down(x)``, as the reference does)
        it first looks for the 2x2 max-pool the preceding ``CBAM(x)`` call left behind (see ``CBAM.forward``): SmaAt-UNet's
        ``cbamN(x)`` -> ``downN(x)`` (models/SmaAt_UNet.py:42-50), UNetAttention's (unet_precip_regression_lightning.py:68-77).
        ``run_kw`` goes to the double conv's ``run`` (DownDS: ``with_maxpool`` / ``pooled_dtype``, DoubleConvDS.run)."""
        if pooled is None:
            pooled = _take_stashed_maxpool(x)
        if pooled is None:
            if _needs_grad(self, x):
                from .autograd import MaxPool2Fn
                pooled = MaxPool2Fn.apply(x) if x.requires_grad else ops.maxpool2(x)
            else:
                pooled = ops.maxpool2(x)
        return self.maxpool_conv[1].run(pooled, **run_kw)


class DownDS(_Down):
    """models/unet_parts_depthwise_separable.py:42-53 -- MaxPool2d(2) then DoubleConvDS."""

    def __init__(self, in_channels, out_channels, kernels_per_layer=1):
        super().__init__()
        self.maxpool_conv = nn.Sequential(
            nn.MaxPool2d(2),
            DoubleConvDS(in_channels, out_channels, kernels_per_layer=kernels_per_layer),
        )


class _TransposedUp(_CachingModule):
    """The upsample step of Up / UpDS: nn.Upsample(x2, bilinear, align_corners=True), or with ``bilinear=False``
    ConvTranspose2d(Cin, Cin // 2, kernel_size=2, stride=2), then F.pad to the skip.  kernel = stride, so the transposed conv is
    one wgmma pointwise GEMM to the 4 packed taps + a pixel shuffle (csrc/convt.cu)."""

    def __init__(self, in_channels, bilinear):
        super().__init__()
        self.bilinear = bilinear
        if bilinear:
            self.up = nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True)
        else:
            self.up = nn.ConvTranspose2d(in_channels, in_channels // 2, kernel_size=2, stride=2)
        self._packed = None

    def _drop_caches(self):
        self._packed = None

    def _packed_weight(self):
        """((4 Cout, Cin) GEMM matrix of the transposed conv, its operands in the current mode (``ops.derived_operands``: None
        where the mode takes it as it is)); cached on the weight's version and the mode."""
        w = self.up.weight
        key = (_versions(w), ops.get_pointwise_mode())
        in_train_capture = self.training and torch.cuda.is_current_stream_capturing()
        if in_train_capture or self._packed is None or self._packed[0] != key:
            with torch.no_grad():
                wp = ops.convt2x2_pack_weight(w.detach())
                split = ops.derived_operands(wp, ops.PW_MODES[ops.get_pointwise_mode()])
            self._packed = (None if in_train_capture else key, wp, split, _held(w))
        return self._packed[1], self._packed[2]

    def _up_transposed(self, x1, Ho, Wo):
        up = self.up
        if (up.kernel_size, up.stride, up.padding, up.output_padding, up.dilation, up.groups) != ((2, 2), (2, 2), (0, 0), (0, 0), (1, 1), 1):
            raise NotImplementedError(f"{type(self).__name__}: only the reference's ConvTranspose2d(kernel_size=2, stride=2) is implemented "
                                      "(parts_ds.py:72, unet_parts.py:50)")
        wp, split = self._packed_weight()
        if _needs_grad(up, x1):
            from .autograd import ConvT2x2PadFn
            return ConvT2x2PadFn.apply(x1, up.weight, up.bias, Ho, Wo, wp, split)
        t = ops.pw1x1(x1, wp, None, None, False, w_split=split)
        return ops.pixel_shuffle2_pad(t, up.bias.detach() if up.bias is not None else None, up.out_channels, Ho, Wo)

    def _upsampled(self, x1, x2):
        """x1 upsampled x2 and padded to x2's plane."""
        Ho, Wo = x2.shape[2], x2.shape[3]
        if not self.bilinear:
            return self._up_transposed(x1, Ho, Wo)
        if torch.is_grad_enabled() and x1.requires_grad:
            from .autograd import Upsample2xPadFn
            return Upsample2xPadFn.apply(x1, Ho, Wo)
        # the bf16 route: the upsampled map joins a bf16 skip, so it is written in bf16 (from fp32 level 4 into up2)
        return ops.upsample2x_pad(x1, Ho, Wo, out_dtype=torch.bfloat16 if ops.is_bf16(x2) else torch.float32)


class UpDS(_TransposedUp):
    """models/unet_parts_depthwise_separable.py:56-86 -- upsample x2, pad to the skip, concat, DoubleConvDS.

    The concat is never materialised: the first depthwise kernel reads [skip, up] as a virtual concat.
    ``bilinear=False`` (ConvTranspose2d(in, in // 2, 2, stride=2), :72-73): kernel = stride, so the transposed conv is one
    wgmma pointwise GEMM to the 4 packed taps + a pixel shuffle (csrc/convt.cu).
    """

    def __init__(self, in_channels, out_channels, bilinear=True, kernels_per_layer=1):
        super().__init__(in_channels, bilinear)
        self.conv = DoubleConvDS(in_channels, out_channels, in_channels // 2 if bilinear else None, kernels_per_layer=kernels_per_layer)

    def forward(self, x1, x2, outconv=None, gate=None, head="logits"):
        """``gate=(sc, sa)`` (serving forward, inference only): x2 is the un-attended skip, and the block reads the CBAM output
        (x2 * sc) * sa as it loads it (DoubleConvDS.run).  ``outconv``: the OutConv's logits of the block's output, or with
        ``head="classes"`` / ``"probs"`` their class map / softmax probabilities."""
        _check_head(head, outconv)
        return self.conv.run(x2, x1=self._upsampled(x1, x2), outconv=outconv, gate=gate, head=head)


class DoubleConv(_DoubleConvBase):
    """models/unet_parts.py:8-25 -- (Conv2d 3x3 => BN => ReLU) * 2, the dense block of UNet / UNetAttention.

    Eval mode runs 2 kernels: conv3x3 (+folded BN +ReLU) twice (csrc/conv3x3_tc.cu; the exact CUDA-core kernel in 'fp32'
    mode and for the shapes the tensor-core kernel declines).  ``run(x, x1)`` reads the virtual concat [x, x1].
    """

    def __init__(self, in_channels, out_channels, mid_channels=None):
        if not mid_channels:
            mid_channels = out_channels
        super().__init__(nn.Sequential(
            nn.Conv2d(in_channels, mid_channels, kernel_size=3, padding=1),
            nn.BatchNorm2d(mid_channels),
            nn.ReLU(inplace=True),
            nn.Conv2d(mid_channels, out_channels, kernel_size=3, padding=1),
            nn.BatchNorm2d(out_channels),
            nn.ReLU(inplace=True),
        ))

    def _drop_caches(self):
        super()._drop_caches()
        self._packed = {}

    def _check(self):
        for idx in (0, 3):
            c = self.double_conv[idx]
            if (c.kernel_size, c.padding, c.stride, c.dilation, c.groups) != ((3, 3), (1, 1), (1, 1), (1, 1), 1) or c.padding_mode != "zeros":
                raise NotImplementedError("smaat_unet_b200 implements the dense conv the reference uses: 3x3, padding=1, stride 1, "
                                          "groups=1 (unet_parts.py:16,19)")

    def packed(self, idx, C0, C1=0, flip_transpose=False):
        """(packed weight, its operands in the current mode (``ops.derived_operands``; None where the mode takes the packed
        weight as it is)) of conv ``idx`` for inputs [C0 | C1]; with ``flip_transpose`` the input-gradient form.  Cached on the
        weight's version and the mode; re-derived inside a training capture."""
        w = self.double_conv[idx].weight
        mode = ops.get_pointwise_mode()
        key = (_versions(w), mode)
        slot = (idx, C0, C1, bool(flip_transpose))
        in_train_capture = self.training and torch.cuda.is_current_stream_capturing()
        hit = self._packed.get(slot)
        if in_train_capture or hit is None or hit[0] != key:
            with torch.no_grad():
                wp = ops.conv3x3_pack_weight(w.detach(), C0, C1, flip_transpose)
                wops = ops.derived_operands(wp, ops.PW_MODES[mode])
            hit = (None if in_train_capture else key, (wp, wops), _held(w))
            self._packed[slot] = hit
        return hit[1]

    def conv(self, idx, x, x1=None, scale=None, shift=None, relu=False, stats=None):
        """Conv ``idx`` (0 or 3) over [x, x1] with the epilogue y = act(scale * acc + shift)."""
        self._check()
        C0, C1 = x.shape[1], (x1.shape[1] if x1 is not None else 0)
        wp, wops = self.packed(idx, C0, C1)
        return ops.conv3x3(x, wp, self.double_conv[idx].out_channels, scale, shift, relu, x1=x1, w_split=wops, stats=stats)

    def run(self, x, x1=None, outconv=None, head="logits"):
        """``outconv`` (an OutConv module): return OutConv(block(x)) ending in ``head`` (``HEADS``) -- its logits, their
        (B, H, W) int64 class map or their (B, K, H, W) softmax probabilities (no gradient): the block, the OutConv kernel and
        the channel argmax / softmax kernel (``apply_head``)."""
        _check_head(head, outconv)
        ops._req(x, "input", 4)
        if x1 is not None:
            ops._req(x1, "input", 4)
        self._check()
        if outconv is not None:
            return self._run_head(x, x1, outconv, head)
        return self._plain(x, x1)

    def _folded_conv(self, idx, x, x1=None, gate=None):
        s, t = self._folded(idx)
        return self.conv(idx, x, x1, scale=s, shift=t, relu=True)

    def _unfolded(self, x, x1):
        if _needs_grad(self, x, x1):
            from .autograd import DoubleConvFn
            return DoubleConvFn.run(self, x, x1)
        from . import functional as Fn       # batch statistics (and running-stat update), no tape
        return Fn.dense_double_conv_fwd(self, x, x1)[0]


class Down(_Down):
    """models/unet_parts.py:28-36 -- MaxPool2d(2) then DoubleConv."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.maxpool_conv = nn.Sequential(nn.MaxPool2d(2), DoubleConv(in_channels, out_channels))


class Up(_TransposedUp):
    """models/unet_parts.py:39-64 -- upsample x2 (bilinear, or ConvTranspose2d), pad to the skip, concat, DoubleConv.

    The concat is never materialised: the first 3x3 conv reads [skip, up] as a virtual concat."""

    def __init__(self, in_channels, out_channels, bilinear=True):
        super().__init__(in_channels, bilinear)
        self.conv = DoubleConv(in_channels, out_channels, in_channels // 2 if bilinear else None)

    def forward(self, x1, x2, outconv=None, head="logits"):
        """``outconv``: return OutConv's logits of the block's output; with ``head="classes"`` / ``"probs"`` their class map /
        softmax probabilities (``DoubleConv.run``)."""
        _check_head(head, outconv)
        ops._req(x1, "x1", 4)
        ops._req(x2, "x2", 4)
        return self.conv.run(x2, x1=self._upsampled(x1, x2), outconv=outconv, head=head)


class OutConv(nn.Module):
    """models/unet_parts.py:67-73 -- 1x1 conv to n_classes."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size=1)

    def forward(self, x):
        if _needs_grad(self, x):
            from .autograd import OutConvFn
            return OutConvFn.apply(x, self.conv.weight, self.conv.bias)
        return ops.outconv(x, self.conv.weight.detach(), self.conv.bias.detach() if self.conv.bias is not None else None)

    def classes(self, x):
        """The (B, H, W) int64 class map argmax_c OutConv(x) (the reference's ``torch.argmax(softmax(y_pred), dim=1)``,
        train_SmaAtUNet.py:76): this module's logits, then the channel argmax kernel.  Inference only: a class map has no gradient."""
        return apply_head(self, x, "classes")

    def probs(self, x):
        """The (B, K, H, W) class probabilities softmax_c OutConv(x) (the reference's ``softmax(y_pred)``, train_SmaAtUNet.py:76):
        this module's logits, then the channel softmax kernel.  Inference only: no gradient."""
        return apply_head(self, x, "probs")


class Flatten(nn.Module):
    """models/layers.py:85-87 (kept so that MLP indices -- state_dict keys MLP.1 / MLP.3 -- match)."""

    def forward(self, x):
        return x.view(x.size(0), -1)


class ChannelAttention(nn.Module):
    """models/layers.py:90-111."""

    def __init__(self, input_channels, reduction_ratio=16):
        super().__init__()
        self.input_channels = input_channels
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.max_pool = nn.AdaptiveMaxPool2d(1)
        self.MLP = nn.Sequential(
            Flatten(),
            nn.Linear(input_channels, input_channels // reduction_ratio),
            nn.ReLU(),
            nn.Linear(input_channels // reduction_ratio, input_channels),
        )

    def gate(self, x, with_maxpool=False, pooled_dtype=torch.float32):
        """sigmoid(MLP(avg) + MLP(max)) as a (B, C) tensor.  ``with_maxpool``: also return MaxPool2d(2)(x) (or None), computed
        in the same read of x as the global pools; a bf16 x (the bf16 route) writes it in ``pooled_dtype``."""
        l1, l2 = self.MLP[1], self.MLP[3]
        # 512 channels: the MLP runs as a second launch instead of in the last-arriving pooling CTA of each image, whose
        # serial 512-channel MLP sits on the critical path of these small planes
        one = None if x.shape[1] >= 512 else ops.cbam_pool_mlp(x, l1.weight.detach(), l1.bias.detach(), l2.weight.detach(), l2.bias.detach(),
                                                               with_maxpool=with_maxpool, pooled_dtype=pooled_dtype)
        if one is not None:          # pools + MLP + sigmoid (+ the 2x2 max-pool) in one launch
            sc, _, _, pooled = one
            return (sc, pooled) if with_maxpool else sc
        pooled = None
        fused = ops.cbam_pool_maxpool(x, pooled_dtype=pooled_dtype) if with_maxpool else None
        if fused is not None:
            avg, mx, pooled = fused
        else:
            avg, mx = ops.cbam_pool(x)
        sc = ops.cbam_mlp(avg, mx, l1.weight.detach(), l1.bias.detach(), l2.weight.detach(), l2.bias.detach())
        return (sc, pooled) if with_maxpool else sc

    def forward(self, x):
        _no_autograd(self, x)
        sc = self.gate(x)
        ones = torch.ones((x.shape[0], 1, x.shape[2], x.shape[3]), device=x.device, dtype=torch.float32)
        return ops.cbam_scale(x, sc, ones)


class SpatialAttention(_CachingModule):
    """models/layers.py:114-129."""

    def __init__(self, kernel_size=7):
        super().__init__()
        assert kernel_size in (3, 7), "kernel size must be 3 or 7"
        padding = 3 if kernel_size == 7 else 1
        self.conv = nn.Conv2d(2, 1, kernel_size=kernel_size, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(1)
        self._fold = None

    def _drop_caches(self):
        self._fold = None

    def bn_affine(self):
        """Device tensor [scale, shift] of the eval-mode BatchNorm2d(1); cached."""
        if self.bn.training:
            raise NotImplementedError("standalone SpatialAttention in train mode is not implemented (CBAM handles it); "
                                      "call .eval() or use CBAM")
        bn = self.bn
        src = (bn.weight, bn.bias, bn.running_mean, bn.running_var)
        key = _versions(*src)
        if self._fold is None or self._fold[0] != key:
            with torch.no_grad():
                s, t = ops.bn_fold(bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var, None, bn.eps)
                self._fold = (key, torch.cat([s, t]), _held(*src))
        return self._fold[1]

    def gate(self, x, sc):
        pooled = ops.cbam_reduce(x, sc)
        return ops.cbam_gate(pooled, self.conv.weight.detach(), self.bn_affine())

    def forward(self, x):
        _no_autograd(self, x)
        ones = torch.ones((x.shape[0], x.shape[1]), device=x.device, dtype=torch.float32)
        return ops.cbam_scale(x, ones, self.gate(x, ones))


class CBAM(nn.Module):
    """models/layers.py:132-141 -- channel attention then spatial attention: 3 kernels, 4|x| of traffic."""

    def __init__(self, input_channels, reduction_ratio=16, kernel_size=7):
        super().__init__()
        self.channel_att = ChannelAttention(input_channels, reduction_ratio=reduction_ratio)
        self.spatial_att = SpatialAttention(kernel_size=kernel_size)
        self.stash_maxpool = True     # False: never produce the max-pool in a plain call (e.g. no DownDS follows)

    def forward(self, x, out=None, with_maxpool=False):
        """``with_maxpool=True`` returns (CBAM(x), MaxPool2d(2)(x) or None) explicitly; a plain ``cbam(x)`` (the reference's
        call) returns CBAM(x) and stashes the max-pool for the DownDS that follows (models/SmaAt_UNet.py:42-50)."""
        if _needs_grad(self, x):
            from .autograd import CBAMFn
            y = CBAMFn.run(self, x)
            return (y, None) if with_maxpool else y
        if self.spatial_att.bn.training or not self.spatial_att.bn.track_running_stats:
            from . import functional as Fn       # batch statistics for the gate's BatchNorm2d(1), no tape
            y = Fn.cbam_fwd(self, ops._dense(x, "x"))[0]
            return (y, None) if with_maxpool else y
        # one read of x gives the global pools AND MaxPool2d(2)(x) (shape permitting); a plain call leaves the latter for
        # the DownDS that the reference calls next on the same x
        pooled = None
        if with_maxpool or self.stash_maxpool:
            sc, pooled = self.channel_att.gate(x, with_maxpool=True)
            if pooled is not None and not with_maxpool:
                _stash_maxpool(x, pooled)
        else:
            sc = self.channel_att.gate(x)
        # three launches: [pools + MLP (+ max-pool)], channel reduce, [k x k gate + scale]
        red = ops.cbam_reduce(x, sc)
        y = ops.cbam_gate_scale(x, sc, red, self.spatial_att.conv.weight.detach(), self.spatial_att.bn_affine(), out=out)
        if y is None:
            sa = ops.cbam_gate(red, self.spatial_att.conv.weight.detach(), self.spatial_att.bn_affine())
            y = ops.cbam_scale(x, sc, sa, out=out)
        return (y, pooled) if with_maxpool else y

    def serving_gates(self, x, pooled_dtype=torch.float32):
        """Serving forward, inference only: CBAM(x)'s two gates (sc (B, C), sa (B, 1, H, W)) and MaxPool2d(2)(x) (or None),
        without writing CBAM(x): pools + MLP (+ max-pool), channel reduce, k x k gate -- the same launches and values as
        ``forward``.  The consumer applies (x * sc) * sa as it loads x (``UpDS.forward(..., gate=(sc, sa))``).  A bf16 x (the
        bf16 route): the gates stay fp32, the max-pool is written in ``pooled_dtype``."""
        sc, pooled = self.channel_att.gate(x, with_maxpool=True, pooled_dtype=pooled_dtype)
        red = ops.cbam_reduce(x, sc)
        return sc, ops.cbam_gate(red, self.spatial_att.conv.weight.detach(), self.spatial_att.bn_affine()), pooled


def cached_tensors(model):
    """Every tensor the eval fast path derived from ``model``'s parameters (folded BatchNorm affine, tf32 hi/lo splits, bf16
    packs, packed 3x3 and transposed-conv weights).  A CUDA graph captured over the eval forward has their addresses baked in:
    whoever owns the graph must keep them alive (``graph_tensors``)."""
    out = []
    for m in model.modules():
        if isinstance(m, DepthwiseSeparableConv) and m._wsplit is not None:
            out.extend(t for t in m._wsplit if t is not None)
        elif isinstance(m, (DoubleConvDS, DoubleConv)):
            for entry in m._fold.values():
                out.extend(entry[1])
            if isinstance(m, DoubleConv):
                for entry in m._packed.values():
                    wp, wops = entry[1]
                    out.append(wp)
                    out.extend(t for t in wops or () if t is not None)
        elif isinstance(m, SpatialAttention) and m._fold is not None:
            out.append(m._fold[1])
        if isinstance(m, _TransposedUp) and m._packed is not None:
            _, wp, split, _ = m._packed
            out.append(wp)
            out.extend(t for t in split or () if t is not None)
    return out


def graph_tensors(model):
    """Everything a CUDA graph captured over ``model``'s eval forward reads by address, other than its own inputs and
    activations: the caches (``cached_tensors``), and aliases of every parameter and buffer, which the kernels read in
    place.  The aliases keep the storage alive after the model lets it go (``TrainSession`` re-points the parameters into
    its flat buffer, ``load_state_dict(..., assign=True)`` replaces them, a mode switch drops the caches)."""
    return cached_tensors(model) + [t.detach() for t in list(model.parameters()) + list(model.buffers())]
