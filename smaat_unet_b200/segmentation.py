"""Multi-class segmentation: cross-entropy loss and IoU bookkeeping on the device, one kernel pass, no host sync.

Host-side mirror of the reference's segmentation workflow (train_SmaAtUNet.py:139-199):
  * ``CrossEntropyLoss``   -- ``nn.CrossEntropyLoss()`` (train_SmaAtUNet.py:182) with the reference's constructor call;
    class-index or probability targets, ``reduction`` "mean" / "sum", any ``ignore_index``
  * ``CrossEntropyLossWithOptions`` -- ``nn.CrossEntropyLoss`` with torch's full constructor: also ``weight``,
    ``label_smoothing`` and ``reduction="none"``
  * ``ConfusionMatrix`` / ``IoU`` -- metric/confusionmatrix.py and metric/iou.py: same constructors, ``add`` / ``value`` /
    ``reset``; the counts stay on the device and ``value()`` makes the one device->host copy
  * ``ce_step(logits, target, metrics)`` -- the loss, its gradient and the IoU update of one training / validation batch
    in ONE pass over the logits: the counterpart of ``metrics.step_loss``
The arithmetic is ``smaat_ce_fwd`` (the plain loss), ``smaat_cross_entropy_fwd`` (any of the options), ``smaat_confusion_add``
and ``smaat_onehot_classes`` (include/smaat_b200.h).

Argmax.  The fused path takes the argmax of the LOGITS; the reference takes it of ``softmax(logits)``
(train_SmaAtUNet.py:76).  Softmax is monotonic, so the two agree except where two logits lie within about one ulp of each
other and softmax rounds their probabilities to the same float: there the reference picks the lower index among the tied
probabilities while the logits may still order them.  ``IoU.add`` with integer predictions counts exactly what it is given.

Labels.  The reference asserts on every batch that labels lie in [0, K) (a device->host sync).  Here an out-of-range label
is counted on the device and never used as an index: the loss comes out NaN (torch raises a device-side assert instead),
the pixel's gradient is 0, and a metric that saw one raises from ``value()``.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from . import _lib
from .ops import _call, _ptr, _stream

MAX_CLASSES = 1024


# ------------------------------------------------------------------------------------------------ kernel wrappers
def _logits_view(logits, name="logits"):
    if not isinstance(logits, torch.Tensor) or not logits.is_cuda or logits.dtype != torch.float32:
        raise RuntimeError(f"smaat segmentation: {name} must be a float32 CUDA tensor (got {getattr(logits, 'dtype', None)} on "
                           f"{getattr(logits, 'device', None)}); there is no CPU fallback")
    if logits.dim() < 2:
        raise RuntimeError(f"smaat segmentation: {name} must be (N, K, ...), got shape {tuple(logits.shape)}")
    return logits if logits.is_contiguous() else logits.contiguous()


def _labels(t, device, name):
    """Class indices as a dense int64 tensor on `device` (a host tensor is copied over: train_SmaAtUNet.py:77 passes it un-moved)."""
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(np.asarray(t))
    if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
        raise RuntimeError(f"smaat segmentation: {name} must hold integer class indices, got {t.dtype}")
    t = t.to(device=device, dtype=torch.int64, non_blocking=True)
    return t if t.is_contiguous() else t.contiguous()


def ce_forward(logits, target, ignore_index=-100, use_ignore=True, want_grad=False, conf=None):
    """One pass of ``smaat_ce_fwd``: returns (batch_acc double[3], dlogits or None).  ``conf``: int64 (K, K) added into."""
    x = _logits_view(logits)
    B, K = x.shape[0], x.shape[1]
    if K > MAX_CLASSES:
        raise NotImplementedError(f"smaat segmentation: {K} classes, the kernel supports at most {MAX_CLASSES}")
    y = _labels(target, x.device, "target")
    if tuple(y.shape) != (B,) + tuple(x.shape[2:]):
        raise RuntimeError(f"smaat segmentation: target {tuple(y.shape)} does not match logits {tuple(x.shape)}")
    P = x.numel() // max(B * K, 1)
    acc = torch.empty(3, device=x.device, dtype=torch.float64)
    dl = torch.empty_like(x) if want_grad else None
    if x.numel() == 0:
        acc.zero_()
        if dl is not None:
            dl.zero_()
        return acc, dl
    lib = _lib.load()
    n = B * P
    _call("smaat_ce_fwd", 4 * x.numel() * (2 if want_grad else 1) + 8 * n, 5 * x.numel(), lib.smaat_ce_fwd, _ptr(x), _ptr(y),
          B, K, P, int(ignore_index), int(bool(use_ignore)), _ptr(acc), _ptr(dl), _ptr(conf), _stream())
    return acc, dl


def _is_prob_target(logits, target):
    """A probability (or one-hot float) target: a floating-point tensor with the logits' shape, as torch decides."""
    return isinstance(target, torch.Tensor) and target.is_floating_point() and tuple(target.shape) == tuple(logits.shape)


def _check_options(logits, target, weight, label_smoothing, ignore_index):
    """Host-side checks of the loss options, with torch's messages; returns the weight as a dense fp32 device tensor."""
    K = logits.shape[1] if isinstance(logits, torch.Tensor) and logits.dim() >= 2 else None
    if K is not None and K > MAX_CLASSES:
        raise NotImplementedError(f"smaat segmentation: {K} classes, the kernel supports at most {MAX_CLASSES}")
    eps = float(label_smoothing)
    if not 0.0 <= eps <= 1.0:
        raise RuntimeError(f"label_smoothing must be between 0.0 and 1.0. Got: {eps}")
    if weight is not None:
        if not isinstance(weight, torch.Tensor) or weight.dim() != 1 or weight.numel() != K:
            raise RuntimeError(f"cross_entropy: weight tensor should be defined either for all {K} classes or no classes but got "
                               f"weight tensor of shape: {list(getattr(weight, 'shape', []))}")
        weight = weight.detach()
        if weight.device != logits.device or weight.dtype != torch.float32 or not weight.is_contiguous():
            weight = weight.to(device=logits.device, dtype=torch.float32).contiguous()
    if _is_prob_target(logits, target) and int(ignore_index) >= 0:
        raise RuntimeError("ignore_index is not supported for floating point target")
    return weight


def ce_forward_opts(logits, target, weight=None, label_smoothing=0.0, ignore_index=-100, use_ignore=True, want_grad=False,
                    want_map=False, conf=None):
    """One pass of ``smaat_cross_entropy_fwd``: returns (batch_acc double[4], per-pixel loss (B, ...) or None, dlogits or
    None).  ``target``: int64 class indices (B, ...) or float probabilities shaped like the logits; ``weight``: fp32 (K,) on
    the logits' device or None; ``conf``: int64 (K, K) added into."""
    x = _logits_view(logits)
    B, K = x.shape[0], x.shape[1]
    if K > MAX_CLASSES:
        raise NotImplementedError(f"smaat segmentation: {K} classes, the kernel supports at most {MAX_CLASSES}")
    prob = _is_prob_target(x, target)
    if prob:
        q = target.detach().to(device=x.device, dtype=torch.float32, non_blocking=True)
        q = q if q.is_contiguous() else q.contiguous()
        y, use_ignore = None, False
    else:
        y, q = _labels(target, x.device, "target"), None
        if tuple(y.shape) != (B,) + tuple(x.shape[2:]):
            raise RuntimeError(f"smaat segmentation: target {tuple(y.shape)} does not match logits {tuple(x.shape)}")
    P = x.numel() // max(B * K, 1)
    acc = torch.empty(4, device=x.device, dtype=torch.float64)
    lmap = torch.empty((B,) + tuple(x.shape[2:]), device=x.device, dtype=torch.float32) if want_map else None
    dl = torch.empty_like(x) if want_grad else None
    if x.numel() == 0:
        acc.zero_()
        for t in (lmap, dl):
            if t is not None:
                t.zero_()
        return acc, lmap, dl
    lib = _lib.load()
    n = B * P
    nbytes = 4 * x.numel() * ((2 if want_grad else 1) + (1 if prob else 0)) + (0 if prob else 8 * n) + (4 * n if want_map else 0)
    _call("smaat_cross_entropy_fwd", nbytes, 8 * x.numel(), lib.smaat_cross_entropy_fwd, _ptr(x), _ptr(y), _ptr(q), _ptr(weight),
          B, K, P, float(label_smoothing), int(ignore_index), int(bool(use_ignore)), _ptr(acc), _ptr(lmap), _ptr(dl), _ptr(conf),
          _stream())
    return acc, lmap, dl


def onehot_classes(target, device, num_classes):
    """``smaat_onehot_classes``: (N, K, ...) one-hot targets -> int64 (N, ...) classes, -1 where a row fails the reference's
    checks (values in [0, 1], row sum 1)."""
    if not isinstance(target, torch.Tensor):
        target = torch.as_tensor(np.asarray(target))
    if target.dim() < 2 or target.shape[1] != num_classes:
        raise AssertionError("Onehot target does not match size of confusion matrix")
    q = target.to(device=device, dtype=torch.float32, non_blocking=True)
    q = q if q.is_contiguous() else q.contiguous()
    N, K = q.shape[0], q.shape[1]
    classes = torch.empty((N,) + tuple(q.shape[2:]), device=device, dtype=torch.int64)
    if q.numel() == 0:
        return classes
    P = q.numel() // (N * K)
    _call("smaat_onehot_classes", 4 * q.numel() + 8 * N * P, 0, _lib.load().smaat_onehot_classes, _ptr(q), _ptr(classes), N, K, P,
          _stream())
    return classes


def confusion_add(pred, target, conf, invalid, num_classes):
    """``smaat_confusion_add``: conf[target][pred] += 1 over the (pred, target) pairs; out-of-range pairs into ``invalid``."""
    p = _labels(pred, conf.device, "predicted")
    t = _labels(target, conf.device, "target")
    if p.numel() != t.numel():
        raise RuntimeError(f"smaat segmentation: {p.numel()} predictions vs {t.numel()} targets")
    if p.numel() == 0:
        return
    lib = _lib.load()
    _call("smaat_confusion_add", 16 * p.numel(), 0, lib.smaat_confusion_add, _ptr(p), _ptr(t), p.numel(), int(num_classes),
          _ptr(conf), _ptr(invalid), _stream())


# ------------------------------------------------------------------------------------------------ loss
class _CrossEntropyFn(torch.autograd.Function):
    """Cross-entropy over class-index targets with the gradient produced by the forward pass."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, reduction, metrics):
        cm = _confusion_of(metrics)
        acc, dl = ce_forward(logits.detach(), target, ignore_index, True, want_grad=logits.requires_grad,
                             conf=None if cm is None else cm._conf)
        if cm is not None:
            cm._add_invalid(acc[2])
        n, bad = acc[1], acc[2] > 0
        if reduction == "mean":
            loss = acc[0] / n                                  # 0 / 0 = NaN when no pixel counts, as in torch
            scale = torch.where(n > 0, 1.0 / n, torch.zeros_like(n))   # device scalar: no sync
        else:
            loss = acc[0]
            scale = torch.ones_like(n)
        loss = torch.where(bad, torch.full_like(loss, float("nan")), loss)
        ctx.save_for_backward(dl, scale)
        return loss.to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        dl, scale = ctx.saved_tensors
        return dl * (g * scale).to(torch.float32), None, None, None, None


class _CrossEntropyOptsFn(torch.autograd.Function):
    """Cross-entropy with class weights, label smoothing, probability targets or ``reduction="none"``
    (``smaat_cross_entropy_fwd``); the gradient is produced by the forward pass and scaled in the backward: by the device
    scalar 1 / D for "mean", by the upstream per-pixel gradient for "none"."""

    @staticmethod
    def forward(ctx, logits, target, weight, label_smoothing, ignore_index, reduction, metrics):
        cm = _confusion_of(metrics)
        prob = _is_prob_target(logits, target)
        acc, lmap, dl = ce_forward_opts(logits.detach(), target, weight, label_smoothing, ignore_index, not prob,
                                        want_grad=logits.requires_grad, want_map=reduction == "none",
                                        conf=None if cm is None else cm._conf)
        if cm is not None:
            cm._add_invalid(acc[2])
        ctx.none = reduction == "none"
        if ctx.none:
            ctx.save_for_backward(dl)
            return lmap                                        # 0 on ignored pixels, NaN on invalid labels
        n, d = acc[1], acc[3]
        nan = torch.full_like(d, float("nan"))
        if reduction == "mean":
            loss = torch.where(d != 0, acc[0] / d, nan)        # torch: NaN when nothing counts, or every counted weight is 0
            scale = torch.where(n > 0, torch.where(d != 0, 1.0 / d, nan), torch.zeros_like(d))   # device scalars: no sync
        else:
            loss = acc[0]
            scale = torch.ones_like(d)
        if not prob:                                           # probability targets are not validated, as in torch
            loss = torch.where(acc[2] > 0, nan, loss)
        ctx.save_for_backward(dl, scale)
        return loss.to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        if ctx.none:
            (dl,) = ctx.saved_tensors
            return dl * g.unsqueeze(1).to(torch.float32), None, None, None, None, None, None
        dl, scale = ctx.saved_tensors
        return dl * (g * scale).to(torch.float32), None, None, None, None, None, None


def _check_target(logits, target):
    if isinstance(target, torch.Tensor) and target.is_floating_point() and not _is_prob_target(logits, target):
        raise RuntimeError(f"smaat CrossEntropyLoss: a floating-point target must have the logits' shape {tuple(logits.shape)} "
                           f"(probabilities), got {tuple(target.shape)}; class indices must be integers")
    if isinstance(target, torch.Tensor) and not target.is_floating_point() and target.dim() == logits.dim():
        raise NotImplementedError("smaat CrossEntropyLoss: integer one-hot targets are not supported; pass class indices or "
                                  "float probabilities")


def _apply(logits, target, metrics, ignore_index, reduction, weight, label_smoothing):
    if reduction not in ("mean", "sum", "none"):
        raise NotImplementedError(f"smaat CrossEntropyLoss: reduction={reduction!r}; 'mean', 'sum' and 'none' are supported")
    _check_target(logits, target)
    weight = _check_options(logits, target, weight, label_smoothing, ignore_index)
    if weight is None and float(label_smoothing) == 0.0 and reduction != "none" and not _is_prob_target(logits, target):
        return _CrossEntropyFn.apply(logits, target, int(ignore_index), reduction, metrics)     # smaat_ce_fwd
    return _CrossEntropyOptsFn.apply(logits, target, weight, float(label_smoothing), int(ignore_index), reduction, metrics)


def cross_entropy(logits, target, ignore_index=-100, reduction="mean", *, weight=None, label_smoothing=0.0):
    """``F.cross_entropy(logits, target, weight=..., ignore_index=..., reduction=..., label_smoothing=...)``; differentiable.
    ``target``: int64 class indices (N, ...) or float probabilities shaped like the logits."""
    return _apply(logits, target, None, ignore_index, reduction, weight, label_smoothing)


def ce_step(logits, target, metrics=None, ignore_index=-100, reduction="mean", *, weight=None, label_smoothing=0.0):
    """``loss_func(logits, target)`` and ``metrics.add(logits, target)`` (train_SmaAtUNet.py:54,73-77) in one pass; the
    gradient for ``loss.backward()`` comes from the same pass.  ``metrics``: an ``IoU``, a ``ConfusionMatrix`` or None.
    Pixels labelled ``ignore_index`` are left out of both the loss and the confusion matrix.  With probability targets the
    confusion row is the target's argmax, and a row that is not one-hot makes the metric's ``value()`` raise."""
    return _apply(logits, target, metrics, ignore_index, reduction, weight, label_smoothing)


class CrossEntropyLoss(nn.Module):
    """``nn.CrossEntropyLoss()`` (train_SmaAtUNet.py:182) for (N, K, ...) float32 CUDA logits: the reference's loss, with
    int64 class-index targets (``smaat_ce_fwd``) or float probability targets shaped like the logits.

    ``reduction`` "mean" (over the pixels not labelled ``ignore_index``; NaN when there are none, as in torch) or "sum".
    A label outside [0, K) that is not ``ignore_index`` makes the loss NaN and that pixel's gradient 0 -- torch raises a
    device-side assert there.  The constructor options beyond the reference's call -- ``weight``, ``label_smoothing`` and
    ``reduction="none"`` -- raise NotImplementedError here: they are ``CrossEntropyLossWithOptions``."""

    def __init__(self, weight=None, size_average=None, ignore_index=-100, reduce=None, reduction="mean", label_smoothing=0.0):
        super().__init__()
        hint = "; use smaat_unet_b200.CrossEntropyLossWithOptions, which takes torch's full constructor"
        if weight is not None:
            raise NotImplementedError("smaat CrossEntropyLoss: class weights are not taken here" + hint)
        if size_average is not None or reduce is not None:
            raise NotImplementedError("smaat CrossEntropyLoss: the deprecated size_average / reduce arguments are not supported")
        if label_smoothing != 0.0:
            raise NotImplementedError("smaat CrossEntropyLoss: label_smoothing is not taken here" + hint)
        if reduction not in ("mean", "sum"):
            raise NotImplementedError(f"smaat CrossEntropyLoss: reduction={reduction!r}; 'mean' and 'sum' are taken here" + hint)
        self.ignore_index = int(ignore_index)
        self.reduction = reduction
        self.label_smoothing = 0.0
        self.weight = None

    def forward(self, input, target):
        return cross_entropy(input, target, self.ignore_index, self.reduction)


class CrossEntropyLossWithOptions(nn.Module):
    """``nn.CrossEntropyLoss`` with torch's full constructor, for (N, K, ...) float32 CUDA logits with int64 class-index
    targets or float probability targets shaped like the logits: ``nn.CrossEntropyLoss(weight=w, label_smoothing=0.1)``
    becomes ``CrossEntropyLossWithOptions(weight=w, label_smoothing=0.1)``.

    ``weight`` (K,) class weights, a registered buffer as in torch (``.to(device)`` moves it); ``label_smoothing`` in
    [0, 1]; ``reduction`` "mean" (class-index targets: divided by the sum of the counted pixels' weights, NaN when it is 0
    or nothing counts, as in torch; probability targets: divided by the pixel count), "sum" or "none" (the per-pixel loss,
    0 on ignored pixels).  A label outside [0, K) that is not ``ignore_index`` makes the loss NaN and that pixel's gradient
    0 -- torch raises a device-side assert there.  Without weights, smoothing, probability targets or "none" the loss is
    ``smaat_ce_fwd``, as ``CrossEntropyLoss``; otherwise ``smaat_cross_entropy_fwd``."""

    def __init__(self, weight=None, size_average=None, ignore_index=-100, reduce=None, reduction="mean", label_smoothing=0.0):
        super().__init__()
        if size_average is not None or reduce is not None:
            raise NotImplementedError("smaat CrossEntropyLossWithOptions: the deprecated size_average / reduce arguments are "
                                      "not supported")
        if reduction not in ("mean", "sum", "none"):
            raise NotImplementedError(f"smaat CrossEntropyLossWithOptions: reduction={reduction!r}; 'mean', 'sum' and 'none' "
                                      "are supported")
        if not 0.0 <= float(label_smoothing) <= 1.0:
            raise RuntimeError(f"label_smoothing must be between 0.0 and 1.0. Got: {float(label_smoothing)}")
        if weight is not None and (not isinstance(weight, torch.Tensor) or weight.dim() != 1):
            raise RuntimeError(f"cross_entropy: weight tensor should be defined either for all classes or no classes but got "
                               f"weight tensor of shape: {list(getattr(weight, 'shape', []))}")
        self.register_buffer("weight", weight)
        self.ignore_index = int(ignore_index)
        self.reduction = reduction
        self.label_smoothing = float(label_smoothing)

    def forward(self, input, target):
        return cross_entropy(input, target, self.ignore_index, self.reduction, weight=self.weight,
                             label_smoothing=self.label_smoothing)


# ------------------------------------------------------------------------------------------------ metrics
def _confusion_of(metrics):
    if metrics is None:
        return None
    return metrics.conf_metric if isinstance(metrics, IoU) else metrics


class ConfusionMatrix:
    """Device-resident K x K confusion matrix with the interface of metric/confusionmatrix.py: rows are targets, columns
    predictions.  ``add`` accepts (N, K, ...) scores (argmax over dim 1, fused kernel) or integer predictions, with class-index
    targets (N, ...) or one-hot targets (N, K, ...) (metric/confusionmatrix.py:57-61: the row's argmax); out-of-range values
    and one-hot rows with a value outside [0, 1] or a sum other than 1 are counted on the device and make ``value()`` raise."""

    def __init__(self, num_classes, normalized=False, device="cuda"):
        if not 2 <= int(num_classes) <= MAX_CLASSES:
            raise NotImplementedError(f"smaat ConfusionMatrix: {num_classes} classes; 2..{MAX_CLASSES} are supported")
        self.num_classes = int(num_classes)
        self.normalized = normalized
        k2 = self.num_classes ** 2
        self._totals = torch.zeros(k2 + 1, device=device, dtype=torch.int64)    # K*K counts, then the invalid-value count
        self._conf = self._totals[:k2].view(self.num_classes, self.num_classes)
        self._invalid = self._totals[k2:]

    def reset(self):
        self._totals.zero_()

    def totals_snapshot(self):
        return self._totals.clone()

    def load_totals(self, snap):
        self._totals.copy_(snap)

    def sync_across_ranks(self):
        """Sum the counts over the ranks of a data-parallel run: one all-reduce of K*K + 1 int64."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self._totals, op=dist.ReduceOp.SUM)

    def _add_invalid(self, n):
        self._invalid.add_(n.to(torch.int64))

    def add(self, predicted, target):
        if not isinstance(predicted, torch.Tensor):
            predicted = torch.as_tensor(np.asarray(predicted))
        tdim = target.dim() if isinstance(target, torch.Tensor) else np.ndim(target)
        if tdim == predicted.dim() + (0 if predicted.is_floating_point() else 1):
            # one-hot (N, K, ...) targets (metric/confusionmatrix.py:57-61): the row's argmax, -1 (invalid) where the row has
            # a value outside [0, 1] or does not sum to 1
            target = onehot_classes(target, self._totals.device, self.num_classes)
            tdim -= 1
        if predicted.is_floating_point():
            if predicted.dim() != tdim + 1:
                raise NotImplementedError(f"smaat ConfusionMatrix: (N, K, ...) scores need (N, ...) class indices or (N, K, ...) "
                                          f"one-hot targets, got {tdim}-D targets for {predicted.dim()}-D scores")
            if predicted.shape[1] != self.num_classes:
                raise AssertionError("number of predictions does not match size of confusion matrix")
            scores = predicted.detach()
            if scores.device != self._totals.device or scores.dtype != torch.float32:
                scores = scores.to(device=self._totals.device, dtype=torch.float32)
            acc, _ = ce_forward(scores, target, 0, False, want_grad=False, conf=self._conf)
            self._add_invalid(acc[2])
        else:
            confusion_add(predicted.reshape(-1), torch.as_tensor(target).reshape(-1), self._conf, self._invalid,
                          self.num_classes)

    def counts(self):
        """(K x K int64 counts, invalid-value count) on the host: ONE device->host copy."""
        t = self._totals.cpu()
        k2 = self.num_classes ** 2
        return t[:k2].view(self.num_classes, self.num_classes).numpy(), int(t[k2])

    def value(self):
        conf, invalid = self.counts()
        if invalid:
            raise AssertionError(f"{invalid} predicted or target values were not between 0 and k-1 (k = {self.num_classes})")
        return confusion_value(conf, self.normalized)


def confusion_value(conf, normalized=False):
    """The reference's ConfusionMatrix.value() on counts: its int32 matrix, or rows scaled to sum to 1 in float32."""
    conf = np.asarray(conf)
    if conf.size and conf.max() > np.iinfo(np.int32).max:
        raise OverflowError("confusion counts exceed the int32 range of the reference's matrix")
    conf = conf.astype(np.int32)
    if not normalized:
        return conf
    c = conf.astype(np.float32)
    return c / c.sum(1).clip(min=1e-12)[:, None]


def iou_value(conf, ignore_index=None):
    """Per-class IoU = TP / (TP + FP + FN) on a (possibly normalised) confusion matrix, and its NaN-ignoring mean; classes
    in ``ignore_index`` have their row and column zeroed first (so their IoU is NaN)."""
    conf = np.array(conf, copy=True)
    if ignore_index is not None:
        conf[:, ignore_index] = 0
        conf[ignore_index, :] = 0
    tp = np.diag(conf)
    fp = np.sum(conf, 0) - tp
    fn = np.sum(conf, 1) - tp
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = tp / (tp + fp + fn)
    return iou, np.nanmean(iou)


class IoU:
    """Per-class intersection over union and its mean, with the interface of metric/iou.py; the confusion matrix lives on
    the device (``conf_metric``).  ``add(predicted, target)``: (N, K, H, W) scores or (N, H, W) integer predictions, (N, H, W)
    integer or (N, K, H, W) one-hot targets on the device or the host.  ``value()`` -> (per-class IoU ndarray, mean IoU)."""

    def __init__(self, num_classes, normalized=False, ignore_index=None, device="cuda"):
        self.conf_metric = ConfusionMatrix(num_classes, normalized, device=device)
        if ignore_index is None:
            self.ignore_index = None
        elif isinstance(ignore_index, int):
            self.ignore_index = (ignore_index,)
        else:
            try:
                self.ignore_index = tuple(ignore_index)
            except TypeError as err:
                raise ValueError("'ignore_index' must be an int or iterable") from err

    @property
    def num_classes(self):
        return self.conf_metric.num_classes

    def reset(self):
        self.conf_metric.reset()

    def totals_snapshot(self):
        return self.conf_metric.totals_snapshot()

    def load_totals(self, snap):
        self.conf_metric.load_totals(snap)

    def sync_across_ranks(self):
        self.conf_metric.sync_across_ranks()

    def add(self, predicted, target):
        if predicted.size(0) != target.size(0):
            raise AssertionError("number of targets and predicted outputs do not match")
        if predicted.dim() not in (3, 4):
            raise AssertionError("predictions must be of dimension (N, H, W) or (N, K, H, W)")
        if target.dim() not in (3, 4):
            raise AssertionError("targets must be of dimension (N, H, W) or (N, K, H, W)")
        if predicted.dim() == 4:
            self.conf_metric.add(predicted, target)
        else:
            if predicted.is_floating_point():
                raise RuntimeError("smaat IoU: (N, H, W) predictions must be integer class indices")
            self.conf_metric.add(predicted, target)

    def value(self):
        return iou_value(self.conf_metric.value(), self.ignore_index)
