"""Multi-class segmentation: cross-entropy loss and IoU bookkeeping on the device, one kernel pass, no host sync.

Host-side mirror of the reference's segmentation workflow (train_SmaAtUNet.py:139-199):
  * ``CrossEntropyLoss``   -- ``nn.CrossEntropyLoss`` (train_SmaAtUNet.py:182) with torch's constructor; class-index
    targets, ``reduction`` "mean" / "sum", any ``ignore_index``
  * ``ConfusionMatrix`` / ``IoU`` -- metric/confusionmatrix.py and metric/iou.py: same constructors, ``add`` / ``value`` /
    ``reset``; the counts stay on the device and ``value()`` makes the one device->host copy
  * ``ce_step(logits, target, metrics)`` -- the loss, its gradient and the IoU update of one training / validation batch
    in ONE pass over the logits: the counterpart of ``metrics.step_loss``
The arithmetic is ``smaat_ce_fwd`` / ``smaat_confusion_add`` (include/smaat_b200.h).

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


def _check_target(logits, target):
    if isinstance(target, torch.Tensor) and target.is_floating_point():
        raise NotImplementedError("smaat CrossEntropyLoss: probability (soft) targets are not supported; pass class indices")
    if isinstance(target, torch.Tensor) and target.dim() == logits.dim():
        raise NotImplementedError("smaat CrossEntropyLoss: one-hot / probability targets are not supported; pass class indices")


def cross_entropy(logits, target, ignore_index=-100, reduction="mean"):
    """``F.cross_entropy(logits, target, ignore_index=..., reduction=...)`` for class-index targets; differentiable."""
    if reduction not in ("mean", "sum"):
        raise NotImplementedError(f"smaat CrossEntropyLoss: reduction={reduction!r}; 'mean' and 'sum' are supported")
    _check_target(logits, target)
    return _CrossEntropyFn.apply(logits, target, int(ignore_index), reduction, None)


def ce_step(logits, target, metrics=None, ignore_index=-100, reduction="mean"):
    """``loss_func(logits, target)`` and ``metrics.add(logits, target)`` (train_SmaAtUNet.py:54,73-77) in one pass; the
    gradient for ``loss.backward()`` comes from the same pass.  ``metrics``: an ``IoU``, a ``ConfusionMatrix`` or None.
    Pixels labelled ``ignore_index`` are left out of both the loss and the confusion matrix."""
    if reduction not in ("mean", "sum"):
        raise NotImplementedError(f"smaat CrossEntropyLoss: reduction={reduction!r}; 'mean' and 'sum' are supported")
    _check_target(logits, target)
    return _CrossEntropyFn.apply(logits, target, int(ignore_index), reduction, metrics)


class CrossEntropyLoss(nn.Module):
    """``nn.CrossEntropyLoss`` (train_SmaAtUNet.py:182) for (N, K, ...) float32 CUDA logits and int64 class-index targets.

    ``reduction`` "mean" (over the pixels not labelled ``ignore_index``; NaN when there are none, as in torch) or "sum".
    A label outside [0, K) that is not ``ignore_index`` makes the loss NaN and that pixel's gradient 0 -- torch raises a
    device-side assert there.  ``weight``, ``label_smoothing`` and probability targets raise NotImplementedError: there is
    no kernel for them and no silent PyTorch fallback."""

    def __init__(self, weight=None, size_average=None, ignore_index=-100, reduce=None, reduction="mean", label_smoothing=0.0):
        super().__init__()
        if weight is not None:
            raise NotImplementedError("smaat CrossEntropyLoss: class weights are not supported")
        if size_average is not None or reduce is not None:
            raise NotImplementedError("smaat CrossEntropyLoss: the deprecated size_average / reduce arguments are not supported")
        if label_smoothing != 0.0:
            raise NotImplementedError("smaat CrossEntropyLoss: label_smoothing is not supported")
        if reduction not in ("mean", "sum"):
            raise NotImplementedError(f"smaat CrossEntropyLoss: reduction={reduction!r}; 'mean' and 'sum' are supported")
        self.ignore_index = int(ignore_index)
        self.reduction = reduction
        self.label_smoothing = 0.0
        self.weight = None

    def forward(self, input, target):
        return cross_entropy(input, target, self.ignore_index, self.reduction)


# ------------------------------------------------------------------------------------------------ metrics
def _confusion_of(metrics):
    if metrics is None:
        return None
    return metrics.conf_metric if isinstance(metrics, IoU) else metrics


class ConfusionMatrix:
    """Device-resident K x K confusion matrix with the interface of metric/confusionmatrix.py: rows are targets, columns
    predictions.  ``add`` accepts (N, K, ...) scores (argmax over dim 1, fused kernel) or integer predictions shaped like
    the target; out-of-range values are counted on the device and make ``value()`` raise."""

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
        if isinstance(target, torch.Tensor) and isinstance(predicted, torch.Tensor) and target.dim() == predicted.dim() \
                and target.is_floating_point():
            raise NotImplementedError("smaat ConfusionMatrix: one-hot targets are not supported; pass class indices")
        if not isinstance(predicted, torch.Tensor):
            predicted = torch.as_tensor(np.asarray(predicted))
        tdim = target.dim() if isinstance(target, torch.Tensor) else np.ndim(target)
        if predicted.is_floating_point():
            if predicted.dim() != tdim + 1:
                raise NotImplementedError("smaat ConfusionMatrix: one-hot targets are not supported; pass class indices")
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
    integer targets on the device or the host.  ``value()`` -> (per-class IoU ndarray, mean IoU)."""

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
        if target.dim() == 4:
            raise NotImplementedError("smaat IoU: one-hot (N, K, H, W) targets are not supported; pass (N, H, W) class indices")
        if target.dim() != 3:
            raise AssertionError("targets must be of dimension (N, H, W) or (N, K, H, W)")
        if predicted.dim() == 4:
            self.conf_metric.add(predicted, target)
        else:
            if predicted.is_floating_point():
                raise RuntimeError("smaat IoU: (N, H, W) predictions must be integer class indices")
            self.conf_metric.add(predicted, target)

    def value(self):
        return iou_value(self.conf_metric.value(), self.ignore_index)
