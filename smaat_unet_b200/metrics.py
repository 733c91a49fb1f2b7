"""Loss and metric bookkeeping of a training / validation step on the device, one kernel pass, no host sync.

Host-side mirror of the reference's interface for this step:
  * ``loss_func(y_pred, y_true)``      -- UNetBase.loss_func, reference models/regression_lightning.py:57-65
  * ``PrecipitationMetrics``           -- reference metric/precipitation_metrics.py:6-147 (same constructor
    arguments, ``update(preds, target)``, ``compute()`` keys, ``reset()``, ``total_*`` state names)
  * ``step_loss(y_pred, y_true, metrics)`` -- what training_step/validation_step do (loss_func + metrics.update,
    regression_lightning.py:67-88) fused into ONE pass that also writes the loss gradient.
  * ``PrecipitationMetricsSweep``        -- PrecipitationMetrics for up to 32 thresholds at once, every sample a batch of
    one (test-set evaluation, ``evaluate.py``; ``smaat_precip_sweep_fwd`` / ``smaat_precip_sweep_commit``).
The arithmetic is ``smaat_mse_metrics_fwd`` / ``smaat_metrics_commit`` (include/smaat_b200.h).  The reference's NaN
guard (`if torch.isnan(...).any()`: a device->host sync every step, precipitation_metrics.py:46) is evaluated on the
device: a batch containing NaN is not added to the totals, and ``skipped_batches`` counts them.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .ops import _call, _dense, _nchw_bstride, _ptr, _stream

FACTOR = 47.83  # precipitation_metrics.py:23


def _match_shapes(preds, target):
    """The reference's shape reconciliation (precipitation_metrics.py:51-58 / regression_lightning.py:59-62)."""
    if preds.shape != target.shape:
        if preds.dim() < target.dim():
            preds = preds.unsqueeze(0)
        elif preds.dim() > target.dim():
            preds = preds.squeeze()
            if preds.dim() < target.dim():
                preds = preds.unsqueeze(0)
    if preds.shape != target.shape:
        raise RuntimeError(f"smaat metrics: preds {tuple(preds.shape)} and target {tuple(target.shape)} do not match")
    return preds


def _check(t, name):
    if t.device.type != "cuda" or t.dtype != torch.float32:
        raise RuntimeError(f"smaat metrics: {name} must be a float32 CUDA tensor (got {t.dtype} on {t.device})")
    return _dense(t, name)


def mse_metrics(preds, target, threshold=0.5, denormalize=True, want_grad=False, grad_scale=1.0, factor=FACTOR):
    """One pass over (preds, target): returns (batch_acc double[8], dpred or None).  See smaat_mse_metrics_fwd."""
    p, t = _check(preds, "preds"), _check(target, "target")
    n = t.numel()
    acc = torch.empty(8, device=t.device, dtype=torch.float64)
    dp = torch.empty_like(p) if want_grad else None
    lib = _lib.load()
    _call("smaat_mse_metrics_fwd", 4 * n * (3 if want_grad else 2), 12 * n, lib.smaat_mse_metrics_fwd, _ptr(p), _ptr(t), n, float(factor),
          float(threshold), int(bool(denormalize)), _ptr(acc), _ptr(dp), float(grad_scale), _stream())
    return acc, dp


class _MseSumFn(torch.autograd.Function):
    """loss = sum((p - y)^2) / B with the gradient produced by the same pass."""

    @staticmethod
    def forward(ctx, y_pred, y_true, metrics):
        B = y_true.size(0)
        need = y_pred.requires_grad
        acc, dp = mse_metrics(y_pred.detach(), y_true.detach(), metrics.threshold if metrics else 0.5,
                              metrics.denormalize if metrics else False, want_grad=need, grad_scale=1.0 / B)
        if metrics is not None:
            metrics._commit(acc, B)
        ctx.save_for_backward(dp)
        return (acc[0] / B).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        (dp,) = ctx.saved_tensors
        return dp * g, None, None


def _loss_shapes(y_pred, y_true):
    if y_pred.dim() > y_true.dim():
        y_pred = y_pred.squeeze(1)
    elif y_true.dim() > y_pred.dim():
        y_pred = y_pred.unsqueeze(1)
    if y_pred.shape != y_true.shape:
        raise RuntimeError(f"smaat loss_func: shapes {tuple(y_pred.shape)} vs {tuple(y_true.shape)}")
    return y_pred


def loss_func(y_pred, y_true):
    """UNetBase.loss_func (regression_lightning.py:57-65): mse_loss(reduction="sum") / batch; differentiable."""
    return _MseSumFn.apply(_loss_shapes(y_pred, y_true), y_true, None)


def step_loss(y_pred, y_true, metrics):
    """loss_func(y_pred, y) and metrics.update(y_pred.detach(), y.detach()) (regression_lightning.py:67-88) in one pass."""
    return _MseSumFn.apply(_loss_shapes(y_pred, y_true), y_true, metrics)


class PrecipitationMetrics:
    """Device-resident accumulator with the reference class's interface (precipitation_metrics.py:6-147)."""

    _NAMES = ("total_loss", "total_loss_denorm", "total_samples", "total_pixels", "total_tn", "total_fp", "total_fn",
              "total_tp", "skipped_batches")

    def __init__(self, threshold=0.5, denormalize=True, dist_sync_on_step=False, device="cuda"):
        self.threshold = threshold
        self.denormalize = denormalize
        self.factor = FACTOR
        self.dist_sync_on_step = dist_sync_on_step
        self._totals = torch.zeros(9, device=device, dtype=torch.float64)

    def to(self, device):
        self._totals = self._totals.to(device)
        return self

    def reset(self):
        self._totals.zero_()

    def totals_snapshot(self):
        return self._totals.clone()

    def load_totals(self, snap):
        self._totals.copy_(snap)

    def __getattr__(self, name):
        names = type(self)._NAMES
        if name in names and "_totals" in self.__dict__:
            v = self.__dict__["_totals"][names.index(name)]
            return v if name.startswith("total_loss") else v.to(torch.int64)
        raise AttributeError(name)

    def _commit(self, acc, batch_size):
        lib = _lib.load()
        _call("smaat_metrics_commit", 0, 0, lib.smaat_metrics_commit, _ptr(acc), _ptr(self._totals), int(batch_size),
              int(bool(self.denormalize)), _stream())

    def update(self, preds, target):
        preds = _match_shapes(preds.detach(), target)
        acc, _ = mse_metrics(preds, target.detach(), self.threshold, self.denormalize, factor=self.factor)
        self._commit(acc, target.size(0))

    def sync_across_ranks(self):
        """dist_reduce_fx="sum" of every state (precipitation_metrics.py:26-34): one all-reduce of 9 doubles."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self._totals, op=dist.ReduceOp.SUM)

    def compute(self):
        """precipitation_metrics.py:97-147; one device->host copy of the 9 totals."""
        t = self._totals.cpu()
        return compute_from_totals(t, self.denormalize)

    def __call__(self, preds, target):
        self.update(preds, target)


MAX_SWEEP_THRESHOLDS = 32


class PrecipitationMetricsSweep:
    """``PrecipitationMetrics`` for several thresholds at once, counting every sample as its own batch of one.

    Each ``update`` is one pass over the batch (``smaat_precip_sweep_fwd``): per image, the two squared-error sums, a NaN
    count and a joint (target bin, prediction bin) histogram over the thresholds, from which every threshold's confusion
    matrix follows exactly.  ``smaat_precip_sweep_commit`` then adds the images one by one to totals that stay on the
    device (no host synchronisation per batch).

    Why a batch of one: the reference's ``PrecipitationMetrics.update`` adds ``mse_loss(sum) / batch_size`` to
    ``total_loss`` and ``batch_size`` to ``total_samples`` (metric/precipitation_metrics.py:62-64), and ``compute()``
    divides by ``total_samples`` again (:105), so ``mse``, ``mse_denorm`` and ``mse_pixel`` come out B times smaller when
    it is fed batches of B.  Its NaN guard drops the whole update (:46-48), good samples included.  The published figures
    use batch size 1 (calc_metrics_test_set.py:95).  Here a batch of B gives exactly what B batch-1 updates of
    ``PrecipitationMetrics(threshold=t)`` give, for every threshold t: each image adds its sums, 1 sample, its pixels and
    its counts, and an image containing NaN adds nothing and is counted in ``skipped_images``.

    ``thresholds``: 1 to 32 strictly increasing values in mm/h, compared in fp32 as the reference does.  ``compute()``
    returns ``{threshold: dict}`` with the reference's ten keys (``compute_from_totals``)."""

    def __init__(self, thresholds, denormalize=True, device="cuda"):
        th = tuple(float(t) for t in thresholds)
        th32 = [float(torch.tensor(t, dtype=torch.float32)) for t in th]
        if not 1 <= len(th) <= MAX_SWEEP_THRESHOLDS or any(not a < b for a, b in zip(th32, th32[1:])) or any(t != t for t in th):
            raise ValueError(f"PrecipitationMetricsSweep: thresholds must be 1..{MAX_SWEEP_THRESHOLDS} strictly increasing "
                             f"values (in float32), got {th}")
        self.thresholds = th
        self.denormalize = denormalize
        self.factor = FACTOR
        self._thr = (C.c_float * len(th))(*th32)
        cells = (len(th) + 1) ** 2
        self._totals = torch.zeros(5 + cells, device=device, dtype=torch.float64)

    def to(self, device):
        self._totals = self._totals.to(device)
        return self

    def reset(self):
        self._totals.zero_()

    def totals_snapshot(self):
        return self._totals.clone()

    def load_totals(self, snap):
        self._totals.copy_(snap)

    @property
    def total_samples(self):
        return self._totals[2].to(torch.int64)

    @property
    def total_pixels(self):
        return self._totals[3].to(torch.int64)

    @property
    def skipped_images(self):
        return self._totals[4].to(torch.int64)

    def _sweep(self, pred, pred_bstride, target, B, P):
        T = len(self.thresholds)
        per_image = torch.empty((B, 3), device=target.device, dtype=torch.float64)
        hist = torch.empty((B, T + 1, T + 1), device=target.device, dtype=torch.int32)
        lib = _lib.load()
        _call("smaat_precip_sweep_fwd", 8 * B * P, 0, lib.smaat_precip_sweep_fwd, pred, int(pred_bstride), _ptr(target), B, P,
              float(self.factor), self._thr, T, int(bool(self.denormalize)), _ptr(per_image), _ptr(hist), _stream())
        _call("smaat_precip_sweep_commit", 0, 0, lib.smaat_precip_sweep_commit, _ptr(per_image), _ptr(hist), B, P, T,
              int(bool(self.denormalize)), _ptr(self._totals), _stream())

    def update(self, preds, target):
        """Add a batch of model outputs (B, 1, H, W) (or any shape the reference's update reconciles with target) against
        target (B, H, W), every image as a batch of one."""
        target = _check(target.detach(), "target")
        preds = _check(_match_shapes(preds.detach(), target), "preds")
        B = target.size(0)
        P = target.numel() // B
        self._sweep(_ptr(preds), P, target, B, P)

    def update_persistence(self, x, target):
        """The persistence baseline's update (regression_lightning.py:202-204: the prediction is the input's last frame
        ``x[:, -1:]``), read in place from x (B, C, H, W) with batch stride C * H * W: no copy of the frame."""
        target = _check(target.detach(), "target")
        x, bstride = _nchw_bstride(x.detach(), "x")
        B, Cc, H, W = x.shape
        if target.shape != (B, H, W):
            raise RuntimeError(f"smaat metrics: persistence input {tuple(x.shape)} and target {tuple(target.shape)} do not match")
        self._sweep(x.data_ptr() + (Cc - 1) * H * W * x.element_size(), bstride, target, B, H * W)

    def sync_across_ranks(self):
        """dist_reduce_fx="sum" of every state: one all-reduce of the totals."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self._totals, op=dist.ReduceOp.SUM)

    def threshold_totals(self):
        """``{threshold: totals}`` in ``PrecipitationMetrics``' layout (float64 CPU: total_loss, total_loss_denorm,
        total_samples, total_pixels, TN, FP, FN, TP, skipped images); one device->host copy."""
        t = self._totals.cpu()
        T1 = len(self.thresholds) + 1
        h = t[5:].to(torch.int64).view(T1, T1)          # [target bin][pred bin], exact integers
        out = {}
        for i, thr in enumerate(self.thresholds, start=1):
            tp = int(h[i:, i:].sum())
            fn = int(h[i:, :i].sum())
            fp = int(h[:i, i:].sum())
            tn = int(h[:i, :i].sum())
            out[thr] = torch.tensor([float(t[0]), float(t[1]), float(t[2]), float(t[3]), tn, fp, fn, tp, float(t[4])],
                                    dtype=torch.float64)
        return out

    def compute(self):
        """``{threshold: dict}``: for each threshold the reference's ``compute()`` dict (precipitation_metrics.py:97-147)."""
        return {thr: compute_from_totals(v, self.denormalize) for thr, v in self.threshold_totals().items()}


def compute_from_totals(t, denormalize=True):
    nan = torch.tensor(float("nan"))
    loss, loss_d, n, px, tn, fp, fn, tp = (t[i] for i in range(8))
    f = lambda v: v.to(torch.float32)
    mse = f(loss / n)
    mse_denorm = f(loss_d / n) if denormalize else nan
    mse_pixel = f(loss_d / px) if denormalize else nan
    precision = f(tp / (tp + fp)) if (tp + fp) > 0 else nan
    recall = f(tp / (tp + fn)) if (tp + fn) > 0 else nan
    accuracy = f((tp + tn) / (tp + tn + fp + fn))
    f1 = 2 * precision * recall / (precision + recall) if (precision + recall) > 0 else nan
    csi = f(tp / (tp + fn + fp)) if (tp + fn + fp) > 0 else nan
    far = f(fp / (tp + fp)) if (tp + fp) > 0 else nan
    denom = (tp + fn) * (fn + tn) + (tp + fp) * (fp + tn)
    hss = f((tp * tn - fn * fp) / denom) if denom > 0 else nan
    return {"mse": mse, "mse_denorm": mse_denorm, "mse_pixel": mse_pixel, "precision": precision, "recall": recall,
            "accuracy": accuracy, "f1": f1, "csi": csi, "far": far, "hss": hss}
