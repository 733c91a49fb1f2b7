"""Train the reference's models from start to finish on the GPU path, without Lightning: its two training recipes on
``TrainSession``, with validation, the plateau learning-rate schedule, early stopping and checkpoints.

  * ``fit_precipitation(model, train_shard, out_dir, ...)`` -- ``train_precip_lightning.py`` with
    ``models/regression_lightning.py``: one of the four precipitation networks (or UNetDSAttention4CBAMs), Adam,
    ``ReduceLROnPlateau(mode="min")`` on ``val_loss``, Lightning's ``EarlyStopping`` and ``ModelCheckpoint`` files, which
    ``evaluate.load_reference_checkpoint`` (and so ``python -m smaat_unet_b200.evaluate``) reads.
  * ``fit_voc(train_prefix, val_prefix, out_dir, ...)`` -- ``fit()`` of ``train_SmaAtUNet.py``: ``SmaAt_UNet(3, 21)`` on the
    VOC shards of ``data.convert_voc``, validated on the IoU's mean, with its early stopping and its ``.pt`` files.
  * ``python -m smaat_unet_b200.fit {precip,voc} ...`` -- the command line of both.

Both recipes share one epoch loop (``_EpochLoop``).  Every batch is one ``TrainSession.step`` (a captured graph; the
epoch's partial last batch has a graph of its own size) or one serving forward plus one loss / metric kernel pass.  The
per-batch losses are copied into a device buffer, the metric totals stay on the device, and each epoch reads them back
once, after its last batch: nothing in the batch loops waits for the GPU (``sync_debug=True`` makes any such wait raise).

Validation runs on the weights and BatchNorm running statistics of the epoch's last step.  ``TrainSession`` writes them by
graph replay, which bumps no tensor's ``_version``, so the validation forward is either the uncaptured serving forward
(``validation="serving"``, the default: the weight caches follow ``ops.bump_weights_generation``, which every step
bumps) or an ``InferenceSession`` re-captured before each validation pass (``validation="captured"``).  The default is
the faster of the two as measured by ``tools/bench_fit.py`` (README "Training from start to finish").  Either way the
model is put back in train mode before the next step.

Data parallelism.  When a process group is initialised (``torchrun --nproc-per-node N python -m smaat_unet_b200.fit ...``
sets one up through ``parallel.process_group_from_env``), both recipes run data-parallel, as Lightning's DDP does:
  * ``batch_size`` is per rank; the global batch is ``N x batch_size``, the learning rate is not scaled;
  * every rank draws the same split and the same per-epoch shuffle, then takes its wrap-padded shard of the train indices
    (``shard_indices``), so every rank steps the same batch sizes; padded samples are seen twice per epoch, as with torch's
    ``DistributedSampler``.  Validation indices are split into disjoint slices (``disjoint=True``): each sample counts once;
  * at the epoch's end rank 0's BatchNorm running statistics replace the others' (DDP's buffer broadcast), then the loss
    sums and counts and the metric totals are summed over the ranks, and rank 0's early-stopping, plateau and stop
    decisions are broadcast, so every rank takes the same ones;
  * rank 0 alone writes checkpoints, ``history.jsonl`` and the printed lines; the others wait at a barrier after each write.
    Checkpoints of a multi-process run hold ``world_size``, and a resume at another world size is refused.
Without a process group nothing of this runs.

Deliberate differences from the reference:
  * the train / validation split is drawn from ``np.random.RandomState(seed)`` (the same draw as the reference's
    ``np.random.shuffle`` after ``np.random.seed(seed)``) and the seed is stored in the checkpoint, so a resumed run keeps
    its split; the reference draws a new split on every start;
  * the per-epoch batch order comes from ``PinnedBatchLoader``'s seeded shuffle (``seed + epoch``), so it is reproducible;
  * checkpoints are written after the epoch's early-stopping and plateau decisions, so a resumed run continues with the
    state the uninterrupted run has (Lightning writes them before the scheduler's step).
"""
from __future__ import annotations

import argparse
import contextlib
import json
import math
import os
import shutil
import time

import numpy as np
import torch

from . import ops, parallel
from .data import PinnedBatchLoader, precipitation_maps_oversampled_shard, precipitation_maps_shard, voc_segmentation_shard
from .engine import InferenceSession
from .evaluate import _CTOR_ARGS
from .metrics import PrecipitationMetrics, mse_metrics
from .model import SmaAt_UNet, UNet, UNetAttention, UNetDS, UNetDSAttention4CBAMs
from .segmentation import IoU, ce_forward
from .train import TrainSession

# the reference's Lightning class name (unet_precip_regression_lightning.py) -> native class; the name is what the checkpoint
# files are called by, so evaluate.checkpoint_class resolves them
PRECIP_MODELS = {"UNet": UNet, "UNetDS": UNetDS, "UNetAttention": UNetAttention, "UNetDSAttention": SmaAt_UNet,
                 "UNetDSAttention4CBAMs": UNetDSAttention4CBAMs}
LIGHTNING_VERSION = "2.5.0.post0"        # the version the reference pins (uv.lock); written as Lightning writes its own
VALIDATION_MODES = ("serving", "captured")
HISTORY_FILE = "history.jsonl"

# hyper-parameters that fix the network or the split: a resumed run must agree with its checkpoint on these
_RESUME_KEYS = ("model", "n_channels", "n_classes", "kernels_per_layer", "bilinear", "reduction_ratio", "num_input_images",
                "num_output_images", "valid_size", "use_oversampled_dataset", "seed", "batch_size")


# ------------------------------------------------------------------------------------------------ recipe pieces
def train_valid_split(num_samples, valid_size, seed):
    """``prepare_data``'s split (regression_lightning.py:163-170): ``split = floor(valid_size * N)``, ``range(N)`` shuffled,
    validation the first ``split`` indices.  ``RandomState(seed).shuffle`` is the draw ``np.random.shuffle`` makes after
    ``np.random.seed(seed)``.  Returns (train indices, validation indices)."""
    indices = list(range(int(num_samples)))
    split = int(np.floor(valid_size * num_samples))
    np.random.RandomState(seed).shuffle(indices)
    return indices[split:], indices[:split]


class EarlyStopping:
    """The stopping rule of both recipes, fed one monitored value per epoch; ``update`` returns True when training stops.

    ``mode="min"`` with ``check_finite=True`` is Lightning's ``EarlyStopping(monitor="val_loss", mode="min", patience=p)``
    with its defaults (``min_delta=0``): an improvement is a value strictly below the best, a non-finite value stops at
    once, and ``patience`` epochs in a row without improvement stop.  ``mode="max"``, ``best=-1.0``,
    ``check_finite=False`` is train_SmaAtUNet.py:94-115: ``mean_iou > best_mIoU`` resets the counter, anything else (a NaN
    included) counts, and ``counter >= earlystopping`` stops."""

    def __init__(self, patience, mode="min", check_finite=True, best=None):
        if mode not in ("min", "max"):
            raise ValueError(f"EarlyStopping: mode must be 'min' or 'max', got {mode!r}")
        self.patience, self.mode, self.check_finite = int(patience), mode, bool(check_finite)
        self.best = float(best) if best is not None else (math.inf if mode == "min" else -math.inf)
        self.wait_count = 0
        self.stopped_epoch = 0
        self.improved = False

    def update(self, value, epoch=0):
        value = float(value)
        self.improved = False
        if self.check_finite and not math.isfinite(value):
            stop = True
        elif (value < self.best) if self.mode == "min" else (value > self.best):
            self.best, self.wait_count, self.improved = value, 0, True
            stop = False
        else:
            self.wait_count += 1
            stop = self.wait_count >= self.patience
        if stop:
            self.stopped_epoch = int(epoch)
        return stop

    def state_dict(self):
        return {"wait_count": self.wait_count, "stopped_epoch": self.stopped_epoch, "best_score": self.best,
                "patience": self.patience}

    def load_state_dict(self, sd):
        self.wait_count, self.stopped_epoch = int(sd["wait_count"]), int(sd["stopped_epoch"])
        self.best = float(sd["best_score"])


class PlateauLR:
    """``torch.optim.lr_scheduler.ReduceLROnPlateau`` itself, on a one-parameter stand-in optimizer whose rate the caller
    copies to ``TrainSession.set_lr``: the session's Adam reads its rate from a device scalar, not a param group."""

    def __init__(self, lr, mode, factor=0.1, patience=4):
        self._opt = torch.optim.SGD([torch.zeros(1, requires_grad=True)], lr=float(lr))
        self.scheduler = torch.optim.lr_scheduler.ReduceLROnPlateau(self._opt, mode=mode, factor=factor, patience=patience)

    @property
    def lr(self):
        return float(self._opt.param_groups[0]["lr"])

    def step(self, value):
        """One epoch's step; returns the rate for the next epoch."""
        self.scheduler.step(float(value))
        return self.lr

    def state_dict(self):
        return self.scheduler.state_dict()

    def load_state_dict(self, sd, lr):
        self.scheduler.load_state_dict(sd)
        self._opt.param_groups[0]["lr"] = float(lr)


def make_metrics_str(metrics):
    """utils/formatting.py's ``make_metrics_str``: ``name: value`` to four decimals, NaN values left out, ``" | "``-joined."""
    parts = []
    for name, v in metrics.items():
        v = v.item() if isinstance(v, torch.Tensor) else v
        if not (isinstance(v, float) and math.isnan(v)):
            parts.append(f"{name}: {v:.4f}")
    return " | ".join(parts)


def _plain_metrics(metrics):
    return {k: float(v.item() if isinstance(v, torch.Tensor) else v) for k, v in metrics.items()}


def _cpu_state_dict(model):
    """The model's state_dict as self-contained CPU tensors (the parameters themselves are views of the flat buffer)."""
    return {k: v.detach().to("cpu", copy=True) for k, v in model.state_dict().items()}


def _cpu_optimizer_state(sd):
    out = {"state": {}, "param_groups": sd["param_groups"]}
    for i, st in sd["state"].items():
        out["state"][i] = {k: (v.detach().to("cpu", copy=True) if isinstance(v, torch.Tensor) else v) for k, v in st.items()}
    return out


# ------------------------------------------------------------------------------------------------ precipitation checkpoints
def precip_file_names(class_name, epoch, val_loss):
    """(best, last) file names of the two ModelCheckpoint callbacks (train_precip_lightning.py:27-41): Lightning expands
    ``{epoch}`` to ``epoch=<e>`` and ``{val_loss:.6f}`` to ``val_loss=<v>``."""
    stem = f"{class_name}_rain_threshold_50_epoch={int(epoch)}-val_loss={float(val_loss):.6f}"
    return stem + ".ckpt", stem + "_last.ckpt"


def precip_checkpoint(state_dict, hyper_parameters, epoch, global_step, optimizer_state, scheduler_state, early_stopping,
                      best_model_score, best_model_path, split, world_size=1):
    """A Lightning-layout checkpoint dict of plain types and CPU tensors only (``evaluate``'s restricted unpickler refuses any
    other class).  A data-parallel run's (``world_size`` > 1) also holds ``world_size``; a single process's has no such
    key."""
    ckpt = {
        "epoch": int(epoch),
        "global_step": int(global_step),
        "pytorch-lightning_version": LIGHTNING_VERSION,
        "state_dict": state_dict,
        "callbacks": {
            "EarlyStopping{'monitor': 'val_loss', 'mode': 'min'}": dict(early_stopping),
            "ModelCheckpoint{'monitor': 'val_loss', 'mode': 'min'}": {
                "monitor": "val_loss", "best_model_score": best_model_score, "best_model_path": best_model_path},
        },
        "optimizer_states": [optimizer_state],
        "lr_schedulers": [scheduler_state],
        "hparams_name": "hparams",
        "hyper_parameters": dict(hyper_parameters),
        "split": dict(split),
    }
    if world_size > 1:
        ckpt["world_size"] = int(world_size)
    return ckpt


def precip_hyper_parameters(model="UNetDSAttention", train_shard=None, batch_size=16, learning_rate=1e-3, epochs=200,
                            lr_patience=4, es_patience=15, valid_size=0.1, use_oversampled_dataset=True, kernels_per_layer=2,
                            bilinear=True, reduction_ratio=16, threshold=0.5, num_input_images=12, num_output_images=6,
                            n_classes=1, seed=0, resume_from_checkpoint=None):
    """Every argument of a precipitation run, with the reference's argparse defaults and the values its ``__main__`` sets
    (train_precip_lightning.py:82-117; regression_lightning.py:14-29, :118-127).  ``n_channels`` is the input frame count."""
    if model == "PersistenceModel":
        raise ValueError("fit_precipitation: PersistenceModel has no parameters to train; it is scored by "
                         "python -m smaat_unet_b200.evaluate as it is")
    if model not in PRECIP_MODELS:
        raise ValueError(f"fit_precipitation: unknown model {model!r}; one of {', '.join(PRECIP_MODELS)}")
    return {"model": model, "n_channels": int(num_input_images), "n_classes": int(n_classes),
            "kernels_per_layer": int(kernels_per_layer), "bilinear": bool(bilinear), "reduction_ratio": int(reduction_ratio),
            "lr_patience": int(lr_patience), "threshold": float(threshold), "num_input_images": int(num_input_images),
            "num_output_images": int(num_output_images), "valid_size": float(valid_size),
            "use_oversampled_dataset": bool(use_oversampled_dataset),
            "dataset_folder": None if train_shard is None or not isinstance(train_shard, (str, os.PathLike)) else os.fspath(train_shard),
            "batch_size": int(batch_size), "learning_rate": float(learning_rate), "epochs": int(epochs),
            "es_patience": int(es_patience), "seed": int(seed),
            "resume_from_checkpoint": None if resume_from_checkpoint is None else os.fspath(resume_from_checkpoint)}


def build_precip_model(hp):
    """The native network of a run's hyper-parameters, with the constructor arguments its reference class reads."""
    cls = PRECIP_MODELS[hp["model"]]
    return cls(**{k: hp[k] for k in _CTOR_ARGS[cls]})


def check_resume(ckpt, hp, num_samples, world=1):
    """Refuse a checkpoint of another network, split, batch size or world size than this run's (``ValueError``).  A
    checkpoint without ``world_size`` was written by a single process."""
    old = ckpt.get("hyper_parameters") or {}
    bad = [f"{k}: checkpoint {old.get(k)!r}, run {hp[k]!r}" for k in _RESUME_KEYS if old.get(k) != hp[k]]
    samples = (ckpt.get("split") or {}).get("samples")
    if samples != num_samples:
        bad.append(f"samples in the train shard: checkpoint {samples!r}, run {num_samples}")
    ckpt_world = int(ckpt.get("world_size", 1))
    if ckpt_world != int(world):
        bad.append(f"world size: checkpoint {ckpt_world}, run {int(world)} (each rank's batches would differ from the "
                   "interrupted run's)")
    if bad:
        raise ValueError("fit_precipitation: the checkpoint to resume from does not match this run: " + "; ".join(bad))


def _replace_file(directory, old_name, new_name, payload):
    """Write ``payload`` (a checkpoint dict, or the path of a file already holding it) as ``new_name`` and remove
    ``old_name``."""
    path = os.path.join(directory, new_name)
    tmp = path + ".tmp"
    if isinstance(payload, str):
        shutil.copyfile(payload, tmp)
    else:
        torch.save(payload, tmp)
    os.replace(tmp, path)
    if old_name and old_name != new_name and os.path.exists(os.path.join(directory, old_name)):
        os.remove(os.path.join(directory, old_name))
    return path


# ------------------------------------------------------------------------------------------------ the shared epoch loop
@contextlib.contextmanager
def _sync_check(enabled):
    """With ``enabled``, any operation that makes the host wait for the GPU raises inside the block
    (``torch.cuda.set_sync_debug_mode("error")``)."""
    if not enabled:
        yield
        return
    old = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(old)


class _EpochLoop:
    """One epoch of either recipe: every train batch through ``sess.step``, then every validation batch through the serving
    forward and ``val_batch(pred, y, row)``, which writes its per-batch sums into a row of the epoch's device buffer.

    ``sess``: the TrainSession.  ``val_input(x, y)`` turns a pinned host batch into device (x, y); ``val_batch(pred, y, row)``
    launches the loss / metric pass.  Returns the buffer's rows on the host (one device->host read): rows 0..nt-1 hold the
    step losses in column 0, the others what ``val_batch`` wrote."""

    def __init__(self, sess, train_loader, val_loader, val_input, val_batch, validation="serving", sync_debug=False):
        if validation not in VALIDATION_MODES:
            raise ValueError(f"fit: validation must be one of {VALIDATION_MODES}, got {validation!r}")
        self.sess, self.train_loader, self.val_loader = sess, train_loader, val_loader
        self.val_input, self.val_batch = val_input, val_batch
        self.validation, self.sync_debug = validation, bool(sync_debug)
        self.device = sess.device
        self.model = sess.model
        self._vsess = None
        self.train_sizes = self._sizes(train_loader)
        self.val_sizes = self._sizes(val_loader)

    @staticmethod
    def _sizes(loader):
        n, b = len(loader.epoch_indices()), loader.batch_size
        return [b] * (n // b) + ([n % b] if n % b else [])

    def _forward(self):
        """The validation forward on the current weights (see the module docstring)."""
        if self.validation == "serving":
            model = self.model
            model.eval()
            return model.forward_serving
        vb = self.val_loader.batch_size
        tail = self.val_sizes[-1] if self.val_sizes and self.val_sizes[-1] != vb else None
        if self._vsess is None:
            self._vsess = InferenceSession(self.model, vb, self.sess.in_shape, device=self.device,
                                           batch_sizes=(tail,) if tail else None)
        else:
            self._vsess.refresh()
        return self._vsess.forward

    def run(self, epoch):
        nt, nv = len(self.train_sizes), len(self.val_sizes)
        buf = torch.zeros((nt + nv, 3), device=self.device, dtype=torch.float64)
        self.train_loader.set_epoch(epoch)
        self.val_loader.set_epoch(epoch)
        with torch.cuda.device(self.device):
            with _sync_check(self.sync_debug):
                for i, batch in enumerate(self.train_loader):
                    loss = self.sess.step(*batch[:2], aug=batch[2] if len(batch) > 2 else None)
                    buf[i, 0].copy_(loss)
                    self.train_loader.guard(self.sess.last_h2d_event())
            if self.sess.world > 1:
                # each replica's BatchNorm running statistics followed its own batches: validation and the checkpoint take
                # rank 0's, which is what DDP's buffer broadcast leaves in every replica
                parallel.broadcast_tensors_(list(self.model.buffers()), self.device)
                ops.bump_weights_generation()
            fwd = self._forward()
            try:
                with torch.no_grad(), _sync_check(self.sync_debug):
                    for j, (x, y) in enumerate(self.val_loader):
                        xd, yd = self.val_input(x.to(self.device, non_blocking=True), y.to(self.device, non_blocking=True))
                        copied = torch.cuda.Event()
                        copied.record()
                        self.val_loader.guard(copied)
                        self.val_batch(fwd(xd), yd, buf[nt + j])
            finally:
                self.model.train()              # TrainSession's eager steps (undeclared sizes) read the flag
                # the session's boundary hook saw the validation forward's CBAM outputs; they are no step's and must not
                # stay referenced until its next eager step
                self.sess._bnd.clear()
        rows = buf.cpu().numpy()
        return rows[:nt], rows[nt:]


def _weighted_sums(values, weights):
    """[sum of values x weights, sum of weights] in float64: one rank's part of an epoch's weighted mean, which
    ``parallel.allreduce_sum`` completes over the ranks."""
    v, w = np.asarray(values, np.float64), np.asarray(weights, np.float64)
    return [(v * w).sum(), w.sum()]


def _agree(stop, value, stopper, plateau, device=None):
    """Rank 0's epoch decisions on every rank, in one broadcast: its stop decision and monitored value, and its
    early-stopping and plateau state (and so the next learning rate).  The ranks' values come from the same reductions,
    but the decisions are made identical by construction, not by floating-point luck: a rank that stopped alone would
    leave the others waiting in a collective.  Returns (stop, value); without a process group, the arguments."""
    if parallel.rank_world()[1] == 1:
        return stop, value
    d = parallel.broadcast_from_rank0({"stop": bool(stop), "value": value, "early_stopping": stopper.state_dict(),
                                       "improved": stopper.improved, "plateau": plateau.state_dict(), "lr": plateau.lr},
                                      device)
    stopper.load_state_dict(d["early_stopping"])
    stopper.improved = d["improved"]
    plateau.load_state_dict(d["plateau"], d["lr"])
    return d["stop"], d["value"]


@contextlib.contextmanager
def _rank0_writes(device=None):
    """A block whose files only rank 0 writes: it yields whether this rank is the writer, and at its end every rank waits
    at a barrier, so that no rank reads (e.g. resumes from) a file rank 0 is still writing."""
    rank, world = parallel.rank_world()
    yield rank == 0
    if world > 1:
        parallel.barrier(device)


def _append_history(out_dir, record):
    with open(os.path.join(out_dir, HISTORY_FILE), "a") as f:
        f.write(json.dumps(record) + "\n")


# ------------------------------------------------------------------------------------------------ precipitation
class FitResult:
    """What a run leaves behind: ``history`` (the per-epoch records also written to ``history.jsonl``), ``model``,
    ``session`` (the TrainSession), the ``split`` (train, validation indices), the data loaders, and the paths of the
    last written checkpoint files (``best_path``, ``last_path``)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def fit_precipitation(model="UNetDSAttention", train_shard=None, out_dir="lightning/precip_regression", batch_size=16,
                      learning_rate=1e-3, epochs=200, lr_patience=4, es_patience=15, valid_size=0.1,
                      use_oversampled_dataset=True, kernels_per_layer=2, bilinear=True, reduction_ratio=16, threshold=0.5,
                      num_input_images=12, num_output_images=6, seed=0, resume_from_checkpoint=None, validation="serving",
                      sync_debug=False, device=None, verbose=True):
    """``train_precip_lightning.train_regression`` for one model (train_precip_lightning.py:13-77 with
    regression_lightning.py:44-199): per epoch, in Lightning's order,

      1. the train batches, each one ``TrainSession.step`` (Adam at ``learning_rate``; ``loss_func`` and the training
         ``PrecipitationMetrics(threshold)`` in the step);
      2. validation on the last step's weights and running statistics: ``val_loss`` and the validation metrics from the
         serving forward and ``metrics.mse_metrics``;
      3. ``EarlyStopping(patience=es_patience)`` on ``val_loss`` (Lightning's defaults);
      4. ``ReduceLROnPlateau(mode="min", factor=0.1, patience=lr_patience)`` on ``val_loss``; the new rate applies from the
         next epoch;
      5. the best (lowest ``val_loss``) and last checkpoints under ``out_dir/<model>/``, one file of each.

    ``train_loss`` / ``val_loss`` are Lightning's epoch values: the batch-size-weighted mean of the per-batch
    ``loss_func``.  ``train_shard``: the ``<prefix>_train.npy`` of ``data.convert_h5`` (or an array of that layout).
    ``resume_from_checkpoint``: a last (or best) checkpoint of this recipe; the run continues with the next epoch."""
    hp = precip_hyper_parameters(model, train_shard, batch_size, learning_rate, epochs, lr_patience, es_patience, valid_size,
                                 use_oversampled_dataset, kernels_per_layer, bilinear, reduction_ratio, threshold,
                                 num_input_images, num_output_images, seed=seed, resume_from_checkpoint=resume_from_checkpoint)
    if train_shard is None:
        raise ValueError("fit_precipitation: train_shard is required (data.convert_h5 writes <prefix>_train.npy)")
    if isinstance(train_shard, (str, os.PathLike)) and not os.path.isfile(train_shard):
        raise FileNotFoundError(f"fit_precipitation: no train shard at {os.fspath(train_shard)!r}")
    ds_cls = precipitation_maps_oversampled_shard if use_oversampled_dataset else precipitation_maps_shard
    dataset = ds_cls(train_shard, num_input_images, num_output_images, train=True)
    n = len(dataset)
    rank, world = parallel.rank_world()
    ckpt = None
    if resume_from_checkpoint is not None:           # every rank loads it; the session's broadcast keeps them identical
        from .evaluate import _RestrictedPickle
        ckpt = torch.load(resume_from_checkpoint, map_location="cpu", pickle_module=_RestrictedPickle, weights_only=False)
        check_resume(ckpt, hp, n, world)
    train_idx, valid_idx = train_valid_split(n, valid_size, seed)
    if not train_idx or not valid_idx:
        raise ValueError(f"fit_precipitation: {n} samples with valid_size={valid_size} leave an empty train or validation split")
    device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    in_shape, _ = dataset.sample_shapes()

    torch.manual_seed(seed)
    net = build_precip_model(hp)
    if ckpt is not None:
        net.load_state_dict(ckpt["state_dict"], strict=True)
    # data-parallel: the same split and per-epoch shuffle on every rank; train shards wrap-padded to equal length (every
    # rank steps the same sizes), validation slices disjoint (every sample counted once)
    train_loader = PinnedBatchLoader(dataset, batch_size, indices=train_idx, shuffle=True, seed=seed, drop_last=False,
                                     rank=rank, world=world)
    val_loader = PinnedBatchLoader(dataset, batch_size, indices=valid_idx, shuffle=True, seed=seed, drop_last=False,
                                   rank=rank, world=world, disjoint=True)
    tail = len(train_loader.epoch_indices()) % batch_size
    sess = TrainSession(net, batch_size, in_shape, lr=learning_rate, device=device, batch_sizes=(tail,) if tail else None,
                        metrics=PrecipitationMetrics(threshold=threshold, device=device))
    sess.check_partial_rows = False                  # equal step sizes on every rank by construction (shard_indices)
    val_metrics = PrecipitationMetrics(threshold=threshold, device=device)

    plateau = PlateauLR(learning_rate, "min", factor=0.1, patience=lr_patience)
    stopper = EarlyStopping(es_patience, mode="min", check_finite=True)
    start, global_step, best_score, best_name, last_name = 0, 0, None, None, None
    ckpt_dir = os.path.join(os.fspath(out_dir), hp["model"])
    if ckpt is not None:
        lr = ckpt["optimizer_states"][0]["param_groups"][0]["lr"]
        sess.load_optimizer_state_dict(ckpt["optimizer_states"][0])
        plateau.load_state_dict(ckpt["lr_schedulers"][0], lr)
        cbs = ckpt["callbacks"]
        stopper.load_state_dict(cbs["EarlyStopping{'monitor': 'val_loss', 'mode': 'min'}"])
        mc = cbs["ModelCheckpoint{'monitor': 'val_loss', 'mode': 'min'}"]
        best_score = mc["best_model_score"]
        best_name = os.path.basename(mc["best_model_path"]) if mc["best_model_path"] else None
        start, global_step = int(ckpt["epoch"]) + 1, int(ckpt["global_step"])
        last_name = os.path.basename(os.fspath(resume_from_checkpoint))
        if not last_name.endswith("_last.ckpt"):
            last_name = None
        del ckpt
    with _rank0_writes(device) as writer:
        if writer:
            os.makedirs(ckpt_dir, exist_ok=True)

    def val_batch(pred, yd, row):
        acc, _ = mse_metrics(pred.reshape(yd.shape), yd, threshold, True)
        val_metrics._commit(acc, yd.shape[0])
        row[:1].copy_(acc[:1])                    # the batch's squared-error sum

    loop = _EpochLoop(sess, train_loader, val_loader, lambda x, y: (x, y), val_batch, validation, sync_debug)
    history, split = [], {"seed": int(seed), "samples": n, "valid_size": float(valid_size)}
    t_start = time.perf_counter()
    for epoch in range(start, epochs):
        t0 = time.perf_counter()
        lr = plateau.lr
        train_rows, val_rows = loop.run(epoch)
        tsz, vsz = np.asarray(loop.train_sizes, np.float64), np.asarray(loop.val_sizes, np.float64)
        step_losses = train_rows[:, 0].astype(np.float32)                                 # loss_func per step (fp32)
        val_losses = (val_rows[:, 0] / vsz).astype(np.float32)
        # one reduction over the ranks (none without a process group): the weighted sums, their weights, the batch count
        t_sum, t_n, v_sum, v_n, v_batches = parallel.allreduce_sum(
            _weighted_sums(step_losses, tsz) + _weighted_sums(val_losses, vsz) + [len(vsz)], device)
        train_loss = float(t_sum / t_n)
        val_loss = float(v_sum / v_n)
        global_step += len(tsz)
        val_metrics.sync_across_ranks()
        sess.metrics.sync_across_ranks()
        val_m, train_m = val_metrics.compute(), sess.metrics.compute()
        val_metrics.reset()
        sess.metrics.reset()
        stop = stopper.update(val_loss, epoch)
        plateau.step(val_loss)
        stop, val_loss = _agree(stop, val_loss, stopper, plateau, device)
        next_lr = plateau.lr
        sess.set_lr(next_lr)
        score = val_loss if math.isfinite(val_loss) else math.inf
        is_best = best_score is None or score < best_score
        best_file, last_file = precip_file_names(hp["model"], epoch, val_loss)
        with _rank0_writes(device) as writer:
            t_ckpt = 0.0
            if writer:
                payload = precip_checkpoint(_cpu_state_dict(net), hp, epoch, global_step,
                                            _cpu_optimizer_state(sess.optimizer_state_dict()), plateau.state_dict(),
                                            stopper.state_dict(), score if is_best else best_score,
                                            os.path.join(ckpt_dir, best_file if is_best else best_name), split, world)
                t_ckpt = time.perf_counter()
                if is_best:
                    payload = _replace_file(ckpt_dir, best_name, best_file, payload)  # the last file is a copy of it
                _replace_file(ckpt_dir, last_name, last_file, payload)
                t_ckpt = time.perf_counter() - t_ckpt
            if is_best:
                best_score, best_name = score, best_file
            last_name = last_file
            rec = {"recipe": "precip", "model": hp["model"], "epoch": epoch, "global_step": global_step,
                   "train_loss": train_loss, "val_loss": val_loss, "lr": lr, "next_lr": next_lr, "train_samples": int(t_n),
                   "val_samples": int(v_n), "train_batches": len(tsz), "val_batches": int(v_batches),
                   "train_metrics": _plain_metrics(train_m), "val_metrics": _plain_metrics(val_m), "best": is_best,
                   "es_wait_count": stopper.wait_count, "stop": stop, "epoch_seconds": time.perf_counter() - t0,
                   "checkpoint_seconds": t_ckpt}
            if world > 1:
                rec["world_size"] = world
            history.append(rec)
            if writer:
                _append_history(os.fspath(out_dir), rec)
            if writer and verbose:
                print(f"\n\nEpoch {epoch} - Validation Metrics: {make_metrics_str(val_m)}")
                print(f"\n\nEpoch {epoch} - Train Metrics: {make_metrics_str(train_m)}")
                print(f"Epoch {epoch}: train_loss={train_loss:.6f}, val_loss={val_loss:.6f}, lr={lr}, "
                      f"time {(time.perf_counter() - t_start) / 60:.3f} min", flush=True)
        if stop:
            if verbose and rank == 0:
                print(f"Early stopping at epoch {epoch}: val_loss "
                      f"{'is not finite' if not math.isfinite(val_loss) else f'did not improve for {es_patience} epochs'}")
            break
    return FitResult(history=history, model=net, session=sess, split=(train_idx, valid_idx), train_loader=train_loader,
                     val_loader=val_loader, best_path=os.path.join(ckpt_dir, best_name) if best_name else None,
                     last_path=os.path.join(ckpt_dir, last_name) if last_name else None, hyper_parameters=hp)


# ------------------------------------------------------------------------------------------------ VOC
def voc_checkpoint(model, epoch, optimizer_state, val_loss, train_loss, miou, world_size=1):
    """train_SmaAtUNet.py:83-96's dict.  ``model`` is a CPU copy of the network (the trained one's parameters live in the
    session's flat buffers and its CBAMs carry the session's hooks).  A data-parallel run's (``world_size`` > 1) also
    holds ``world_size``."""
    copy = SmaAt_UNet(model.n_channels, model.n_classes, kernels_per_layer=model.inc.double_conv[0].kernels_per_layer,
                      bilinear=model.bilinear)
    sd = _cpu_state_dict(model)
    copy.load_state_dict(sd, strict=True)
    ckpt = {"model": copy, "epoch": int(epoch), "state_dict": sd, "optimizer_state_dict": optimizer_state,
            "val_loss": float(val_loss), "train_loss": float(train_loss), "mIOU": float(miou)}
    if world_size > 1:
        ckpt["world_size"] = int(world_size)
    return ckpt


def voc_file_names(class_name, epoch):
    """(best, per-epoch) file names of train_SmaAtUNet.py:97, :128."""
    return f"best_mIoU_model_{class_name}.pt", f"model_{class_name}_epoch_{int(epoch)}.pt"


def fit_voc(train_prefix, val_prefix, out_dir="checkpoints", epochs=200, batch_size=8, learning_rate=1e-3, earlystopping=30,
            save_every=1, lr_patience=4, seed=0, validation="serving", sync_debug=False, device=None, verbose=True):
    """``fit()`` of train_SmaAtUNet.py:23-136 with its ``__main__`` (:139-199): ``SmaAt_UNet(3, 21)``, Adam,
    ``nn.CrossEntropyLoss()``, batches of ``batch_size`` from the ``data.convert_voc`` shards (train: augmented and shuffled,
    validation: neither).  Per epoch: ``train_loss`` is the mean of the per-batch losses; validation gives ``val_loss``
    (the mean of the per-batch cross-entropy means) and ``IoU(21)``'s mean; ``mean_iou > best_mIoU`` writes the best file
    and resets the early-stopping counter, otherwise it counts and training stops at ``earlystopping``; every
    ``save_every`` epochs a per-epoch file; then ``ReduceLROnPlateau(mode="max", factor=0.1, patience=lr_patience)`` on
    the mean IoU."""
    for p in (train_prefix, val_prefix):
        for suffix in ("_images.npy", "_masks.npy"):
            if not os.path.isfile(f"{os.fspath(p)}{suffix}"):
                raise FileNotFoundError(f"fit_voc: no VOC shard at {os.fspath(p)}{suffix!r} (data.convert_voc writes it)")
    device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    train_ds = voc_segmentation_shard(train_prefix, augmentations=True, seed=seed)
    val_ds = voc_segmentation_shard(val_prefix, augmentations=False)
    (H, W, _), _ = train_ds.sample_shapes()
    torch.manual_seed(seed)
    net = SmaAt_UNet(3, 21)
    K = net.n_classes
    rank, world = parallel.rank_world()
    # the sharding of fit_precipitation: wrap-padded train shards, disjoint validation slices
    train_loader = PinnedBatchLoader(train_ds, batch_size, shuffle=True, seed=seed, drop_last=False, rank=rank, world=world)
    val_loader = PinnedBatchLoader(val_ds, batch_size, shuffle=False, drop_last=False, rank=rank, world=world, disjoint=True)
    tail = len(train_loader.epoch_indices()) % batch_size
    sess = TrainSession(net, batch_size, (3, H, W), lr=learning_rate, device=device, loss="cross_entropy",
                        input_transform=ops.VOCNormalize(), batch_sizes=(tail,) if tail else None, metrics=None)
    sess.check_partial_rows = False
    iou = IoU(K, normalized=False, device=device)
    norm = ops.VOCNormalize()

    def val_batch(pred, yd, row):
        acc, _ = ce_forward(pred, yd, -100, True, want_grad=False, conf=iou.conf_metric._conf)
        row.copy_(acc)                            # loss sum, counted pixels, invalid labels

    loop = _EpochLoop(sess, train_loader, val_loader, lambda x, y: norm(x, y), val_batch, validation, sync_debug)
    plateau = PlateauLR(learning_rate, "max", factor=0.1, patience=lr_patience)
    stopper = EarlyStopping(earlystopping, mode="max", check_finite=False, best=-1.0)
    with _rank0_writes(device) as writer:
        if writer:
            os.makedirs(os.fspath(out_dir), exist_ok=True)
    class_name = type(net).__name__
    history, t_start = [], time.perf_counter()
    for epoch in range(epochs):
        t0 = time.perf_counter()
        lr = plateau.lr
        train_rows, val_rows = loop.run(epoch)
        step_losses = train_rows[:, 0].astype(np.float32)
        with np.errstate(invalid="ignore", divide="ignore"):
            per_batch = np.where(val_rows[:, 2] > 0, np.nan, val_rows[:, 0] / val_rows[:, 1]).astype(np.float32)
        # the reference's losses are plain means of the per-batch losses: every batch weighs 1, over all ranks' batches
        t_sum, t_n, v_sum, v_n, invalid, t_samples, v_samples = parallel.allreduce_sum(
            _weighted_sums(step_losses, np.ones(len(step_losses))) + _weighted_sums(per_batch, np.ones(len(per_batch)))
            + [val_rows[:, 2].sum(), sum(loop.train_sizes), sum(loop.val_sizes)], device)
        train_loss = float(t_sum / t_n)
        val_loss = float(v_sum / v_n)
        iou.sync_across_ranks()
        iou.conf_metric._invalid.add_(int(invalid))
        _, mean_iou = iou.value()
        mean_iou = float(mean_iou)
        iou.reset()
        stop = stopper.update(mean_iou, epoch)
        if not stop:                              # the reference breaks before its scheduler step
            plateau.step(mean_iou)
        stop, mean_iou = _agree(stop, mean_iou, stopper, plateau, device)
        next_lr = plateau.lr
        best_file, epoch_file = voc_file_names(class_name, epoch)
        with _rank0_writes(device) as writer:
            if writer and stopper.improved:
                torch.save(voc_checkpoint(net, epoch, _cpu_optimizer_state(sess.optimizer_state_dict()), val_loss,
                                          train_loss, mean_iou, world), os.path.join(os.fspath(out_dir), best_file))
            rec = {"recipe": "voc", "model": class_name, "epoch": epoch, "train_loss": train_loss, "val_loss": val_loss,
                   "mIOU": mean_iou, "lr": lr, "best": stopper.improved, "earlystopping_counter": stopper.wait_count,
                   "stop": stop, "train_batches": len(train_rows), "val_batches": int(v_n),
                   "train_samples": int(t_samples), "val_samples": int(v_samples)}
            if world > 1:
                rec["world_size"] = world
            if not stop:                          # the reference breaks before its print and per-epoch file
                if writer and verbose:
                    print(f"Epoch: {epoch:5d}, Time: {(time.perf_counter() - t_start) / 60:.3f} min,"
                          f"Train_loss: {train_loss:2.10f}, Val_loss: {val_loss:2.10f},", f"mIOU: {mean_iou:.10f},",
                          f"lr: {lr},", f"Early stopping counter: {stopper.wait_count}/{earlystopping}", flush=True)
                if writer and save_every is not None and epoch % save_every == 0:
                    torch.save(voc_checkpoint(net, epoch, _cpu_optimizer_state(sess.optimizer_state_dict()), val_loss,
                                              train_loss, mean_iou, world), os.path.join(os.fspath(out_dir), epoch_file))
                sess.set_lr(next_lr)
            rec.update(next_lr=next_lr, epoch_seconds=time.perf_counter() - t0)
            history.append(rec)
            if writer:
                _append_history(os.fspath(out_dir), rec)
            if writer and stop and verbose:
                print(f"Stopping early --> mean IoU has not decreased over {earlystopping} epochs")
        if stop:
            break
    return FitResult(history=history, model=net, session=sess, train_loader=train_loader, val_loader=val_loader,
                     best_path=os.path.join(os.fspath(out_dir), voc_file_names(class_name, 0)[0]))


# ------------------------------------------------------------------------------------------------ command line
def _bool(v):
    if isinstance(v, bool):
        return v
    s = str(v).strip().lower()
    if s in ("1", "true", "yes", "y", "on"):
        return True
    if s in ("0", "false", "no", "n", "off"):
        return False
    raise argparse.ArgumentTypeError(f"expected a boolean, got {v!r}")


_BATCH_HELP = ("samples per step on each GPU: under torchrun --nproc-per-node N the global batch is N x this, as in "
               "Lightning's DDP; the learning rate is not scaled")


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Train the reference's models on the GPU path, without Lightning.  Under torchrun "
                                "(one process per GPU) the run is data-parallel; only rank 0 writes files")
    sub = p.add_subparsers(dest="recipe", required=True)
    pr = sub.add_parser("precip", help="train_precip_lightning.py: a precipitation network on a data.convert_h5 train shard")
    pr.add_argument("--model", default="UNetDSAttention", help=f"one of {', '.join(PRECIP_MODELS)}")
    pr.add_argument("--train-shard", "--train_shard", dest="train_shard", required=True,
                    help="(samples, T, H, W) float32 .npy of the train split (data.convert_h5 writes <prefix>_train.npy)")
    pr.add_argument("--out", "--out-dir", dest="out_dir", default="lightning/precip_regression",
                    help="checkpoints go to OUT/<model>/, the per-epoch history to OUT/history.jsonl")
    pr.add_argument("--batch_size", "--batch-size", type=int, default=16, help=_BATCH_HELP)
    pr.add_argument("--learning_rate", "--learning-rate", type=float, default=1e-3)
    pr.add_argument("--epochs", type=int, default=200)
    pr.add_argument("--lr_patience", "--lr-patience", type=int, default=4)
    pr.add_argument("--es_patience", "--es-patience", type=int, default=15)
    pr.add_argument("--valid_size", "--valid-size", type=float, default=0.1)
    pr.add_argument("--use_oversampled_dataset", "--use-oversampled-dataset", type=_bool, default=True)
    pr.add_argument("--kernels_per_layer", "--kernels-per-layer", type=int, default=2)
    pr.add_argument("--bilinear", type=_bool, default=True)
    pr.add_argument("--reduction_ratio", "--reduction-ratio", type=int, default=16)
    pr.add_argument("--threshold", type=float, default=0.5)
    pr.add_argument("--num_input_images", "--num-input-images", type=int, default=12)
    pr.add_argument("--num_output_images", "--num-output-images", type=int, default=6)
    pr.add_argument("--seed", type=int, default=0, help="the split's and the batch order's seed (stored in the checkpoint)")
    pr.add_argument("--resume-from-checkpoint", "--resume_from_checkpoint", dest="resume_from_checkpoint", default=None)
    vc = sub.add_parser("voc", help="train_SmaAtUNet.py: SmaAt_UNet(3, 21) on data.convert_voc shards")
    vc.add_argument("--train-prefix", required=True, help="data.convert_voc prefix of the train split")
    vc.add_argument("--val-prefix", required=True, help="data.convert_voc prefix of the val split")
    vc.add_argument("--out", "--out-dir", dest="out_dir", default="checkpoints")
    vc.add_argument("--batch-size", "--batch_size", dest="batch_size", type=int, default=8, help=_BATCH_HELP)
    vc.add_argument("--learning-rate", "--learning_rate", dest="learning_rate", type=float, default=1e-3)
    vc.add_argument("--epochs", type=int, default=200)
    vc.add_argument("--earlystopping", type=int, default=30)
    vc.add_argument("--save-every", "--save_every", dest="save_every", type=int, default=1)
    vc.add_argument("--lr-patience", "--lr_patience", dest="lr_patience", type=int, default=4)
    vc.add_argument("--seed", type=int, default=0)
    for s in (pr, vc):
        s.add_argument("--validation", choices=VALIDATION_MODES, default="serving",
                       help="validation forward: the uncaptured serving forward, or an InferenceSession re-captured per epoch")
        s.add_argument("--sync-debug", action="store_true", help="raise if anything in a batch loop waits for the GPU")
    return p.parse_args(argv)


def main(argv=None):
    a = vars(parse_args(argv))
    recipe = a.pop("recipe")
    with parallel.process_group_from_env():
        if recipe == "precip":
            return fit_precipitation(**a)
        return fit_voc(**a)


if __name__ == "__main__":
    main()
