"""Test-set evaluation of precipitation models on the GPU: what the reference's ``calc_metrics_test_set.py`` computes,
for several thresholds in one pass.

  * ``evaluate_precipitation(models, dataset, batch, thresholds, denormalize)`` -- one ``PinnedBatchLoader`` pass over the
    test shard.  Each batch crosses PCIe once; every model runs its captured ``InferenceSession`` on it and feeds its
    ``PrecipitationMetricsSweep``; a ``PersistenceModel`` is scored from the batch itself (its last input frame), with no
    forward.  Every sample counts as a batch of one, as in the reference script (batch_size=1, calc_metrics_test_set.py:95),
    whatever ``batch`` is.
  * ``load_reference_checkpoint(path)`` -- a reference Lightning ``.ckpt`` as a native model, without ``lightning``.
  * ``python -m smaat_unet_b200.evaluate`` -- the reference script's command line and output files
    (calc_metrics_test_set.py:18-72, :209-232), with ``--thresholds`` taking several values and ``--test-shard`` the shard
    written by ``data.convert_h5``.  Under ``torchrun --nproc-per-node N`` every rank scores its own contiguous slice of
    the test set and the totals are summed over the ranks before ``compute()``; rank 0 writes the files.
"""
from __future__ import annotations

import argparse
import csv
import json
import math
import os
import pickle

import torch

from . import parallel
from .data import PinnedBatchLoader, precipitation_maps_oversampled_shard
from .engine import InferenceSession
from .metrics import PrecipitationMetricsSweep
from .model import PersistenceModel, SmaAt_UNet, UNet, UNetAttention, UNetDS, UNetDSAttention4CBAMs

PERSISTENCE = "PersistenceModel"


# ------------------------------------------------------------------------------------------------ evaluation
def evaluate_precipitation(models, dataset, batch=32, thresholds=(0.5,), denormalize=True, device=None):
    """Score ``models`` ({name: native model}, ``PersistenceModel`` instances included) on every sample of ``dataset``
    (a ``precipitation_maps_oversampled_shard(..., train=False)``, or any shard dataset with ``sample_shapes``).

    Returns ``{name: {threshold: metrics}}``, in ``models``' order, where ``metrics`` is the reference's ``compute()`` dict
    (``PrecipitationMetricsSweep.compute``).  The batches are ``batch`` samples; the last, partial one runs on a graph
    captured for its size (``InferenceSession(batch_sizes=(tail,))``), so each sample is counted exactly once.

    With a process group, rank r scores the contiguous slice ``parallel.shard_range(len(dataset), r, world)`` at its own
    batch and tail sizes, and every accumulator's totals are summed over the ranks before ``compute()``: the counts equal
    a single process's exactly, the squared-error sums up to their summation order."""
    device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
    n = len(dataset)
    if n < 1:
        raise ValueError("evaluate_precipitation: the dataset is empty")
    rank, world = parallel.rank_world()
    lo, hi = parallel.shard_range(n, rank, world)
    accs = {name: PrecipitationMetricsSweep(thresholds, denormalize=denormalize, device=device) for name in models}
    if hi > lo:                                      # a rank of a test set smaller than the world scores nothing
        batch = min(int(batch), hi - lo)
        tail = (hi - lo) % batch
        in_shape, _ = dataset.sample_shapes()
        sessions = {name: InferenceSession(m, batch, in_shape, device=device, batch_sizes=(tail,) if tail else None)
                    for name, m in models.items() if not isinstance(m, PersistenceModel)}
        loader = PinnedBatchLoader(dataset, batch, drop_last=False, rank=rank, world=world, disjoint=True)
        score_batches(loader, sessions, accs, device)
    for acc in accs.values():
        acc.sync_across_ranks()
    return {name: acc.compute() for name, acc in accs.items()}


def score_batches(loader, sessions, accs, device):
    """The evaluation loop: every (x, y) batch of ``loader`` is copied to ``device`` once, then each accumulator in ``accs``
    is updated from its session's output (``sessions[name]``), or from the batch's last input frame where ``name`` has no
    session (the persistence baseline)."""
    with torch.cuda.device(device), torch.no_grad():
        for x, y in loader:
            xd = x.to(device, non_blocking=True)
            yd = y.to(device, non_blocking=True)
            copied = torch.cuda.Event()
            copied.record()
            loader.guard(copied)
            for name, acc in accs.items():
                if name in sessions:
                    acc.update(sessions[name].forward(xd), yd)
                else:
                    acc.update_persistence(xd, yd)


# ------------------------------------------------------------------------------------------------ checkpoints
# utils/model_classes.py:5-33, tested in its order: (file-name pattern, display name, native class)
CHECKPOINT_CLASSES = (
    ("UNetAttention", "UNet Attention", UNetAttention),
    ("UNetDSAttention4kpl", "UNetDS Attention with 4kpl", SmaAt_UNet),
    ("UNetDSAttention1kpl", "UNetDS Attention with 1kpl", SmaAt_UNet),
    ("UNetDSAttention4CBAMs", "UNetDS Attention 4CBAMs", UNetDSAttention4CBAMs),
    ("UNetDSAttention", "SmaAt-UNet", SmaAt_UNet),
    ("UNetDS", "UNetDS", UNetDS),
    ("UNet", "UNet", UNet),
)

# the constructor arguments each native class takes from ckpt["hyper_parameters"] (the ones the reference's class reads)
_CTOR_ARGS = {
    UNet: ("n_channels", "n_classes", "bilinear"),
    UNetAttention: ("n_channels", "n_classes", "bilinear", "reduction_ratio"),
    UNetDS: ("n_channels", "n_classes", "kernels_per_layer", "bilinear"),
    UNetDSAttention4CBAMs: ("n_channels", "n_classes", "kernels_per_layer", "bilinear", "reduction_ratio"),
    SmaAt_UNet: ("n_channels", "n_classes", "kernels_per_layer", "bilinear", "reduction_ratio"),
}


def checkpoint_class(file_name):
    """(display name, native class) for a reference checkpoint's file name (utils/model_classes.py:5-33)."""
    base = os.path.basename(os.fspath(file_name))
    for pattern, display, cls in CHECKPOINT_CLASSES:
        if pattern in base:
            return display, cls
    raise ValueError(f"load_reference_checkpoint: no model class for checkpoint file {base!r}: the name must contain one of "
                     f"{', '.join(p for p, _, _ in CHECKPOINT_CLASSES)} (utils/model_classes.py)")


class _PlainMapping(dict):
    """What a pickled Lightning ``AttributeDict`` or ``argparse.Namespace`` is loaded as: a dict, holding whatever state the
    pickle sets on it."""

    def __setstate__(self, state):
        if isinstance(state, dict):
            self.update(state)


# Lightning classes a checkpoint may pickle, mapped to plain mappings.  Matched by class name under a lightning package;
# the modules are never imported.
_LIGHTNING_PACKAGES = ("lightning", "pytorch_lightning", "lightning_fabric")
_LIGHTNING_MAPPINGS = {"AttributeDict": _PlainMapping}

_SAFE_GLOBALS = {
    ("collections", "OrderedDict"), ("collections", "defaultdict"), ("builtins", "set"), ("builtins", "frozenset"),
    ("builtins", "slice"), ("builtins", "complex"),
    ("torch._utils", "_rebuild_tensor_v2"), ("torch._utils", "_rebuild_parameter"),
    ("torch._utils", "_rebuild_parameter_with_state"), ("torch", "Size"), ("torch", "device"),
    ("pathlib", "PosixPath"), ("pathlib", "WindowsPath"), ("pathlib", "PurePosixPath"), ("pathlib", "PureWindowsPath"),
    ("pathlib", "Path"), ("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar"), ("numpy", "dtype"),
}


class _CheckpointUnpickler(pickle.Unpickler):
    def find_class(self, module, name):
        root = module.split(".")[0]
        if root in _LIGHTNING_PACKAGES:
            if name in _LIGHTNING_MAPPINGS:
                return _LIGHTNING_MAPPINGS[name]
            raise pickle.UnpicklingError(
                f"load_reference_checkpoint: the checkpoint pickles {module}.{name}, which the loader does not map to a plain "
                "type; it is not imported")
        if (module, name) == ("argparse", "Namespace"):
            return _PlainMapping
        if (module, name) in _SAFE_GLOBALS or (module == "torch" and isinstance(getattr(torch, name, None), torch.dtype)):
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"load_reference_checkpoint: the checkpoint pickles {module}.{name}, which the loader "
                                     "does not allow; it is not imported")


class _RestrictedPickle:
    """The ``pickle_module`` handed to ``torch.load``: its unpickler maps or refuses every global the file names."""

    Unpickler = _CheckpointUnpickler

    @staticmethod
    def load(f, **kw):
        return _CheckpointUnpickler(f, **kw).load()


def load_reference_checkpoint(path):
    """A reference Lightning checkpoint as a native model (CPU, eval mode), without importing ``lightning``.

    The class comes from the file name (``checkpoint_class``), the constructor arguments from ``ckpt["hyper_parameters"]``,
    the weights from ``ckpt["state_dict"]`` with ``strict=True``.  The pickle is read by a restricted unpickler: Lightning's
    ``AttributeDict`` and ``argparse.Namespace`` become plain mappings, tensors and plain containers load as usual, and any
    other class the file names raises ``pickle.UnpicklingError`` naming it, without importing it."""
    _, cls = checkpoint_class(path)
    ckpt = torch.load(path, map_location="cpu", pickle_module=_RestrictedPickle, weights_only=False)
    hp = ckpt.get("hyper_parameters")
    if hp is None or "state_dict" not in ckpt:
        raise ValueError(f"load_reference_checkpoint: {path} has no hyper_parameters / state_dict")
    missing = [k for k in _CTOR_ARGS[cls] if k not in hp]
    if missing:
        raise ValueError(f"load_reference_checkpoint: {path}: hyper_parameters lack {missing}")
    model = cls(**{k: hp[k] for k in _CTOR_ARGS[cls]})
    model.load_state_dict(ckpt["state_dict"], strict=True)
    return model.eval()


# ------------------------------------------------------------------------------------------------ command line
def _python(v):
    """convert_tensors_to_python (calc_metrics_test_set.py:37-48) for one metric value."""
    v = v.item() if isinstance(v, torch.Tensor) else v
    return float("nan") if isinstance(v, float) and math.isnan(v) else v


def metrics_file_name(threshold, denormalize, file_type):
    """calc_metrics_test_set.py:218 (the threshold as the reference's ``--threshold`` float prints it)."""
    return f"model_metrics_{float(threshold)}_{'denorm' if denormalize else 'norm'}.{file_type}"


def save_metrics(results, file_path, file_type="json"):
    """calc_metrics_test_set.py:51-72: csv rows of model name + values, else json (json and txt alike)."""
    with open(file_path, "w") as f:
        if file_type == "csv":
            writer = csv.writer(f)
            if results:
                first_model = next(iter(results.values()))
                writer.writerow(["Model"] + list(first_model.keys()))
                for model_name, metrics in results.items():
                    writer.writerow([model_name] + list(metrics.values()))
        else:
            json.dump(results, f, indent=4)


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Calculate metrics for precipitation models on the test set, on the GPU")
    p.add_argument("--model-folder", type=str, required=True, help="folder with the reference's .ckpt files")
    p.add_argument("--test-shard", type=str, required=True,
                   help="(samples, T, H, W) float32 .npy of the test split (data.convert_h5 writes <prefix>_test.npy)")
    p.add_argument("--thresholds", type=float, nargs="+", default=[0.5], help="precipitation thresholds in mm/h")
    p.add_argument("--normalized", action="store_false", dest="denormalize", default=True,
                   help="calculate metrics for normalized data")
    p.add_argument("--file-type", type=str, default="txt", choices=["json", "txt", "csv"], help="output file format")
    p.add_argument("--save-dir", type=str, default=None, help="where to save the metrics (default: under --model-folder)")
    p.add_argument("--batch", type=int, default=32, help="samples per forward (every sample still counts as a batch of one)")
    p.add_argument("--num-input-images", type=int, default=12)
    p.add_argument("--num-output-images", type=int, default=6)
    return p.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    with parallel.process_group_from_env() as (rank, world, _):
        writer = rank == 0                           # every rank loads the models and scores its slice; rank 0 writes
        thresholds = sorted(set(args.thresholds))
        tag = "denorm" if args.denormalize else "norm"
        save_dir = args.save_dir or os.path.join(args.model_folder, f"calc_metrics_test_set_results_{tag}")
        if writer:
            os.makedirs(save_dir, exist_ok=True)
        models = {PERSISTENCE: PersistenceModel()}
        for f in sorted(os.listdir(args.model_folder)):
            if f.endswith(".ckpt"):
                name, _ = checkpoint_class(f)
                if writer:
                    print(f"Loading model: {name}")
                models[name] = load_reference_checkpoint(os.path.join(args.model_folder, f))
        dataset = precipitation_maps_oversampled_shard(args.test_shard, args.num_input_images, args.num_output_images,
                                                       train=False)
        results = evaluate_precipitation(models, dataset, batch=args.batch, thresholds=thresholds,
                                         denormalize=args.denormalize)
        if writer:
            for t in thresholds:
                per_model = {name: {k: _python(v) for k, v in res[t].items()} for name, res in results.items()}
                path = os.path.join(save_dir, metrics_file_name(t, args.denormalize, args.file_type))
                save_metrics(per_model, path, args.file_type)
                print(f"Metrics saved to {path}")
        if world > 1:
            parallel.barrier(torch.device("cuda", torch.cuda.current_device()))
    return results


if __name__ == "__main__":
    main()
