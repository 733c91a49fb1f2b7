"""Test-set evaluation without a GPU: the sweep oracle against the reference's batch-1 numbers, the batch-size trap, the
checkpoint loader, the command line's files, and the sweep entry points' argument checks."""
import csv
import ctypes
import json
import math
import os
import pathlib
import pickle
import sys
import types
from collections import OrderedDict

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle import metrics_oracle as MO
from oracle import sweep_oracle as SO
from smaat_unet_b200 import evaluate as E

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "precip_eval.npz"))
TH = SO.GOLDEN_THRESHOLDS
KEYS = ("mse", "mse_denorm", "mse_pixel", "precision", "recall", "accuracy", "f1", "csi", "far", "hss")
COUNTS = ("total_tp", "total_fp", "total_tn", "total_fn", "total_samples", "total_pixels")


def _same(a, b, tol, what):
    a, b = float(a), float(b)
    if math.isnan(b):
        assert math.isnan(a), what
    else:
        assert abs(a - b) <= tol * max(abs(b), 1e-30), f"{what}: {a} vs {b}"


def _persistence_rows():
    x, y = GOLD["x"], GOLD["y"]
    return x[:, -1].reshape(len(x), -1), y.reshape(len(y), -1)


# ----------------------------------------------------------------------------------------------- oracle vs reference
def test_golden_samples_are_the_oracle_samples():
    x, y = SO.eval_samples()
    np.testing.assert_array_equal(x, GOLD["x"])
    np.testing.assert_array_equal(y, GOLD["y"])
    assert tuple(GOLD["thresholds"]) == TH


@pytest.mark.parametrize("denorm", [True, False])
def test_oracle_sweep_matches_reference_batch1(denorm):
    tag = "denorm" if denorm else "norm"
    p, y = _persistence_rows()
    st = SO.sweep(p, y, TH, denorm)
    assert st["skipped"] == 2
    out = SO.compute(st, TH, denorm)
    for i, t in enumerate(TH):
        s = SO.threshold_state(st, i)
        for k in COUNTS:                                # integer states: exact
            assert int(s[k]) == int(GOLD[f"{tag}/{t}/{k}"]), (t, k)
        for k in KEYS:                                  # the reference accumulates in float32
            _same(out[t][k], GOLD[f"{tag}/{t}/{k}"], 2e-6, f"{tag}/{t}/{k}")


def test_golden_reaches_every_threshold_cell():
    # the denormalised rain fields fill all four cells at 0.5-10 mm/h; the boundary samples put values on both sides of
    # every threshold
    for t in TH[:-1]:
        assert all(int(GOLD[f"denorm/{t}/{k}"]) > 0 for k in ("total_tp", "total_fp", "total_tn", "total_fn")), t
    for t in TH:
        assert int(GOLD[f"norm/{t}/total_fp"]) + int(GOLD[f"norm/{t}/total_fn"]) > 0, t


def test_batch_size_trap():
    """The reference's update divides each batch's sum by B and compute() divides by the sample count again: at B = 4 its
    mse is a quarter of the batch-1 figure.  The sweep's totals are the batch-1 figures whatever the grouping."""
    p, y = _persistence_rows()
    keep = ~(np.isnan(p).any(1) | np.isnan(y).any(1))
    p, y = p[keep][:8], y[keep][:8]
    b1, b4 = MO.new_state(), MO.new_state()
    for i in range(8):
        MO.update(b1, p[i:i + 1], y[i:i + 1], 0.5, True)
    for i in range(0, 8, 4):
        MO.update(b4, p[i:i + 4], y[i:i + 4], 0.5, True)
    m1, m4 = MO.compute(b1), MO.compute(b4)
    for k in ("mse", "mse_denorm", "mse_pixel"):
        assert m4[k] == pytest.approx(m1[k] / 4, rel=1e-12), k
    st = SO.sweep(p, y, (0.5,), True)
    s = SO.threshold_state(st, 0)
    for k in COUNTS:
        assert int(s[k]) == int(b1[k]), k
    assert s["total_loss"] == pytest.approx(b1["total_loss"], rel=1e-12)
    assert s["total_loss_denorm"] == pytest.approx(b1["total_loss_denorm"], rel=1e-12)


def test_sweep_threshold_totals_layout():
    """threshold_totals() turns the summed histogram into PrecipitationMetrics' nine totals per threshold."""
    m = S.PrecipitationMetricsSweep(TH[:3], device="cpu")
    T1 = 4
    h = torch.arange(T1 * T1, dtype=torch.float64)
    m._totals.copy_(torch.cat([torch.tensor([10.0, 20.0, 3.0, 300.0, 1.0]), h]))
    hn = h.view(T1, T1).to(torch.int64)
    for i, (t, v) in enumerate(m.threshold_totals().items(), start=1):
        assert t == TH[i - 1]
        assert v[:4].tolist() == [10.0, 20.0, 3.0, 300.0] and v[8] == 1.0
        assert v[4:8].tolist() == [hn[:i, :i].sum(), hn[:i, i:].sum(), hn[i:, :i].sum(), hn[i:, i:].sum()]


@pytest.mark.parametrize("bad", [(), (1.0, 0.5), (0.5, 0.5), (0.5, float("nan")), tuple(range(1, 34))])
def test_sweep_refuses_bad_thresholds(bad):
    with pytest.raises(ValueError, match="strictly increasing"):
        S.PrecipitationMetricsSweep(bad, device="cpu")


# ----------------------------------------------------------------------------------------------- C ABI argument checks
def _thr(*v):
    return (ctypes.c_float * max(len(v), 1))(*v)


_F = 16          # a non-null address; every call below is refused before anything is read through it


@pytest.mark.parametrize("args,msg", [
    ((_F, 4, _F, 2, 4, 47.83, _thr(1.0, 0.5), 2, 1, _F, _F), b"strictly increasing"),
    ((_F, 4, _F, 2, 4, 47.83, _thr(0.5, 0.5), 2, 1, _F, _F), b"strictly increasing"),
    ((_F, 4, _F, 2, 4, 47.83, _thr(float("nan")), 1, 1, _F, _F), b"NaN"),
    ((_F, 4, _F, 2, 4, 47.83, _thr(0.5), 0, 1, _F, _F), b"T=0"),
    ((_F, 4, _F, 2, 4, 47.83, _thr(*range(1, 34)), 33, 1, _F, _F), b"T=33"),
    ((_F, 4, _F, 2, 0, 47.83, _thr(0.5), 1, 1, _F, _F), b"P=0"),
    ((_F, 4, _F, 0, 4, 47.83, _thr(0.5), 1, 1, _F, _F), b"B=0"),
    ((_F, 3, _F, 2, 4, 47.83, _thr(0.5), 1, 1, _F, _F), b"batch stride"),
    ((None, 4, _F, 2, 4, 47.83, _thr(0.5), 1, 1, _F, _F), b"null"),
    ((_F, 4, None, 2, 4, 47.83, _thr(0.5), 1, 1, _F, _F), b"null"),
    ((_F, 4, _F, 2, 4, 47.83, None, 1, 1, _F, _F), b"null"),
    ((_F, 4, _F, 2, 4, 47.83, _thr(0.5), 1, 1, None, _F), b"null"),
    ((_F, 4, _F, 2, 4, 47.83, _thr(0.5), 1, 1, _F, None), b"null"),
])
def test_sweep_fwd_refuses_before_launch(args, msg):
    lib = S._lib.load()
    assert lib.smaat_precip_sweep_fwd(*args, None) == -1
    assert msg in lib.smaat_last_error()


@pytest.mark.parametrize("args", [(None, _F, 2, 4, 1, 1, _F), (_F, None, 2, 4, 1, 1, _F), (_F, _F, 2, 4, 1, 1, None),
                                  (_F, _F, 0, 4, 1, 1, _F), (_F, _F, 2, 0, 1, 1, _F), (_F, _F, 2, 4, 0, 1, _F),
                                  (_F, _F, 2, 4, 33, 1, _F)])
def test_sweep_commit_refuses_before_launch(args):
    lib = S._lib.load()
    assert lib.smaat_precip_sweep_commit(*args, None) == -1
    assert b"precip_sweep_commit" in lib.smaat_last_error()


# ----------------------------------------------------------------------------------------------- PersistenceModel
def test_persistence_model_is_the_last_frame():
    m = S.PersistenceModel()
    assert list(m.parameters()) == [] and m.state_dict() == {}
    x = torch.randn(2, 5, 3, 4)
    assert torch.equal(m(x), x[:, -1:])


# ----------------------------------------------------------------------------------------------- checkpoints
LIGHTNING_DATA = "lightning.fabric.utilities.data"
LIGHTNING_CB = "lightning.pytorch.callbacks.model_checkpoint"


@pytest.fixture
def lightning_standin(monkeypatch):
    """Stand-in Lightning modules, registered only while checkpoints are written: AttributeDict (a dict) and a
    ModelCheckpoint-like class, so the pickles name them as a Lightning checkpoint would."""
    mods = {}
    for name in ("lightning", "lightning.fabric", "lightning.fabric.utilities", LIGHTNING_DATA, "lightning.pytorch",
                 "lightning.pytorch.callbacks", LIGHTNING_CB):
        mods[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, mods[name])

    class AttributeDict(dict):
        pass

    class ModelCheckpoint:
        pass

    AttributeDict.__module__, AttributeDict.__qualname__ = LIGHTNING_DATA, "AttributeDict"
    ModelCheckpoint.__module__, ModelCheckpoint.__qualname__ = LIGHTNING_CB, "ModelCheckpoint"
    mods[LIGHTNING_DATA].AttributeDict = AttributeDict
    mods[LIGHTNING_CB].ModelCheckpoint = ModelCheckpoint
    return types.SimpleNamespace(AttributeDict=AttributeDict, ModelCheckpoint=ModelCheckpoint)


def _no_lightning(monkeypatch):
    """From here on `import lightning` fails, as on a machine without it."""
    for name in list(sys.modules):
        if name.split(".")[0] in ("lightning", "pytorch_lightning", "lightning_fabric"):
            monkeypatch.delitem(sys.modules, name)
    for name in ("lightning", "pytorch_lightning", "lightning_fabric"):
        monkeypatch.setitem(sys.modules, name, None)
    with pytest.raises(ImportError):
        import lightning  # noqa: F401


def _hparams(ld, **kw):
    hp = ld.AttributeDict(n_channels=12, n_classes=1, kernels_per_layer=2, bilinear=True, reduction_ratio=16,
                          learning_rate=1e-3, lr_patience=4, model="UNetDSAttention",
                          dataset_folder=pathlib.PosixPath("/data/precipitation/train_test.h5"))
    hp.update(kw)
    return hp


def _write_ckpt(path, model, hp, extra=None):
    ck = {"epoch": 7, "global_step": 1234, "pytorch-lightning_version": "2.5.0", "state_dict": OrderedDict(model.state_dict()),
          "hyper_parameters": hp, "hparams_name": "hparams", "loops": {"fit_loop": {"state_dict": {}, "epoch_progress": {}}},
          "optimizer_states": [{"state": {}, "param_groups": [{"lr": 1e-3, "params": [0, 1]}]}],
          "lr_schedulers": [{"factor": 0.1, "patience": 4, "mode": "min", "best": float("inf")}]}
    ck.update(extra or {})
    torch.save(ck, path)


# (file name, expected native class, kernels_per_layer in the hyper-parameters)
CKPT_NAMES = [
    ("UNetAttention_rain_threshold_50_epoch=40.ckpt", S.UNetAttention, 1),
    ("UNetDSAttention4kpl_rain_threshold_50.ckpt", S.SmaAt_UNet, 4),
    ("UNetDSAttention1kpl_rain_threshold_50.ckpt", S.SmaAt_UNet, 1),
    ("UNetDSAttention4CBAMs_rain_threshold_50.ckpt", S.UNetDSAttention4CBAMs, 2),
    ("UNetDSAttention_rain_threshold_50.ckpt", S.SmaAt_UNet, 2),
    ("UNetDS_rain_threshold_50.ckpt", S.UNetDS, 2),
    ("UNet_rain_threshold_50.ckpt", S.UNet, 1),
]


def _build(cls, k, n_channels=12):
    torch.manual_seed(k)
    if cls in (S.UNet,):
        return cls(n_channels, 1, bilinear=True)
    if cls is S.UNetAttention:
        return cls(n_channels, 1, bilinear=True, reduction_ratio=16)
    if cls is S.UNetDS:
        return cls(n_channels, 1, kernels_per_layer=k, bilinear=True)
    return cls(n_channels, 1, kernels_per_layer=k, bilinear=True, reduction_ratio=16)


@pytest.mark.parametrize("fname,cls,k", CKPT_NAMES)
def test_load_reference_checkpoint_without_lightning(tmp_path, monkeypatch, lightning_standin, fname, cls, k):
    ref = _build(cls, k, n_channels=6)
    path = tmp_path / fname
    _write_ckpt(path, ref, _hparams(lightning_standin, n_channels=6, kernels_per_layer=k))
    _no_lightning(monkeypatch)
    assert E.checkpoint_class(fname)[1] is cls
    got = E.load_reference_checkpoint(str(path))
    assert type(got) is cls and not got.training
    assert got.n_channels == 6 and got.n_classes == 1
    if hasattr(got.inc, "double_conv") and hasattr(got.inc.double_conv[0], "kernels_per_layer"):
        assert got.inc.double_conv[0].kernels_per_layer == k
    sd, want = got.state_dict(), ref.state_dict()
    assert list(sd) == list(want)
    for key in want:
        assert torch.equal(sd[key], want[key]), key
    assert not any(n.split(".")[0] == "lightning" and m is not None for n, m in sys.modules.items())


def test_checkpoint_class_names_follow_the_reference_order():
    assert E.checkpoint_class("a/b/UNetDSAttention4CBAMs.ckpt") == ("UNetDS Attention 4CBAMs", S.UNetDSAttention4CBAMs)
    assert E.checkpoint_class("UNetDSAttention.ckpt") == ("SmaAt-UNet", S.SmaAt_UNet)
    assert E.checkpoint_class("UNetAttention.ckpt") == ("UNet Attention", S.UNetAttention)
    with pytest.raises(ValueError, match="no model class for checkpoint file 'ConvLSTM.ckpt'"):
        E.checkpoint_class("ConvLSTM.ckpt")
    with pytest.raises(ValueError, match="no model class"):
        E.load_reference_checkpoint("/nonexistent/ConvLSTM.ckpt")


def test_unmapped_pickled_class_is_named_and_not_imported(tmp_path, monkeypatch, lightning_standin):
    path = tmp_path / "UNet_rain.ckpt"
    _write_ckpt(path, _build(S.UNet, 1, 4), _hparams(lightning_standin, n_channels=4),
                extra={"callbacks": {"ModelCheckpoint{'monitor': 'val_loss'}": lightning_standin.ModelCheckpoint()}})
    _no_lightning(monkeypatch)
    with pytest.raises(pickle.UnpicklingError, match=f"{LIGHTNING_CB}.ModelCheckpoint"):
        E.load_reference_checkpoint(str(path))
    assert sys.modules.get("lightning.pytorch.callbacks.model_checkpoint") is None


def test_non_lightning_globals_are_refused(tmp_path, monkeypatch, lightning_standin):
    path = tmp_path / "UNet_rain.ckpt"
    _write_ckpt(path, _build(S.UNet, 1, 4), _hparams(lightning_standin, n_channels=4), extra={"fn": os.getcwd})
    _no_lightning(monkeypatch)
    with pytest.raises(pickle.UnpicklingError, match="posix.getcwd"):
        E.load_reference_checkpoint(str(path))


def test_checkpoint_load_is_strict(tmp_path, monkeypatch, lightning_standin):
    m = _build(S.UNet, 1, 4)
    path = tmp_path / "UNet_rain.ckpt"
    sd = OrderedDict(m.state_dict())
    sd["extra.weight"] = torch.zeros(1)
    ck_model = types.SimpleNamespace(state_dict=lambda: sd)
    _write_ckpt(path, ck_model, _hparams(lightning_standin, n_channels=4))
    _no_lightning(monkeypatch)
    with pytest.raises(RuntimeError, match="Unexpected key"):
        E.load_reference_checkpoint(str(path))
    path2 = tmp_path / "UNetDS_rain.ckpt"
    _write_ckpt(path2, _build(S.UNetDS, 2, 4), {"n_channels": 4, "n_classes": 1})
    with pytest.raises(ValueError, match="kernels_per_layer"):
        E.load_reference_checkpoint(str(path2))


# ----------------------------------------------------------------------------------------------- command line
def _fake_results(models, dataset, batch=32, thresholds=(0.5,), denormalize=True, device=None):
    """What evaluate_precipitation returns, with values that identify model and threshold."""
    out = {}
    for j, name in enumerate(models):
        out[name] = {t: {k: torch.tensor(float("nan") if k == "far" else 100 * j + t + i / 10, dtype=torch.float32)
                         for i, k in enumerate(KEYS)} for t in thresholds}
    _fake_results.seen = dict(models=models, n=len(dataset), batch=batch, thresholds=thresholds, denormalize=denormalize)
    return out


@pytest.mark.parametrize("file_type", ["json", "txt", "csv"])
@pytest.mark.parametrize("normalized", [False, True])
def test_cli_writes_reference_layout(tmp_path, monkeypatch, lightning_standin, file_type, normalized):
    folder = tmp_path / "comparison"
    folder.mkdir()
    _write_ckpt(folder / "UNetDS_rain_threshold_50.ckpt", _build(S.UNetDS, 2, 12), _hparams(lightning_standin))
    _write_ckpt(folder / "UNetDSAttention_rain_threshold_50.ckpt", _build(S.SmaAt_UNet, 2, 12), _hparams(lightning_standin))
    (folder / "notes.txt").write_text("not a checkpoint")
    shard = tmp_path / "test.npy"
    np.save(shard, np.zeros((5, 18, 32, 32), np.float32))
    monkeypatch.setattr(E, "evaluate_precipitation", _fake_results)
    _no_lightning(monkeypatch)
    argv = ["--model-folder", str(folder), "--test-shard", str(shard), "--thresholds", "1", "0.5", "--file-type", file_type,
            "--batch", "4"] + (["--normalized"] if normalized else [])
    E.main(argv)
    seen = _fake_results.seen
    assert list(seen["models"]) == ["PersistenceModel", "SmaAt-UNet", "UNetDS"]
    assert isinstance(seen["models"]["PersistenceModel"], S.PersistenceModel)
    assert seen["n"] == 5 and seen["batch"] == 4 and list(seen["thresholds"]) == [0.5, 1.0]
    assert seen["denormalize"] is (not normalized)
    tag = "norm" if normalized else "denorm"
    out_dir = folder / f"calc_metrics_test_set_results_{tag}"
    assert sorted(os.listdir(out_dir)) == sorted(f"model_metrics_{t}_{tag}.{file_type}" for t in ("0.5", "1.0"))
    for t in (0.5, 1.0):
        path = out_dir / f"model_metrics_{t}_{tag}.{file_type}"
        want = {name: {k: (float("nan") if k == "far" else float(np.float32(100 * j + t + i / 10))) for i, k in enumerate(KEYS)}
                for j, name in enumerate(["PersistenceModel", "SmaAt-UNet", "UNetDS"])}
        text = path.read_text()
        if file_type == "csv":
            rows = list(csv.reader(text.splitlines()))
            assert rows[0] == ["Model"] + list(KEYS)
            assert [r[0] for r in rows[1:]] == list(want)
            for r in rows[1:]:
                assert r[1:] == [str(v) for v in want[r[0]].values()]
        else:
            assert text == json.dumps(want, indent=4)
            assert "NaN" in text


def test_cli_save_dir_and_file_names(tmp_path, monkeypatch):
    assert E.metrics_file_name(0.5, True, "txt") == "model_metrics_0.5_denorm.txt"
    assert E.metrics_file_name(2, False, "csv") == "model_metrics_2.0_norm.csv"
    folder = tmp_path / "models"
    folder.mkdir()
    shard = tmp_path / "test.npy"
    np.save(shard, np.zeros((3, 18, 32, 32), np.float32))
    monkeypatch.setattr(E, "evaluate_precipitation", _fake_results)
    E.main(["--model-folder", str(folder), "--test-shard", str(shard), "--save-dir", str(tmp_path / "out")])
    assert os.listdir(tmp_path / "out") == ["model_metrics_0.5_denorm.txt"]
    assert list(json.loads((tmp_path / "out" / "model_metrics_0.5_denorm.txt").read_text())) == ["PersistenceModel"]
