"""The training driver's host logic (smaat_unet_b200.fit), on the CPU: the train / validation split, the plateau and
early-stopping decisions, checkpoint file names and contents, and the argument checks that run before any GPU work."""
import math
import os

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from smaat_unet_b200 import evaluate as E
from smaat_unet_b200 import fit as F


# ------------------------------------------------------------------------------------------------ split
@pytest.mark.parametrize("n", [1, 9, 10, 37, 1000, 5734])
@pytest.mark.parametrize("valid_size", [0.0, 0.1, 0.25, 0.5])
@pytest.mark.parametrize("seed", [0, 7, 1234])
def test_split_is_prepare_data_under_np_random_seed(n, valid_size, seed):
    np.random.seed(seed)
    indices = list(range(n))
    np.random.shuffle(indices)                        # regression_lightning.py:163-168
    split = int(np.floor(valid_size * n))
    train, valid = F.train_valid_split(n, valid_size, seed)
    assert train == indices[split:] and valid == indices[:split]
    assert sorted(train + valid) == list(range(n))


# ------------------------------------------------------------------------------------------------ plateau LR
SEQUENCES = {
    "falls": [1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4],
    "plateau": [1.0, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9, 0.9],
    "ties_and_tiny_gains": [1.0, 1.0, 0.99995, 1.0, 0.9999, 0.99, 0.99, 0.99, 0.99, 0.99, 0.99, 0.5, 0.5],
    "rises": [0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0, 1.1, 1.2, 1.3, 1.4],
    "with_nan": [1.0, 0.8, float("nan"), 0.8, 0.9, 0.9, 0.9, 0.7, 0.7, 0.7, 0.7, 0.7, 0.7],
}


@pytest.mark.parametrize("mode", ["min", "max"])
@pytest.mark.parametrize("patience", [0, 1, 4])
@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_plateau_lr_sequence_is_torch_reduce_lr_on_plateau(mode, patience, name):
    seq = SEQUENCES[name]
    w = torch.zeros(3, requires_grad=True)
    opt = torch.optim.Adam([w], lr=1e-3)
    ref = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, mode=mode, factor=0.1, patience=patience)
    ours = F.PlateauLR(1e-3, mode, factor=0.1, patience=patience)
    got, want = [], []
    for v in seq:
        ref.step(v)
        want.append(opt.param_groups[0]["lr"])
        got.append(ours.step(v))
    assert got == want


def test_plateau_state_round_trips_through_a_checkpoint_dict():
    a = F.PlateauLR(1e-3, "min", patience=2)
    for v in (1.0, 1.0, 1.0):
        a.step(v)
    b = F.PlateauLR(1e-3, "min", patience=2)
    b.load_state_dict(a.state_dict(), a.lr)
    for v in (1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 0.5):
        assert a.step(v) == b.step(v)


# ------------------------------------------------------------------------------------------------ early stopping
def stop_epoch(values, **kw):
    es = F.EarlyStopping(**kw)
    for e, v in enumerate(values):
        if es.update(v, e):
            return e
    return None


def test_early_stopping_lightning_rules():
    nan, inf = float("nan"), float("inf")
    # ties are no improvement (min_delta = 0, strictly below the best)
    assert stop_epoch([1.0, 0.9, 0.9, 0.95, 0.9], patience=3) == 4
    assert stop_epoch([1.0, 0.9, 0.9, 0.95, 0.89, 0.9, 0.9], patience=3) is None
    assert stop_epoch([1.0, 0.9, 0.9, 0.95, 0.89, 0.9, 0.9, 0.89], patience=3) == 7
    # patience counts epochs without improvement: patience 1 stops at the first one
    assert stop_epoch([1.0, 1.0], patience=1) == 1
    assert stop_epoch([1.0, 0.5], patience=1) is None
    # check_finite: a NaN or an infinite value stops at once, whatever the counter
    assert stop_epoch([1.0, nan, 0.1], patience=15) == 1
    assert stop_epoch([inf], patience=15) == 0
    assert stop_epoch([1.0, -inf], patience=15) == 1
    es = F.EarlyStopping(15)
    for e, v in enumerate([1.0, 0.5, 0.6, 0.7]):
        assert not es.update(v, e)
    assert es.best == 0.5 and es.wait_count == 2
    assert es.update(nan, 4) and es.stopped_epoch == 4 and es.wait_count == 2 and es.best == 0.5


def test_early_stopping_voc_fit_rules():
    nan = float("nan")
    kw = dict(mode="max", check_finite=False, best=-1.0)
    # mean_iou > best_mIoU resets the counter; a tie or a NaN counts; counter >= earlystopping stops
    assert stop_epoch([0.1, 0.2, 0.2, nan, 0.15], patience=3, **kw) == 4
    assert stop_epoch([0.1, 0.1, 0.3, 0.3, 0.3, 0.3], patience=3, **kw) == 5
    assert stop_epoch([nan, nan], patience=2, **kw) == 1
    assert stop_epoch([0.0, 0.0], patience=30, **kw) is None
    es = F.EarlyStopping(30, **kw)
    assert not es.update(0.0) and es.improved and es.best == 0.0        # 0.0 > -1.0: the first epoch always saves
    assert not es.update(0.0) and not es.improved and es.wait_count == 1


def test_early_stopping_state_round_trips():
    a = F.EarlyStopping(4)
    for e, v in enumerate([1.0, 0.7, 0.8, 0.9]):
        a.update(v, e)
    b = F.EarlyStopping(4)
    b.load_state_dict(a.state_dict())
    for e, v in enumerate([0.8, 0.8, 0.6, 0.9, 0.9, 0.9, 0.9], start=4):
        assert a.update(v, e) == b.update(v, e)
        assert a.state_dict() == b.state_dict()


# ------------------------------------------------------------------------------------------------ checkpoints
def test_file_names():
    best, last = F.precip_file_names("UNetDSAttention", 12, 0.0123456789)
    assert best == "UNetDSAttention_rain_threshold_50_epoch=12-val_loss=0.012346.ckpt"
    assert last == "UNetDSAttention_rain_threshold_50_epoch=12-val_loss=0.012346_last.ckpt"
    assert F.voc_file_names("SmaAt_UNet", 3) == ("best_mIoU_model_SmaAt_UNet.pt", "model_SmaAt_UNet_epoch_3.pt")


def _plain(obj, path="ckpt"):
    """Every leaf of a checkpoint is a plain Python value or a tensor that owns its storage exactly."""
    if isinstance(obj, dict):
        for k, v in obj.items():
            assert isinstance(k, (str, int)), f"{path}: key {k!r}"
            _plain(v, f"{path}[{k!r}]")
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _plain(v, f"{path}[{i}]")
    elif isinstance(obj, torch.Tensor):
        assert type(obj) is torch.Tensor and obj.device.type == "cpu", path
        assert obj.untyped_storage().nbytes() == obj.numel() * obj.element_size(), f"{path} is a view of a larger buffer"
    else:
        assert obj is None or type(obj) in (bool, int, float, str), f"{path}: {type(obj).__name__}"


CLASSES = [("UNet", S.UNet, {}), ("UNetAttention", S.UNetAttention, {"reduction_ratio": 8}),
           ("UNetDS", S.UNetDS, {"kernels_per_layer": 1}), ("UNetDSAttention", S.SmaAt_UNet, {"kernels_per_layer": 2}),
           ("UNetDSAttention4CBAMs", S.UNetDSAttention4CBAMs, {"kernels_per_layer": 1, "reduction_ratio": 8})]


@pytest.mark.parametrize("name,cls,extra", CLASSES, ids=[c[0] for c in CLASSES])
def test_precip_checkpoint_loads_through_evaluate(tmp_path, name, cls, extra):
    hp = F.precip_hyper_parameters(name, str(tmp_path / "train.npy"), seed=3, **extra)
    torch.manual_seed(0)
    model = F.build_precip_model(hp)
    assert type(model) is cls
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn_like(p) * 0.01)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    plateau = F.PlateauLR(1e-3, "min", patience=hp["lr_patience"])
    plateau.step(0.5)
    es = F.EarlyStopping(hp["es_patience"])
    es.update(0.5, 0)
    best, _ = F.precip_file_names(name, 0, 0.5)
    ck = F.precip_checkpoint(F._cpu_state_dict(model), hp, 0, 7, opt.state_dict(), plateau.state_dict(), es.state_dict(), 0.5,
                             str(tmp_path / best), {"seed": 3, "samples": 37, "valid_size": 0.1})
    assert set(ck) >= {"state_dict", "hyper_parameters", "epoch", "global_step", "optimizer_states", "lr_schedulers",
                       "callbacks", "pytorch-lightning_version"}
    _plain(ck)
    path = tmp_path / best
    torch.save(ck, path)
    display, got_cls = E.checkpoint_class(path)
    assert got_cls is cls
    loaded = E.load_reference_checkpoint(path)
    assert type(loaded) is cls and not loaded.training
    for k in E._CTOR_ARGS[cls]:
        assert getattr(loaded, k, hp[k]) == hp[k]
    if "kernels_per_layer" in E._CTOR_ARGS[cls]:
        assert loaded.inc.double_conv[0].kernels_per_layer == hp["kernels_per_layer"]
    sd, ref = loaded.state_dict(), model.state_dict()
    assert sd.keys() == ref.keys()
    for k in ref:
        assert torch.equal(sd[k], ref[k]), k
    raw = torch.load(path, map_location="cpu", pickle_module=E._RestrictedPickle, weights_only=False)
    assert raw["hyper_parameters"] == hp and raw["epoch"] == 0 and raw["global_step"] == 7


def test_state_dict_of_views_is_self_contained():
    flat = torch.arange(100, dtype=torch.float32)
    m = torch.nn.Linear(3, 2)
    with torch.no_grad():
        m.weight.data = flat[10:16].view(2, 3)
        m.bias.data = flat[40:42]
    sd = F._cpu_state_dict(m)
    _plain(sd)
    assert torch.equal(sd["weight"], flat[10:16].view(2, 3))


def test_voc_checkpoint_keys():
    torch.manual_seed(0)
    model = S.SmaAt_UNet(3, 21)
    opt = torch.optim.Adam(model.parameters())
    ck = F.voc_checkpoint(model, 4, opt.state_dict(), 1.5, 2.5, 0.25)
    assert set(ck) == {"model", "epoch", "state_dict", "optimizer_state_dict", "val_loss", "train_loss", "mIOU"}
    assert type(ck["model"]) is S.SmaAt_UNet and ck["model"] is not model
    for k, v in model.state_dict().items():
        assert torch.equal(ck["state_dict"][k], v) and torch.equal(ck["model"].state_dict()[k], v)
    assert (ck["epoch"], ck["val_loss"], ck["train_loss"], ck["mIOU"]) == (4, 1.5, 2.5, 0.25)


def test_make_metrics_str():
    nan = float("nan")
    s = F.make_metrics_str({"mse": torch.tensor(0.5), "precision": torch.tensor(nan), "f1": 0.25, "far": nan})
    assert s == "mse: 0.5000 | f1: 0.2500"


# ------------------------------------------------------------------------------------------------ argument checks
def _shard(tmp_path, n=20, hw=64):
    rng = np.random.default_rng(0)
    path = tmp_path / "p_train.npy"
    np.save(path, rng.random((n, 13, hw, hw), dtype=np.float32))
    return path


@pytest.mark.parametrize("model", ["PersistenceModel", "UNetDSAttention1kpl", "SmaAt_UNet", ""])
def test_refused_models(tmp_path, model):
    with pytest.raises(ValueError, match="PersistenceModel|unknown model"):
        F.fit_precipitation(model, _shard(tmp_path), tmp_path / "out")


def test_refused_models_from_the_command_line(tmp_path):
    with pytest.raises(ValueError, match="PersistenceModel"):
        F.main(["precip", "--model", "PersistenceModel", "--train-shard", str(_shard(tmp_path)), "--out", str(tmp_path)])
    with pytest.raises(ValueError, match="unknown model"):
        F.main(["precip", "--model", "Foo", "--train-shard", str(_shard(tmp_path)), "--out", str(tmp_path)])


def test_missing_shards(tmp_path):
    with pytest.raises(FileNotFoundError):
        F.fit_precipitation("UNetDS", tmp_path / "nope_train.npy", tmp_path / "out")
    with pytest.raises(FileNotFoundError):
        F.fit_voc(tmp_path / "nope_train", tmp_path / "nope_val", tmp_path / "out")
    assert not (tmp_path / "out").exists()


def _resume_file(tmp_path, hp, samples):
    torch.manual_seed(0)
    model = F.build_precip_model(hp)
    ck = F.precip_checkpoint(F._cpu_state_dict(model), hp, 1, 4, torch.optim.Adam(model.parameters()).state_dict(),
                             F.PlateauLR(1e-3, "min").state_dict(), F.EarlyStopping(15).state_dict(), 0.5, "",
                             {"seed": hp["seed"], "samples": samples, "valid_size": hp["valid_size"]})
    best, last = F.precip_file_names(hp["model"], 1, 0.5)
    path = tmp_path / last
    torch.save(ck, path)
    return path


@pytest.mark.parametrize("change", [{"model": "UNetDS"}, {"seed": 1}, {"kernels_per_layer": 1}, {"valid_size": 0.2},
                                    {"batch_size": 8}, {"samples": 21}])
def test_mismatched_resume_is_refused(tmp_path, change):
    shard = _shard(tmp_path)
    change = dict(change)
    samples = change.pop("samples", 20)
    kw = dict(model="UNetDSAttention", seed=0)
    kw.update(change)
    hp = F.precip_hyper_parameters(train_shard=str(shard), **kw)
    path = _resume_file(tmp_path, hp, samples)
    with pytest.raises(ValueError, match="does not match"):
        F.fit_precipitation("UNetDSAttention", shard, tmp_path / "out", resume_from_checkpoint=path)
    # the same checkpoint is accepted by the run it belongs to
    F.check_resume(torch.load(path, weights_only=False), hp, samples)


def test_checkpoint_names_resolve_to_their_class():
    for name, cls, _ in CLASSES:
        best, last = F.precip_file_names(name, 3, 0.25)
        assert E.checkpoint_class(best)[1] is cls and E.checkpoint_class(last)[1] is cls
    assert math.isinf(F.EarlyStopping(1).best)


def test_history_and_hyper_parameters_defaults():
    hp = F.precip_hyper_parameters()
    assert (hp["model"], hp["n_channels"], hp["n_classes"], hp["kernels_per_layer"], hp["bilinear"], hp["reduction_ratio"],
            hp["batch_size"], hp["learning_rate"], hp["epochs"], hp["lr_patience"], hp["es_patience"], hp["valid_size"],
            hp["use_oversampled_dataset"]) == ("UNetDSAttention", 12, 1, 2, True, 16, 16, 1e-3, 200, 4, 15, 0.1, True)
    args = F.parse_args(["precip", "--train-shard", "x.npy"])
    assert (args.model, args.batch_size, args.epochs, args.kernels_per_layer, args.use_oversampled_dataset) == \
        ("UNetDSAttention", 16, 200, 2, True)
    voc = F.parse_args(["voc", "--train-prefix", "a", "--val-prefix", "b"])
    assert (voc.batch_size, voc.learning_rate, voc.earlystopping, voc.save_every, voc.lr_patience) == (8, 1e-3, 30, 1, 4)
    assert os.path.basename(F.HISTORY_FILE) == "history.jsonl"
