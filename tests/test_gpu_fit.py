"""-m gpu: the training driver (smaat_unet_b200.fit) end to end on small seeded synthetic shards.

Precipitation: 37 samples of 13 x 64 x 64 whose target is the last input frame (learnable), batches of 8: the split leaves
34 train samples (four full batches and a tail of 2) and 3 validation samples (one partial batch).  VOC: 19 train and 11
validation uint8 samples of 64 x 64.  Each check compares what the driver reports with an independent computation: the
plain forward of a fresh copy of the trained weights, the step losses the session returned, the indices the loaders read,
and the checkpoint files."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import smaat_unet_b200 as S
from smaat_unet_b200 import data as D
from smaat_unet_b200 import evaluate as E
from smaat_unet_b200 import fit as F
from smaat_unet_b200 import ops
from smaat_unet_b200.train import TrainSession

pytestmark = pytest.mark.gpu

N, T, HW, B, SEED = 37, 13, 64, 8, 5
VAL_TOL = 1e-4          # NET_TOL (tf32x3): the serving forward against the plain forward of the same weights


def make_shard(path, nan_valid_targets=False):
    rng = np.random.default_rng(11)
    a = (rng.random((N, T, HW, HW), dtype=np.float32) ** 3 * np.float32(0.08)).astype(np.float32)
    a[:, -1] = a[:, -2]                                 # the target is the last input frame
    if nan_valid_targets:
        _, valid = F.train_valid_split(N, 0.1, SEED)
        a[valid, -1, 0, 0] = np.nan
    np.save(path, a)
    return path


class Recorder:
    """Wraps TrainSession.step and the shard's read_into: the step sizes, whether each ran a captured graph, the returned
    losses, and every sample index the loaders read, in order."""

    def __init__(self, mp, dataset_cls):
        self.steps, self.reads = [], []
        step, read_into = TrainSession.step, dataset_cls.read_into
        rec = self

        def recording_step(sess, x=None, y=None, aug=None):
            n = int(x.shape[0])
            loss = step(sess, x, y, aug)
            rec.steps.append((n, n in sess._size_graphs, loss.clone()))
            return loss

        def recording_read(ds, index, x_out, y_out):
            rec.reads.append(int(index))
            return read_into(ds, index, x_out, y_out)

        mp.setattr(TrainSession, "step", recording_step)
        mp.setattr(dataset_cls, "read_into", recording_read)


def run_precip(out_dir, rec_cls=D.precipitation_maps_oversampled_shard, shard=None, **kw):
    args = dict(model="UNetDSAttention", train_shard=shard, out_dir=out_dir, batch_size=B, epochs=3, seed=SEED,
                verbose=False)
    args.update(kw)
    with pytest.MonkeyPatch.context() as mp:
        rec = Recorder(mp, rec_cls)
        res = F.fit_precipitation(**args)
    torch.cuda.synchronize()
    return res, rec


@pytest.fixture(scope="module")
def shard(tmp_path_factory):
    return make_shard(tmp_path_factory.mktemp("precip") / "p_train.npy")


@pytest.fixture(scope="module")
def run3(shard, tmp_path_factory):
    out = tmp_path_factory.mktemp("run3")
    res, rec = run_precip(out, shard=shard)
    return res, rec, out


def test_every_sample_once_per_epoch_and_tail_on_its_graph(run3):
    res, rec, _ = run3
    train, valid = res.split
    assert (len(train), len(valid)) == (34, 3)
    assert res.session.sizes == (2, B)
    per_epoch = len(train) + len(valid)
    assert len(rec.reads) == 3 * per_epoch
    for e in range(3):
        chunk = rec.reads[e * per_epoch:(e + 1) * per_epoch]
        assert sorted(chunk[:len(train)]) == sorted(train), e
        assert sorted(chunk[len(train):]) == sorted(valid), e
    orders = [tuple(rec.reads[e * per_epoch:e * per_epoch + len(train)]) for e in range(3)]
    assert len(set(orders)) == 3                        # reshuffled every epoch
    assert [n for n, _, _ in rec.steps] == [B, B, B, B, 2] * 3
    assert all(captured for _, captured, _ in rec.steps)


def test_train_loss_is_the_batch_weighted_mean_of_the_step_losses(run3):
    res, rec, _ = run3
    for e, h in enumerate(res.history):
        steps = rec.steps[5 * e:5 * (e + 1)]
        want = sum(float(loss) * n for n, _, loss in steps) / sum(n for n, _, _ in steps)
        assert h["train_loss"] == pytest.approx(want, rel=1e-6), e
        assert h["train_samples"] == 34 and h["val_samples"] == 3 and h["global_step"] == 5 * (e + 1)


def test_history_file_and_checkpoint_files(run3):
    res, _, out = run3
    with open(os.path.join(out, "history.jsonl")) as f:
        lines = [json.loads(line) for line in f]
    assert [r["epoch"] for r in lines] == [0, 1, 2]
    assert [r["val_loss"] for r in lines] == [h["val_loss"] for h in res.history]
    files = sorted(os.listdir(os.path.join(out, "UNetDSAttention")))
    last = [f for f in files if f.endswith("_last.ckpt")]
    best = [f for f in files if f.endswith(".ckpt") and not f.endswith("_last.ckpt")]
    assert len(last) == 1 and len(best) == 1, files
    h = res.history[-1]
    assert last[0] == F.precip_file_names("UNetDSAttention", 2, h["val_loss"])[1]
    best_epoch = min(range(3), key=lambda e: (res.history[e]["val_loss"], e))
    assert best[0] == F.precip_file_names("UNetDSAttention", best_epoch, res.history[best_epoch]["val_loss"])[0]


def test_learnable_target_trains(run3):
    res, _, _ = run3
    losses = [h["train_loss"] for h in res.history]
    assert losses[-1] < losses[0], losses


def test_validation_equals_a_separate_computation_on_the_trained_weights(run3, shard):
    res, _, _ = run3
    hp = res.hyper_parameters
    copy = F.build_precip_model(hp)
    copy.load_state_dict(F._cpu_state_dict(res.model), strict=True)
    copy = copy.cuda().eval()
    ds = D.precipitation_maps_oversampled_shard(str(shard), 12, 6)
    _, valid = res.split
    x = torch.stack([torch.from_numpy(ds[i][0]) for i in valid]).cuda()
    y = torch.stack([torch.from_numpy(ds[i][1]) for i in valid]).cuda()
    met = S.PrecipitationMetrics(threshold=hp["threshold"])
    with torch.no_grad():
        pred = copy(x)
        loss = float(S.loss_func(pred, y))
        met.update(pred, y)
    ref = met.compute()
    got = res.history[-1]
    assert got["val_loss"] == pytest.approx(loss, rel=VAL_TOL)
    for k in ("mse", "mse_denorm", "mse_pixel"):
        assert got["val_metrics"][k] == pytest.approx(float(ref[k]), rel=VAL_TOL), k
    for k in ("precision", "recall", "accuracy", "f1", "csi", "far", "hss"):
        a, b = got["val_metrics"][k], float(ref[k])
        assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 2e-3, (k, a, b)


def test_checkpoint_serves_bit_for_bit(run3, shard):
    res, _, _ = run3
    loaded = E.load_reference_checkpoint(res.last_path).cuda().eval()
    assert type(loaded) is S.SmaAt_UNet
    x = torch.from_numpy(np.load(shard)[:B, :12].copy()).cuda()
    model = res.model
    try:
        model.eval()
        with torch.no_grad():
            want = model.forward_serving(x).clone()
            got = loaded.forward_serving(x)
    finally:
        model.train()
    assert torch.equal(got, want)
    best = E.load_reference_checkpoint(res.best_path)
    assert type(best) is S.SmaAt_UNet


def test_resume_restores_the_state_at_the_checkpoint(run3, shard, tmp_path):
    res3, rec3, _ = run3
    first, _ = run_precip(tmp_path / "a", shard=shard, epochs=2)
    path = first.last_path
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert ck["epoch"] == 1 and ck["global_step"] == 10

    # resumed with nothing left to run: the session holds exactly the checkpoint's state
    restored, rec = run_precip(tmp_path / "b", shard=shard, epochs=2, resume_from_checkpoint=path)
    assert not restored.history and not rec.steps
    sd = restored.model.state_dict()
    for k, v in ck["state_dict"].items():
        assert torch.equal(sd[k].cpu(), v), k
    opt, want = restored.session.optimizer_state_dict(), ck["optimizer_states"][0]
    for i, st in want["state"].items():
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(opt["state"][i][k].cpu(), st[k]), (i, k)
    h1 = first.history[1]
    assert restored.session.get_lr() == pytest.approx(h1["next_lr"], rel=1e-7)
    cb = ck["callbacks"]["EarlyStopping{'monitor': 'val_loss', 'mode': 'min'}"]
    assert cb["wait_count"] == h1["es_wait_count"]
    assert ck["lr_schedulers"][0]["last_epoch"] == 2

    # resumed for one more epoch: the third epoch's sample order is the uninterrupted run's
    cont, rec = run_precip(tmp_path / "c", shard=shard, epochs=3, resume_from_checkpoint=path)
    assert [h["epoch"] for h in cont.history] == [2] and cont.history[0]["global_step"] == 15
    assert rec.reads[:34] == rec3.reads[2 * 37:2 * 37 + 34]
    assert sorted(rec.reads[34:]) == sorted(rec3.reads[2 * 37 + 34:3 * 37])
    assert os.path.basename(cont.last_path) == F.precip_file_names("UNetDSAttention", 2, cont.history[0]["val_loss"])[1]


def test_nan_validation_stops_at_once_and_plateau_drops_the_lr(tmp_path):
    shard = make_shard(tmp_path / "nan_train.npy", nan_valid_targets=True)
    res, rec = run_precip(tmp_path / "out", shard=shard, epochs=5, lr_patience=0)
    assert len(res.history) == 1 and res.history[0]["stop"]
    h = res.history[0]
    assert np.isnan(h["val_loss"]) and h["lr"] == 1e-3
    assert h["next_lr"] == pytest.approx(1e-4) and res.session.get_lr() == pytest.approx(1e-4)


def test_no_host_synchronisation_in_the_batch_loops(shard, tmp_path):
    res, _ = run_precip(tmp_path / "ok", shard=shard, epochs=1, sync_debug=True)
    assert len(res.history) == 1
    res, _ = run_precip(tmp_path / "captured", shard=shard, epochs=2, sync_debug=True, validation="captured")
    assert len(res.history) == 2
    step = TrainSession.step

    def syncing_step(sess, x=None, y=None, aug=None):
        loss = step(sess, x, y, aug)
        float(loss)                                      # a host read of the loss: waits for the GPU
        return loss

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(TrainSession, "step", syncing_step)
        with pytest.raises(RuntimeError, match="synchroniz"):
            F.fit_precipitation("UNetDSAttention", shard, tmp_path / "bad", batch_size=B, epochs=1, seed=SEED,
                                sync_debug=True, verbose=False)
    assert torch.cuda.get_sync_debug_mode() == 0


def test_captured_validation_matches_serving_validation(shard, tmp_path):
    """Both validation forwards see the same weights: two runs of one epoch with lr = 0 from the same initialisation end
    with the same parameters and running statistics, and the two modes report the same validation loss."""
    outs = {}
    for mode in F.VALIDATION_MODES:
        r, _ = run_precip(tmp_path / mode, shard=shard, epochs=1, learning_rate=0.0, validation=mode)
        outs[mode] = r.history[0]["val_loss"]
    assert outs["captured"] == pytest.approx(outs["serving"], rel=VAL_TOL)


# ------------------------------------------------------------------------------------------------ VOC
def make_voc(prefix, n, seed):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (n, HW, HW, 3), dtype=np.uint8)
    masks = rng.integers(0, 21, (n, HW, HW), dtype=np.uint8)
    masks[:, :4] = 255                                   # the border label, mapped to 0
    np.save(f"{prefix}_images.npy", imgs)
    np.save(f"{prefix}_masks.npy", masks)
    return prefix


@pytest.fixture(scope="module")
def voc_run(tmp_path_factory):
    d = tmp_path_factory.mktemp("voc")
    train, val = make_voc(str(d / "voc_train"), 19, 1), make_voc(str(d / "voc_val"), 11, 2)
    with pytest.MonkeyPatch.context() as mp:
        rec = Recorder(mp, D.voc_segmentation_shard)
        res = F.fit_voc(train, val, d / "out", epochs=2, batch_size=B, seed=SEED, verbose=False)
    torch.cuda.synchronize()
    return res, rec, d, val


def test_voc_samples_steps_and_train_loss(voc_run):
    res, rec, _, _ = voc_run
    assert res.session.sizes == (3, B)
    assert [n for n, _, _ in rec.steps] == [B, B, 3] * 2 and all(c for _, c, _ in rec.steps)
    per_epoch = 19 + 11
    for e in range(2):
        chunk = rec.reads[e * per_epoch:(e + 1) * per_epoch]
        assert sorted(chunk[:19]) == list(range(19)) and chunk[19:] == list(range(11))
        steps = rec.steps[3 * e:3 * (e + 1)]
        assert res.history[e]["train_loss"] == pytest.approx(np.mean([float(loss) for _, _, loss in steps]), rel=1e-6)


def test_voc_validation_equals_a_separate_computation(voc_run):
    res, _, d, val = voc_run
    copy = S.SmaAt_UNet(3, 21)
    copy.load_state_dict(F._cpu_state_dict(res.model), strict=True)
    copy = copy.cuda().eval()
    imgs, masks = np.load(f"{val}_images.npy"), np.load(f"{val}_masks.npy")
    losses, conf = [], np.zeros((21, 21), np.int64)
    with torch.no_grad():
        for i in range(0, 11, B):
            x, y = ops.voc_augment(torch.from_numpy(imgs[i:i + B]).cuda(), torch.from_numpy(masks[i:i + B]).cuda())
            logits = copy(x)
            losses.append(float(TF.cross_entropy(logits, y)))
            pred = logits.argmax(1).cpu().numpy().ravel()
            conf += np.bincount(y.cpu().numpy().ravel() * 21 + pred, minlength=21 * 21).reshape(21, 21)
    tp = np.diag(conf).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        miou = np.nanmean(tp / (tp + conf.sum(0) - tp + conf.sum(1) - tp))
    h = res.history[-1]
    assert h["val_loss"] == pytest.approx(np.mean(losses), rel=VAL_TOL)
    assert abs(h["mIOU"] - miou) <= 2e-3
    names = sorted(os.listdir(d / "out"))
    assert names == ["best_mIoU_model_SmaAt_UNet.pt", "history.jsonl", "model_SmaAt_UNet_epoch_0.pt",
                     "model_SmaAt_UNet_epoch_1.pt"]
    ck = torch.load(d / "out" / "model_SmaAt_UNet_epoch_1.pt", map_location="cpu", weights_only=False)
    assert set(ck) == {"model", "epoch", "state_dict", "optimizer_state_dict", "val_loss", "train_loss", "mIOU"}
    assert ck["epoch"] == 1 and ck["mIOU"] == h["mIOU"] and ck["val_loss"] == h["val_loss"]
    for k, v in copy.state_dict().items():
        assert torch.equal(ck["state_dict"][k], v.cpu()), k
