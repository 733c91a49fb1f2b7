"""-m gpu: the training driver and the test-set evaluator data-parallel over 2 NCCL ranks (one process per GPU, spawned
with torch.multiprocessing), checked against single-process computations.

Precipitation: the 37-sample 13 x 64 x 64 shard of test_gpu_fit.py, batches of 8 per rank.  The split leaves 34 train
samples (17 per rank: steps of 8, 8 and a tail of 1 on both) and 3 validation samples (2 on rank 0, 1 on rank 1).  VOC: 19
train and 11 validation uint8 samples of 64 x 64, batches of 4.  Evaluation: 13 test samples, one with a NaN target,
batches of 4 (one process: 4, 4, 4, 1; two ranks: 4, 3 and 4, 2).

Every test needs two GPUs and is skipped with fewer.  Every spawned process destroys its process group and exits before
the test returns."""
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from smaat_unet_b200 import evaluate as E
from smaat_unet_b200 import fit as F
from smaat_unet_b200 import parallel as P
from smaat_unet_b200.metrics import PrecipitationMetrics, PrecipitationMetricsSweep
from smaat_unet_b200.segmentation import ConfusionMatrix

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(torch.cuda.device_count() < 2,
                                 reason=f"needs 2 GPUs for 2 NCCL ranks; {torch.cuda.device_count()} visible")]

WORLD, N, T, HW, B, SEED = 2, 37, 13, 64, 8, 5


def make_shard(path, n=N, nan_sample=None):
    rng = np.random.default_rng(11)
    a = (rng.random((n, T, HW, HW), dtype=np.float32) ** 3 * np.float32(0.08)).astype(np.float32)
    a[:, -1] = a[:, -2]
    if nan_sample is not None:
        a[nan_sample, -1, 3, 3] = np.nan
    np.save(path, a)
    return str(path)


def make_voc(prefix, n, seed):
    rng = np.random.default_rng(seed)
    np.save(f"{prefix}_images.npy", rng.integers(0, 256, (n, HW, HW, 3), dtype=np.uint8))
    masks = rng.integers(0, 21, (n, HW, HW), dtype=np.uint8)
    masks[:, :4] = 255
    np.save(f"{prefix}_masks.npy", masks)
    return prefix


def untimed(history):
    return [{k: v for k, v in h.items() if not k.endswith("_seconds")} for h in history]


def spawn(target, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + os.getpid() % 2000
    procs = [ctx.Process(target=_entry, args=(target, r, port, args, q)) for r in range(WORLD)]
    [p.start() for p in procs]
    try:
        res = sorted((q.get(timeout=600) for _ in range(WORLD)), key=lambda r: r["rank"])
    finally:
        [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for r in res:
        assert "error" not in r, r["error"]
    return res


def _entry(target, rank, port, args, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(WORLD), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    P.init_from_env("nccl", torch.device("cuda", rank))
    res = {"rank": rank}
    try:
        target(res, *args)
    except BaseException:
        res["error"] = traceback.format_exc()
    finally:
        q.put(res)
        dist.destroy_process_group()


def _record_replicas(sums):
    """Wrap _EpochLoop.run: after every epoch, the all-gathered checksums of the parameters and of the buffers."""
    run = F._EpochLoop.run

    def recording_run(loop, epoch):
        out = run(loop, epoch)
        params = loop.sess.replica_checksums()
        b = torch.cat([t.detach().double().reshape(-1) for t in loop.model.buffers()])
        mine = torch.stack([b.sum(), (b * b).sum()])
        bufs = [torch.zeros_like(mine) for _ in range(WORLD)]
        dist.all_gather(bufs, mine)
        sums.append((params, [x.tolist() for x in bufs]))
        return out

    F._EpochLoop.run = recording_run


def _record_writes(writes):
    replace, append, save = F._replace_file, F._append_history, torch.save

    def rec(fn, tag):
        def wrapped(*a, **kw):
            writes.append(tag)
            return fn(*a, **kw)
        return wrapped

    F._replace_file, F._append_history = rec(replace, "checkpoint"), rec(append, "history")
    F.torch.save = rec(save, "torch.save")


# ------------------------------------------------------------------------------------------------ precipitation
def _precip_worker(res, shard, out):
    sums, writes, samples = [], [], []
    _record_replicas(sums)
    _record_writes(writes)
    compute = PrecipitationMetrics.compute

    def recording_compute(m):
        samples.append((id(m), int(m._totals[2])))
        return compute(m)

    PrecipitationMetrics.compute = recording_compute
    r = F.fit_precipitation(model="UNetDSAttention", train_shard=shard, out_dir=out, batch_size=B, epochs=2, seed=SEED,
                            verbose=False)
    res.update(sums=sums, writes=list(writes), history=r.history, split=r.split, steps=F._EpochLoop._sizes(r.train_loader),
               val_samples=[n for i, n in samples if i != id(r.session.metrics)])
    r2 = F.fit_precipitation(model="UNetDSAttention", train_shard=shard, out_dir=out, batch_size=B, epochs=3, seed=SEED,
                             verbose=False, resume_from_checkpoint=r.last_path)
    res.update(resumed=r2.history, resumed_sums=sums[2:], last=r2.last_path, best=r2.best_path)


def test_fit_precipitation_two_ranks(tmp_path):
    shard = make_shard(tmp_path / "p_train.npy")
    out = str(tmp_path / "out")
    res = spawn(_precip_worker, shard, out)
    r0, r1 = res
    train, valid = r0["split"]
    assert (len(train), len(valid)) == (34, 3)
    assert r0["steps"] == r1["steps"] == [8, 8, 1]
    for params, bufs in r0["sums"] + r0["resumed_sums"]:           # every epoch, both runs: bitwise equal replicas
        assert params[0] == params[1] and bufs[0] == bufs[1], (params, bufs)
    assert len(r0["sums"]) == 3
    assert r0["val_samples"] == r1["val_samples"] == [3, 3]        # each validation sample counted once per epoch
    assert all(h["val_samples"] == 3 and h["train_samples"] == 34 and h["world_size"] == 2 for h in r0["history"])
    assert [h["epoch"] for h in r0["resumed"]] == [2]               # resume at world 2 continues with the next epoch
    assert untimed(r0["history"]) == untimed(r1["history"]) and untimed(r0["resumed"]) == untimed(r1["resumed"])
    assert r1["writes"] == [] and "checkpoint" in r0["writes"] and "history" in r0["writes"]

    files = sorted(os.listdir(os.path.join(out, "UNetDSAttention")))
    last = [f for f in files if f.endswith("_last.ckpt")]
    best = [f for f in files if f.endswith(".ckpt") and not f.endswith("_last.ckpt")]
    assert len(last) == 1 and len(best) == 1 and len(files) == 2, files
    for f in files:
        E.load_reference_checkpoint(os.path.join(out, "UNetDSAttention", f))       # strict=True
    ckpt = torch.load(r0["last"], map_location="cpu", weights_only=False)
    assert ckpt["world_size"] == 2 and ckpt["epoch"] == 2

    # val_loss: one process validating the final weights over the whole validation split
    model = E.load_reference_checkpoint(r0["last"]).cuda()
    a = np.load(shard)
    x, y = torch.from_numpy(a[valid, :12]).cuda(), torch.from_numpy(a[valid, -1]).cuda()
    with torch.no_grad():
        pred = model(x).reshape(y.shape).double()
    want = float(((pred - y.double()) ** 2).sum() / len(valid))
    assert r0["resumed"][-1]["val_loss"] == pytest.approx(want, rel=1e-4)

    with pytest.raises(ValueError, match="world size: checkpoint 2, run 1"):       # resume at world 1
        F.fit_precipitation(model="UNetDSAttention", train_shard=shard, out_dir=out, batch_size=B, epochs=4, seed=SEED,
                            verbose=False, resume_from_checkpoint=r0["last"])


# ------------------------------------------------------------------------------------------------ VOC
def _voc_worker(res, train, val, out):
    sums, writes, pixels = [], [], []
    _record_replicas(sums)
    _record_writes(writes)
    counts = ConfusionMatrix.counts

    def recording_counts(cm):
        conf, invalid = counts(cm)
        pixels.append((int(conf.sum()), invalid))
        return conf, invalid

    ConfusionMatrix.counts = recording_counts
    r = F.fit_voc(train, val, out, epochs=1, batch_size=4, seed=SEED, verbose=False)
    res.update(sums=sums, writes=writes, pixels=pixels, history=r.history)


def test_fit_voc_two_ranks(tmp_path):
    train, val = make_voc(str(tmp_path / "voc_train"), 19, 1), make_voc(str(tmp_path / "voc_val"), 11, 2)
    out = str(tmp_path / "out")
    r0, r1 = spawn(_voc_worker, train, val, out)
    for params, bufs in r0["sums"]:
        assert params[0] == params[1] and bufs[0] == bufs[1], (params, bufs)
    assert r0["pixels"] == r1["pixels"] == [(11 * HW * HW, 0)]      # every validation pixel counted once
    assert untimed(r0["history"]) == untimed(r1["history"]) and r0["history"][0]["val_samples"] == 11
    assert r1["writes"] == [] and r0["writes"].count("torch.save") == 2
    assert sorted(os.listdir(out)) == ["best_mIoU_model_SmaAt_UNet.pt", "history.jsonl", "model_SmaAt_UNet_epoch_0.pt"]


# ------------------------------------------------------------------------------------------------ evaluate
def _record_totals(totals):
    compute = PrecipitationMetricsSweep.compute

    def recording_compute(acc):
        totals.append({t: v.tolist() for t, v in acc.threshold_totals().items()})
        return compute(acc)

    PrecipitationMetricsSweep.compute = recording_compute


def _eval_argv(folder, shard, save):
    return ["--model-folder", folder, "--test-shard", shard, "--thresholds", "0.5", "2.0", "--save-dir", save, "--batch", "4",
            "--file-type", "json"]


def _eval_worker(res, folder, shard, save):
    totals, writes = [], []
    _record_totals(totals)
    save_metrics = E.save_metrics

    def recording_save(*a, **kw):
        writes.append(a[1])
        return save_metrics(*a, **kw)

    E.save_metrics = recording_save
    E.main(_eval_argv(folder, shard, save))
    res.update(totals=totals, writes=writes)


def test_evaluate_two_ranks_equals_one(tmp_path):
    folder = tmp_path / "models"
    folder.mkdir()
    for i, name in enumerate(("UNetDS", "UNetDSAttention")):
        torch.manual_seed(i)
        hp = F.precip_hyper_parameters(model=name)
        net = F.build_precip_model(hp)
        ckpt = F.precip_checkpoint(F._cpu_state_dict(net), hp, 0, 1, {"state": {}, "param_groups": []}, {}, {}, 0.1, "",
                                   {"seed": 0, "samples": 1, "valid_size": 0.1})
        torch.save(ckpt, folder / f"{name}_rain_threshold_50_epoch=0-val_loss=0.100000.ckpt")
    shard = make_shard(tmp_path / "p_test.npy", n=13, nan_sample=5)
    r0, r1 = spawn(_eval_worker, str(folder), shard, str(tmp_path / "two"))
    assert r1["writes"] == [] and len(r0["writes"]) == 2
    assert sorted(os.listdir(tmp_path / "two")) == ["model_metrics_0.5_denorm.json", "model_metrics_2.0_denorm.json"]

    one = []
    with pytest.MonkeyPatch.context() as m:
        compute = PrecipitationMetricsSweep.compute

        def recording_compute(acc):
            one.append({t: v.tolist() for t, v in acc.threshold_totals().items()})
            return compute(acc)

        m.setattr(PrecipitationMetricsSweep, "compute", recording_compute)
        E.main(_eval_argv(str(folder), shard, str(tmp_path / "one")))
    assert len(one) == 3                                            # persistence and the two networks
    for got in (r0["totals"], r1["totals"]):
        assert len(got) == len(one)
        for g, w in zip(got, one):
            for t in (0.5, 2.0):
                assert g[t][2:] == w[t][2:]                          # samples, pixels, TN, FP, FN, TP, skipped: exact
                assert g[t][2] == 12 and g[t][8] == 1
                for k in (0, 1):                                      # squared-error sums: summation order only
                    assert abs(g[t][k] - w[t][k]) <= 1e-12 * abs(w[t][k]), (t, k, g[t][k], w[t][k])
