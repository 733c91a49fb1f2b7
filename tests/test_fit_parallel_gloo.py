"""CPU tests of the data-parallel host logic of the training driver and the evaluator (smaat_unet_b200.fit /
evaluate under torch.distributed): the sharding of train, validation and test indices, the epoch-end reductions, the
decisions every rank must share, rank-0-only writes and the world-size check on resume.  The collective parts run gloo
process groups of 2 and 3 ranks, spawned as tests/test_parallel_gloo.py does; the single-process parts check that without
a process group the host arithmetic and the checkpoint dicts are what they were before data parallelism existed."""
import math
import os
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from smaat_unet_b200 import data as D
from smaat_unet_b200 import fit as F
from smaat_unet_b200 import parallel as P


class _Tiny:
    """A dataset of n one-value samples: enough for PinnedBatchLoader's index logic."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def sample_shapes(self):
        return (1,), (1,)


# ------------------------------------------------------------------------------------------------ sharding
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("n", [0, 1, 2, 5, 7, 17, 34, 37])
def test_disjoint_shards_cover_every_index_exactly_once(world, n):
    order = list(np.random.default_rng(n).permutation(100)[:n])
    shards = [D.shard_indices(order, r, world, disjoint=True) for r in range(world)]
    assert sum(shards, []) == order                      # contiguous, in rank order, nothing padded or dropped
    assert max(map(len, shards)) - min(map(len, shards)) <= 1
    for batch in (1, 2, 4):
        loaders = [D.PinnedBatchLoader(_Tiny(100), batch, indices=order, shuffle=True, seed=3, drop_last=False, rank=r,
                                       world=world, disjoint=True, pin_memory=False) for r in range(world)]
        for epoch in (0, 1):
            for ld in loaders:
                ld.set_epoch(epoch)
            mine = [ld.epoch_indices() for ld in loaders]
            assert sorted(sum(mine, [])) == sorted(order), (batch, epoch)
            assert [len(ld) for ld in loaders] == [-(-len(m) // batch) for m in mine]
            assert [sum(F._EpochLoop._sizes(ld)) for ld in loaders] == [len(m) for m in mine]


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("n", [1, 2, 7, 34, 37, 101])
@pytest.mark.parametrize("batch", [1, 4, 8, 16])
def test_padded_train_shards_step_equal_sizes_on_every_rank(world, n, batch):
    loaders = [D.PinnedBatchLoader(_Tiny(200), batch, indices=range(n), shuffle=True, seed=5, drop_last=False, rank=r,
                                   world=world, pin_memory=False) for r in range(world)]
    for epoch in (0, 3):
        for ld in loaders:
            ld.set_epoch(epoch)
        sizes = [F._EpochLoop._sizes(ld) for ld in loaders]
        assert all(s == sizes[0] for s in sizes), (epoch, sizes)       # same step count and the same tail
        seen = sum((ld.epoch_indices() for ld in loaders), [])
        assert set(seen) == set(range(n)) and len(seen) == -(-n // world) * world


# ------------------------------------------------------------------------------------------------ without a process group
def test_single_process_epoch_values_are_the_former_expressions():
    """What fit computed per epoch before the ranks were reduced: the same float64 values, bit for bit."""
    rng = np.random.default_rng(0)
    for trial in range(50):
        nt, nv, b = int(rng.integers(1, 40)), int(rng.integers(1, 9)), int(rng.integers(1, 17))
        tsz = np.asarray([b] * (nt - 1) + [int(rng.integers(1, b + 1))], np.float64)
        vsz = np.asarray([b] * (nv - 1) + [int(rng.integers(1, b + 1))], np.float64)
        step_losses = rng.random(nt).astype(np.float32) * np.float32(10.0 ** rng.integers(-6, 3))
        val_rows = rng.random((nv, 3)) * 100
        if trial % 7 == 0:
            step_losses[0] = np.nan
        val_losses = (val_rows[:, 0] / vsz).astype(np.float32)
        t_sum, t_n, v_sum, v_n, v_b = P.allreduce_sum(F._weighted_sums(step_losses, tsz) + F._weighted_sums(val_losses, vsz)
                                                      + [len(vsz)])
        old_train = float((step_losses * tsz).sum() / tsz.sum())
        old_val = float((val_losses * vsz).sum() / vsz.sum())
        assert (float(t_sum / t_n), float(v_sum / v_n)) == (old_train, old_val) or math.isnan(old_train)
        assert (int(t_n), int(v_n), int(v_b)) == (int(tsz.sum()), int(vsz.sum()), nv)
        # VOC: plain means of the per-batch losses
        s, c = P.allreduce_sum(F._weighted_sums(step_losses, np.ones(nt)))
        old = float(step_losses.astype(np.float64).mean())
        assert float(s / c) == old or math.isnan(old)


def test_single_process_decisions_and_writes_are_local():
    stopper, plateau = F.EarlyStopping(3), F.PlateauLR(1e-3, "min", patience=0)
    stop = stopper.update(0.5, 0)
    plateau.step(0.5)
    assert F._agree(stop, 0.5, stopper, plateau) == (False, 0.5)
    with F._rank0_writes() as writer:
        assert writer
    assert P.broadcast_from_rank0({"a": 1}) == {"a": 1}
    t = torch.arange(3.0)
    P.broadcast_tensors_([t])
    assert t.tolist() == [0.0, 1.0, 2.0]


def _ckpt(world_size=1):
    hp = F.precip_hyper_parameters(model="UNetDS")
    return F.precip_checkpoint({"w": torch.zeros(2)}, hp, 3, 30, {"state": {}, "param_groups": []}, {}, {"wait_count": 0},
                               0.5, "best.ckpt", {"seed": 0, "samples": 20, "valid_size": 0.1}, world_size=world_size)


def test_single_process_checkpoints_have_no_world_size_key():
    keys = {"epoch", "global_step", "pytorch-lightning_version", "state_dict", "callbacks", "optimizer_states",
            "lr_schedulers", "hparams_name", "hyper_parameters", "split"}
    assert set(_ckpt()) == keys
    assert set(_ckpt(4)) == keys | {"world_size"} and _ckpt(4)["world_size"] == 4
    model = F.SmaAt_UNet(3, 21)
    voc = F.voc_checkpoint(model, 0, {}, 1.0, 1.0, 0.5)
    assert set(voc) == {"model", "epoch", "state_dict", "optimizer_state_dict", "val_loss", "train_loss", "mIOU"}
    assert F.voc_checkpoint(model, 0, {}, 1.0, 1.0, 0.5, world_size=2)["world_size"] == 2


def _shard_and_ckpt(tmp_path, world_size):
    shard = tmp_path / "p_train.npy"
    np.save(shard, np.zeros((20, 13, 64, 64), np.float32))
    path = tmp_path / "UNetDS_rain_threshold_50_epoch=3-val_loss=0.500000_last.ckpt"
    torch.save(_ckpt(world_size), path)
    return str(shard), str(path)


def test_resume_of_a_multi_process_checkpoint_in_one_process_is_refused(tmp_path):
    shard, path = _shard_and_ckpt(tmp_path, 2)
    F.check_resume(_ckpt(2), F.precip_hyper_parameters(model="UNetDS"), 20, world=2)      # the same world is accepted
    with pytest.raises(ValueError, match=r"world size: checkpoint 2, run 1"):
        F.fit_precipitation(model="UNetDS", train_shard=shard, out_dir=str(tmp_path / "out"), resume_from_checkpoint=path,
                            verbose=False)
    assert not (tmp_path / "out").exists()


# ------------------------------------------------------------------------------------------------ gloo process groups
def _worker(rank, world, port, shard, ckpt, out_file, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    P.init_from_env(backend="gloo")
    res = {"rank": rank}
    try:
        # epoch-end reduction: each rank holds its own steps (sizes and losses differ by rank)
        rng = np.random.default_rng(100 + rank)
        tsz = np.asarray([4] * (3 + rank) + [1 + rank], np.float64)
        losses = rng.random(len(tsz)).astype(np.float32)
        t_sum, t_n = P.allreduce_sum(F._weighted_sums(losses, tsz))
        res["train_loss"], res["train_n"] = float(t_sum / t_n), int(t_n)
        res["local"] = (losses.tolist(), tsz.tolist())

        # decisions: local monitored values that disagree on purpose (rank 1 would stop at once on its NaN)
        stopper, plateau = F.EarlyStopping(2), F.PlateauLR(1e-3, "min", patience=0)
        trace = []
        for epoch, base in enumerate([1.0, 0.9, 0.95, 0.97, 0.99]):
            value = float("nan") if (rank == 1 and epoch == 1) else base + 0.01 * rank
            stop = stopper.update(value, epoch)
            plateau.step(value)
            stop, value = F._agree(stop, value, stopper, plateau)
            trace.append((stop, value, stopper.state_dict(), stopper.improved, plateau.lr, plateau.state_dict()))
            if stop:
                break
        res["trace"] = trace

        # rank 0 writes, the others may read once the block is over
        with F._rank0_writes() as writer:
            res["writer"] = writer
            if writer:
                with open(out_file + ".tmp", "w") as f:
                    f.write("x" * 1000)
                time.sleep(0.5)
                os.replace(out_file + ".tmp", out_file)
        with open(out_file) as f:
            res["read"] = len(f.read())

        # buffers take rank 0's values
        bufs = [torch.full((3,), float(rank)), torch.full((2,), rank, dtype=torch.int64)]
        P.broadcast_tensors_(bufs)
        res["buffers"] = [b.tolist() for b in bufs]

        # a single-process checkpoint at world > 1: refused before the session (or any device work) exists
        try:
            F.fit_precipitation(model="UNetDS", train_shard=shard, out_dir=os.path.dirname(ckpt), resume_from_checkpoint=ckpt,
                                verbose=False)
            res["resume"] = None
        except ValueError as e:
            res["resume"] = str(e)
        res["cuda_initialized"] = torch.cuda.is_initialized()
    finally:
        q.put(res)
        torch.distributed.destroy_process_group()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("world", [2, 3])
def test_gloo_reductions_decisions_writes_and_resume(tmp_path, world):
    shard, ckpt = _shard_and_ckpt(tmp_path, 1)
    out_file = str(tmp_path / "written.txt")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000 + 10 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, shard, ckpt, out_file, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted((q.get(timeout=150) for _ in range(world)), key=lambda r: r["rank"])
    [p.join(30) for p in procs]
    assert all(p.exitcode == 0 for p in procs)

    # the reduced train loss is the single-process weighted mean over every rank's steps
    losses = np.concatenate([np.asarray(r["local"][0], np.float32) for r in res])
    sizes = np.concatenate([np.asarray(r["local"][1], np.float64) for r in res])
    want = float((losses * sizes).sum() / sizes.sum())
    for r in res:
        assert r["train_loss"] == pytest.approx(want, rel=1e-12) and r["train_n"] == int(sizes.sum())

    # every rank took rank 0's decisions and state, epoch by epoch, although rank 1's own values said otherwise
    assert all(r["trace"] == res[0]["trace"] for r in res)
    assert [t[1] for t in res[0]["trace"]] == [1.0, 0.9, 0.95, 0.97]                  # rank 0's values; stops at epoch 3
    assert [t[0] for t in res[0]["trace"]] == [False, False, False, True]

    assert [r["writer"] for r in res] == [True] + [False] * (world - 1)
    assert all(r["read"] == 1000 for r in res)
    assert sorted(os.listdir(tmp_path)) == sorted([os.path.basename(shard), os.path.basename(ckpt), "written.txt"])

    assert all(r["buffers"] == [[0.0] * 3, [0] * 2] for r in res)

    for r in res:
        assert r["resume"] is not None and f"world size: checkpoint 1, run {world}" in r["resume"], r["resume"]
        assert not r["cuda_initialized"]
