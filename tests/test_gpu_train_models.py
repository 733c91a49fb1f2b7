"""A captured TrainSession step of every network the project trains, against float64 at its training shape.

test_gpu_train_tail.py part D holds SmaAt_UNet(12, 1, 2) to the float64 port through two captured steps at 288x288.  The
other networks compose the same kernels differently -- an encoder map feeding both a max-pool and a decoder concat (UNetDS),
an un-attended bottleneck that makes the two-phase backward unsound (UNetDSAttention4CBAMs), a conv bias before a
train-mode BatchNorm (UNet, UNetAttention), the transposed-conv upsample into the bucket (bilinear=False) -- and errors of
composition (a gradient contribution dropped or doubled, a gradient in the wrong bucket slot, a cache stale across the
optimizer step, the wrong backward structure) are invisible to the per-kernel files.  Here each row gets part D's
treatment at its own training shape:

  row          model                                           loss           B, H x W    backward
  unet         UNet(12, 1)                                     mse            2, 288^2    one phase (no CBAM)
  unet_convt   UNet(12, 1, bilinear=False)                     mse            2, 288^2    one phase (no CBAM)
  unetatt      UNetAttention(12, 1)                            mse            2, 288^2    two phases
  unetds       UNetDS(12, 1, kernels_per_layer=2)              mse            2, 288^2    one phase (no CBAM)
  unetds4      UNetDSAttention4CBAMs(12, 1, 2)                 mse            2, 288^2    one phase (split rejected by
                                                                                          _verify_split: up1 reads x5 un-attended)
  smaat_convt  SmaAt_UNet(12, 1, 2, bilinear=False)            mse            2, 288^2    two phases
  smaat_voc    SmaAt_UNet(3, 21) (train_SmaAtUNet.py:178)      cross_entropy  8, 224^2    two phases

Every row runs in the tf32x3 pointwise mode (what training runs); unet and unetds also in fp32 (the CUDA-core 3x3 conv,
pw1x1 and weight gradients through a whole captured step).  Two steps per (row, mode), each checked against the float64
port (oracle/dense_oracle.py, oracle/torch_port.py) on the GPU at the parameters and statistics the session held before the
step: the gradient bucket (live parameters to a multiple of the port's own fp32-vs-float64 movement, mathematically-zero
conv biases below 1e-3 max|g|, padding exactly 0), Adam on the session's own gradient and moments, BatchNorm running
statistics and step counters, the logits (through a forward hook on outc, captured with the graph), the loss and the metric
totals.  The conventions and helpers are part D's.  The CPU tests at the end check that each row's parameter schema is the
model's state_dict and that the port reads every parameter, so a key mismatch fails on any machine.

Bounds.  The bucket is held to part D's rule -- every live parameter within F x the port's fp32-vs-float64 movement on its
worst parameter (rel max and rel L2), or NOISE_FLOOR -- with F = NOISE_FACTOR (5) except where the table says otherwise.
Statistics, logits and loss use part D's NOISE_FLOOR / NOISE_FACTOR except the statistics floors named below.  Worst error
observed over both steps and four runs on an H100 80GB HBM3 (700 W power limit); bucket errors in units of the port's
noise (error / max(floor / F, noise)):

  row / mode           bucket (units)     statistics (rel)        logits (rel)        loss vs port (rel)
                       observed / bound   observed / bound        observed / bound    observed / bound
  unet tf32x3          3.3 / 10           2.9e-5 / 1e-4           9.0e-5 / 3e-4       1.3e-6 / 1e-5
  unet_convt tf32x3    3.6 / 10           1.8e-5 / 1e-4           1.4e-5 / 3e-4       1.0e-6 / 1e-5
  unetatt tf32x3       11.5 / 30          1.2e-5 / 1e-4           1.5e-4 / 3e-4       7.5e-7 / 1e-5
  unetds tf32x3        2.2 / 5            2.8e-6 / 2e-5           2.1e-5 / 3e-4       3.7e-8 / 1e-5
  unetds4 tf32x3       6.0 / 15           3.2e-6 / 2e-5           8.1e-5 / 3e-4       2.0e-7 / 1e-5
  smaat_convt tf32x3   2.7 / 5            1.7e-6 / 2e-5           2.4e-5 / 3e-4       1.0e-7 / 1e-5
  smaat_voc tf32x3     2.2 / 5            2.7e-6 / 2e-5           5.4e-5 / 3e-4       2.5e-8 / 1e-5
  unet fp32            2.6 / 5            1.1e-7 / 1e-6           1.3e-5 / 3e-4       9.3e-8 / 1e-5
  unetds fp32          1.1 / 5            9.7e-8 / 1e-6           1.1e-5 / 3e-4       2.2e-8 / 1e-5

The logits and loss floors are part D's, shared by every row; for the rows whose observation is lower they sit more than
10x above it.  Mathematically-zero gradients stay exactly 0 in the dense rows (the conv bias gradient is never written in
train mode) and reach 1.0e-5 max|g| in the DS rows (bound 1e-3); Adam's m', v', p' reach 2.0 / 3.7 / 5.7 units
(part D's bounds 8 / 8 / 16); confusion counts and metric totals are exact.

Why some rows have their own bounds.  Each was localised before it was raised:
  * the dense rows in tf32x3: running statistics up to 2.9e-5 (at up1's first BatchNorm), 200x the port's noise, where
    the same rows in fp32 stay within it; test_gpu_dense_kernels.py measures the 3x3 conv's 3xTF32 BatchNorm sums at 6.2e-5
    from float64 at these layer shapes, ~20x its fp32 error.  Hence the statistics floor 1e-4 (DENSE_TF32X3_STATS); fp32
    mode gets 1e-6 (FP32_STATS) instead of part D's 2e-5;
  * the bucket of UNetAttention in tf32x3 reached 11.5 units (the BatchNorm biases of down1 / down2, then up1's last 3x3
    conv and cbam4's spatial BatchNorm), UNetDSAttention4CBAMs 6.0 (cbam4.spatial_att.bn.weight: a one-element gradient,
    one sum over the whole 36x36 map); in fp32 mode the same rows stay within 3.2 units,
    and so does part D's SmaAt_UNet.  Train-mode BatchNorm over the 18x18 and 36x36 levels amplifies the 3xTF32 kernels'
    error there (20x fp32's in the dense kernel file), and the noise unit itself, one sample of the port's rounding,
    moves 2x between runs.  The dense rows at 3.6 get 10 for the same reason;
  * the unit is the port's noise on its worst parameter, not each parameter's own: on one-element parameters that is a
    single rounding sample, and the ratio of error to it reaches 128 in fp32 mode on these rows and on part D's model.

The port runs in fp32 without cuDNN (im2col + cuBLAS, TF32 off): cuDNN's fp32 algorithms for the dense 3x3 convs at
288x288 take ~15 GiB of workspace.  The whole file runs in ~28 s on one H100 at a peak of 8.4 GiB allocated (smaat_voc;
the 288x288 rows peak at 3.0-5.4 GiB).
"""
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import dense_oracle as D
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from oracle.cases_dense import unet_schema
from smaat_unet_b200 import ops
from tests._util import load_np_state_dict
from tests.test_gpu_train_tail import (CE_LOSS_BOUND, F32_ROUND, NOISE_FACTOR, NOISE_FLOOR, SSE_BOUND, _exact, _rel_l2, _rel_max,  # noqa: F401
                                       ce_ref, check_adam, metric_ref, no_tf32)

gpu = pytest.mark.gpu

# make: the model; schema: its reference-keyed parameter schema; forward(x, sd): the port's train-mode forward;
# split: the backward TrainSession must choose ("two-phase", "none": _find_split finds no CBAM boundary, "rejected": it finds
# one and _verify_split refuses it)
Row = namedtuple("Row", "make schema forward loss B in_shape split seed")
ROWS = {
    "unet": Row(lambda: S.UNet(12, 1), lambda: unet_schema(12, 1),
                lambda x, sd: D.port_unet_forward(x, sd, True), "mse", 2, (12, 288, 288), "none", 301),
    "unet_convt": Row(lambda: S.UNet(12, 1, bilinear=False), lambda: unet_schema(12, 1, bilinear=False),
                      lambda x, sd: D.port_unet_forward(x, sd, True), "mse", 2, (12, 288, 288), "none", 302),
    "unetatt": Row(lambda: S.UNetAttention(12, 1), lambda: unet_schema(12, 1, attention=True),
                   lambda x, sd: D.port_unet_forward(x, sd, True, attention=True), "mse", 2, (12, 288, 288), "two-phase", 303),
    "unetds": Row(lambda: S.UNetDS(12, 1, kernels_per_layer=2), lambda: smaat_unet_schema(12, 1, 2, n_cbams=0),
                  lambda x, sd: TP.smaat_unet_forward(x, sd, True, 0), "mse", 2, (12, 288, 288), "none", 304),
    "unetds4": Row(lambda: S.UNetDSAttention4CBAMs(12, 1, kernels_per_layer=2), lambda: smaat_unet_schema(12, 1, 2, n_cbams=4),
                   lambda x, sd: TP.smaat_unet_forward(x, sd, True, 4), "mse", 2, (12, 288, 288), "rejected", 305),
    "smaat_convt": Row(lambda: S.SmaAt_UNet(12, 1, kernels_per_layer=2, bilinear=False),
                       lambda: smaat_unet_schema(12, 1, 2, bilinear=False),
                       lambda x, sd: TP.smaat_unet_forward(x, sd, True, 5), "mse", 2, (12, 288, 288), "two-phase", 306),
    "smaat_voc": Row(lambda: S.SmaAt_UNet(3, 21), lambda: smaat_unet_schema(3, 21, 2),
                     lambda x, sd: TP.smaat_unet_forward(x, sd, True, 5), "cross_entropy", 8, (3, 224, 224), "two-phase", 307),
}
CASES = [(r, "tf32x3") for r in ROWS] + [("unet", "fp32"), ("unetds", "fp32")]
# Running statistics of the dense rows in tf32x3: the 3x3 conv's 3xTF32 BatchNorm sums sit up to 6.2e-5 off float64 at these
# layer shapes (test_gpu_dense_kernels.py A, bound 3e-4), two orders above the port's fp32 noise; in fp32 mode the same rows'
# statistics are within the port's noise.  The DS rows' pointwise GEMM keeps theirs under NOISE_FLOOR["stats"].
DENSE_TF32X3_STATS = 1e-4
FP32_STATS = 1e-6             # fp32 mode: the session's statistics are as close to float64 as the port's own fp32 run
# Bucket bounds above part D's NOISE_FACTOR, in units of the port's noise on its worst parameter (module docstring)
BUCKET_FACTOR = {("unet", "tf32x3"): 10.0, ("unet_convt", "tf32x3"): 10.0, ("unetatt", "tf32x3"): 30.0, ("unetds4", "tf32x3"): 15.0}


# ==================================================================================================================== GPU
def _port_step(forward, state, x, y, loss_kind, dtype, names):
    """The port's train-mode forward, loss and backward in `dtype` on the GPU at `state` (reference-keyed, float64).
    Returns (loss, logits, {name: grad}, {buffer name: updated running statistic})."""
    sd = {}
    for k, v in state.items():
        if v.dtype == torch.int64:
            sd[k] = v.clone()
        elif k.endswith(("running_mean", "running_var")):
            sd[k] = v.to(dtype).clone()
        else:
            sd[k] = v.to(dtype).clone().requires_grad_(k in names)
    # fp32 runs without cuDNN (im2col + cuBLAS GEMM, TF32 off): cuDNN's fp32 algorithms for the dense 3x3 convs at 288x288
    # allocate ~15 GiB of workspace
    with torch.backends.cudnn.flags(enabled=dtype != torch.float32, benchmark=False, allow_tf32=False):
        out = forward(x.to(dtype), sd)
        if loss_kind == "mse":
            loss = F.mse_loss(out.squeeze(1), y.to(dtype), reduction="sum") / x.shape[0]
        else:
            loss = F.cross_entropy(out, y)
        grads = torch.autograd.grad(loss, [sd[k] for k in names])
    stats = {k: v.detach().double() for k, v in sd.items() if k.endswith(("running_mean", "running_var"))}
    return loss.item(), out.detach().double(), {k: g.double() for k, g in zip(names, grads)}, stats


def _batch(rng, r, K):
    B, (C, H, W) = r.B, r.in_shape
    x = torch.from_numpy(rng.uniform(0, 1, (B, C, H, W))).float().cuda()
    if r.loss == "mse":
        return x, torch.from_numpy(rng.uniform(0, 1, (B, H, W))).float().cuda()
    yn = rng.integers(0, K, (B, H, W))
    yn[rng.random((B, H, W)) < 0.05] = -100
    return x, torch.from_numpy(yn).cuda()


@gpu
@pytest.mark.parametrize("row,mode", CASES, ids=[f"{r}-{m}" for r, m in CASES])
def test_captured_train_step_matches_float64(row, mode, no_tf32):
    old = ops.get_pointwise_mode()
    ops.set_pointwise_mode(mode)
    try:
        _check_session(row, mode)
    finally:
        ops.set_pointwise_mode(old)


def _check_session(row, mode):
    from smaat_unet_b200.train import TrainSession
    r = ROWS[row]
    what = f"{row} {mode}"
    B, (C, H, W) = r.B, r.in_shape
    model = r.make()
    K = model.n_classes
    model = load_np_state_dict(model, cast_sd(fill_schema(r.schema(), r.seed), np.float32)).cuda().train()
    logits = torch.zeros(B, K, H, W, device="cuda")
    calls = [0]

    def keep_logits(mod, inp, out):   # the copy is captured with the graph: each replay leaves its step's logits here
        calls[0] += 1
        logits.copy_(out.detach())

    hook = model.outc.register_forward_hook(keep_logits)
    torch.cuda.reset_peak_memory_stats()
    sess = TrainSession(model, B, r.in_shape, lr=1e-3, use_graph=True, loss=r.loss)
    try:
        # 0  the backward's structure: the cheapest sign of a model taking the wrong path
        split = "two-phase" if sess._split is not None else ("rejected" if sess._find_split() is not None else "none")
        assert split == r.split, (what, split, r.split)
        assert sess.graphs is not None and calls[0] > 0
        names = [k for k, _ in model.named_parameters()]
        params = dict(model.named_parameters())
        spans = {k: (o, params[k].numel()) for k, o in zip(names, sess._offsets)}
        live = torch.zeros(sess.n_flat, dtype=torch.bool, device="cuda")
        for o, n in spans.values():
            live[o:o + n] = True
        rng = np.random.default_rng(r.seed + (0 if mode == "tf32x3" else 1000))
        lr32 = float(np.float32(1e-3))
        for k in (1, 2):
            x, y = _batch(rng, r, K)
            logits.fill_(float("nan"))
            torch.cuda.synchronize()
            P0, M0, V0 = sess.flat_param.clone(), sess.exp_avg.clone(), sess.exp_avg_sq.clone()
            state = {kk: v.detach().double().clone() if v.dtype != torch.int64 else v.clone() for kk, v in model.state_dict().items()}
            for kk in names:                                                     # the parameters as the bucket holds them
                o, n = spans[kk]
                state[kk] = P0[o:o + n].view(params[kk].shape).double()
            tot0 = sess.metrics.totals_snapshot()
            n_calls = calls[0]
            loss = sess.step(x, y)
            torch.cuda.synchronize()
            assert calls[0] == n_calls, "the step ran eagerly, not from the captured graphs"
            assert bool(torch.isfinite(logits).all()), "the hook's copy did not run in the replay"
            G = sess.flat_grad.clone()
            l64, y64, g64, s64 = _port_step(r.forward, state, x, y, r.loss, torch.float64, names)
            l32, y32, g32, s32 = _port_step(r.forward, state, x, y, r.loss, torch.float32, names)

            # 1  the gradient bucket: every parameter within the row's factor x the port's noise on its worst parameter
            gmax = max(g.abs().max().item() for g in g64.values())
            on = [kk for kk in names if g64[kk].abs().max().item() >= 1e-6 * gmax]
            factor = BUCKET_FACTOR.get((row, mode), NOISE_FACTOR)
            worst, bad = {}, []
            for norm, rel in (("max", _rel_max), ("l2", _rel_l2)):
                noise = max(rel(g32[kk], g64[kk]) for kk in on)
                tol = max(NOISE_FLOOR["grad_" + norm], factor * noise)
                errs = {kk: rel(G[spans[kk][0]:sum(spans[kk])].view(params[kk].shape), g64[kk]) for kk in on}
                kk_w = max(errs, key=errs.get)
                worst[norm] = f"{errs[kk_w]:.2e} at {kk_w} (port noise {noise:.2e}, {errs[kk_w] / max(tol / factor, 1e-30):.1f} units)"
                bad += [f"{kk}: rel {norm} {e:.2e} (tol {tol:.1e})" for kk, e in errs.items() if e > tol]
            zero = {kk: G[spans[kk][0]:sum(spans[kk])].abs().max().item() / gmax for kk in names if kk not in on}
            bad += [f"{kk}: {e:.2e} max|g| where the gradient is 0" for kk, e in zero.items() if e > 1e-3]   # bias before a train BN
            print(f"ERR {what} step {k} bucket: rel max {worst['max']}, L2 {worst['l2']} (bound {factor} units); "
                  f"{len(zero)} zero gradients up to {max(zero.values(), default=0.0):.1e} max|g|")
            assert not bad, f"{what} step {k} bucket: " + "; ".join(bad)
            assert not bool(G[~live].any()), "gradient in a padding slot"

            # 2  the optimizer, on the session's own gradient and moments
            check_adam((sess.flat_param, sess.exp_avg, sess.exp_avg_sq), (P0, M0, V0), G, k, lr32, f"{what} step {k}")
            assert float(sess.opt_step) == k
            for buf in (sess.flat_param, sess.exp_avg, sess.exp_avg_sq):
                assert not bool(buf[~live].any()), "padding slot written"

            # 3  BatchNorm running statistics (the port updates them in place) and the step counters
            bufs = dict(model.named_buffers())
            n_st = max(_rel_max(s32[kk], s64[kk]) for kk in s64)
            floor_st = {"fp32": FP32_STATS, "tf32x3": DENSE_TF32X3_STATS if row in ("unet", "unet_convt", "unetatt") else NOISE_FLOOR["stats"]}[mode]
            tol_st = max(floor_st, NOISE_FACTOR * n_st)
            e_st, kk_st = max((_rel_max(bufs[kk], s64[kk]), kk) for kk in s64)
            print(f"ERR {what} step {k} running statistics: rel max {e_st:.2e} at {kk_st} (port noise {n_st:.2e})")
            assert e_st <= tol_st, (what, k, e_st, tol_st)
            counters = [kk for kk in bufs if kk.endswith("num_batches_tracked")]
            assert len(counters) == len(s64) // 2
            for kk in counters:
                assert int(bufs[kk]) == k, kk                                   # the warm-up was rolled back

            # 4  logits, loss and metrics
            n_lg = _rel_max(y32, y64)
            e_lg = _rel_max(logits, y64)
            print(f"ERR {what} step {k} logits: rel max {e_lg:.2e} (port noise {n_lg:.2e})")
            assert e_lg <= max(NOISE_FLOOR["logits"], NOISE_FACTOR * n_lg), (what, k, e_lg, n_lg)
            tot = sess.metrics.totals_snapshot() - tot0
            if r.loss == "mse":
                sse, sse_d, counts = metric_ref(logits.squeeze(1), y, 0.5, True)
                e = abs(float(loss) - sse / B) / (sse / B)
                print(f"ERR {what} step {k} loss against its own logits: {e:.2e}")
                assert e <= SSE_BOUND + F32_ROUND
                t = tot.cpu().tolist()
                assert abs(t[0] - sse / B) <= SSE_BOUND * sse / B and abs(t[1] - sse_d / B) <= SSE_BOUND * sse_d / B
                assert t[2] == B and t[3] == B * H * W and [int(c) for c in t[4:8]] == counts and t[8] == 0
            else:
                rc = ce_ref(logits, y, -100)
                e = abs(float(loss) - rc["loss"] / rc["counted"]) / (rc["loss"] / rc["counted"])
                print(f"ERR {what} step {k} loss against its own logits: {e:.2e}")
                assert e <= CE_LOSS_BOUND + F32_ROUND
                _exact(tot[:K * K].view(K, K), rc["conf"], f"{what} IoU counts step {k}")
                assert int(tot[K * K]) == 0
            e_l, n_l = abs(float(loss) - l64) / abs(l64), abs(l32 - l64) / abs(l64)
            print(f"ERR {what} step {k} loss against the port: {e_l:.2e} (port noise {n_l:.2e})")
            assert e_l <= max(NOISE_FLOOR["loss"], NOISE_FACTOR * n_l), (what, k, e_l, n_l)
        print(f"ERR {what}: peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated")
    finally:
        hook.remove()
        sess.close()


# ==================================================================================================================== CPU
class _Reads(dict):
    """A state_dict that records the keys read from it."""

    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)


@pytest.mark.parametrize("row", list(ROWS))
def test_schema_is_the_models_state_dict(row):
    """Keys and shapes equal; key order equal, except that the schemas list the CBAMs as one block (the order fill_schema
    draws values in, which the golden fixtures depend on) where the models register each after its level."""
    r = ROWS[row]
    schema = r.schema()
    sd = r.make().state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(s) for k, s in schema.items()}
    for part in (lambda k: k.startswith("cbam"), lambda k: not k.startswith("cbam")):
        assert [k for k in schema if part(k)] == [k for k in sd if part(k)]
    if not any(k.startswith("cbam") for k in sd):
        assert list(schema) == list(sd)


@pytest.mark.parametrize("row", list(ROWS))
def test_port_reads_every_parameter(row):
    """One train-mode forward of the port at 32x32 (CPU, fp32) reads every key in named_parameters() and the running
    statistics of every BatchNorm."""
    r = ROWS[row]
    model = r.make()
    sd = _Reads({k: torch.from_numpy(v).float() if v.dtype != np.int64 else torch.from_numpy(v)
                 for k, v in fill_schema(r.schema(), r.seed).items()})
    x = torch.from_numpy(np.random.default_rng(r.seed).uniform(0, 1, (2, r.in_shape[0], 32, 32))).float()
    with torch.no_grad():
        out = r.forward(x, sd)
    assert tuple(out.shape) == (2, model.n_classes, 32, 32)
    names = {k for k, _ in model.named_parameters()}
    assert names <= sd.read, sorted(names - sd.read)
    stats = {k for k, _ in model.named_buffers() if k.endswith(("running_mean", "running_var"))}
    assert stats <= sd.read, sorted(stats - sd.read)
