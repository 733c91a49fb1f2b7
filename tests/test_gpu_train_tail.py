"""The kernels that run after the backward pass, and one captured TrainSession step, against float64 at the training shapes.

The forward and backward kernels are held to float64 at the 288x288 layer shapes by the other kernel files.  What a
training step does after them -- the optimizer over the flat bucket, the fused loss / metric passes, and the session that
strings the pieces into CUDA graphs -- was only compared with eager torch on the same modules, at small sizes or loose
bounds.  Here:

  A  smaat_adam_step (C ABI) against float64 Adam: the real bucket of TrainSession(SmaAt_UNet(12, 1, 2)) (~4 M floats,
     so every thread of the 8*SMs*256 grid loops), n = 4, and a ragged size just past three grid strides.  Gradient scales
     log-uniform per tensor from 1e-30 to 1e2, parameters with a share at |p| <= 1e-3, non-trivial prior moments,
     completed-step counts 0 .. 1e5, lr 1e-3 / 1e-4 / 0.  One call captured in a CUDA graph and replayed with lr changed
     between replays; elements with g^2 beyond the fp32 range bit-equal to torch.optim.Adam on the GPU
  B  smaat_mse_metrics_fwd + smaat_metrics_commit at B = 32, 288x288 (bench.py's training batch): the squared-error sums
     against float64, the TN/FP/FN/TP counts bit-exact against the reference's fp32 expression with threshold ties
     planted in the 128-bit and the scalar path, the loss gradient bit-equal to torch's fp32 autograd, the NaN guard,
     and the running totals over three batches
  C  smaat_ce_fwd + smaat_confusion_add at the segmentation shapes: (32, 8, 288, 288) (SmaAt_UNet(12, 8), grid-stride
     loop asserted from the launch rule), the VOC shape (8, 21, 224, 224), K = 96 / 97 on both sides of the shared-memory
     histogram limit, K = 1024, K = 2; continuous logits and logits on a 1/4 grid (exact ties among the top logits)
  D  one captured TrainSession step at 288x288, B = 2, twice, against the float64 port (oracle/torch_port.py): the
     gradient bucket, the optimizer (isolated from gradient noise by feeding the reference the session's own gradient),
     BatchNorm running statistics, the logits, the loss and the metric totals; MSE and cross-entropy sessions

Conventions of the references:
  * Adam (adam_ref) is computed in float64 from the fp32 inputs: m' = b1 m + (1 - b1) g, v' = b2 v + (1 - b2) g^2,
    p' = p - lr / (1 - b1^t) * m' / (sqrt(v') / sqrt(1 - b2^t) + eps), t = completed steps + 1, with lr the fp32 value
    the kernel reads.  m' and v' are measured in units of 2^-24 of the magnitude of their terms (b1|m| + (1 - b1)|g|, and
    v' itself: both its terms are >= 0).  p' is allowed 1/2 ulp(p') for its own rounding plus c 2^-24 of the magnitude
    of the update's terms, step_size (b1|m| + (1 - b1)|g|) / denom; that is |dp| except where m' cancels.  Quantities
    in the fp32 subnormal range get one subnormal ulp (2^-149) on top;
  * the metric counts are the reference's own fp32 expression (preds * factor * 12 > threshold, products left to right)
    evaluated by torch on the GPU; the squared-error sums are float64 sums of float64 squares of the fp32 inputs;
  * the cross-entropy reference is float64 log-sum-exp over the fp32 logits, dlogits = softmax - onehot (exactly 0 on
    ignored and invalid pixels), and the confusion matrix is bincount(t K + torch.argmax(fp32 logits)) over the counted
    pixels: torch.argmax returns the first of tied maxima;
  * the session's reference is the port in float64 on the GPU at the parameters and statistics the session held before
    the step; its distance from the port in fp32 (TF32 off) is the reference algorithm's own rounding noise, and the
    gradient, statistic and logit bounds are multiples of that noise, as in test_gpu_api_paths.py's 288x288 check.

Threshold ties.  At the default threshold 0.5 no fp32 value is decided differently by (x * 47.83) * 12 and
x * (47.83 * 12): a scan of 4 000 values around 0.5 / 573.96 finds the two orders differing by one ulp in a third of them,
but never across 0.5.  At 5, 10 and 20 mm/h they do decide differently, so part B runs thresholds 0.5 and 10.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than 10x
above it (everything not listed is bit-exact and was):

  quantity                                                   worst observed                 bound
  A  m', v' (units of 2^-24 of their terms)                  2.0, 3.7                       8, 8
     p' beyond 1/2 ulp (units of 2^-24 of the update)        6.3                            16
  B  sum (p - y)^2, sum (pf - yf)^2 (relative)               1.7e-9                         1e-8
     returned fp32 loss (relative), MSE / cross-entropy      2.2e-8 / 4.3e-8                bound above + 2^-24
  C  loss sum (relative), dlogits (absolute)                 1.8e-7, 2.7e-7                 1e-6, 1e-6
  D  bucket, rel max / rel L2, in units of the port's noise  2.3 / 2.6                      5 (or 2e-3 / 1e-3)
     BatchNorm running statistics (relative)                 3.0e-6                         2e-5 (or 5x noise)
     logits (relative)                                       4.9e-5                         3e-4 (or 5x noise)
     loss against the float64 port (relative)                1.3e-6                         1e-5 (or 5x noise)

The optimizer needs no slack beyond these units: the kernel's (float)(1 - beta2) is within half an ulp of 1 - beta2, while
1.f - (float)beta2 is 1.3e-5 off: ~220 units on every v' that g^2 dominates, and half that on its update.  The session's optimizer check feeds
the reference the session's own gradient and moments and measures the same 2.0 / 3.6 / 5.5 units as the kernel alone.
The whole file runs in ~14 s on one H100 at a peak of 3.8 GiB allocated.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from smaat_unet_b200 import _lib, ops
from smaat_unet_b200.metrics import FACTOR, PrecipitationMetrics, mse_metrics, step_loss
from smaat_unet_b200.segmentation import ce_forward, confusion_add
from tests._util import load_np_state_dict

gpu = pytest.mark.gpu
B1, B2, EPS = 0.9, 0.999, 1e-8
U24 = 2.0 ** -24              # unit of the Adam bounds
SUB = 2.0 ** -149             # one fp32 subnormal ulp
G_OVERFLOW = 2.0 ** 70        # |g| whose square overflows fp32

# bounds (see the module docstring for the observed figures)
ADAM_BOUND = {"m": 8.0, "v": 8.0, "p": 16.0}      # units of 2^-24 (see the conventions)
SSE_BOUND = 1e-8              # relative error of the fp32-partial / fp64-merged squared-error sums
CE_LOSS_BOUND = 1e-6          # relative error of the loss sum
CE_DL_BOUND = 1e-6            # absolute error of dlogits (softmax probabilities, |ref| <= 1)
F32_ROUND = 2.0 ** -24        # the fp32 loss a step returns is its float64 sum / count rounded once more
NOISE_FACTOR = 5.0            # session quantities: at most this x the port's own fp32-vs-fp64 movement ...
NOISE_FLOOR = {"grad_max": 2e-3, "grad_l2": 1e-3, "stats": 2e-5, "logits": 3e-4, "loss": 1e-5}   # ... or these, whichever is larger


# ------------------------------------------------------------------------------------------------------------------ helpers
def _abi(name, *args):
    _lib.check(getattr(_lib.load(), name)(*args), name)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(seed, device="cuda"):
    return torch.Generator(device=device).manual_seed(seed)


def _exact(got, ref, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = got != ref
    n = int(bad.sum())
    print(f"ERR {what}: {n} of {got.numel()} differ (bit-exact)")
    if n:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} values differ, first at {idx}: {got[idx].item()!r} vs {ref[idx].item()!r}")


def _rel_max(a, b):
    a, b = a.double(), b.double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return (a - b).norm().item() / max(b.norm().item(), 1e-30)


@pytest.fixture
def no_tf32():
    """fp32 references on the GPU run in true fp32: cuDNN and cuBLAS TF32 off while the test runs, restored after."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ================================================================================================================ A  Adam
def adam_ref(p, g, m, v, t, lr):
    """One Adam step in float64 from fp32 state (torch.optim.Adam's arithmetic, betas (0.9, 0.999), eps 1e-8).  t: this
    step's number.  Returns (p', m', v', magnitude of m''s terms, magnitude of the update's terms)."""
    p, g, m, v = (a.double() for a in (p, g, m, v))
    m1 = B1 * m + (1.0 - B1) * g
    v1 = B2 * v + (1.0 - B2) * g * g
    step_size = lr / (1.0 - B1 ** t)
    denom = v1.sqrt() / math.sqrt(1.0 - B2 ** t) + EPS
    m_mag = B1 * m.abs() + (1.0 - B1) * g.abs()
    return p - step_size * m1 / denom, m1, v1, m_mag, step_size * m_mag / denom


def _ulp32(x):
    """ulp of the fp32 value nearest to x (float64 in, float64 out)."""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


def adam_errors(got, before, g, t, lr, mask=None):
    """(m', v', p') errors of a kernel step in the units of the module docstring, over the elements in `mask`."""
    p1, m1, v1, m_mag, d_mag = adam_ref(*before[:1], g, *before[1:], t, lr)
    gp, gm, gv = (a.double() for a in got)
    em = (gm - m1).abs() / (U24 * m_mag + SUB)
    ev = (gv - v1).abs() / (U24 * v1 + SUB)
    ep = ((gp - p1).abs() - 0.5 * _ulp32(p1)).clamp_min(0.0) / (U24 * d_mag + SUB)
    if mask is not None:
        em, ev, ep = em[mask], ev[mask], ep[mask]
    return em.max().item(), ev.max().item(), ep.max().item()


def check_adam(got, before, g, t, lr, what, mask=None):
    em, ev, ep = adam_errors(got, before, g, t, lr, mask)
    print(f"ERR adam {what}: m' {em:.2f}  v' {ev:.2f}  p' {ep:.2f} (units of 2^-24; bounds {ADAM_BOUND})")
    assert em <= ADAM_BOUND["m"] and ev <= ADAM_BOUND["v"] and ep <= ADAM_BOUND["p"], (what, em, ev, ep)


def _adam_call(p, g, m, v, lr, step):
    _abi("smaat_adam_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), lr.data_ptr(), step.data_ptr(),
         B1, B2, EPS, ops._stream())


def adam_contents(n, segments, seed, device="cuda"):
    """fp32 (p, g, m, v) of n floats: live data in `segments` [(offset, length)], zero elsewhere (the bucket's padding).
    Per segment (a parameter tensor) one gradient scale, log-uniform in [1e-30, 1e2]; p ~ N(0, 0.05) with a fifth at
    |p| <= 1e-3; m a prior of the gradient's scale; v >= 0 from 0 up to 10 g-scale^2, a tenth exactly 0."""
    gen = _gen(seed, device)
    scale = torch.zeros(n, device=device, dtype=torch.float64)
    live = torch.zeros(n, device=device, dtype=torch.bool)
    logs = torch.rand(len(segments), generator=gen, device=device, dtype=torch.float64) * 32.0 - 30.0
    for (o, k), e in zip(segments, logs.tolist()):
        scale[o:o + k] = 10.0 ** e
        live[o:o + k] = True

    def randn():
        return torch.randn(n, generator=gen, device=device, dtype=torch.float64)

    def rand():
        return torch.rand(n, generator=gen, device=device, dtype=torch.float64)

    p = randn() * 0.05
    p = torch.where(rand() < 0.2, (rand() * 2 - 1) * 1e-3, p)
    g = randn() * scale
    m = randn() * scale * 0.5
    v = (scale * scale) * 10.0 ** (rand() * 9.0 - 8.0)
    v = torch.where(rand() < 0.1, torch.zeros_like(v), v)
    out = [torch.where(live, a, torch.zeros_like(a)).float() for a in (p, g, m, v)]
    return out, live


def _grid_threads():
    return 8 * _sms() * 256          # smaat_adam_step's grid cap x block size


@pytest.fixture(scope="module")
def bucket():
    """The four flat buffers of a TrainSession over SmaAt_UNet(12, 1, kernels_per_layer=2) and the live (offset, length)
    of every parameter in them: the production layout, 64-float slots with zero padding."""
    from smaat_unet_b200.train import TrainSession
    torch.manual_seed(0)
    sess = TrainSession(S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda(), 2, (12, 32, 32), use_graph=False, warmup=1)
    segs = [(o, p.numel()) for p, o in zip(sess.params, sess._offsets)]
    yield sess, segs
    sess.close()


def test_adam_reference_matches_torch_adam_float64():
    """adam_ref, chained over 6 steps with an lr change, against torch.optim.Adam(foreach=False) in float64 on the CPU."""
    gen = torch.Generator().manual_seed(3)
    n = 4096
    p0 = torch.randn(n, generator=gen, dtype=torch.float64)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref], lr=1e-3, foreach=False)
    p, m, v = p0.clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    lr = 1e-3
    for t in range(1, 7):
        if t == 4:
            lr = 1e-4
            opt.param_groups[0]["lr"] = lr
        g = torch.randn(n, generator=gen, dtype=torch.float64) * 10.0 ** (t - 4)
        ref.grad = g.clone()
        opt.step()
        p_new, m, v, _, d_mag = adam_ref(p, g, m, v, t, lr)
        assert ((p_new - p).abs() - d_mag).max() <= 1e-15      # the update's magnitude bounds the update
        p = p_new
        st = opt.state[ref]
        assert (p - ref.detach()).abs().max().item() <= 1e-14 * max(p.abs().max().item(), 1.0)
        for mine, theirs in ((m, st["exp_avg"]), (v, st["exp_avg_sq"])):
            assert (mine - theirs).abs().max().item() <= 1e-14 * theirs.abs().max().item()


def _adam_layouts(bucket):
    sess, segs = bucket
    n_rag = 4 * (_grid_threads() * 3 + 5)
    rag = torch.zeros(4, n_rag, device="cuda")
    return {
        "bucket": ((sess.flat_param, sess.flat_grad, sess.exp_avg, sess.exp_avg_sq), segs),
        "n4": (tuple(torch.zeros(4, 4, device="cuda")), [(0, 4)]),
        "ragged": (tuple(rag), [(o, min(4096, n_rag - o)) for o in range(0, n_rag, 4096)]),
    }


@gpu
@pytest.mark.parametrize("layout", ["bucket", "n4", "ragged"])
def test_adam_step_matches_float64_adam(bucket, layout):
    (p, g, m, v), segs = _adam_layouts(bucket)[layout]
    n = p.numel()
    if layout == "bucket":
        assert n // 4 > _grid_threads(), (n, _grid_threads())         # every thread takes more than one grid-stride pass
    lr_t, step = torch.zeros((), device="cuda"), torch.zeros((), device="cuda")
    seed = 0
    for done in (0, 1, 9, 999, 100000):
        for lr in (1e-3, 1e-4, 0.0):
            seed += 1
            (p0, g0, m0, v0), live = adam_contents(n, segs, seed)
            for dst, src in zip((p, g, m, v), (p0, g0, m0, v0)):
                dst.copy_(src)
            lr_t.fill_(lr)
            step.fill_(float(done))
            _adam_call(p, g, m, v, lr_t, step)
            torch.cuda.synchronize()
            assert float(step) == done + 1
            check_adam((p, m, v), (p0, m0, v0), g0, done + 1, float(np.float32(lr)), f"{layout} t={done + 1} lr={lr}")
            for buf in (p, g, m, v):
                assert not bool(buf[~live].any()), "padding slot written"
            if lr == 0.0:
                _exact(p, p0, f"{layout} lr=0 parameters")
                assert bool((m != m0).any())
                v_term = ((1.0 - B2) * g0.double() ** 2).float()               # 0 where g^2 underflows fp32
                assert bool((v != v0).any()) or not bool(v_term.any())


@gpu
def test_adam_step_captured_in_a_graph_follows_lr_and_step_count():
    """One call captured, replayed 5 times with lr (fill_) and the gradient changed between replays: each replay is one
    float64 Adam step with t = 1..5 and that replay's lr -- bias correction and lr are read on the device."""
    n = 4 * (_grid_threads() + 3)
    (p0, g0, m0, v0), _ = adam_contents(n, [(0, n)], 100)
    p, g, m, v = (a.clone() for a in (p0, g0, m0, v0))
    lr, step = torch.full((), 1e-3, device="cuda"), torch.zeros((), device="cuda")
    _adam_call(p, g, m, v, lr, step)                       # first launch outside the capture
    for dst, src in zip((p, m, v), (p0, m0, v0)):
        dst.copy_(src)
    step.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _adam_call(p, g, m, v, lr, step)
    torch.cuda.synchronize()
    assert float(step) == 0 and torch.equal(p, p0)         # captured, not run
    for k, lr_k in enumerate((1e-3, 3e-4, 1e-4, 0.0, 2e-3), start=1):
        (_, g_new, _, _), _ = adam_contents(n, [(0, n)], 100 + k)
        g.copy_(g_new)
        lr.fill_(lr_k)
        before = (p.clone(), m.clone(), v.clone())
        graph.replay()
        torch.cuda.synchronize()
        assert float(step) == k
        check_adam((p, m, v), before, g, k, float(np.float32(lr_k)), f"graph replay {k}")


@gpu
def test_adam_step_with_overflowing_g_squared_matches_torch_fp32_bitwise():
    """|g| = 2^70: g^2 overflows fp32, v' = inf, the update is 0.  float64 cannot stand in there; torch.optim.Adam
    (single-tensor, fp32 on the GPU) does.  Every other element is held to float64 as usual."""
    n = 4096
    (p0, g0, m0, v0), _ = adam_contents(n, [(0, n)], 7)
    idx = torch.tensor([0, 3, 5, 1000, 2047, 4095], device="cuda")
    g0[idx] = torch.tensor([1.0, -1.0, 1.0, -1.0, 1.0, -1.0], device="cuda") * G_OVERFLOW
    done = 9
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref], lr=1e-3, foreach=False)
    opt.state[ref] = {"step": torch.tensor(float(done)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    ref.grad = g0.clone()
    opt.step()
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    _adam_call(p, g0, m, v, torch.full((), 1e-3, device="cuda"), torch.full((), float(done), device="cuda"))
    torch.cuda.synchronize()
    st = opt.state[ref]
    assert bool(torch.isinf(v[idx]).all())
    _exact(p[idx], ref.detach()[idx], "overflow p'")
    _exact(m[idx], st["exp_avg"][idx], "overflow m'")
    _exact(v[idx], st["exp_avg_sq"][idx], "overflow v'")
    rest = torch.ones(n, dtype=torch.bool, device="cuda")
    rest[idx] = False
    check_adam((p, m, v), (p0, m0, v0), g0, done + 1, float(np.float32(1e-3)), "overflow batch, other elements", rest)


# ================================================================================================== B  MSE loss + metrics
F32_FACTOR = np.float32(FACTOR)


def threshold_products(x, denormalize, order="reference"):
    """fp32 (x * factor) * 12 (the reference's order), x * (factor * 12) (order="folded"), or x * 12."""
    x = np.asarray(x, np.float32)
    if not denormalize:
        return x * np.float32(12)
    if order == "reference":
        return (x * F32_FACTOR) * np.float32(12)
    return x * (F32_FACTOR * np.float32(12))


def threshold_ties(threshold, denormalize, n_scan=4000):
    """fp32 values around threshold / (12 factor) (or threshold / 12) whose product in the reference's order lands within
    two ulp of the threshold: just below, exactly on, just above."""
    thr = np.float32(threshold)
    x0 = np.float32(threshold / (12.0 * float(F32_FACTOR)) if denormalize else threshold / 12.0)
    x = (x0.view(np.int32) + np.arange(-n_scan // 2, n_scan // 2, dtype=np.int32)).view(np.float32)
    d = threshold_products(x, denormalize).view(np.int32) - thr.view(np.int32)
    return x[np.abs(d) <= 2]


@pytest.mark.parametrize("threshold", [0.5, 10.0])
@pytest.mark.parametrize("denormalize", [True, False])
def test_threshold_tie_scan(threshold, denormalize):
    """The planted values really sit on the decision: some land below, on and above the threshold, so `>` and `>=`
    decide differently on some; with the factor and threshold 10 the two product orders decide differently on some, at
    the default threshold 0.5 on none."""
    thr = np.float32(threshold)
    x = threshold_ties(threshold, denormalize)
    a = threshold_products(x, denormalize)
    assert (a < thr).any() and (a == thr).any() and (a > thr).any()
    assert ((a > thr) != (a >= thr)).any()
    if denormalize:
        b = threshold_products(x, True, "folded")
        assert ((a > thr) != (b > thr)).any() == (threshold == 10.0)


B_METRIC, HW = 32, (288, 288)


def precip_batch(B, seed, ties=(), share=0.01):
    """(pred, target): fp32 maps in [0, 1) on the GPU, a share of each planted with the values in `ties`."""
    gen = _gen(seed)
    out = []
    for _ in range(2):
        a = torch.rand((B,) + HW, generator=gen, device="cuda")
        if len(ties):
            tv = torch.from_numpy(np.asarray(ties, np.float32)).cuda()
            pick = torch.rand(a.shape, generator=gen, device="cuda") < share
            which = torch.randint(0, len(tv), a.shape, generator=gen, device="cuda")
            a = torch.where(pick, tv[which], a)
        out.append(a)
    return out


def _unaligned(t):
    """A copy of t that is 4-byte but not 16-byte aligned: the kernel's scalar path."""
    base = torch.empty(t.numel() + 1, device=t.device, dtype=t.dtype)
    v = base[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def metric_ref(pred, target, threshold, denormalize):
    """float64 sum (p - y)^2, sum (p f - y f)^2 and the reference's fp32 TN/FP/FN/TP (torch on the GPU)."""
    p64, y64 = pred.double(), target.double()
    f = float(F32_FACTOR)
    sse = ((p64 - y64) ** 2).sum().item()
    sse_d = ((p64 * f - y64 * f) ** 2).sum().item() if denormalize else sse
    pu, yu = (pred * FACTOR, target * FACTOR) if denormalize else (pred, target)
    pm, tm = (pu * 12 > threshold).view(-1), (yu * 12 > threshold).view(-1)
    counts = torch.bincount(tm.long() * 2 + pm.long(), minlength=4)
    return sse, sse_d, [int(c) for c in counts.tolist()]


def check_batch_acc(acc, pred, target, threshold, denormalize, what):
    sse, sse_d, counts = metric_ref(pred, target, threshold, denormalize)
    a = acc.cpu().tolist()
    e0, e1 = abs(a[0] - sse) / sse, abs(a[1] - sse_d) / sse_d
    print(f"ERR {what}: sse {e0:.2e}  sse_denorm {e1:.2e} (bound {SSE_BOUND:.0e})")
    assert e0 <= SSE_BOUND and e1 <= SSE_BOUND, (what, e0, e1)
    assert a[2] == 0 and a[7] == pred.numel()
    assert [int(c) for c in a[3:7]] == counts, (what, a[3:7], counts)
    return sse, sse_d, counts


@gpu
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("threshold", [0.5, 10.0])
@pytest.mark.parametrize("denormalize", [True, False])
def test_mse_metrics_sums_and_counts_at_b32(denormalize, threshold, aligned):
    ties = threshold_ties(threshold, denormalize)
    pred, target = precip_batch(B_METRIC, 11 + int(threshold), ties)
    if not aligned:
        pred, target = _unaligned(pred), _unaligned(target)
    acc, _ = mse_metrics(pred, target, threshold, denormalize)
    check_batch_acc(acc, pred, target, threshold, denormalize, f"batch sums (denorm={denormalize}, thr={threshold}, aligned={aligned})")
    # the planted ties are in this batch and sit on the decision
    a = torch.from_numpy(threshold_products(pred.cpu().numpy(), denormalize))
    thr = np.float32(threshold)
    assert int((a == float(thr)).sum()) > 100


@gpu
@pytest.mark.parametrize("B", [32, 3])
def test_mse_loss_gradient_is_bitwise_torch_autograd(B):
    """dpred = 2 (p - y) (1 / B): 2 d is exact, so the kernel rounds once, as ATen's mse_loss backward does; 1/3 is not a
    power of two, so B = 3 tests that the scale is rounded the way torch rounds it."""
    pred, target = precip_batch(B, 21)
    p = pred.clone().requires_grad_(True)
    metrics = PrecipitationMetrics(device="cuda")
    loss = step_loss(p, target, metrics)
    loss.backward()
    p2 = pred.clone().requires_grad_(True)
    ref = F.mse_loss(p2, target, reduction="sum") / B
    ref.backward()
    _exact(p.grad, p2.grad, f"dpred B={B}")
    sse, _, _ = metric_ref(pred, target, 0.5, True)
    e = abs(loss.item() - sse / B) / (sse / B)
    print(f"ERR fp32 loss B={B}: {e:.2e}")
    assert e <= SSE_BOUND + F32_ROUND


def _acc_terms(acc, B, denormalize):
    """What smaat_metrics_commit adds for one clean batch, in float64 on the host."""
    a = acc.cpu().double()
    return torch.tensor([a[0] / B, a[1] / B if denormalize else 0.0, float(B), a[7], a[3], a[4], a[5], a[6], 0.0],
                        dtype=torch.float64)


@gpu
@pytest.mark.parametrize("where", ["pred_last", "target_first", "both"])
def test_nan_guard_at_full_size(where):
    """A NaN anywhere drops the whole batch: batch_acc[2] holds the exact count of pixels with a NaN, the totals stay
    bit-unchanged, skipped_batches goes up by one; a clean batch after it adds exactly its own terms."""
    B = B_METRIC
    metrics = PrecipitationMetrics(device="cuda")
    metrics.update(*precip_batch(B, 30))
    before = metrics.totals_snapshot().cpu()
    pred, target = precip_batch(B, 31)
    pf, tf = pred.view(-1), target.view(-1)
    mid = pf.numel() // 2 + 1
    if where in ("pred_last", "both"):
        pf[-1] = math.nan
    if where in ("target_first", "both"):
        tf[0] = math.nan
    if where == "both":
        pf[mid] = math.nan
        tf[mid] = math.nan
    acc, _ = mse_metrics(pred, target, metrics.threshold, metrics.denormalize)
    assert float(acc[2]) == (3 if where == "both" else 1)
    metrics._commit(acc, B)
    after = metrics.totals_snapshot().cpu()
    _exact(after[:8], before[:8], "totals after a NaN batch")
    assert after[8] == before[8] + 1
    clean = precip_batch(B, 32)
    acc2, _ = mse_metrics(*clean, metrics.threshold, metrics.denormalize)
    check_batch_acc(acc2, *clean, metrics.threshold, metrics.denormalize, "clean batch after a NaN batch")
    metrics._commit(acc2, B)
    _exact(metrics.totals_snapshot().cpu(), after + _acc_terms(acc2, B, True), "totals after the clean batch")


@gpu
@pytest.mark.parametrize("denormalize", [True, False])
def test_metric_totals_over_three_batches(denormalize):
    B = B_METRIC
    metrics = PrecipitationMetrics(threshold=0.5, denormalize=denormalize, device="cuda")
    want = np.zeros(8)
    for i in range(3):
        pred, target = precip_batch(B, 40 + i, threshold_ties(0.5, denormalize))
        metrics.update(pred, target)
        sse, sse_d, counts = metric_ref(pred, target, 0.5, denormalize)
        want += [sse / B, sse_d / B if denormalize else 0.0, B, pred.numel()] + counts
    t = metrics.totals_snapshot().cpu().numpy()
    e0 = abs(t[0] - want[0]) / want[0]
    e1 = abs(t[1] - want[1]) / want[1] if denormalize else 0.0
    print(f"ERR totals over 3 batches: loss {e0:.2e}  loss_denorm {e1:.2e}")
    assert e0 <= SSE_BOUND and e1 <= SSE_BOUND
    if not denormalize:
        assert t[1] == 0.0
    assert t[2] == 3 * B and t[3] == 3 * pred.numel() and list(t[4:8]) == list(want[4:8]) and t[8] == 0


# ========================================================================================================= C  cross-entropy
def ce_ref(logits, target, ignore_index):
    """float64 reference of smaat_ce_fwd: dict(loss, counted, invalid, dlogits (float64), conf (K x K int64))."""
    K = logits.shape[1]
    ign = target == ignore_index
    ok = ~ign & (target >= 0) & (target < K)
    l64 = logits.double()
    tt = torch.where(ok, target, torch.zeros_like(target))
    lt = l64.gather(1, tt[:, None])[:, 0]
    loss = (torch.logsumexp(l64, 1) - lt)[ok].sum().item()
    d = torch.softmax(l64, 1)
    d.scatter_add_(1, tt[:, None], -torch.ones_like(lt)[:, None])
    d *= ok[:, None]
    am = logits.argmax(1)
    conf = torch.bincount((target[ok] * K + am[ok]).view(-1), minlength=K * K).view(K, K)
    return {"loss": loss, "counted": int(ok.sum()), "invalid": int((~ign & ~ok).sum()), "dlogits": d, "conf": conf, "ok": ok}


def ce_case(B, K, H, W, kind, ignore_index, invalid, seed, device="cuda"):
    """(fp32 logits, int64 labels): continuous logits in +-4, or logits on a 1/4 grid in [-2, 2] (exact ties among the top
    logits are common); 5 % of the labels ignore_index, with `invalid` another 1 % out of range (K, -1, 1000)."""
    gen = _gen(seed, device)
    if kind == "continuous":
        lg = (torch.rand(B, K, H, W, generator=gen, device=device) * 2 - 1) * 4
    else:
        lg = torch.randint(-8, 9, (B, K, H, W), generator=gen, device=device).float() / 4
    t = torch.randint(0, K, (B, H, W), generator=gen, device=device)
    r = torch.rand(B, H, W, generator=gen, device=device)
    t = torch.where(r < 0.05, torch.full_like(t, ignore_index), t)
    if invalid:
        bad = torch.tensor([K, -1, 1000], device=device)[torch.randint(0, 3, (B, H, W), generator=gen, device=device)]
        t = torch.where((r >= 0.05) & (r < 0.06), bad, t)
    return lg, t


def ce_grid(B, K, P, sms, l2):
    """smaat_ce_fwd's launch rule: (pixel groups, CTAs) of the 128-bit kernel."""
    groups = B * (P // 4)
    cap = min(max(l2 // 2 // (256 * 4 * K * 4), sms), 8 * sms)
    return groups, max(1, min(-(-groups // 256), cap))


def test_ce_reference_matches_cross_entropy_autograd():
    """ce_ref on the CPU against F.cross_entropy + autograd in float64 (invalid labels mapped to ignored), and its confusion
    matrix against a per-pixel first-maximum loop, on quantised logits with ties."""
    K = 5
    lg, t = ce_case(2, K, 6, 7, "quantised", -100, True, 1, device="cpu")
    r = ce_ref(lg, t, -100)
    ok = r["ok"]
    l64 = lg.double().requires_grad_(True)
    want = F.cross_entropy(l64, torch.where(ok, t, torch.full_like(t, -100)), ignore_index=-100, reduction="sum")
    want.backward()
    assert abs(r["loss"] - want.item()) <= 1e-12 * want.item()
    assert torch.allclose(r["dlogits"], l64.grad, rtol=0, atol=1e-15)
    assert r["counted"] == int(ok.sum()) and r["invalid"] == int(((t != -100) & ~ok).sum()) > 0
    conf = torch.zeros(K, K, dtype=torch.int64)
    ties = 0
    for b, y, x in zip(*torch.nonzero(ok, as_tuple=True)):
        col = lg[b, :, y, x]
        first = next(c for c in range(K) if col[c] == col.max())
        ties += int((col == col.max()).sum() > 1)
        conf[t[b, y, x], first] += 1
    assert ties > 0 and torch.equal(conf, r["conf"])


def test_ce_launch_rule_loops_at_the_production_shape():
    """(32, 8, 288, 288) on an H100 (132 SMs, 50 MB L2): 800 CTAs for 663 552 pixel groups, so every thread loops."""
    groups, blocks = ce_grid(32, 8, 288 * 288, 132, 50 << 20)
    assert (groups, blocks) == (663552, 800) and groups > 3 * blocks * 256


# B, K, H, W, ignore_index, invalid labels
CE_SHAPES = [
    (32, 8, 288, 288, -100, True),     # SmaAt_UNet(12, 8) on the classification data: the grid-stride production launch
    (8, 21, 224, 224, 255, False),     # the VOC shape of tools/bench_seg.py
    (4, 96, 96, 96, 255, False),       # the largest K with the shared-memory histogram
    (4, 97, 96, 96, -100, False),      # the smallest K with the global-atomic histogram
    (2, 1024, 12, 20, -100, False),    # the largest K the kernel takes
    (32, 2, 288, 288, 255, False),
]


@gpu
@pytest.mark.parametrize("kind", ["continuous", "quantised"])
@pytest.mark.parametrize("shape", CE_SHAPES, ids=lambda s: "x".join(map(str, s[:4])))
def test_ce_fwd_matches_float64_at_segmentation_shapes(shape, kind):
    B, K, H, W, ig, invalid = shape
    if (B, K) == (32, 8):
        groups, blocks = ce_grid(B, K, H * W, _sms(), torch.cuda.get_device_properties(0).L2_cache_size)
        assert groups > blocks * 256, (groups, blocks)                # every thread takes more than one grid-stride pass
    lg, t = ce_case(B, K, H, W, kind, ig, invalid, seed=K * 7 + H)
    r = ce_ref(lg, t, ig)
    if kind == "quantised":
        top2 = lg.topk(2, dim=1).values
        assert float((top2[:, 0] == top2[:, 1]).float().mean()) > 0.02   # ties among the top logits are common
    conf0 = torch.randint(0, 50, (K, K), generator=_gen(9), device="cuda")
    conf = conf0.clone()
    acc, dl = ce_forward(lg, t, ig, True, want_grad=True, conf=conf)
    a = acc.cpu().tolist()
    e_loss = abs(a[0] - r["loss"]) / r["loss"]
    e_dl = (dl.double() - r["dlogits"]).abs().max().item()
    print(f"ERR ce {shape} {kind}: loss {e_loss:.2e} (bound {CE_LOSS_BOUND:.0e})  dlogits {e_dl:.2e} (bound {CE_DL_BOUND:.0e})")
    assert e_loss <= CE_LOSS_BOUND and e_dl <= CE_DL_BOUND
    assert int(a[1]) == r["counted"] and int(a[2]) == r["invalid"] and (r["invalid"] > 0) == invalid
    assert not bool(dl.permute(0, 2, 3, 1)[~r["ok"]].any())           # exactly 0 on ignored and invalid pixels
    _exact(conf - conf0, r["conf"], f"confusion {shape} {kind}")
    conf2 = conf0.clone()
    acc2, dl2 = ce_forward(lg, t, ig, True, want_grad=True, conf=conf2)
    _exact(dl2, dl, "dlogits, second call")
    _exact(conf2, conf, "confusion, second call")
    assert acc2.cpu().tolist()[1:] == a[1:]


@gpu
@pytest.mark.parametrize("K", [8, 150])
def test_confusion_add_at_full_size(K):
    n = B_METRIC * HW[0] * HW[1]
    gen = _gen(K)
    pred = torch.randint(0, K, (n,), generator=gen, device="cuda")
    target = torch.randint(0, K, (n,), generator=gen, device="cuda")
    bad_vals = torch.tensor([-1, K, 1000], device="cuda")
    for a in (pred, target):
        pick = torch.rand(n, generator=gen, device="cuda") < 0.01
        a.copy_(torch.where(pick, bad_vals[torch.randint(0, 3, (n,), generator=gen, device="cuda")], a))
    conf0 = torch.randint(0, 50, (K, K), generator=gen, device="cuda")
    conf, inv = conf0.clone(), torch.full((1,), 7, dtype=torch.int64, device="cuda")
    confusion_add(pred, target, conf, inv, K)
    ok = (pred >= 0) & (pred < K) & (target >= 0) & (target < K)
    _exact(conf - conf0, torch.bincount(target[ok] * K + pred[ok], minlength=K * K).view(K, K), f"confusion_add K={K}")
    assert int(inv) - 7 == int((~ok).sum()) > 0


# ===================================================================================================== D  TrainSession step
SESSION_B, SESSION_HW = 2, (288, 288)


def _port_step(state, x, y, loss_kind, dtype, names):
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
    out = TP.smaat_unet_forward(x.to(dtype), sd, True)
    if loss_kind == "mse":
        loss = F.mse_loss(out.squeeze(1), y.to(dtype), reduction="sum") / x.shape[0]
    else:
        loss = F.cross_entropy(out, y)
    grads = torch.autograd.grad(loss, [sd[k] for k in names])
    stats = {k: v.detach().double() for k, v in sd.items() if k.endswith(("running_mean", "running_var"))}
    return loss.item(), out.detach().double(), {k: g.double() for k, g in zip(names, grads)}, stats


@gpu
@pytest.mark.parametrize("loss_kind", ["mse", "cross_entropy"])
def test_captured_train_session_step_matches_float64(loss_kind, no_tf32):
    from smaat_unet_b200.train import TrainSession
    B, (H, W) = SESSION_B, SESSION_HW
    K = 1 if loss_kind == "mse" else 8
    sd_np = fill_schema(smaat_unet_schema(12, K, 2), 12)
    model = load_np_state_dict(S.SmaAt_UNet(12, K, kernels_per_layer=2), cast_sd(sd_np, np.float32)).cuda().train()
    logits = torch.zeros(B, K, H, W, device="cuda")

    def keep_logits(mod, inp, out):   # the copy is captured with the graph: each replay leaves its step's logits here
        logits.copy_(out.detach())

    hook = model.outc.register_forward_hook(keep_logits)
    sess = TrainSession(model, B, (12, H, W), lr=1e-3, use_graph=True, loss=loss_kind)
    assert sess._split is not None and sess.graphs is not None                 # two-phase backward, replayed graphs
    names = [k for k, _ in model.named_parameters()]
    params = dict(model.named_parameters())
    spans = {k: (o, params[k].numel()) for k, o in zip(names, sess._offsets)}
    live = torch.zeros(sess.n_flat, dtype=torch.bool, device="cuda")
    for o, n in spans.values():
        live[o:o + n] = True
    rng = np.random.default_rng(5 if loss_kind == "mse" else 6)
    lr32 = float(np.float32(1e-3))
    for k in (1, 2):
        x = torch.from_numpy(rng.uniform(0, 1, (B, 12, H, W))).float().cuda()
        if loss_kind == "mse":
            y = torch.from_numpy(rng.uniform(0, 1, (B, H, W))).float().cuda()
        else:
            yn = rng.integers(0, K, (B, H, W))
            yn[rng.random((B, H, W)) < 0.05] = -100
            y = torch.from_numpy(yn).cuda()
        torch.cuda.synchronize()
        P0, M0, V0 = sess.flat_param.clone(), sess.exp_avg.clone(), sess.exp_avg_sq.clone()
        state = {kk: v.detach().double().clone() if v.dtype != torch.int64 else v.clone() for kk, v in model.state_dict().items()}
        for kk in names:                                                         # the parameters as the bucket holds them
            o, n = spans[kk]
            state[kk] = P0[o:o + n].view(params[kk].shape).double()
        tot0 = sess.metrics.totals_snapshot()
        loss = sess.step(x, y)
        torch.cuda.synchronize()
        G = sess.flat_grad.clone()
        l64, y64, g64, s64 = _port_step(state, x, y, loss_kind, torch.float64, names)
        l32, y32, g32, s32 = _port_step(state, x, y, loss_kind, torch.float32, names)

        # 1  the gradient bucket
        gmax = max(g.abs().max().item() for g in g64.values())
        on = [kk for kk in names if g64[kk].abs().max().item() >= 1e-6 * gmax]
        n_max = max(_rel_max(g32[kk], g64[kk]) for kk in on)
        n_l2 = max(_rel_l2(g32[kk], g64[kk]) for kk in on)
        tol_max = max(NOISE_FLOOR["grad_max"], NOISE_FACTOR * n_max)
        tol_l2 = max(NOISE_FLOOR["grad_l2"], NOISE_FACTOR * n_l2)
        worst_max = worst_l2 = 0.0
        for kk in names:
            o, n = spans[kk]
            got = G[o:o + n].view(params[kk].shape)
            if kk not in on:                  # mathematically zero (bias before a train-mode BatchNorm): summation noise only
                assert got.abs().max().item() <= 1e-3 * gmax, kk
                continue
            e_max, e_l2 = _rel_max(got, g64[kk]), _rel_l2(got, g64[kk])
            worst_max, worst_l2 = max(worst_max, e_max), max(worst_l2, e_l2)
            assert e_max <= tol_max and e_l2 <= tol_l2, f"step {k} bucket {kk}: rel max {e_max:.2e} (tol {tol_max:.1e}), L2 {e_l2:.2e} (tol {tol_l2:.1e})"
        print(f"ERR session {loss_kind} step {k} bucket: rel max {worst_max:.2e} (port noise {n_max:.2e}), "
              f"L2 {worst_l2:.2e} (port noise {n_l2:.2e})")
        assert not bool(G[~live].any()), "gradient in a padding slot"

        # 2  the optimizer, on the session's own gradient and moments
        check_adam((sess.flat_param, sess.exp_avg, sess.exp_avg_sq), (P0, M0, V0), G, k, lr32, f"session {loss_kind} step {k}")
        assert float(sess.opt_step) == k
        for buf in (sess.flat_param, sess.exp_avg, sess.exp_avg_sq):
            assert not bool(buf[~live].any()), "padding slot written"

        # 3  BatchNorm running statistics (the port updates them in place) and the step counters
        bufs = dict(model.named_buffers())
        n_st = max(_rel_max(s32[kk], s64[kk]) for kk in s64)
        tol_st = max(NOISE_FLOOR["stats"], NOISE_FACTOR * n_st)
        e_st = max(_rel_max(bufs[kk], s64[kk]) for kk in s64)
        print(f"ERR session {loss_kind} step {k} running statistics: rel max {e_st:.2e} (port noise {n_st:.2e})")
        assert e_st <= tol_st, (k, e_st, tol_st)
        for kk, v in bufs.items():
            if kk.endswith("num_batches_tracked"):
                assert int(v) == k, kk                                          # the warm-up was rolled back

        # 4  logits, loss and metrics
        n_lg = _rel_max(y32, y64)
        e_lg = _rel_max(logits, y64)
        print(f"ERR session {loss_kind} step {k} logits: rel max {e_lg:.2e} (port noise {n_lg:.2e})")
        assert e_lg <= max(NOISE_FLOOR["logits"], NOISE_FACTOR * n_lg)
        tot = sess.metrics.totals_snapshot() - tot0
        if loss_kind == "mse":
            sse, sse_d, counts = metric_ref(logits.squeeze(1), y, 0.5, True)
            e = abs(float(loss) - sse / B) / (sse / B)
            print(f"ERR session {loss_kind} step {k} loss against its own logits: {e:.2e}")
            assert e <= SSE_BOUND + F32_ROUND
            t = tot.cpu().tolist()
            assert abs(t[0] - sse / B) <= SSE_BOUND * sse / B and abs(t[1] - sse_d / B) <= SSE_BOUND * sse_d / B
            assert t[2] == B and t[3] == B * H * W and [int(c) for c in t[4:8]] == counts and t[8] == 0
        else:
            r = ce_ref(logits, y, -100)
            e = abs(float(loss) - r["loss"] / r["counted"]) / (r["loss"] / r["counted"])
            print(f"ERR session {loss_kind} step {k} loss against its own logits: {e:.2e}")
            assert e <= CE_LOSS_BOUND + F32_ROUND
            _exact(tot[:K * K].view(K, K), r["conf"], f"session IoU counts step {k}")
            assert int(tot[K * K]) == 0
        e_l, n_l = abs(float(loss) - l64) / abs(l64), abs(l32 - l64) / abs(l64)
        print(f"ERR session {loss_kind} step {k} loss against the port: {e_l:.2e} (port noise {n_l:.2e})")
        assert e_l <= max(NOISE_FLOOR["loss"], NOISE_FACTOR * n_l)
    hook.remove()
    sess.close()
