"""-m gpu: the state the Python layer keeps BETWEEN calls, which the kernels read through raw pointers, is never stale and
never freed while something can still read it.

* Weight caches (tf32 hi/lo splits, folded BatchNorm, packed 3x3 and transposed-conv weights) follow every write path.
* A captured InferenceSession graph keeps alive every address it reads, whatever the model does afterwards.
* The CBAM -> Down max-pool stash is taken only for the very tensor the CBAM saw, and never under autograd.

The comparator is a FRESH model: a new instance loaded with the model's state_dict, in eval mode, that never built a cache.
The same kernels on the same inputs and weights give the same bits, so outputs are compared bit for bit: any difference is
a stale or recycled read.  Each family's fresh model is anchored once to the float64 CPU port (NET_TOL)."""
import gc

import pytest
import torch
from torch import nn

import smaat_unet_b200 as S
from oracle import dense_oracle as DO
from oracle import torch_port as TP
from smaat_unet_b200 import functional as Fn
from smaat_unet_b200 import metrics as Mt
from smaat_unet_b200 import ops
from smaat_unet_b200 import segmentation as Sg
from smaat_unet_b200.engine import InferenceSession
from smaat_unet_b200.modules import _TransposedUp, cached_tensors
from smaat_unet_b200.train import TrainSession
from tests._util import NET_TOL, assert_close

pytestmark = pytest.mark.gpu

B, HW = 2, 64
# name -> (constructor, input channels, classes)
FAMILIES = {
    "smaat_12_1": (lambda: S.SmaAt_UNet(12, 1), 12, 1),
    "smaat_3_21_convt": (lambda: S.SmaAt_UNet(3, 21, bilinear=False), 3, 21),
    "unet_12_1": (lambda: S.UNet(12, 1), 12, 1),
    "unet_3_21_convt": (lambda: S.UNet(3, 21, bilinear=False), 3, 21),
    "unetatt_12_1": (lambda: S.UNetAttention(12, 1), 12, 1),
}
NAMES = list(FAMILIES)

# one tensor per cache kind, where the family has it
TARGETS = (
    "inc.double_conv.0.pointwise.weight",      # tf32 split of a DS conv's pointwise weight
    "up2.conv.double_conv.3.pointwise.weight",
    "inc.double_conv.1.running_var",           # folded BatchNorm (DoubleConvDS / DoubleConv)
    "down2.maxpool_conv.1.double_conv.4.running_mean",
    "inc.double_conv.0.weight",                # packed 3x3 weight, slot without a concat
    "up4.conv.double_conv.0.weight",           # packed 3x3 weight, slot of the virtual concat [skip, up]
    "up1.up.weight",                           # packed transposed-conv weight (bilinear=False)
    "cbam1.spatial_att.bn.running_mean",       # folded spatial-attention BatchNorm
)
# caches derived from ONE tensor: a single replaced tensor that lands on the cached address at the cached version hits them
SINGLE_SOURCE = ("inc.double_conv.0.pointwise.weight", "inc.double_conv.0.weight", "up1.up.weight")


def make(name, seed=0):
    """The family's model with default initialisation and random BatchNorm statistics and affines (so that every fold
    matters), on the GPU in eval mode."""
    torch.manual_seed(seed)
    m = FAMILIES[name][0]()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.running_mean.uniform_(-0.2, 0.2, generator=g)
                mod.running_var.uniform_(0.5, 1.5, generator=g)
                mod.weight.uniform_(0.8, 1.2, generator=g)
                mod.bias.uniform_(-0.1, 0.1, generator=g)
    return m.cuda().eval()


def fresh(m, name):
    f = FAMILIES[name][0]()
    f.load_state_dict(m.state_dict())
    return f.cuda().eval()


def inputs(name, seed, batch=B, hw=HW):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(batch, FAMILIES[name][1], hw, hw, device="cuda", generator=g)


def run(m, x, fn=None):
    with torch.no_grad():
        y = (fn or m)(x).clone()
    torch.cuda.synchronize()
    return y


def train_session(m, name, use_graph=True, steps=0, seed=7):
    """A TrainSession on ``m`` (cross-entropy for the multi-class families), after ``steps`` steps on random batches."""
    K = FAMILIES[name][2]
    ts = TrainSession(m, B, (FAMILIES[name][1], HW, HW), lr=1e-2, use_graph=use_graph, loss="cross_entropy" if K > 1 else "mse")
    g = torch.Generator(device="cuda").manual_seed(seed)
    for _ in range(steps):
        x = inputs(name, int(torch.randint(1 << 30, (1,), device="cuda", generator=g)))
        y = (torch.randint(K, (B, HW, HW), device="cuda", generator=g) if K > 1
             else torch.rand(B, HW, HW, device="cuda", generator=g))
        ts.step(x, y)
    torch.cuda.synchronize()
    ts.close()
    return ts


def grow_counters(m, name):
    """An eager forward at a batch larger than the CBAM hand-off counters hold: ``ops._counters`` takes a larger buffer."""
    cur = ops._cbam_counters.get(torch.device("cuda", torch.cuda.current_device()))
    n = max(300, cur.numel() + 1 if cur is not None else 0)
    run(m, inputs(name, 99, batch=n, hw=32))


def blocks():
    """(start, size, state, stream, pool id) of every block the caching allocator holds."""
    out = []
    for seg in torch.cuda.memory_snapshot():
        a, pool = seg["address"], tuple(seg.get("segment_pool_id", (0, 0)))
        for b in seg["blocks"]:
            out.append((a, b["size"], b["state"], seg["stream"], pool))
            a += b["size"]
    return out


def block_of(addr, blks):
    for blk in blks:
        if blk[0] <= addr < blk[0] + blk[1]:
            return blk
    return None


class PtrRecorder:
    """Records every pointer handed to a launch while a CUDA graph is being captured: ``ops._ptr`` and the aliases bound in
    ``functional``, ``segmentation`` and ``metrics``."""

    def __init__(self, monkeypatch):
        self.ptrs = set()
        orig = ops._ptr

        def _ptr(t):
            p = orig(t)
            if p is not None and torch.cuda.is_current_stream_capturing():
                self.ptrs.add(p)
            return p
        for mod in (ops, Fn, Sg, Mt):
            monkeypatch.setattr(mod, "_ptr", _ptr)


def owners(m):
    """(start, end, label) of what a model's graph may read: parameters, buffers, caches, the CBAM counters."""
    out = [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), f"parameter/buffer {n}")
           for n, t in list(m.named_parameters()) + list(m.named_buffers())]
    for mn, mod in m.named_modules():
        if isinstance(mod, _TransposedUp) and mod._packed is not None:
            out += [(t.data_ptr(), t.data_ptr() + t.numel() * 4, f"packed transposed-conv weight of {mn}")
                    for t in [mod._packed[1]] + list(mod._packed[2] or ())]
    out += [(t.data_ptr(), t.data_ptr() + t.numel() * 4, "weight cache") for t in cached_tensors(m)]
    out += [(t.data_ptr(), t.data_ptr() + t.numel() * 4, "CBAM counters") for t in ops._cbam_counters.values()]
    return out


def label(addr, own):
    return next((lab for a, e, lab in own if a <= addr < e), "activation / other")


# ---------------------------------------------------------------------------------------------------------------------
# the comparator against the maths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_fresh_model_matches_float64_port(name):
    m = make(name)
    x = inputs(name, 1)
    y = run(m, x)
    sd = {k: (v.detach().cpu() if v.dtype == torch.int64 else v.detach().cpu().double()) for k, v in m.state_dict().items()}
    xd = x.cpu().double()
    with torch.no_grad():
        if name.startswith("smaat"):
            ref = TP.smaat_unet_forward(xd, sd)
        else:
            ref = DO.port_unet_forward(xd, sd, attention=name.startswith("unetatt"))
    assert_close(y, ref.numpy(), NET_TOL["tf32x3"], f"{name} fresh model vs float64 port")


# ---------------------------------------------------------------------------------------------------------------------
# A. weight caches stay coherent on every write path
# ---------------------------------------------------------------------------------------------------------------------
def targets(m):
    named = dict(m.named_parameters())
    named.update(m.named_buffers())
    return {n: named[n] for n in TARGETS if n in named}


def assign_twice(m):
    """Two load_state_dict(..., assign=True) calls with no forward in between, both replacing the target tensors only (the
    others are passed as aliases).  After the first, the tensors the caches were derived from are no longer the model's;
    the second call's tensors are allocated after that, so where the allocator can hand a cached address out again, one
    of them is put there, at the cached version (value-preserving in-place no-ops set it)."""
    params = dict(m.named_parameters())
    cached = {n: (params[n].data_ptr(), params[n]._version) for n in SINGLE_SOURCE if n in params}
    del params                                       # hold no reference to the original tensors
    sd = m.state_dict()
    for n in list(targets(m)):
        sd[n] = sd[n] * 1.25
    m.load_state_dict(sd, assign=True)
    del sd
    torch.cuda.synchronize()
    blks = blocks()
    plugs, held = [], []
    sd2 = m.state_dict()
    for n, (ptr, ver) in cached.items():
        blk = block_of(ptr, blks)
        if blk is not None and blk[2] == "active_allocated":
            held.append(n)                           # a cache holds its source: nothing can be allocated there
            continue
        vals = sd2[n]
        for _ in range(256):
            t = torch.empty(vals.numel(), device="cuda", dtype=vals.dtype)
            plugs.append(t)
            if t.data_ptr() == ptr:
                t.data.copy_(vals.reshape(-1))       # through .data: the version counter stays at 0
                while t._version < ver:
                    t.add_(0.0)                      # value-preserving in-place no-op: one version step
                sd2[n] = t.view_as(vals)
                break
    m.load_state_dict(sd2, assign=True)
    del sd2
    on_cached = [n for n in cached if (m.get_parameter(n).data_ptr(), m.get_parameter(n)._version) == cached[n]]
    assert held or on_cached, ("precondition: no new tensor landed on a cached address at the cached version, and no cache "
                               f"holds its source ({cached})")


WRITES = ["inplace_no_grad", "detach_copy", "load_state_dict", "train_session_graph", "train_session_eager",
          "train_mode_forward", "assign_twice"]


@pytest.mark.parametrize("write", WRITES)
@pytest.mark.parametrize("name", NAMES)
def test_weight_caches_follow_every_write(name, write):
    m = make(name)
    x = inputs(name, 2)
    y0 = run(m, x)                                   # builds every cache of the eval forward
    if write == "inplace_no_grad":
        with torch.no_grad():
            for t in targets(m).values():
                t.mul_(1.25)
    elif write == "detach_copy":
        for t in targets(m).values():
            t.detach().copy_(t.detach() * 1.25)
    elif write == "load_state_dict":
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        for n in targets(m):
            sd[n] *= 1.25
        m.load_state_dict(sd)
    elif write in ("train_session_graph", "train_session_eager"):
        train_session(m, name, use_graph=write == "train_session_graph", steps=2)
        m.eval()
    elif write == "train_mode_forward":
        m.train()
        run(m, inputs(name, 3) * 2.0)                # running statistics move by raw pointer (no _version bump)
        m.eval()
    elif write == "assign_twice":
        assign_twice(m)
    y1 = run(m, x)
    want = run(fresh(m, name), x)
    assert not torch.equal(y0, want), f"{name} / {write}: the write did not change the output (test is not sensitive)"
    assert torch.equal(y1, want), \
        f"{name} / {write}: eval forward after the write differs from a fresh model (max |diff| {float((y1 - want).abs().max()):.3e})"


@pytest.mark.parametrize("name", NAMES)
def test_weight_caches_follow_pointwise_mode_changes(name):
    m = make(name)
    x = inputs(name, 4)
    run(m, x)
    try:
        for mode in ("tf32", "fp32", "tf32x3"):
            S.set_pointwise_mode(mode)
            y = run(m, x)
            want = run(fresh(m, name), x)
            assert torch.equal(y, want), f"{name}: '{mode}' after the caches were built in another mode differs from a fresh model"
    finally:
        S.set_pointwise_mode("tf32x3")


@pytest.mark.parametrize("name", ["smaat_12_1", "unet_3_21_convt"])
def test_data_writes_are_followed_after_eval(name):
    """``p.data.copy_()`` bumps no version and cannot be seen; the documented remedy is ``model.eval()``."""
    m = make(name)
    x = inputs(name, 5)
    run(m, x)
    for t in targets(m).values():
        t.data.copy_(t.data * 1.25)
    m.eval()
    assert torch.equal(run(m, x), run(fresh(m, name), x))


# ---------------------------------------------------------------------------------------------------------------------
# B. what a captured session points at stays alive
# ---------------------------------------------------------------------------------------------------------------------
def session_output_fn(model, output, fusions):
    """What an InferenceSession(model, output=..., serving_fusions=...) captures, as an eager call."""
    if fusions:
        return {"logits": model.forward_serving, "classes": model.forward_classes, "probs": model.forward_probs}[output]
    return {"logits": model, "classes": lambda x: ops.argmax_channels(model(x)),
            "probs": lambda x: ops.softmax_channels(model(x))}[output]


def _struct_cases():
    out = []
    for name in NAMES:
        outputs = ("logits", "classes", "probs") if FAMILIES[name][2] > 1 else ("logits", "classes")
        for output in outputs:
            for fusions in (True, False):
                out.append((name, output, fusions))
    return out


def disrupt(m, name):
    """Everything a user may do with the model after building a session on it."""
    m.eval()
    m.train()
    run(m, inputs(name, 11))                         # train-mode eager forward: running statistics move
    m.eval()
    run(m, inputs(name, 12))                         # rebuilds the caches
    ts = train_session(m, name)                      # re-points every parameter into the session's flat buffer
    del ts
    m.eval()
    grow_counters(m, name)
    gc.collect()
    torch.cuda.synchronize()


@pytest.mark.parametrize("name,output,fusions", _struct_cases())
def test_session_keeps_alive_every_address_its_graph_reads(name, output, fusions, monkeypatch):
    m = make(name)
    with monkeypatch.context() as mp:
        rec = PtrRecorder(mp)
        sess = InferenceSession(m, B, (FAMILIES[name][1], HW, HW), output=output, serving_fusions=fusions)
    assert sess.graph is not None and rec.ptrs
    own = owners(m)
    pool = tuple(sess.graph.pool())
    blks0 = blocks()
    # the graph's own activations live in its private pool, which the graph keeps reserved for itself
    outside = [p for p in rec.ptrs if (block_of(p, blks0) or (0, 0, "", 0, None))[4] != pool]
    # a block that is freed and handed out again is active at the end: the allocator's free events show it
    torch.cuda.memory._record_memory_history("all", context=None, max_entries=1 << 20, clear_history=True)
    try:
        disrupt(m, name)
        trace = torch.cuda.memory._snapshot()["device_traces"][torch.cuda.current_device()]
    finally:
        torch.cuda.memory._record_memory_history(None)
    freed = [(e["addr"], e["size"]) for e in trace if e["action"] in ("free_requested", "free_completed")]
    blks = blocks()
    stale = []
    for p in sorted(outside):
        blk = block_of(p, blks)
        if blk is None or blk[2] != "active_allocated" or any(a <= p < a + s for a, s in freed):
            stale.append(label(p, own))
    assert not stale, (f"{name} output={output} fusions={fusions}: {len(stale)} of {len(rec.ptrs)} "
                       f"addresses the graph reads were freed: {sorted(set(stale))[:12]}")


@pytest.mark.parametrize("name", ["unet_3_21_convt", "smaat_12_1"])
def test_session_never_replays_onto_recycled_memory(name, monkeypatch):
    """The model moves on after the session was built; every block the graph read that the allocator could hand out again
    is handed out and filled with NaN (int32 counter-sized blocks with 7).  The session's output for a NEW input must still
    be bit for bit the fresh model's at the construction-time weights (TrainSession restores them after its warm-up).
    No kernel of the inference forward uses this data as an index or address: weights and BatchNorm statistics are
    values, and the CBAM counters are only compared with the channel count (a wrong start skips or repeats the MLP)."""
    m = make(name)
    want_model = fresh(m, name)
    with monkeypatch.context() as mp:
        rec = PtrRecorder(mp)
        sess = InferenceSession(m, B, (FAMILIES[name][1], HW, HW))
    counters = [(t.data_ptr(), t.numel() * 4) for t in ops._cbam_counters.values()]
    blks0 = blocks()
    # (start, size, stream, holds the CBAM counters) of every allocator block outside the graph's pool that it reads
    graph_blocks = {(blk[0], blk[1], blk[3], any(blk[0] <= c < blk[0] + blk[1] for c, _ in counters))
                    for blk in (block_of(p, blks0) for p in rec.ptrs) if blk is not None and blk[2] == "active_allocated"}
    sess.forward(inputs(name, 21))                   # the last replay before the refill: a skipped CBAM MLP keeps its gate
    disrupt(m, name)
    blks = blocks()
    fills = []
    cur = torch.cuda.current_stream()
    for start, size, stream, is_counter in sorted(graph_blocks):
        blk = block_of(start, blks)
        if blk is not None and blk[2] == "active_allocated":
            continue
        s = sess.compute if stream == sess.compute.cuda_stream else (cur if stream == cur.cuda_stream else torch.cuda.ExternalStream(stream))
        with torch.cuda.stream(s):
            for _ in range(64):
                t = torch.empty(size // 4, device="cuda", dtype=torch.float32)
                fills.append(t)
                if is_counter:
                    t.view(torch.int32).fill_(7)
                else:
                    t.fill_(float("nan"))
                if t.data_ptr() <= start < t.data_ptr() + size:
                    break
    torch.cuda.synchronize()
    b = inputs(name, 22)
    got = sess.forward(b).clone()
    torch.cuda.synchronize()
    want = run(want_model, b, want_model.forward_serving)
    assert torch.equal(got, want), (f"{name}: the session's output after the model moved on differs from the construction-time "
                                    f"weights' ({int(torch.isnan(got).sum())} NaN, max |diff| {float((got - want).abs().nan_to_num(float('inf')).max()):.3e})")
    del fills


@pytest.mark.parametrize("name", NAMES)
def test_refresh_after_training_equals_fresh_model(name):
    m = make(name)
    x = inputs(name, 30)
    sess = InferenceSession(m, B, (FAMILIES[name][1], HW, HW))
    y0 = sess.forward(x).clone()
    train_session(m, name, steps=2)
    sess.refresh()
    y1 = sess.forward(x).clone()
    f = fresh(m, name)
    want = run(f, x, f.forward_serving)
    assert not torch.equal(y0, want), f"{name}: training did not change the output (test is not sensitive)"
    assert torch.equal(y1, want), f"{name}: refresh() after TrainSession steps differs from a fresh model"


# ---------------------------------------------------------------------------------------------------------------------
# C. the max-pool stash: the very tensor, never under autograd
# ---------------------------------------------------------------------------------------------------------------------
def _blocks_cbam_down(seed=0):
    torch.manual_seed(seed)
    inc = S.DoubleConvDS(12, 64, kernels_per_layer=2).cuda().eval()
    cbam = S.CBAM(64).cuda().eval()
    down = S.DownDS(64, 128, kernels_per_layer=2).cuda().eval()
    return inc, cbam, down


def test_maxpool_stash_is_not_taken_for_a_tensor_on_a_recycled_address():
    _, cbam, down = _blocks_cbam_down()
    inc = S.OutConv(12, 64).cuda().eval()           # a one-kernel producer: its output is its only allocation
    g = torch.Generator(device="cuda").manual_seed(40)
    a, b = (torch.rand(B, 12, 32, 32, device="cuda", generator=g) for _ in range(2))
    with torch.no_grad():
        f = inc(a)
        cbam(f)
        down(f)                                      # builds the weight caches outside the pool below
        del f
        pool = torch.cuda.MemPool()
        with torch.cuda.use_mem_pool(pool):          # a fresh pool: f1 opens its first segment
            f1 = inc(a)
            cbam(f1)                                 # stashes MaxPool2d(2)(f1)
            key, shape = (f1.data_ptr(), f1._version), f1.shape
            del f1
            # every free block the allocator would choose before f1's is plugged, so inc(b)'s output goes to f1's block
            plugs = []
            for _ in range(64):
                t = torch.empty(shape, device="cuda")
                if t.data_ptr() == key[0]:
                    del t
                    break
                plugs.append(t)
            f2 = inc(b)
        try:
            assert (f2.data_ptr(), f2._version) == key, "precondition: f2 sits on f1's block at f1's version"
            got = down(f2)
            want = down(f2.clone())
        finally:
            S.modules._maxpool_stash = None          # no tensor of the pool outlives the test
            del f2, plugs
    assert torch.equal(got, want), "down(f2) took the max-pool the CBAM stashed for the freed f1"


def test_maxpool_stash_is_not_taken_under_autograd():
    inc, cbam, down = _blocks_cbam_down(1)
    down.train()                                     # batch statistics: the gradient does not depend on the running ones
    x0 = torch.rand(B, 64, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(41))

    def grad_of_down(with_cbam):
        x = x0.clone().requires_grad_(True)
        if with_cbam:
            with torch.no_grad():
                cbam(x)                              # stashes a max-pool produced without a tape
        down(x).sum().backward()
        torch.cuda.synchronize()
        return x.grad

    want = grad_of_down(False)
    got = grad_of_down(True)
    assert got is not None, "x.grad is None: down(x) took the no-grad stashed max-pool and cut the gradient path to x"
    assert_close(got, want.double().cpu().numpy(), 1e-5, "dL/dx after a no-grad CBAM call")


def test_maxpool_stash_of_one_model_is_not_taken_by_another():
    """UNetAttention at 128 x 128 leaves cbam5's stash of (B, 512, 8, 8); UNet at 64 x 64 calls down4 on an x4 of that shape."""
    att = make("unetatt_12_1")
    run(att, inputs("unetatt_12_1", 50, hw=128))
    m = make("unet_12_1", seed=3)
    x = inputs("unet_12_1", 51)
    assert torch.equal(run(m, x), run(fresh(m, "unet_12_1"), x))
