"""TrainSession -- the training-side public API: one optimisation step of the reference's Lightning loop
(``training_step`` + ``configure_optimizers``: forward, ``loss_func``, metric update, backward, Adam;
reference models/regression_lightning.py:44-78) as a static-shape step captured in CUDA graphs.

    sess = TrainSession(model, batch=32, in_shape=(12, 288, 288), lr=1e-3)
    loss = sess.step(x, y)          # x: (B, 12, H, W), y: (B, H, W); device or pinned-host tensors; returns a 0-dim device tensor
    sess.set_lr(1e-4)               # e.g. from ReduceLROnPlateau (regression_lightning.py:49-55); no re-capture needed
    sess.metrics.compute()          # PrecipitationMetrics over the steps so far

Memory layout.  Parameters, gradients and both Adam moments live in four flat fp32 buffers with one layout (every tensor
starts on a 256-byte boundary): the model's ``nn.Parameter``s are re-pointed into the parameter buffer, ``.grad`` of every
parameter is a view of the gradient buffer, the block backward passes accumulate straight into those views
(functional.add_grad_sinks), and the optimizer step is ONE kernel over the four buffers (csrc/optim.cu) reading the learning
rate from a device scalar.  ``optimizer_state_dict()`` exports torch.optim.Adam's schema (train_SmaAtUNet.py:85-96 saves it).

Data parallelism (SURVEY 8e, BASELINE configs[3]): one process per GPU, each with its own session on its shard of the global
batch.  Replicas start identical (rank 0's parameters and buffers are broadcast at construction, as DDP / Lightning do).
The gradient bucket is all-reduced (average) by NCCL over NVLink in TWO pieces so that the collective overlaps the
backward pass: the decoder's slice (its gradients are final once the backward pass has reached the attention maps) is
reduced on a side stream while the encoder's backward is still running; the encoder's slice follows.  BatchNorm statistics
stay per rank, as in the reference (no SyncBatchNorm).

Segmentation (train_SmaAtUNet.py:139-199): ``loss="cross_entropy"`` trains with ``nn.CrossEntropyLoss()`` semantics instead
of the default ``"mse"``.  The target buffer is then int64 (B, H, W) class indices, the step's loss + gradient + IoU update
is ``segmentation.ce_step`` (one kernel pass), ``metrics`` defaults to ``IoU(K)`` with K the logits' channel count (pass
``metrics=None`` for none), and ``step`` returns the mean cross-entropy over the pixels not labelled -100.  With several
ranks the averaged per-rank mean gradients equal the gradient of the global mean only when every rank counts the same
number of pixels (no ignored or invalid labels, equal shards) -- the same caveat as the MSE path's sum / B_local.

    sess = TrainSession(SmaAt_UNet(3, 21), batch=8, in_shape=(3, 224, 224), loss="cross_entropy")
    loss = sess.step(x, y)          # y: (B, H, W) int64
    iou, miou = sess.metrics.value()
"""
from __future__ import annotations

import weakref

import torch
import torch.distributed as dist

from . import _lib, ops
from . import functional as Fn
from .metrics import PrecipitationMetrics, step_loss
from .modules import CBAM
from .segmentation import IoU, ce_step

_ALIGN = 64          # floats: every parameter starts on a 256-byte boundary of the flat buffers (TMA needs 16)
_DEFAULT = object()  # metrics argument not given: the loss's own default metric


class TrainSession:
    def __init__(self, model, batch, in_shape, lr=1e-3, device=None, use_graph=True, metrics=_DEFAULT, warmup=3,
                 betas=(0.9, 0.999), eps=1e-8, overlap_allreduce=True, recompute_depthwise=False, loss="mse"):
        if loss not in ("mse", "cross_entropy"):
            raise ValueError(f"TrainSession: loss={loss!r}; 'mse' or 'cross_entropy'")
        self.loss_kind = loss
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.model = model.to(self.device).train()
        self.batch, self.in_shape = int(batch), tuple(in_shape)
        self.world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
        self.use_graph = bool(use_graph)
        self.recompute_depthwise = bool(recompute_depthwise)   # functional.set_recompute_depthwise for this session's forwards
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        if self.world > 1:
            # replicas must start identical (what DDP / Lightning do at construction): rank 0's parameters AND buffers
            with torch.no_grad():
                for t in list(self.model.parameters()) + list(self.model.buffers()):
                    dist.broadcast(t, src=0)
        self.params = [p for p in self.model.parameters() if p.requires_grad]
        self._flatten()
        self.x = torch.zeros((self.batch,) + self.in_shape, device=self.device, dtype=torch.float32)
        if loss == "mse":
            self.metrics = metrics if metrics is not None and metrics is not _DEFAULT else PrecipitationMetrics(device=self.device)
            self.y = torch.zeros((self.batch,) + self.in_shape[1:], device=self.device, dtype=torch.float32)
        else:
            self.metrics = IoU(self._n_classes(), device=self.device) if metrics is _DEFAULT else metrics
            self.y = torch.zeros((self.batch,) + self.in_shape[1:], device=self.device, dtype=torch.int64)
        self.loss = torch.zeros((), device=self.device, dtype=torch.float32)
        self.lr = torch.full((), float(lr), device=self.device, dtype=torch.float32)      # device scalar: graphs follow set_lr()
        self.opt_step = torch.zeros((), device=self.device, dtype=torch.float32)          # completed optimizer steps
        self.stream = torch.cuda.Stream(self.device)
        self.comm = torch.cuda.Stream(self.device, priority=-1)       # the early (decoder) all-reduce rides beside the backward
        self._ev_dec = torch.cuda.Event()
        self._ev_comm = torch.cuda.Event()
        # two-phase backward: boundary = the attention maps (outputs of the CBAM children), the decoder's parameters are the
        # tail of the bucket (registration order ... up1..up4, outc) -- else one phase, one all-reduce
        self._split = self._find_split() if overlap_allreduce else None
        self._bnd = []
        self._hooks = []
        if self._split is not None:
            for m in self._split["boundary"]:
                self._hooks.append(m.register_forward_hook(lambda mod, inp, out: self._bnd.append(out)))
        self.graphs = None
        self.launches_per_step = 0
        self.allreduce_events = None        # (start, end) pairs of the last step when record_comm_timing is on
        self.record_comm_timing = False
        self.skip_allreduce = False         # measurement only (bench.py: step time without the collective); replicas diverge
        self._build(warmup)

    def _n_classes(self):
        """Channel count of the model's logits, from one eval-mode forward of a single zero sample (no statistics move)."""
        with torch.no_grad(), torch.cuda.device(self.device):
            self.model.eval()
            try:
                out = self.model(self.x[:1])
            finally:
                self.model.train()
        return int(out.shape[1])

    # ---- flat buffers ------------------------------------------------------------------------------------
    def _flatten(self):
        offs, n = [], 0
        for p in self.params:
            offs.append(n)
            n += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        self.n_flat = n
        self.flat_param = torch.zeros(n, device=self.device, dtype=torch.float32)
        self.flat_grad = torch.zeros(n, device=self.device, dtype=torch.float32)
        self.exp_avg = torch.zeros(n, device=self.device, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(n, device=self.device, dtype=torch.float32)
        self._offsets = offs
        self._views = []
        with torch.no_grad():
            for p, o in zip(self.params, offs):
                v = self.flat_param[o:o + p.numel()].view_as(p)
                v.copy_(p.detach())
                p.data = v                                  # the module's own Parameter now lives in the flat buffer
                gv = self.flat_grad[o:o + p.numel()].view_as(p)
                p.grad = gv
                self._views.append(gv)
        ops.bump_weights_generation()

    def _find_split(self):
        """{'boundary': [CBAM modules], 'tail': first flat offset of the decoder's parameters} or None."""
        kids = list(self.model.named_children())
        cbams = [m for _, m in kids if isinstance(m, CBAM)]
        if not cbams:
            return None
        last = max(i for i, (_, m) in enumerate(kids) if isinstance(m, CBAM))
        dec_ids = {id(p) for _, m in kids[last + 1:] for p in m.parameters()}
        enc_ids = {id(p) for _, m in kids[:last + 1] for p in m.parameters()}
        if not dec_ids or (dec_ids & enc_ids):
            return None
        flags = [id(p) in dec_ids for p in self.params]
        first = flags.index(True)
        if not all(flags[first:]) or any(flags[:first]):
            return None                                     # decoder parameters are not the tail of the bucket
        # every decoder input must be a boundary output or downstream of one: true for the reference's UNet variants with
        # CBAMs on every skip (SmaAt_UNet, UNetDSAttention); UNetDSAttention4CBAMs feeds x5 un-attended -> single phase
        return {"boundary": cbams, "tail": self._offsets[first]}

    # ---- the pieces of a step ----------------------------------------------------------------------------
    def _forward_loss(self):
        self._bnd.clear()
        old = Fn.set_recompute_depthwise(self.recompute_depthwise)
        try:
            pred = self.model(self.x)
        finally:
            Fn.set_recompute_depthwise(old)
        if self.loss_kind == "cross_entropy":
            return ce_step(pred, self.y, self.metrics)    # nn.CrossEntropyLoss + IoU.add in one pass (segmentation.py)
        return step_loss(pred, self.y, self.metrics)      # loss_func + metrics.update in one pass (metrics.py)

    def _phase1(self):
        """Zero the bucket, forward, loss, backward down to the attention maps (all decoder gradients)."""
        self.flat_grad.zero_()
        loss = self._forward_loss()
        self.loss.copy_(loss.detach())
        if self._split is None or not self._bnd or not all(t.requires_grad for t in self._bnd):
            loss.backward()
            self._carry = None
            return
        bnd = list(self._bnd)
        self._bnd.clear()
        grads = torch.autograd.grad(loss, bnd, retain_graph=False, allow_unused=False)
        self._carry = (bnd, grads)

    def _phase2(self):
        """The encoder's backward, from the attention maps' gradients."""
        if self._carry is not None:
            bnd, grads = self._carry
            torch.autograd.backward(bnd, grads)
            self._carry = None

    def _optimise(self):
        lib = _lib.load()
        ops._call("smaat_adam_step", 28 * self.n_flat, 0, lib.smaat_adam_step, self.flat_param.data_ptr(), self.flat_grad.data_ptr(),
                  self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), self.n_flat, self.lr.data_ptr(), self.opt_step.data_ptr(),
                  self.betas[0], self.betas[1], self.eps, ops._stream())

    def _reduce(self, lo, hi, stream):
        """In-place average of flat_grad[lo:hi] over the ranks on `stream`."""
        if self.world == 1 or hi <= lo or self.skip_allreduce:
            return
        with torch.cuda.stream(stream):
            if self.record_comm_timing:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
            dist.all_reduce(self.flat_grad[lo:hi], op=dist.ReduceOp.AVG)
            if self.record_comm_timing:
                e1.record(stream)
                self.allreduce_events.append((e0, e1, (hi - lo) * 4))

    def _snapshot(self):
        return [t.detach().clone() for t in list(self.model.parameters()) + list(self.model.buffers())]

    def _restore(self, snap):
        with torch.no_grad():
            for t, s in zip(list(self.model.parameters()) + list(self.model.buffers()), snap):
                t.copy_(s)
            self.exp_avg.zero_()
            self.exp_avg_sq.zero_()
            self.opt_step.zero_()
        if self.metrics is not None:
            self.metrics.load_totals(self._metrics_snap)  # warm-up must not disturb totals the caller already holds
        ops.bump_weights_generation()

    def _verify_split(self):
        """The two-phase backward assumes that everything the decoder's parameters depend on hangs below the attention maps.
        Checked, not assumed: the same batch and weights through the one-phase backward must give the same bucket (a model
        whose decoder also reads an un-attended encoder map, e.g. UNetDSAttention4CBAMs, fails this and gets one phase)."""
        if self._split is None:
            return
        split, self._split = self._split, None
        self._phase1()                                   # one phase: loss.backward()
        ref = self.flat_grad.clone()
        self._split = split
        self._phase1()
        self._phase2()
        scale = float(ref.abs().max())
        err = float((self.flat_grad - ref).abs().max())
        if not (err <= 1e-3 * max(scale, 1e-30)):        # atomics reorder sums: equal up to fp32 summation noise, or not at all
            self._split = None
            for h in self._hooks:
                h.remove()
            self._hooks = []

    def _eager_step(self):
        self._phase1()
        self._sync_grads_and_phase2(eager=True)
        self._optimise()

    def _sync_grads_and_phase2(self, eager):
        two = self._split is not None and self.world > 1
        tail = self._split["tail"] if self._split is not None else self.n_flat
        if two:
            self._ev_dec.record(self.stream)
            self.comm.wait_event(self._ev_dec)
            self._reduce(tail, self.n_flat, self.comm)           # decoder slice, beside the encoder's backward
        if eager:
            self._phase2()
        else:
            self.graphs[1].replay()
        if two:
            self._reduce(0, tail, self.stream)
            self._ev_comm.record(self.comm)
            self.stream.wait_event(self._ev_comm)
        else:
            self._reduce(0, self.n_flat, self.stream)

    def _build(self, warmup):
        snap = self._snapshot()          # warm-up steps must not change the model the caller handed in
        self._metrics_snap = self.metrics.totals_snapshot() if self.metrics is not None else None
        self._sink_keys = Fn.add_grad_sinks(self.params, self._views)
        weakref.finalize(self, Fn.remove_grad_sinks, self._sink_keys)
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            self.allreduce_events = []
            self._verify_split()
            for _ in range(max(1, warmup)):   # builds caches, sizes the allocator, warms NCCL
                self._eager_step()
            self.stream.synchronize()
            n0 = _lib.launch_count()
            if self.use_graph:
                g1, g2, g3 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(g1, stream=self.stream):
                    self._phase1()
                with torch.cuda.graph(g2, stream=self.stream, pool=g1.pool()):
                    self._phase2()
                with torch.cuda.graph(g3, stream=self.stream, pool=g1.pool()):
                    self._optimise()
                self.graphs = (g1, g2, g3)
            else:
                self._phase1()
                self._phase2()
                self._optimise()
            self.launches_per_step = int(_lib.launch_count() - n0)
            self.stream.synchronize()
        self._restore(snap)
        cur.wait_stream(self.stream)

    # ---- public ------------------------------------------------------------------------------------------
    def set_lr(self, lr: float):
        """Change the learning rate (device scalar read by the captured optimizer kernel)."""
        self.lr.fill_(float(lr))

    def get_lr(self) -> float:
        return float(self.lr)

    def optimizer_state_dict(self):
        """torch.optim.Adam's state_dict schema (what train_SmaAtUNet.py:85-96 checkpoints), built from the flat buffers."""
        state = {}
        for i, (p, o) in enumerate(zip(self.params, self._offsets)):
            n = p.numel()
            state[i] = {"step": self.opt_step.detach().clone(), "exp_avg": self.exp_avg[o:o + n].view_as(p).clone(),
                        "exp_avg_sq": self.exp_avg_sq[o:o + n].view_as(p).clone()}
        group = {"lr": self.get_lr(), "betas": self.betas, "eps": self.eps, "weight_decay": 0, "amsgrad": False, "maximize": False,
                 "foreach": None, "capturable": False, "differentiable": False, "fused": None, "params": list(range(len(self.params)))}
        return {"state": state, "param_groups": [group]}

    def load_optimizer_state_dict(self, sd):
        with torch.no_grad():
            for i, (p, o) in enumerate(zip(self.params, self._offsets)):
                st = sd["state"].get(i)
                if st is None:
                    continue
                n = p.numel()
                self.exp_avg[o:o + n].copy_(st["exp_avg"].reshape(-1))
                self.exp_avg_sq[o:o + n].copy_(st["exp_avg_sq"].reshape(-1))
                self.opt_step.fill_(float(st["step"]))
        self.set_lr(sd["param_groups"][0]["lr"])

    def replica_checksums(self):
        """(sum, sum of squares) of the flat parameter buffer, gathered over the ranks: replicas of a data-parallel run must
        agree exactly (same initial state, same averaged gradients, same optimizer arithmetic)."""
        t = torch.stack([self.flat_param.double().sum(), (self.flat_param.double() ** 2).sum()])
        if self.world == 1:
            return [t.tolist()]
        out = [torch.zeros_like(t) for _ in range(self.world)]
        dist.all_gather(out, t)
        return [o.tolist() for o in out]

    def _stage(self, x, y):
        """Host batch -> device staging slot on the copy stream (overlaps the previous step's compute), then a
        device-to-device copy into the graph's static inputs on the compute stream."""
        if not hasattr(self, "_slots"):
            self.h2d = torch.cuda.Stream(self.device)
            self._slots = [(torch.empty_like(self.x), torch.empty_like(self.y)) for _ in range(2)]
            self._h2d_done = [torch.cuda.Event() for _ in range(2)]
            self._slot_free = [torch.cuda.Event() for _ in range(2)]
            self._n = 0
        i = self._n % 2
        self._n += 1
        sx, sy = self._slots[i]
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(self._slot_free[i])
            sx.copy_(x, non_blocking=True)
            sy.copy_(y.reshape(sy.shape), non_blocking=True)
            self._h2d_done[i].record(self.h2d)
        self.stream.wait_event(self._h2d_done[i])
        self.x.copy_(sx, non_blocking=True)
        self.y.copy_(sy, non_blocking=True)
        self._slot_free[i].record(self.stream)

    def last_h2d_event(self):
        """Event marking the end of the most recent host->device batch copy (None before the first host batch).  Hand it to
        ``PinnedBatchLoader.guard`` so the loader does not overwrite a pinned buffer that is still being copied."""
        if not hasattr(self, "_slots") or self._n == 0:
            return None
        return self._h2d_done[(self._n - 1) % 2]

    def load_batch(self, x, y):
        """Copy a batch into the static input buffers (async).  Host tensors (pinned for true overlap) are staged on a
        separate copy stream so the transfer of step i+1 hides behind the compute of step i."""
        if x.device.type == "cpu":
            self._stage(x, y)
        else:
            self.x.copy_(x, non_blocking=True)
            self.y.copy_(y.reshape(self.y.shape), non_blocking=True)

    def step(self, x=None, y=None):
        """One training step on (x, y) (or on the batch already loaded).  Returns the loss (0-dim device tensor, valid in
        stream order; it is overwritten by the next step)."""
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        if self.record_comm_timing:
            self.allreduce_events = []
        with torch.cuda.stream(self.stream):
            if x is not None:
                self.load_batch(x, y)
            if self.use_graph:
                self.graphs[0].replay()
                self._sync_grads_and_phase2(eager=False)
                self.graphs[2].replay()
            else:
                self._eager_step()
        cur.wait_stream(self.stream)
        ops.bump_weights_generation()    # parameters / running statistics were written by graph replay: no _version bump
        return self.loss

    def close(self):
        """Detach the session from the process-wide gradient sinks (the parameters stay in the flat buffer)."""
        Fn.remove_grad_sinks(self._sink_keys)
        for h in self._hooks:
            h.remove()
