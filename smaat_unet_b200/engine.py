"""InferenceSession -- the serving-side public API: a static-shape eval forward captured once
in a CUDA graph (~90 kernel launches -> one graph launch) with pinned-host, double-buffered,
stream-overlapped input/output staging.

    sess = InferenceSession(model, batch=32, in_shape=(12, 288, 288))
    y_dev = sess.forward(x_dev)                  # device-resident input
    sess.submit(x_host_pinned); ...; y = sess.collect()   # host buffers, H2D/D2H overlapped with compute

A request may carry fewer rows than ``batch``: it runs the smallest captured size that holds it (``batch_sizes`` adds
sizes to the one captured at ``batch``) and returns its own rows only.

No collective is involved: eval samples are independent, so N GPUs run N sessions on
disjoint batch shards (SURVEY 8e).
"""
from __future__ import annotations

import collections

import torch

from . import _lib, ops
from .modules import apply_head


class InferenceSession:
    def __init__(self, model, batch, in_shape, device=None, use_graph=True, slots=2, serving_fusions=True, output="logits",
                 batch_sizes=None, dtype=torch.float32):
        """``output="logits"`` (default): the model's fp32 output.  ``output="classes"``: the (batch, H, W) int64 class map
        argmax over its channels (the reference's ``torch.argmax(softmax(y_pred), dim=1)``, train_SmaAtUNet.py:76), computed
        inside the captured graph: ``model.forward_classes`` where the model has it (SmaAt_UNet: OutConv and argmax in the last
        kernel's epilogue), otherwise ``model(x)`` followed by the channel argmax kernel.  Only the class map crosses PCIe.
        ``output="probs"``: the (batch, K, H, W) fp32 softmax probabilities over the model's K output channels (the reference's
        ``softmax(y_pred)``), likewise from ``model.forward_probs`` where the model has it, otherwise ``model(x)`` followed by
        the channel softmax kernel; only the probabilities cross PCIe.  A model with one output channel raises ``ValueError``
        (softmax over one channel is identically 1).

        ``batch`` is the capacity: the largest request and the size captured in any case.  ``batch_sizes``: further sizes in
        ``1..batch``, each captured in a graph of its own over the leading rows of the one input buffer.  ``forward`` /
        ``submit`` take any 1 <= n <= batch rows and run the smallest captured size m >= n; rows n..m are padding (eval
        samples are independent, so they change no real row) and only the n real rows are returned.

        ``dtype=torch.bfloat16`` captures SmaAt_UNet's bf16 storage route (``SmaAt_UNet._serve_bf16``): the input and its
        staging buffers are bf16, and so are the logits and probabilities (class maps stay int64); requests must be bf16.
        Models and settings without that route raise ``ValueError`` here."""
        if dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"InferenceSession: dtype must be torch.float32 or torch.bfloat16, got {dtype}")
        if output not in ("logits", "classes", "probs"):
            raise ValueError(f"InferenceSession: output must be one of 'probs', 'logits' or 'classes', got {output!r}")
        batch = int(batch)
        extra = [int(m) for m in (batch_sizes or ())]
        if batch < 1 or any(not 1 <= m <= batch for m in extra):
            raise ValueError(f"InferenceSession: batch_sizes must lie in 1..batch={batch}, got {tuple(extra)}")
        self.sizes = tuple(sorted(set(extra) | {batch}))     # captured sizes, ascending; the last is the capacity
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.model = model.to(self.device).eval()
        self.batch, self.in_shape = batch, tuple(in_shape)
        self.output = output
        self.use_graph = use_graph
        self.compute = torch.cuda.Stream(self.device)
        self.h2d = torch.cuda.Stream(self.device)
        self.d2h = torch.cuda.Stream(self.device)
        self.dtype = dtype
        self.static_in = torch.zeros((batch,) + self.in_shape, device=self.device, dtype=dtype)
        self.launches_per_forward = 0
        self.graph = None            # the capacity size's graph
        self._graphs = {}            # size -> captured graph
        self._outs = {}              # size -> its static output
        # the serving forward may fuse what plain module calls cannot express (OutConv in the last epilogue, model.py);
        # serving_fusions=False captures exactly the reference-API call sequence (+ the argmax / softmax kernel for class maps /
        # probabilities)
        name = {"logits": "forward_serving", "classes": "forward_classes", "probs": "forward_probs"}[output]
        self._fwd = getattr(self.model, name, None) if serving_fusions else None
        if self._fwd is None:
            model = self.model                  # not self: a session must not sit in a reference cycle
            self._fwd = lambda x: apply_head(model, x, output)
        self._capture()
        self.out_shape = tuple(self.static_out.shape)
        # staging slots (device side) so H2D of step i+1 and D2H of step i-1 overlap compute of step i
        self.slots = slots
        self.in_stage = [torch.empty_like(self.static_in) for _ in range(slots)]
        self.out_stage = [torch.empty_like(self.static_out) for _ in range(slots)]
        self.out_host = [torch.empty(self.out_shape, dtype=self.static_out.dtype, pin_memory=True) for _ in range(slots)]
        self._h2d_done = [torch.cuda.Event() for _ in range(slots)]
        self._in_free = [torch.cuda.Event() for _ in range(slots)]
        self._out_ready = [torch.cuda.Event() for _ in range(slots)]
        self._d2h_done = [torch.cuda.Event() for _ in range(slots)]
        self._pending = collections.deque()
        self._step = 0

    def _capture(self):
        with torch.cuda.device(self.device), torch.no_grad():
            # warm-up of every size on the compute stream, capacity first, before any capture: builds the folded-BN /
            # split-weight caches and the CBAM scratch (their allocations must not be captured) and sizes the allocator
            self.compute.wait_stream(torch.cuda.current_stream(self.device))
            self._graphs, self._outs = {}, {}
            out_like = {}
            with torch.cuda.stream(self.compute):
                for m in reversed(self.sizes):
                    for _ in range(2):
                        out = self._fwd(self.static_in[:m])
                    out_like[m] = (out.shape, out.dtype)
            self.compute.synchronize()
            if self.output == "probs" and out.shape[1] == 1:
                raise ValueError("InferenceSession(output='probs'): the model has one output channel, whose softmax is "
                                 "identically 1; serve its logits instead")
            # Every size captures into the capacity graph's private pool, so an extra size costs little more than its
            # output.  Sharing scratch is safe: all graphs replay on the one compute stream, so no two run at once, and
            # every pool block a graph uses is written by that graph before it reads it.  Outputs must outlive other sizes'
            # replays, so none of them may sit in a block another graph uses as scratch.  Left to the allocator, an extra
            # size's output would land in blocks the graphs captured before it freed, and those graphs write them on every
            # replay.  So the extra sizes' buffers are allocated first thing in the capacity capture (no kernel), before
            # any scratch block, and each extra graph copies its result into its buffer.  The capacity graph is captured
            # first; its output is its own last write.  All outputs stay referenced for the session's life, so no later
            # capture is handed their blocks.
            pool = None
            for m in reversed(self.sizes):
                n0 = _lib.launch_count()
                if self.use_graph:
                    g = torch.cuda.CUDAGraph()
                    with ops.gc_paused(), torch.cuda.graph(g, pool=pool, stream=self.compute):
                        if m == self.batch:
                            for k in self.sizes[:-1]:
                                self._outs[k] = torch.empty(out_like[k][0], dtype=out_like[k][1], device=self.device)
                            self._outs[m] = self._fwd(self.static_in[:m])
                        else:
                            self._outs[m].copy_(self._fwd(self.static_in[:m]))
                    pool = g.pool() if pool is None else pool
                    self._graphs[m] = g
                else:
                    with torch.cuda.stream(self.compute):
                        self._outs[m] = self._fwd(self.static_in[:m])
                if m == self.batch:
                    self.launches_per_forward = _lib.launch_count() - n0
            self.compute.synchronize()
        self.graph = self._graphs.get(self.batch)
        # the graph has the addresses of the weight caches, parameters and buffers baked in: the session holds them alive,
        # whatever the model does with them afterwards (mode switches drop the caches, TrainSession re-points the parameters)
        from .modules import graph_tensors
        self._keepalive = graph_tensors(self.model)

    @property
    def static_out(self):
        """The capacity size's output buffer."""
        return self._outs[self.batch]

    def size_for(self, n):
        """The captured size a request of ``n`` rows runs: the smallest one >= n.  ``ValueError`` outside 1..batch."""
        if not 1 <= n <= self.batch:
            raise ValueError(f"InferenceSession: a request must have 1..{self.batch} rows, got {n}")
        return next(m for m in self.sizes if m >= n)

    def _rows(self, x):
        if self.dtype == torch.bfloat16 and x.dtype != torch.bfloat16:
            raise ValueError(f"InferenceSession(dtype=torch.bfloat16): requests must be bfloat16, got {x.dtype}")
        if x.dim() != 1 + len(self.in_shape) or tuple(x.shape[1:]) != self.in_shape:
            raise ValueError(f"InferenceSession: expected (n, {', '.join(map(str, self.in_shape))}) with 1 <= n <= {self.batch}, "
                             f"got {tuple(x.shape)}")
        n = int(x.shape[0])
        return n, self.size_for(n)

    def refresh(self):
        """Re-derive the weight caches and re-capture every size's graph: call after the model's parameters / BatchNorm
        statistics changed (e.g. more training).  The session is not a snapshot: the folded BatchNorm, tf32 splits and packed weights
        are derived at capture, but the other parameters (depthwise and tf32-mode pointwise weights, the CBAM MLP, OutConv,
        biases) are read in place, so until refresh() the outputs mix old and new weights."""
        ops.bump_weights_generation()
        self.model.eval()
        self.graph = None
        self._graphs = {}
        self._capture()          # static_out may be a new tensor: read it again after refresh()

    # -- device-resident path ---------------------------------------------------------------
    def _run(self, m):
        """Run captured size m on static_in[:m]; returns its output."""
        if self.use_graph:
            self._graphs[m].replay()
        else:
            with torch.no_grad():
                self._outs[m] = self._fwd(self.static_in[:m])
        return self._outs[m]

    def forward(self, x_dev):
        """x_dev: (n, *in_shape) CUDA tensor, 1 <= n <= batch -> its n output rows, a view of the static output of the size
        it ran (valid until the next request of that size; requests of other sizes leave it alone)."""
        n, m = self._rows(x_dev)
        cur = torch.cuda.current_stream(self.device)     # the caller's stream, which produced x_dev
        with torch.cuda.stream(self.compute):
            self.compute.wait_stream(cur)
            self.static_in[:n].copy_(x_dev, non_blocking=True)
            out = self._run(m)
        cur.wait_stream(self.compute)
        return out if n == m else out[:n]

    def replay(self, m=None):
        """Re-run the captured forward of size ``m`` (default: the capacity) on whatever static_in holds (kernel-only
        timing)."""
        with torch.cuda.stream(self.compute):
            self._run(self.batch if m is None else m)

    # -- host-buffer path ----------------------------------------------------------------------
    def submit(self, x_host):
        """Enqueue one batch of 1 <= n <= batch rows from PINNED host memory; returns immediately."""
        n, m = self._rows(x_host)
        assert x_host.is_pinned(), "InferenceSession.submit needs pinned host memory for async copies"
        s = self._step % self.slots
        if self._step >= self.slots:          # slot reuse: its previous D2H must have been collected
            assert len(self._pending) < self.slots, "collect() results before submitting more batches"
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(self._in_free[s])
            self.in_stage[s][:n].copy_(x_host, non_blocking=True)
            self._h2d_done[s].record(self.h2d)
        with torch.cuda.stream(self.compute):
            self.compute.wait_event(self._h2d_done[s])
            self.static_in[:n].copy_(self.in_stage[s][:n], non_blocking=True)
            self._in_free[s].record(self.compute)
            out = self._run(m)
            self.compute.wait_event(self._d2h_done[s])
            self.out_stage[s][:n].copy_(out[:n], non_blocking=True)
            self._out_ready[s].record(self.compute)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self._out_ready[s])
            self.out_host[s][:n].copy_(self.out_stage[s][:n], non_blocking=True)
            self._d2h_done[s].record(self.d2h)
        self._pending.append((s, n))
        self._step += 1

    def collect(self):
        """Block until the oldest submitted batch is back in pinned host memory; returns its n rows, a view of a pinned
        buffer (reused after ``slots`` further submits)."""
        s, n = self._pending.popleft()
        self._d2h_done[s].synchronize()
        return self.out_host[s] if n == self.batch else self.out_host[s][:n]

    @property
    def h2d_bytes_per_step(self):
        """Bytes one capacity-size request moves host -> device (a request of n rows moves n / batch of it)."""
        return self.static_in.numel() * self.static_in.element_size()

    @property
    def d2h_bytes_per_step(self):
        """Bytes one capacity-size request moves device -> host."""
        return self.static_out.numel() * self.static_out.element_size()
