"""InferenceSession -- the serving-side public API: a static-shape eval forward captured once
in a CUDA graph (~90 kernel launches -> one graph launch) with pinned-host, double-buffered,
stream-overlapped input/output staging.

    sess = InferenceSession(model, batch=32, in_shape=(12, 288, 288))
    y_dev = sess.forward(x_dev)                  # device-resident input
    sess.submit(x_host_pinned); ...; y = sess.collect()   # host buffers, H2D/D2H overlapped with compute

No collective is involved: eval samples are independent, so N GPUs run N sessions on
disjoint batch shards (SURVEY 8e).
"""
from __future__ import annotations

import collections

import torch

from . import _lib
from .modules import apply_head


class InferenceSession:
    def __init__(self, model, batch, in_shape, device=None, use_graph=True, slots=2, serving_fusions=True, output="logits"):
        """``output="logits"`` (default): the model's fp32 output.  ``output="classes"``: the (batch, H, W) int64 class map
        argmax over its channels (the reference's ``torch.argmax(softmax(y_pred), dim=1)``, train_SmaAtUNet.py:76), computed
        inside the captured graph: ``model.forward_classes`` where the model has it (SmaAt_UNet: OutConv and argmax in the last
        kernel's epilogue), otherwise ``model(x)`` followed by the channel argmax kernel.  Only the class map crosses PCIe.
        ``output="probs"``: the (batch, K, H, W) fp32 softmax probabilities over the model's K output channels (the reference's
        ``softmax(y_pred)``), likewise from ``model.forward_probs`` where the model has it, otherwise ``model(x)`` followed by
        the channel softmax kernel; only the probabilities cross PCIe.  A model with one output channel raises ``ValueError``
        (softmax over one channel is identically 1)."""
        if output not in ("logits", "classes", "probs"):
            raise ValueError(f"InferenceSession: output must be one of 'probs', 'logits' or 'classes', got {output!r}")
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.model = model.to(self.device).eval()
        self.batch, self.in_shape = batch, tuple(in_shape)
        self.output = output
        self.use_graph = use_graph
        self.compute = torch.cuda.Stream(self.device)
        self.h2d = torch.cuda.Stream(self.device)
        self.d2h = torch.cuda.Stream(self.device)
        self.static_in = torch.zeros((batch,) + self.in_shape, device=self.device, dtype=torch.float32)
        self.launches_per_forward = 0
        self.graph = None
        # the serving forward may fuse what plain module calls cannot express (OutConv in the last epilogue, model.py);
        # serving_fusions=False captures exactly the reference-API call sequence (+ the argmax / softmax kernel for class maps /
        # probabilities)
        name = {"logits": "forward_serving", "classes": "forward_classes", "probs": "forward_probs"}[output]
        self._fwd = getattr(self.model, name, None) if serving_fusions else None
        if self._fwd is None:
            self._fwd = lambda x: apply_head(self.model, x, output)
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
            # warm-up on the compute stream: builds the folded-BN / split-weight caches (their small
            # kernels must not be captured) and sizes the allocator
            self.compute.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.compute):
                for _ in range(2):
                    self.static_out = self._fwd(self.static_in)
            self.compute.synchronize()
            if self.output == "probs" and self.static_out.shape[1] == 1:
                raise ValueError("InferenceSession(output='probs'): the model has one output channel, whose softmax is "
                                 "identically 1; serve its logits instead")
            n0 = _lib.launch_count()
            if self.use_graph:
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, stream=self.compute):
                    self.static_out = self._fwd(self.static_in)
            else:
                with torch.cuda.stream(self.compute):
                    self.static_out = self._fwd(self.static_in)
            self.launches_per_forward = _lib.launch_count() - n0
            self.compute.synchronize()
        # the graph has the addresses of the weight caches, parameters and buffers baked in: the session holds them alive,
        # whatever the model does with them afterwards (mode switches drop the caches, TrainSession re-points the parameters)
        from .modules import graph_tensors
        self._keepalive = graph_tensors(self.model)

    def refresh(self):
        """Re-derive the weight caches and re-capture the graph: call after the model's parameters / BatchNorm statistics
        changed (e.g. more training).  The session is not a snapshot: the folded BatchNorm, tf32 splits and packed weights
        are derived at capture, but the other parameters (depthwise and tf32-mode pointwise weights, the CBAM MLP, OutConv,
        biases) are read in place, so until refresh() the outputs mix old and new weights."""
        from . import ops
        ops.bump_weights_generation()
        self.model.eval()
        self.graph = None
        self._capture()          # static_out may be a new tensor: read it again after refresh()

    # -- device-resident path ---------------------------------------------------------------
    def _run(self):
        if self.graph is not None:
            self.graph.replay()
        else:
            with torch.no_grad():
                self.static_out = self._fwd(self.static_in)

    def forward(self, x_dev):
        """x_dev: (batch, *in_shape) CUDA tensor -> static output tensor (valid until the next call)."""
        with torch.cuda.stream(self.compute):
            self.compute.wait_stream(torch.cuda.current_stream(self.device))
            self.static_in.copy_(x_dev, non_blocking=True)
            self._run()
        torch.cuda.current_stream(self.device).wait_stream(self.compute)
        return self.static_out

    def replay(self):
        """Re-run the captured forward on whatever static_in holds (kernel-only timing)."""
        with torch.cuda.stream(self.compute):
            self._run()

    # -- host-buffer path ----------------------------------------------------------------------
    def submit(self, x_host):
        """Enqueue one batch from PINNED host memory; returns immediately."""
        assert x_host.is_pinned(), "InferenceSession.submit needs pinned host memory for async copies"
        s = self._step % self.slots
        if self._step >= self.slots:          # slot reuse: its previous D2H must have been collected
            assert len(self._pending) < self.slots, "collect() results before submitting more batches"
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(self._in_free[s])
            self.in_stage[s].copy_(x_host, non_blocking=True)
            self._h2d_done[s].record(self.h2d)
        with torch.cuda.stream(self.compute):
            self.compute.wait_event(self._h2d_done[s])
            self.static_in.copy_(self.in_stage[s], non_blocking=True)
            self._in_free[s].record(self.compute)
            self._run()
            self.compute.wait_event(self._d2h_done[s])
            self.out_stage[s].copy_(self.static_out, non_blocking=True)
            self._out_ready[s].record(self.compute)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self._out_ready[s])
            self.out_host[s].copy_(self.out_stage[s], non_blocking=True)
            self._d2h_done[s].record(self.d2h)
        self._pending.append(s)
        self._step += 1

    def collect(self):
        """Block until the oldest submitted batch is back in pinned host memory; returns that tensor
        (reused after ``slots`` further submits)."""
        s = self._pending.popleft()
        self._d2h_done[s].synchronize()
        return self.out_host[s]

    @property
    def h2d_bytes_per_step(self):
        return self.static_in.numel() * self.static_in.element_size()

    @property
    def d2h_bytes_per_step(self):
        return self.static_out.numel() * self.static_out.element_size()
