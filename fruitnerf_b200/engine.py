"""CUDA-graph execution of the training hot step.

One FruitNeRF training iteration on the hot path is a handful of kernels that together run for a few
milliseconds; enqueueing them op by op from Python costs a large share of that.  ``GraphedTrainStep``
captures the body of ``FruitPipeline.get_train_loss_dict`` + ``backward`` for a fixed batch shape --
fused render forward, MSE / BCE-with-logits loss (fruit_nerf/fruit_nerf.py:359-366), field
backward into the flat gradient buffer -- into ONE CUDA graph and replays it per step.  Inputs live in
static device buffers that ``load_batch`` refreshes (asynchronous H2D copies from pinned memory).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch
from torch import Tensor

from . import _lib as L
from . import ops


def default_loss(outputs: Dict[str, Tensor], image: Tensor, fruit_mask: Tensor, semantic_loss_weight: float = 1.0) -> Tensor:
    """rgb MSE + semantic BCE-with-logits (get_loss_dict without the interlevel term)."""
    mse, bce, _ = ops.render_losses(outputs["rgb"], outputs["semantics"], image, fruit_mask, semantic_loss_weight)  # one launch
    return mse + bce


class GraphedTrainStep:
    def __init__(self, field, num_rays: int, num_samples: int, impl: int = L.FNR_IMPL_AUTO, semantic_loss_weight: float = 1.0,
                 use_graph: bool = True, flat_grad: Optional[Tensor] = None):
        self.field = field
        self._flat_grad_buffer = flat_grad  # persistent (e.g. symmetric / multicast-mapped) gradient buffer, or None
        self.impl = impl
        self.semantic_loss_weight = semantic_loss_weight
        dev = next(field.parameters()).device
        self.device = dev
        R, S = num_rays, num_samples
        # every static input is a view of ONE device byte buffer, so a batch that arrives packed in one pinned host
        # buffer (``pack_batch``) is a single host->device copy per step (``load_packed``)
        spec = (("origins", (R, 3), torch.float32), ("directions", (R, 3), torch.float32), ("starts", (R, S), torch.float32),
                ("ends", (R, S), torch.float32), ("camera_indices", (R,), torch.int32), ("image", (R, 3), torch.float32),
                ("fruit_mask", (R, 1), torch.float32))
        self._layout, off = {}, 0
        for name, shape, dtype in spec:
            n = 1
            for v in shape:
                n *= v
            self._layout[name] = (off, n * 4, shape, dtype)
            off += (n * 4 + 255) // 256 * 256
        self._flat_bytes = off
        self._flat = torch.zeros(off, dtype=torch.uint8, device=dev)
        self.static = {name: self._flat[o:o + nb].view(dtype).view(shape) for name, (o, nb, shape, dtype) in self._layout.items()}
        self.static["ends"].fill_(1.0)
        self.params = field.kernel_params()
        self.loss: Optional[Tensor] = None
        self.outputs: Optional[Dict[str, Tensor]] = None
        self.flat_grad: Optional[Tensor] = None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.use_graph = use_graph
        self._captured = False
        self._copy_stream = None
        self._staging = None
        self._copy_done = None
        self.launches_per_step = 0

    # ---- inputs -----------------------------------------------------------------------------------
    def load_batch(self, origins, directions, starts, ends, camera_indices, image, fruit_mask, non_blocking: bool = True) -> int:
        """Copy one batch (host pinned or device tensors) into the static buffers; returns bytes copied."""
        src = dict(origins=origins, directions=directions, starts=starts, ends=ends, camera_indices=camera_indices, image=image,
                   fruit_mask=fruit_mask)
        n = 0
        for k, t in src.items():
            dst = self.static[k]
            if t.dtype != dst.dtype:
                t = t.to(dst.dtype)
            dst.copy_(t.reshape(dst.shape), non_blocking=non_blocking)
            n += dst.numel() * dst.element_size()
        return n

    def pack_batch(self, origins, directions, starts, ends, camera_indices, image, fruit_mask) -> Tensor:
        """Pack one batch into a pinned host byte buffer with the layout of the static device buffer (what a data loader
        worker would fill)."""
        flat = torch.zeros(self._flat_bytes, dtype=torch.uint8).pin_memory()
        src = dict(origins=origins, directions=directions, starts=starts, ends=ends, camera_indices=camera_indices, image=image,
                   fruit_mask=fruit_mask)
        for name, (o, nb, shape, dtype) in self._layout.items():
            flat[o:o + nb].view(dtype).view(shape).copy_(src[name].to(dtype).reshape(shape))
        return flat

    def load_packed(self, flat_host: Tensor, non_blocking: bool = True) -> int:
        """ONE host->device copy of a packed batch; returns the payload bytes (without alignment padding)."""
        self._flat.copy_(flat_host, non_blocking=non_blocking)
        return sum(nb for _, nb, _, _ in self._layout.values())

    def prefetch_packed(self, flat_host: Tensor) -> int:
        """Start the host->device copy of the NEXT packed batch on a side stream while the current step runs;
        ``commit_prefetched`` swaps it in with one device-to-device copy."""
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._staging = torch.empty_like(self._flat)
            self._copy_done = torch.cuda.Event()
        self._copy_stream.wait_stream(torch.cuda.current_stream(self.device))  # the staging buffer was read by the last commit
        with torch.cuda.stream(self._copy_stream):
            self._staging.copy_(flat_host, non_blocking=True)
            self._copy_done.record(self._copy_stream)
        return sum(nb for _, nb, _, _ in self._layout.values())

    def commit_prefetched(self) -> None:
        torch.cuda.current_stream(self.device).wait_event(self._copy_done)
        self._flat.copy_(self._staging, non_blocking=True)

    # ---- result read-back ----------------------------------------------------------------------------
    def read_loss_async(self):
        """Start the device->host copy of the current step's loss into pinned memory; returns a handle whose ``value()``
        waits for that copy only (not for later work) -- the way a training loop logs its loss without draining the GPU."""
        if not hasattr(self, "_loss_ring"):
            self._loss_ring = [(torch.zeros(1).pin_memory(), torch.cuda.Event()) for _ in range(4)]
            self._loss_next = 0
        buf, ev = self._loss_ring[self._loss_next]
        self._loss_next = (self._loss_next + 1) % len(self._loss_ring)
        buf.copy_(self.loss.reshape(1), non_blocking=True)
        ev.record(torch.cuda.current_stream(self.device))

        class _Handle:
            def value(self_inner) -> float:
                ev.synchronize()
                return float(buf[0])

        return _Handle()

    # ---- the step ---------------------------------------------------------------------------------
    def _eager(self) -> Tensor:
        f, st = self.field, self.static
        for p in self.params:
            p.grad = None
        out = ops.render(f.kernel_shape(), self.params, st["origins"], st["directions"], st["starts"], st["ends"], st["camera_indices"],
                         f.position_mode(), f.appearance_mode(), impl=self.impl, flat_grad=self._flat_grad_buffer)
        loss = default_loss(out, st["image"], st["fruit_mask"], self.semantic_loss_weight)
        loss.backward()
        self.outputs, self.loss = out, loss.detach()
        self.flat_grad = ops._Render.last_flat_grad
        return self.loss

    def capture(self, warmup: int = 3) -> None:
        if not self.use_graph:
            lib = L.load()
            lib.fnr_launch_count(1)
            self._eager()
            self.launches_per_step = int(lib.fnr_launch_count(1))
            self._captured = True
            return
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._eager()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        for p in self.params:
            p.grad = None
        self.graph = torch.cuda.CUDAGraph()
        lib = L.load()
        lib.fnr_launch_count(1)
        with torch.cuda.graph(self.graph):
            self._eager()
        self.launches_per_step = int(lib.fnr_launch_count(1))  # kernels of THIS library recorded into the step's graph
        self._captured = True

    def __call__(self) -> Tensor:
        """Run one step on the current static batch; returns the (static) scalar loss tensor.  Parameter
        ``.grad`` tensors are views of ``flat_grad`` (one buffer for the multi-GPU all-reduce)."""
        if not self._captured:
            self.capture()
        if self.graph is not None:
            self.graph.replay()
        else:
            self._eager()
        return self.loss
