"""Inference engine: the call a user makes to classify batches of clouds at full throughput.

One forward of the point-set-abstraction models is ~25 small-to-medium kernel launches, several of them latency-bound
on a fraction of the SMs (FPS: one CTA per cloud).  The engine therefore
  * captures one forward per *slot* into a CUDA graph (static input / output buffers, private workspace pool), and
  * keeps `slots` independent batches in flight on `slots` streams (batch i -> slot i % slots), so the next batch's
    FPS overlaps the current batch's tensor-core kernels (which hand out their tiles dynamically).
Host batches are copied from pinned memory on the slot's stream; results come back as pinned host tensors.
"""
from __future__ import annotations

from typing import Callable, List

import torch


class InferenceEngine:
    def __init__(self, forward: Callable[[torch.Tensor], torch.Tensor], batch_shape, out_shape, slots: int = 3, device=None):
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.slots = max(1, int(slots))
        self.streams: List[torch.cuda.Stream] = [torch.cuda.Stream(device=self.device) for _ in range(self.slots)]
        self.static_in, self.static_out, self.graphs, self.host_out = [], [], [], []
        probe = torch.zeros(batch_shape, dtype=torch.float32, device=self.device)
        probe[..., 0] = torch.linspace(-1, 1, batch_shape[-2], device=self.device)      # any finite input: warm-up only
        for j in range(self.slots):
            buf = probe.clone()
            self.streams[j].wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.streams[j]):
                for _ in range(2):                    # warm-up: builds weight images / caches outside the capture
                    out = forward(buf)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.streams[j]):
                out = forward(buf)
            torch.cuda.synchronize()
            if tuple(out.shape) != tuple(out_shape):
                raise ValueError(f"forward returned {tuple(out.shape)}, expected {tuple(out_shape)}")
            self.static_in.append(buf); self.static_out.append(out); self.graphs.append(g)
            self.host_out.append(torch.empty(out_shape, dtype=torch.float32).pin_memory())
        self._n = 0

    def submit(self, batch: torch.Tensor, to_host: bool = False) -> int:
        """Enqueue one batch (device tensor, or pinned host tensor) on the next slot; returns the slot index.
        The previous result of that slot is overwritten: read it (``result``) before the slot comes round again."""
        j = self._n % self.slots
        self._n += 1
        if batch.is_cuda:
            # the producer of a device batch ran on the caller's current stream: order the slot stream behind it, and keep the
            # caching allocator from recycling the (possibly temporary) tensor while the copy is still pending
            self.streams[j].wait_stream(torch.cuda.current_stream(self.device))
            batch.record_stream(self.streams[j])
        with torch.cuda.stream(self.streams[j]):
            self.static_in[j].copy_(batch, non_blocking=True)
            self.graphs[j].replay()
            if to_host:
                self.host_out[j].copy_(self.static_out[j], non_blocking=True)
        return j

    def result(self, slot: int, host: bool = False) -> torch.Tensor:
        """Wait for the slot's stream and return its logits (device tensor, or the pinned host copy).  Both are the slot's
        STATIC buffers: they are overwritten when the slot comes round again (after ``slots`` further submits) -- clone to keep."""
        self.streams[slot].synchronize()
        return self.host_out[slot] if host else self.static_out[slot]

    def fence_begin(self, event: torch.cuda.Event) -> None:
        for st in self.streams:
            st.wait_event(event)

    def fence_end(self, stream: torch.cuda.Stream) -> None:
        for st in self.streams:
            stream.wait_stream(st)


def pointnet2_cls_ssg_engine(params, batch: int = 32, npoints: int = 2048, num_class: int = 15, slots: int = 3, device=None):
    from . import pointnet2_cls_ssg

    def forward(x):
        logits, _ = pointnet2_cls_ssg.get_model(x, False, params=params)
        return logits

    return InferenceEngine(forward, (batch, npoints, 3), (batch, num_class), slots=slots, device=device)


def pointcnn_cls_engine(params, batch: int = 32, npoints: int = 1024, num_class: int = 15, slots: int = 3, device=None):
    from . import pointcnn_cls

    def forward(x):
        return pointcnn_cls.get_model(x, False, num_class, params=params)

    return InferenceEngine(forward, (batch, npoints, 3), (batch, 1, num_class), slots=slots, device=device)
