"""CUDA-graph execution of the two-stream detector (inference).

At batch 1 the forward is ~110 short kernels; launching them one by one from Python is 10x slower than the
kernels themselves.  :class:`GraphedDetector` captures one ``Model`` forward (all libicaf_b200 launches on the
capture stream, intermediate buffers in the graph's private pool) and replays it per step.  Inputs are staged
through static device buffers: device tensors are copied in with one D2D memcpy, host tensors (ideally pinned)
with one async H2D memcpy each; `uint8` frames are scaled by 1/255 inside the packing kernel, like the
reference's ``img.half() / 255`` staging (detect_twostream.py:70-80).
"""
from __future__ import annotations

from typing import Iterable, Iterator, Optional, Tuple

import torch

from . import ops
from .yolo_test import Model


class GraphedDetector:
    def __init__(self, model: Model, batch: int, height: int, width: int, in_dtype: torch.dtype = torch.float16,
                 device: Optional[torch.device] = None, warmup: int = 2, nms: Optional[dict] = None,
                 frame_hw: Optional[Tuple[int, int]] = None, confluence: Optional[dict] = None):
        """`frame_hw`: (H0, W0) of the raw decoded BGR frames; when given, the device letterbox (utils/datasets.py:1404-1427 +
        the BGR->RGB / HWC->CHW of :238) is captured in front of the forward and ``infer_frames`` takes the raw uint8
        (B, H0, W0, 3) frames -- the whole detect_twostream.py:70-86 loop body as one graph.
        `nms`: keyword arguments of :func:`icafusion_b200.ops.nms` (e.g. ``dict(conf_thres=0.25, iou_thres=0.45)``); when
        given, the batched device NMS (utils/general.py:518-607) is captured behind the forward and ``infer_detections``
        returns its fixed-capacity result -- the whole detect_twostream.py:84-86 step without a host round trip in between.
        `confluence`: keyword arguments of :func:`icafusion_b200.ops.confluence` (e.g. ``dict(conf_thres=0.1, p_thres=0.5)``),
        the reference's alternative to NMS (utils/confluence.py), captured in its place; its count is the true number kept
        and may exceed max_det."""
        if nms is not None and confluence is not None:
            raise ValueError("GraphedDetector: pass nms= or confluence=, not both")
        if model.training:
            raise ValueError("GraphedDetector needs model.eval()")
        self.model = model
        self.device = device or next(model.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("GraphedDetector needs the model on a CUDA device")
        self.shape = (batch, 3, height, width)
        self.rgb = torch.zeros(self.shape, dtype=in_dtype, device=self.device)
        self.ir = torch.zeros(self.shape, dtype=in_dtype, device=self.device)
        self.frame_hw = frame_hw
        self.rgb_raw = self.ir_raw = None
        if frame_hw is not None:
            from .datasets import letterbox, letterbox_geometry
            if in_dtype != torch.uint8:
                raise ValueError("GraphedDetector(frame_hw=...) stages uint8 frames: use in_dtype=torch.uint8")
            (nw, nh), _, _, (top, bottom, left, right) = letterbox_geometry(frame_hw, (height, width))
            if (nh + top + bottom, nw + left + right) != (height, width):
                raise ValueError(f"letterboxing {frame_hw} frames to {(height, width)} does not give {(height, width)}")
            self.rgb_raw = torch.zeros(batch, frame_hw[0], frame_hw[1], 3, dtype=torch.uint8, device=self.device)
            self.ir_raw = torch.zeros_like(self.rgb_raw)
            self._letterbox = lambda t, o: letterbox(t, (height, width), out=o)[0]
        self.stream = torch.cuda.Stream(self.device)
        self.launches_per_step = 0
        with torch.no_grad(), torch.cuda.stream(self.stream):
            if frame_hw is not None:
                self._letterbox(self.rgb_raw, self.rgb)    # uploads the tap tables outside the capture
            for _ in range(max(1, warmup)):            # packs filters, configures kernels, warms the allocator
                self.model(self.rgb, self.ir)
            if self.model.__dict__.get("_icaf_arena") is None:
                self.model.consolidate_weights(self.rgb, self.ir)     # one contiguous filter arena -> per-step L2 prefetch
                self.model(self.rgb, self.ir)
            self.stream.synchronize()
            self.det = self.count = None
            if nms is not None:                         # static NMS buffers live outside the graph's private pool
                z0 = self.model(self.rgb, self.ir)[0]
                self.det, self.count = ops.nms(z0, **nms)
                need = ops.nms_workspace_bytes(*z0.shape, nms.get("multi_label", False))
                self._nms_ws = torch.empty((need + 7) // 8, dtype=torch.int64, device=self.device)
                self.stream.synchronize()
            if confluence is not None:
                z0 = self.model(self.rgb, self.ir)[0]
                self._cf_ws = torch.empty((ops.confluence_workspace_bytes(*z0.shape) + 15) // 16, 2, dtype=torch.int64,
                                          device=self.device)
                self.det, self.count = ops.confluence(z0, workspace=self._cf_ws, **confluence)
                self.stream.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count()
            with torch.cuda.graph(self.graph, stream=self.stream):
                if frame_hw is not None:
                    self._letterbox(self.rgb_raw, self.rgb)
                    self._letterbox(self.ir_raw, self.ir)
                self.z, self.logits, self.xs = self.model(self.rgb, self.ir)
                if nms is not None:
                    ops.nms(self.z, det=self.det, count=self.count, workspace=self._nms_ws, **nms)
                if confluence is not None:
                    ops.confluence(self.z, det=self.det, count=self.count, workspace=self._cf_ws, **confluence)
            self.launches_per_step = ops.launch_count() - n0
        self.stream.synchronize()
        self._z_host = torch.empty(self.z.shape, dtype=self.z.dtype, pin_memory=True)
        if self.det is not None:
            self._det_host = torch.empty(self.det.shape, dtype=self.det.dtype, pin_memory=True)
            self._count_host = torch.empty(self.count.shape, dtype=self.count.dtype, pin_memory=True)

    # -- device-resident path ------------------------------------------------------------------
    def replay(self):
        """Re-run the captured forward on whatever the static input buffers hold (current stream)."""
        self.graph.replay()
        return self.z, self.logits, self.xs

    def __call__(self, rgb: torch.Tensor, ir: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, list]:
        """The reference-facing call: ``pred = model(img_rgb, img_ir)``.  Device or host inputs of the captured
        shape / dtype.  Returns device tensors (z, logits, [x0,x1,x2]) valid until the next call."""
        if tuple(rgb.shape) != self.shape or tuple(ir.shape) != self.shape:
            raise ValueError(f"GraphedDetector was captured for {self.shape}, got {tuple(rgb.shape)}")
        if self.rgb_raw is not None:
            raise RuntimeError("this GraphedDetector letterboxes raw frames inside its graph: call infer_frames(rgb_frames, ir_frames)")
        self.rgb.copy_(rgb, non_blocking=True)
        self.ir.copy_(ir, non_blocking=True)
        self.graph.replay()
        return self.z, self.logits, self.xs

    def infer_to_host(self, rgb_host: torch.Tensor, ir_host: torch.Tensor) -> torch.Tensor:
        """End-to-end step from (pinned) host frames to the decoded predictions on the host: H2D, forward, D2H, sync."""
        self(rgb_host, ir_host)
        self._z_host.copy_(self.z, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return self._z_host


    def infer_detections(self, rgb_host: torch.Tensor, ir_host: torch.Tensor):
        """End-to-end step with the captured NMS: H2D, forward, NMS, D2H of the (B, max_det, 6) detections and their counts.
        Returns (det_host fp32, count_host int32), valid until the next call."""
        if self.det is None:
            raise RuntimeError("GraphedDetector was built without nms=... or confluence=...")
        self(rgb_host, ir_host)
        self._det_host.copy_(self.det, non_blocking=True)
        self._count_host.copy_(self.count, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return self._det_host, self._count_host


    def infer_frames(self, rgb_frames_host: torch.Tensor, ir_frames_host: torch.Tensor):
        """The detect_twostream.py loop body for one batch of raw decoded frames (uint8 (B, H0, W0, 3) BGR, ideally pinned):
        H2D, letterbox + channel swap, staging, forward, NMS, D2H of the detections.  Needs frame_hw= and nms=."""
        if self.rgb_raw is None or self.det is None:
            raise RuntimeError("GraphedDetector.infer_frames needs frame_hw=... and nms=...")
        self.rgb_raw.copy_(rgb_frames_host, non_blocking=True)
        self.ir_raw.copy_(ir_frames_host, non_blocking=True)
        self.graph.replay()
        self._det_host.copy_(self.det, non_blocking=True)
        self._count_host.copy_(self.count, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return self._det_host, self._count_host


class PipelinedDetector:
    """Streaming front end: `depth` captured replicas of the forward (shared weights, private static buffers) used round
    robin so that the H2D copy of frame i+1 (copy stream) overlaps the forward of frame i (compute stream) and the host
    only blocks on the oldest frame in flight.  Every frame still pays its own H2D, forward and D2H.

        for z_host in PipelinedDetector(model, 1, 512, 640).infer_stream(frames):   # frames: iterable of (rgb_u8, ir_u8) host tensors
            ...                                                                     # z_host valid until `depth` more frames are submitted
    """

    def __init__(self, model: Model, batch: int, height: int, width: int, in_dtype: torch.dtype = torch.uint8,
                 device: Optional[torch.device] = None, depth: int = 2):
        self.replicas = [GraphedDetector(model, batch, height, width, in_dtype, device) for _ in range(depth)]
        self.device = self.replicas[0].device
        self.compute = torch.cuda.Stream(self.device)
        self.copy = torch.cuda.Stream(self.device)
        self.launches_per_step = self.replicas[0].launches_per_step
        for r in self.replicas:
            r._h2d_ev = torch.cuda.Event()
            r._done_ev = torch.cuda.Event()
            r._done_ev.record(self.compute)

    def submit(self, i: int, rgb_host: torch.Tensor, ir_host: torch.Tensor) -> None:
        r = self.replicas[i % len(self.replicas)]
        with torch.cuda.stream(self.copy):
            self.copy.wait_event(r._done_ev)            # replica's previous frame fully retired (inputs + z free)
            r.rgb.copy_(rgb_host, non_blocking=True)
            r.ir.copy_(ir_host, non_blocking=True)
            r._h2d_ev.record(self.copy)
        with torch.cuda.stream(self.compute):
            self.compute.wait_event(r._h2d_ev)
            r.graph.replay()
            r._z_host.copy_(r.z, non_blocking=True)
            r._done_ev.record(self.compute)

    def collect(self, i: int) -> torch.Tensor:
        r = self.replicas[i % len(self.replicas)]
        r._done_ev.synchronize()
        return r._z_host

    def infer_stream(self, frames: Iterable[Tuple[torch.Tensor, torch.Tensor]]) -> Iterator[torch.Tensor]:
        depth = len(self.replicas)
        submitted = collected = 0
        for rgb, ir in frames:
            if submitted - collected >= depth:          # oldest frame in flight; retiring it frees its replica
                yield self.collect(collected)
                collected += 1
            self.submit(submitted, rgb, ir)
            submitted += 1
        while collected < submitted:
            yield self.collect(collected)
            collected += 1
