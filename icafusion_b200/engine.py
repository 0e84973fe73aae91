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
from .common import C3, Conv, CrossAttention, CrossTransformerBlock, TransformerFusionBlock
from .yolo_test import Detect, Model


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


def refresh_packed_(model: Model) -> int:
    """Bring every packed-filter cache of `model` up to date with its parameters and BatchNorm buffers, in place.

    Each cache whose key moved (``ModelEMA.update``, ``load_state_dict``, an optimiser step) is packed again by the code the
    forward uses, and the result is copied into the tensors already cached (:func:`ops.copy_packed_`): Conv filters (the
    image stem and the fused Bottleneck read these too), C3's stacked cv1 | cv2 bank, the DMFF projections with their
    LayerNorm fold and colsum, the DMFF front tensors and Detect's filters.  No tensor is rebound, so a CUDA graph captured
    on them (:class:`ValidationGraphs`) stays valid.  A re-pack of another shape or layout raises ValueError.  Detect's
    anchors are not packed: the decode takes them by value.  Returns the number of caches re-packed."""
    n = 0
    for m in reversed(list(model.modules())):                   # children first: C3's cv1 and cv2 before its stack
        d = m.__dict__
        if isinstance(m, C3) and "_icaf_pack12" in d:
            before = d["_icaf_pack12"][3]
            m.packed_cv12(in_place=True)
            n += int(d["_icaf_pack12"][3] != before)
        if isinstance(m, (Conv, CrossAttention, CrossTransformerBlock)) and "_icaf_pack" in d:
            before = d["_icaf_pack"][0]
            m.packed(in_place=True)
            n += int(d["_icaf_pack"][0] != before)
        elif isinstance(m, TransformerFusionBlock) and "_icaf_pack" in d:
            before = d["_icaf_pack"][0]
            m._front(in_place=True)
            n += int(d["_icaf_pack"][0] != before)
        elif isinstance(m, Detect):
            cache = d.get("_icaf_pack", {})
            for i, (key, old) in list(cache.items()):
                m._packed(i)                                     # re-packs into a new pack when the key moved
                if cache[i][0] != key:
                    cache[i] = (cache[i][0], ops.copy_packed_(old, cache[i][1], f"Detect.m[{i}]"))
                    n += 1
    return n


def broadcast_model_(model: Model, src: int = 0, group=None) -> None:
    """Give every rank of `group` rank `src`'s weights, in place: every parameter and buffer of `model` (Detect's anchors
    included) is broadcast into the tensor it already is, so the packed-filter caches and the CUDA graphs of a
    :class:`ValidationGraphs` keep their addresses, and the next ``begin`` refreshes the packs.  For a sharded
    ``test.test(..., group=)`` when only rank `src` holds the EMA model; ``TrainStep(..., ema=True)`` on every rank keeps
    identical EMA weights without it."""
    import torch.distributed as dist
    with torch.no_grad():
        for t in list(model.parameters()) + list(model.buffers()):
            buf = t.detach().clone()
            dist.broadcast(buf, src=src, group=group)
            t.copy_(buf)                    # an in-place copy moves the tensor's version, which the packed caches are keyed on


def decode_values(model: Model) -> tuple:
    """What the Detect decode launches take by value, as the next forward reads them: the anchors in pixels per level and
    the strides (one device to host copy)."""
    det = model.model[-1]
    return det.anchor_grid.detach().float().cpu().view(det.nl, -1).tolist(), [float(s) for s in det.stride]


class ValidationGraphs:
    """CUDA-graph replay of :func:`icafusion_b200.test.test`'s batch loop, bound to one eval-mode model for a whole training
    run: ``test.test(..., model=ema.ema, graphs=ValidationGraphs(ema.ema))``.

    Per batch shape (B, H, W) it keeps static inputs (the uint8 (B, 6, H, W) image, the targets at a capacity that grows,
    unused rows at image -1, which the loss and the matching skip; ``ratio_pad``; the KAIST image positions) and two graphs:
    the forward plus the optional validation loss, accumulated into the static ``loss``, and multi-label NMS plus
    icaf_match_detections plus the optional icaf_kaist_round_detections.  The first batch of a shape runs eagerly on the
    static buffers (the warm-up, which packs the filters) and is then captured; later batches of the shape are replays.
    Each call of test.test starts with ``begin``, which refreshes the model's packed filters in place
    (:func:`refresh_packed_`), so the graphs see the weights of that epoch.

    A new shape, a batch with more targets than the shape's capacity, or other test.test settings capture again.  At most
    ``max_shapes`` shapes are held; batches of further shapes run eagerly.  The decode launches hold Detect's anchors by
    value, and ModelEMA.update moves them by rounding, so the graphs are captured again whenever those values changed."""

    max_shapes = 4
    max_det = 300                 # ops.nms's default, what test.test keeps per image

    def __init__(self, model: Model):
        if not isinstance(model, Model):
            raise TypeError(f"ValidationGraphs needs an icafusion_b200 Model, got {type(model).__name__}")
        if model.training:
            raise ValueError("ValidationGraphs needs model.eval()")
        self.model = model
        self.device = next(model.parameters()).device
        if self.device.type != "cuda" and not (ops.dry_running() and self.device.type == "meta"):
            raise RuntimeError("ValidationGraphs needs the model on a CUDA device")
        self.entries = {}                 # (B, H, W, image dtype) -> _ShapeGraphs
        self.captures = 0                 # shapes captured so far, re-captures included
        self.settings = None
        self.per_batch = False
        self.loss = self.iouv = None
        self._stream = None
        self._values = None               # what the captured decodes hold by value: Detect's anchors and strides
        self._held = []                   # the packs the graphs were captured on (kept alive; see begin)
        self._kaist = None

    def check(self, model, device) -> None:
        if model is not self.model:
            raise ValueError("test: graphs= was built for another model")
        if device != self.device:
            raise ValueError(f"test: graphs= was built for the model on {self.device}, the model is now on {device}")

    def begin(self, iouv: torch.Tensor, settings: tuple, per_batch: bool = False) -> torch.Tensor:
        """Start one test.test call: refresh the packed filters in place, drop the graphs whose by-value arguments or settings
        changed, and zero the loss accumulator, which is returned.  per_batch: the captured forward writes each batch's loss
        items to the returned tensor instead of adding them (``run(..., loss_row=)`` then copies them out)."""
        refresh_packed_(self.model)
        values = decode_values(self.model)
        packs = self._packs()
        if values != self._values or settings != self.settings or per_batch != self.per_batch or \
                len(packs) != len(self._held) or any(a is not b for a, b in zip(packs, self._held)):
            # an eager forward after a weight change re-packs into new tensors: the graphs' filters are then stale
            self.entries.clear()
            self._values, self.settings, self.per_batch = values, settings, per_batch
        if self.loss is None:
            self.loss = torch.zeros(4, device=self.device)
            self.iouv = iouv.clone()
        else:
            self.loss.zero_()
            self.iouv.copy_(iouv)
        return self.loss

    def kaist_buffers(self, kaist):
        """The (rows, span) buffers every batch's icaf_kaist_round_detections writes, span zeroed for a new call."""
        if self._kaist is None or self._kaist[0] is not kaist:
            self._kaist = (kaist, torch.empty(kaist.images * self.max_det, 5, dtype=torch.float64, device=self.device),
                           torch.zeros(kaist.images, 2, dtype=torch.int32, device=self.device))
        else:
            self._kaist[2].zero_()
        return self._kaist[1], self._kaist[2]

    def entry(self, img: torch.Tensor, n_targets: int):
        """The graphs of this batch's shape, made if needed; None when the batch is to run eagerly."""
        B, _, H, W = img.shape
        key = (B, H, W, img.dtype)
        e = self.entries.get(key)
        if e is not None and n_targets > e.capacity:
            del self.entries[key]                    # frees the graphs and their pool before the larger capture
            e = None
        if e is None:
            if len(self.entries) >= self.max_shapes:
                return None
            cap = 64
            while cap < n_targets:
                cap *= 2
            e = self.entries[key] = _ShapeGraphs(self, B, H, W, img.dtype, cap)
        return e

    def _packs(self) -> list:
        """Every packed-filter object the model's caches hold now."""
        out = []
        for m in self.model.modules():
            c = m.__dict__.get("_icaf_pack")
            if isinstance(c, dict):
                out += [e[1] for e in c.values()]
            elif c is not None:
                out.append(c[1])
            if "_icaf_pack12" in m.__dict__:
                out.append(m.__dict__["_icaf_pack12"][2])
        return out

    def stream(self) -> torch.cuda.Stream:
        if self._stream is None:
            self._stream = torch.cuda.Stream(self.device)
        return self._stream


class _ShapeGraphs:
    """Static buffers and the two graphs of one batch shape (see ValidationGraphs)."""

    def __init__(self, owner: ValidationGraphs, B: int, H: int, W: int, dtype: torch.dtype, capacity: int):
        conf_thres, iou_thres, single_cls, compute_loss, need_native, kaist = owner.settings
        dev = owner.device
        self.owner, self.B, self.H, self.W, self.capacity = owner, B, H, W, capacity
        self.img = torch.zeros(B, 6, H, W, dtype=dtype, device=dev)
        self.targets = torch.zeros(capacity, 6, dtype=torch.float32, device=dev)
        self._unused = torch.zeros(capacity, 6, dtype=torch.float32, device=dev)
        self._unused[:, 0] = -1.0
        self.ratio_pad = torch.zeros(B, 5, dtype=torch.float32, device=dev)
        self.image = torch.zeros(B, dtype=torch.int32, device=dev) if kaist is not None else None
        self.det = torch.zeros(B, owner.max_det, 6, dtype=torch.float32, device=dev)
        self.count = torch.zeros(B, dtype=torch.int32, device=dev)
        self.correct = torch.zeros(B, owner.max_det, owner.iouv.numel(), dtype=torch.uint8, device=dev)
        self.native = torch.zeros(B, owner.max_det, 4, dtype=torch.float32, device=dev) if need_native else None
        need = int(ops._lib.lib().icaf_match_detections_workspace_bytes(capacity))
        self.match_ws = torch.empty(max((need + 3) // 4, 1), dtype=torch.int32, device=dev)
        self.nms_ws = self.z = None
        self.fwd = self.post = None

    def _forward(self):
        compute_loss = self.owner.settings[3]
        out, _, train_out = self.owner.model(self.img[:, :3], self.img[:, 3:])
        if compute_loss:
            items = compute_loss([x.float() for x in train_out], self.targets)[1][:4]
            if self.owner.per_batch:
                self.owner.loss.copy_(items)
            else:
                self.owner.loss += items
        self.z = (out if out.dtype == torch.float16 else out.half()).contiguous()

    def _post(self):
        conf_thres, iou_thres, single_cls, _, _, kaist = self.owner.settings
        ops.nms(self.z, conf_thres, iou_thres, agnostic=single_cls, multi_label=True, max_det=self.owner.max_det,
                det=self.det, count=self.count, workspace=self.nms_ws)
        ops.match_detections(self.det, self.count, self.targets, self.ratio_pad, self.H, self.W, self.owner.iouv, single_cls,
                             correct=self.correct, native=self.native, workspace=self.match_ws)
        if kaist is not None:
            rows, span = self.owner._kaist[1], self.owner._kaist[2]
            ops.kaist_round_detections(self.native, self.det, self.count, self.image, rows, span)

    def run(self, img, targets, ratio_pad, image, ev, loss_row=None):
        """One batch: stage it into the static inputs, then replay (or, for the shape's first batch, run eagerly and capture).
        ev: four CUDA events, recorded around the forward (+ loss) and around the NMS and matching.  loss_row: with
        ``begin(..., per_batch=True)``, a (4,) device tensor that receives this batch's loss items.  Returns per-batch device
        copies (det, count, correct, native); nothing waits for the device."""
        T = int(targets.shape[0])
        self.img.copy_(img, non_blocking=True)
        self.targets[:T].copy_(targets, non_blocking=True)
        self.targets[T:].copy_(self._unused[T:])
        self.ratio_pad.copy_(ratio_pad.pin_memory(), non_blocking=True)
        if self.image is not None:
            self.image.copy_(image.pin_memory(), non_blocking=True)
        with torch.no_grad():
            ev[0].record()
            if self.fwd is None:
                self._forward()
            else:
                self.fwd.replay()
            if loss_row is not None:
                loss_row.copy_(self.owner.loss)
            ev[1].record()
            ev[2].record()
            if self.fwd is None:
                if self.nms_ws is None:
                    need = ops.nms_workspace_bytes(*self.z.shape, True)
                    self.nms_ws = torch.empty((need + 7) // 8, dtype=torch.int64, device=self.owner.device)
                self._post()
            else:
                self.post.replay()
            ev[3].record()
            out = (self.det.clone(), self.count.clone(), self.correct.clone(),
                   self.native.clone() if self.native is not None else None)
            if self.fwd is None:
                self._capture()
        return out

    def _capture(self):
        """Capture the two graphs; nothing runs.  The graphs share one private pool (they replay in capture order)."""
        s = self.owner.stream()
        s.wait_stream(torch.cuda.current_stream(self.owner.device))
        fwd, post = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(fwd, stream=s):
            self._forward()
        with torch.cuda.graph(post, stream=s, pool=fwd.pool()):
            self._post()
        self.fwd, self.post = fwd, post
        self.owner.captures += 1
        self.owner._held = self.owner._packs()
