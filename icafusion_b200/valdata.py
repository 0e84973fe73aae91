"""Validation batches on the device: what train.py's testloader -- ``create_dataloader_rgb_ir(..., rect=True, pad=0.5)``,
i.e. ``LoadMultiModalImagesAndLabels(augment=False)`` (utils/datasets.py:948-1024) + ``collate_fn`` (:1026-1031) -- hands
to ``test.test``, one kernel launch per batch.

The host reproduces the dataset's rect order and batch shapes (:827-860), the load_image_rgb_ir size (:1097-1125), the
letterbox geometry with scaleup=False (:1404-1427), the label rows and the ``shapes`` tuple, with the reference's own
expressions.  The kernel (csrc/image.cu, ``icaf_val_stage``) writes every output pixel of the uint8 (B, 6, H, W) batch:
the 114 border, or the load_image resize of the decoded frame -- a copy at r = 1, cv2.resize INTER_LINEAR at r > 1 and
INTER_AREA at r < 1, bit-exact against cv2 -- channel-swapped to RGB, the RGB frame in channels 0-2 and the IR frame in 3-5.

cv2.resize INTER_AREA on uint8 takes one of two paths (imgproc/resize.cpp), chosen per image from scale = src / dst in double
for each axis:
  * both scales integer (``resizeAreaFast``): the sum of the sx x sy source block; 2 x 2 blocks round as (sum + 2) >> 2 (the
    SIMD path), every other block as saturate_cast<uchar>(sum * (1.f / area)) (float, round half to even);
  * otherwise (``resizeArea_``), also when only one axis is integer or the two scales differ: per axis a float weight table
    (computeResizeAreaTab, built here in cv2's order); each output pixel sums, for every source row tap in order,
    beta * (sum over the column taps in order of src * alpha), every product and sum rounded to float, then
    saturate_cast<uchar>.
With pad >= 0 the letterbox never resizes a second time (the batch shape holds every load_image size of its batch);
a geometry that would need it raises NotImplementedError.  Decoding stays with the caller.

:func:`stage_reference` is the numpy restatement of the kernel's arithmetic (tests, and the CPU side of
scripts/val_loader_times.py)."""
from __future__ import annotations

import functools
import math
import time
from typing import Callable, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, ops
from .augment import load_size, resize_fixed, xywhn2xyxy, xyxy2xywh
from .datasets import ParamBlock, frames_on_device, letterbox_geometry, resize_taps

PAD = 114
MODE_COPY, MODE_LINEAR, MODE_AREA_FAST, MODE_AREA = 0, 1, 2, 3
_F32 = np.float32


# ---------------------------------------------------------------- reference expressions (utils/datasets.py)
def rect_batches(hw0: Sequence[Tuple[int, int]], batch_size: int, img_size: int, stride: int, pad: float):
    """The rect order, batch index and batch shapes of LoadMultiModalImagesAndLabels(rect=True) (:801-860): (irect int64 (n,),
    bi int64 (n,) over the sorted order, batch_shapes int64 (nb, 2) rows (H, W))."""
    s = np.array([(w, h) for h, w in hw0], dtype=np.float64)          # the label cache's shapes are (w, h)
    n = len(s)
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    ar = s[:, 1] / s[:, 0]
    irect = ar.argsort()
    ar = ar[irect]
    shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [maxi, 1]
        elif mini > 1:
            shapes[i] = [1, 1 / mini]
    batch_shapes = np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride
    return irect, bi, batch_shapes


def sample_geometry(h0: int, w0: int, shape, img_size: int):
    """(h, w) of load_image_rgb_ir, then letterbox(img, shape, auto=False, scaleup=False) of that image: (h, w, ratio, pad
    (dw, dh), top, left).  shape: the batch's (H, W) row of batch_shapes (numpy integers, so every scalar has the type the
    reference computes it in)."""
    h, w = load_size(h0, w0, img_size)
    (nw, nh), ratio, pad, (top, bottom, left, right) = letterbox_geometry((h, w), shape, scaleup=False)
    if (nh, nw) != (h, w):
        raise NotImplementedError(f"val: a {h}x{w} load_image result letterboxed to {tuple(int(v) for v in shape)} needs a "
                                  "second resize (pad < 0)")
    return h, w, ratio, pad, top, left


def sample_labels(lab: np.ndarray, h: int, w: int, ratio, pad, H: int, W: int) -> np.ndarray:
    """__getitem__'s label path without augmentation: float32 (nL, 5) rows (cls, x, y, w, h) normalised to the batch shape."""
    lab = lab.copy()
    if lab.size:
        lab[:, 1:] = xywhn2xyxy(lab[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    if len(lab):
        lab[:, 1:5] = xyxy2xywh(lab[:, 1:5])
        lab[:, [2, 4]] /= H
        lab[:, [1, 3]] /= W
    return lab


def collate(per_sample: Sequence[np.ndarray]) -> torch.Tensor:
    """collate_fn on the samples' labels_out: float32 (n, 6) rows (image, cls, x, y, w, h)."""
    outs = []
    for i, lab in enumerate(per_sample):
        t = torch.zeros((len(lab), 6))
        if len(lab):
            t[:, 1:] = torch.from_numpy(lab)
        t[:, 0] = i
        outs.append(t)
    return torch.cat(outs, 0)


# ---------------------------------------------------------------- cv2.resize's choice and tables
def stage_mode(H0: int, W0: int, h: int, w: int) -> Tuple[int, int, int]:
    """(mode, sx, sy) of cv2.resize(frame, (w, h)) as load_image_rgb_ir calls it (INTER_AREA when shrinking, INTER_LINEAR
    when enlarging): sx, sy are the integer scales of MODE_AREA_FAST."""
    if (h, w) == (H0, W0):
        return MODE_COPY, 0, 0
    if h >= H0 and w >= W0:
        return MODE_LINEAR, 0, 0
    scale_x, scale_y = 1. / (w / W0), 1. / (h / H0)
    isx, isy = int(round(scale_x)), int(round(scale_y))
    if abs(scale_x - isx) < np.finfo(np.float64).eps and abs(scale_y - isy) < np.finfo(np.float64).eps:
        return MODE_AREA_FAST, isx, isy
    return MODE_AREA, 0, 0


@functools.lru_cache(maxsize=64)
def area_taps(src: int, dst: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """computeResizeAreaTab (imgproc/resize.cpp) along one axis: (span int32 (dst, 2) rows {first tap, tap count}, si int32
    (n,), alpha float32 (n,)), the taps of each destination index contiguous and in cv2's order."""
    scale = 1. / (dst / src)
    si, alpha, span = [], [], np.zeros((dst, 2), np.int32)
    for d in range(dst):
        fsx1 = d * scale
        fsx2 = fsx1 + scale
        cell = min(scale, src - fsx1)
        sx1, sx2 = math.ceil(fsx1), math.floor(fsx2)
        sx2 = min(sx2, src - 1)
        sx1 = min(sx1, sx2)
        span[d, 0] = len(si)
        if sx1 - fsx1 > 1e-3:
            si.append(sx1 - 1)
            alpha.append((sx1 - fsx1) / cell)
        for sx in range(sx1, sx2):
            si.append(sx)
            alpha.append(1.0 / cell)
        if fsx2 - sx2 > 1e-3:
            si.append(sx2)
            alpha.append(min(min(fsx2 - sx2, 1.), cell) / cell)
        span[d, 1] = len(si) - span[d, 0]
    return span, np.array(si, np.int32), np.array(alpha, _F32)


def area_table_words(src: int, dst: int) -> np.ndarray:
    """The device form of area_taps: int32 words -- dst {first tap word (relative to the table), count} pairs, then the taps
    as {si, alpha bits} pairs."""
    span, si, alpha = area_taps(src, dst)
    head = span.copy()
    head[:, 0] = 2 * dst + 2 * span[:, 0]
    body = np.stack([si, alpha.view(np.int32)], 1)
    return np.concatenate([head.reshape(-1), body.reshape(-1)]).astype(np.int32)


# ---------------------------------------------------------------- numpy restatement of the kernel
def _area_axis(x: np.ndarray, src: int, dst: int, axis: int) -> np.ndarray:
    """Weighted sums along one axis of a float32 array in cv2's tap order (every product and sum rounded to float32)."""
    span, si, alpha = area_taps(src, dst)
    x = np.moveaxis(x, axis, 0)
    acc = np.zeros((dst,) + x.shape[1:], _F32)
    for t in range(int(span[:, 1].max())):
        live = np.nonzero(span[:, 1] > t)[0]
        k = span[live, 0] + t
        a = alpha[k].reshape((-1,) + (1,) * (x.ndim - 1))
        acc[live] = acc[live] + x[si[k]] * a
    return np.moveaxis(acc, 0, axis)


def resize_area(img: np.ndarray, h: int, w: int) -> np.ndarray:
    """cv2.resize(img, (w, h), INTER_AREA) on a uint8 (H0, W0, 3) image that shrinks along both axes."""
    H0, W0 = img.shape[:2]
    mode, sx, sy = stage_mode(H0, W0, h, w)
    if mode == MODE_AREA_FAST:
        blk = img.reshape(h, sy, w, sx, 3).astype(np.int64).sum((1, 3))
        if sx == 2 and sy == 2:
            return ((blk + 2) >> 2).astype(np.uint8)
        out = np.rint(blk.astype(_F32) * (_F32(1) / _F32(sx * sy)))
    else:
        rows = _area_axis(img.astype(_F32), W0, w, 1)          # per source row: sum over the column taps (cv2's buf)
        span, si, alpha = area_taps(H0, h)
        out = np.zeros((h, w, 3), _F32)
        for t in range(int(span[:, 1].max())):
            live = np.nonzero(span[:, 1] > t)[0]
            k = span[live, 0] + t
            out[live] = out[live] + alpha[k][:, None, None] * rows[si[k]]
        out = np.rint(out)
    return np.clip(out, 0, 255).astype(np.uint8)


def load_resize(img: np.ndarray, h: int, w: int) -> np.ndarray:
    """load_image_rgb_ir's cv2.resize of one decoded frame to (h, w), as the kernel computes it."""
    mode = stage_mode(img.shape[0], img.shape[1], h, w)[0]
    if mode == MODE_COPY:
        return img
    if mode == MODE_LINEAR:
        return resize_fixed(img, h, w)
    return resize_area(img, h, w)


def stage_reference(rgb: np.ndarray, ir: np.ndarray, h: int, w: int, top: int, left: int, H: int, W: int) -> np.ndarray:
    """One sample of the batch in numpy: uint8 (6, H, W) -- both frames resized, placed on the 114 border, BGR -> RGB, CHW."""
    out = np.full((6, H, W), PAD, np.uint8)
    for m, f in enumerate((rgb, ir)):
        out[3 * m:3 * m + 3, top:top + h, left:left + w] = load_resize(f, h, w)[:, :, ::-1].transpose(2, 0, 1)
    return out


# ---------------------------------------------------------------- public interface
Frames = Tuple[object, object]


class ValBatches:
    """Device-side testloader of train.py: LoadMultiModalImagesAndLabels(augment=False, rect=True) + collate_fn.

    labels: per dataset index a float32 (n, 5) array of (cls, x, y, w, h) normalised, as in the label cache.
    frames: index -> (rgb, ir) decoded BGR uint8 (H0, W0, 3) frames of one pair (numpy arrays or CUDA tensors).
    hw0: per dataset index the decoded (H0, W0) -- the label cache's shapes, which are (w, h), reversed.
    paths: per dataset index the RGB image path the batches report (default: the index as a string).
    Iterating yields what the reference loader yields, in its order: (img uint8 (B, 6, H, W) CUDA, targets float32 (n, 6),
    paths, shapes) with shapes[i] = ((h0, w0), ((h / h0, w / w0), (dw, dh))), so ``test.test(dataloader=ValBatches(...))``
    runs unchanged.  Dataset indices are those of the label cache; the batches visit them in the rect order."""

    def __init__(self, labels: Sequence[np.ndarray], frames: Callable[[int], Frames], hw0: Sequence[Tuple[int, int]],
                 img_size: int, batch_size: int = 1, stride: int = 32, pad: float = 0.5, single_cls: bool = False,
                 paths: Optional[Sequence[str]] = None, device=None):
        n = len(labels)
        if n < 1:
            raise ValueError("val: empty dataset")
        if len(hw0) != n or (paths is not None and len(paths) != n):
            raise ValueError(f"val: {n} labels, {len(hw0)} hw0 rows and {len(paths) if paths is not None else n} paths")
        if img_size < 1 or stride < 1 or batch_size < 1:
            raise ValueError("val: img_size, stride and batch_size must be positive")
        for i, lb in enumerate(labels):
            if lb.ndim != 2 or lb.shape[1] != 5:
                raise NotImplementedError(f"val: labels[{i}] has shape {lb.shape}: only (n, 5) box labels are built (no segments)")
        self.hw0 = [(int(h), int(w)) for h, w in hw0]
        if min(min(hw) for hw in self.hw0) < 1:
            raise ValueError("val: every hw0 must be positive")
        self.labels = [np.asarray(lb, dtype=np.float32) for lb in labels]
        if single_cls:
            for x in self.labels:
                x[:, 0] = 0
        self.frames = frames
        self.paths = [str(p) for p in paths] if paths is not None else [str(i) for i in range(n)]
        self.img_size = img_size
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.order, bi, self.batch_shapes = rect_batches(self.hw0, batch_size, img_size, stride, pad)
        self.batch_size = min(batch_size, n)                   # create_dataloader_rgb_ir's loader batch
        self.geometry = [sample_geometry(*self.hw0[i], self.batch_shapes[bi[k]], img_size) for k, i in enumerate(self.order)]
        self.shape_of = [self.batch_shapes[b] for b in bi]
        self.host_seconds = 0.0                      # time spent on the host per batch (labels, tables, uploads, launch)
        self.params = None

    def __len__(self):
        return (len(self.order) + self.batch_size - 1) // self.batch_size

    def batch(self, j: int):
        """Batch j of the rect order: (img, targets, paths, shapes)."""
        t0 = time.perf_counter()
        ks = range(j * self.batch_size, min((j + 1) * self.batch_size, len(self.order)))
        idx = [int(self.order[k]) for k in ks]
        B = len(idx)
        H, W = (int(v) for v in self.shape_of[ks[0]])
        frames = frames_on_device(self.frames, idx, self.device, "val")
        samples = (_lib.ValSample * B)()
        block = ParamBlock()
        per_labels, shapes = [], []
        for b, (k, i) in enumerate(zip(ks, idx)):
            h0, w0 = self.hw0[i]
            rgb, ir = frames[i]
            if tuple(rgb.shape[:2]) != (h0, w0):
                raise ValueError(f"val: frame {i} is {tuple(rgb.shape[:2])}, hw0 says {(h0, w0)}")
            h, w, ratio, pad, top, left = self.geometry[k]
            mode, sx, sy = stage_mode(h0, w0, h, w)
            S = samples[b]
            S.rgb, S.ir = ops._addr(rgb), ops._addr(ir)
            S.H0, S.W0, S.h, S.w, S.top, S.left, S.mode, S.sx, S.sy = h0, w0, h, w, top, left, mode, sx, sy
            if mode == MODE_LINEAR:
                S.xtab = block.table(("linear", w0, w, False), lambda: resize_taps(w0, w))
                S.ytab = block.table(("linear", h0, h, True), lambda: resize_taps(h0, h, vertical=True))
            elif mode == MODE_AREA:
                S.xtab = block.table(("area", w0, w), lambda: area_table_words(w0, w))
                S.ytab = block.table(("area", h0, h), lambda: area_table_words(h0, h))
            per_labels.append(sample_labels(self.labels[i], h, w, ratio, pad, H, W))
            shapes.append(((h0, w0), ((h / h0, w / w0), pad)))
        n_words = block.n_words
        nbytes = int(_lib.lib().icaf_val_stage_params_bytes(B, n_words))
        if nbytes == 0:
            raise ValueError(f"val: unsupported batch {B} / {n_words} table words")
        params = block.upload(samples, (), nbytes, self.device)
        self.params = params                         # the latest batch's parameter block (re-launched by scripts/val_loader_times.py)
        targets = collate(per_labels)
        if not ops.dry_running():
            targets = targets.pin_memory()
        img = torch.empty(B, 6, H, W, dtype=torch.uint8, device=self.device)
        ops._call("icaf_val_stage", _lib.lib().icaf_val_stage, (ops._ptr(params), nbytes, B, H, W, n_words, ops._ptr(img)),
                  {"bytes": float(img.numel() + sum(2 * f[0].numel() for f in frames.values()) + nbytes)})
        self.host_seconds += time.perf_counter() - t0
        return img, targets, tuple(self.paths[i] for i in idx), tuple(shapes)

    def __iter__(self):
        for j in range(len(self)):
            yield self.batch(j)

    def reference(self, j: int, frames_host: Optional[Callable[[int], Frames]] = None):
        """Batch j through the numpy restatement: uint8 (B, 6, H, W) numpy images (targets, paths and shapes are batch()'s)."""
        ks = range(j * self.batch_size, min((j + 1) * self.batch_size, len(self.order)))
        H, W = (int(v) for v in self.shape_of[ks[0]])
        out = []
        for k in ks:
            i = int(self.order[k])
            pair = (frames_host or self.frames)(i)
            rgb, ir = (f.cpu().numpy() if isinstance(f, torch.Tensor) else np.asarray(f) for f in pair)
            h, w, _, _, top, left = self.geometry[k]
            out.append(stage_reference(rgb, ir, h, w, top, left, H, W))
        return np.stack(out)
