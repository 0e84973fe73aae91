"""Training augmentation of RGB/IR pairs on the device: what ``LoadMultiModalImagesAndLabels.__getitem__`` (utils/datasets.py:
948-1024, augment=True) followed by ``collate_fn`` (:1026-1031) hands to the training step, one kernel launch per batch.

The host draws every random number in the reference's order, from Python's ``random`` and numpy's global ``np.random`` --
per sample: the mosaic coin, the mosaic centre, ``random.choices(k=3)``, the 8 ``random.uniform`` of
``random_perspective_rgb_ir``, ``np.random.uniform(-1, 1, 3)`` for the RGB and then the IR ``augment_hsv``, flipud, fliplr -- so
with the same seeds and indices a batch equals the reference's ``dataset[i]`` samples (single-process loading order).  The host
also builds what the kernel needs (the inverted warp matrix as cv2's fixed-point per-column / per-row terms, the mosaic tile
rectangles, the cv2.resize tap tables, the HSV LUTs) and runs the label path in numpy with the reference's own expressions.
The kernel (csrc/augment.cu, ``icaf_augment``) evaluates warp -> mosaic canvas -> resize -> HSV jitter -> flips per output
pixel without materialising the canvas.  JPEG decoding stays with the caller.

Not built (raises NotImplementedError): ``perspective != 0`` (warpPerspective), segment labels, ``rect``, ``--quad``
(collate_fn4), mixup.  :func:`render_reference` is the numpy restatement of the kernel's arithmetic (tests, and the CPU side
of scripts/augment_times.py)."""
from __future__ import annotations

import ctypes as C
import math
import random
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, ops
from .datasets import ParamBlock, frames_on_device, letterbox_geometry, resize_taps

PAD = 114
AB_BITS, INTER_BITS = 10, 5                 # cv2 imgwarp.cpp: AB_SCALE = 1 << 10, INTER_TAB_SIZE = 32
ROUND_DELTA = (1 << AB_BITS) // (1 << INTER_BITS) // 2


# ---------------------------------------------------------------- reference expressions (utils/general.py, utils/datasets.py)
def xywhn2xyxy(x, w=640, h=640, padw=0, padh=0):
    """utils/general.py:342-349 (numpy arrays)."""
    y = np.copy(x)
    y[:, 0] = w * (x[:, 0] - x[:, 2] / 2) + padw
    y[:, 1] = h * (x[:, 1] - x[:, 3] / 2) + padh
    y[:, 2] = w * (x[:, 0] + x[:, 2] / 2) + padw
    y[:, 3] = h * (x[:, 1] + x[:, 3] / 2) + padh
    return y


def xyxy2xywh(x):
    """utils/general.py:322-329 (numpy arrays)."""
    y = np.copy(x)
    y[:, 0] = (x[:, 0] + x[:, 2]) / 2
    y[:, 1] = (x[:, 1] + x[:, 3]) / 2
    y[:, 2] = x[:, 2] - x[:, 0]
    y[:, 3] = x[:, 3] - x[:, 1]
    return y


def box_candidates(box1, box2, wh_thr=2, ar_thr=20, area_thr=0.1, eps=1e-16):
    """utils/datasets.py:1633-1638."""
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + eps), h2 / (w2 + eps))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + eps) > area_thr) & (ar < ar_thr)


def rotation_matrix_2d(angle: float, scale: float) -> np.ndarray:
    """cv2.getRotationMatrix2D(center=(0, 0), angle, scale) (imgproc/imgwarp.cpp), in double."""
    a = angle * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    cx = cy = 0.0
    return np.array([[alpha, beta, (1 - alpha) * cx - beta * cy], [-beta, alpha, beta * cx + (1 - alpha) * cy]])


def load_size(h0: int, w0: int, img_size: int) -> Tuple[int, int]:
    """(h, w) of load_image_rgb_ir (utils/datasets.py:1116-1123): the long side scaled to img_size, truncated."""
    r = img_size / max(h0, w0)
    if r != 1:
        return int(h0 * r), int(w0 * r)
    return h0, w0


def mosaic_rects(i: int, xc: int, yc: int, h: int, w: int, s: int):
    """Canvas rectangle (x1a, y1a, x2a, y2a) and tile offset (x1b, y1b) of mosaic tile i (utils/datasets.py:1233-1246)."""
    if i == 0:
        x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
        x1b, y1b = w - (x2a - x1a), h - (y2a - y1a)
    elif i == 1:
        x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
        x1b, y1b = 0, h - (y2a - y1a)
    elif i == 2:
        x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
        x1b, y1b = w - (x2a - x1a), 0
    else:
        x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
        x1b, y1b = 0, 0
    return (x1a, y1a, x2a, y2a), (x1b, y1b)


def draw_affine(canvas: int, border: Sequence[int], degrees: float, translate: float, scale: float, shear: float,
                perspective: float) -> Tuple[np.ndarray, float]:
    """The matrix of random_perspective_rgb_ir (utils/datasets.py:1544-1576) for a (canvas, canvas) image; consumes the same 8
    random.uniform draws.  Returns (M 3x3, scale s)."""
    height = canvas + border[0] * 2
    width = canvas + border[1] * 2
    Cm = np.eye(3)
    Cm[0, 2] = -canvas / 2
    Cm[1, 2] = -canvas / 2
    P = np.eye(3)
    P[2, 0] = random.uniform(-perspective, perspective)
    P[2, 1] = random.uniform(-perspective, perspective)
    R = np.eye(3)
    a = random.uniform(-degrees, degrees)
    s = random.uniform(1 - scale, 1 + scale)
    R[:2] = rotation_matrix_2d(a, s)
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-shear, shear) * math.pi / 180)
    S[1, 0] = math.tan(random.uniform(-shear, shear) * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - translate, 0.5 + translate) * width
    T[1, 2] = random.uniform(0.5 - translate, 0.5 + translate) * height
    M = T @ S @ R @ P @ Cm
    return M, s


def warp_tables(M: np.ndarray, dsize: int) -> np.ndarray:
    """cv2.warpAffine(src, M[:2], (dsize, dsize)) fixed-point terms: int32 (4, dsize) rows adelta[x], bdelta[x], X0[y], Y0[y] of
    the inverted matrix (imgwarp.cpp: invertAffineTransform in double, cvRound(M0 x 1024), cvRound((M1 y + M2) 1024) + 16)."""
    m = [float(v) for v in np.asarray(M, dtype=np.float64)[:2].reshape(-1)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1. / D if D != 0 else 0.
    A11, A22 = m[4] * D, m[0] * D
    m[0] = A11
    m[1] *= -D
    m[3] *= -D
    m[4] = A22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    x = np.arange(dsize, dtype=np.float64)
    ab = float(1 << AB_BITS)
    out = np.empty((4, dsize), dtype=np.int64)
    out[0] = np.rint(m[0] * x * ab)
    out[1] = np.rint(m[3] * x * ab)
    out[2] = np.rint((m[1] * x + m[2]) * ab) + ROUND_DELTA
    out[3] = np.rint((m[4] * x + m[5]) * ab) + ROUND_DELTA
    return out.astype(np.int32)


def hsv_luts(r: np.ndarray) -> np.ndarray:
    """augment_hsv's three LUTs (utils/datasets.py:1134-1137) for gains r: uint8 (3, 256)."""
    dtype = np.uint8
    x = np.arange(0, 256, dtype=np.int16)
    lut_hue = ((x * r[0]) % 180).astype(dtype)
    lut_sat = np.clip(x * r[1], 0, 255).astype(dtype)
    lut_val = np.clip(x * r[2], 0, 255).astype(dtype)
    return np.stack([lut_hue, lut_sat, lut_val])


# ---------------------------------------------------------------- per-sample draws and geometry
class SampleDraw:
    """The random decisions of one sample, in the order __getitem__ makes them."""
    __slots__ = ("index", "mosaic", "xc", "yc", "indices", "M", "scale", "gains", "flipud", "fliplr")


def draw_sample(index: int, n: int, img_size: int, hyp: Dict[str, float]) -> SampleDraw:
    """Consume Python `random` / `np.random` exactly as LoadMultiModalImagesAndLabels.__getitem__(index) does with
    augment=True, rect=False (n = dataset length)."""
    d = SampleDraw()
    d.index = index
    d.mosaic = random.random() < hyp['mosaic']
    d.xc = d.yc = 0
    d.indices = [index]
    d.M, d.scale = None, 1.0
    if d.mosaic:
        s = img_size
        border = [-img_size // 2, -img_size // 2]
        d.yc, d.xc = [int(random.uniform(-x, 2 * s + x)) for x in border]
        d.indices = [index] + random.choices(range(n), k=3)
        d.M, d.scale = draw_affine(2 * s, border, hyp['degrees'], hyp['translate'], hyp['scale'], hyp['shear'], hyp['perspective'])
    d.gains = [np.random.uniform(-1, 1, 3) * [hyp['hsv_h'], hyp['hsv_s'], hyp['hsv_v']] + 1 for _ in range(2)]   # RGB, then IR
    d.flipud = random.random() < hyp['flipud']
    d.fliplr = random.random() < hyp['fliplr']
    return d


def sample_layout(d: SampleDraw, shapes: Dict[int, Tuple[int, int]], img_size: int):
    """Tiles [(index, (h, w), (x1a, y1a, x2a, y2a), (x1b, y1b), (padw, padh))] of the canvas, canvas side, and for the
    letterbox branch (ratio, pad).  shapes: index -> decoded (H0, W0)."""
    s = img_size
    if d.mosaic:
        tiles = []
        for i, idx in enumerate(d.indices):
            h, w = load_size(*shapes[idx], s)
            a, b = mosaic_rects(i, d.xc, d.yc, h, w, s)
            tiles.append((idx, (h, w), a, b, (a[0] - b[0], a[1] - b[1])))
        return tiles, 2 * s, None
    h, w = load_size(*shapes[d.index], s)
    (nw, nh), ratio, pad, (top, bottom, left, right) = letterbox_geometry((h, w), s, scaleup=True)
    if (nh, nw) != (h, w):
        raise NotImplementedError(f"augment: a {h}x{w} load_image result letterboxed to {s} needs a second resize")
    return [(d.index, (h, w), (left, top, left + w, top + h), (0, 0), (left, top))], s, (ratio, pad)


def sample_labels(d: SampleDraw, labels: Sequence[np.ndarray], tiles, letterbox, img_size: int) -> np.ndarray:
    """Label path of __getitem__ for one sample (float32 (nL, 5) rows cls, x, y, w, h normalised), with the reference's
    expressions and dtypes: xywhn2xyxy per tile, clip to 2s, the 4-corner warp + box_candidates (load_mosaic_RGB_IR /
    random_perspective_rgb_ir), or the letterbox placement; then xyxy2xywh, normalisation, flips."""
    s = img_size
    if d.mosaic:
        labels4 = []
        for idx, (h, w), _, _, (padw, padh) in tiles:
            lb = labels[idx].copy()
            if lb.size:
                lb[:, 1:] = xywhn2xyxy(lb[:, 1:], w, h, padw, padh)
            labels4.append(lb)
        labels4 = np.concatenate(labels4, 0)
        np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
        targets = labels4
        M = d.M
        width = height = 2 * s + (-img_size // 2) * 2
        n = len(targets)
        if n:
            xy = np.ones((n * 4, 3))
            xy[:, :2] = targets[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)
            xy = xy @ M.T
            xy = xy[:, :2].reshape(n, 8)
            x = xy[:, [0, 2, 4, 6]]
            y = xy[:, [1, 3, 5, 7]]
            new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
            new[:, [0, 2]] = new[:, [0, 2]].clip(0, width)
            new[:, [1, 3]] = new[:, [1, 3]].clip(0, height)
            i = box_candidates(box1=targets[:, 1:5].T * d.scale, box2=new.T, area_thr=0.10)
            targets = targets[i]
            targets[:, 1:5] = new[i]
        lab = targets
    else:
        ratio, pad = letterbox
        (h, w) = tiles[0][1]
        lab = labels[d.index].copy()
        if lab.size:
            lab[:, 1:] = xywhn2xyxy(lab[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    nL = len(lab)
    if nL:
        lab[:, 1:5] = xyxy2xywh(lab[:, 1:5])
        lab[:, [2, 4]] /= s
        lab[:, [1, 3]] /= s
        if d.flipud:
            lab[:, 2] = 1 - lab[:, 2]
        if d.fliplr:
            lab[:, 1] = 1 - lab[:, 1]
    return lab


def collate_targets(per_sample: Sequence[np.ndarray]) -> np.ndarray:
    """collate_fn (utils/datasets.py:1026-1031) on the labels_out of each sample: float32 (n, 6) rows (image, cls, x, y, w, h)."""
    outs = []
    for i, lab in enumerate(per_sample):
        t = torch.zeros((len(lab), 6))
        if len(lab):
            t[:, 1:] = torch.from_numpy(lab)
        t[:, 0] = i
        outs.append(t)
    return torch.cat(outs, 0).numpy() if outs else np.zeros((0, 6), np.float32)


def check_hyp(hyp: Dict[str, float]) -> None:
    if hyp.get('perspective', 0.0) != 0:
        raise NotImplementedError("augment: perspective != 0 (cv2.warpPerspective) is not built")
    if hyp.get('mixup', 0.0) > 0:
        raise NotImplementedError("augment: mixup is not built")


# ---------------------------------------------------------------- numpy restatement of the kernel
def resize_fixed(img: np.ndarray, h: int, w: int) -> np.ndarray:
    """cv2.resize(img, (w, h), INTER_LINEAR) on uint8 with the resize_taps tables and cv2's integer arithmetic."""
    H0, W0 = img.shape[:2]
    if (h, w) == (H0, W0):
        return img
    xt, yt = resize_taps(W0, w).astype(np.int64), resize_taps(H0, h, vertical=True).astype(np.int64)
    f = img.astype(np.int64)
    hz = f[:, xt[:, 0]] * xt[None, :, 2, None] + f[:, xt[:, 1]] * xt[None, :, 3, None]
    r0, r1 = hz[yt[:, 0]], hz[yt[:, 1]]
    out = (((yt[:, 2, None, None] * (r0 >> 4)) >> 16) + ((yt[:, 3, None, None] * (r1 >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


def warp_fixed(canvas: np.ndarray, tab: np.ndarray, dsize: int) -> np.ndarray:
    """cv2.warpAffine(canvas, M[:2], (dsize, dsize), borderValue=(114,)*3) from warp_tables(M): fixed-point INTER_LINEAR."""
    tab = tab.astype(np.int64)
    X = (tab[2][:, None] + tab[0][None, :]) >> INTER_BITS
    Y = (tab[3][:, None] + tab[1][None, :]) >> INTER_BITS
    sx, sy = np.clip(X >> INTER_BITS, -32768, 32767), np.clip(Y >> INTER_BITS, -32768, 32767)
    ax, ay = X & 31, Y & 31
    Hc, Wc = canvas.shape[:2]
    acc = np.zeros((dsize, dsize, 3), np.int64)
    for dy, dx, wgt in ((0, 0, (32 - ay) * (32 - ax)), (0, 1, (32 - ay) * ax), (1, 0, ay * (32 - ax)), (1, 1, ay * ax)):
        xx, yy = sx + dx, sy + dy
        inside = (xx >= 0) & (yy >= 0) & (xx < Wc) & (yy < Hc)
        v = np.where(inside[..., None], canvas[np.clip(yy, 0, Hc - 1), np.clip(xx, 0, Wc - 1)].astype(np.int64), PAD)
        acc += v * (wgt * 32)[..., None]
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)


def _hsv_tables():
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i > 0, np.rint((255 << 12) / np.maximum(i, 1)), 0).astype(np.int64)
        hdiv = np.where(i > 0, np.rint((180 << 12) / (6. * np.maximum(i, 1))), 0).astype(np.int64)
    return sdiv, hdiv


def bgr2hsv_fixed(img: np.ndarray) -> np.ndarray:
    """cv2.cvtColor(img, COLOR_BGR2HSV) on uint8 (hsv_shift = 12 integer tables)."""
    sdiv, hdiv = _hsv_tables()
    f = img.astype(np.int64)
    b, g, r = f[..., 0], f[..., 1], f[..., 2]
    v = np.maximum(np.maximum(b, g), r)
    vmin = np.minimum(np.minimum(b, g), r)
    diff = v - vmin
    vr = np.where(v == r, -1, 0)
    vg = np.where(v == g, -1, 0)
    s = (diff * sdiv[v] + (1 << 11)) >> 12
    h = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + (~vg & (r - g + 4 * diff))))
    h = (h * hdiv[diff] + (1 << 11)) >> 12
    h += np.where(h < 0, 180, 0)
    return np.stack([h, s, v], -1).astype(np.uint8)


_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def hsv2bgr_fixed(hsv: np.ndarray) -> np.ndarray:
    """cv2.cvtColor(hsv, COLOR_HSV2BGR) on uint8 as cv2's vectorised path computes it: float32, h * (6/180), s and v * (1/255),
    v(1 - s h) and v(1 - s(1 - h)) with the inner product fused (an FMA, emulated exactly in double), x 255, truncated."""
    f32 = np.float32
    H = hsv[..., 0].astype(f32)
    s = hsv[..., 1].astype(f32) * f32(1.0 / 255.0)
    v = hsv[..., 2].astype(f32) * f32(1.0 / 255.0)
    hs = H * f32(6.0 / 180.0)
    sector = np.trunc(hs)
    fr = hs - sector
    sector = sector.astype(np.int64)
    sector[(sector < 0) | (sector >= 6)] = 0
    one = np.float64(1.0)
    s64 = s.astype(np.float64)
    tab = np.stack([v, v * (f32(1) - s), v * (-s64 * fr.astype(np.float64) + one).astype(f32),
                    v * (-s64 * (f32(1) - fr).astype(np.float64) + one).astype(f32)], -1)
    out = np.take_along_axis(tab, _SECTOR[sector], -1)
    return np.minimum(np.trunc(out * f32(255.0)), 255).astype(np.uint8)


def hsv_jitter_fixed(img: np.ndarray, lut: np.ndarray) -> np.ndarray:
    """augment_hsv with the LUTs of hsv_luts: BGR -> HSV -> LUT -> BGR."""
    hsv = bgr2hsv_fixed(img)
    hsv = np.stack([lut[c][hsv[..., c]] for c in range(3)], -1)
    return hsv2bgr_fixed(hsv)


def render_reference(d: SampleDraw, tiles, canvas: int, frames: Dict[int, Tuple[np.ndarray, np.ndarray]], img_size: int):
    """The kernel's arithmetic for one sample in numpy (the canvas is materialised here): uint8 (3, s, s) RGB and IR."""
    s = img_size
    out = []
    for m in range(2):
        cv = np.full((canvas, canvas, 3), PAD, dtype=np.uint8)
        for idx, (h, w), (x1a, y1a, x2a, y2a), (x1b, y1b), _ in tiles:
            t = resize_fixed(frames[idx][m], h, w)
            cv[y1a:y2a, x1a:x2a] = t[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
        img = warp_fixed(cv, warp_tables(d.M, s), s) if d.mosaic else cv
        img = hsv_jitter_fixed(img, hsv_luts(d.gains[m]))
        if d.flipud:
            img = img[::-1]
        if d.fliplr:
            img = img[:, ::-1]
        out.append(np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1)))
    return out[0], out[1]


# ---------------------------------------------------------------- public interface
Frames = Tuple[object, object]


class Augment:
    """Device-side LoadMultiModalImagesAndLabels(augment=True) + collate_fn for training batches.

    labels: per dataset index a float32 (n, 5) array of (cls, x, y, w, h) normalised, as in the label cache.
    frames: index -> (rgb, ir) decoded BGR uint8 (H0, W0, 3) frames of one pair (numpy arrays or CUDA tensors).
    hyp: the hyperparameter dict of hyp.scratch.yaml (mosaic, degrees, translate, scale, shear, perspective, hsv_*, flip*).
    ``aug(indices)`` -> (rgb, ir, targets): uint8 (B, 3, s, s) CUDA tensors and float32 (n, 6) CUDA targets, ready for
    TrainStep / GraphedTrainStep."""

    def __init__(self, labels: Sequence[np.ndarray], frames: Callable[[int], Frames], img_size: int = 640,
                 hyp: Optional[Dict[str, float]] = None, device=None, rect: bool = False, quad: bool = False):
        if rect:
            raise NotImplementedError("augment: rectangular batches (rect=True) are not built")
        if quad:
            raise NotImplementedError("augment: --quad (collate_fn4 / 4-image batches) is not built")
        if hyp is None:
            raise ValueError("augment: hyp is required (e.g. data/hyp.scratch.yaml)")
        check_hyp(hyp)
        for i, lb in enumerate(labels):
            if lb.ndim != 2 or lb.shape[1] != 5:
                raise NotImplementedError(f"augment: labels[{i}] has shape {lb.shape}: only (n, 5) box labels are built (no segments)")
        if img_size % 2:
            raise ValueError("augment: img_size must be even")
        self.labels = [np.asarray(lb, dtype=np.float32) for lb in labels]
        self.frames = frames
        self.img_size = img_size
        self.hyp = dict(hyp)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.host_seconds = 0.0                      # time spent in __call__ on the host (draws, tables, labels, uploads)
        self.params = None

    def __len__(self):
        return len(self.labels)

    def draw(self, indices: Sequence[int]) -> List[SampleDraw]:
        return [draw_sample(int(i), len(self.labels), self.img_size, self.hyp) for i in indices]

    def __call__(self, indices: Sequence[int], out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        import time
        t0 = time.perf_counter()
        s, B = self.img_size, len(indices)
        if B < 1:
            raise ValueError("augment: empty batch")
        draws = self.draw(indices)
        needed = sorted({i for d in draws for i in d.indices})
        frames = frames_on_device(self.frames, needed, self.device, "augment")
        shapes = {i: (int(frames[i][0].shape[0]), int(frames[i][0].shape[1])) for i in needed}
        samples = (_lib.AugSample * B)()
        warp = np.zeros((B, 4, s), dtype=np.int32)
        block = ParamBlock()
        per_labels = []
        for b, d in enumerate(draws):
            tiles, canvas, lbox = sample_layout(d, shapes, s)
            S = samples[b]
            S.ntiles, S.canvas, S.warp, S.flipud, S.fliplr = len(tiles), canvas, int(d.mosaic), int(d.flipud), int(d.fliplr)
            for t, (idx, (h, w), (x1a, y1a, x2a, y2a), (x1b, y1b), _) in enumerate(tiles):
                T = S.tile[t]
                H0, W0 = shapes[idx]
                T.rgb, T.ir = ops._addr(frames[idx][0]), ops._addr(frames[idx][1])
                T.H0, T.W0, T.h, T.w = H0, W0, h, w
                T.x1a, T.y1a, T.x2a, T.y2a, T.x1b, T.y1b = x1a, y1a, x2a, y2a, x1b, y1b
                if (h, w) != (H0, W0):                # offsets in int4 rows: every resize_taps row is 4 words
                    T.xtab = block.table((W0, w, False), lambda: resize_taps(W0, w)) // 4
                    T.ytab = block.table((H0, h, True), lambda: resize_taps(H0, h, vertical=True)) // 4
            lut = np.stack([hsv_luts(g) for g in d.gains])
            C.memmove(C.addressof(S.lut), lut.ctypes.data, lut.nbytes)
            if d.mosaic:
                warp[b] = warp_tables(d.M, s)
            per_labels.append(sample_labels(d, self.labels, tiles, lbox, s))
        n_taps = block.n_words // 4
        nbytes = int(_lib.lib().icaf_augment_params_bytes(B, s, n_taps))
        if nbytes == 0:
            raise ValueError(f"augment: unsupported batch {B} / size {s}")
        params = block.upload(samples, (warp,), nbytes, self.device)
        self.params = params                         # the latest batch's parameter block (re-launched by scripts/augment_times.py)
        targets = torch.from_numpy(collate_targets(per_labels)).to(self.device, non_blocking=True)
        if out is None:
            rgb = torch.empty(B, 3, s, s, dtype=torch.uint8, device=self.device)
            ir = torch.empty_like(rgb)
        else:
            rgb, ir = out
            for o in (rgb, ir):
                if tuple(o.shape) != (B, 3, s, s) or o.dtype != torch.uint8 or not o.is_contiguous():
                    raise ValueError(f"augment: `out` must be contiguous uint8 {(B, 3, s, s)}")
        self.host_seconds += time.perf_counter() - t0
        ops._call("icaf_augment", _lib.lib().icaf_augment,
                  (ops._ptr(params), nbytes, B, s, n_taps, ops._ptr(rgb), ops._ptr(ir)),
                  {"bytes": float(2 * rgb.numel() + nbytes)})
        return rgb, ir, targets

    def reference(self, indices: Sequence[int], frames_host: Optional[Dict[int, Frames]] = None):
        """The same batch through the numpy restatement (consumes the random state like __call__): uint8 (B, 3, s, s) RGB and IR
        numpy arrays and float32 (n, 6) targets."""
        s = self.img_size
        draws = self.draw(indices)
        needed = sorted({i for d in draws for i in d.indices})
        fr = {}
        for i in needed:
            pair = frames_host[i] if frames_host is not None else self.frames(i)
            fr[i] = tuple(f.cpu().numpy() if isinstance(f, torch.Tensor) else np.asarray(f) for f in pair)
        shapes = {i: fr[i][0].shape[:2] for i in needed}
        rgb, ir, labs = [], [], []
        for d in draws:
            tiles, canvas, lbox = sample_layout(d, shapes, s)
            a, b = render_reference(d, tiles, canvas, fr, s)
            rgb.append(a)
            ir.append(b)
            labs.append(sample_labels(d, self.labels, tiles, lbox, s))
        return np.stack(rgb), np.stack(ir), collate_targets(labs)
