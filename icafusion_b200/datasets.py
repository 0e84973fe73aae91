"""Input-side helpers with the reference's names (utils/datasets.py), running on the device.

``letterbox`` is what ``LoadImages.__next__`` applies to every decoded frame before the model sees it
(datasets.py:235-239: letterbox -> BGR to RGB -> HWC to CHW); here a batch of RGB/IR frames is letterboxed, channel-swapped
and transposed by one kernel (icaf_letterbox), bit-exact against the cv2 pipeline (cv2.resize INTER_LINEAR is fixed-point;
its tap tables are rebuilt on the host by :func:`resize_taps`).  The result is the uint8 (B,3,H,W) tensor the detector's
staging kernel (/255 -> fp16, space-to-depth) consumes."""
from __future__ import annotations

import ctypes as C
import functools
from typing import Callable, Sequence, Tuple

import numpy as np
import torch

from . import _lib, ops

INTER_RESIZE_COEF_SCALE = 2048          # OpenCV: INTER_RESIZE_COEF_BITS = 11


@functools.lru_cache(maxsize=64)
def resize_taps(src: int, dst: int, vertical: bool = False) -> np.ndarray:
    """cv2.resize(..., INTER_LINEAR) taps along one axis for uint8 images: int32 (dst, 4) rows {i0, i1, w0, w1}, weights x 2048
    (imgproc/resize.cpp: f = (d + 0.5) * scale - 0.5 in double -> float, floor, cvRound(w * 2048)).  Horizontally a tap that
    falls off the image is snapped onto the edge pixel with weight 1; vertically OpenCV keeps the fractional weights and only
    clamps the two row indices (so an edge row is blended with itself, which rounds differently)."""
    scale = 1.0 / (dst / src)                                   # double, like inv_scale -> scale in cv::resize
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    i0 = np.floor(f).astype(np.int32)
    f = f - i0.astype(np.float32)
    if not vertical:
        lo = i0 < 0
        f[lo], i0[lo] = 0.0, 0
        hi = i0 >= src - 1
        f[hi], i0[hi] = 0.0, src - 1
    w1 = np.rint(f * np.float32(INTER_RESIZE_COEF_SCALE)).astype(np.int32)             # saturate_cast<short> = round half to even
    w0 = np.rint((np.float32(1.0) - f) * np.float32(INTER_RESIZE_COEF_SCALE)).astype(np.int32)
    i1 = np.clip(i0 + 1, 0, src - 1).astype(np.int32)
    i0 = np.clip(i0, 0, src - 1).astype(np.int32)
    return np.ascontiguousarray(np.stack([i0, i1, w0, w1], 1).astype(np.int32))


def _align16(n: int) -> int:
    return (n + 15) // 16 * 16


class ParamBlock:
    """The parameter block of one staging launch (icaf_val_stage, icaf_augment): a ctypes struct array at 0, then int32
    regions, each 16-byte aligned; the last region holds the resize tables, interned by key."""

    def __init__(self):
        self.offsets, self.tables, self.n_words = {}, [], 0

    def table(self, key, make: Callable[[], np.ndarray]) -> int:
        """Offset in int32 words of the table `key` in the table region; make() builds it on the key's first use.  Every
        table starts 16-byte aligned."""
        if key not in self.offsets:
            t = np.asarray(make(), dtype=np.int32).reshape(-1)
            self.offsets[key] = self.n_words
            self.tables.append(np.pad(t, (0, -t.size % 4)))
            self.n_words += self.tables[-1].size
        return self.offsets[key]

    def upload(self, structs, regions: Sequence[np.ndarray], nbytes: int, device) -> torch.Tensor:
        """The block on `device`: structs, then `regions` and the table region, assembled in a pinned buffer (plain host
        memory in a dry run) of nbytes, the size the library computes for this layout."""
        blob = torch.zeros(nbytes, dtype=torch.uint8, pin_memory=not ops.dry_running())
        bn = blob.numpy()
        bn[:C.sizeof(structs)] = np.frombuffer(structs, dtype=np.uint8)
        off = _align16(C.sizeof(structs))
        for r in (*regions, *self.tables):
            bn[off:off + r.nbytes] = r.view(np.uint8).reshape(-1)
            off = _align16(off + r.nbytes)
        if off != nbytes:
            raise ValueError(f"parameter block: the layout takes {off} bytes, the library expects {nbytes}")
        return blob.to(device, non_blocking=True)


_TAPS_ON_DEVICE = {}


def _device_taps(src: int, dst: int, vertical: bool, device) -> torch.Tensor:
    """Tap table on the device, cached per (geometry, device): a CUDA-graph capture must not see the upload."""
    key = (src, dst, vertical, str(device))
    t = _TAPS_ON_DEVICE.get(key)
    if t is None:
        t = _TAPS_ON_DEVICE[key] = torch.from_numpy(resize_taps(src, dst, vertical)).to(device)
    return t


def frames_on_device(frames: Callable[[int], Tuple[object, object]], needed: Sequence[int], device, what: str):
    """index -> (rgb, ir) device uint8 frames for the decoded BGR uint8 (H0, W0, 3) pairs frames(index) returns (numpy arrays
    or tensors); host frames go up in one pinned copy.  `what` names the caller in error messages."""
    got, host = {}, []
    for idx in needed:
        rgb, ir = frames(idx)
        for f in (rgb, ir):
            if f.dtype not in (np.uint8, torch.uint8) or f.ndim != 3 or f.shape[2] != 3:
                raise ValueError(f"{what}: frame {idx} must be uint8 (H0, W0, 3) BGR, got {f.dtype} {tuple(f.shape)}")
        if tuple(rgb.shape) != tuple(ir.shape):
            raise ValueError(f"{what}: RGB and IR frames of index {idx} differ in size: {tuple(rgb.shape)} vs {tuple(ir.shape)}")
        got[idx] = [rgb, ir]
        for m, f in enumerate((rgb, ir)):
            if isinstance(f, torch.Tensor):
                if not ops.on_device(f):
                    f = f.numpy()
                else:
                    got[idx][m] = f.contiguous()
                    continue
            host.append((idx, m, np.ascontiguousarray(f)))
    if host:
        sizes = [a.nbytes for _, _, a in host]
        offs = np.concatenate([[0], np.cumsum([(n + 255) // 256 * 256 for n in sizes])]).astype(np.int64)
        buf = torch.empty(int(offs[-1]), dtype=torch.uint8, pin_memory=not ops.dry_running())
        bn = buf.numpy()
        for (idx, m, a), o in zip(host, offs):
            bn[o:o + a.nbytes] = a.reshape(-1)
        dev = buf.to(device, non_blocking=True)
        for (idx, m, a), o in zip(host, offs):
            got[idx][m] = dev[o:o + a.nbytes].view(a.shape)
    return {k: (v[0], v[1]) for k, v in got.items()}


def letterbox_geometry(shape: Tuple[int, int], new_shape=(640, 640), scaleup: bool = True):
    """reference arithmetic of utils/datasets.py:1404-1424 -> (new_unpad (w, h), ratio, (dw, dh), (top, bottom, left, right))."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = (new_shape[1] - new_unpad[0]) / 2, (new_shape[0] - new_unpad[1]) / 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, (r, r), (dw, dh), (top, bottom, left, right)


def letterbox(img: torch.Tensor, new_shape=(640, 640), color=(114, 114, 114), auto: bool = True, scaleFill: bool = False,
              scaleup: bool = True, stride: int = 32, out: torch.Tensor = None):
    """reference: utils/datasets.py:1404-1427 (`auto` / `scaleFill` / `stride` are accepted and, as in the reference, unused:
    its minimum-rectangle branch is commented out).  img: CUDA uint8 (B, H0, W0, 3) BGR frames (or (H0, W0, 3)).
    Returns (uint8 (B, 3, H, W) RGB planar -- letterboxed, channel-swapped, transposed: what datasets.py:238-239 hands to the
    model --, ratio, (dw, dh))."""
    if img.dim() == 3:
        img = img[None]
    if img.dim() != 4 or img.shape[3] != 3 or img.dtype != torch.uint8 or not ops.on_device(img):
        raise ValueError(f"letterbox: expected CUDA uint8 (B, H0, W0, 3) frames, got {img.dtype} {tuple(img.shape)} on {img.device}")
    if len(set(color)) != 1:
        raise NotImplementedError("letterbox: the border colour must be grey (one value for the three channels)")
    img = img.contiguous()
    B, H0, W0, _ = img.shape
    (new_w, new_h), ratio, pad, (top, bottom, left, right) = letterbox_geometry((H0, W0), new_shape, scaleup)
    H, W = new_h + top + bottom, new_w + left + right
    if out is None:
        out = torch.empty(B, 3, H, W, dtype=torch.uint8, device=img.device)
    elif tuple(out.shape) != (B, 3, H, W) or out.dtype != torch.uint8 or not out.is_contiguous():
        raise ValueError(f"letterbox: `out` must be contiguous uint8 {(B, 3, H, W)}")
    xt = yt = None
    if (new_h, new_w) != (H0, W0):
        xt = _device_taps(W0, new_w, False, img.device)
        yt = _device_taps(H0, new_h, True, img.device)
    ops._call("icaf_letterbox", _lib.lib().icaf_letterbox,
              (ops._ptr(img), B, H0, W0, ops._ptr(out), H, W, top, left, new_h, new_w, ops._ptr(xt), ops._ptr(yt), int(color[0])),
              {"bytes": float(img.numel() + out.numel())})
    return out, ratio, pad
