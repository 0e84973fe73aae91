"""Confluence with the reference's names and signatures (utils/confluence.py), running on the device.

Confluence is the reference's alternative to NMS: boxes of one class are clustered by a normalised Manhattan distance
instead of IoU, and the box with the smallest confidence-weighted distance to its neighbours represents each cluster.
The whole batch is one launch group (icaf_confluence); these wrappers only size its output so that nothing is cut and
slice it into the reference's forms.  Use :func:`icafusion_b200.ops.confluence` directly to stay asynchronous (e.g. inside
a CUDA graph: ``GraphedDetector(..., confluence=dict(conf_thres=0.1, p_thres=0.5))``)."""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch

from . import ops

MIN_CONF = 2.5e-4     # below 2e-4 the reference's selection scan (starting at 10000) can find no box and raises


def confluence_process(prediction: torch.Tensor, conf_thres: float = 0.1, p_thres: float = 0.6) -> List[Optional[torch.Tensor]]:
    """reference: utils/confluence.py:50-106.  prediction: CUDA fp16 or fp32 (B, R, nc+5) decoded predictions.  Returns one
    fp32 (n, 6) tensor [x1, y1, x2, y2, conf, cls] per image, rows in ascending candidate order, or None for an image
    without candidates.  Like the reference, nothing is cut at max_det (300 there is unused)."""
    if not prediction.is_cuda:
        raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
    if prediction.dtype not in (torch.float16, torch.float32):
        raise ValueError(f"confluence_process: fp16 or fp32 predictions, got {prediction.dtype}")
    z = prediction.contiguous()
    B, R, no = z.shape
    det, count = ops.confluence(z, conf_thres, p_thres, max_det=R * (no - 5))
    counts = count.tolist()                       # the one host sync of the list-shaped API
    return [det[i, :n] if n else None for i, n in enumerate(counts)]


def confluence(prediction: np.ndarray, class_num: int, p_thres: float = 0.6) -> np.ndarray:
    """reference: utils/confluence.py:109-193.  prediction: (n, 6) rows [x1, y1, x2, y2, conf, cls] whose values are exactly
    representable in fp32 (what confluence_process passes the reference's version); rows of class 0 .. class_num-1 are
    clustered on the device.  Returns the kept row indices in ascending order, as np.unique(keep) does."""
    a = np.asarray(prediction)
    if a.ndim != 2 or a.shape[1] < 6:
        raise ValueError(f"confluence: expected (n, 6) detection rows, got shape {a.shape}")
    f = np.ascontiguousarray(a[:, :6], dtype=np.float32)
    if not np.array_equal(f.astype(a.dtype), a[:, :6], equal_nan=True):
        raise ValueError("confluence: the rows must be exactly representable in fp32")
    if a.shape[0] == 0 or class_num < 1:
        return np.unique([])
    in_class = np.isin(f[:, 5], np.arange(class_num, dtype=np.float32))
    if (f[in_class, 4] < MIN_CONF).any() or np.isnan(f[in_class, 4]).any():
        raise ValueError(f"confluence: every conf must be >= {MIN_CONF}")
    n = f.shape[0]
    z = torch.from_numpy(f)[None].cuda()
    index = torch.empty(1, n, dtype=torch.int32, device=z.device)
    _, count = ops.confluence(z, p_thres=p_thres, max_det=n, index=index, class_num=int(class_num))
    return index[0, :int(count[0])].cpu().numpy().astype(np.int64)
