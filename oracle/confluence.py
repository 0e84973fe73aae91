"""Vectorised fp64 restatement of the reference's Confluence (utils/confluence.py:50-193), for the tests.

Same candidates (fp32 cls * obj and xywh2xyxy, one per (row, class) above conf_thres in row-major order), same fp64
distances on the widened fp32 values, same selection: per class, the first box with the smallest
min over p < 2 of p / conf (0 without such a neighbour) is kept, and it and every box with p < p_thres leave.  The whole
distance matrix of a class is formed once; each live row keeps its minimum over the live neighbours, recomputed only
when the neighbour that gave it leaves."""
from __future__ import annotations

import numpy as np


def pair_p(box: np.ndarray) -> np.ndarray:
    """(n, 4) fp64 boxes [x1, y1, x2, y2] -> (n, n) p, as confluence.py:140-162 computes it for each ordered pair."""
    def axis(a1, a2):
        A1, A2, B1, B2 = a1[:, None], a2[:, None], a1[None, :], a2[None, :]
        mn = np.minimum(np.minimum(A1, A2), np.minimum(B1, B2))
        mx = np.maximum(np.maximum(A1, A2), np.maximum(B1, B2))
        d = mx - mn
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.abs((A1 - mn) / d - (B1 - mn) / d), np.abs((A2 - mn) / d - (B2 - mn) / d)
    x1, x2 = axis(box[:, 0], box[:, 2])
    y1, y2 = axis(box[:, 1], box[:, 3])
    return x1 + x2 + y1 + y2


def confluence(dets: np.ndarray, class_num: int, p_thres: float = 0.6) -> np.ndarray:
    """(n, 6) rows [x1, y1, x2, y2, conf, cls] -> kept row indices, ascending (confluence.py:109-193)."""
    infos = dets.astype(np.float64)
    keep = []
    for c in range(class_num):
        idx = np.nonzero(infos[:, 5] == c)[0]
        if not len(idx):
            continue
        P = pair_p(infos[idx, :4])
        with np.errstate(invalid="ignore"):
            P2 = np.where(P < 2, P, np.inf)                 # the neighbours that count toward value
        np.fill_diagonal(P2, np.inf)
        conf = infos[idx, 4]
        live = np.ones(len(idx), dtype=bool)
        part = P2.argmin(1)                               # the row minimum's neighbour; rescanned once it leaves
        rowmin = P2[np.arange(len(idx)), part]
        while live.any():
            # min(p / conf) == min(p) / conf: correctly rounded division by a positive constant is monotone
            value = np.where(np.isfinite(rowmin), rowmin / conf, 0.0)
            value[~live] = np.inf
            best = int(np.argmin(value))                  # the first of the smallest, like the reference's strict < scan
            keep.append(int(idx[best]))
            with np.errstate(invalid="ignore"):
                live &= ~(P[best] < p_thres)
            live[best] = False
            stale = np.nonzero(live & np.isfinite(rowmin) & ~live[part])[0]
            if len(stale):
                sub = np.where(live[None, :], P2[stale], np.inf)
                part[stale] = sub.argmin(1)
                rowmin[stale] = sub[np.arange(len(stale)), part[stale]]
    return np.unique(np.array(keep, dtype=np.int64))


def candidates(x: np.ndarray, conf_thres: float) -> np.ndarray:
    """One image's fp32 (R, nc+5) predictions -> fp32 (n, 6) candidate rows [x1, y1, x2, y2, conf, cls] in the
    reference's order (confluence.py:73-91)."""
    x = x.astype(np.float32)
    thr = np.float32(conf_thres)
    x = x[x[:, 4] > thr]
    nc = x.shape[1] - 5
    conf = x[:, 5:] * x[:, 4:5]
    box = np.stack([x[:, 0] - x[:, 2] / np.float32(2), x[:, 1] - x[:, 3] / np.float32(2),
                    x[:, 0] + x[:, 2] / np.float32(2), x[:, 1] + x[:, 3] / np.float32(2)], 1)
    if nc > 1:
        i, j = np.nonzero(conf > thr)
        return np.concatenate([box[i], conf[i, j, None], j[:, None].astype(np.float32)], 1)
    keep = conf[:, 0] > thr
    return np.concatenate([box, conf, np.zeros_like(conf)], 1)[keep]


def confluence_process(prediction: np.ndarray, conf_thres: float = 0.1, p_thres: float = 0.6):
    """(B, R, nc+5) predictions (fp16 widened to fp32, fp32 as is) -> per image fp32 (n, 6) kept rows or None."""
    out = []
    for x in np.asarray(prediction):
        d = candidates(x.astype(np.float32), conf_thres)
        out.append(d[confluence(d, x.shape[1] - 5, p_thres)] if len(d) else None)
    return out
