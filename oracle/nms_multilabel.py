"""CPU oracle of the multi-label branch of utils/general.py:518-607 non_max_suppression -- TEST INFRASTRUCTURE.

What test.py:139 calls (`multi_label=True`) for detectors with nc > 1: one row per (i, j) of
`(x[:, 5:] > conf_thres).nonzero()` (:566-568), in that row-major order.  The reference cuts to max_nms with
`argsort(descending=True)`, which is not stable on the CPU; this restatement cuts with a STABLE descending sort, so ties
keep the nonzero() order (the order the device kernel produces).  The suppression is oracle.icaf_oracle.greedy_nms.
With nc == 1 the reference switches the branch off itself (:535), and so does this function.
"""
from __future__ import annotations

import torch

from oracle import icaf_oracle as O


def non_max_suppression_multilabel(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, max_det=300):
    """Returns one (n,6) fp32 tensor [x1, y1, x2, y2, conf, cls] per image."""
    if prediction.shape[2] - 5 <= 1:
        return O.non_max_suppression(prediction, conf_thres, iou_thres, classes=classes, agnostic=agnostic, max_det=max_det)
    max_wh, max_nms = 4096, 30000
    out = []
    for x in prediction.float():
        x = x[x[:, 4] > conf_thres].clone()
        if not x.shape[0]:
            out.append(torch.zeros((0, 6)))
            continue
        x[:, 5:] *= x[:, 4:5]
        box = x[:, :4].clone()
        box[:, 0] = x[:, 0] - x[:, 2] / 2
        box[:, 1] = x[:, 1] - x[:, 3] / 2
        box[:, 2] = x[:, 0] + x[:, 2] / 2
        box[:, 3] = x[:, 1] + x[:, 3] / 2
        i, j = (x[:, 5:] > conf_thres).nonzero(as_tuple=False).T
        x = torch.cat((box[i], x[i, j + 5, None], j[:, None].float()), 1)
        if classes is not None:
            x = x[(x[:, 5:6] == torch.tensor(classes, dtype=x.dtype)).any(1)]
        n = x.shape[0]
        if not n:
            out.append(torch.zeros((0, 6)))
            continue
        if n > max_nms:
            x = x[torch.sort(x[:, 4], descending=True, stable=True)[1][:max_nms]]
        c = x[:, 5:6] * (0 if agnostic else max_wh)
        i = O.greedy_nms(x[:, :4] + c, x[:, 4], iou_thres)[:max_det]
        out.append(x[i])
    return out
