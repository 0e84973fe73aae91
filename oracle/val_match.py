"""CPU oracle of test.py:196-227 -- which detections of one image are true positives -- TEST INFRASTRUCTURE.

An independent torch restatement with the reference's structure: one image at a time, one label class at a time, fp32 CPU
tensor arithmetic in the reference's operation order (scale_coords divides by the gain).  The device kernel
(icaf_match_detections) does the same work for a whole batch in one launch; the tests hold the two equal bit for bit.
"""
from __future__ import annotations

import torch


def scale_boxes(boxes, h0, w0, gain, padw, padh):
    """utils/general.py:386-407 with ratio_pad = ((gain, gain), (padw, padh)), on a copy of an (n, 4) xyxy fp32 tensor."""
    b = boxes.clone()
    b[:, [0, 2]] -= padw
    b[:, [1, 3]] -= padh
    b /= gain
    b[:, [0, 2]] = b[:, [0, 2]].clamp(0, w0)
    b[:, [1, 3]] = b[:, [1, 3]].clamp(0, h0)
    return b


def pair_iou(a, b):
    """utils/general.py:455-477: (n, 4) x (m, 4) xyxy -> (n, m)."""
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    iw = (torch.min(a[:, None, 2], b[None, :, 2]) - torch.max(a[:, None, 0], b[None, :, 0])).clamp(0)
    ih = (torch.min(a[:, None, 3], b[None, :, 3]) - torch.max(a[:, None, 1], b[None, :, 1])).clamp(0)
    inter = iw * ih
    return inter / (area_a[:, None] + area_b[None, :] - inter)


def match_image(pred, labels, shape, iouv, single_cls=False):
    """pred: fp32 (n, 6) NMS rows [x1, y1, x2, y2, conf, cls] in batch pixels; labels: fp32 (nl, 5) [cls, x, y, w, h] in batch
    pixels (test.py:136 applied); shape: ((h0, w0), ((gain, gain), (padw, padh))).  Returns (correct bool (n, niou),
    pred with the class column as test.py appends it, native boxes fp32 (n, 4))."""
    (h0, w0), ((gain, _), (padw, padh)) = shape
    pred = pred.clone()
    if single_cls:
        pred[:, 5] = 0
    native = scale_boxes(pred[:, :4], h0, w0, gain, padw, padh)
    correct = torch.zeros(pred.shape[0], iouv.numel(), dtype=torch.bool)
    if not labels.shape[0] or not pred.shape[0]:
        return correct, pred, native
    xy, half = labels[:, 1:3], labels[:, 3:5] / 2
    tbox = scale_boxes(torch.cat((xy - half, xy + half), 1), h0, w0, gain, padw, padh)
    taken = set()
    for c in torch.unique(labels[:, 0]).tolist():
        li = torch.where(labels[:, 0] == c)[0]
        pi = torch.where(pred[:, 5] == c)[0]
        if not pi.numel():
            continue
        best, arg = pair_iou(native[pi], tbox[li]).max(1)
        for k in range(pi.numel()):               # confidence (row) order
            lab = int(li[arg[k]])
            if best[k] > iouv[0] and lab not in taken:
                taken.add(lab)
                correct[pi[k]] = best[k] > iouv
    return correct, pred, native


def match_batch(dets, targets, height, width, shapes, iouv, single_cls=False):
    """dets: one (n, 6) tensor per image; targets: fp32 (T, 6) [image, cls, x, y, w, h] normalised.  Returns one
    (correct, pred, native) per image."""
    px = targets.clone()
    px[:, 2:] *= torch.tensor([width, height, width, height], dtype=torch.float32)
    return [match_image(d, px[px[:, 0] == i, 1:], shapes[i], iouv, single_cls) for i, d in enumerate(dets)]
