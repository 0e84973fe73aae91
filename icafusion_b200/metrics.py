"""Validation metrics with the reference's names and signatures (utils/metrics.py), on the host in numpy.

They run once per validation, over the statistics test.test() gathers from the device, so there is no hot path here.  The
numbers equal the reference's exactly: the same numpy operations in the same order and dtypes (``tp`` bool, ``conf`` and
``pred_cls`` float32, ``target_cls`` float64).  ``plot=True`` draws nothing (matplotlib is not a dependency) and changes no
result."""
from __future__ import annotations

import numpy as np


def fitness(x):
    """reference: utils/metrics.py:12-15 -- mAP@0.5 of the rows [tp, fp, fn, f1, mp, mr, map50, map]."""
    w = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    return (x[:, :8] * w).sum(1)


def compute_ap(recall, precision):
    """reference: utils/metrics.py:85-110.  101-point interpolated area under the precision envelope.
    Returns (ap, envelope precision, recall with sentinels)."""
    mrec = np.concatenate(([0.0], recall, [recall[-1] + 0.01]))
    mpre = np.flip(np.maximum.accumulate(np.flip(np.concatenate(([1.0], precision, [0.0])))))
    x = np.linspace(0, 1, 101)
    return np.trapezoid(np.interp(x, mrec, mpre), x), mpre, mrec


def ap_per_class(tp, conf, pred_cls, target_cls, plot=False, save_dir=".", names=()):
    """reference: utils/metrics.py:18-82 (the variant that also returns TP / FP / FN).  tp: bool (n, niou); conf, pred_cls:
    (n,); target_cls: (nt,).  Returns (tp, fp, fn, p, r, ap (nc, niou), f1, classes int32), every per-class vector taken at
    the confidence of the best mean F1.  As in the reference, tp / fp / fn are derived from the label count of the last
    class."""
    order = np.argsort(-conf)
    tp, conf, pred_cls = tp[order], conf[order], pred_cls[order]
    classes = np.unique(target_cls)
    nc = classes.shape[0]
    px = np.linspace(0, 1, 1000)
    ap, p, r = np.zeros((nc, tp.shape[1])), np.zeros((nc, 1000)), np.zeros((nc, 1000))
    n_l = 0
    for ci, c in enumerate(classes):
        sel = pred_cls == c
        n_l = (target_cls == c).sum()
        if sel.sum() == 0 or n_l == 0:
            continue
        tpc = tp[sel].cumsum(0)
        fpc = (1 - tp[sel]).cumsum(0)
        recall = tpc / (n_l + 1e-16)
        precision = tpc / (tpc + fpc)
        r[ci] = np.interp(-px, -conf[sel], recall[:, 0], left=0)
        p[ci] = np.interp(-px, -conf[sel], precision[:, 0], left=1)
        for j in range(tp.shape[1]):
            ap[ci, j] = compute_ap(recall[:, j], precision[:, j])[0]
    f1 = 2 * p * r / (p + r + 1e-16)
    best = f1.mean(0).argmax()
    tps = (r * n_l).round()
    fn = n_l - tps
    fp = (tps / (p + 1e-16) - tps).round()
    return tps[:, best], fp[:, best], fn[:, best], p[:, best], r[:, best], ap, f1[:, best], classes.astype("int32")
