"""Focal branch of the oracle's ComputeLoss (utils/loss.py:37-64 FocalLoss, switched on by hyp fl_gamma at :341-344).

The reference wraps its two BCEWithLogitsLoss criteria in FocalLoss and leaves build_targets and the reductions alone.
`compute_loss` does the same around `icaf_oracle.compute_loss`: it runs that restatement with its BCE replaced by the
focal form, so target assignment, CIoU and the means stay the code the plain-BCE goldens pin.  fl_gamma <= 0 calls
`icaf_oracle.compute_loss` unchanged, like the reference's `if g > 0`.
"""
from __future__ import annotations

import contextlib
import types

import torch
import torch.nn.functional as F

from oracle import icaf_oracle as O

ALPHA = 0.25          # FocalLoss(loss_fcn, gamma, alpha=0.25): ComputeLoss passes only gamma


def focal_bce_with_logits(x, y, gamma: float, pos_weight=None, alpha: float = ALPHA):
    """FocalLoss(nn.BCEWithLogitsLoss(pos_weight), gamma, alpha).forward with reduction 'mean', in the reference's order."""
    loss = F.binary_cross_entropy_with_logits(x, y, pos_weight=pos_weight, reduction="none")
    pred_prob = torch.sigmoid(x)
    p_t = y * pred_prob + (1 - y) * (1 - pred_prob)
    alpha_factor = y * alpha + (1 - y) * (1 - alpha)
    modulating_factor = (1.0 - p_t) ** gamma
    loss = loss * (alpha_factor * modulating_factor)
    return loss.mean()


@contextlib.contextmanager
def _focal_criterion(gamma: float):
    """icaf_oracle.compute_loss reaches its BCE through the module name `F`: point that name at a namespace whose
    binary_cross_entropy_with_logits is the focal form for the duration of one call."""
    real = O.F
    ns = types.SimpleNamespace(**{k: getattr(real, k) for k in dir(real) if not k.startswith("__")})
    ns.binary_cross_entropy_with_logits = lambda x, y, pos_weight=None: focal_bce_with_logits(x, y, gamma, pos_weight)
    O.F = ns
    try:
        yield
    finally:
        O.F = real


def compute_loss(p, targets, anchors, hyp: dict, gr: float = 1.0):
    """icaf_oracle.compute_loss with the reference's focal branch: same arguments and return value."""
    g = float(hyp.get("fl_gamma", 0.0))
    if not g > 0:
        return O.compute_loss(p, targets, anchors, hyp, gr)
    with _focal_criterion(g):
        return O.compute_loss(p, targets, anchors, hyp, gr)
