"""Post-processing helpers with the reference's names and signatures (utils/general.py), running on the device.

``non_max_suppression`` is what ``detect_twostream.py:86`` / ``test.py:139`` call on the model's first output.  The
suppression itself (candidate filter, confidence sort, greedy IoU suppression, max_det cut) is one kernel launch for the
whole batch (icaf_nms); this wrapper only slices the fixed-capacity result into the reference's list-of-(n,6) form, which
costs the single device->host read of the per-image counts that the list form makes unavoidable.  Use
:func:`icafusion_b200.ops.nms` directly to stay asynchronous (e.g. inside a CUDA graph)."""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import ops


def xywh2xyxy(x: torch.Tensor) -> torch.Tensor:
    """reference: utils/general.py:332-339 (host-side helper; the NMS kernel does this conversion itself)."""
    y = x.clone()
    y[:, 0] = x[:, 0] - x[:, 2] / 2
    y[:, 1] = x[:, 1] - x[:, 3] / 2
    y[:, 2] = x[:, 0] + x[:, 2] / 2
    y[:, 3] = x[:, 1] + x[:, 3] / 2
    return y


def non_max_suppression(prediction: torch.Tensor, conf_thres: float = 0.25, iou_thres: float = 0.45,
                        classes: Optional[Sequence[int]] = None, agnostic: bool = False, multi_label: bool = False,
                        labels=()) -> List[torch.Tensor]:
    """reference: utils/general.py:518-607.  Returns a list with one (n,6) fp32 tensor [xyxy, conf, cls] per image.
    `multi_label` (test.py:139) keeps every (box, class) pair above conf_thres; it is off when nc == 1, as in the reference."""
    if labels:
        raise NotImplementedError("non_max_suppression: autolabelling (labels=...) is outside the hot path built here")
    if not prediction.is_cuda:
        raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
    z = prediction if prediction.dtype == torch.float16 else prediction.to(torch.float16)
    det, count = ops.nms(z.contiguous(), conf_thres, iou_thres, agnostic, classes, multi_label=multi_label)
    counts = count.tolist()                       # the one host sync of the list-shaped API
    return [det[i, :n] for i, n in enumerate(counts)]
