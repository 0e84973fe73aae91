"""Time of the device NMS on test.py's validation batch: B = 32 images at its rect shape 544 x 672 (22 491 rows), nc = 3
(FLIR), conf 0.001 / iou 0.6 -- every row x class pair is a candidate (67 473 per image), cut to max_nms = 30 000.

Reported, each as ms per call from CUDA events around `--reps` calls after warm-up:
  * multi_label: ops.nms(..., multi_label=True) (icaf_nms_multi_label: filter, radix sort, suppression)
  * best_class:  ops.nms(...) on the same batch (icaf_nms: filter, rank sort, suppression)
  * reference_torchvision: the reference's per-image expression (utils/general.py:540-602, multi-label branch, with
    torchvision.ops.nms) restated on the GPU tensors, when torchvision imports; "not measured" otherwise.
The inputs are seeded synthetic predictions (uniform boxes, scores in [0.05, 0.95]).  The card name, power limit and max
SM clock are printed with the numbers.

    python scripts/nms_times.py [--reps 20] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown (nvidia-smi printed nothing)"
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def predictions(B, R, nc, device, seed=7):
    import torch
    g = torch.Generator().manual_seed(seed)
    z = torch.empty(B, R, 5 + nc)
    z[..., 0] = torch.rand(B, R, generator=g) * 672
    z[..., 1] = torch.rand(B, R, generator=g) * 544
    z[..., 2:4] = torch.rand(B, R, 2, generator=g) * 120 + 4
    z[..., 4:] = torch.rand(B, R, 1 + nc, generator=g) * 0.9 + 0.05
    return z.half().to(device)


def reference_multilabel(prediction, conf_thres, iou_thres):
    """utils/general.py:540-602 for multi_label=True, classes=None, agnostic=False, restated on the given tensors."""
    import torch
    import torchvision
    max_wh, max_det, max_nms = 4096, 300, 30000
    xc = prediction[..., 4] > conf_thres
    output = [torch.zeros((0, 6), device=prediction.device)] * prediction.shape[0]
    for xi, x in enumerate(prediction):
        x = x[xc[xi]]
        if not x.shape[0]:
            continue
        x[:, 5:] *= x[:, 4:5]
        box = x[:, :4].clone()
        box[:, 0] = x[:, 0] - x[:, 2] / 2
        box[:, 1] = x[:, 1] - x[:, 3] / 2
        box[:, 2] = x[:, 0] + x[:, 2] / 2
        box[:, 3] = x[:, 1] + x[:, 3] / 2
        i, j = (x[:, 5:] > conf_thres).nonzero(as_tuple=False).T
        x = torch.cat((box[i], x[i, j + 5, None], j[:, None].float()), 1)
        n = x.shape[0]
        if not n:
            continue
        elif n > max_nms:
            x = x[x[:, 4].argsort(descending=True)[:max_nms]]
        c = x[:, 5:6] * max_wh
        i = torchvision.ops.nms(x[:, :4] + c, x[:, 4], iou_thres)[:max_det]
        output[xi] = x[i]
    return output


def _time(fn, reps, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rows", type=int, default=22491)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("nms_times.py measures the device path: no CUDA device")
    from icafusion_b200 import ops
    dev = torch.device("cuda:0")
    B, R, nc, conf, iou = a.batch, a.rows, 3, 0.001, 0.6
    z = predictions(B, R, nc, dev)
    res = {"card": _card(), "batch": B, "rows": R, "nc": nc, "conf_thres": conf, "iou_thres": iou, "reps": a.reps}
    bufs = {}
    for tag, ml in (("multi_label", True), ("best_class", False)):
        det = torch.zeros(B, 300, 6, dtype=torch.float32, device=dev)
        count = torch.zeros(B, dtype=torch.int32, device=dev)
        ws = torch.empty((ops.nms_workspace_bytes(B, R, 5 + nc, ml) + 7) // 8, dtype=torch.int64, device=dev)
        res[tag] = {"ms": _time(lambda: ops.nms(z, conf, iou, det=det, count=count, workspace=ws, multi_label=ml), a.reps),
                    "workspace_MB": ws.numel() * 8 / 1e6}
        bufs[tag] = (det, count)
    try:
        import torchvision  # noqa: F401
    except Exception as e:  # noqa: BLE001
        res["reference_torchvision"] = f"not measured (torchvision does not import: {e})"
    else:
        zf = z.float()
        res["reference_torchvision"] = {"ms": _time(lambda: reference_multilabel(zf.clone(), conf, iou), max(2, a.reps // 4), 1),
                                        "torchvision": torchvision.__version__}
        ref = reference_multilabel(zf.clone(), conf, iou)
        det, count = bufs["multi_label"]
        cnt = count.tolist()
        res["reference_torchvision"]["images_equal_device"] = sum(
            int(cnt[b] == r.shape[0] and torch.equal(det[b, :cnt[b]], r)) for b, r in enumerate(ref))
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
