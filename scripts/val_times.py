"""Validation timings on the GPU (prints one JSON line):

* ``match_ms``: icaf_match_detections per batch (CUDA events over 200 launches) on a FLIR detector's own multi-label NMS
  output, B = 32 at test.py's rect shape 544 x 672 with 10 labels per image;
* ``dropin_img_s`` / ``loop_img_s``: whole-validation images/s of icafusion_b200.test.test against test.py's per-image loop
  (test.py:144-230, restated here on the same device forward and NMS: per image a boolean mask, `unique`, `nonzero`,
  `.item()` / `.tolist()` / `.cpu()` host round trips), yolov5l FLIR with synthetic weights at 544 x 672, at B = 1
  (train.py's setting) and B = 32;
* the card name, power limit and max SM clock, read in the same run.

    python scripts/val_times.py [--images 64]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from icafusion_b200 import Model, ops  # noqa: E402
from icafusion_b200 import test as T  # noqa: E402
from icafusion_b200.metrics import ap_per_class  # noqa: E402
from icafusion_b200.synth import load_synth  # noqa: E402

H, W = 544, 672
SHAPE = ((512, 640), ((1.0, 1.0), (16.0, 16.0)))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def batches(n_images, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in range(n_images // B):
        img = (torch.rand(B, 6, H, W, generator=g) * 255).to(torch.uint8).pin_memory()
        tg = torch.cat([torch.arange(B).repeat_interleave(10)[:, None].float(), torch.randint(0, 3, (B * 10, 1), generator=g).float(),
                        torch.rand(B * 10, 2, generator=g) * 0.8 + 0.1, torch.rand(B * 10, 2, generator=g) * 0.2 + 0.02], 1)
        out.append((img, tg.pin_memory(), [f"/d/{k}_{i}.jpg" for i in range(B)], [SHAPE] * B))
    return out


def reference_loop(model, loader, dev, iouv):
    """test.py:115-230 on the device: forward, NMS, then the per-image Python loop; returns the stats list."""
    stats = []
    for img, targets, paths, shapes in loader:
        img = img.to(dev, non_blocking=True)
        targets = targets.to(dev)
        nb, _, height, width = img.shape
        with torch.no_grad():
            z = model(img[:, :3], img[:, 3:])[0]
            targets[:, 2:] *= torch.tensor([width, height, width, height], device=dev)
            det, count = ops.nms(z, 0.001, 0.5, multi_label=True)
            out = [det[i, :n] for i, n in enumerate(count.tolist())]
        for si, pred in enumerate(out):
            labels = targets[targets[:, 0] == si, 1:]
            nl = len(labels)
            tcls = labels[:, 0].tolist() if nl else []
            if len(pred) == 0:
                continue
            (h0, w0), ((gain, _), (pw, ph)) = shapes[si]
            predn = pred.clone()
            predn[:, [0, 2]] -= pw
            predn[:, [1, 3]] -= ph
            predn[:, :4] /= gain
            predn[:, [0, 2]] = predn[:, [0, 2]].clamp(0, w0)
            predn[:, [1, 3]] = predn[:, [1, 3]].clamp(0, h0)
            correct = torch.zeros(pred.shape[0], iouv.numel(), dtype=torch.bool, device=dev)
            if nl:
                detected = []
                tbox = torch.cat((labels[:, 1:3] - labels[:, 3:5] / 2, labels[:, 1:3] + labels[:, 3:5] / 2), 1)
                tbox[:, [0, 2]] = ((tbox[:, [0, 2]] - pw) / gain).clamp(0, w0)
                tbox[:, [1, 3]] = ((tbox[:, [1, 3]] - ph) / gain).clamp(0, h0)
                for cls in torch.unique(labels[:, 0]):
                    ti = (cls == labels[:, 0]).nonzero(as_tuple=False).view(-1)
                    pi = (cls == pred[:, 5]).nonzero(as_tuple=False).view(-1)
                    if pi.shape[0]:
                        a, b = predn[pi, :4], tbox[ti]
                        inter = (torch.min(a[:, None, 2:], b[:, 2:]) - torch.max(a[:, None, :2], b[:, :2])).clamp(0).prod(2)
                        area = lambda x: (x[:, 2] - x[:, 0]) * (x[:, 3] - x[:, 1])  # noqa: E731
                        ious, i = (inter / (area(a)[:, None] + area(b) - inter)).max(1)
                        done = set()
                        for j in (ious > iouv[0]).nonzero(as_tuple=False):
                            d = ti[i[j]]
                            if d.item() not in done:
                                done.add(d.item())
                                detected.append(d)
                                correct[pi[j]] = ious[j] > iouv
                                if len(detected) == nl:
                                    break
            stats.append((correct.cpu(), pred[:, 4].cpu(), pred[:, 5].cpu(), tcls))
    return stats


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    model = Model("yolov5l_Transfusion_FLIR").eval()
    load_synth(model, 3)
    model = model.fuse().to(dev)
    iouv = torch.linspace(0.5, 0.95, 10).to(dev)
    res = {"card": card()}

    # kernel time per batch: B = 32 on the detector's own NMS output
    (img, tg, _, shapes), = batches(32, 32, seed=1)
    with torch.no_grad():
        z = model(img[:, :3].to(dev), img[:, 3:].to(dev))[0]
    det, count = ops.nms(z, 0.001, 0.5, multi_label=True)
    tg_d, rp = tg.to(dev), T.ratio_pad_rows(shapes).to(dev)
    correct = torch.empty(32, det.shape[1], 10, dtype=torch.uint8, device=dev)
    ws = torch.empty(tg.shape[0], dtype=torch.int32, device=dev)
    for _ in range(10):
        ops.match_detections(det, count, tg_d, rp, H, W, iouv, correct=correct, workspace=ws)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        ops.match_detections(det, count, tg_d, rp, H, W, iouv, correct=correct, workspace=ws)
    e1.record()
    torch.cuda.synchronize()
    res["match_ms_b32"] = round(e0.elapsed_time(e1) / 200, 4)
    res["detections_b32"] = int(count.sum())

    data = {"nc": 3, "names": ["person", "car", "bicycle"]}
    with tempfile.TemporaryDirectory() as tmp:
        for B in (1, 32):
            loader = batches(max(args.images, B) // B * B, B, seed=2)
            n = len(loader) * B
            t_drop = timed(lambda: T.test(data, model=model, dataloader=loader, save_dir=tmp, batch_size=B, imgsz=W))
            t_loop = timed(lambda: ap_per_class(*[np.concatenate(x, 0) for x in zip(*reference_loop(model, loader, dev, iouv))]))
            res[f"dropin_img_s_b{B}"] = round(n / t_drop, 1)
            res[f"loop_img_s_b{B}"] = round(n / t_loop, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
