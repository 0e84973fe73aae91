"""Throughput of the device training augmentation (icafusion_b200.augment.Augment) at B = 16, s = 640, against a single-thread
cv2 restatement of the same transform.

Dataset: 64 synthetic 512 x 640 RGB/IR pairs (the KAIST / FLIR frame size; at s = 640 the load_image resize is the identity)
with 0-8 boxes each, hyp.scratch.  Decoding is not part of either path: the frames are already decoded, on the device for the
device path ("frames on device") and, as a second variant, in host memory (uploaded by Augment in one pinned copy per batch).

Reported per variant: pairs/s of whole batches (host draws + label path + parameter upload + kernel, ending in a device
synchronise), the host's share of that time (Augment.host_seconds: the random draws, warp tables, LUTs and labels), and the
kernel alone (CUDA events around re-launches of the last batch's icaf_augment).  The cv2 path builds the same sample with
cv2.resize / np.full canvas / cv2.warpAffine / cvtColor + LUT / flips / transpose on one thread (cv2.setNumThreads(1)).
The card name, power limit and max SM clock are printed with the numbers.

    python scripts/augment_times.py [--batches 20] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HYP_SCRATCH = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0,
                   flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.0)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown (nvidia-smi printed nothing)"
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def _dataset(n, seed=3):
    import numpy as np
    g = np.random.default_rng(seed)
    frames, labels = {}, []
    yy, xx = np.mgrid[0:512, 0:640]
    for k in range(n):
        base = (xx * (k + 3) // 7 + yy * (k + 5) // 9) % 256
        rgb = np.stack([(base + 60 * c + g.integers(0, 24, base.shape)) % 256 for c in range(3)], -1).astype(np.uint8)
        ir = np.repeat(((base // 2 + g.integers(0, 16, base.shape)) % 256)[..., None], 3, -1).astype(np.uint8)
        frames[k] = (rgb, ir)
        nb = int(g.integers(0, 9))
        wh = g.uniform(0.02, 0.4, (nb, 2))
        labels.append(np.concatenate([g.integers(0, 2, (nb, 1)), g.uniform(wh / 2, 1 - wh / 2), wh], 1).astype(np.float32))
    return frames, labels


def cv2_batch(aug, indices, frames):
    """The same transform with cv2 calls, one sample after another (draws and labels from icafusion_b200.augment)."""
    import cv2
    import numpy as np
    from icafusion_b200.augment import hsv_luts, sample_labels, sample_layout, collate_targets
    s = aug.img_size
    draws = aug.draw(indices)
    shapes = {i: frames[i][0].shape[:2] for d in draws for i in d.indices}
    imgs, labs = [], []
    for d in draws:
        tiles, canvas, lbox = sample_layout(d, shapes, s)
        pair = []
        for m in range(2):
            cv = np.full((canvas, canvas, 3), 114, dtype=np.uint8)
            for idx, (h, w), (x1a, y1a, x2a, y2a), (x1b, y1b), _ in tiles:
                f = frames[idx][m]
                if (h, w) != f.shape[:2]:
                    f = cv2.resize(f, (w, h), interpolation=cv2.INTER_LINEAR)
                cv[y1a:y2a, x1a:x2a] = f[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
            img = cv2.warpAffine(cv, d.M[:2], dsize=(s, s), borderValue=(114, 114, 114)) if d.mosaic else cv
            lut = hsv_luts(d.gains[m])
            hue, sat, val = cv2.split(cv2.cvtColor(img, cv2.COLOR_BGR2HSV))
            img = cv2.cvtColor(cv2.merge((cv2.LUT(hue, lut[0]), cv2.LUT(sat, lut[1]), cv2.LUT(val, lut[2]))), cv2.COLOR_HSV2BGR)
            if d.flipud:
                img = np.flipud(img)
            if d.fliplr:
                img = np.fliplr(img)
            pair.append(np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1)))
        imgs.append(np.concatenate(pair, 0))
        labs.append(sample_labels(d, aug.labels, tiles, lbox, s))
    return np.stack(imgs), collate_targets(labs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("augment_times.py measures the device path: no CUDA device")
    import cv2
    from icafusion_b200 import _lib
    from icafusion_b200.augment import Augment
    dev = torch.device("cuda:0")
    frames, labels = _dataset(64)
    frames_dev = {k: tuple(torch.from_numpy(f).to(dev) for f in v) for k, v in frames.items()}
    B, s = a.batch, a.size
    res = {"card": _card(), "batch": B, "img_size": s, "hyp": "hyp.scratch", "frames": "512x640"}
    g = np.random.default_rng(0)
    batches = [list(g.choice(64, B, replace=False)) for _ in range(a.batches + 3)]
    for tag, src in (("frames_on_device", frames_dev), ("frames_on_host", frames)):
        aug = Augment(labels, src.__getitem__, s, HYP_SCRATCH, device=dev)
        random.seed(0)
        np.random.seed(0)
        for idx in batches[:3]:                                           # warm-up
            aug(idx)
        torch.cuda.synchronize()
        aug.host_seconds = 0.0
        t0 = time.perf_counter()
        for idx in batches[3:]:
            rgb, ir, tg = aug(idx)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[tag] = {"pairs_per_s": B * a.batches / dt, "ms_per_batch": 1e3 * dt / a.batches,
                    "host_share": aug.host_seconds / dt, "host_ms_per_batch": 1e3 * aug.host_seconds / a.batches}
    # kernel alone: re-launch icaf_augment on the parameter block of one batch (same frames, same outputs)
    L = _lib.lib()
    aug = Augment(labels, frames_dev.__getitem__, s, HYP_SCRATCH, device=dev)
    from icafusion_b200 import ops
    calls = []
    saved = ops._call

    def spy(name, fn, args, work=None):
        if name == "icaf_augment":
            calls.append(args)
        return saved(name, fn, args, work)
    ops._call = spy
    try:
        random.seed(1)
        np.random.seed(1)
        rgb, ir, tg = aug(batches[0])
    finally:
        ops._call = saved
    args = calls[-1]                      # its parameter block stays alive as aug.params until the next batch
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(5):
        _lib.check(L.icaf_augment(*args, st), "icaf_augment")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 200
    e0.record()
    for _ in range(reps):
        _lib.check(L.icaf_augment(*args, st), "icaf_augment")
    e1.record()
    torch.cuda.synchronize()
    k_ms = e0.elapsed_time(e1) / reps
    out_bytes = 2 * B * 3 * s * s
    res["kernel"] = {"ms": k_ms, "pairs_per_s": B / (k_ms * 1e-3), "output_GBps": out_bytes / (k_ms * 1e-3) / 1e9}
    # single-thread cv2 restatement of the same transform
    cv2.setNumThreads(1)
    aug_c = Augment(labels, frames.__getitem__, s, HYP_SCRATCH, device=dev)
    random.seed(0)
    np.random.seed(0)
    cv2_batch(aug_c, batches[0], frames)
    nb = max(2, a.batches // 4)
    t0 = time.perf_counter()
    for idx in batches[3:3 + nb]:
        cv2_batch(aug_c, idx, frames)
    dt = time.perf_counter() - t0
    res["cv2_single_thread"] = {"pairs_per_s": B * nb / dt, "ms_per_batch": 1e3 * dt / nb, "cv2": cv2.__version__}
    # same draws: the cv2 path and the device path agree on this batch
    random.seed(1)
    np.random.seed(1)
    img, t = cv2_batch(aug_c, batches[0], frames)
    res["device_equals_cv2"] = bool(np.array_equal(img[:, :3], rgb.cpu().numpy()) and np.array_equal(img[:, 3:], ir.cpu().numpy())
                                    and np.array_equal(t, tg.cpu().numpy()))
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
