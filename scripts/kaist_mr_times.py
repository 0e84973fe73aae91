"""KAIST miss-rate timings on the GPU (prints one JSON line):

* ``mlpd_ms`` / ``arcnn_ms``: icaf_kaist_mr on the MLPD result file (5,939 detections) and on ARCNN's detections with a
  score of at least 0.001 (19,951 of its 76,743; the fixture keeps those), packed layout, with the curves evaluate()
  returns, CUDA events over 50 calls;
* ``dense_ms``: icaf_kaist_mr on a seeded 2,252 x 300-detection dense input (test.test's layout at conf_thres 0.001, its
  worst case: every image full), CUDA events over 50 calls;
* ``test_added_ms``: the added wall time of test.test(mr_annotations=...) over test.test on a seeded loader of 2,252
  images (B = 32, a stub detector whose NMS keeps 300 detections per image), median of alternating runs;
* the card name, power limit and max SM clock, read in the same run.

For comparison, the reference's pure-Python evaluate() on the CPU of the development machine (not an H100 host) took
4.2 s (MLPD, 5,939 detections), 7.1 s (MBNet, 12,937), 8.2 s (MSDS-RCNN, 13,547), 28.1 s (ARCNN, 76,743) and 10.8 s
(ARCNN at score >= 0.001, 19,951).

    python scripts/kaist_mr_times.py
"""
from __future__ import annotations

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

from icafusion_b200 import kaist_eval as K  # noqa: E402
from icafusion_b200 import ops  # noqa: E402
from icafusion_b200 import test as T  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def event_ms(fn, reps=50, warmup=5):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


class _Stub(torch.nn.Module):
    """Decoded predictions around the annotation boxes plus noise: (B, R, 6) fp16, the same for every batch."""

    def __init__(self, z):
        super().__init__()
        self.z = z
        self.anchor = torch.nn.Parameter(torch.zeros(1))
        self.names = ["person"]

    def forward(self, x, x2, augment=False):
        return self.z[:x.shape[0]], None, []


def main():
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ann = K.KaistAnnotations(os.path.join(GOLDEN, "kaist_annotation.json.gz"), dev)
    out = {"gpu": card()}
    # result files, packed
    for key, name in (("mlpd_ms", "kaist_mr_MLPD.txt.gz"), ("arcnn_ms", "kaist_mr_ARCNN_conf0.001.txt.gz")):
        rows, span, mx = K.load_detections(os.path.join(GOLDEN, name), ann)
        r, s = torch.from_numpy(rows).to(dev), torch.from_numpy(span).to(dev)
        ws = torch.empty(int(ops._lib.lib().icaf_kaist_mr_workspace_bytes(ann.images, int(ann.id.numel()), r.shape[0])) + 256,
                         dtype=torch.uint8, device=dev)
        out[key] = event_ms(lambda: ops.kaist_mr(ann, r, s, mx, curves=True, workspace=ws))
    # 2,252 x 300 dense: jittered gts and random boxes, scores uniform
    g = np.random.Generator(np.random.PCG64(5))
    per = 300
    dense = np.empty((ann.images, per, 5))
    dense[..., 0] = g.uniform(0, 600, (ann.images, per))
    dense[..., 1] = g.uniform(0, 450, (ann.images, per))
    dense[..., 2] = g.uniform(10, 60, (ann.images, per))
    dense[..., 3] = dense[..., 2] * g.uniform(1.8, 2.8, (ann.images, per))
    dense[..., 4] = g.uniform(0.001, 1, (ann.images, per))
    box, off = ann.host["box"], ann.host["offset"]
    for p in range(ann.images):
        n = off[p + 1] - off[p]
        dense[p, :n, :4] = box[off[p]:off[p + 1]] + g.normal(0, 2, (n, 4))
    dspan = np.stack([np.arange(ann.images) * per, np.full(ann.images, per)], 1).astype(np.int32)
    r = torch.from_numpy(dense.reshape(-1, 5)).to(dev)
    s = torch.from_numpy(dspan).to(dev)
    ws = torch.empty(int(ops._lib.lib().icaf_kaist_mr_workspace_bytes(ann.images, int(ann.id.numel()), r.shape[0])) + 256,
                     dtype=torch.uint8, device=dev)
    out["dense_ms"] = event_ms(lambda: ops.kaist_mr(ann, r, s, per, workspace=ws))
    # test.test with and without the miss rate: 2,252 images in batches of 32
    B, R = 32, 1200
    z = np.zeros((B, R, 6), np.float32)
    z[..., 0] = g.uniform(20, 650, (B, R))
    z[..., 1] = g.uniform(20, 520, (B, R))
    z[..., 2] = g.uniform(10, 60, (B, R))
    z[..., 3] = z[..., 2] * 2.4
    z[..., 4] = g.uniform(0.01, 1, (B, R))
    z[..., 5] = 1.0
    stub = _Stub(torch.from_numpy(z).half().to(dev)).to(dev)
    img = torch.zeros(B, 6, 544, 672, dtype=torch.uint8).pin_memory()
    labels_list = [f"img_{i:05d}.txt" for i in range(ann.images)]
    shapes = [((512, 640), ((1.0, 1.0), (16.0, 16.0)))] * B
    loader = []
    for b0 in range(0, ann.images, B):
        n = min(B, ann.images - b0)
        loader.append((img[:n], torch.zeros(0, 6), [f"/d/img_{i:05d}.jpg" for i in range(b0, b0 + n)], shapes[:n]))
    times = {True: [], False: []}
    with tempfile.TemporaryDirectory() as tmp:
        for k in range(7):
            for mr in (False, True):
                t0 = time.perf_counter()
                _, _, res, _ = T.test({"nc": 1, "names": ["person"]}, model=stub, dataloader=loader, save_dir=tmp,
                                      labels_list=labels_list, mr_annotations=ann if mr else None)
                if k:                                    # the first round warms both paths up
                    times[mr].append(time.perf_counter() - t0)
    out["test_ms"] = float(np.median(times[False]) * 1e3)
    out["test_mr_ms"] = float(np.median(times[True]) * 1e3)
    out["test_added_ms"] = out["test_mr_ms"] - out["test_ms"]
    out["test_mr_result"] = [round(v, 6) for v in res]
    out["cpu_reference_s"] = {"MLPD": 4.2, "MBNet": 7.1, "MSDS-RCNN": 8.2, "ARCNN": 28.1, "ARCNN_conf0.001": 10.8}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
