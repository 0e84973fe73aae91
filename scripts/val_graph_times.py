"""Graphed against eager validation on the GPU (prints one JSON line):

* ``eager_img_s`` / ``graphed_img_s``: images/s of icafusion_b200.test.test without and with ``graphs=ValidationGraphs``,
  as train.py calls it per epoch: yolov5l FLIR with synthetic weights (not fused, like ``ema.ema``), 544 x 672, B = 1,
  ``compute_loss`` and ``save_txt=True``.  The two are alternated pass by pass in one run; each figure is the median of
  ``--passes`` passes, and ``*_spread`` is (max - min) / median over them.  The graphs are captured before the first
  timed pass, so a graphed pass is replays plus one in-place refresh;
* ``refresh_ms``: one ``engine.refresh_packed_(model)`` after every parameter and buffer of the model moved (median of 5);
* the card name, power limit and max SM clock, read in the same run.

    python scripts/val_graph_times.py [--images 128] [--passes 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from icafusion_b200 import Model  # noqa: E402
from icafusion_b200 import test as T  # noqa: E402
from icafusion_b200.engine import ValidationGraphs, refresh_packed_  # noqa: E402
from icafusion_b200.loss import ComputeLoss  # noqa: E402
from icafusion_b200.synth import load_synth  # noqa: E402

H, W = 544, 672
SHAPE = ((512, 640), ((1.0, 1.0), (16.0, 16.0)))
HYP = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def batches(n_images, seed=2):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in range(n_images):
        img = (torch.rand(1, 6, H, W, generator=g) * 255).to(torch.uint8).pin_memory()
        tg = torch.cat([torch.zeros(10, 1), torch.randint(0, 3, (10, 1), generator=g).float(),
                        torch.rand(10, 2, generator=g) * 0.8 + 0.1, torch.rand(10, 2, generator=g) * 0.2 + 0.02], 1)
        out.append((img, tg.pin_memory(), [f"/d/{k:05d}.jpg"], [SHAPE]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--passes", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    model = Model("yolov5l_Transfusion_FLIR").eval()
    load_synth(model, 3)
    model = model.to(dev)
    model.hyp, model.gr = dict(HYP), 1.0
    loader = batches(args.images)
    labels_list = sorted(os.path.basename(b[2][0])[:-4] + ".txt" for b in loader)
    data = {"nc": 3, "names": ["person", "car", "bicycle"]}
    res = {"card": card(), "model": "yolov5l_Transfusion_FLIR", "shape": [1, H, W], "images": len(loader)}
    graphs = ValidationGraphs(model)
    compute_loss = ComputeLoss(model)
    times = {"eager": [], "graphed": []}
    with tempfile.TemporaryDirectory() as tmp:
        def run(g):
            return T.test(data, model=model, dataloader=loader, save_dir=tmp, batch_size=1, imgsz=W, save_txt=True,
                          compute_loss=compute_loss, labels_list=labels_list, graphs=g)
        want = run(None)                                    # warm-up of both paths (packs, captures)
        got = run(graphs)
        res["graphed_equals_eager"] = bool(list(want[0]) == list(got[0]) and (want[1] == got[1]).all())
        for _ in range(args.passes):
            for name, g in (("eager", None), ("graphed", graphs)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(g)
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
    for name, ts in times.items():
        med = statistics.median(ts)
        res[f"{name}_img_s"] = round(len(loader) / med, 1)
        res[f"{name}_spread"] = round((max(ts) - min(ts)) / med, 3)
    res["speedup"] = round(res["graphed_img_s"] / res["eager_img_s"], 2)
    res["captures"] = graphs.captures

    refresh = []
    for _ in range(5):
        with torch.no_grad():
            for v in model.state_dict().values():
                if v.dtype.is_floating_point:
                    v.mul_(1.0)                             # moves every cache key, keeps the values
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = refresh_packed_(model)
        torch.cuda.synchronize()
        refresh.append(time.perf_counter() - t0)
    res["refresh_ms"] = round(statistics.median(refresh) * 1e3, 2)
    res["refreshed_caches"] = n
    print(json.dumps(res))


if __name__ == "__main__":
    main()
