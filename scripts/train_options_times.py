"""Cost of gradient accumulation and focal loss in the training step (prints one JSON line):

  * a GraphedTrainStep of yolov5l at batch 16 and 640 x 512: CUDA events time one replay of the fresh graph (writes .grad)
    and one replay of the accumulating graph (adds into .grad), alternated, each after an L2 flush;
  * ComputeLoss forward + backward on yolov5l's three Detect maps at the same size (fp16, 40 labels): fl_gamma 0 (plain BCE)
    against 1.5 (focal), alternated, each after an L2 flush.

The card name and power limit are read in the same run.

    python scripts/train_options_times.py [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from icafusion_b200 import Model  # noqa: E402
from icafusion_b200.loss import ComputeLoss  # noqa: E402
from icafusion_b200.synth import load_synth  # noqa: E402
from icafusion_b200.trainer import GraphedTrainStep, TrainStep  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def alternated(fns, reps, flush):
    """Median us per call of each fn, calls alternated, an L2 flush before each."""
    times = [[] for _ in fns]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(reps):
        for i, fn in enumerate(fns):
            flush.zero_()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[i].append(e0.elapsed_time(e1) * 1e3)
    return [sorted(t)[len(t) // 2] for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)          # > the H100's 50 MB L2
    B, H, W = 16, 512, 640
    g = torch.Generator().manual_seed(0)
    rgb = torch.randint(0, 256, (B, 3, H, W), generator=g).to(torch.uint8).to(dev)
    ir = torch.randint(0, 256, (B, 3, H, W), generator=g).to(torch.uint8).to(dev)
    t = torch.rand(40, 6, generator=g) * 0.5 + 0.25
    t[:, 0] = torch.arange(40) % B
    t[:, 1] = 0
    t = t.to(dev)

    model = Model("yolov5l_Transfusion_kaist")
    load_synth(model, 5)
    model = model.to(dev).train()
    ts = TrainStep(model, None, total_batch_size=B, imgsz=W)
    step = GraphedTrainStep(ts, B, H, W, 64, dev)
    step(rgb, ir, t, optimizer_step=False)                                  # fresh graph
    step(rgb, ir, t, optimizer_step=False)                                  # captures the accumulating graph
    torch.cuda.synchronize()
    fresh, acc = alternated([step.graph.replay, step.acc_graph.replay], args.reps, flush)
    step.close()

    ny = [H // s for s in (8, 16, 32)]
    nx = [W // s for s in (8, 16, 32)]
    p = [(torch.randn(B, 3, y, x, 6, generator=g) * 1.5).half().to(dev).requires_grad_(True) for y, x in zip(ny, nx)]
    losses = {}
    for gamma in (0.0, 1.5):
        m = Model("yolov5l_Transfusion_kaist")
        m.hyp = dict(ts.hyp, fl_gamma=gamma)
        m.model[-1].anchors = m.model[-1].anchors.to(dev)
        losses[gamma] = ComputeLoss(m)

    def loss_step(fn):
        def run():
            loss, _ = fn(p, t)
            loss.backward()
        return run
    plain, focal = alternated([loss_step(losses[0.0]), loss_step(losses[1.5])], args.reps * 5, flush)
    print(json.dumps({
        "card": card(), "model": "yolov5l", "batch": B, "image": f"{W}x{H}", "reps": args.reps,
        "graph_replay_us": {"fresh": round(fresh, 1), "accumulating": round(acc, 1)},
        "loss_fwd_bwd_us": {"fl_gamma_0": round(plain, 1), "fl_gamma_1.5": round(focal, 1)},
    }))


if __name__ == "__main__":
    main()
