"""Train.py iterations with the optimiser step on the device against the eager torch step (prints one JSON line).

The loop is train.py-shaped: yolov5l, batch 16 of 640 x 512 pairs (uint8, on the device), accumulate 4 (nominal batch 64),
EMA on, GraphedTrainStep, and every call writes the warm-up interpolation of each group's lr and momentum first
(train.py:314-326).  Two per-call sequences run on the same GraphedTrainStep, alternated block by block:

* ``device``: ``GraphedTrainStep.__call__`` -- graph replay, then on a stepping call the step graph (unscale, SGD gated on
  the device flag, scale update, EMA); no read-back;
* ``eager``: the parent commit's call -- the same graph replay, then on a stepping call ``scaler.step(optimizer)``,
  ``scaler.update()`` and ``ema.update(model)`` through torch, which reads GradScaler's inf flag on the host.

Reported, median over ``--blocks`` blocks of ``--iters`` iterations per sequence (at least 40, after 8 warm-up iterations):

* ``*_ms_per_iter``: host clock over a block that starts and ends with a device synchronise; the script reads nothing back
  inside it (the eager sequence's own read of the inf flag is part of what it measures);
* ``*_step_gpu_ms``: CUDA events around the optimiser step alone (step graph replay against torch's sequence), each behind
  a fresh backward replay, median of ``--steps`` alternated steps per sequence;
* the card name, power limit and max SM clock, read in the same run.

    python scripts/train_iteration_times.py [--iters 48] [--blocks 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from icafusion_b200 import Model, synth  # noqa: E402
from icafusion_b200.synth import load_synth  # noqa: E402
from icafusion_b200.trainer import GraphedTrainStep, TrainStep  # noqa: E402

B, H, W = 16, 512, 640
NW = 1000                                 # warm-up batches: every timed call writes lr / momentum


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=48)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20, help="optimiser steps timed alone per sequence")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_iteration_times: needs a CUDA device")
    if args.iters < 40:
        raise SystemExit("train_iteration_times: --iters must be at least 40")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = Model("yolov5l_Transfusion_kaist")
    load_synth(model, 0)
    model = model.to(dev).train()
    ts = TrainStep(model, None, total_batch_size=B, imgsz=max(H, W), ema=True)
    assert ts.accumulate == 4
    lf = lambda x: (1 - x / 300) * (1.0 - 0.2) + 0.2      # noqa: E731 (train.py:148)
    torch.optim.lr_scheduler.LambdaLR(ts.optimizer, lr_lambda=lf)
    rgb, ir = [(t * 255).to(torch.uint8).to(dev) for t in synth.synth_images(B, H, W, 0)]
    g = torch.Generator().manual_seed(0)
    tg = torch.zeros(4 * B, 6)
    tg[:, 0] = torch.arange(4 * B) % B
    tg[:, 2:4] = 0.1 + 0.8 * torch.rand(4 * B, 2, generator=g)
    tg[:, 4:6] = 0.03 + 0.2 * torch.rand(4 * B, 2, generator=g)
    tg = tg.to(dev)
    step = GraphedTrainStep(ts, B, H, W, 4 * B, dev)

    def eager_call(optimizer_step):              # the parent commit's GraphedTrainStep.__call__
        step.rgb.copy_(rgb, non_blocking=True)
        step.ir.copy_(ir, non_blocking=True)
        step.tg.copy_(tg, non_blocking=True)
        (step.graph if step.fresh else step.acc_graph).replay()
        step.fresh = optimizer_step
        if optimizer_step:
            ts.scaler.step(ts.optimizer)
            ts.scaler.update()
            ts.ema.update(ts.raw_model)

    ni = [0]

    def one(mode):
        k = ni[0]
        ni[0] += 1
        for j, x in enumerate(ts.optimizer.param_groups):                # train.py:322-326
            x["lr"] = np.interp(k, [0, NW], [0.1 if j == 2 else 0.0, x["initial_lr"] * lf(0)])
            x["momentum"] = np.interp(k, [0, NW], [0.8, 0.937])
        flag = k % ts.accumulate == 0
        if mode == "eager":
            eager_call(flag)
        else:
            step(rgb, ir, tg, optimizer_step=flag)

    for _ in range(8):
        one("device")
        one("eager")
    torch.cuda.synchronize()
    per_iter = {"device": [], "eager": []}
    for b in range(args.blocks):
        for mode in (("device", "eager") if b % 2 == 0 else ("eager", "device")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                one(mode)
            torch.cuda.synchronize()
            per_iter[mode].append((time.perf_counter() - t0) * 1e3 / args.iters)
    # the optimiser step alone, behind a fresh backward each time, alternated
    step_ms = {"device": [], "eager": []}
    for r in range(2 * args.steps):
        mode = ("device", "eager")[r % 2]
        step.graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if mode == "device":
            step.opt.stage()
            step.step_graph.replay()
        else:
            ts.scaler.step(ts.optimizer)
            ts.scaler.update()
            ts.ema.update(ts.raw_model)
        e1.record()
        torch.cuda.synchronize()
        step_ms[mode].append(e0.elapsed_time(e1))
    step.close()
    out = {"workload": f"yolov5l train.py loop, {B} x {W}x{H} uint8 pairs, accumulate {ts.accumulate}, EMA, warm-up lr every call",
           "iters_per_block": args.iters, "blocks": args.blocks}
    for mode in ("device", "eager"):
        out[f"{mode}_ms_per_iter"] = round(statistics.median(per_iter[mode]), 3)
        out[f"{mode}_ms_per_iter_all"] = [round(x, 3) for x in per_iter[mode]]
        out[f"{mode}_step_gpu_ms"] = round(statistics.median(step_ms[mode]), 3)
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
