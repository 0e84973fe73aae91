"""Cost of the two-phase (synchronised) BatchNorm on one GPU, with no exchange (prints one JSON line):

for every BatchNorm layer of a yolov5l training step at batch 16 and 640 x 512 (its shapes taken from a dry-run walk of the
train-mode forward), CUDA events time the one-call icaf_bn_act_fwd / icaf_bn_act_bwd against the two-phase
icaf_bn_act_fwd_stats + icaf_bn_act_fwd_apply / icaf_bn_act_bwd_sums + icaf_bn_act_bwd_apply, back to back on one stream.
The sums over the step's layers give the cost of the split per training step.  The exchange itself (one all-reduce per
layer and direction) needs several GPUs and is not part of this number.  The calls are eager: where the host issues them
slower than the GPU runs them, the events measure the host's issue time.  The card name and power limit are read in the
same run.

    python scripts/sync_bn_times.py [--reps 50]
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

from icafusion_b200 import Model, ops  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def layers(B=16, H=512, W=640):
    """(rows, C, act) of every BatchNorm layer of one yolov5l training forward, in walk order."""
    m = Model("yolov5l_Transfusion_kaist").to("meta").train()
    rgb = torch.empty(B, 3, H, W, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        m(rgb, rgb)
    return [(int(a[8]), int(a[9]), int(a[12])) for n, a, _ in dr.records if n == "icaf_bn_act_fwd"]


def timed(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3            # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    shapes = layers()
    per = {}
    for rows, C, act in sorted(set(shapes)):
        g = torch.Generator().manual_seed(rows + C)
        x = torch.randn(rows, C, generator=g).half().to(dev)
        dy = (0.1 * torch.randn(rows, C, generator=g)).half().to(dev)
        gam, bet = torch.ones(C, device=dev), torch.zeros(C, device=dev)
        rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
        dg, db = torch.empty(C, device=dev), torch.empty(C, device=dev)
        _, sm, si = ops.bn_act_fwd(x, gam, bet, rm, rv, 1e-3, 0.03, act)
        stats = ops.bn_act_fwd_stats(x)

        def fwd2():
            ops.bn_act_fwd_apply(x, gam, bet, rm, rv, ops.bn_act_fwd_stats(x), 1e-3, 0.03, act)

        def bwd2():
            s = ops.bn_act_bwd_sums(x, dy, gam, bet, sm, si, act, dg, db)
            ops.bn_act_bwd_apply(x, dy, gam, bet, sm, si, s, stats[-1:], act)

        per[(rows, C, act)] = dict(fwd1=timed(lambda: ops.bn_act_fwd(x, gam, bet, rm, rv, 1e-3, 0.03, act), args.reps), fwd2=timed(fwd2, args.reps),
                                   bwd1=timed(lambda: ops.bn_act_bwd(x, dy, gam, bet, sm, si, act, dg, db), args.reps), bwd2=timed(bwd2, args.reps))
    tot = {k: sum(per[s][k] for s in shapes) for k in ("fwd1", "fwd2", "bwd1", "bwd2")}
    worst = max(shapes, key=lambda s: (per[s]["fwd2"] + per[s]["bwd2"]) - (per[s]["fwd1"] + per[s]["bwd1"]))
    print(json.dumps({
        "card": card(), "model": "yolov5l", "batch": 16, "image": "640x512", "bn_layers": len(shapes), "reps": args.reps,
        "step_us": {k: round(v, 1) for k, v in tot.items()},
        "split_cost_us_per_step": round(tot["fwd2"] + tot["bwd2"] - tot["fwd1"] - tot["bwd1"], 1),
        "worst_layer": {"rows": worst[0], "C": worst[1], **{k: round(v, 2) for k, v in per[worst].items()}},
    }))


if __name__ == "__main__":
    main()
