"""Device time of icaf_confluence (ops.confluence) per batch: batch 1 and 16, about 100, 1 000 and 5 000 candidates per
image, clustered (jittered copies around n/12 centres) and spread boxes, fp16 (B, 25200, 6) predictions.

    python scripts/confluence_times.py [--rounds 3] [--iters 5]

Configurations run alternately, round after round, so that drift in clocks or in other work on the card touches them
all alike; each figure is the range over rounds of the mean of `iters` launches timed by CUDA events.  Prints the card,
its power limit and its maximum SM clock first."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from icafusion_b200 import ops  # noqa: E402

R = 25200


def image(n, seed, spread):
    g = np.random.Generator(np.random.PCG64(seed))
    x = np.zeros((R, 6), np.float32)
    rows = np.sort(g.choice(R, n, replace=False))
    if spread:
        ctr, wh = g.uniform(0, 640, size=(n, 2)), g.uniform(4, 40, size=(n, 2))
    else:
        k = max(1, n // 12)
        c, s = g.uniform(0, 640, size=(k, 2)), g.uniform(8, 120, size=(k, 2))
        pick = g.integers(0, k, size=n)
        ctr, wh = c[pick] + g.normal(0, 2, size=(n, 2)), s[pick] * g.uniform(0.9, 1.1, size=(n, 2))
    x[rows, :2], x[rows, 2:4] = ctr, wh
    x[rows, 4] = g.uniform(0.2, 1.0, size=n)
    x[rows, 5] = g.uniform(0.6, 1.0, size=n)
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("confluence_times: needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(dev))
    cfgs = []
    for B in (1, 16):
        for n in (100, 1000, 5000):
            for spread in (False, True):
                z = torch.from_numpy(np.stack([image(n, 100 * b + n, spread) for b in range(B)])).half().to(dev)
                ws = torch.empty((ops.confluence_workspace_bytes(B, R, 6) + 15) // 16, 2, dtype=torch.int64, device=dev)
                det, count = ops.confluence(z, 0.1, 0.6, max_det=n, workspace=ws)
                cfgs.append(dict(B=B, n=n, kind="spread" if spread else "clustered", z=z, ws=ws, det=det, count=count, ms=[]))
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for c in cfgs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                ops.confluence(c["z"], 0.1, 0.6, det=c["det"], count=c["count"], workspace=c["ws"])
            e1.record()
            e1.synchronize()
            c["ms"].append(e0.elapsed_time(e1) / a.iters)
    for c in cfgs:
        kept = c["count"].float().mean().item()
        print(f"B={c['B']:2d} candidates={c['n']:5d} {c['kind']:9s} kept/image={kept:7.1f} "
              f"ms/batch={min(c['ms']):9.3f}-{max(c['ms']):9.3f}")


if __name__ == "__main__":
    main()
