"""Cost of fp32 DMFF token streams in the training step (TrainStep(dmff_fp32=True)); prints one JSON line:

  * a GraphedTrainStep of yolov5l at batch 16 and 640 x 512, built twice -- fp16 streams (the default) and fp32 streams --
    CUDA events time one replay of each step graph, alternated, each after an L2 flush;
  * the forward + backward of each of yolov5l's three TransformerFusionBlocks at the shapes that step gives them (P3 / P4 /
    P5 maps of batch 16), captured alone as a CUDA graph per precision and timed the same way (5 x reps replays).  Their sum
    over the step time is printed as dmff_isolated_sum_pct: in the step the blocks overlap the backbone and each other on
    side streams, so it is an upper bound on their share, not the share.

The card name, power limit and SM clock are read in the same run.

    python scripts/dmff_fp32_times.py [--reps 20]
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

from icafusion_b200 import Model, TransformerFusionBlock  # noqa: E402
from icafusion_b200 import autograd as A  # noqa: E402
from icafusion_b200.synth import load_synth  # noqa: E402
from icafusion_b200.trainer import GraphedTrainStep, TrainStep, set_dmff_stream_dtype  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
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


def block_graph(blk, rgb, ir, dy):
    """One CUDA graph of the block's training forward + backward on static NHWC inputs."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            A.fusion_block(blk, rgb, ir).backward(dy)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        A.fusion_block(blk, rgb, ir).backward(dy)
    return g


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

    steps = {}
    for fp32 in (False, True):
        model = Model("yolov5l_Transfusion_kaist")
        load_synth(model, 5)
        model = model.to(dev).train()
        ts = TrainStep(model, None, total_batch_size=B, imgsz=W, dmff_fp32=fp32)
        steps[fp32] = GraphedTrainStep(ts, B, H, W, 64, dev)
        steps[fp32](rgb, ir, t, optimizer_step=False)
    torch.cuda.synchronize()
    off, on = alternated([steps[False].graph.replay, steps[True].graph.replay], args.reps, flush)
    for s in steps.values():
        s.close()
    del steps
    torch.cuda.empty_cache()

    # the three DMFF blocks at the maps the step gives them (P3 / P4 / P5 of a 640 x 512 batch)
    model = Model("yolov5l_Transfusion_kaist")
    load_synth(model, 5)
    blocks = [m for m in model.model if isinstance(m, TransformerFusionBlock)]
    blk_us = {}
    for blk, s in zip(blocks, (8, 16, 32)):
        blk = blk.to(dev).train()
        C = blk.n_embd
        x = [(torch.randn(B, H // s, W // s, C, generator=g) * 0.5).half().to(dev).requires_grad_(True) for _ in range(2)]
        dy = (torch.randn(B, H // s, W // s, C, generator=g) * 0.01).half().to(dev)
        graphs = {}
        for fp32 in (False, True):
            set_dmff_stream_dtype(blk, fp32)
            graphs[fp32] = block_graph(blk, x[0], x[1], dy)
        b_off, b_on = alternated([graphs[False].replay, graphs[True].replay], args.reps * 5, flush)
        blk_us[f"P{s.bit_length() - 1}"] = {"fp16": round(b_off, 1), "fp32": round(b_on, 1)}
        del graphs
    print(json.dumps({
        "card": card(), "model": "yolov5l", "batch": B, "image": f"{W}x{H}", "reps": args.reps,
        "step_replay_us": {"fp16_streams": round(off, 1), "fp32_streams": round(on, 1), "cost_pct": round(100 * (on - off) / off, 2)},
        "dmff_block_fwd_bwd_us": blk_us,
        "dmff_isolated_sum_pct": {k: round(100 * sum(v[k] for v in blk_us.values()) / (off if k == "fp16" else on), 2) for k in ("fp16", "fp32")},
    }))


if __name__ == "__main__":
    main()
