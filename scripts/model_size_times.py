"""Forward step times of the five detector sizes, and the cross-attention launch time per DMFF head dim.

For yolov5{n,s,m,l,x}_Transfusion_FLIR at batch 1 and 16, 512 x 640 RGB+IR (seeded synthetic weights, BN folded, fp16), the way
bench.py builds its detector:
  - step: CUDA-graph replay of the forward (GraphedDetector), device-resident uint8 inputs, one CUDA event pair per step, the
    L2 flushed (256 MiB memset) between steps; the median and the spread over the timed steps are printed.
  - attention: eager forwards on one stream with a CUDA event after every library launch (ops.profile), each pass queued
    behind a spin kernel and after an L2 flush; every icaf_cross_attention launch keeps its fastest pass.  Head dims:
    n 8/16/32, s 16/32/64, m 24/48/96, l 32/64/128, x 40/80/160 (DMFF C / 8 heads at P3 / P4 / P5).
The card name, power limit and the SM clocks nvidia-smi reports during the timed steps are printed with the numbers.

    python scripts/model_size_times.py [--sizes n,s,m,l,x] [--batches 1,16] [--steps 50] [--warmup 10] [--passes 5]
"""
from __future__ import annotations

import argparse
import os
import statistics
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


def measure(size, B, steps, warmup, passes, dev, flush):
    import torch
    from bench import ClockSampler
    from icafusion_b200 import Model, ops, synth
    from icafusion_b200.engine import GraphedDetector
    from icafusion_b200.synth import load_synth

    H, W = 512, 640
    model = Model(f"yolov5{size}_Transfusion_FLIR").eval()
    load_synth(model, 0)
    model = model.fuse().half().to(dev)
    rgb, ir = [(t * 255).to(torch.uint8) for t in synth.synth_images(B, H, W, 0)]
    eng = GraphedDetector(model, B, H, W, in_dtype=torch.uint8, device=dev)
    eng.rgb.copy_(rgb)
    eng.ir.copy_(ir)
    for _ in range(warmup):
        eng.replay()
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    sampler.start()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for s, e in ev:
        flush.zero_()
        s.record()
        eng.replay()
        e.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = sorted(s.elapsed_time(e) for s, e in ev)
    del eng

    # attention launches, event-timed in eager forwards on one stream
    rgb_d, ir_d = rgb.to(dev), ir.to(dev)
    with torch.no_grad():
        for _ in range(2):
            model(rgb_d, ir_d)
        torch.cuda.synchronize()
        model.__dict__["_icaf_concurrent"] = False
        with ops.profile() as prof:
            for _ in range(passes):
                flush.zero_()
                torch.cuda._sleep(int(6e7))
                prof.mark()
                model(rgb_d, ir_d)
                torch.cuda.synchronize()
        model.__dict__["_icaf_concurrent"] = True
    recs = prof.records
    per = len(recs) // passes
    attn = []
    for i in range(per):
        name, work, _, _ = recs[i]
        if name != "icaf_cross_attention":
            continue
        us = 1e3 * min(recs[r * per + i][2].elapsed_time(recs[r * per + i][3]) for r in range(passes))
        attn.append((work["d"], work["N"], us))
    return dict(ms_median=statistics.median(ms), ms_min=ms[0], ms_max=ms[-1], clocks=clocks, attn=attn)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="n,s,m,l,x")
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--passes", type=int, default=5)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("model_size_times.py measures on the GPU: no CUDA device is available")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # > 50 MB L2

    print(f"card: {_card()}  (name, power limit, max SM clock)")
    print(f"512x640 RGB+IR, CUDA-graph forward, L2 flushed between steps, {args.steps} timed steps after {args.warmup} warm-up")
    print(f"{'model':<9} {'B':>3} {'ms/step':>8} {'min':>7} {'max':>7} {'SM MHz':>7} {'reasons':<24} attention launches (head dim d, tokens N: us)")
    for size in args.sizes.split(","):
        for B in (int(b) for b in args.batches.split(",")):
            r = measure(size, B, args.steps, args.warmup, args.passes, dev, flush)
            c = r["clocks"]
            attn = "  ".join(f"d{d} N{n}: {us:.1f}" for d, n, us in r["attn"])
            print(f"yolov5{size:<3} {B:>3} {r['ms_median']:>8.3f} {r['ms_min']:>7.3f} {r['ms_max']:>7.3f} {str(c['sm_mhz']):>7} "
                  f"{','.join(c['reasons']) or '-':<24} {attn}", flush=True)


if __name__ == "__main__":
    main()
