"""Per-launch times of the conv GEMMs of one yolov5l batch-16 forward (512 x 640 RGB+IR), against the roofline.

Builds the detector the way bench.py does (seeded synthetic weights, BN folded, fp16), warms it up and runs eager forwards
on one stream with a CUDA event after every library launch (ops.profile).  Each pass is queued behind a spin kernel so the
launches execute back to back; the L2 is flushed before each pass and every launch keeps its fastest of the passes.

For every icaf_conv2d_fwd launch (and every fused Bottleneck launch, icaf_bottleneck_fwd) it prints the kernel the dispatcher picks (persist / one-tile), K, the tile count, the
time, the achieved TFLOP/s and GB/s (algorithmic bytes: input + output + filter, + residual) and the roofline fraction:
max(FLOPs / tensor peak, bytes / HBM peak) / time.  The launches are then summed per K class.  The peaks are the H100 SXM
data-sheet figures (989 TFLOP/s dense FP16, 3.35 TB/s), which hold at 700 W; the card name and power limit are printed
with the table.

    python scripts/conv_launch_times.py [--batch 16] [--passes 3] [--csv out.csv] [--unfused]
"""
from __future__ import annotations

import argparse
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0     # H100 SXM, dense FP16, 700 W
PEAK_GBS = 3350.0       # H100 SXM HBM3


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown (nvidia-smi printed nothing)"
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def _k_class(persistent: bool, K: int) -> str:
    if not persistent:
        return "one-tile kernel"
    if K <= 256:
        return "persist K <= 256"
    if K <= 1152:
        return "persist K 257-1152"
    return "persist K >= 2048" if K >= 2048 else "persist K 1153-2047"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--size", default="l", choices=["s", "l"])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--csv", default=None, help="also write the per-launch table to this CSV file")
    ap.add_argument("--unfused", action="store_true", help="run the 64-channel Bottlenecks as two conv launches each instead "
                    "of the fused launch (icaf_bottleneck_fwd), to compare the two")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("conv_launch_times.py measures kernels on the GPU: no CUDA device is available")
    from icafusion_b200 import Model, _lib, ops, synth
    from icafusion_b200.synth import load_synth

    if args.unfused:
        from icafusion_b200 import common
        common.Bottleneck.fusable = staticmethod(lambda mods, xs, outs=None: False)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    B, H, W = args.batch, 512, 640
    model = Model(f"yolov5{args.size}_Transfusion_kaist").eval()
    load_synth(model, 0)
    model = model.fuse().half().to(dev)
    rgb, ir = [(t * 255).to(torch.uint8).to(dev) for t in synth.synth_images(B, H, W, 0)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # > 50 MB L2
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    L = _lib.lib()

    with torch.no_grad():
        for _ in range(3):
            model(rgb, ir)
        torch.cuda.synchronize()
        model.__dict__["_icaf_concurrent"] = False        # one stream: every launch is timed against its predecessor
        with ops.profile() as prof:
            for _ in range(args.passes):
                flush.zero_()
                torch.cuda._sleep(int(6e7))
                prof.mark()
                model(rgb, ir)
                torch.cuda.synchronize()
        model.__dict__["_icaf_concurrent"] = True
    recs = prof.records
    per = len(recs) // args.passes
    rows = []
    for i in range(per):
        name, work, _, _ = recs[i]
        if name not in ("icaf_conv2d_fwd", "icaf_bottleneck_fwd"):
            continue
        ms = min(recs[r * per + i][2].elapsed_time(recs[r * per + i][3]) for r in range(args.passes))
        fl, by = work["flops"], work["bytes"]
        us = ms * 1e3
        flop_us, hbm_us = fl / (PEAK_TFLOPS * 1e6), by / (PEAK_GBS * 1e3)
        if name == "icaf_bottleneck_fwd":           # 1x1 (on the patch halo) + 3x3 + residual, 4 x 32-pixel patches
            rows.append(dict(tag=work["tag"], kernel="fused", K=64 + 576, tiles=0, us=us, tflops=fl / (us * 1e-6) / 1e12,
                             gbs=by / (us * 1e-6) / 1e9, frac=max(flop_us, hbm_us) / us, bound="flop" if flop_us >= hbm_us else "hbm",
                             cls="fused bottleneck", flops=fl, bytes=by, bound_us=max(flop_us, hbm_us)))
            continue
        pl = _lib.ConvPlan()
        if L.icaf_conv2d_plan(ctypes.byref(work["geom"]), work["n_io"], sms, 0, ctypes.byref(pl)) != 0:
            raise RuntimeError(L.icaf_last_error().decode())
        g = work["geom"]
        K = g.kh * g.kw * g.Cin
        persistent = pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z
        bound_us = max(flop_us, hbm_us)
        rows.append(dict(tag=work["tag"], kernel="persist" if persistent else "one-tile", K=K, tiles=pl.work_items, us=us,
                         tflops=fl / (us * 1e-6) / 1e12, gbs=by / (us * 1e-6) / 1e9, frac=bound_us / us,
                         bound="flop" if flop_us >= hbm_us else "hbm", cls=_k_class(persistent, K),
                         flops=fl, bytes=by, bound_us=bound_us))

    print(f"card: {_card()}  (name, power limit, max SM clock)")
    print(f"yolov5{args.size} batch {B} {H}x{W}: {len(rows)} conv launches, fastest of {args.passes} event-timed eager passes, "
          f"peaks {PEAK_TFLOPS:.0f} TFLOP/s / {PEAK_GBS / 1e3:.2f} TB/s")
    hdr = f"{'#':>3} {'tag':<36} {'kernel':<8} {'K':>5} {'tiles':>5} {'us':>8} {'TFLOP/s':>8} {'GB/s':>7} {'bound':>5} {'frac':>5}"
    print(hdr)
    for i, r in enumerate(rows):
        print(f"{i:>3} {r['tag']:<36} {r['kernel']:<8} {r['K']:>5} {r['tiles']:>5} {r['us']:>8.1f} {r['tflops']:>8.1f} "
              f"{r['gbs']:>7.0f} {r['bound']:>5} {r['frac']:>5.2f}")
    print()
    print(f"{'class':<20} {'launches':>8} {'GFLOP':>7} {'GB':>6} {'us':>8} {'bound us':>9} {'TFLOP/s':>8} {'GB/s':>6} {'frac':>5}")
    classes = ["persist K <= 256", "persist K 257-1152", "persist K 1153-2047", "persist K >= 2048", "one-tile kernel",
               "fused bottleneck", "all"]
    for c in classes:
        sel = [r for r in rows if c == "all" or r["cls"] == c]
        if not sel:
            continue
        us = sum(r["us"] for r in sel)
        fl, by, bu = sum(r["flops"] for r in sel), sum(r["bytes"] for r in sel), sum(r["bound_us"] for r in sel)
        print(f"{c:<20} {len(sel):>8} {fl / 1e9:>7.0f} {by / 1e9:>6.2f} {us:>8.0f} {bu:>9.0f} {fl / (us * 1e-6) / 1e12:>8.1f} "
              f"{by / (us * 1e-6) / 1e9:>6.0f} {bu / us:>5.2f}")
    if args.csv:
        with open(args.csv, "w") as f:
            f.write("tag,kernel,K,tiles,us,tflops,gbs,bound,frac\n")
            for r in rows:
                f.write(f"{r['tag']},{r['kernel']},{r['K']},{r['tiles']},{r['us']:.2f},{r['tflops']:.2f},{r['gbs']:.1f},{r['bound']},"
                        f"{r['frac']:.3f}\n")


if __name__ == "__main__":
    main()
