"""Host seconds per validation batch: the reference's CPU staging against icafusion_b200.valdata.ValBatches.

Datasets: 64 synthetic decoded RGB/IR pairs of one size -- KAIST 512 x 640 (at img_size 640 load_image keeps the frame) and
LLVIP 1024 x 1280 (INTER_AREA 2x to 512 x 640); both letterbox to 544 x 672 batches -- at batch 1 and 32, rect=True,
pad=0.5.  Decoding is not part of either path: the frames sit decoded in host
memory, as cv2.imread leaves them.

  * cv2: what the reference's loader does per batch on the host thread after imread -- cv2.resize (INTER_AREA when r < 1),
    cv2.copyMakeBorder to the batch shape, BGR -> RGB, HWC -> CHW, the 6-channel concatenate, collate_fn's torch.stack, the
    pin and the upload test.test makes, ending in a device synchronise.  Labels are left out (both paths build the same rows).
  * ValBatches: a whole batch (labels, tables, the pinned upload of the frames, the icaf_val_stage launch), ending in a device
    synchronise; `host` is ValBatches.host_seconds, the part spent on the host thread.
  * kernel: CUDA events around re-launches of the last batch's icaf_val_stage.

The card name, power limit and max SM clock are printed with the numbers.

    python scripts/val_loader_times.py [--passes 3] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown (nvidia-smi printed nothing)"
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def _dataset(n, h, w, seed=3):
    import numpy as np
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    frames, labels = {}, []
    for k in range(n):
        base = (xx * (k + 3) // 7 + yy * (k + 5) // 9) % 256
        rgb = np.stack([(base + 60 * c + g.integers(0, 24, base.shape)) % 256 for c in range(3)], -1).astype(np.uint8)
        ir = np.repeat(((base // 2 + g.integers(0, 16, base.shape)) % 256)[..., None], 3, -1).astype(np.uint8)
        frames[k] = (rgb, ir)
        nb = int(g.integers(0, 9))
        wh = g.uniform(0.02, 0.4, (nb, 2))
        labels.append(np.concatenate([g.integers(0, 2, (nb, 1)), g.uniform(wh / 2, 1 - wh / 2), wh], 1).astype(np.float32))
    return frames, labels


def cv2_batch(vb, j, frames, dev):
    """Batch j of the reference's staging with cv2 (geometry from vb), uploaded as test.test uploads it."""
    import cv2
    import numpy as np
    import torch
    bs = vb.batch_size
    ks = range(j * bs, min((j + 1) * bs, len(vb.order)))
    H, W = (int(v) for v in vb.shape_of[ks[0]])
    imgs = []
    for k in ks:
        h, w, _, _, top, left = vb.geometry[k]
        pair = []
        for f in frames[int(vb.order[k])]:
            if f.shape[:2] != (h, w):
                f = cv2.resize(f, (w, h), interpolation=cv2.INTER_AREA if h < f.shape[0] else cv2.INTER_LINEAR)
            f = cv2.copyMakeBorder(f, top, H - h - top, left, W - w - left, cv2.BORDER_CONSTANT, value=(114, 114, 114))
            pair.append(np.ascontiguousarray(f[:, :, ::-1].transpose(2, 0, 1)))
        imgs.append(torch.from_numpy(np.concatenate(pair, 0)))
    return torch.stack(imgs, 0).pin_memory().to(dev, non_blocking=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=3, help="timed passes over the 64 pairs")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("val_loader_times.py measures the device path: no CUDA device")
    import cv2
    from icafusion_b200 import _lib, ops
    from icafusion_b200.valdata import ValBatches
    dev = torch.device("cuda:0")
    res = {"card": _card(), "cv2_threads": cv2.getNumThreads(), "pairs": 64, "passes": a.passes, "runs": []}
    for name, (h0, w0) in (("KAIST 512x640", (512, 640)), ("LLVIP 1024x1280", (1024, 1280))):
        frames, labels = _dataset(64, h0, w0)
        for B in (1, 32):
            vb = ValBatches(labels, frames.__getitem__, [(h0, w0)] * 64, 640, batch_size=B, device=dev)
            nb = len(vb)
            for j in range(min(nb, 2)):                                     # warm-up (pinned blocks, module load)
                cv2_batch(vb, j, frames, dev)
                vb.batch(j)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.passes):
                for j in range(nb):
                    cv2_batch(vb, j, frames, dev)
            torch.cuda.synchronize()
            t_cv2 = (time.perf_counter() - t0) / (a.passes * nb)
            vb.host_seconds = 0.0
            t0 = time.perf_counter()
            for _ in range(a.passes):
                for j in range(nb):
                    img = vb.batch(j)[0]
            torch.cuda.synchronize()
            t_dev = (time.perf_counter() - t0) / (a.passes * nb)
            host = vb.host_seconds / (a.passes * nb)
            want = cv2_batch(vb, nb - 1, frames, dev)
            same = bool(torch.equal(img, want))
            # kernel alone: re-launch the last batch's icaf_val_stage
            L, params = _lib.lib(), vb.params
            Bl, _, H, W = img.shape
            n_words = (params.numel() - int(L.icaf_val_stage_params_bytes(Bl, 0))) // 4
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 50
            e0.record()
            for _ in range(reps):
                _lib.check(L.icaf_val_stage(params.data_ptr(), params.numel(), Bl, H, W, n_words, img.data_ptr(),
                                            ops._stream()), "icaf_val_stage")
            e1.record()
            torch.cuda.synchronize()
            r = {"frames": name, "batch": B, "batch_shape": [int(H), int(W)], "cv2_ms_per_batch": 1e3 * t_cv2,
                 "valbatches_ms_per_batch": 1e3 * t_dev, "valbatches_host_ms_per_batch": 1e3 * host,
                 "kernel_us": 1e3 * e0.elapsed_time(e1) / reps, "equal_to_cv2": same}
            print(json.dumps(r))
            res["runs"].append(r)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
