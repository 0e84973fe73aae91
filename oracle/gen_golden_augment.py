"""Generate tests/golden/augment_cases.npz by running the REAL reference's training loader (build container only).

    python -m oracle.gen_golden_augment

A synthetic dataset tree (visible/, infrared/, labels/; lossless PNG frames of mixed sizes and random box labels) is loaded by
utils/datasets.py:LoadMultiModalImagesAndLabels(..., augment=True, hyp=hyp.scratch + overrides); under fixed seeds of
`random` and `np.random` each case takes dataset[i] for a list of indices and collates them (collate_fn).  Stored: the decoded
frames (what cv2.imread returned), the parsed labels, per case the seed, indices, image size, hyp, the (B, 6, s, s) images,
the (n, 6) targets and the next draw of `random` / `np.random` after the batch (the sampler must leave both in that state).
"""
from __future__ import annotations

import json
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "augment_cases.npz")
FRAME_HW = [(96, 128), (90, 120), (128, 80), (96, 128), (60, 80), (120, 120)]
HYP_SCRATCH = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0,
                   flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.0)
CASES = [  # name, img_size, seed, indices, hyp overrides
    ("mosaic_r1", 128, 11, [0, 3], {}),                                  # 96x128 frames at s = 128: r = 1 tiles
    ("mosaic_resize", 96, 12, [1, 4, 5], {}),                            # every tile resized (down and up)
    ("letterbox", 96, 13, [2, 4, 0], dict(mosaic=0.0)),                  # the non-mosaic branch
    ("degrees_shear", 64, 14, [5, 2], dict(degrees=10.0, shear=5.0)),
    ("flipud", 64, 15, [3, 1], dict(flipud=1.0, hsv_h=0.1)),
]


def synth_frames(seed=5):
    """Smooth colour / grey frames with mild noise (kept small so the golden stays well under 1 MB): BGR uint8 (h, w, 3) RGB-camera and IR-camera pairs."""
    g = np.random.Generator(np.random.PCG64(seed))
    out = []
    for h, w in FRAME_HW:
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        ph = g.uniform(0, 2 * np.pi, 6)
        rgb = np.stack([127 + 110 * np.sin(xx / (9 + 5 * c) + yy / (12 + 3 * c) + ph[c]) for c in range(3)], -1)
        rgb += g.normal(0, 1, rgb.shape)
        ir = 120 + 100 * np.cos(xx / 16 + ph[3]) * np.sin(yy / 10 + ph[4]) + g.normal(0, 1, (h, w))
        ir = np.repeat(ir[..., None], 3, -1)
        out.append((np.clip(rgb, 0, 255).astype(np.uint8), np.clip(ir, 0, 255).astype(np.uint8)))
    return out


def synth_labels(n, seed=6):
    g = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k in range(n):
        nb = int(g.integers(0, 7)) if k != 2 else 0                        # image 2 has no labels
        wh = g.uniform(0.03, 0.45, (nb, 2))
        xy = g.uniform(wh / 2, 1 - wh / 2)
        cls = g.integers(0, 3, (nb, 1)).astype(np.float64)
        out.append(np.concatenate([cls, xy, wh], 1))
    return out


def main():
    load_reference()
    import cv2
    from utils.datasets import LoadMultiModalImagesAndLabels
    frames = synth_frames()
    labels = synth_labels(len(frames))
    arrays, meta = {}, {"cases": [], "frames": len(frames)}
    with tempfile.TemporaryDirectory(prefix="augtree") as tmp:
        # img2label_paths maps .../visible/x.png and .../infrared/x.png to .../labels/x.txt: one labels/ per modality, so the
        # two label caches the loader writes do not collide
        vis, inf = os.path.join(tmp, "rgb", "visible"), os.path.join(tmp, "ir", "infrared")
        caches = [os.path.join(tmp, m, "labels.cache") for m in ("rgb", "ir")]
        for d in (vis, inf, os.path.join(tmp, "rgb", "labels"), os.path.join(tmp, "ir", "labels")):
            os.makedirs(d)
        for k, ((rgb, ir), lb) in enumerate(zip(frames, labels)):
            cv2.imwrite(os.path.join(vis, f"{k:03d}.png"), rgb)
            cv2.imwrite(os.path.join(inf, f"{k:03d}.png"), ir)
            for m in ("rgb", "ir"):
                with open(os.path.join(tmp, m, "labels", f"{k:03d}.txt"), "w") as f:
                    f.writelines(f"{int(r[0])} {r[1]:.6f} {r[2]:.6f} {r[3]:.6f} {r[4]:.6f}\n" for r in lb)
        for k in range(len(frames)):
            arrays[f"rgb{k}"] = cv2.imread(os.path.join(vis, f"{k:03d}.png"))
            arrays[f"ir{k}"] = cv2.imread(os.path.join(inf, f"{k:03d}.png"))
        for name, s, seed, indices, over in CASES:
            hyp = dict(HYP_SCRATCH, **over)
            for c in caches:               # rebuilt every time: torch >= 2.6 refuses to torch.load the numpy-holding cache
                if os.path.exists(c):
                    os.remove(c)
            ds = LoadMultiModalImagesAndLabels(vis, inf, img_size=s, batch_size=16, augment=True, hyp=hyp)
            if name == CASES[0][0]:
                for k in range(len(frames)):
                    arrays[f"labels{k}"] = np.asarray(ds.labels_rgb[k], dtype=np.float32)
            random.seed(seed)
            np.random.seed(seed)
            batch = [ds[i] for i in indices]
            img, targets, _, _ = LoadMultiModalImagesAndLabels.collate_fn(batch)
            arrays[f"{name}_img"] = img.numpy()
            arrays[f"{name}_targets"] = targets.numpy().astype(np.float32)
            arrays[f"{name}_next"] = np.array([random.random(), np.random.random()])
            meta["cases"].append(dict(name=name, img_size=s, seed=seed, indices=indices, hyp=hyp))
            print(name, img.shape, targets.shape)
    meta["reference"] = "utils/datasets.py:948-1031 LoadMultiModalImagesAndLabels(augment=True)[i] + collate_fn"
    meta["cv2"] = cv2.__version__
    np.savez_compressed(OUT, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
