"""Generate tests/golden/val_loader_cases.npz by running the REAL reference's validation loader (build container only).

    python -m oracle.gen_golden_val_loader

A synthetic dataset tree (visible/, infrared/, labels/; seeded JPEG pairs of mixed sizes and random box labels) is loaded the
way train.py:211-214 builds its testloader: utils/datasets.py:create_dataloader_rgb_ir(..., img_size 320, stride 32,
rect=True, pad=0.5, workers=0), i.e. LoadMultiModalImagesAndLabels(augment=False) + collate_fn.  At img_size 320 the
frames take every staging path: r = 1 (a copy), r = 0.5 (INTER_AREA's integer fast path), fractional INTER_AREA with equal
and with unequal x / y scales, and r > 1 (INTER_LINEAR); their aspect ratios span both sides of 1, so the rect sort and
several batch shapes matter.  Cases: batch 1, batch 4, batch 4 with single_cls.

Stored: the decoded frames (what cv2.imread returned), the parsed labels (file order), and per case every batch the loader
yielded -- the SHA-256 and shape of the (B, 6, H, W) uint8 images (the images themselves would be most of the file), the
(n, 6) targets, the paths relative to the dataset root and the shapes tuples.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "val_loader_cases.npz")
IMG_SIZE = 320
# (h0, w0) at img_size 320: r = 1 | 2x area | area 1.5625 | linear 1.25 | area 1.5 (tall) | area x 1.03125, y 1.0345 |
# linear, tall | area 1.03125 / 1.0345, tall
FRAME_HW = [(240, 320), (512, 640), (400, 500), (200, 256), (480, 360), (300, 330), (257, 250), (330, 300)]
CASES = [("b1", 1, False), ("b4", 4, False), ("b4_single_cls", 4, True)]   # name, batch size, single_cls


def synth_frames(seed=7):
    """BGR uint8 (h, w, 3) RGB-camera / IR-camera pairs: colour waves along x, steps along y and flat boxes with sharp edges,
    so both the averaging and the edges of a resize are exercised.  The waves repeat every 32 columns and the steps every 16
    rows (whole JPEG blocks), so the decoded rows repeat too and the golden stays small."""
    g = np.random.Generator(np.random.PCG64(seed))
    out = []
    for h, w in FRAME_HW:
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        ph = g.uniform(0, 2 * np.pi, 4)
        rgb = np.stack([127 + 100 * np.sin(xx * (np.pi / 16) + ph[c]) + 20 * (yy // 16 % 3) for c in range(3)], -1)
        ir = np.full((h, w), 60.0) + 50 * np.cos(yy / 40 + ph[3])
        for _ in range(5):
            bh, bw = int(g.integers(8, h // 3)), int(g.integers(8, w // 3))
            y0, x0 = int(g.integers(0, h - bh)), int(g.integers(0, w - bw))
            rgb[y0:y0 + bh, x0:x0 + bw] = g.integers(0, 256, 3)
            ir[y0:y0 + bh, x0:x0 + bw] = g.integers(120, 256)
        ir = np.repeat(ir[..., None], 3, -1)
        out.append((np.clip(rgb, 0, 255).astype(np.uint8), np.clip(ir, 0, 255).astype(np.uint8)))
    return out


def synth_labels(n, seed=8):
    g = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k in range(n):
        nb = int(g.integers(1, 6)) if k != 3 else 0                         # image 3 has no labels
        wh = g.uniform(0.03, 0.45, (nb, 2))
        xy = g.uniform(wh / 2, 1 - wh / 2)
        cls = g.integers(0, 3, (nb, 1)).astype(np.float64)
        out.append(np.concatenate([cls, xy, wh], 1))
    return out


def main():
    load_reference()
    import cv2
    from utils.datasets import LoadMultiModalImagesAndLabels, create_dataloader_rgb_ir
    frames = synth_frames()
    labels = synth_labels(len(frames))
    arrays, meta = {}, {"cases": [], "frames": len(frames), "img_size": IMG_SIZE, "stride": 32, "pad": 0.5}
    with tempfile.TemporaryDirectory(prefix="valtree") as tmp:
        vis, inf = os.path.join(tmp, "rgb", "visible"), os.path.join(tmp, "ir", "infrared")
        caches = [os.path.join(tmp, m, "labels.cache") for m in ("rgb", "ir")]
        for d in (vis, inf, os.path.join(tmp, "rgb", "labels"), os.path.join(tmp, "ir", "labels")):
            os.makedirs(d)
        for k, ((rgb, ir), lb) in enumerate(zip(frames, labels)):
            cv2.imwrite(os.path.join(vis, f"{k:03d}.jpg"), rgb, [cv2.IMWRITE_JPEG_QUALITY, 90])
            cv2.imwrite(os.path.join(inf, f"{k:03d}.jpg"), ir, [cv2.IMWRITE_JPEG_QUALITY, 90])
            for m in ("rgb", "ir"):
                with open(os.path.join(tmp, m, "labels", f"{k:03d}.txt"), "w") as f:
                    f.writelines(f"{int(r[0])} {r[1]:.6f} {r[2]:.6f} {r[3]:.6f} {r[4]:.6f}\n" for r in lb)
        for k in range(len(frames)):
            arrays[f"rgb{k}"] = cv2.imread(os.path.join(vis, f"{k:03d}.jpg"))
            arrays[f"ir{k}"] = cv2.imread(os.path.join(inf, f"{k:03d}.jpg"))

        def fresh():
            for c in caches:               # rebuilt every time: torch >= 2.6 refuses to torch.load the numpy-holding cache
                if os.path.exists(c):
                    os.remove(c)

        fresh()
        ds = LoadMultiModalImagesAndLabels(vis, inf, img_size=IMG_SIZE, batch_size=1)      # file order, for the labels
        for k in range(len(frames)):
            arrays[f"labels{k}"] = np.asarray(ds.labels_rgb[k], dtype=np.float32)
        meta["paths"] = [os.path.relpath(p, tmp) for p in ds.img_files_rgb]
        for name, bs, single_cls in CASES:
            fresh()
            opt = types.SimpleNamespace(single_cls=single_cls)
            loader, _ = create_dataloader_rgb_ir(vis, inf, IMG_SIZE, bs, 32, opt, hyp=None, rect=True, pad=0.5, workers=0)
            case = dict(name=name, batch_size=bs, single_cls=single_cls, batches=[])
            for i, (img, targets, paths, shapes) in enumerate(loader):
                arrays[f"{name}_targets{i}"] = targets.numpy().astype(np.float32)
                case["batches"].append(dict(
                    img_shape=list(img.shape), img_sha256=hashlib.sha256(img.numpy().tobytes()).hexdigest(),
                    paths=[os.path.relpath(p, tmp) for p in paths],
                    shapes=[[[int(h0), int(w0)], [[float(a), float(b)], [float(c), float(d)]]]
                            for (h0, w0), ((a, b), (c, d)) in shapes]))
                print(name, i, tuple(img.shape), tuple(targets.shape))
            meta["cases"].append(case)
    meta["reference"] = ("utils/datasets.py:create_dataloader_rgb_ir(rect=True, pad=0.5, workers=0): "
                         "LoadMultiModalImagesAndLabels(augment=False) + collate_fn")
    meta["cv2"] = cv2.__version__
    np.savez_compressed(OUT, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
