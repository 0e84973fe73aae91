"""Generate tests/golden/confluence_cases.npz by executing the REAL reference's utils/confluence.py:confluence_process
(build container only; needs the reference tree, see oracle/ref_shim.py).

    python -m oracle.gen_golden_confluence

Inputs are built by `build_inputs()` (seeded PCG64) from the committed detector goldens: the reference's own decoded
yolov5s output (tests/golden/yolov5s_512x640.npz, nc = 1) and yolov5m FLIR output (yolov5m_flir_512x640.npz, nc = 3).
Most rows get obj = 0; a few hundred rows become jittered copies of real boxes, so that clusters form, with objectness
re-spread above the threshold.  The images cover exact duplicates (p = 0), zero-width boxes sharing an x (0/0 = NaN),
equal confidences, a class with a single candidate, an image without candidates, fp32 (nc = 1) and fp16 (nc = 3,
multi-label) inputs, each at the reference defaults (0.1, 0.6) and at test.py:140's (0.1, 0.5).  Only the reference's
kept rows are stored, with the SHA-256 of each input; the tests rebuild the inputs and check them against it.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.confluence import confluence_process as oracle_process  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SETTINGS = [("default", 0.1, 0.6), ("test", 0.1, 0.5)]


def _clusters(g, z, n_clusters, copies, jitter):
    """Rows of jittered copies of n_clusters real boxes of z, objectness above 0.1: (rows, no) fp32."""
    base = z[g.choice(z.shape[0], n_clusters, replace=False)]
    out = []
    for b in base:
        for _ in range(int(g.integers(1, copies + 1))):
            r = b.copy()
            r[:4] *= g.uniform(1 - jitter, 1 + jitter, size=4).astype(np.float32)
            r[4] = g.uniform(0.12, 1.0)
            r[5:] = g.uniform(0.15, 1.0, size=len(r) - 5)
            out.append(r)
    return np.array(out, dtype=np.float32)


def _place(g, z, rows):
    """z with every obj cleared and `rows` written at random row positions (kept in their order)."""
    x = z.copy()
    x[:, 4] = 0.0
    pos = np.sort(g.choice(z.shape[0], len(rows), replace=False))
    x[pos] = rows
    return x


def build_inputs(seed=7):
    """{"kaist": fp32 (3, 20160, 6), "flir": fp16 (2, 20160, 8)} predictions."""
    g = np.random.Generator(np.random.PCG64(seed))
    zs = np.load(os.path.join(OUT, "yolov5s_512x640.npz"))["z"][0].astype(np.float32)           # (20160, 6)
    zf = np.load(os.path.join(OUT, "yolov5m_flir_512x640.npz"))["z16"][0].astype(np.float32)    # (20160, 8)

    c = _clusters(g, zs, 60, 7, 0.04)                      # clustered
    dup = c[g.choice(len(c), 20, replace=False)]           # exact duplicates: p = 0, equal values
    zw = c[:6].copy()
    zw[:, 2] = 0.0                                         # zero-width boxes ...
    zw = np.concatenate([zw, zw])                          # ... sharing their x with a copy: 0/0 on the x axis
    zw[6:, 1] += 3.0
    eq = c[6:12].copy()
    eq[:, 4:] = 0.5                                        # equal confidences
    rows = np.concatenate([c, dup, zw, eq])
    im0 = _place(g, zs, rows[g.permutation(len(rows))])
    spread = _clusters(g, zs, 150, 1, 0.0)                 # spread boxes: mostly isolated
    im1 = _place(g, zs, spread)
    im2 = zs.copy()
    im2[:, 4] = 0.0                                        # no candidate
    kaist = np.stack([im0, im1, im2]).astype(np.float32)

    f = _clusters(g, zf, 40, 6, 0.05)
    f[:, 5:] *= (g.uniform(size=(len(f), 3)) < 0.6)        # some (row, class) pairs below the threshold
    f[:, 7] = 0.0
    f[0, 7] = 0.9                                          # class 2: a single candidate
    f = np.concatenate([f, f[1:11]])                       # duplicates across the classes
    fim0 = _place(g, zf, f[g.permutation(len(f))])
    f1 = _clusters(g, zf, 30, 8, 0.08)
    fim1 = _place(g, zf, f1)
    flir = np.stack([fim0, fim1]).astype(np.float16)
    return {"kaist": kaist, "flir": flir}


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def checked_inputs(meta) -> dict:
    """build_inputs(), each input asserted byte-identical to the one the golden was generated from."""
    inputs = build_inputs()
    for entry in meta["inputs"]:
        p = inputs[entry["name"]]
        assert list(p.shape) == entry["shape"] and digest(p) == entry["sha256"], \
            f"rebuilt input {entry['name']} differs from the golden's (numpy {np.__version__}, golden made with {meta['numpy']})"
    return inputs


def main():
    load_reference()
    from utils.confluence import confluence_process      # the reference's own function
    arrays, meta = {}, {"inputs": []}
    for name, pred in build_inputs().items():
        entry = dict(name=name, nc=int(pred.shape[2] - 5), dtype=str(pred.dtype), shape=list(pred.shape),
                     sha256=digest(pred), settings=[])
        for sname, conf, p_thres in SETTINGS:
            t0 = time.time()
            out = confluence_process(torch.from_numpy(pred), conf, p_thres)
            dt = time.time() - t0
            mine = oracle_process(pred, conf, p_thres)
            counts = []
            for b, (o, m) in enumerate(zip(out, mine)):
                assert (o is None) == (m is None), (name, sname, b)
                if o is not None:
                    assert np.array_equal(o.numpy(), m), (name, sname, b)
                    arrays[f"{name}_{sname}_{b}"] = o.numpy().astype(np.float32)
                counts.append(None if o is None else int(o.shape[0]))
            cand = (pred.astype(np.float32)[..., 4] > np.float32(conf)).sum(1).tolist()
            entry["settings"].append(dict(name=sname, conf=conf, p_thres=p_thres, counts=counts, rows_above=cand,
                                          seconds=round(dt, 1)))
            print(name, sname, "rows above", cand, "kept", counts, f"{dt:.1f} s")
        meta["inputs"].append(entry)
    meta["reference"] = "utils/confluence.py:50-106 confluence_process on the CPU; every case equals oracle.confluence"
    meta["torch"] = torch.__version__
    meta["numpy"] = np.__version__
    path = os.path.join(OUT, "confluence_cases.npz")
    np.savez_compressed(path, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
