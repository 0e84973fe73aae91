"""Generate tests/golden/nms_multilabel_cases.npz by executing the REAL reference's
utils/general.py:non_max_suppression(..., multi_label=True) (build container only; needs /root/reference).

    python -m oracle.gen_golden_nms_multilabel

Inputs are fp16 predictions built by `build_inputs()` from the committed detector golden
tests/golden/yolov5m_flir_512x640.npz (`z16`: the reference's own decoded yolov5m FLIR output, nc = 3): the image as is,
a perturbed copy and an image without candidates (one batch whose images have different counts), and a 9-class
(VEDAI-like) batch whose class scores are re-spread copies of the three real ones.  Settings: test.py's (conf 0.001 /
iou 0.6: 60 480 candidates, above max_nms = 30000), detect's (0.25 / 0.45), agnostic (what test.py's single_cls passes)
and a class filter.  The inputs are not stored: the tests rebuild them with `build_inputs()` (seeded PCG64) and check
them against the SHA-256 stored per input, so only the reference's kept rows are kept in the repository.

The reference cuts to max_nms with `argsort(descending=True)`, which is not stable on the CPU; every stored case is
asserted equal to the stable-order restatement (oracle.nms_multilabel), so the golden pins the order a stable sort gives
and no case rests on how the CPU sort happened to break ties.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.nms_multilabel import non_max_suppression_multilabel  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SETTINGS = {  # input -> [(name, conf, iou, agnostic, classes)]
    "flir": [("test", 0.001, 0.6, False, None),         # test.py:139 with test.py's defaults
             ("detect", 0.25, 0.45, False, None),       # detect_twostream.py defaults
             ("agnostic", 0.001, 0.6, True, None),      # test.py --single-cls
             ("classes", 0.25, 0.45, False, [0, 2])],
    "vedai": [("test", 0.001, 0.6, False, None),
              ("detect", 0.25, 0.45, False, None)],
}


def build_inputs(seed=11):
    """{"flir": (3, 20160, 8), "vedai": (2, 20160, 14)} fp16 predictions."""
    g = np.random.Generator(np.random.PCG64(seed))
    z = np.load(os.path.join(OUT, "yolov5m_flir_512x640.npz"))["z16"].astype(np.float32)[0]    # (20160, 8)
    R = z.shape[0]
    pert = z[::-1].copy()                                   # other row order, other sizes, other scores
    pert[:, 2:4] *= g.uniform(0.8, 1.25, size=(R, 2)).astype(np.float32)
    pert[:, 4] = g.beta(0.6, 2.0, size=R).astype(np.float32)
    pert[g.uniform(size=R) < 0.6, 4] = 0.0                  # below max_nms at test.py's setting: no tie-breaking cut
    pert[:, 5:] = np.clip(pert[:, 5:] * g.uniform(0.3, 1.4, size=(R, 3)).astype(np.float32), 0, 1)
    empty = z.copy()
    empty[:, 4] = 0.0                                       # no row passes obj > conf_thres
    flir = np.stack([z, pert, empty]).astype(np.float16)
    cls9 = np.concatenate([z[:, 5:] * f for f in (1.0, 0.7, 0.45)], 1)
    cls9 = np.clip(cls9 * g.uniform(0.5, 1.3, size=cls9.shape), 0, 1).astype(np.float32)
    v0 = np.concatenate([z[:, :5], cls9], 1)
    v0[g.uniform(size=R) < 0.85, 4] = 0.0                   # < 30000 candidates of 9 classes: no tie-breaking cut
    v1 = v0[g.permutation(R)].copy()
    v1[:, 4] = g.beta(0.3, 3.0, size=R).astype(np.float32)
    vedai = np.stack([v0, v1]).astype(np.float16)
    return {"flir": flir, "vedai": vedai}


def digest(pred16: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(pred16).tobytes()).hexdigest()


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
    from utils.general import non_max_suppression      # the reference's own function
    arrays, meta = {}, {"inputs": []}
    for inp, pred16 in build_inputs().items():
        pred = torch.from_numpy(pred16).float()
        entry = dict(name=inp, nc=int(pred16.shape[2] - 5), shape=list(pred16.shape), sha256=digest(pred16), settings=[])
        for name, conf, iou, agn, classes in SETTINGS[inp]:
            out = non_max_suppression(pred, conf, iou, classes=classes, agnostic=agn, multi_label=True)
            stable = non_max_suppression_multilabel(pred, conf, iou, classes=classes, agnostic=agn)
            for b, (o, s) in enumerate(zip(out, stable)):
                assert np.array_equal(o.numpy(), s.numpy()), f"{inp}/{name} image {b}: the reference's unstable cut differs"
            pair = (pred[..., 4:5] > conf) & (pred[..., 5:] * pred[..., 4:5] > conf)
            if classes is not None:
                pair &= torch.isin(torch.arange(pair.shape[2]), torch.tensor(classes))
            n_cand = pair.sum((1, 2)).tolist()
            counts = [int(o.shape[0]) for o in out]
            entry["settings"].append(dict(name=name, conf=conf, iou=iou, agnostic=agn, classes=classes, counts=counts,
                                          candidates=n_cand))
            for b, o in enumerate(out):
                arrays[f"{inp}_{name}_{b}"] = o.numpy().astype(np.float32)
            print(inp, name, "candidates", n_cand, "kept", counts)
        meta["inputs"].append(entry)
    meta["reference"] = ("utils/general.py:518-607 non_max_suppression(multi_label=True) on pred.float() (CPU, "
                         "torchvision.ops.nms); every case equals the stable-order restatement")
    meta["torch"] = torch.__version__
    meta["numpy"] = np.__version__
    path = os.path.join(OUT, "nms_multilabel_cases.npz")
    np.savez_compressed(path, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
