"""Generate the goldens at the shapes training and validation run, by executing the REAL reference (build container only).

    python -m oracle.gen_golden_shapes          # needs /root/reference (read-only, never copied)

test.py and train.py's validation loader batch the 512x640 frames of both datasets as rectangles (rect=True, pad=0.5):
ceil(shape * 640 / 32 + 0.5) * 32 = 544x672.  There P5 is 17x21 and the DMFF token pooling runs irregular overlapping
windows (P3 68x84 -> 20x20: kernel (11, 8), stride (3, 4); P4 34x42 -> 16x16: (4, 12), (2, 2); P5 17x21 -> 10x10: (8, 3),
(1, 2)).  train.py's mosaic batches are img_size x img_size = 640x640.  Same scheme as gen_golden_sizes.py (model forwards:
z in fp16 plus float64 fingerprints of every fp32 output) and gen_golden_train.py (one training step).  Writes to
tests/golden/:
  yolov5s_544x672, yolov5l_flir_544x672 : Model(...).eval() forward, unfused and .fuse()d, with the reference's fp16
                                          self-deviation
  train_yolov5s_640                     : train.py:334-344 on KAIST at 640x640, batch 2: loss, gradient fingerprints, dead
                                          parameters, BN probes
"""
from __future__ import annotations

import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from oracle.gen_golden import OUT, _load_synth, _save  # noqa: E402
from oracle.gen_golden_train import BN_PROBES, HYP, fingerprint, synth_targets  # noqa: E402
from oracle.ref_shim import REF_ROOT, load_reference  # noqa: E402

MODEL_CASES = [
    # name,                  size, dataset, B, H,   W
    ("yolov5s_544x672", "s", "kaist", 1, 544, 672),
    ("yolov5l_flir_544x672", "l", "FLIR", 1, 544, 672),
]
TRAIN_CASE = dict(name="train_yolov5s_640", size="s", dataset="kaist", nc=1, B=2, H=640, W=640, nt=16, seed=1234)


def _model(yolo, size, dataset):
    cfg = os.path.join(REF_ROOT, "models", "transformer", f"yolov5{size}_Transfusion_{dataset}.yaml")
    return yolo.Model(cfg, ch=3, nc=1) if dataset == "kaist" else yolo.Model(cfg, ch=3)


def models(yolo, seed=1234):
    for name, size, dataset, B, H, W in MODEL_CASES:
        model = _model(yolo, size, dataset).eval()
        nc = model.yaml["nc"]
        _load_synth(model, seed)
        rgb, ir = synth.synth_images(B, H, W, seed)
        z, logits, xs = model(rgb, ir)
        fused = _model(yolo, size, dataset).eval()
        _load_synth(fused, seed)
        fused.fuse()
        zf = fused(rgb, ir)[0]
        dev16 = None
        try:     # how far the reference's own fp16 path (detect_twostream.py:40-41) sits from its fp32 path
            z16 = fused.half()(rgb.half(), ir.half())[0].float()
            dev16 = float((z16 - zf).abs().max() / zf.abs().max())
        except Exception as e:  # noqa: BLE001
            print("fp16 CPU run failed:", e)
        fused_dev = float((zf - z).abs().max() / z.abs().max())
        assert fused_dev < 1e-5, fused_dev          # one fp16 z stands for both
        outs = dict(z=z, z_fused=zf, logits=logits, x0=xs[0], x1=xs[1], x2=xs[2])
        meta = dict(kind="model", size=size, dataset=dataset, nc=nc, B=B, H=H, W=W, seed=seed, ref_fp16_self_dev=dev16,
                    fused_dev=fused_dev, shapes={k: list(v.shape) for k, v in outs.items()},
                    reference=f"models/yolo_test.py Model(yolov5{size}_Transfusion_{dataset}.yaml).eval() forward, plus .fuse() variant",
                    torch=torch.__version__)
        _save(name, meta, z16=z.numpy().astype(np.float16), **{"fp:" + k: fingerprint(v.numpy(), k) for k, v in outs.items()})


def train_step(yolo):
    """gen_golden_train.main at 640x640."""
    from utils.loss import ComputeLoss
    c = TRAIN_CASE
    model = _model(yolo, c["size"], c["dataset"])
    assert model.yaml["nc"] == c["nc"]
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    missing = model.load_state_dict(synth.synth_state_dict(shapes, c["seed"]), strict=False)
    assert all(k.endswith(("anchors", "anchor_grid")) for k in missing.missing_keys) and not missing.unexpected_keys
    model.train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.hyp, model.gr = dict(HYP), 1.0
    rgb, ir = synth.synth_images(c["B"], c["H"], c["W"], c["seed"])
    t = synth_targets(c["nt"], c["B"], c["seed"])
    pred = model(rgb, ir)                                                        # train.py:336
    loss, items = ComputeLoss(model)(pred, torch.from_numpy(t))                  # train.py:338
    loss.backward()                                                              # train.py:344
    arrays = {"targets": t, "out": np.concatenate([loss.detach().numpy().reshape(1), items.numpy()]).astype(np.float32)}
    names, dead = [], []
    for k, p in model.named_parameters():
        if p.grad is None:
            dead.append(k)
            continue
        names.append(k)
        arrays["g:" + k] = fingerprint(p.grad.numpy(), k)
    for i, x in enumerate(pred):
        arrays[f"pred{i}"] = fingerprint(x.detach().numpy(), f"pred{i}")
    state = model.state_dict()
    for k in BN_PROBES:
        arrays["rm:" + k] = state[k + ".running_mean"].numpy().copy()
        arrays["rv:" + k] = state[k + ".running_var"].numpy().copy()
    meta = dict(c, hyp=HYP, gr=1.0, params=names, dead_params=dead, bn_probes=BN_PROBES,
                reference="models/yolo_test.py Model.train() forward + utils/loss.py ComputeLoss + backward (train.py:334-344), dropout p=0, fp32 CPU",
                torch=torch.__version__)
    path = os.path.join(OUT, c["name"] + ".npz")
    np.savez_compressed(path, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print(f"loss {arrays['out']}  {len(names)} live / {len(dead)} dead parameters  -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


def main():
    warnings.filterwarnings("ignore")
    _, yolo = load_reference()
    with torch.no_grad():
        models(yolo)
    train_step(yolo)


if __name__ == "__main__":
    main()
