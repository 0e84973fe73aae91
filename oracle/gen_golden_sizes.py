"""Generate the yolov5n / yolov5m golden files by executing the REAL reference (build container only).

    python -m oracle.gen_golden_sizes            # needs /root/reference (read-only, never copied)

Same scheme as gen_golden.py (model forwards) and gen_golden_train.py (one training step); weights, images and targets are
rebuilt from their seeds by the tests.  Writes to tests/golden/:
  yolov5n_flir_320, yolov5m_flir_320, yolov5m_flir_512x640 : Model(yolov5{n,m}_Transfusion_FLIR.yaml).eval() forward,
                                                              unfused and .fuse()d, with the reference's fp16 self-deviation
  train_yolov5n_flir_320                                    : loss, gradient fingerprints, dead parameters, BN probes
  reference_yaml_sizes.json                                 : models/transformer/yolov5{n,m}_Transfusion_{kaist,FLIR}.yaml as
                                                              parsed by yaml.safe_load

The model files stay small: they hold the detections z rounded to fp16 (what the fp16 CUDA path is compared with, at 3e-3;
the rounding is <= 2^-11 of each element) and a float64 fingerprint (gen_golden_train.fingerprint: L2 norm and two seeded
projections) of each fp32 output -- z, z of the fused model, logits and the three head maps -- which pins the fp32 oracle to
the reference at 2e-5 without storing the arrays.  The fused and unfused z differ by ~1e-6 of their maximum (meta
'fused_dev'), far below fp16's resolution, so the one fp16 z serves both.
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
    # name,                  size, B, H,   W
    ("yolov5n_flir_320", "n", 2, 320, 320),
    ("yolov5m_flir_320", "m", 2, 320, 320),
    ("yolov5m_flir_512x640", "m", 1, 512, 640),
]
TRAIN_CASE = dict(name="train_yolov5n_flir_320", size="n", dataset="FLIR", nc=3, B=2, H=320, W=320, nt=12, seed=1234)
YAMLS = [(s, ds) for s in ("n", "m") for ds in ("kaist", "FLIR")]


def _yaml(size, dataset="FLIR"):
    return os.path.join(REF_ROOT, "models", "transformer", f"yolov5{size}_Transfusion_{dataset}.yaml")


def models(yolo, seed=1234):
    for name, size, B, H, W in MODEL_CASES:
        model = yolo.Model(_yaml(size), ch=3).eval()
        nc = model.yaml["nc"]
        _load_synth(model, seed)
        rgb, ir = synth.synth_images(B, H, W, seed)
        z, logits, xs = model(rgb, ir)
        fused = yolo.Model(_yaml(size), ch=3).eval()
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
        meta = dict(kind="model", size=size, dataset="FLIR", nc=nc, B=B, H=H, W=W, seed=seed, ref_fp16_self_dev=dev16,
                    fused_dev=fused_dev, shapes={k: list(v.shape) for k, v in outs.items()},
                    reference=f"models/yolo_test.py Model(yolov5{size}_Transfusion_FLIR.yaml).eval() forward, plus .fuse() variant",
                    torch=torch.__version__)
        _save(name, meta, z16=z.numpy().astype(np.float16), **{"fp:" + k: fingerprint(v.numpy(), k) for k, v in outs.items()})


def train_step(yolo):
    """gen_golden_train.main on yolov5n_Transfusion_FLIR."""
    from utils.loss import ComputeLoss
    c = TRAIN_CASE
    model = yolo.Model(_yaml(c["size"], c["dataset"]), ch=3)
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
    t[:, 1] = np.arange(c["nt"]) % c["nc"]                                       # every class present
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


def yamls():
    import yaml
    cfgs = {}
    for size, ds in YAMLS:
        with open(_yaml(size, ds)) as f:
            cfgs[f"yolov5{size}_Transfusion_{ds}"] = yaml.safe_load(f)
    path = os.path.join(OUT, "reference_yaml_sizes.json")
    with open(path, "w") as f:
        json.dump(cfgs, f, separators=(",", ":"))
    print(f"wrote {path}")


def main():
    warnings.filterwarnings("ignore")
    _, yolo = load_reference()
    yamls()
    with torch.no_grad():
        models(yolo)
    train_step(yolo)


if __name__ == "__main__":
    main()
