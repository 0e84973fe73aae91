"""Generate the yolov5x golden files by executing the REAL reference (build container only).

    python -m oracle.gen_golden_sizes_x          # needs /root/reference (read-only, never copied)

The reference ships no yolov5x_Transfusion_*.yaml, but its Model accepts a config dict (models/yolo_test.py:77).  The x
config is its own yolov5l_Transfusion_{kaist,FLIR}.yaml with YOLOv5's x multiples (depth 1.33, width 1.25) in place of
l's; everything else in the rows is shared by the sizes.  Writes to tests/golden/, in the scheme of gen_golden_sizes.models
(z rounded to fp16, float64 fingerprints of the fp32 z, fused z, logits and head maps, the fused / unfused deviation and
the reference's own fp16 self-deviation):
  yolov5x_flir_320, yolov5x_flir_512x640 : Model(x config, FLIR).eval() forward, unfused and .fuse()d
  reference_cfg_x.json                   : the config dicts the reference's Model was built from (Model.yaml), kaist and FLIR
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
from oracle.gen_golden_train import fingerprint  # noqa: E402
from oracle.ref_shim import REF_ROOT, load_reference  # noqa: E402

X_MULT = {"depth_multiple": 1.33, "width_multiple": 1.25}
MODEL_CASES = [
    # name,                  B, H,   W
    ("yolov5x_flir_320", 2, 320, 320),
    ("yolov5x_flir_512x640", 1, 512, 640),
]


def x_cfg(dataset):
    """The reference's l YAML for `dataset` with the x multiples."""
    import yaml
    with open(os.path.join(REF_ROOT, "models", "transformer", f"yolov5l_Transfusion_{dataset}.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg.update(X_MULT)
    return cfg


def configs(yolo):
    """Build the reference's Model from each x config and record the dict it parsed."""
    out = {}
    for ds in ("kaist", "FLIR"):
        model = yolo.Model(x_cfg(ds), ch=3)
        out[f"yolov5x_Transfusion_{ds}"] = model.yaml
    path = os.path.join(OUT, "reference_cfg_x.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print(f"wrote {path}")


def models(yolo, seed=1234):
    for name, B, H, W in MODEL_CASES:
        model = yolo.Model(x_cfg("FLIR"), ch=3).eval()
        nc = model.yaml["nc"]
        _load_synth(model, seed)
        rgb, ir = synth.synth_images(B, H, W, seed)
        z, logits, xs = model(rgb, ir)
        fused = yolo.Model(x_cfg("FLIR"), ch=3).eval()
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
        meta = dict(kind="model", size="x", dataset="FLIR", nc=nc, B=B, H=H, W=W, seed=seed, ref_fp16_self_dev=dev16,
                    fused_dev=fused_dev, shapes={k: list(v.shape) for k, v in outs.items()},
                    reference="models/yolo_test.py Model(yolov5l_Transfusion_FLIR.yaml with depth 1.33 / width 1.25).eval() "
                              "forward, plus .fuse() variant",
                    torch=torch.__version__)
        _save(name, meta, z16=z.numpy().astype(np.float16), **{"fp:" + k: fingerprint(v.numpy(), k) for k, v in outs.items()})
        print(f"{name}: fused_dev {fused_dev:.2e}  reference fp16 self-dev {dev16}")


def main():
    warnings.filterwarnings("ignore")
    _, yolo = load_reference()
    configs(yolo)
    with torch.no_grad():
        models(yolo)


if __name__ == "__main__":
    main()
