"""Generate tests/golden/loss_focal_cases.npz by executing the REAL reference's utils/loss.py:ComputeLoss with focal loss on
(hyp fl_gamma > 0, loss.py:341-344) (build container only).

    python -m oracle.gen_golden_loss_focal

The cases and seeded inputs are gen_golden_loss.py's (KAIST nc=1, nc=3 with label smoothing and non-unit BCE weights,
gr = 0.5, no targets), each run with fl_gamma 1.5 (the hyp files' "efficientDet default") and 2.0.  Per case and gamma:
the reference's outputs, the coarsest level's gradient in full and a 3-number fingerprint per level.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.gen_golden_loss import CASES, HYP, OUT, grad_fingerprint, synth_case  # noqa: E402
from oracle.ref_shim import REF_ROOT, load_reference  # noqa: E402

GAMMAS = (1.5, 2.0)


def main():
    _, yolo = load_reference()
    from utils.loss import ComputeLoss
    arrays, meta = {}, {"cases": []}
    for gamma in GAMMAS:
        for name, nc, B, nt, gr, over in CASES:
            key = f"{name}_g{gamma:g}"
            cfg = os.path.join(REF_ROOT, "models", "transformer", "yolov5s_Transfusion_kaist.yaml")
            model = yolo.Model(cfg, ch=3, nc=nc)
            hyp = dict(HYP, **over, fl_gamma=gamma)
            model.hyp, model.gr = hyp, gr
            loss_fn = ComputeLoss(model)
            assert type(loss_fn.BCEcls).__name__ == "FocalLoss" and type(loss_fn.BCEobj).__name__ == "FocalLoss"
            p, t = synth_case(name, nc, B, nt)
            pt = [torch.from_numpy(x).requires_grad_(True) for x in p]
            loss, items = loss_fn(pt, torch.from_numpy(t))
            loss.sum().backward()
            for lvl, x in enumerate(pt):
                arrays[f"{key}_gproj{lvl}"] = grad_fingerprint(x.grad.numpy(), lvl)
            arrays[f"{key}_grad2"] = pt[2].grad.numpy().astype(np.float32)
            arrays[f"{key}_targets"] = t
            arrays[f"{key}_out"] = np.concatenate([loss.detach().numpy().reshape(1), items.numpy()]).astype(np.float32)
            arrays[f"{key}_anchors"] = model.model[-1].anchors.numpy().astype(np.float32)
            meta["cases"].append(dict(key=key, name=name, nc=nc, B=B, nt=nt, gr=gr, hyp=hyp))
            print(key, arrays[f"{key}_out"])
    meta["reference"] = "utils/loss.py:37-64,325-463 ComputeLoss(model)(p, targets) with hyp fl_gamma > 0, fp32 CPU"
    meta["torch"] = torch.__version__
    np.savez_compressed(os.path.join(OUT, "loss_focal_cases.npz"), meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print("wrote", os.path.join(OUT, "loss_focal_cases.npz"))


if __name__ == "__main__":
    main()
