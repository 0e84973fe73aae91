"""Generate tests/golden/train_accumulate_yolov5s_320.npz by executing train.py's accumulating loop around the REAL
reference's Model, ComputeLoss, SGD and ModelEMA (build container only).

    python -m oracle.gen_golden_train_accumulate

train.py:117-141 (groups, nominal batch 64, scaled weight decay, nesterov SGD), 238-244 (loss gains) and 291-352 (forward,
loss, backward, and an optimiser step + zero_grad + EMA update when ``ni % accumulate == 0``) transcribed on CPU fp32 with
GradScaler off, as it is on CPU.  yolov5s at 320 x 320, seeded synthetic weights (oracle/synth.py), dropout p = 0, micro-batches
of 2 images; total_batch_size 32 gives accumulate = 2, and four micro-batches make two optimiser steps (ni = 1 .. 4, past
warm-up: the LR stays lr0).  Stored: every micro-batch's loss, a fingerprint of the update of every parameter in the
optimiser's groups and of every EMA
entry's change, the running statistics of four BatchNorm layers and the num_batches_tracked counters.

``oracle_loop`` runs the same loop through oracle.icaf_oracle.train_step; the tests use it as the yardstick of the device.
"""
from __future__ import annotations

import json
import math
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from oracle.gen_golden_train import BN_PROBES, fingerprint, synth_targets  # noqa: E402
from oracle.ref_shim import REF_ROOT, load_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=0.0005, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0,
           fl_gamma=0.0)
CASE = dict(name="train_accumulate_yolov5s_320", size="s", B=2, H=320, W=320, nt=12, seed=1234, total_batch_size=32,
            micro_batches=4)


def batches(c=CASE):
    """The seeded micro-batches: (rgb, ir) float images in [0, 1] and (nt, 6) targets."""
    out = []
    for i in range(c["micro_batches"]):
        rgb, ir = synth.synth_images(c["B"], c["H"], c["W"], c["seed"] + 1 + i)
        out.append((rgb, ir, torch.from_numpy(synth_targets(c["nt"] + i, c["B"], c["seed"] + 1 + i))))
    return out


def scaled_hyp(nc: int = 1, nl: int = 3, c=CASE):
    """train.py:121 and 238-240: weight decay for the nominal batch, loss gains for nc, nl and the image size."""
    nbs = 64
    accumulate = max(round(nbs / c["total_batch_size"]), 1)
    h = dict(HYP)
    h["weight_decay"] *= c["total_batch_size"] * accumulate / nbs
    h["box"] *= 3.0 / nl
    h["cls"] *= nc / 80.0 * 3.0 / nl
    h["obj"] *= (c["H"] / 640) ** 2 * 3.0 / nl
    return h, accumulate


def _record(arrays, init, final, ema, losses):
    arrays["losses"] = np.asarray(losses, dtype=np.float64)
    for k in init:
        if init[k].is_floating_point():
            arrays["e:" + k] = fingerprint((ema[k].double() - init[k].double()).numpy(), "e:" + k)
    for k in BN_PROBES:
        arrays["rm:" + k] = final[k + ".running_mean"].numpy().copy()
        arrays["rv:" + k] = final[k + ".running_var"].numpy().copy()


def oracle_loop(sd, cfg, meta, data, autocast_device=None, loss_scale: float = 1.0):
    """The loop of main() through the oracle: -> ({name: parameter update}, final state, EMA state, [losses]).  Under
    autocast_device the forward and backward run in the reference's fp16 regime (static loss scale) on that device."""
    from oracle import icaf_oracle as O
    hyp, accumulate = scaled_hyp()
    groups = meta["groups"]
    state = {k: v.clone() for k, v in sd.items()}
    leaves = {k: state[k].clone() for g in groups for k in g}
    opt = torch.optim.SGD([leaves[k] for k in groups[0]], lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)
    opt.add_param_group({"params": [leaves[k] for k in groups[1]], "weight_decay": hyp["weight_decay"]})
    opt.add_param_group({"params": [leaves[k] for k in groups[2]]})
    ema, updates = {k: v.clone() for k, v in state.items()}, 0
    losses = []
    for ni, (rgb, ir, t) in enumerate(data, 1):
        for k, v in leaves.items():
            state[k] = v.detach().clone()
        loss, _, grads, _, new = O.train_step(state, cfg, rgb, ir, t, hyp, 1.0, autocast_device=autocast_device, loss_scale=loss_scale)
        losses.append(float(loss.reshape(-1)[0]))
        for k, v in new.items():
            if k.endswith(("running_mean", "running_var")):
                state[k] = v.detach().float().cpu()
            elif k.endswith("num_batches_tracked"):
                state[k] = state[k] + 1
        for k, g in grads.items():
            if k in leaves:
                g = g.float().cpu()
                leaves[k].grad = g if leaves[k].grad is None else leaves[k].grad + g
        if ni % accumulate == 0:                                                  # train.py:346-352
            opt.step()
            opt.zero_grad()
            for k, v in leaves.items():
                state[k] = v.detach().clone()
            updates += 1
            d = 0.9999 * (1 - math.exp(-updates / 2000))
            for k, v in ema.items():
                if v.is_floating_point():
                    ema[k] = v * d + (1.0 - d) * state[k]
    upd = {k: leaves[k].detach() - sd[k] for k in leaves}
    return upd, state, ema, losses


def main():
    warnings.filterwarnings("ignore")
    _, yolo = load_reference()
    from utils.loss import ComputeLoss
    from utils.torch_utils import ModelEMA
    c = CASE
    cfg = os.path.join(REF_ROOT, "models", "transformer", f"yolov5{c['size']}_Transfusion_kaist.yaml")
    model = yolo.Model(cfg, ch=3, nc=1)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = synth.synth_state_dict(shapes, c["seed"])
    missing = model.load_state_dict(sd, strict=False)
    assert all(k.endswith(("anchors", "anchor_grid")) for k in missing.missing_keys) and not missing.unexpected_keys
    model.train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    init = {k: v.detach().clone() for k, v in model.state_dict().items()}
    hyp, accumulate = scaled_hyp()
    assert accumulate == 2
    names = {id(p): k for k, p in model.named_parameters()}
    pg0, pg1, pg2 = [], [], []                                                   # train.py:126-131
    for k, v in model.named_modules():
        if hasattr(v, "bias") and isinstance(v.bias, torch.nn.Parameter):
            pg2.append(v.bias)
        if isinstance(v, torch.nn.BatchNorm2d):
            pg0.append(v.weight)
        elif hasattr(v, "weight") and isinstance(v.weight, torch.nn.Parameter):
            pg1.append(v.weight)
    optimizer = torch.optim.SGD(pg0, lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)      # train.py:136
    optimizer.add_param_group({"params": pg1, "weight_decay": hyp["weight_decay"]})
    optimizer.add_param_group({"params": pg2})
    ema = ModelEMA(model)                                                        # train.py:154
    model.nc, model.hyp, model.gr = 1, hyp, 1.0                                  # train.py:242-244
    compute_loss = ComputeLoss(model)
    losses = []
    optimizer.zero_grad()                                                        # train.py:291
    for ni, (rgb, ir, t) in enumerate(batches(), 1):
        pred = model(rgb, ir)                                                    # train.py:336
        loss, _ = compute_loss(pred, t)                                          # train.py:338
        loss.backward()                                                          # train.py:344 (GradScaler off on CPU)
        losses.append(float(loss))
        if ni % accumulate == 0:                                                 # train.py:346-352
            optimizer.step()
            optimizer.zero_grad()
            ema.update(model)
    final = {k: v.detach().clone() for k, v in model.state_dict().items()}
    arrays = {}
    grouped = sorted(names[id(p)] for g in (pg0, pg1, pg2) for p in g)
    for k in grouped:
        arrays["u:" + k] = fingerprint((final[k].double() - init[k].double()).numpy(), "u:" + k)
    _record(arrays, init, final, ema.ema.state_dict(), losses)
    nbt = {k: int(v) for k, v in final.items() if k.endswith("num_batches_tracked")}
    meta = dict(c, hyp=hyp, accumulate=accumulate, gr=1.0, bn_probes=BN_PROBES, num_batches_tracked=nbt,
                groups=[[names[id(p)] for p in g] for g in (pg0, pg1, pg2)],
                reference="train.py:117-141,238-244,291-352 around models/yolo_test.py Model, utils/loss.py ComputeLoss, "
                          "torch.optim.SGD and utils/torch_utils.py ModelEMA; dropout p=0, fp32 CPU, GradScaler off",
                torch=torch.__version__)
    path = os.path.join(OUT, c["name"] + ".npz")
    np.savez_compressed(path, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print(f"losses {losses}  {len(grouped)} parameters in the optimiser's groups  -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
