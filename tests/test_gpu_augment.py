"""Device training augmentation (icaf_augment via icafusion_b200.augment.Augment) against the reference's loader (golden from
utils/datasets.py:LoadMultiModalImagesAndLabels(augment=True) + collate_fn) and against the numpy restatement at B = 16,
s = 640, byte for byte."""
import json
import os
import random

import numpy as np
import pytest
import torch

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "augment_cases.npz")
CASES = ["mosaic_r1", "mosaic_resize", "letterbox", "degrees_shear", "flipud"]
HYP_SCRATCH = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0,
                   flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.0)


def _golden():
    g = np.load(GOLDEN)
    meta = json.loads(bytes(g["meta"]).decode())
    n = meta["frames"]
    return g, meta, {k: (g[f"rgb{k}"], g[f"ir{k}"]) for k in range(n)}, [g[f"labels{k}"] for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("frames_on", ["host", "device"])
@pytest.mark.parametrize("name", CASES)
def test_device_batch_equals_the_reference_loader(cuda_device, name, frames_on):
    from icafusion_b200.augment import Augment
    g, meta, frames, labels = _golden()
    if frames_on == "device":
        frames = {k: tuple(torch.from_numpy(f).to(cuda_device) for f in v) for k, v in frames.items()}
    case = next(c for c in meta["cases"] if c["name"] == name)
    aug = Augment(labels, frames.__getitem__, case["img_size"], case["hyp"], device=cuda_device)
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    rgb, ir, targets = aug(case["indices"])
    torch.cuda.synchronize()
    img = g[f"{name}_img"]
    assert rgb.shape == (len(case["indices"]), 3, case["img_size"], case["img_size"]) and rgb.dtype == torch.uint8
    assert np.array_equal(rgb.cpu().numpy(), img[:, :3])
    assert np.array_equal(ir.cpu().numpy(), img[:, 3:])
    assert targets.is_cuda and np.array_equal(targets.cpu().numpy(), g[f"{name}_targets"])
    assert [random.random(), np.random.random()] == list(g[f"{name}_next"])


def _kaist_like(n, seed=3):
    """n RGB/IR pairs, mostly 512 x 640 (KAIST / FLIR) and a few other sizes, with 0-8 random boxes each."""
    g = np.random.default_rng(seed)
    frames, labels = {}, []
    for k in range(n):
        h, w = (512, 640) if k % 4 else [(480, 640), (720, 1280), (600, 600)][k // 4 % 3]
        yy, xx = np.mgrid[0:h, 0:w]
        base = (xx * (k + 3) // 7 + yy * (k + 5) // 9) % 256
        rgb = np.stack([(base + 60 * c + g.integers(0, 24, (h, w))) % 256 for c in range(3)], -1).astype(np.uint8)
        ir = np.repeat(((base // 2 + g.integers(0, 16, (h, w))) % 256)[..., None], 3, -1).astype(np.uint8)
        frames[k] = (rgb, ir)
        nb = int(g.integers(0, 9))
        wh = g.uniform(0.02, 0.4, (nb, 2))
        labels.append(np.concatenate([g.integers(0, 2, (nb, 1)), g.uniform(wh / 2, 1 - wh / 2), wh], 1).astype(np.float32))
    return frames, labels


@pytest.mark.gpu
@pytest.mark.parametrize("over", [{}, dict(degrees=10.0, shear=5.0, flipud=0.5, mosaic=0.7)])
def test_batch16_640_equals_the_restatement(cuda_device, over):
    from icafusion_b200.augment import Augment
    frames, labels = _kaist_like(24)
    hyp = dict(HYP_SCRATCH, **over)
    aug = Augment(labels, frames.__getitem__, 640, hyp, device=cuda_device)
    indices = list(range(16))
    random.seed(7)
    np.random.seed(7)
    rgb, ir, targets = aug(indices)
    torch.cuda.synchronize()
    random.seed(7)
    np.random.seed(7)
    want_rgb, want_ir, want_t = aug.reference(indices)
    assert rgb.shape == (16, 3, 640, 640)
    assert np.array_equal(rgb.cpu().numpy(), want_rgb)
    assert np.array_equal(ir.cpu().numpy(), want_ir)
    assert np.array_equal(targets.cpu().numpy(), want_t)


@pytest.mark.gpu
def test_unsupported_settings_and_bad_arguments_raise(cuda_device):
    from icafusion_b200 import _lib
    from icafusion_b200.augment import Augment
    g, meta, frames, labels = _golden()
    hyp = meta["cases"][0]["hyp"]
    with pytest.raises(NotImplementedError):
        Augment(labels, frames.__getitem__, 320, dict(hyp, perspective=0.0005), device=cuda_device)
    with pytest.raises(NotImplementedError):
        Augment(labels, frames.__getitem__, 320, dict(hyp, mixup=0.1), device=cuda_device)
    bad = dict(frames)
    bad[0] = (frames[0][0], frames[0][1][:-2])                          # RGB / IR of one pair differ in size
    aug = Augment(labels, bad.__getitem__, 320, dict(hyp, mosaic=0.0), device=cuda_device)
    with pytest.raises(ValueError):
        aug([0])
    L = _lib.lib()
    need = L.icaf_augment_params_bytes(2, 320, 0)
    buf = torch.zeros(need, dtype=torch.uint8, device=cuda_device)
    out = torch.empty(2, 3, 320, 320, dtype=torch.uint8, device=cuda_device)
    assert L.icaf_augment(buf.data_ptr(), need - 1, 2, 320, 0, out.data_ptr(), out.data_ptr(), None) == 1
    assert L.icaf_augment(buf.data_ptr() + 4, need, 2, 320, 0, out.data_ptr(), out.data_ptr(), None) == 1
