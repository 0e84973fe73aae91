"""Host half of the device training augmentation (icafusion_b200/augment.py): the numpy restatement of the kernel's
arithmetic equals cv2 bit for bit (warpAffine, the HSV round trip over every colour, resize), the sampler draws what the
reference's loader draws and leaves `random` / `np.random` where it leaves them, and the whole transform -- images and
targets -- equals the golden taken from the reference's LoadMultiModalImagesAndLabels (tests/golden/augment_cases.npz)."""
import json
import math
import os
import random

import numpy as np
import pytest

from conftest import ROOT

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(ROOT, "tests", "golden", "augment_cases.npz")


def _golden():
    g = np.load(GOLDEN)
    meta = json.loads(bytes(g["meta"]).decode())
    n = meta["frames"]
    frames = {k: (g[f"rgb{k}"], g[f"ir{k}"]) for k in range(n)}
    labels = [g[f"labels{k}"] for k in range(n)]
    return g, meta, frames, labels


def _drawn_matrices(n, degrees, shear, s, seed):
    from icafusion_b200.augment import draw_affine
    random.seed(seed)
    return [draw_affine(2 * s, [-s // 2, -s // 2], degrees, 0.1, 0.5, shear, 0.0)[0] for _ in range(n)]


@pytest.mark.parametrize("degrees,shear", [(0.0, 0.0), (10.0, 5.0), (45.0, 20.0)])
def test_warp_affine_matches_cv2(degrees, shear):
    """warp_tables + the fixed-point gather == cv2.warpAffine(INTER_LINEAR, border 114) on drawn matrices, 2s canvases -> s."""
    from icafusion_b200.augment import warp_fixed, warp_tables
    s = 320
    g = np.random.default_rng(1)
    canvas = g.integers(0, 256, (2 * s, 2 * s, 3), dtype=np.uint8)
    canvas[:, : s // 3] = 114                       # grey like the mosaic background, so border taps mix with it
    for M in _drawn_matrices(6, degrees, shear, s, seed=int(degrees * 7 + shear)):
        want = cv2.warpAffine(canvas, M[:2], dsize=(s, s), borderValue=(114, 114, 114))
        got = warp_fixed(canvas, warp_tables(M, s), s)
        assert np.array_equal(got, want)
    # a matrix that moves most of the canvas off the output (border taps everywhere along one side)
    M = np.array([[1.3, 0.2, -500.0], [-0.1, 0.9, 40.5], [0, 0, 1]])
    assert np.array_equal(warp_fixed(canvas, warp_tables(M, s), s),
                          cv2.warpAffine(canvas, M[:2], dsize=(s, s), borderValue=(114, 114, 114)))


def test_rotation_matrix_matches_cv2():
    from icafusion_b200.augment import rotation_matrix_2d
    g = np.random.default_rng(2)
    for a, sc in zip(g.uniform(-45, 45, 50), g.uniform(0.5, 1.5, 50)):
        want = cv2.getRotationMatrix2D(angle=float(a), center=(0, 0), scale=float(sc))
        assert np.array_equal(rotation_matrix_2d(float(a), float(sc)), want)


def test_bgr2hsv_matches_cv2_on_every_colour():
    from icafusion_b200.augment import bgr2hsv_fixed
    img = np.arange(1 << 24, dtype=np.uint32).view(np.uint8).reshape(4096, 4096, 4)[..., :3].copy()
    for r0 in range(0, 4096, 1024):
        part = img[r0:r0 + 1024]
        assert np.array_equal(bgr2hsv_fixed(part), cv2.cvtColor(part, cv2.COLOR_BGR2HSV))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_hsv_jitter_matches_cv2_on_every_colour(seed):
    """augment_hsv (utils/datasets.py:1129-1140, restated with cv2) == hsv_jitter_fixed over all 2^24 colours."""
    from icafusion_b200.augment import hsv_jitter_fixed, hsv_luts
    np.random.seed(seed)
    r = np.random.uniform(-1, 1, 3) * [0.015 if seed < 2 else 0.3, 0.7, 0.4] + 1
    lut = hsv_luts(r)
    img = np.arange(1 << 24, dtype=np.uint32).view(np.uint8).reshape(4096, 4096, 4)[..., :3].copy()
    for r0 in range(0, 4096, 1024):
        part = img[r0:r0 + 1024]
        hue, sat, val = cv2.split(cv2.cvtColor(part, cv2.COLOR_BGR2HSV))
        hsv = cv2.merge((cv2.LUT(hue, lut[0]), cv2.LUT(sat, lut[1]), cv2.LUT(val, lut[2])))
        want = cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)
        assert np.array_equal(hsv_jitter_fixed(part, lut), want)


def test_hsv2bgr_matches_cv2_on_every_hsv_triple():
    from icafusion_b200.augment import hsv2bgr_fixed
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([h, s, v], -1).astype(np.uint8).reshape(180 * 256, 256, 3)
    assert np.array_equal(hsv2bgr_fixed(hsv), cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR))


@pytest.mark.parametrize("img_size", [160, 320, 416, 512, 800, 1024])
def test_load_image_resize_matches_cv2(img_size):
    from icafusion_b200.augment import load_size, resize_fixed
    g = np.random.default_rng(img_size)
    for H0, W0 in ((512, 640), (300, 400), (333, 250)):
        img = g.integers(0, 256, (H0, W0, 3), dtype=np.uint8)
        h, w = load_size(H0, W0, img_size)
        want = img if (h, w) == (H0, W0) else cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(resize_fixed(img, h, w), want)


def test_sampler_draws_like_the_loader():
    """draw_sample consumes random / np.random in __getitem__'s order: the state after a batch is the reference's (golden)."""
    from icafusion_b200.augment import draw_sample
    g, meta, frames, labels = _golden()
    for case in meta["cases"]:
        random.seed(case["seed"])
        np.random.seed(case["seed"])
        for i in case["indices"]:
            draw_sample(i, len(labels), case["img_size"], case["hyp"])
        assert [random.random(), np.random.random()] == list(g[f"{case['name']}_next"]), case["name"]


@pytest.mark.parametrize("name", ["mosaic_r1", "mosaic_resize", "letterbox", "degrees_shear", "flipud"])
def test_restatement_equals_the_reference_loader(name):
    """The numpy restatement of the kernel + the label path == LoadMultiModalImagesAndLabels(augment=True)[i] + collate_fn."""
    from icafusion_b200.augment import Augment
    g, meta, frames, labels = _golden()
    case = next(c for c in meta["cases"] if c["name"] == name)
    aug = Augment(labels, frames.__getitem__, case["img_size"], case["hyp"], device="cpu")
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    rgb, ir, targets = aug.reference(case["indices"])
    img = g[f"{name}_img"]
    assert np.array_equal(rgb, img[:, :3]) and np.array_equal(ir, img[:, 3:])
    assert np.array_equal(targets, g[f"{name}_targets"])


def test_unsupported_settings_raise():
    from icafusion_b200.augment import Augment
    g, meta, frames, labels = _golden()
    hyp = meta["cases"][0]["hyp"]
    for over in (dict(perspective=0.001), dict(mixup=0.2)):
        with pytest.raises(NotImplementedError):
            Augment(labels, frames.__getitem__, 320, dict(hyp, **over), device="cpu")
    with pytest.raises(NotImplementedError):
        Augment(labels, frames.__getitem__, 320, hyp, device="cpu", rect=True)
    with pytest.raises(NotImplementedError):
        Augment(labels, frames.__getitem__, 320, hyp, device="cpu", quad=True)
    seg = [np.zeros((1, 9), np.float32)] + labels[1:]
    with pytest.raises(NotImplementedError):
        Augment(seg, frames.__getitem__, 320, hyp, device="cpu")
