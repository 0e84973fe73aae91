"""Host half of the device validation loader (icafusion_b200/valdata.py): the rect order, batch shapes, targets, shapes
tuples and paths equal what the reference's testloader yielded (tests/golden/val_loader_cases.npz, from
create_dataloader_rgb_ir(rect=True, pad=0.5) + collate_fn), the numpy restatement of the kernel equals its images byte for
byte (the golden keeps their SHA-256) and cv2.resize on every staging path, and bad arguments are refused on the host."""
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_conv_ptxas_cpu import _nvcc

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(ROOT, "tests", "golden", "val_loader_cases.npz")


def _golden():
    g = np.load(GOLDEN)
    meta = json.loads(bytes(g["meta"]).decode())
    n = meta["frames"]
    frames = {k: (g[f"rgb{k}"], g[f"ir{k}"]) for k in range(n)}
    labels = [g[f"labels{k}"] for k in range(n)]
    return g, meta, frames, labels


def _loader(meta, frames, labels, case, **kw):
    from icafusion_b200.valdata import ValBatches
    hw0 = [frames[k][0].shape[:2] for k in range(meta["frames"])]
    return ValBatches(labels, frames.__getitem__, hw0, meta["img_size"], case["batch_size"], meta["stride"], meta["pad"],
                      case["single_cls"], paths=meta["paths"], device="meta", **kw)


@pytest.mark.parametrize("name", ["b1", "b4", "b4_single_cls"])
def test_batches_equal_the_reference_loader(name):
    """Order, batch shapes, targets, shapes tuples and paths exactly; the images through the numpy restatement byte for byte;
    one icaf_val_stage call per batch with the batch's shape."""
    from icafusion_b200 import ops
    g, meta, frames, labels = _golden()
    case = next(c for c in meta["cases"] if c["name"] == name)
    vb = _loader(meta, frames, labels, case)
    assert len(vb) == len(case["batches"])
    with ops.dry_run() as d:
        got = list(vb)
    assert [r[0] for r in d.records] == ["icaf_val_stage"] * len(vb)
    for i, ((img, targets, paths, shapes), want) in enumerate(zip(got, case["batches"])):
        shape = tuple(want["img_shape"])
        assert tuple(img.shape) == shape and img.dtype == torch.uint8
        assert d.records[i][1][2:5] == (shape[0], shape[2], shape[3])
        assert targets.dtype == torch.float32 and np.array_equal(targets.numpy(), g[f"{name}_targets{i}"])
        assert list(paths) == want["paths"]
        assert [[list(hw), [list(r), list(p)]] for hw, (r, p) in shapes] == want["shapes"]
        ref = vb.reference(i)
        assert ref.shape == shape and hashlib.sha256(ref.tobytes()).hexdigest() == want["img_sha256"]


def test_restatement_matches_cv2_on_every_path():
    """load_resize == cv2.resize with load_image's interpolation: copy, INTER_LINEAR up, INTER_AREA's 2x2 / other integer
    fast paths (equal and unequal scales) and its fractional path (equal and unequal scales, one axis integer)."""
    from icafusion_b200.augment import load_size
    from icafusion_b200.valdata import MODE_AREA, MODE_AREA_FAST, MODE_COPY, MODE_LINEAR, load_resize, stage_mode
    rng = np.random.default_rng(4)
    seen = set()
    for (h0, w0, s) in [(512, 640, 640), (512, 640, 320), (1024, 1280, 640), (768, 960, 320), (96, 1280, 320),
                        (6, 200, 100), (400, 500, 320), (333, 1000, 500), (300, 330, 320), (480, 360, 320),
                        (200, 256, 320), (257, 250, 320), (77, 91, 59), (1024, 1024, 640), (37, 641, 640)]:
        img = rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
        img[h0 // 3:h0 // 2] = (img[h0 // 3:h0 // 2] // 4) * 4 + 2          # rows whose 2 x 2 sums tie at .5
        h, w = load_size(h0, w0, s)
        r = s / max(h0, w0)
        want = img if (h, w) == (h0, w0) else cv2.resize(
            img, (w, h), interpolation=cv2.INTER_AREA if r < 1 else cv2.INTER_LINEAR)
        mode, sx, sy = stage_mode(h0, w0, h, w)
        seen.add((mode, sx == sy == 2))
        assert np.array_equal(load_resize(img, h, w), want), (h0, w0, s, mode, sx, sy)
    assert {m for m, _ in seen} == {MODE_COPY, MODE_LINEAR, MODE_AREA_FAST, MODE_AREA}
    assert (MODE_AREA_FAST, True) in seen and (MODE_AREA_FAST, False) in seen


def test_area_fast_needs_both_scales_integer():
    """cv2 takes resizeAreaFast only when both scales are integers; one integer axis takes the fractional tables."""
    from icafusion_b200.valdata import MODE_AREA, MODE_AREA_FAST, stage_mode
    assert stage_mode(512, 640, 256, 320) == (MODE_AREA_FAST, 2, 2)
    assert stage_mode(6, 200, 2, 100) == (MODE_AREA_FAST, 2, 3)
    assert stage_mode(333, 1000, 166, 500)[0] == MODE_AREA          # x scale 2, y scale 2.006
    assert stage_mode(300, 330, 290, 320)[0] == MODE_AREA           # x 1.03125, y 1.0345


def test_bad_arguments_are_refused_on_the_host():
    from icafusion_b200 import _lib, ops
    from icafusion_b200.valdata import ValBatches
    g, meta, frames, labels = _golden()
    case = {"batch_size": 1, "single_cls": False}
    hw0 = [frames[k][0].shape[:2] for k in range(meta["frames"])]
    with pytest.raises(ValueError):
        ValBatches(labels, frames.__getitem__, hw0[:-1], 320, device="meta")              # one hw0 row short
    with pytest.raises(NotImplementedError):
        ValBatches(labels, frames.__getitem__, hw0, 320, pad=-1.0, device="meta")         # letterbox would resize again
    with pytest.raises(NotImplementedError):
        ValBatches([np.zeros((2, 9), np.float32)] + labels[1:], frames.__getitem__, hw0, 320, device="meta")
    bad = [
        lambda f: (f[0], f[1][:-2]),                                   # RGB and IR differ in size
        lambda f: (f[0][..., :2], f[1][..., :2]),                      # two channels
        lambda f: (f[0].astype(np.float32), f[1].astype(np.float32)),  # not uint8
        lambda f: (f[0][:-4], f[1][:-4]),                              # not the size hw0 gives
    ]
    for make in bad:
        fr = dict(frames)
        vb = _loader(meta, fr, labels, case)
        j = next(j for j in range(len(vb)) if int(vb.order[j]) == 0)
        fr[0] = make(frames[0])
        with ops.dry_run(), pytest.raises(ValueError):
            vb.batch(j)
    L = _lib.lib()
    assert L.icaf_val_stage_params_bytes(0, 0) == 0 and L.icaf_val_stage_params_bytes(2, 6) == 0
    need = L.icaf_val_stage_params_bytes(2, 8)
    assert need == 2 * 64 + 32
    n0 = L.icaf_kernel_launches()
    fake = 1 << 20                                                     # never dereferenced: refused before any launch
    assert L.icaf_val_stage(fake, need - 1, 2, 288, 352, 8, fake, None) == 1
    assert b"params_bytes" in L.icaf_last_error()
    assert L.icaf_val_stage(fake, need, 2, 288, 350, 8, fake, None) == 1      # W % 4 != 0
    assert L.icaf_val_stage(fake + 4, need, 2, 288, 352, 8, fake, None) == 1  # misaligned block
    assert L.icaf_val_stage(None, need, 2, 288, 352, 8, fake, None) == 1
    assert L.icaf_kernel_launches() == n0


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_val_stage_kernel_spill_free(tmp_path):
    """ptxas report of image.cu: val_stage_kernel spills nothing."""
    from icafusion_b200 import build as B
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "image.cu"), "-o", str(tmp_path / "image.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = (out.stdout + out.stderr).splitlines()
    at = next(i for i, l in enumerate(log) if re.search(r"Compiling entry function '\w*val_stage_kernel\w*'", l))
    spill = next(re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l) for l in log[at:] if "spill" in l)
    assert spill.groups() == ("0", "0"), log[at:at + 4]
