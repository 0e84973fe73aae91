"""Device validation loader (icaf_val_stage via icafusion_b200.valdata.ValBatches): its batches equal the reference's
testloader (tests/golden/val_loader_cases.npz, which keeps the images' SHA-256) byte for byte, with frames on the host and
on the device; test.test fed by ValBatches returns what it returns fed the reference's batches; at the dataset sizes
(KAIST / FLIR 512 x 640, LLVIP 1024 x 1280, VEDAI 1024 x 1024 at 640) the kernel equals the numpy restatement at batch 8."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from helpers import load_synth

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "val_loader_cases.npz")


def _golden():
    g = np.load(GOLDEN)
    meta = json.loads(bytes(g["meta"]).decode())
    n = meta["frames"]
    return g, meta, {k: (g[f"rgb{k}"], g[f"ir{k}"]) for k in range(n)}, [g[f"labels{k}"] for k in range(n)]


def _loader(meta, frames, labels, case, dev):
    from icafusion_b200.valdata import ValBatches
    hw0 = [tuple(frames[k][0].shape[:2]) for k in range(meta["frames"])]
    return ValBatches(labels, frames.__getitem__, hw0, meta["img_size"], case["batch_size"], meta["stride"], meta["pad"],
                      case["single_cls"], paths=meta["paths"], device=dev)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _golden_batches(g, meta, frames, labels, case):
    """The reference loader's batches: images rebuilt by the numpy restatement and checked against the golden's SHA-256,
    targets, paths and shapes as stored."""
    vb = _loader(meta, frames, labels, case, "meta")
    out = []
    for i, b in enumerate(case["batches"]):
        img = torch.from_numpy(vb.reference(i))
        assert _sha(img.numpy()) == b["img_sha256"], i
        shapes = tuple(((h0, w0), ((r0, r1), (p0, p1))) for (h0, w0), ((r0, r1), (p0, p1)) in b["shapes"])
        out.append((img, torch.from_numpy(g[f"{case['name']}_targets{i}"]), tuple(b["paths"]), shapes))
    return out


@pytest.mark.parametrize("frames_on", ["host", "device"])
@pytest.mark.parametrize("name", ["b1", "b4", "b4_single_cls"])
def test_device_batches_equal_the_reference_loader(cuda_device, name, frames_on):
    g, meta, frames, labels = _golden()
    if frames_on == "device":
        frames = {k: tuple(torch.from_numpy(f).to(cuda_device) for f in v) for k, v in frames.items()}
    case = next(c for c in meta["cases"] if c["name"] == name)
    got = list(_loader(meta, frames, labels, case, cuda_device))
    torch.cuda.synchronize()
    assert len(got) == len(case["batches"])
    for i, ((img, targets, paths, shapes), b) in enumerate(zip(got, case["batches"])):
        assert img.is_cuda and img.dtype == torch.uint8 and list(img.shape) == b["img_shape"]
        assert _sha(img.cpu().numpy()) == b["img_sha256"], i
        assert np.array_equal(targets.numpy(), g[f"{name}_targets{i}"]) and list(paths) == b["paths"]
        assert [[list(hw), [list(r), list(p)]] for hw, (r, p) in shapes] == b["shapes"]


@pytest.mark.parametrize("name", ["b4", "b4_single_cls"])
def test_dropin_test_fed_by_val_batches_equals_the_reference_batches(cuda_device, tmp_path, name):
    """yolov5n FLIR (synthetic weights) through test.test with save_txt: results, maps and result.txt are identical whether
    the batches come from ValBatches or are the reference loader's own (a plain list).  The P5 fusion block pools to 8 x 8
    tokens instead of 10 x 10, so the 288 x 352 batch (a 9 x 11 P5 map) is admitted."""
    from icafusion_b200 import Model
    from icafusion_b200 import test as T
    from icafusion_b200.cfg import load_cfg
    g, meta, frames, labels = _golden()
    case = next(c for c in meta["cases"] if c["name"] == name)
    cfg = load_cfg("yolov5n_Transfusion_FLIR")
    p5 = next(r for r in cfg["backbone"] if r[2] == "TransformerFusionBlock" and r[3][1] == 10)
    p5[3] = [p5[3][0], 8, 8]
    model = Model(cfg).eval()
    load_synth(model, 23)
    model = model.fuse().to(cuda_device)
    labels_list = [f"{k:03d}.txt" for k in range(meta["frames"])]
    runs = []
    for src, loader in (("golden", _golden_batches(g, meta, frames, labels, case)), ("device", _loader(meta, frames, labels, case, cuda_device))):
        res, maps, mr, _ = T.test({"nc": 3, "names": ["p", "c", "b"]}, model=model, dataloader=loader,
                                  save_dir=tmp_path / src, save_txt=True, single_cls=case["single_cls"],
                                  labels_list=labels_list)
        runs.append(([float(x) for x in res], maps, mr, (tmp_path / src / "labels" / "pred" / "result.txt").read_bytes()))
    (r0, m0, mr0, t0), (r1, m1, mr1, t1) = runs
    assert r0 == r1 and np.array_equal(m0, m1) and mr0 == mr1 and t0 == t1
    assert len(t0) > 0


def _dataset(sizes, seed=5):
    g = np.random.default_rng(seed)
    frames, labels = {}, []
    for k, (h, w) in enumerate(sizes):
        yy, xx = np.mgrid[0:h, 0:w]
        base = (xx * (k + 3) // 7 + yy * (k + 5) // 9) % 256
        rgb = np.stack([(base + 60 * c + g.integers(0, 24, (h, w))) % 256 for c in range(3)], -1).astype(np.uint8)
        ir = np.repeat(((base // 2 + g.integers(0, 16, (h, w))) % 256)[..., None], 3, -1).astype(np.uint8)
        frames[k] = (rgb, ir)
        nb = int(g.integers(0, 6))
        wh = g.uniform(0.02, 0.4, (nb, 2))
        labels.append(np.concatenate([g.integers(0, 2, (nb, 1)), g.uniform(wh / 2, 1 - wh / 2), wh], 1).astype(np.float32))
    return frames, labels


@pytest.mark.parametrize("img_size,sizes", [
    (640, [(512, 640)] * 6 + [(1024, 1280)] * 5 + [(1024, 1024)] * 5),      # copy, 2x2 fast area, fractional area (1.6)
    (320, [(960, 1280), (768, 960), (96, 1280), (333, 1000), (200, 256), (257, 250), (77, 91), (300, 330)]),
])
def test_batch8_equals_the_restatement(cuda_device, img_size, sizes):
    from icafusion_b200.valdata import ValBatches
    frames, labels = _dataset(sizes)
    vb = ValBatches(labels, frames.__getitem__, [s for s in sizes], img_size, batch_size=8, device=cuda_device)
    for j, (img, _, _, _) in enumerate(vb):
        torch.cuda.synchronize()
        assert np.array_equal(img.cpu().numpy(), vb.reference(j)), j
