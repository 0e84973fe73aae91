"""Device multi-label NMS (icaf_nms_multi_label, test.py's non_max_suppression(..., multi_label=True)) against golden rows
from the real reference and against the CPU oracle: the golden settings, a FLIR detector's own output, the nc == 1
identity, a captured GraphedDetector and one full-size test.py batch."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import load_synth
from oracle.gen_golden_nms_multilabel import checked_inputs
from oracle.nms_multilabel import non_max_suppression_multilabel as oracle_nms
from oracle import synth

pytestmark = pytest.mark.gpu


def _assert_equal_oracle(det, count, ref, where, images=None):
    torch.cuda.synchronize()
    cnt = count.tolist()
    for b in (range(len(ref)) if images is None else images):
        r = ref[b] if images is None else ref[images.index(b)]
        assert cnt[b] == r.shape[0], (where, b, cnt[b], r.shape[0])
        assert np.array_equal(det[b, :cnt[b]].cpu().numpy(), r.numpy()), (where, b)


def test_multilabel_matches_reference_golden_bit_exact(cuda_device):
    from icafusion_b200 import ops
    from icafusion_b200.general import non_max_suppression
    m, d = load_golden("nms_multilabel_cases")
    inputs = checked_inputs(m)
    for inp in m["inputs"]:
        pred = torch.from_numpy(inputs[inp["name"]]).to(cuda_device)
        for st in inp["settings"]:
            where = (inp["name"], st["name"])
            det, count = ops.nms(pred, st["conf"], st["iou"], st["agnostic"], st["classes"], multi_label=True)
            torch.cuda.synchronize()
            assert count.tolist() == st["counts"], (where, count.tolist())
            lst = non_max_suppression(pred, st["conf"], st["iou"], classes=st["classes"], agnostic=st["agnostic"],
                                      multi_label=True)
            for b, n in enumerate(st["counts"]):
                want = d[f"{inp['name']}_{st['name']}_{b}"]
                assert np.array_equal(det[b, :n].cpu().numpy(), want), (where, b)
                assert np.array_equal(lst[b].cpu().numpy(), want), (where, b)


def _flir_detector(cuda_device, size="n", seed=9):
    from icafusion_b200 import Model
    model = Model(f"yolov5{size}_Transfusion_FLIR").eval()
    load_synth(model, seed)
    return model.fuse().to(cuda_device)


def test_multilabel_on_flir_detector_output_vs_oracle(cuda_device):
    """A FLIR detector (nc = 3) at B = 4, 512 x 640: its own decoded predictions through the device multi-label NMS equal
    the oracle's, at test.py's setting (every row x class pair is a candidate: cut at max_nms) and at detect's."""
    from icafusion_b200 import ops
    model = _flir_detector(cuda_device)
    rgb, ir = synth.synth_images(4, 512, 640, 9)
    with torch.no_grad():
        z = model(rgb.to(cuda_device), ir.to(cuda_device))[0]
    assert z.shape == (4, 20160, 8)
    for conf, iou in ((0.001, 0.6), (0.25, 0.45)):
        det, count = ops.nms(z, conf, iou, multi_label=True)
        _assert_equal_oracle(det, count, oracle_nms(z.cpu(), conf, iou), (conf, iou))


def test_multilabel_is_best_class_when_single_class(cuda_device):
    """KAIST (nc = 1): multi_label=True returns exactly what the best-class call returns (general.py:535)."""
    from icafusion_b200 import Model, ops
    from icafusion_b200.general import non_max_suppression
    model = Model("yolov5s_Transfusion_kaist").eval()
    load_synth(model, 4)
    model = model.fuse().to(cuda_device)
    rgb, ir = synth.synth_images(2, 320, 320, 4)
    with torch.no_grad():
        z = model(rgb.to(cuda_device), ir.to(cuda_device))[0]
    for conf, iou in ((0.001, 0.6), (0.25, 0.45)):
        d0, c0 = ops.nms(z, conf, iou)
        d1, c1 = ops.nms(z, conf, iou, multi_label=True)
        torch.cuda.synchronize()
        assert torch.equal(c0, c1) and torch.equal(d0, d1)
        l0 = non_max_suppression(z, conf, iou)
        l1 = non_max_suppression(z, conf, iou, multi_label=True)
        assert all(torch.equal(a, b) for a, b in zip(l0, l1))


def test_graphed_detector_with_captured_multilabel_nms(cuda_device):
    """GraphedDetector(nms=dict(..., multi_label=True)) captures the multi-label path; two replays on different inputs each
    equal the oracle's multi-label NMS of that replay's own z."""
    from icafusion_b200.engine import GraphedDetector
    model = _flir_detector(cuda_device, seed=5).half()
    eng = GraphedDetector(model, 2, 320, 320, in_dtype=torch.uint8, device=cuda_device,
                          nms=dict(conf_thres=0.001, iou_thres=0.6, multi_label=True))
    dets = []
    for sd in (31, 32):
        a, b = synth.synth_images(2, 320, 320, sd)
        a, b = (a * 255).to(torch.uint8).pin_memory(), (b * 255).to(torch.uint8).pin_memory()
        det, count = eng.infer_detections(a, b)
        ref = oracle_nms(eng.z.cpu(), 0.001, 0.6)
        assert count.tolist() == [int(r.shape[0]) for r in ref]
        for i, r in enumerate(ref):
            assert np.array_equal(det[i, :r.shape[0]].numpy(), r.numpy()), (sd, i)
        dets.append(det.clone())
    assert not torch.equal(dets[0], dets[1])


def test_multilabel_full_size_test_batch(cuda_device):
    """test.py's batch at its rect shape: B = 32 x 22 491 rows (544 x 672) x nc 3 at conf 0.001 / iou 0.6 -- 67 473
    candidates per image, cut at 30 000 -- equals the oracle on the first and the last image."""
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(7)
    B, R = 32, 22491
    z = torch.empty(B, R, 8)
    z[..., 0] = torch.rand(B, R, generator=g) * 672
    z[..., 1] = torch.rand(B, R, generator=g) * 544
    z[..., 2:4] = torch.rand(B, R, 2, generator=g) * 120 + 4
    z[..., 4:] = torch.rand(B, R, 4, generator=g) * 0.9 + 0.05
    z = z.half()
    det, count = ops.nms(z.to(cuda_device), 0.001, 0.6, multi_label=True)
    images = [0, B - 1]
    ref = oracle_nms(z[images], 0.001, 0.6)
    _assert_equal_oracle(det, count, ref, "B32", images)
    assert min(count.tolist()) == 300
