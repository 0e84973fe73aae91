"""Device validation: icaf_match_detections against the real reference's test.py (golden) and the CPU oracle, and the drop-in
icafusion_b200.test.test against the golden, the oracle and ComputeLoss, with no host sync inside its batch loop."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import load_synth
from oracle import synth
from oracle.gen_golden_val import SETTINGS, StubDetector, _batch, _image, checked_inputs, labels_list_for, loader
from oracle.val_match import match_batch

pytestmark = pytest.mark.gpu

SCALED = [((590, 758), ((0.85, 0.85), (13.7, 21.3))), ((512, 640), ((1.0, 1.0), (16.0, 16.0))),
          ((480, 600), ((1.1, 1.1), (5.9, 8.1))), ((600, 770), ((0.84375, 0.84375), (11.25, 18.875)))]


def _device_match(z16, tg, shapes, iouv, single_cls, dev, conf=0.001, iou=0.5, max_det=300, H=544, W=672):
    from icafusion_b200 import ops
    from icafusion_b200.test import ratio_pad_rows
    z = torch.from_numpy(z16).to(dev)
    det, count = ops.nms(z, conf, iou, agnostic=single_cls, multi_label=True, max_det=max_det)
    native = torch.full((z.shape[0], max_det, 4), 7.0, device=dev)
    correct = torch.full((z.shape[0], max_det, iouv.numel()), 9, dtype=torch.uint8, device=dev)
    ops.match_detections(det, count, torch.from_numpy(tg).to(dev), ratio_pad_rows(shapes).to(dev), H, W, iouv.to(dev),
                         single_cls, correct=correct, native=native)
    torch.cuda.synchronize()
    return det.cpu(), count.cpu().tolist(), correct.cpu(), native.cpu()


def _check_vs_oracle(det, count, correct, native, tg, shapes, iouv, single_cls, where, H=544, W=672):
    dets = [det[b, :n] for b, n in enumerate(count)]
    for b, (c_ref, _, nat_ref) in enumerate(match_batch(dets, torch.from_numpy(tg), H, W, shapes, iouv, single_cls)):
        n = count[b]
        assert torch.equal(correct[b, :n].bool(), c_ref), (where, b)
        assert torch.equal(native[b, :n], nat_ref), (where, b)
        assert not correct[b, n:].any() and not native[b, n:].any(), (where, b)


def test_kernel_matches_reference_golden_bit_exact(cuda_device):
    meta, d = load_golden("val_cases")
    inputs = checked_inputs(meta)
    iouv = torch.from_numpy(d["iouv"])
    same = torch.equal(torch.linspace(0.5, 0.95, 10, device=cuda_device).cpu(), iouv)
    print(f"CUDA torch.linspace(0.5, 0.95, 10) equals the CPU one test.py uses: {same}")
    for name, st in meta["settings"].items():
        rows, conf, pcls = [], [], []
        for z16, tg, shapes, _ in inputs[st["dataset"]]:
            det, count, correct, _ = _device_match(z16, tg, shapes, iouv, st["single_cls"], cuda_device)
            for b, n in enumerate(count):
                rows.append(correct[b, :n].numpy().astype(bool))
                conf.append(det[b, :n, 4].numpy())
                pcls.append(np.zeros(n, np.float32) if st["single_cls"] else det[b, :n, 5].numpy())
        assert np.array_equal(np.concatenate(rows), d[f"{name}_tp"]), name
        assert np.array_equal(np.concatenate(conf), d[f"{name}_conf"]), name
        assert np.array_equal(np.concatenate(pcls), d[f"{name}_pcls"]), name


def test_dropin_with_stub_detector_matches_reference_golden(cuda_device, tmp_path):
    from icafusion_b200 import test as T
    meta, d = load_golden("val_cases")
    inputs = checked_inputs(meta)
    for name, st in meta["settings"].items():
        batches = inputs[st["dataset"]]
        stub = StubDetector([b[0] for b in batches], st["nc"]).to(cuda_device)
        labels_list = labels_list_for(batches) if st["save_txt"] else None
        res, maps, mr, t = T.test({"nc": st["nc"], "names": stub.names}, model=stub, dataloader=loader(batches, pin=True),
                                  save_dir=tmp_path / name, save_txt=st["save_txt"], single_cls=st["single_cls"],
                                  labels_list=labels_list, verbose=True)
        assert [float(x) for x in res] == st["results"], name
        assert np.array_equal(maps, d[f"{name}_maps"]), name
        assert mr == st["mr"] == [0.0] * 10 and len(t) == 6
        if st["save_txt"]:
            txt = (tmp_path / name / "labels" / "pred" / "result.txt").read_bytes()
            assert txt == d[f"{name}_result_txt"].tobytes(), name


@pytest.mark.parametrize("case", ["b32", "labels2000", "max_det1000", "single_cls_scaled"])
def test_kernel_matches_oracle_on_larger_cases(cuda_device, case):
    iouv = torch.linspace(0.5, 0.95, 10)
    g = np.random.Generator(np.random.PCG64({"b32": 1, "labels2000": 2, "max_det1000": 3, "single_cls_scaled": 4}[case]))
    max_det, single_cls, shapes = 300, False, [((512, 640), ((1.0, 1.0), (16.0, 16.0)))] * 32
    if case == "b32":                             # test.py's batch: B = 32 at 544 x 672, nc = 3, conf 0.001 / iou 0.6
        z16, tg = _batch(g, 3, 32, 256)
    elif case in ("labels2000", "max_det1000"):   # one image with 2 000 labels (targets unsorted), two ordinary ones
        parts = [_image(g, 3, n) for n in (2000, 6, 6)]
        z = np.zeros((3, max(r.shape[0] for _, r in parts), 8), np.float32)
        tg = []
        for i, (lab, rows) in enumerate(parts):
            z[i, :rows.shape[0]] = rows
            tg.append(np.concatenate([np.full((lab.shape[0], 1), i), lab], 1))
        tg = np.concatenate(tg).astype(np.float32)
        tg = tg[g.permutation(tg.shape[0])]
        z16 = z.astype(np.float16)
        max_det = 1000 if case == "max_det1000" else 300
        shapes = SCALED[:3]
    else:
        z16, tg = _batch(g, 3, 4, 256, special=True)
        tg[:, 1] = 0
        single_cls, shapes = True, SCALED
    B = z16.shape[0]
    det, count, correct, native = _device_match(z16, tg, shapes[:B], iouv, single_cls, cuda_device, iou=0.6, max_det=max_det)
    if case == "max_det1000":
        assert count[0] == 1000
    if case == "labels2000":
        assert (tg[:, 0] == 0).sum() >= 2000
    _check_vs_oracle(det, count, correct, native, tg, shapes[:B], iouv, single_cls, case)
    assert correct[..., 0].sum() > 0


class _PinnedLoader:
    """Pinned batches; from the second batch on, any synchronising call in the consumer's loop body raises."""

    def __init__(self, batches):
        self.batches = batches

    def __len__(self):
        return len(self.batches)

    def __iter__(self):
        try:
            for i, b in enumerate(self.batches):
                torch.cuda.set_sync_debug_mode("error" if i else 0)
                yield b
        finally:
            torch.cuda.set_sync_debug_mode(0)


def test_dropin_on_flir_detector_vs_oracle_and_loss(cuda_device, tmp_path):
    """yolov5n FLIR (synthetic weights) through test.test at 544 x 672, B = 2, three batches, with compute_loss: the metrics
    equal the oracle's matching and metrics on the device's own NMS rows, the loss equals ComputeLoss called directly, and
    the batch loop makes no synchronising call after the first batch."""
    from icafusion_b200 import Model, ops
    from icafusion_b200 import test as T
    from icafusion_b200.loss import ComputeLoss
    model = Model("yolov5n_Transfusion_FLIR").eval()
    load_synth(model, 21)
    model = model.fuse().to(cuda_device)
    model.hyp = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    model.gr = 1.0
    g = np.random.Generator(np.random.PCG64(5))
    batches = []
    for k in range(3):
        rgb, ir = synth.synth_images(2, 544, 672, 40 + k)
        img = (torch.cat([rgb, ir], 1) * 255).to(torch.uint8)
        lab = [np.concatenate([np.full((5, 1), i), _image(g, 3, 5)[0]], 1) for i in range(2)]
        tg = torch.from_numpy(np.concatenate(lab).astype(np.float32))
        shapes = [((512, 640), ((1.0, 1.0), (16.0, 16.0))), SCALED[0]]
        batches.append((img.pin_memory(), tg.pin_memory(), [f"/d/a{k}_{i}.jpg" for i in range(2)], shapes))
    compute_loss = ComputeLoss(model)
    res, maps, _, _ = T.test({"nc": 3, "names": ["p", "c", "b"]}, model=model, dataloader=_PinnedLoader(batches),
                             save_dir=tmp_path, compute_loss=compute_loss)
    iouv = torch.linspace(0.5, 0.95, 10)
    stats, seen, loss = [], 0, torch.zeros(4, device=cuda_device)
    with torch.no_grad():
        for img, tg, _, shapes in batches:
            img = img.to(cuda_device)
            z, _, train_out = model(img[:, :3], img[:, 3:])
            loss += compute_loss([x.float() for x in train_out], tg.to(cuda_device))[1][:4]
            det, count = ops.nms(z, 0.001, 0.5, multi_label=True)
            dets = [det[b, :n].cpu() for b, n in enumerate(count.tolist())]
            for b, (c, pred, _) in enumerate(match_batch(dets, tg, 544, 672, shapes, iouv)):
                seen += 1
                tcls = tg[tg[:, 0] == b, 1].tolist()
                if pred.shape[0]:
                    stats.append((c.numpy(), pred[:, 4].numpy(), pred[:, 5].numpy(), tcls))
                elif tcls:
                    stats.append((np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls))
    want, want_maps = T.summarise(stats, 3, {0: "p", 1: "c", 2: "b"}, seen)
    assert [float(x) for x in res[:8]] == [float(x) for x in want]
    assert np.array_equal(maps, want_maps)
    assert [float(x) for x in res[8:]] == (loss.cpu() / len(batches)).tolist()
