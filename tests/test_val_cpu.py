"""Validation without a GPU: the CPU oracle of test.py's matching (oracle.val_match) with the oracle NMS and the host-side
metrics (icafusion_b200.metrics, icafusion_b200.test's summary and save_txt writers) reproduce the real reference's
test.test on every golden case exactly; test.test refuses what is not built; icaf_match_detections rejects bad arguments
before any CUDA call."""
import ctypes
from pathlib import Path

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import icaf_oracle as O
from oracle.gen_golden_val import SETTINGS, StubDetector, checked_inputs, labels_list_for
from oracle.nms_multilabel import non_max_suppression_multilabel
from oracle.val_match import match_batch


def _oracle_validation(batches, iouv, single_cls, labels_dir=None, labels_list=None):
    """test.py's per-image loop on the CPU oracles -> (stats list, images seen)."""
    from icafusion_b200 import test as T
    stats, seen = [], 0
    for z16, tg, shapes, paths in batches:
        z = torch.from_numpy(z16).float()
        nms = non_max_suppression_multilabel if z.shape[2] > 6 else O.non_max_suppression
        dets = nms(z, 0.001, 0.5, agnostic=single_cls)
        for si, (correct, pred, native) in enumerate(match_batch(dets, torch.from_numpy(tg), 544, 672, shapes, iouv, single_cls)):
            seen += 1
            tcls = [float(c) for c in tg[tg[:, 0] == si, 1]]
            if not pred.shape[0]:
                if tcls:
                    stats.append((np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls))
                continue
            if labels_dir is not None:
                stem = Path(paths[si]).stem
                T.append_txt(labels_dir, stem, labels_list.index(stem + ".txt"), native.numpy(), pred[:, 4].numpy())
            stats.append((correct.numpy(), pred[:, 4].numpy(), pred[:, 5].numpy(), tcls))
    return stats, seen


@pytest.mark.parametrize("name", list(SETTINGS))
def test_oracles_reproduce_reference_validation(name, tmp_path):
    from icafusion_b200 import test as T
    meta, d = load_golden("val_cases")
    inputs = checked_inputs(meta)
    st = meta["settings"][name]
    iouv = torch.from_numpy(d["iouv"])
    assert torch.equal(iouv, torch.linspace(0.5, 0.95, 10))
    batches = inputs[st["dataset"]]
    labels_dir = labels_list = None
    if st["save_txt"]:
        labels_dir, labels_list = tmp_path / "pred", labels_list_for(batches)
        labels_dir.mkdir()
    stats, seen = _oracle_validation(batches, iouv, st["single_cls"], labels_dir, labels_list)
    cat = [np.concatenate(x, 0) for x in zip(*stats)]
    for k, a in zip(("tp", "conf", "pcls", "tcls"), cat):
        want = d[f"{name}_{k}"]
        assert a.dtype == want.dtype and np.array_equal(a, want), (name, k)
    nc = 1 if st["single_cls"] else st["nc"]
    results, maps = T.summarise(stats, nc, {i: f"c{i}" for i in range(nc)}, seen, verbose=True)
    assert [float(x) for x in results] + [0.0] * 4 == st["results"], name
    assert np.array_equal(maps, d[f"{name}_maps"]), name
    if st["save_txt"]:
        T.write_result_txt(labels_dir)
        assert (labels_dir / "result.txt").read_bytes() == d[f"{name}_result_txt"].tobytes()


def test_golden_covers_the_matching_cases():
    """The golden exercises what the matching must get right: false positives next to true positives at every setting,
    IoUs between the thresholds (rows correct at 0.5 but not at 0.95), and images without predictions."""
    meta, d = load_golden("val_cases")
    for name in SETTINGS:
        tp = d[f"{name}_tp"]
        assert 0 < tp[:, 0].sum() < tp.shape[0], name
        assert (tp[:, 0] & ~tp[:, -1]).any(), name
    assert meta["settings"]["flir"]["n_labels"] > meta["settings"]["flir"]["tp50"]


def test_test_refuses_what_is_not_built(tmp_path):
    from icafusion_b200 import test as T
    stub = StubDetector([np.zeros((1, 4, 8), np.float16)], 3)
    data = {"nc": 3, "names": ["a", "b", "c"]}
    with pytest.raises(NotImplementedError, match="command-line"):
        T.test(data, weights="best.pt", save_dir=tmp_path)
    with pytest.raises(NotImplementedError, match="pycocotools"):
        T.test(data, model=stub, dataloader=[], save_json=True, save_dir=tmp_path)
    with pytest.raises(NotImplementedError, match="save_hybrid"):
        T.test(data, model=stub, dataloader=[], save_hybrid=True, save_dir=tmp_path)
    with pytest.raises(NotImplementedError, match="augmented"):
        T.test(data, model=stub, dataloader=[], augment=True, save_dir=tmp_path)
    with pytest.raises(RuntimeError, match="CUDA"):
        T.test(data, model=stub, dataloader=[], save_dir=tmp_path)


def test_match_detections_rejects_bad_arguments_without_a_gpu():
    from icafusion_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(16)                    # never dereferenced: validation fails first
    assert L.icaf_match_detections_workspace_bytes(100) == 400 and L.icaf_match_detections_workspace_bytes(-1) == 0
    good = dict(det=one, count=one, B=2, max_det=300, targets=one, T=10, ratio_pad=one, height=544, width=672, iouv=one,
                niou=10, single_cls=0, correct=one, native=None, ws=one, ws_bytes=40)

    def call(**kw):
        a = dict(good, **kw)
        return L.icaf_match_detections(a["det"], a["count"], a["B"], a["max_det"], a["targets"], a["T"], a["ratio_pad"],
                                       a["height"], a["width"], a["iouv"], a["niou"], a["single_cls"], a["correct"],
                                       a["native"], a["ws"], a["ws_bytes"], None)
    n0 = L.icaf_kernel_launches()
    for bad in (dict(det=None), dict(count=None), dict(ratio_pad=None), dict(iouv=None), dict(correct=None),
                dict(targets=None), dict(ws=None), dict(B=0), dict(max_det=0), dict(T=-1), dict(niou=0), dict(niou=33),
                dict(height=0), dict(width=-4), dict(ws_bytes=39), dict(native=ctypes.c_void_p(24))):
        assert call(**bad) == 1, bad
        assert L.icaf_last_error()
    assert b"workspace" in (call(ws_bytes=39) and L.icaf_last_error())
    assert L.icaf_kernel_launches() == n0
