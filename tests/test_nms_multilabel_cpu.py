"""Multi-label NMS without a GPU: the oracle's multi-label branch reproduces the real reference's rows
(tests/golden/nms_multilabel_cases.npz from oracle/gen_golden_nms_multilabel.py), and icaf_nms_multi_label is declared,
exported and rejects bad arguments on the host before any launch."""
import ctypes

import numpy as np
import torch

from conftest import load_golden
from oracle.gen_golden_nms_multilabel import checked_inputs
from oracle.nms_multilabel import non_max_suppression_multilabel


def test_multilabel_oracle_matches_reference_golden():
    m, d = load_golden("nms_multilabel_cases")
    inputs = checked_inputs(m)
    cut = 0
    for inp in m["inputs"]:
        pred = torch.from_numpy(inputs[inp["name"]])
        assert pred.shape[2] - 5 == inp["nc"]
        for st in inp["settings"]:
            out = non_max_suppression_multilabel(pred, st["conf"], st["iou"], classes=st["classes"], agnostic=st["agnostic"])
            for b, o in enumerate(out):
                want = d[f"{inp['name']}_{st['name']}_{b}"]
                assert o.shape[0] == st["counts"][b] == want.shape[0], (inp["name"], st["name"], b)
                assert np.array_equal(o.numpy(), want), (inp["name"], st["name"], b)
            cut += sum(n > 30000 for n in st["candidates"])
    assert {i["nc"] for i in m["inputs"]} == {3, 9} and cut >= 2      # both class counts, and cases above max_nms


def test_multilabel_entry_is_declared_and_exported():
    from test_abi_cpu import _header_symbols
    from icafusion_b200 import _lib
    for s in ("icaf_nms_multi_label", "icaf_nms_multi_label_workspace_bytes"):
        assert s in _header_symbols() and s in _lib.SIGNATURES and hasattr(_lib.lib(), s)


def test_multilabel_entry_validates_arguments_without_a_gpu():
    from icafusion_b200 import _lib, ops
    L = _lib.lib()
    one = ctypes.c_void_p(16)                     # non-null, never dereferenced: validation fails first
    B, R, no = 2, 1000, 8
    need = L.icaf_nms_multi_label_workspace_bytes(B, R, no)
    assert need == B * R * 3 * 16 == ops.nms_workspace_bytes(B, R, no, True)
    assert ops.nms_workspace_bytes(B, R, no, False) == L.icaf_nms_workspace_bytes(B, R)
    assert ops.nms_workspace_bytes(B, R, 6, True) == L.icaf_nms_workspace_bytes(B, R)      # nc == 1: best-class path
    assert L.icaf_nms_multi_label_workspace_bytes(0, R, no) == 0 and L.icaf_nms_multi_label_workspace_bytes(B, R, 5) == 0
    assert L.icaf_nms_multi_label_workspace_bytes(B, 1 << 30, 10) == 0                     # R * nc overflows int
    ws = ctypes.c_void_p(1 << 20)
    n0 = L.icaf_kernel_launches()

    def call(z=one, B=B, R=R, no=no, mask=0, max_det=300, det=one, count=one, ws=ws, ws_bytes=need):
        return L.icaf_nms_multi_label(z, B, R, no, 0.001, 0.6, 0, ctypes.c_uint64(mask), max_det, det, count, ws, ws_bytes, None)

    assert call(z=None) == 1 and call(det=None) == 1 and call(count=None) == 1 and call(ws=None) == 1
    assert b"null" in L.icaf_last_error()
    assert call(no=5) == 1 and call(B=0) == 1 and call(R=0) == 1
    assert call(max_det=0) == 1 and call(max_det=1025) == 1
    assert call(ws_bytes=need - 1) == 1 and b"icaf_nms_multi_label_workspace_bytes" in L.icaf_last_error()
    assert call(ws=ctypes.c_void_p((1 << 20) + 4)) == 1                                    # not 8-byte aligned
    assert call(no=5 + 65, mask=1, ws_bytes=1 << 40) == 2                                  # class filter over 65 classes
    assert call(R=1 << 30, no=10, ws_bytes=1 << 62) == 2                                   # R * nc overflows int
    assert L.icaf_kernel_launches() == n0
