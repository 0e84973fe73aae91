"""KAIST miss rate without a GPU: the annotation arrays and per-setup ignore flags against the reference's _prepare, the
result-file parser against float(), the %g rounding formula (numpy mirror of icaf_kaist_round_detections) against
float('%g' % v), host-side refusals of icaf_kaist_mr / icaf_kaist_round_detections, and test.test(mr_annotations=...)'s
launches in a dry run."""
import ctypes
import gzip
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden
from oracle.gen_golden_kaist_mr import ANN, CASES, SMALL_ANN, build_small, gunzip_to

P10 = np.array([float(f"1e{k}") for k in range(23)])


def round_g6(v32: np.ndarray) -> np.ndarray:
    """numpy mirror of the device rounding (exact for 0 and 1e-7 <= |v| < 1e6): rint(v * 10^k) / 10^k, k = 5 - decade."""
    v = np.asarray(v32, dtype=np.float32).astype(np.float64)
    x = np.abs(v) * 1e12
    e = 5 + sum((x >= P10[k]).astype(np.int64) for k in range(6, 18))
    k = 17 - e
    out = np.rint(v * P10[k]) / P10[k]
    return np.where(v == 0, v, out)


def _setup_ignore(h, occ, box, json_ig):
    """_prepare's flag per setup (evaluation_script.py:59-71), as icaf_kaist_mr computes it."""
    ht = [[55, 1e10], [115, 1e10], [45, 115], [1, 45], [1, 1e10], [1, 1e10], [1, 1e10]]
    occs = [[0, 1], [0], [0], [0], [0], [1], [2]]
    out = []
    for s in range(7):
        out.append((json_ig != 0) | (h < ht[s][0]) | (h > ht[s][1]) | ~np.isin(occ, occs[s]) | (box[:, 0] < 5) |
                   (box[:, 1] < 5) | (box[:, 0] + box[:, 2] > 635) | (box[:, 1] + box[:, 3] > 507))
    return np.stack(out).astype(np.uint8)


def test_annotations_and_setup_ignore_flags_match_reference_prepare():
    from icafusion_b200.kaist_eval import KaistAnnotations
    meta, d = load_golden("kaist_mr_cases")
    ann = KaistAnnotations(os.path.join(GOLDEN, ANN), "cpu")
    h = ann.host
    assert ann.images == 2252 and ann.image_ids == list(range(2252)) and h["id"].shape == (4254,)
    assert h["offset"][0] == 0 and h["offset"][-1] == 4254 and np.diff(h["offset"]).max() == 21
    flags = np.zeros_like(d["ignore_flags"])
    flags[:, h["id"]] = _setup_ignore(h["height"], h["occlusion"], h["box"], h["ignore"])
    assert np.array_equal(flags, d["ignore_flags"])
    assert 0 < d["ignore_flags"][0].sum() < 4254 and not np.array_equal(d["ignore_flags"][1], d["ignore_flags"][3])


@pytest.mark.parametrize("case", [c for c, (_, f) in CASES.items() if ".txt" in f])
def test_parser_equals_float_on_every_token(case, tmp_path):
    from icafusion_b200.kaist_eval import KaistAnnotations, load_detections
    a, f = CASES[case]
    ann = KaistAnnotations(os.path.join(GOLDEN, a), "cpu")
    rows, span, mx = load_detections(os.path.join(GOLDEN, f), ann)
    lines = gzip.open(os.path.join(GOLDEN, f), "rt").read().splitlines()
    want = {}
    for line in lines:
        v = [float(t) for t in line.split(",")]
        want.setdefault(ann.position[v[0] - 1], []).append(v[1:6])
    assert rows.shape == (len(lines), 5) and mx == max(len(v) for v in want.values())
    for p, vals in want.items():
        o, n = span[p]
        assert n == len(vals)
        assert np.array_equal(rows[o:o + n], np.array(vals)), p      # bitwise: == on doubles, no NaN in the fixtures


def test_json_results_parse_to_the_txt_values():
    from icafusion_b200.kaist_eval import KaistAnnotations, load_detections
    ann = KaistAnnotations(os.path.join(GOLDEN, ANN), "cpu")
    rows, span, _ = load_detections(os.path.join(GOLDEN, CASES["MLPD_json"][1]), ann)
    rt, st, _ = load_detections(os.path.join(GOLDEN, CASES["MLPD"][1]), ann)
    assert np.array_equal(span, st) and np.abs(rows - rt).max() < 2e-4      # the .txt has 4 / 8 decimals


def test_rounding_mirror_equals_printf_g():
    g = np.random.Generator(np.random.PCG64(3))
    mag = np.exp(g.uniform(np.log(1e-7), np.log(1e6), 1_000_000)).astype(np.float32)
    v = np.where(g.uniform(size=mag.size) < 0.1, -mag, mag).astype(np.float32)
    v = v[(np.abs(v) >= 1e-7) & (np.abs(v) < 1e6)]
    edges = []
    for k in range(-7, 6):
        p = np.float32(10.0 ** k)
        edges += [p, np.nextafter(p, np.float32(0)), np.nextafter(p, np.float32(np.inf)), -p]
    # exact ties at the 6th digit: x.5 units of the last place, representable in fp32 (ties go to even, as printf does)
    ties = np.array([0.5, 1.5, 2.5, 1234.5, 2345.5, 12345.5 / 8, 640.0625, 0.0009765625, 99999.5, 999999.5 / 4, 0.0],
                    dtype=np.float32)
    v = np.concatenate([v, np.array(edges, np.float32), ties])
    v = v[(v == 0) | ((np.abs(v) >= 1e-7) & (np.abs(v) < 1e6))]
    got = round_g6(v)
    want = np.array([float("%g" % x) for x in v.tolist()])
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(float(v[i]), got[i], want[i]) for i in bad[:5]]
    assert (ties[:-1].astype(np.float64) != round_g6(ties[:-1])).any()        # the ties do round


def test_kaist_mr_rejects_bad_arguments_without_a_gpu():
    from icafusion_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(256)
    good = dict(box=one, height=one, occ=one, ig=one, id=one, offset=one, images=2252, gts=4254, day=1455, rows=one,
                span=one, nrows=5939, mpi=300, ys=one, counts=one, curves=None, ws=one, ws_bytes=1 << 30)

    def call(**kw):
        a = dict(good, **kw)
        return L.icaf_kaist_mr(a["box"], a["height"], a["occ"], a["ig"], a["id"], a["offset"], a["images"], a["gts"],
                               a["day"], a["rows"], a["span"], a["nrows"], a["mpi"], a["ys"], a["counts"], a["curves"],
                               a["ws"], a["ws_bytes"], None)
    n0 = L.icaf_kernel_launches()
    for bad in (dict(box=None), dict(height=None), dict(occ=None), dict(ig=None), dict(id=None), dict(offset=None),
                dict(rows=None), dict(span=None), dict(ys=None), dict(counts=None), dict(ws=None), dict(images=0),
                dict(gts=-1), dict(nrows=-1), dict(day=-1), dict(mpi=-1), dict(mpi=1001), dict(ws=ctypes.c_void_p(264))):
        assert call(**bad) == 1, bad
        assert L.icaf_last_error()
    assert call(mpi=1001) == 1 and b"more than 1000" in L.icaf_last_error()
    assert L.icaf_kaist_mr_workspace_bytes(0, 10, 10) == 0 and L.icaf_kaist_mr_workspace_bytes(10, -1, 10) == 0
    assert L.icaf_kaist_mr_workspace_bytes(10, 10, -1) == 0
    rd = dict(native=one, det=one, count=one, image=one, B=4, max_det=300, images=40, rows=one, span=one)

    def rcall(**kw):
        a = dict(rd, **kw)
        return L.icaf_kaist_round_detections(a["native"], a["det"], a["count"], a["image"], a["B"], a["max_det"],
                                             a["images"], a["rows"], a["span"], None)
    for bad in (dict(native=None), dict(det=None), dict(count=None), dict(image=None), dict(rows=None), dict(span=None),
                dict(B=0), dict(max_det=0), dict(images=0), dict(images=1 << 22, max_det=1000)):
        assert rcall(**bad) == 1, bad
    assert L.icaf_kernel_launches() == n0


def test_more_than_1000_detections_in_one_image_is_refused(tmp_path):
    from icafusion_b200 import ops
    from icafusion_b200.kaist_eval import KaistAnnotations, load_detections
    ann = KaistAnnotations(os.path.join(GOLDEN, SMALL_ANN), "cpu")
    p = tmp_path / "many_result.txt"
    p.write_text("".join("3,10,20,30,60,0.5\n" for _ in range(1001)) + "1,10,20,30,60,0.5\n")
    with pytest.raises(ValueError, match="image 2 has 1001 detections"):
        load_detections(str(p), ann)
    p.write_text("".join("3,10,20,30,60,0.5\n" for _ in range(1000)))
    assert load_detections(str(p), ann)[2] == 1000
    with pytest.raises(ValueError, match="more than 1000"):
        ops.kaist_mr(ann, torch.zeros(1001, 5, dtype=torch.float64), torch.zeros(40, 2, dtype=torch.int32), 1001)
    p.write_text("0,10,20,30,60,0.5\n")                  # image id -1: not in the annotations (the reference asserts)
    with pytest.raises(ValueError, match="do not correspond"):
        load_detections(str(p), ann)


def test_new_symbols_in_header_and_signatures():
    from icafusion_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "icaf_b200.h")).read()
    for name in ("icaf_kaist_mr_workspace_bytes", "icaf_kaist_mr", "icaf_kaist_round_detections"):
        assert re.search(r"\b%s\(" % name, hdr), name
        assert name in _lib.SIGNATURES
        assert hasattr(_lib.lib(), name)


def test_dry_run_test_with_mr_annotations_launches(tmp_path, monkeypatch):
    """test.test(mr_annotations=...) records one icaf_kaist_round_detections per batch and one icaf_kaist_mr, all before
    its single synchronise (the run stops there: a dry run has no values to gather)."""
    from icafusion_b200 import ops
    from icafusion_b200 import test as T
    from oracle.gen_golden_val import StubDetector, loader

    class _Event:
        def __init__(self, **k):
            pass

        def record(self):
            pass

    class _Synchronised(Exception):
        pass

    def _sync():
        raise _Synchronised()
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "synchronize", _sync)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    batches, labels_list, _ = build_small()
    stub = StubDetector([b[0] for b in batches], 1).to("meta")
    ann = gunzip_to(SMALL_ANN, tmp_path)
    with torch.no_grad(), ops.dry_run() as dr, pytest.raises(_Synchronised):
        T.test({"nc": 1, "names": ["person"]}, model=stub, dataloader=loader(batches, device="meta"), save_dir=tmp_path,
               labels_list=labels_list, mr_annotations=ann)
    names = [n for n, _, _ in dr.records]
    assert names.count("icaf_kaist_round_detections") == len(batches) == names.count("icaf_match_detections")
    assert names.count("icaf_kaist_mr") == 1 and names[-1] == "icaf_kaist_mr"
    with ops.dry_run(), pytest.raises(ValueError, match="labels_list"):
        T.test({"nc": 1, "names": ["person"]}, model=stub, dataloader=[], save_dir=tmp_path, mr_annotations=ann)
