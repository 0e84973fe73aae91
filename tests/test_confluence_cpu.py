"""Confluence without a GPU: the fp64 restatement reproduces the real reference's rows (tests/golden/confluence_cases.npz
from oracle/gen_golden_confluence.py), the properties the kernel relies on hold, and icaf_confluence is declared,
exported, sized by a pure query, recorded by a dry run and refuses bad arguments on the host before any launch."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.confluence import confluence_process, pair_p
from oracle.gen_golden_confluence import checked_inputs
from test_conv_ptxas_cpu import _nvcc


def test_oracle_matches_reference_golden():
    m, d = load_golden("confluence_cases")
    inputs = checked_inputs(m)
    nones = kept = 0
    for inp in m["inputs"]:
        pred = inputs[inp["name"]]
        assert pred.shape[2] - 5 == inp["nc"] and str(pred.dtype) == inp["dtype"]
        for st in inp["settings"]:
            out = confluence_process(pred, st["conf"], st["p_thres"])
            for b, o in enumerate(out):
                if st["counts"][b] is None:
                    assert o is None, (inp["name"], st["name"], b)
                    nones += 1
                    continue
                want = d[f"{inp['name']}_{st['name']}_{b}"]
                assert o.shape[0] == st["counts"][b] == want.shape[0], (inp["name"], st["name"], b)
                assert np.array_equal(o, want), (inp["name"], st["name"], b)
                kept += o.shape[0]
    assert {i["nc"] for i in m["inputs"]} == {1, 3} and {i["dtype"] for i in m["inputs"]} == {"float16", "float32"}
    assert nones == 2 and kept > 500
    assert {(s["conf"], s["p_thres"]) for i in m["inputs"] for s in i["settings"]} == {(0.1, 0.6), (0.1, 0.5)}


def test_golden_inputs_cover_the_edge_cases():
    """Duplicates (p = 0), zero-width boxes sharing an x (NaN p), equal confidences and a single-candidate class."""
    from oracle.confluence import candidates
    m, _ = load_golden("confluence_cases")
    inputs = checked_inputs(m)
    d = candidates(inputs["kaist"][0], 0.1)
    P = pair_p(d[:, :4].astype(np.float64))
    off = ~np.eye(len(d), dtype=bool)
    assert (P[off] == 0).any() and np.isnan(P).any()
    assert np.unique(d[:, 4], return_counts=True)[1].max() >= 6
    f = candidates(inputs["flir"][0].astype(np.float32), 0.1)
    assert (f[:, 5] == 2).sum() == 1


def test_p_is_symmetric_and_division_is_monotone():
    g = np.random.Generator(np.random.PCG64(3))
    xy = g.uniform(0, 600, size=(400, 2)).astype(np.float32)
    wh = g.uniform(0, 80, size=(400, 2)).astype(np.float32)
    wh[:40, 0] = 0.0
    xy[40:80] = xy[:40]
    box = np.concatenate([xy, xy + wh], 1).astype(np.float64)
    P = pair_p(box)
    assert np.array_equal(P, P.T, equal_nan=True)
    conf = g.uniform(2.5e-4, 1, size=400).astype(np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        Pm = np.where(P < 2, P, np.inf)
    np.fill_diagonal(Pm, np.inf)
    has = np.isfinite(Pm).any(1)
    assert np.array_equal((Pm / conf[:, None]).min(1)[has], (Pm.min(1) / conf)[has])


def test_entry_is_declared_exported_and_validates_arguments_without_a_gpu():
    from test_abi_cpu import _header_symbols
    from icafusion_b200 import _lib, ops
    L = _lib.lib()
    for s in ("icaf_confluence", "icaf_confluence_workspace_bytes"):
        assert s in _header_symbols() and s in _lib.SIGNATURES and hasattr(L, s)
    B, R, no = 2, 1000, 8
    need = L.icaf_confluence_workspace_bytes(B, R, no)
    assert need == B * 3 * 1008 * 37 + B * R * 3 == ops.confluence_workspace_bytes(B, R, no)
    assert L.icaf_confluence_workspace_bytes(0, R, no) == 0 and L.icaf_confluence_workspace_bytes(B, R, 5) == 0
    assert L.icaf_confluence_workspace_bytes(B, 1 << 30, 10) == 0                       # R * nc overflows int
    one, ws = ctypes.c_void_p(16), ctypes.c_void_p(1 << 20)                            # never dereferenced
    n0 = L.icaf_kernel_launches()

    def call(z=one, dtype=0, B=B, R=R, no=no, conf=0.1, p=0.6, det=one, max_det=300, count=one, ws=ws, ws_bytes=need):
        return L.icaf_confluence(z, dtype, B, R, no, conf, p, det, None, max_det, count, ws, ws_bytes, None)

    assert call(z=None) == 1 and call(det=None) == 1 and call(count=None) == 1 and call(ws=None) == 1
    assert b"null" in L.icaf_last_error()
    assert call(dtype=3) == 1 and call(dtype=-1) == 1
    assert call(no=5) == 1 and call(B=0) == 1 and call(R=0) == 1 and call(max_det=0) == 1
    assert call(conf=2e-4) == 1 and b"2.5e-4" in L.icaf_last_error() and call(conf=float("nan")) == 1
    assert call(p=float("nan")) == 1
    assert call(ws_bytes=need - 1) == 1 and b"icaf_confluence_workspace_bytes" in L.icaf_last_error()
    assert call(ws=ctypes.c_void_p((1 << 20) + 8)) == 1                                # not 16-byte aligned
    assert call(R=1 << 30, no=10, ws_bytes=1 << 62) == 2 and call(B=70000, ws_bytes=1 << 62) == 2
    assert L.icaf_kernel_launches() == n0


def test_python_wrappers_refuse_bad_input():
    from icafusion_b200 import confluence as CF, ops
    with pytest.raises(ValueError):
        ops.confluence(torch.zeros(1, 10, 6, dtype=torch.float16, device="meta").transpose(0, 1))
    with pytest.raises(ValueError):
        CF.confluence(np.zeros((3, 6)) + 0.1, 1)                                       # not exact in fp32
    rows = np.array([[0, 0, 1, 1, 1e-4, 0]], dtype=np.float32)
    with pytest.raises(ValueError):
        CF.confluence(rows, 1)                                                          # conf below 2.5e-4
    assert CF.confluence(np.zeros((0, 6), np.float32), 1).shape == (0,)


def test_dry_run_records_one_call():
    from icafusion_b200 import ops
    z = torch.empty(4, 20160, 8, dtype=torch.float16, device="meta")
    with ops.dry_run() as d:
        det, count = ops.confluence(z, 0.1, 0.5, max_det=500)
    assert [r[0] for r in d.records] == ["icaf_confluence"]
    args = d.records[0][1]
    assert args[1:5] == (0, 4, 20160, 8) and args[9] == 500
    assert args[5] == pytest.approx(0.1) and args[6] == 0.5
    assert tuple(det.shape) == (4, 500, 6) and tuple(count.shape) == (4,)


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_confluence_kernels_spill_free(tmp_path):
    """ptxas report of confluence.cu: no kernel spills (the fp64 division stays inline, without a call)."""
    from icafusion_b200 import build as B
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    assert "confluence.cu" in B.SOURCES and not any("fast" in f for f in flags)
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "confluence.cu"), "-o", str(tmp_path / "c.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    kernels = re.findall(r"Compiling entry function '(\w*confluence_\w+_kernel\w*)'", log)
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(kernels) == 6 and len(spills) == 6, log
    assert all(s == ("0", "0", "0") for s in spills), log
