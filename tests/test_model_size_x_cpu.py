"""yolov5x (DMFF head dims 40 / 80 / 160) without a GPU: the stock configs equal the config the reference's Model parsed, the
CPU oracle reproduces the reference's outputs (tests/golden/yolov5x_flir_*.npz, oracle/gen_golden_sizes_x.py), every
convolution plans in the dispatcher, training is refused before any launch, the attention entry points accept / refuse
the right head dims, and the exact-width D = 160 attention kernel compiles without spills or serialised wgmmas."""
import ctypes
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, normwise
from icafusion_b200.cfg import load_cfg
from oracle import icaf_oracle as O
from oracle import synth
from test_conv_ptxas_cpu import _nvcc
from test_model_sizes_cpu import _plan_all

TOL_FP32 = 2e-5


@pytest.mark.parametrize("dataset", ["kaist", "FLIR"])
def test_stock_cfg_equals_reference_parsed_cfg(dataset):
    name = f"yolov5x_Transfusion_{dataset}"
    with open(os.path.join(GOLDEN, "reference_cfg_x.json")) as f:
        ref = json.load(f)[name]
    mine = json.loads(json.dumps(load_cfg(name)))
    ref = json.loads(json.dumps(load_cfg(ref)))          # the same symbolic Detect arguments resolved on both sides
    for k in ("nc", "depth_multiple", "width_multiple", "anchors", "backbone", "head"):
        assert mine[k] == ref[k], k
    assert (mine["depth_multiple"], mine["width_multiple"]) == (1.33, 1.25)
    assert load_cfg(name + ".yaml") == load_cfg(name)


@pytest.mark.parametrize("name", ["yolov5x_flir_320", "yolov5x_flir_512x640"])
def test_model_oracle_matches_reference(name):
    """As tests/test_model_sizes_cpu.py: each fp32 output of the oracle matches the reference's fingerprint to 2e-5 of its
    norm, and z matches the stored fp16 z to its rounding."""
    from oracle.gen_golden_train import fingerprint
    m, d = load_golden(name)
    cfg = load_cfg("yolov5x_Transfusion_FLIR")
    assert m["size"] == "x" and cfg["nc"] == m["nc"] == 3
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    with torch.no_grad():
        z, lg, xs = O.model_forward(sd, cfg, rgb, ir)
        zf = O.model_forward(O.fold_bn(sd), cfg, rgb, ir)[0]
    outs = dict(z=z, z_fused=zf, logits=lg, x0=xs[0], x1=xs[1], x2=xs[2])
    for k, v in outs.items():
        assert list(v.shape) == m["shapes"][k], k
        want = d["fp:" + k]
        assert np.abs(fingerprint(v.numpy(), k) - want).max() < TOL_FP32 * want[0], k
    assert z.shape[2] == 8 and d["z16"].shape == z.shape
    assert normwise(z.numpy(), d["z16"].astype(np.float32)) < 1e-3
    assert m["fused_dev"] < 1e-5


@pytest.mark.parametrize("B", [1, 16])
def test_dispatcher_plans_every_inference_geometry_yolov5x(B):
    from icafusion_b200 import Model, ops
    m = Model("yolov5x_Transfusion_FLIR").eval().fuse().half()
    rgb = torch.empty(B, 3, 512, 640, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run() as dr:
        z, _, _ = m(rgb, rgb)
    assert tuple(z.shape) == (B, 20160, 8)
    counts, n_geoms = _plan_all(dr.records)
    assert n_geoms == 50
    attn = [args for name, args, _ in dr.records if name == "icaf_cross_attention"]
    assert [a[9] // a[10] for a in attn] == [40, 80, 160]                  # C / heads of the P3 / P4 / P5 blocks
    assert [a[7] for a in attn] == [400, 256, 100]                         # tokens: the 20x20 / 16x16 / 10x10 grids


def test_training_yolov5x_refused_before_any_launch():
    from icafusion_b200 import Model, ops
    m = Model("yolov5x_Transfusion_FLIR").to("meta").train()
    rgb = torch.empty(1, 3, 320, 320, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        with pytest.raises(NotImplementedError, match="head dim 40"):
            m(rgb, rgb)
    assert dr.records == []


def test_attention_head_dim_160_accepted_by_the_tensor_core_forward_only():
    """Head dim 160 passes the fused and split forms' shape checks (a misaligned pointer then stops the call before any
    launch, ICAF_ERR_BAD_ARG = 1); the CUDA-core and training forwards refuse it (ICAF_ERR_UNSUPPORTED = 2), as every entry
    point refuses 136, 168 and 200."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    one, odd = ctypes.c_void_p(16), ctypes.c_void_p(18)
    C = 8 * 160
    assert L.icaf_cross_attention(odd, odd, None, None, one, one, 1, 100, 104, C, 8, None) == 1
    assert b"16-byte aligned" in L.icaf_last_error()
    assert L.icaf_cross_attention(odd, odd, odd, odd, one, one, 1, 100, 104, C, 8, None) == 1
    assert b"16-byte aligned" in L.icaf_last_error()
    assert L.icaf_cross_attention_simt(one, one, None, None, one, one, 1, 100, 104, C, 8, None) == 2
    assert b"multiple of 8 in [8, 128]" in L.icaf_last_error()
    assert L.icaf_cross_attention_train(one, one, one, one, 1, 100, 104, C, 8, 0.1, 0, None) == 2
    assert L.icaf_cross_attention_train(one, one, one, one, 1, 100, 104, C, 8, 0.0, 0, None) == 2
    assert b"multiple of 8 in [8, 128]" in L.icaf_last_error()
    for d in (136, 168, 200):
        C = 8 * d
        assert L.icaf_cross_attention(one, one, None, None, one, one, 1, 100, 104, C, 8, None) == 2, d
        assert L.icaf_cross_attention(one, one, one, one, one, one, 1, 100, 104, C, 8, None) == 2, d
        assert b"multiple of 8" in L.icaf_last_error()
        assert L.icaf_cross_attention_simt(one, one, None, None, one, one, 1, 100, 104, C, 8, None) == 2, d
        assert L.icaf_cross_attention_train(one, one, one, one, 1, 100, 104, C, 8, 0.1, 0, None) == 2, d
    from icafusion_b200.autograd import ATTN_BWD_HEAD_DIMS
    assert not {40, 80, 160} & set(ATTN_BWD_HEAD_DIMS)


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_attention_d160_unserialised_and_spill_free(tmp_path):
    """ptxas report of attn.cu: the two D = 160 instantiations (fused and split V) exist, spill nothing and keep their
    wgmmas unserialised (warning C7510)."""
    from icafusion_b200 import build as B
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "attn.cu"), "-o", str(tmp_path / "attn.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    serialised = [l for l in log.splitlines() if "C7510" in l and "cross_attn_tma_kernelILi160E" in l]
    assert not serialised, serialised
    d160, entry = [], None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and entry and "cross_attn_tma_kernelILi160E" in entry:
            d160.append((entry, int(m.group(1)), int(m.group(2))))
            entry = None
    assert len(d160) == 2, log
    assert all(st == 0 and ld == 0 for _, st, ld in d160), d160
