"""yolov5n / yolov5m (DMFF head dims 8 / 24 / 48 / 96) without a GPU: the stock configs equal the reference's YAMLs, the CPU
oracle reproduces the reference's outputs for these sizes (tests/golden/*_flir_*.npz, oracle/gen_golden_sizes.py), every
convolution they issue plans in the dispatcher, and the attention entry points accept / refuse the right head dims."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, normwise
from icafusion_b200.cfg import load_cfg
from oracle import icaf_oracle as O
from oracle import synth
from test_abi_cpu import _check_plan

TOL_FP32 = 2e-5


@pytest.mark.parametrize("size", ["n", "m"])
@pytest.mark.parametrize("dataset", ["kaist", "FLIR"])
def test_stock_cfg_equals_reference_yaml(size, dataset):
    name = f"yolov5{size}_Transfusion_{dataset}"
    with open(os.path.join(GOLDEN, "reference_yaml_sizes.json")) as f:
        ref = json.load(f)[name]
    mine = json.loads(json.dumps(load_cfg(name)))
    ref = json.loads(json.dumps(load_cfg(ref)))          # the same symbolic Detect arguments resolved on both sides
    for k in ("nc", "depth_multiple", "width_multiple", "anchors", "backbone", "head"):
        assert mine[k] == ref[k], k
    assert load_cfg(name + ".yaml") == load_cfg(name)


def test_kaist_names_unchanged():
    from icafusion_b200.cfg import transfusion_kaist_cfg
    for size in "nsml":
        assert load_cfg(f"yolov5{size}_Transfusion_kaist") == load_cfg(transfusion_kaist_cfg(size))
        assert load_cfg(f"yolov5{size}_Transfusion_kaist")["nc"] == 1
        assert load_cfg(f"yolov5{size}_Transfusion_FLIR")["nc"] == 3
    with pytest.raises(FileNotFoundError):
        load_cfg("yolov5s_Transfusion_VEDAI")


@pytest.mark.parametrize("name", ["yolov5n_flir_320", "yolov5m_flir_320", "yolov5m_flir_512x640"])
def test_model_oracle_matches_reference(name):
    """The files keep the reference's z in fp16 and a float64 fingerprint (norm + two seeded projections) of every fp32
    output: the oracle's outputs must match each fingerprint to 2e-5 of the output's norm, and z element by element to the
    fp16 rounding."""
    from oracle.gen_golden_train import fingerprint
    m, d = load_golden(name)
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_FLIR")
    assert cfg["nc"] == m["nc"] == 3
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
    assert normwise(z.numpy(), d["z16"].astype(np.float32)) < 1e-3          # stored as fp16: rounding <= 2^-11 of max|z|
    assert m["fused_dev"] < 1e-5


def test_training_step_oracle_matches_reference_yolov5n():
    check_training_step_oracle("train_yolov5n_flir_320")


def test_training_step_oracle_matches_reference_yolov5l():
    """yolov5l (head dim 128 in the attention backward, up to nine Bottlenecks per C3; oracle/gen_golden_train_l.py): the
    oracle the GPU training-step test holds the device to."""
    # one-element gradients: one cancelling fp32 sum each over a 109 M-parameter model's token streams; the oracle run in
    # float64 lands 2 % from both fp32 steps on model.20.crosstransformer.0.coefficient7.bias, so summation order alone
    # moves them past 2e-4 (1.6e-3 measured)
    m, _ = check_training_step_oracle("train_yolov5l_320", scalar_tol=3e-3)
    assert len(m["params"]) == 633


def check_training_step_oracle(name, scalar_tol=2e-4):
    """The fp32 oracle's step against the reference's: loss, every gradient's fingerprint, the Detect maps, the BN probes."""
    from oracle.gen_golden_train import fingerprint
    m, d = load_golden(name)
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_{m['dataset']}")
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    loss, items, grads, pred, state = O.train_step(sd, cfg, rgb, ir, torch.from_numpy(d["targets"]), m["hyp"], m["gr"])
    got = np.concatenate([loss.numpy().reshape(1), items.numpy()])
    assert np.allclose(got, d["out"], rtol=1e-4, atol=1e-6), (got, d["out"])
    assert sorted(grads) == sorted(m["params"]) and len(m["dead_params"]) == 30
    dev = {k: float(np.abs(fingerprint(grads[k].numpy(), k) - d["g:" + k]).max() / max(d["g:" + k][0], 1e-3)) for k in m["params"]}
    worst = max(e for k, e in dev.items() if grads[k].numel() > 1)
    assert worst < 2e-4, worst
    worst = max(e for k, e in dev.items() if grads[k].numel() == 1)
    assert worst < scalar_tol, worst
    for i in range(3):
        want = d[f"pred{i}"]
        assert np.abs(fingerprint(pred[i].numpy(), f"pred{i}") - want).max() < 1e-4 * want[0]
    for k in m["bn_probes"]:
        assert np.allclose(state[k + ".running_mean"].numpy(), d["rm:" + k], rtol=1e-4, atol=1e-6)
        assert np.allclose(state[k + ".running_var"].numpy(), d["rv:" + k], rtol=1e-4, atol=1e-6)
    return m, d


def _plan_all(records):
    from icafusion_b200 import _lib
    L = _lib.lib()
    seen, counts = set(), {}
    for name, args, work in records:
        counts[name] = counts.get(name, 0) + 1
        if name != "icaf_conv2d_fwd":
            continue
        g, n = work["geom"], work["n_io"]
        key = tuple(getattr(g, f) for f, _ in g._fields_) + (n,)
        if key in seen:
            continue
        seen.add(key)
        pl = _lib.ConvPlan()
        rc = L.icaf_conv2d_plan(ctypes.byref(g), n, 132, -1, ctypes.byref(pl))
        assert rc == 0, f"{work['tag']}: {L.icaf_last_error().decode()}"
        _check_plan(g, n, pl, 132, work["tag"])
    return counts, len(seen)


@pytest.mark.parametrize("size,B", [("n", 1), ("n", 16), ("m", 1), ("m", 16)])
def test_dispatcher_plans_every_inference_geometry(size, B):
    from icafusion_b200 import Model, ops
    m = Model(f"yolov5{size}_Transfusion_FLIR").eval().fuse().half()
    rgb = torch.empty(B, 3, 512, 640, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run() as dr:
        z, _, _ = m(rgb, rgb)
    assert tuple(z.shape) == (B, 20160, 8)
    counts, n_geoms = _plan_all(dr.records)
    assert n_geoms >= 25 and counts["icaf_cross_attention"] == 3


def test_training_dry_run_yolov5n_plans_every_geometry():
    from icafusion_b200 import Model, ops
    m = Model("yolov5n_Transfusion_FLIR").to("meta").train()
    rgb = torch.empty(2, 3, 512, 640, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        pred = m(rgb, rgb)
        assert [tuple(p.shape) for p in pred] == [(2, 3, 64, 80, 8), (2, 3, 32, 40, 8), (2, 3, 16, 20, 8)]
        torch.autograd.backward(pred, [torch.empty_like(p) for p in pred])
    counts, _ = _plan_all(dr.records)
    assert counts["icaf_cross_attention_train"] == counts["icaf_cross_attention_bwd"] == 3
    heads = [args[11] // args[12] for name, args, _ in dr.records if name == "icaf_cross_attention_bwd"]   # C / heads
    assert sorted(heads) == [8, 16, 32]


def test_training_yolov5m_refused_before_any_launch():
    from icafusion_b200 import Model, ops
    m = Model("yolov5m_Transfusion_FLIR").to("meta").train()
    rgb = torch.empty(1, 3, 320, 320, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        with pytest.raises(NotImplementedError, match="head dim 24"):
            m(rgb, rgb)
    assert dr.records == []
    # the module-level training path refuses too
    from icafusion_b200 import common
    blk = common.CrossTransformerBlock(192, 192, 192, 8, 4, 0.1, 0.1).train()
    tok = torch.empty(1, 400, 192, dtype=torch.float16, device="meta")
    with ops.dry_run() as dr, pytest.raises(NotImplementedError, match="head dim 24"):
        blk([tok, tok])
    assert not any(name.startswith("icaf_cross_attention") for name, _, _ in dr.records)


def test_attention_head_dims_accepted_and_refused():
    """Head dims that are not a multiple of 8 in [8, 128] are refused on the host (ICAF_ERR_UNSUPPORTED = 2) by all three
    forward entry points; the backward takes 8 / 16 / 32 / 64 / 128 only.  Accepted calls would launch, so only refusals are
    exercised with dummy pointers."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(16)
    for C in (96, 1088, 8 * 4, 8 * 200):            # head dims 12, 136, 4, 200
        assert L.icaf_cross_attention(one, one, None, None, one, one, 1, 100, 104, C, 8, None) == 2, C
        assert L.icaf_cross_attention(one, one, one, one, one, one, 1, 100, 104, C, 8, None) == 2, C
        assert L.icaf_cross_attention_simt(one, one, None, None, one, one, 1, 100, 104, C, 8, None) == 2, C
        assert L.icaf_cross_attention_train(one, one, one, one, 1, 100, 104, C, 8, 0.1, 0, None) == 2, C
    assert b"multiple of 8" in L.icaf_last_error()
    ws = L.icaf_cross_attention_bwd_workspace_bytes(2, 104, 8)
    for C in (384, 768):                            # head dims 48, 96: no backward
        assert L.icaf_cross_attention_bwd(one, one, one, one, one, one, one, one, 2, 100, 104, C, 8, 0.0, 0, one, ws, None) == 2
    from icafusion_b200.autograd import ATTN_BWD_HEAD_DIMS
    assert 8 in ATTN_BWD_HEAD_DIMS and not {24, 48, 96} & set(ATTN_BWD_HEAD_DIMS)
