"""CPU-side checks of the boundary: the shared library loads, exports every symbol include/icaf_b200.h declares,
argument validation works without a GPU, and the product path refuses to run without CUDA (no fallback)."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "icaf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(icaf_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from icafusion_b200 import _lib
    L = _lib.lib()
    syms = _header_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/icaf_b200.h but not exported"
    assert set(syms) == set(_lib.SIGNATURES), set(syms) ^ set(_lib.SIGNATURES)
    assert L.icaf_version() >= 100


def test_argument_validation_needs_no_gpu():
    """Bad arguments are rejected on the host before any launch; the error string is readable through the ABI."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    g = _lib.ConvGeom(1, 8, 8, 12, 8, 8, 16, 1, 1, 1, 0, 64, 32, 0, 0)      # Cin=12: not 4 / multiple of 8
    io = (_lib.ConvIO * 1)()
    rc = L.icaf_conv2d_fwd(ctypes.byref(g), io, 1, None)
    assert rc == 2 and b"Cin" in L.icaf_last_error()
    rc = L.icaf_cross_attention(None, None, None, None, None, None, 1, 10, 16, 128, 8, None)
    assert rc == 1
    with pytest.raises(_lib.IcafError):
        _lib.check(rc, "icaf_cross_attention")


def test_no_cpu_fallback():
    from icafusion_b200 import Conv, Model, TransformerFusionBlock
    x = torch.randn(1, 64, 8, 8)
    with pytest.raises(RuntimeError):
        Conv(64, 64).eval()(x)
    with pytest.raises(RuntimeError):
        TransformerFusionBlock(128, 4, 4).eval()([torch.randn(1, 128, 8, 8)] * 2)
    m = Model("yolov5s_Transfusion_kaist").eval()
    with pytest.raises(RuntimeError):
        m(torch.rand(1, 3, 320, 320), torch.rand(1, 3, 320, 320))


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from icafusion_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.IcafError):
        _lib.lib()


def test_shipped_library_has_no_probe_hooks_and_counts_launches():
    """The library exports no debug hook (icaf_debug_set) beyond the header's symbols.  The launch tally behind bench.py's `gpu_launches` starts at zero and does not move on rejected calls."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    assert not hasattr(L, "icaf_debug_set")
    n0 = L.icaf_kernel_launches()
    g = _lib.ConvGeom(1, 8, 8, 12, 8, 8, 16, 1, 1, 1, 0, 64, 32, 0, 0)      # rejected on the host (Cin = 12)
    io = (_lib.ConvIO * 1)()
    assert L.icaf_conv2d_fwd(ctypes.byref(g), io, 1, None) != 0
    assert L.icaf_kernel_launches() == n0


# ---------------------------------------------------------------------------------------------------------------
# Host-only walk of the conv dispatcher over every layer geometry the detectors issue (no GPU): the product path is run
# in dry mode (meta tensors, nothing launched), every recorded icaf_conv2d_fwd geometry goes through icaf_conv2d_plan --
# the same planner + invariant checks icaf_conv2d_fwd runs before it launches.
def _dry_geometries(size: str, B: int, H: int = 512, W: int = 640):
    from icafusion_b200 import Model, ops
    m = Model(f"yolov5{size}_Transfusion_kaist").eval().fuse().half()
    rgb = torch.empty(B, 3, H, W, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run() as dr:
        z, logits, xs = m(rgb, rgb)
    assert z.shape[0] == B and z.shape[2] == 6
    seen, out = set(), []
    for name, args, work in dr.records:
        if name != "icaf_conv2d_fwd":
            continue
        g, n = work["geom"], work["n_io"]
        key = tuple(getattr(g, f) for f, _ in g._fields_) + (n,)
        if key not in seen:
            seen.add(key)
            out.append((g, n, work["tag"]))
    return out, len(dr.records)


def _check_plan(g, n, pl, sms, tag):
    from icafusion_b200 import _lib
    where = f"{tag}: kernel {pl.kernel} bn {pl.bn} a_mode {pl.a_mode} halo {pl.halo}"
    assert pl.kernel == _lib.KERNEL_TC and pl.bn in (32, 64, 128), where
    assert 0 < pl.smem_bytes <= 227 * 1024, where
    assert pl.grid_x >= 1 and pl.grid_y >= 1 and pl.grid_z >= 1 and pl.stages >= 1, where
    ctas = pl.grid_x * pl.grid_y * pl.grid_z
    if pl.a_mode == 2:       # 4-D TMA tiles cover the output map with <= 128 pixels per tile
        assert 1 <= pl.tile_w * pl.tile_h <= 128, where
        assert pl.tiles_x * pl.tile_w >= g.Wo and pl.tiles_y * pl.tile_h >= g.Ho, where
        assert (pl.tiles_x - 1) * pl.tile_w < g.Wo and (pl.tiles_y - 1) * pl.tile_h < g.Ho, where
        assert pl.cblk == 64 and g.Cin % pl.cblk == 0, where
    assert pl.halo == 0, where
    assert pl.cluster == pl.splits and 1 <= pl.splits <= 8 and pl.grid_x % pl.splits == 0, where
    assert ctas == pl.work_items * pl.splits, where


@pytest.mark.parametrize("size,B", [("s", 1), ("s", 16), ("l", 1), ("l", 16)])
def test_dispatcher_plans_every_layer_geometry(size, B):
    from icafusion_b200 import _lib
    L = _lib.lib()
    geoms, n_calls = _dry_geometries(size, B)
    assert len(geoms) >= 25 and n_calls >= 60
    kernels = set()
    for g, n, tag in geoms:
        for sms in (132, 148):
            for pair_mode in (0, 1, 2):
                pl = _lib.ConvPlan()
                rc = L.icaf_conv2d_plan(ctypes.byref(g), n, sms, pair_mode, ctypes.byref(pl))
                assert rc == 0, f"{tag} (sms {sms}, pair mode {pair_mode}): {L.icaf_last_error().decode()}"
                _check_plan(g, n, pl, sms, tag)
                if sms == 132 and pair_mode == 1:
                    kernels.add((pl.bn, pl.a_mode))
    if (size, B) == ("l", 16):     # the compute-bound config exercises every tile width and every activation staging mode
        assert {32, 64, 128} <= {k[0] for k in kernels} and {0, 1, 2} <= {k[1] for k in kernels}, kernels


def test_dispatcher_plan_matches_small_and_odd_geometries():
    """The GPU parity cases of tests/test_gpu_conv.py (ragged N, odd maps, strides, split-K shapes) plan cleanly too."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    cases = [(1, 8, 8, 64, 96, 1, 1, 0), (2, 20, 16, 64, 64, 3, 1, 1), (1, 16, 20, 512, 512, 3, 1, 1), (8, 64, 80, 64, 64, 3, 1, 1),
             (1, 33, 47, 64, 128, 3, 2, 1), (16, 128, 160, 64, 64, 3, 1, 1), (1, 10, 10, 1024, 4096, 1, 1, 0),
             (16, 256, 320, 16, 64, 3, 1, 1), (1, 256, 320, 16, 32, 3, 1, 1), (3, 17, 19, 24, 40, 3, 1, 1)]
    for B, Hi, Wi, Cin, Cout, k, s, p in cases:
        Ho, Wo = (Hi + 2 * p - k) // s + 1, (Wi + 2 * p - k) // s + 1
        kp = (k * k * Cin + 63) // 64 * 64
        g = _lib.ConvGeom(B, Hi, Wi, Cin, Ho, Wo, Cout, k, k, s, p, kp, (Cout + 31) // 32 * 32, 1, 0)
        for n in (1, 2):
            for pair_mode in (0, 1, 2):
                pl = _lib.ConvPlan()
                rc = L.icaf_conv2d_plan(ctypes.byref(g), n, 132, pair_mode, ctypes.byref(pl))
                assert rc == 0, L.icaf_last_error().decode()
                _check_plan(g, n, pl, 132, f"B{B} {Hi}x{Wi} {Cin}->{Cout} k{k}s{s}")
    bad = _lib.ConvGeom(1, 8, 8, 12, 8, 8, 16, 1, 1, 1, 0, 64, 32, 0, 0)
    assert L.icaf_conv2d_plan(ctypes.byref(bad), 1, 132, -1, ctypes.byref(_lib.ConvPlan())) == 2
    assert L.icaf_conv2d_plan(ctypes.byref(g), 1, 0, -1, ctypes.byref(_lib.ConvPlan())) == 1


@pytest.mark.parametrize("size,B", [("s", 2), ("l", 16)])
def test_training_step_dry_run_plans_every_geometry(size, B):
    """The training step (train-mode forward + backward of the whole model) walked on `meta` tensors in the GPU-less container:
    every convolution it issues -- forward filters and the flipped / transposed data-gradient filters over (zero-stuffed)
    gradient maps -- plans cleanly in the dispatcher, every weight-gradient geometry is one icaf_conv2d_wgrad supports (the wrapper
    raises when its host-side plan returns no workspace size), and exactly the reference's live parameters receive a gradient."""
    from icafusion_b200 import Model, _lib, ops
    L = _lib.lib()
    m = Model(f"yolov5{size}_Transfusion_kaist").to("meta").train()
    rgb = torch.empty(B, 3, 512, 640, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        pred = m(rgb, rgb)
        assert [tuple(p.shape) for p in pred] == [(B, 3, 64, 80, 6), (B, 3, 32, 40, 6), (B, 3, 16, 20, 6)]
        torch.autograd.backward(pred, [torch.empty_like(p) for p in pred])
    count = {}
    seen = set()
    for name, args, work in dr.records:
        count[name] = count.get(name, 0) + 1
        if name == "icaf_conv2d_fwd":
            g, n = work["geom"], work["n_io"]
            key = tuple(getattr(g, f) for f, _ in g._fields_) + (n,)
            if key in seen:
                continue
            seen.add(key)
            pl = _lib.ConvPlan()
            rc = L.icaf_conv2d_plan(ctypes.byref(g), n, 132, -1, ctypes.byref(pl))
            assert rc == 0, f"{work['tag']}: {L.icaf_last_error().decode()}"
            _check_plan(g, n, pl, 132, work["tag"])
    n_bn = sum(isinstance(x, torch.nn.BatchNorm2d) for x in m.modules())
    assert count["icaf_bn_act_fwd"] == count["icaf_bn_act_bwd"] == n_bn
    # one weight gradient per Conv / Detect conv / live Linear (the three q, k, v projections of a modality share one GEMM)
    n_lin = sum(isinstance(x, torch.nn.Linear) for x in m.modules())
    n_dmff = sum(type(x).__name__ == "CrossTransformerBlock" for x in m.modules())
    assert count["icaf_conv2d_wgrad"] == n_bn + 3 + (n_lin - n_dmff * (2 + 6)) + 2 * n_dmff
    assert count["icaf_cross_attention_train"] == count["icaf_cross_attention_bwd"] == 3
    dead = sorted(k for k, p in m.named_parameters() if p.grad is None)
    from icafusion_b200.trainer import dead_parameters
    assert dead == sorted(dead_parameters(m)) and len(dead) == 30


def test_training_entry_points_validate_arguments_without_a_gpu():
    """The backward / training entry points reject bad arguments on the host, before any CUDA call (return code + readable
    icaf_last_error), and their workspace-size queries are pure functions."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    P = ctypes.c_void_p
    one = P(16)                                   # a non-null pointer that is never dereferenced: validation fails first
    assert L.icaf_train_workspace_bytes(64) > 0 and L.icaf_train_workspace_bytes(256) == 4 * L.icaf_train_workspace_bytes(64)
    # BatchNorm: C not a multiple of 8 / workspace too small
    assert L.icaf_bn_act_fwd(one, one, one, None, None, one, one, one, 100, 12, 1e-3, 0.03, 1, one, 1 << 30, None) == 1
    assert L.icaf_bn_act_fwd(one, one, one, None, None, one, one, one, 100, 64, 1e-3, 0.03, 1, one, 16, None) == 1
    assert b"workspace" in L.icaf_last_error()
    assert L.icaf_bn_act_bwd(one, one, one, one, one, one, one, None, None, 100, 64, 1, 1.0, 0, one, 16, None) == 1
    # attention backward: head dim 24 is not built; dropout probability must be < 1
    ws = L.icaf_cross_attention_bwd_workspace_bytes(2, 104, 8)
    assert ws == 2 * 2 * 8 * 104 * 2 * 4
    assert L.icaf_cross_attention_bwd(one, one, one, one, one, one, one, one, 2, 100, 104, 192, 8, 0.0, 0, one, ws, None) == 2
    assert L.icaf_cross_attention_bwd(one, one, one, one, one, one, one, one, 2, 100, 104, 256, 8, 1.0, 0, one, ws, None) == 1
    assert L.icaf_cross_attention_train(one, one, one, one, 2, 100, 104, 256, 8, 1.5, 0, None) == 1
    # weight gradient: unsupported channel count -> no workspace size, and the call itself refuses
    bad = _lib.ConvGeom(1, 16, 16, 24, 16, 16, 64, 3, 3, 1, 1, 256, 64, 0, 0)          # Cin = 24
    assert L.icaf_conv2d_wgrad_workspace_bytes(ctypes.byref(bad)) == 0
    good = _lib.ConvGeom(2, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 576, 64, 0, 0)
    need = L.icaf_conv2d_wgrad_workspace_bytes(ctypes.byref(good))
    assert need > 0
    assert L.icaf_conv2d_wgrad(ctypes.byref(good), one, 64, one, 64, one, 1.0, 0, one, need - 1, None) != 0
    # filter packing: padded sizes smaller than the filter
    assert L.icaf_pack_weight(one, 64, 64, 3, 3, 64, 32, 576, 0, one, None) == 1
    assert L.icaf_pack_weight_pair(one, 64, 64, 3, 3, 64, 576, one, 64, 64, 512, one, None) == 1
    # DMFF tail backward exists for the training-mode (nearest) tail only
    assert L.icaf_dmff_upsample_cat_bwd(one, 256, one, one, 1, 16, 16, 128, 8, 8, 64, 0, None) == 2
    assert L.icaf_dmff_pool_tokens_bwd(one, one, 128, one, one, one, one, one, 1, 16, 16, 128, 8, 8, 64, one, 8, None) == 1
    assert L.icaf_maxpool5_bwd(one, one, one, 1, 8, 8, 64, one, 8, None) == 1
    # loss backward: needs the backward workspace (no_bwd = no) and a gradient pointer
    ny, nx = (ctypes.c_int * 3)(8, 4, 2), (ctypes.c_int * 3)(8, 4, 2)
    w_f, w_b = L.icaf_loss_workspace_bytes(2, 3, 4, ny, nx, 3, 0), L.icaf_loss_workspace_bytes(2, 3, 4, ny, nx, 3, 6)
    assert 0 < w_f < w_b
    ptrs = (ctypes.c_void_p * 3)(16, 16, 16)
    anch = (ctypes.c_float * 18)(*([1.0] * 18))
    hyp = _lib.LossHyp(0.05, 1.0, 0.5, 1.0, 1.0, 4.0, 0.0, 1.0, 1.0, 0.0, (ctypes.c_float * 5)(4.0, 1.0, 0.4, 0.0, 0.0))
    assert L.icaf_compute_loss_bwd(ptrs, 0, 0, ny, nx, 3, 2, 3, 6, one, 4, anch, ctypes.byref(hyp), None, ptrs, one, w_b, None) == 1
    assert L.icaf_compute_loss_bwd(ptrs, 0, 0, ny, nx, 3, 2, 3, 6, one, 4, anch, ctypes.byref(hyp), one, ptrs, P(256), w_f, None) == 1
    assert L.icaf_set_seed_offset(None) == 0
