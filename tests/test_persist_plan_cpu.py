"""Host-only check of the rule that sends a conv launch to the persistent kernel (conv_gemm_persist_kernel): a 128 x 128
tile, TMA-staged activations, no split-K and more tiles than SMs.  The detector forwards are walked on `meta` tensors (nothing
is launched) and every recorded icaf_conv2d_fwd geometry goes through icaf_conv2d_plan."""
import ctypes

import pytest
import torch

SMS = 132


def _plans(size: str, B: int):
    from icafusion_b200 import Model, _lib, ops
    L = _lib.lib()
    m = Model(f"yolov5{size}_Transfusion_kaist").eval().fuse().half()
    rgb = torch.empty(B, 3, 512, 640, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run() as dr:
        m(rgb, rgb)
    out = []
    for name, args, work in dr.records:
        if name != "icaf_conv2d_fwd":
            continue
        pl = _lib.ConvPlan()
        assert L.icaf_conv2d_plan(ctypes.byref(work["geom"]), work["n_io"], SMS, 0, ctypes.byref(pl)) == 0, L.icaf_last_error().decode()
        out.append((work.get("tag", ""), work.get("flops", 0.0), pl))
    return out


def _eligible(pl):
    return pl.bn == 128 and pl.a_mode in (1, 2) and pl.splits == 1 and pl.work_items > SMS


@pytest.mark.parametrize("size,B", [("l", 16), ("s", 1)])
def test_persistent_kernel_takes_exactly_the_multi_wave_128_wide_tma_launches(size, B):
    plans = _plans(size, B)
    n_persist, flops_persist, flops_all = 0, 0.0, 0.0
    for tag, flops, pl in plans:
        grid = pl.grid_x * pl.grid_y * pl.grid_z
        assert grid == pl.work_items * pl.splits, tag           # grid_x/y/z stay the tile grid
        persistent = pl.ctas < grid
        assert persistent == _eligible(pl), f"{tag}: bn {pl.bn} a_mode {pl.a_mode} splits {pl.splits} tiles {pl.work_items} ctas {pl.ctas}"
        flops_all += flops
        if persistent:
            n_persist += 1
            flops_persist += flops
            assert pl.ctas == SMS, tag
            assert pl.stages >= 2 and pl.smem_bytes <= 227 * 1024, tag
        else:
            assert pl.ctas == grid, tag
    if (size, B) == ("l", 16):
        # the multi-wave 128 x 128 launches carry almost all of the step's work
        assert n_persist == 101 and flops_persist > 0.9 * flops_all, (n_persist, flops_persist / flops_all)
    else:
        assert n_persist == 0
