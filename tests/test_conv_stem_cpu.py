"""Host-only checks of the image-stem conv kernel (conv_stem_kernel): which launches the dispatcher sends to it, the plan
icaf_conv2d_plan reports for them (one tile per CTA, BN 64, cp.async gather, one stage, the kernel's shared memory),
and its ptxas report (cross-compiled for sm_90a: no spills, and few enough registers for four CTAs per SM)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from icafusion_b200 import build as B

SMS = 132


def _plan(B_, H, W, Cin, Cout, k=3, s=1, p=1, n_io=2, act=1, epi=0):
    """Plan of a conv over a (B_, H, W, Cin) map whose filter is packed as pack_conv_weight does."""
    from icafusion_b200 import _lib
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    g = _lib.ConvGeom(B_, H, W, Cin, Ho, Wo, Cout, k, k, s, p, (k * k * Cin + 63) // 64 * 64, (Cout + 31) // 32 * 32, act, epi)
    pl = _lib.ConvPlan()
    L = _lib.lib()
    assert L.icaf_conv2d_plan(ctypes.byref(g), n_io, SMS, 0, ctypes.byref(pl)) == 0, L.icaf_last_error().decode()
    return pl


def _stem_smem(Wo):
    """The kernel's layout: three 8 KB filter boxes, 1 KB for the bias and the mbarrier, then the halo -- runs x 3 input
    rows x (min(Wo, 128) + 2) pixels of 32 bytes, or the 16 KB output tile if that is larger -- and 1 KB of alignment
    slack."""
    runs = 1 + -(-127 // Wo)
    halo = runs * 3 * (min(Wo, 128) + 2) * 32
    return 3 * 8192 + 1024 + max(halo, 16384) + 1024


@pytest.mark.parametrize("Cout", [64, 48])
def test_yolov5_stem_plan(Cout):
    """yolov5l (N = 64) and yolov5m (N = 48) stems at batch 16: 16 x 256 x 320 space-to-depth frames, both streams."""
    pl = _plan(16, 256, 320, 16, Cout)
    got = {f: getattr(pl, f) for f in ("kernel", "bn", "a_mode", "halo", "splits", "cluster", "stages", "grid_x", "grid_y",
                                       "grid_z", "work_items", "ctas", "smem_bytes")}
    assert got == dict(kernel=0, bn=64, a_mode=0, halo=0, splits=1, cluster=1, stages=1, grid_x=10240, grid_y=1, grid_z=2,
                       work_items=20480, ctas=20480, smem_bytes=_stem_smem(320)), got
    assert _stem_smem(320) == 51584 and 4 * (51584 + 1024) <= 228 * 1024      # four CTAs per SM


@pytest.mark.parametrize("H,W", [(50, 36), (40, 1), (64, 127), (132, 132)])
def test_stem_plan_smem_follows_the_map_width(H, W):
    """Narrow maps take more, shorter runs per tile; the halo (or the output tile) sizes the shared memory."""
    pl = _plan(400, H, W, 16, 64)
    assert (pl.bn, pl.a_mode, pl.stages, pl.smem_bytes) == (64, 0, 1, _stem_smem(W))
    assert pl.smem_bytes <= 64 * 1024


def test_other_launches_keep_their_kernels():
    """BN = 32 stems (yolov5s / n), residual launches and other channel counts or strides stay on the one-tile kernel."""
    from icafusion_b200 import _lib
    assert _plan(16, 256, 320, 16, 32).stages > 1                                  # yolov5s stem: BN 32
    assert _plan(16, 256, 320, 16, 64, epi=_lib.EPI_ADD_RES).stages > 1           # residual
    assert _plan(16, 256, 320, 32, 64).stages > 1                                  # 32 channels
    assert _plan(16, 256, 320, 16, 64, s=2).stages > 1                             # stride 2


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_stem_kernel_spill_free(tmp_path):
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "conv_gemm.cu"), "-o", str(tmp_path / "conv_gemm.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = (out.stdout + out.stderr).splitlines()
    i = next(i for i, line in enumerate(log) if re.search(r"Compiling entry function '\w*conv_stem_kernel\w*'", line))
    report = " ".join(log[i + 1:i + 4])
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    regs = re.search(r"Used (\d+) registers", report)
    assert spills and regs, report
    assert spills.groups() == ("0", "0"), report
    assert int(regs.group(1)) <= 128, report                  # 4 CTAs of 128 threads per SM
