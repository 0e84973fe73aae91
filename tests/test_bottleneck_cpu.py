"""The fused Bottleneck (bottleneck.cu, ops.bottleneck) without a GPU: its kernel compiles for sm_90a without spills or
serialised wgmmas, the detector forwards send exactly the P2 Bottlenecks of yolov5l to it, and the entry point refuses
overlapping input and output maps before it touches CUDA."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from icafusion_b200 import build as B


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_bottleneck_kernel_unserialised_and_spill_free(tmp_path):
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "bottleneck.cu"), "-o", str(tmp_path / "bottleneck.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    assert "C7510" not in log, [l for l in log.splitlines() if "C7510" in l]
    spills = [(int(a), int(b)) for a, b in re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)]
    assert len(spills) == 1 and spills[0] == (0, 0), log


def _records(size, B):
    from icafusion_b200 import Model, ops
    m = Model(f"yolov5{size}_Transfusion_kaist").eval().fuse().half()
    rgb = torch.empty(B, 3, 512, 640, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run() as dr:
        m(rgb, rgb)
    return [(name, work) for name, _, work in dr.records]


def test_dry_run_fuses_the_p2_bottlenecks_of_yolov5l():
    fused = [w for n, w in _records("l", 16) if n == "icaf_bottleneck_fwd"]
    # the three Bottlenecks of the P2 C3 (128 x 160, 64 channels), RGB and IR grouped
    assert [w["tag"] for w in fused] == ["bottleneck M327680 C64 x2"] * 3
    patches = 16 * 32 * 5
    assert fused[0]["flops"] == 2 * 2.0 * 64 * (204 * 64 + 128 * 576) * patches
    assert fused[0]["bytes"] == 2 * 2.0 * (2 * 327680 * 64 + 64 * 64 + 64 * 576)


def test_dry_run_fused_launches_replace_two_conv_launches_each():
    from icafusion_b200 import common
    l16 = _records("l", 16)
    n_conv = sum(n == "icaf_conv2d_fwd" for n, _ in l16)
    orig = common.Bottleneck.fusable
    try:
        common.Bottleneck.fusable = staticmethod(lambda mods, xs, outs=None: False)
        n_conv_unfused = sum(n == "icaf_conv2d_fwd" for n, _ in _records("l", 16))
    finally:
        common.Bottleneck.fusable = orig
    assert n_conv_unfused - n_conv == 6


def test_dry_run_yolov5s_b1_keeps_the_two_launch_path():
    # its only 64-channel Bottlenecks (P3, 64 x 80) have too few patches to fill the GPU
    assert not any(n == "icaf_bottleneck_fwd" for n, _ in _records("s", 1))


def test_entry_point_refuses_overlapping_maps_and_bad_counts():
    from icafusion_b200 import _lib
    L = _lib.lib()
    base = 1 << 20
    io = (_lib.BottleneckIO * 2)()
    for i in range(2):
        io[i].x, io[i].x_ld = base + i * (1 << 24), 64
        io[i].w1, io[i].b1, io[i].w3, io[i].b2 = base + (1 << 28), base + (1 << 28), base + (1 << 28), base + (1 << 28)
    io[0].y, io[0].y_ld = base + 64 * 64 * 2, 64                 # inside problem 0's input
    io[1].y, io[1].y_ld = base + (1 << 26), 64
    assert L.icaf_bottleneck_fwd(2, 32, 64, io, 2, None) == 1 and b"overlap" in L.icaf_last_error()
    io[0].y = base + (1 << 24) - 16                              # ends inside problem 1's input
    assert L.icaf_bottleneck_fwd(2, 32, 64, io, 2, None) == 1 and b"overlap" in L.icaf_last_error()
    assert L.icaf_bottleneck_fwd(2, 32, 64, io, 3, None) == 1
    io[0].y, io[0].x_ld = base + (1 << 25), 60
    assert L.icaf_bottleneck_fwd(2, 32, 64, io, 2, None) == 1 and b"aligned" in L.icaf_last_error()
