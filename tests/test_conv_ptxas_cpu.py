"""ptxas report of the conv kernels (cross-compiled for sm_90a, no GPU needed): no wgmma is serialised (warning C7510, which
a call such as printf reachable from a wgmma kernel causes) and no conv_gemm kernel spills registers."""
import os
import re
import shutil
import subprocess

import pytest

from icafusion_b200 import build as B


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_conv_kernels_unserialised_and_spill_free(tmp_path):
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "conv_gemm.cu"), "-o", str(tmp_path / "conv_gemm.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    assert "C7510" not in log, [l for l in log.splitlines() if "C7510" in l]
    # "Compiling entry function '<mangled>' for 'sm_90a'", then "... N bytes spill stores, M bytes spill loads"
    conv, entry = [], None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and entry and "conv_gemm_" in entry:
            conv.append((entry, int(m.group(1)), int(m.group(2))))
            entry = None
    # 6 one-tile instantiations (BN 32 / 64 / 128 x XM), 2 persistent ones and the CUDA-core reference
    assert len(conv) == 9, log
    spilling = [(k, st, ld) for k, st, ld in conv if st or ld]
    assert not spilling, spilling
