"""Every launch reports its own result.  Where the CUDA runtime sees no device, an entry point whose arguments pass
validation fails at its launch: it returns ICAF_ERR_CUDA with the entry's label in icaf_last_error(), and the launch
tally behind bench.py's `gpu_launches` does not count the refused launch."""
import ctypes

import pytest

ICAF_ERR_CUDA = 3


@pytest.fixture
def lib_without_device():
    from icafusion_b200 import _lib
    L = _lib.lib()
    if L.icaf_sm_count() >= 0:
        pytest.skip("the runtime sees a CUDA device: these calls would launch kernels on dummy pointers")
    return L


def test_single_launch_reports_its_own_failure(lib_without_device):
    L = lib_without_device
    p = ctypes.c_void_p(16)                       # never dereferenced: no kernel can run
    n0 = L.icaf_kernel_launches()
    assert L.icaf_upsample2x(p, 64, p, 64, 1, 4, 4, 64, None) == ICAF_ERR_CUDA
    assert L.icaf_last_error().startswith(b"upsample2x: ")
    assert L.icaf_kernel_launches() == n0


def test_first_of_two_launches_stops_the_entry(lib_without_device):
    L = lib_without_device
    p = ctypes.c_void_p(16)
    n0 = L.icaf_kernel_launches()
    assert L.icaf_colsum(p, 100, 64, p, 1.0, 0, p, 64 * 64 * 4, None) == ICAF_ERR_CUDA
    assert L.icaf_last_error().startswith(b"colsum(partial): ")
    assert L.icaf_kernel_launches() == n0
