"""Shared helpers for the parity tests (test infrastructure)."""
from __future__ import annotations

import numpy as np
import torch

from oracle import synth


from icafusion_b200.synth import load_synth  # noqa: E402,F401  (same loader the benchmark uses)


def nhwc(x_nchw: torch.Tensor) -> torch.Tensor:
    return x_nchw.permute(0, 2, 3, 1).contiguous()


def nchw(x_nhwc: torch.Tensor) -> torch.Tensor:
    return x_nhwc.permute(0, 3, 1, 2).contiguous()


def sm_count() -> int:
    """SM count of the current CUDA device."""
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def conv_plan(fn):
    """The icaf_conv2d_plan of the one conv launch `fn` makes, on this device."""
    import ctypes
    from icafusion_b200 import _lib, ops
    with ops.dry_run() as dr:
        fn()
    (_, _, work), = dr.records
    pl = _lib.ConvPlan()
    assert _lib.lib().icaf_conv2d_plan(ctypes.byref(work["geom"]), work["n_io"], sm_count(), 0, ctypes.byref(pl)) == 0
    return pl


def err(a, b) -> float:
    """max|a-b| / max|b|"""
    a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float32)
    b = b.detach().float().cpu().numpy() if torch.is_tensor(b) else np.asarray(b, dtype=np.float32)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.isfinite(a).all(), "non-finite values in the CUDA result"
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max() / max(np.abs(b).max(), 1e-30))
