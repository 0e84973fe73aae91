"""Flash cross-attention (wgmma) vs the CPU oracle and vs the on-device CUDA-core reference."""
import math

import pytest
import torch

from helpers import err

pytestmark = pytest.mark.gpu
TOL = 1e-3   # the north-star tolerance: P is rounded to fp16 before the PV MMA (as in the reference's fp16 path) + fp16 output;
             # observed 4e-4 .. 9e-4 (printed per case)


def _oracle(qk_q, qk_k, vt, B, N, n_pad, C, h):
    """softmax(q k^T / sqrt(d)) v per head (common.py:670-684), q from one modality, k/v from the other."""
    d = C // h
    q = qk_q[:, :N, :C].float().reshape(B, N, h, d).permute(0, 2, 1, 3)
    k = qk_k[:, :N, C:].float().reshape(B, N, h, d).permute(0, 2, 1, 3)
    v = vt.float().reshape(C, B, n_pad)[:, :, :N].permute(1, 0, 2).reshape(B, h, d, N).permute(0, 1, 3, 2)
    att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), -1)
    return (att @ v).permute(0, 2, 1, 3).reshape(B, N, C)


@pytest.mark.parametrize("B,N,C", [(2, 100, 128), (1, 256, 256), (1, 400, 128), (1, 400, 512), (2, 100, 1024), (1, 1280, 256),
                                   (1, 77, 128)])
def test_cross_attention(cuda_device, B, N, C):
    from icafusion_b200 import ops
    h = 8
    n_pad = ops.round_up(N, 8)
    g = torch.Generator().manual_seed(7)
    qk_v, qk_i = torch.randn(B, n_pad, 2 * C, generator=g).half(), torch.randn(B, n_pad, 2 * C, generator=g).half()
    vt_v, vt_i = torch.randn(C, B * n_pad, generator=g).half(), torch.randn(C, B * n_pad, generator=g).half()
    args = [t.to(cuda_device) for t in (qk_v, qk_i, vt_v, vt_i)]
    o_v, o_i = ops.cross_attention(*args, B, N, n_pad, C, h)
    s_v, s_i = ops.cross_attention(*args, B, N, n_pad, C, h, simt=True)
    torch.cuda.synchronize()
    r_v = _oracle(qk_i, qk_v, vt_v, B, N, n_pad, C, h)      # RGB output: IR queries on RGB keys/values (common.py:670,682)
    r_i = _oracle(qk_v, qk_i, vt_i, B, N, n_pad, C, h)
    es, eo = max(err(s_v[:, :N], r_v), err(s_i[:, :N], r_i)), max(err(o_v[:, :N], r_v), err(o_i[:, :N], r_i))
    print(f"\n[attention B{B} N{N} C{C} d{C // h}] wgmma {eo:.2e}  cuda-core {es:.2e}  (tol {TOL:.0e})")
    assert es < TOL, "CUDA-core reference disagrees with the oracle"
    assert eo < TOL
    if n_pad > N:
        assert float(o_v[:, N:].abs().max()) == 0 and float(o_i[:, N:].abs().max()) == 0    # pad rows stay finite (zero)


@pytest.mark.parametrize("B,N,C", [(2, 100, 128), (1, 400, 256), (1, 256, 512), (2, 100, 1024), (1, 1280, 128), (1, 77, 256)])
def test_cross_attention_fused_qkv(cuda_device, B, N, C):
    """Fused form: one (B, Npad, 3C) [q|k|v] matrix per modality; V tiles are consumed as MN-major UMMA operands."""
    from icafusion_b200 import ops
    h = 8
    n_pad = ops.round_up(N, 8)
    g = torch.Generator().manual_seed(11)
    qkv_v, qkv_i = torch.randn(B, n_pad, 3 * C, generator=g).half(), torch.randn(B, n_pad, 3 * C, generator=g).half()
    args = [qkv_v.to(cuda_device), qkv_i.to(cuda_device), None, None]
    o_v, o_i = ops.cross_attention(*args, B, N, n_pad, C, h)
    s_v, s_i = ops.cross_attention(*args, B, N, n_pad, C, h, simt=True)
    torch.cuda.synchronize()

    def vt(t):      # (B, Npad, C) value rows -> the split form's (C, B*Npad) layout the oracle helper expects
        return t[:, :, 2 * C:].permute(2, 0, 1).reshape(C, B * n_pad).contiguous()
    r_v = _oracle(qkv_i[:, :, :2 * C], qkv_v[:, :, :2 * C], vt(qkv_v), B, N, n_pad, C, h)
    r_i = _oracle(qkv_v[:, :, :2 * C], qkv_i[:, :, :2 * C], vt(qkv_i), B, N, n_pad, C, h)
    es, eo = max(err(s_v[:, :N], r_v), err(s_i[:, :N], r_i)), max(err(o_v[:, :N], r_v), err(o_i[:, :N], r_i))
    print(f"\n[attention fused-qkv B{B} N{N} C{C} d{C // h}] wgmma {eo:.2e}  cuda-core {es:.2e}  (tol {TOL:.0e})")
    assert es < TOL, "CUDA-core reference disagrees with the oracle"
    assert eo < TOL
