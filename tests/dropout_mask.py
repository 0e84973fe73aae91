"""The counter-based dropout masks restated on the host (test helper): csrc/ptx.cuh's dropout_hash and attn_keep, and the
element-wise keep test of csrc/train.cu's eltwise_kernel, bit for bit (tests/test_dropout_mask_cpu.py compiles the source's
own functions and compares).

Torch int64 arithmetic on any device: every 32-bit product is formed from 16-bit halves, so that no intermediate exceeds
2^49, and every step is reduced mod 2^32.  The keep test is the kernels' fp32 compare, float32(h >> 8) * 2^-24 >= float32(p):
the left side is exact in fp32 and p reaches the kernels as a C float."""
from __future__ import annotations

import numpy as np
import torch

M32 = 0xFFFFFFFF


def _mul(a: torch.Tensor, c: int) -> torch.Tensor:
    """a * c mod 2^32, a int64 in [0, 2^32), c a 32-bit constant."""
    return ((a & 0xFFFF) * c + (((a >> 16) * (c & 0xFFFF)) << 16)) & M32


def dropout_hash(a, b, c) -> torch.Tensor:
    """dropout_hash(a, b, c) of broadcastable int64 tensors (each taken mod 2^32)."""
    a, b, c = (torch.as_tensor(t, dtype=torch.int64) & M32 for t in (a, b, c))
    h = _mul(a, 0x9E3779B1) ^ _mul((b + 0x7F4A7C15) & M32, 0x85EBCA77) ^ _mul((c + 0x165667B1) & M32, 0xC2B2AE3D)
    h = h ^ (h >> 15)
    h = _mul(h, 0x2C1B3C6D)
    h = h ^ (h >> 12)
    h = _mul(h, 0x297A2D39)
    return h ^ (h >> 15)


def f32(p: float) -> float:
    """p rounded to fp32, as the C ABI receives it."""
    return float(np.float32(p))


def keep(h: torch.Tensor, p: float) -> torch.Tensor:
    return (h >> 8).to(torch.float32) * 2.0 ** -24 >= f32(p)


def attn_keep(seed: int, dir, bh, q, k, p: float) -> torch.Tensor:
    """attn_keep(seed, dir, bh, q, k, p) over broadcastable int64 tensors dir, bh, q, k."""
    q, k = torch.as_tensor(q, dtype=torch.int64), torch.as_tensor(k, dtype=torch.int64)
    a = ((q & M32) * 65536 + (k & 0xFFFF)) & M32
    b = (torch.as_tensor(bh, dtype=torch.int64) * 2 + torch.as_tensor(dir, dtype=torch.int64) + ((k & M32) >> 16) * 0x10001) & M32
    return keep(dropout_hash(a, b, torch.tensor(seed & M32, device=a.device)), p)


def attn_keep_mask(seed: int, offset: int, B: int, heads: int, N: int, p: float, device="cpu") -> torch.Tensor:
    """Keep mask of the cross-attention probabilities, bool (2 directions, B * heads, N queries, N keys).  Direction 0 is the
    RGB output (IR queries on RGB keys), direction 1 the IR output; `offset` is the device-side seed offset."""
    r = torch.arange(N, dtype=torch.int64, device=device)
    d = torch.arange(2, dtype=torch.int64, device=device).view(2, 1, 1, 1)
    bh = torch.arange(B * heads, dtype=torch.int64, device=device).view(1, -1, 1, 1)
    return attn_keep((seed + offset) & M32, d, bh, r.view(1, 1, N, 1), r.view(1, 1, 1, N), p)


def eltwise_keep(n: int, seed: int, offset: int, p: float, device="cpu", first: int = 0) -> torch.Tensor:
    """Keep mask of icaf_eltwise's dropout (mode 2) over elements first .. first + n - 1, bool (n,)."""
    idx = torch.arange(first, first + n, dtype=torch.int64, device=device)
    return keep(dropout_hash(idx & M32, idx >> 32, torch.tensor((seed + offset) & M32, device=device)), p)


def eltwise_dropout(x: torch.Tensor, keep_mask: torch.Tensor, p: float) -> torch.Tensor:
    """icaf_eltwise mode 2 on fp16 x: fp16(fp32(x) / (1 - fp32(p))) where kept, +0 where dropped."""
    kept = (x.float() / float(np.float32(1) - np.float32(p))).half()
    return torch.where(keep_mask.view(x.shape), kept, torch.zeros_like(kept))
