"""Tensor-level wrappers over the C ABI: torch tensors in, torch tensors out, kernels on the current stream.

Activations are fp16 NHWC tensors (shape (B,H,W,C)); a channel slice ``t[..., a:b]`` of a
contiguous tensor is a valid "view" (pixel pitch = t.stride(2)).  PyTorch only provides device
memory and the stream here -- every computation is a kernel from libicaf_b200.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, fields
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import (ACT_GELU, ACT_NONE, ACT_SILU, EPI_ADD_RES, EPI_BIAS_ROW, EPI_EMIT_STATS, EPI_LN_FOLD,  # noqa: F401
                   EPI_SCALED_RES)


_PROFILE = None        # when a list: every call appends (name, work dict, start event, end event)


def launch_count() -> int:
    """Kernels of libicaf_b200 enqueued so far (the library's own tally: a C-ABI call may launch more than one)."""
    return int(_lib.lib().icaf_kernel_launches())


class profile:
    """Context manager: time every libicaf_b200 launch with CUDA events on its stream.  One event is recorded after
    each launch; a launch's duration is the gap to the previous event (so with the launches queued back to back it is
    kernel time + inter-kernel gap).  Use on a single stream: `with ops.profile() as p: ...; torch.cuda.synchronize()`."""

    def __enter__(self):
        global _PROFILE
        self.records = []
        _PROFILE = self
        self.last = None
        return self

    def __exit__(self, *a):
        global _PROFILE
        _PROFILE = None

    def mark(self):
        """Start a new timing chain (call after queueing work that must not be attributed to the next launch)."""
        self.last = torch.cuda.Event(enable_timing=True)
        self.last.record()

    def per_launch(self):
        """[(name, tag, ms, flops, bytes)] in launch order (call after a device synchronize)."""
        return [(n, w.get("tag", ""), e0.elapsed_time(e1), w.get("flops", 0.0), w.get("bytes", 0.0)) for n, w, e0, e1 in self.records]

    def summary(self):
        out = {}
        for name, work, e0, e1 in self.records:
            d = out.setdefault(name, {"launches": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            d["launches"] += 1
            d["ms"] += e0.elapsed_time(e1)
            d["flops"] += work.get("flops", 0.0)
            d["bytes"] += work.get("bytes", 0.0)
        return out


_DRY = None            # when a list: no kernel is launched; every C-ABI call is recorded as (name, args, work)


class dry_run:
    """Context manager: walk the product path without a GPU.  Tensors live on the ``meta`` device (shapes and strides
    only), packed filters stay where the module is (CPU), and every C-ABI call is recorded instead of launched:
    ``records`` = [(entry point, ctypes args, work dict)].  Convolution records keep their ``ConvGeom`` so a test can feed
    the exact geometries of a model to ``icaf_conv2d_plan`` (tests/test_abi_cpu.py)."""

    def __enter__(self):
        global _DRY
        self.records = []
        _DRY = self.records
        return self

    def __exit__(self, *a):
        global _DRY
        _DRY = None


def dry_running() -> bool:
    return _DRY is not None


_SM_TARGET = 0         # the library's icaf_set_sm_count_target, as last set through sm_count_target


class sm_count_target:
    """Context manager: every launch planned inside plans for min(n, SM count of the device) SMs (icaf_set_sm_count_target),
    as it would on a part or MIG slice with that many SMs; n = 0 plans for the device's own count.  The previous target is
    restored on exit.  Process-wide, and read when a call plans its launch: graphs captured earlier keep their plans."""

    def __init__(self, n: int):
        self.n = int(n)

    def __enter__(self):
        global _SM_TARGET
        _lib.check(_lib.lib().icaf_set_sm_count_target(self.n), "icaf_set_sm_count_target")
        self.prev, _SM_TARGET = _SM_TARGET, self.n
        return self

    def __exit__(self, *a):
        global _SM_TARGET
        _lib.check(_lib.lib().icaf_set_sm_count_target(self.prev), "icaf_set_sm_count_target")
        _SM_TARGET = self.prev


def on_device(t: torch.Tensor) -> bool:
    """True for CUDA tensors (and for anything while a dry run is recording: meta activations, CPU-resident filters)."""
    return t.is_cuda or _DRY is not None


_WEIGHT_TRACE = None   # when a list: (container, key) of every weight tensor a forward consumes


def note_weight(container, key) -> None:
    if _WEIGHT_TRACE is not None:
        _WEIGHT_TRACE.append((container, key))


class trace_weights:
    """Context manager: record which packed weight tensors a forward touches (for consolidate_weights)."""

    def __enter__(self):
        global _WEIGHT_TRACE
        self.items = []
        _WEIGHT_TRACE = self.items
        return self

    def __exit__(self, *a):
        global _WEIGHT_TRACE
        _WEIGHT_TRACE = None


def consolidate_weights(items):
    """Move every traced weight tensor into one contiguous fp16 arena (in use order) and rebind its owner to the arena
    view; returns the arena.  One arena = one L2 prefetch per step and sequential DRAM pages for the filter stream."""
    seen, uniq = set(), []
    for cont, key in items:
        k = (id(cont), key)
        if k not in seen:
            seen.add(k)
            uniq.append((cont, key))
    def get(cont, key):
        return cont[key] if isinstance(cont, dict) else getattr(cont, key)
    sizes = [round_up(get(c, k).numel(), 128) for c, k in uniq]
    dev = get(*uniq[0]).device
    arena = torch.zeros(sum(sizes), dtype=torch.float16, device=dev)
    off = 0
    for (cont, key), sz in zip(uniq, sizes):
        t = get(cont, key)
        assert t.dtype == torch.float16 and t.is_contiguous()
        view = arena[off:off + t.numel()].view(t.shape)
        view.copy_(t)
        if isinstance(cont, dict):
            cont[key] = view
        else:
            setattr(cont, key, view)
        off += sz
    return arena


def prefetch_l2(t: torch.Tensor) -> None:
    _call("icaf_prefetch_l2", _lib.lib().icaf_prefetch_l2, (_ptr(t), t.numel() * t.element_size()),
          {"bytes": float(t.numel() * t.element_size())})


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name: str, fn, args, work=None):
    """Invoke one C-ABI kernel launcher on the current stream (optionally event-bracketed)."""
    if _DRY is not None:
        _DRY.append((name, args, work or {}))
        return
    if _PROFILE is not None:
        if _PROFILE.last is None:
            _PROFILE.mark()
        rc = fn(*args, _stream())
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        _PROFILE.records.append((name, work or {}, _PROFILE.last, e1))
        _PROFILE.last = e1
    else:
        rc = fn(*args, _stream())
    _lib.check(rc, name)


def _check_view(t: torch.Tensor, what: str) -> int:
    """Validate an fp16 NHWC view and return its pixel pitch (elements)."""
    if t.dtype != torch.float16 or not on_device(t) or t.dim() != 4:
        raise ValueError(f"{what}: expected a CUDA fp16 (B,H,W,C) tensor, got {t.dtype} {tuple(t.shape)} on {t.device}")
    B, H, W, Cc = t.shape
    ld = t.stride(2) if W > 1 else (t.stride(1) if H > 1 else (t.stride(0) if B > 1 else Cc))
    ok = t.stride(3) == 1 and (W == 1 or t.stride(2) == ld) and (H == 1 or t.stride(1) == W * ld) and \
        (B == 1 or t.stride(0) == H * W * ld)
    if not ok:
        raise ValueError(f"{what}: not a dense NHWC view (shape {tuple(t.shape)}, strides {t.stride()})")
    return ld


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


@dataclass
class PackedConv:
    """Filter bank in the layout the implicit-GEMM kernel consumes: fp16 [w_rows][k_pad], K order (ky,kx,c)."""
    w: torch.Tensor
    bias: Optional[torch.Tensor]      # fp32 [Cout]
    cin: int                          # channels consumed per tap (4 for the packed image)
    cout: int
    kh: int
    kw: int
    stride: int
    pad: int
    act: int
    is_weight: bool = True            # False when the "filter" operand is an activation (swap-AB linears)
    colsum: Optional[torch.Tensor] = None   # LN fold (pack_linear_ln): fp32 [w_rows] row sums of the gamma-folded fp16 filter
    ln_eps: float = 0.0


def copy_packed_(old, new, what: str = "packed weights"):
    """Copy a fresh pack `new` into the cached pack `old`, tensor by tensor, and return `old`.  Both are a PackedConv, a
    tensor, or a dict / tuple / list of them.  No tensor is rebound, so every address a launch, a tensor map or a captured
    CUDA graph holds stays valid.  Raises ValueError where a shape, dtype, stride, device or non-tensor field differs."""
    if isinstance(old, PackedConv) and isinstance(new, PackedConv):
        for f in fields(PackedConv):
            a, b = getattr(old, f.name), getattr(new, f.name)
            if torch.is_tensor(a) or torch.is_tensor(b):
                copy_packed_(a, b, f"{what}.{f.name}")
            elif a != b:
                raise ValueError(f"{what}: {f.name} changed from {a!r} to {b!r}; the pack cannot be refreshed in place")
    elif isinstance(old, dict) and isinstance(new, dict) and old.keys() == new.keys():
        for k in old:
            copy_packed_(old[k], new[k], f"{what}[{k!r}]")
    elif isinstance(old, (tuple, list)) and type(old) is type(new) and len(old) == len(new):
        for i, (a, b) in enumerate(zip(old, new)):
            copy_packed_(a, b, f"{what}[{i}]")
    elif torch.is_tensor(old) and torch.is_tensor(new):
        if (old.shape, old.dtype, old.stride(), old.device) != (new.shape, new.dtype, new.stride(), new.device):
            raise ValueError(f"{what}: {new.dtype} {tuple(new.shape)} strides {new.stride()} on {new.device} does not fit the "
                             f"cached {old.dtype} {tuple(old.shape)} strides {old.stride()} on {old.device}")
        if old.device.type != "meta" and old.data_ptr() != new.data_ptr():   # a bias may be the parameter itself
            old.copy_(new)
    elif old is not None or new is not None:
        raise ValueError(f"{what}: {type(new).__name__} does not fit the cached {type(old).__name__}")
    return old


def pack_conv_weight(weight: torch.Tensor, bias: Optional[torch.Tensor], stride: int, pad: int, act: int,
                     device=None) -> PackedConv:
    """(Cout,Cin,kh,kw) fp32 filter (BN already folded) -> PackedConv.  A 3-channel filter is padded to 4
    input channels to match the packed image layout (icaf_pack_image)."""
    cout, cin, kh, kw = weight.shape
    w = weight.detach().float()
    if cin == 3:
        w = torch.cat([w, w.new_zeros(cout, 1, kh, kw)], 1)
        cin = 4
    if not (cin == 4 or cin % 8 == 0):
        raise ValueError(f"conv input channels must be 3/4 or a multiple of 8, got {cin}")
    K = kh * kw * cin
    k_pad, rows = round_up(K, 64), round_up(cout, 32)
    m = w.permute(0, 2, 3, 1).reshape(cout, K)
    out = torch.zeros(rows, k_pad, dtype=torch.float16, device=device or weight.device)
    out[:cout, :K] = m.to(out.device, torch.float16)
    b = None if bias is None else bias.detach().float().to(out.device).contiguous()
    return PackedConv(out, b, cin, cout, kh, kw, stride, pad, act)


def pack_linear(weight: torch.Tensor, bias: Optional[torch.Tensor], act: int = ACT_NONE, device=None) -> PackedConv:
    """nn.Linear weight (out,in) as a 1x1 filter bank."""
    return pack_conv_weight(weight.detach()[:, :, None, None], bias, 1, 0, act, device)


def _addr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    return 0 if t.device.type == "meta" else t.data_ptr()


def pack_linear_ln(weight: torch.Tensor, bias: Optional[torch.Tensor], ln_weight: torch.Tensor, ln_bias: torch.Tensor,
                   ln_eps: float, act: int = ACT_NONE, device=None) -> PackedConv:
    """nn.Linear applied to nn.LayerNorm(x) (common.py:660-668, 749-750 + 704), LayerNorm folded into the GEMM:
    filter W diag(gamma), bias b + W beta, colsum[n] = sum_k fp16(W'[n][k]) -- the kernel normalises in its epilogue
    (ICAF_EPI_LN_FOLD, include/icaf_b200.h)."""
    w = weight.detach().float()
    wf = w * ln_weight.detach().float()[None, :]
    b = (bias.detach().float() if bias is not None else torch.zeros(w.shape[0], device=w.device)) + w @ ln_bias.detach().float()
    pk = pack_conv_weight(wf[:, :, None, None], b, 1, 0, act, device)
    pk.colsum = pk.w.float().sum(1).contiguous()                # of the ROUNDED filter: the identity holds for what the MMA sees
    pk.ln_eps = float(ln_eps)
    return pk


def row_stats(x0: torch.Tensor, x1: Optional[torch.Tensor] = None):
    """(sum, sum of squares) per row of (rows, C) fp16 matrices -> fp32 (rows, 1, 2) each (ln_parts = 1)."""
    rows, Cc = x0.shape
    assert x0.is_contiguous() and x0.dtype == torch.float16 and (x1 is None or (x1.shape == x0.shape and x1.is_contiguous()))
    s0 = torch.empty(rows, 1, 2, dtype=torch.float32, device=x0.device)
    s1 = torch.empty_like(s0) if x1 is not None else None
    _call("icaf_row_stats", _lib.lib().icaf_row_stats, (_ptr(x0), _ptr(x1), _ptr(s0), _ptr(s1), rows, Cc),
          {"bytes": 2.0 * x0.numel() * (2 if x1 is not None else 1)})
    return (s0, s1) if x1 is not None else s0


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(_addr(t) or 0)


def conv2d(xs: Sequence[torch.Tensor], packs: Sequence[PackedConv], outs: Optional[Sequence[torch.Tensor]] = None,
           res: Optional[Sequence[torch.Tensor]] = None, scaled: Optional[Sequence] = None,
           bias_row: bool = False, simt: bool = False, ln_stats: Optional[Sequence[torch.Tensor]] = None,
           stats_out: Optional[Sequence[torch.Tensor]] = None) -> List[torch.Tensor]:
    """Grouped (1 or 2 problems of identical geometry) Conv+bias+act(+residual).
    `scaled`: per problem (alpha, beta) device fp32 scalars -> y = alpha*res + beta*(acc+bias).
    `ln_stats`: per problem fp32 (M, parts, 2) row statistics of the input -> LayerNorm-folded linear (packs from
    pack_linear_ln).  `stats_out`: per problem fp32 (M, ceil(Cout/32), 2) receiving the row statistics of the output
    (with `scaled` only)."""
    n = len(xs)
    assert n in (1, 2) and len(packs) == n
    p0 = packs[0]
    B, Hi, Wi, Cx = xs[0].shape
    if Cx != p0.cin:
        raise ValueError(f"conv2d: input has {Cx} channels, filter expects {p0.cin}")
    Ho = (Hi + 2 * p0.pad - p0.kh) // p0.stride + 1
    Wo = (Wi + 2 * p0.pad - p0.kw) // p0.stride + 1
    epi = (EPI_BIAS_ROW if bias_row else 0) | (EPI_SCALED_RES if scaled is not None else (EPI_ADD_RES if res is not None else 0)) | \
        (EPI_LN_FOLD if ln_stats is not None else 0) | (EPI_EMIT_STATS if stats_out is not None else 0)
    g = _lib.ConvGeom(B, Hi, Wi, p0.cin, Ho, Wo, p0.cout, p0.kh, p0.kw, p0.stride, p0.pad, p0.w.shape[1],
                      p0.w.shape[0], p0.act, epi)
    if outs is None:
        outs = [torch.empty(B, Ho, Wo, p0.cout, dtype=torch.float16, device=xs[0].device) for _ in range(n)]
    ios = (_lib.ConvIO * n)()
    for i in range(n):
        pk = packs[i]
        if pk.is_weight:
            note_weight(pk, "w")
        if (pk.cin, pk.cout, pk.kh, pk.kw, pk.stride, pk.pad, pk.act) != (p0.cin, p0.cout, p0.kh, p0.kw, p0.stride, p0.pad, p0.act) \
                or tuple(xs[i].shape) != tuple(xs[0].shape):
            raise ValueError("conv2d: grouped problems must share one geometry")
        if tuple(outs[i].shape) != (B, Ho, Wo, p0.cout):
            raise ValueError(f"conv2d: output shape {tuple(outs[i].shape)} != {(B, Ho, Wo, p0.cout)}")
        ios[i].x, ios[i].x_ld = _addr(xs[i]), _check_view(xs[i], "conv2d input")
        ios[i].w = _addr(pk.w)
        ios[i].bias = _addr(pk.bias)
        ios[i].y, ios[i].y_ld = _addr(outs[i]), _check_view(outs[i], "conv2d output")
        if res is not None:
            if tuple(res[i].shape) != (B, Ho, Wo, p0.cout):
                raise ValueError("conv2d: residual shape mismatch")
            ios[i].res, ios[i].res_ld = _addr(res[i]), _check_view(res[i], "conv2d residual")
        if scaled is not None:
            ios[i].alpha, ios[i].beta = _addr(scaled[i][0]), _addr(scaled[i][1])
        if ln_stats is not None:
            st = ln_stats[i]
            if pk.colsum is None or st.dtype != torch.float32 or st.dim() != 3 or st.shape[0] != B * Ho * Wo or st.shape[2] != 2 or \
                    not st.is_contiguous():
                raise ValueError("conv2d: ln_stats must be contiguous fp32 (M, parts, 2) and the filter packed by pack_linear_ln")
            ios[i].ln_stats, ios[i].ln_colsum, ios[i].ln_parts, ios[i].ln_eps = _addr(st), _addr(pk.colsum), st.shape[1], pk.ln_eps
        if stats_out is not None:
            so = stats_out[i]
            if tuple(so.shape) != (B * Ho * Wo, (p0.cout + 31) // 32, 2) or so.dtype != torch.float32 or not so.is_contiguous():
                raise ValueError(f"conv2d: stats_out must be contiguous fp32 {(B * Ho * Wo, (p0.cout + 31) // 32, 2)}")
            ios[i].stats_out = _addr(so)
    fn = _lib.lib().icaf_conv2d_fwd_simt if simt else _lib.lib().icaf_conv2d_fwd
    M = B * Ho * Wo
    kk = p0.kh * p0.kw * p0.cin
    work = {"tag": f"M{M} N{p0.cout} K{kk} k{p0.kh}s{p0.stride} x{n}" + (" +res" if res is not None else ""),
            "flops": 2.0 * M * p0.cout * kk * n,
            "bytes": 2.0 * n * (B * Hi * Wi * p0.cin + M * p0.cout * (2 if res is not None else 1) + p0.cout * kk)}
    work["geom"], work["n_io"] = g, n
    _call("icaf_conv2d_fwd_simt" if simt else "icaf_conv2d_fwd", fn, (C.byref(g), ios, n), work)
    return list(outs)


def linear(xs: Sequence[torch.Tensor], packs: Sequence[PackedConv], outs=None, res=None, scaled=None,
           bias_row: bool = False, simt: bool = False, ln_stats=None, stats_out=None) -> List[torch.Tensor]:
    """Rows-as-pixels view of conv2d: xs are (rows, K) fp16 matrices (row pitch = stride(0))."""
    def as4(t):
        return None if t is None else t.unflatten(0, (1, 1, t.shape[0])) if t.dim() == 2 else t
    o = conv2d([as4(x) for x in xs], packs, None if outs is None else [as4(t) for t in outs],
               None if res is None else [as4(t) for t in res], scaled, bias_row, simt, ln_stats, stats_out)
    return [t[0, 0] for t in o]


def bottleneck(xs: Sequence[torch.Tensor], p1s: Sequence[PackedConv], p3s: Sequence[PackedConv],
               outs: Optional[Sequence[torch.Tensor]] = None) -> List[torch.Tensor]:
    """Grouped (1 or 2 problems) Bottleneck with shortcut, 64 channels: y = x + cv2(cv1(x)) in one launch that keeps the
    hidden map on chip (icaf_bottleneck_fwd).  p1s: the packed 1x1 SiLU cv1 filters, p3s: the packed 3x3 / pad 1 SiLU cv2
    filters.  Outputs must not overlap the inputs."""
    n = len(xs)
    assert n in (1, 2) and len(p1s) == n and len(p3s) == n
    B, H, W, Cx = xs[0].shape
    for p1, p3 in zip(p1s, p3s):
        if (p1.cin, p1.cout, p1.kh, p1.stride, p1.pad, p1.act, tuple(p1.w.shape)) != (64, 64, 1, 1, 0, ACT_SILU, (64, 64)) or \
                (p3.cin, p3.cout, p3.kh, p3.kw, p3.stride, p3.pad, p3.act, tuple(p3.w.shape)) != (64, 64, 3, 3, 1, 1, ACT_SILU, (64, 576)) or \
                p1.bias is None or p3.bias is None:
            raise ValueError("bottleneck: needs a 64-channel 1x1 and a 3x3 / pad 1 filter, both with bias and SiLU")
    if outs is None:
        outs = [torch.empty(B, H, W, 64, dtype=torch.float16, device=xs[0].device) for _ in range(n)]
    ios = (_lib.BottleneckIO * n)()
    for i in range(n):
        if tuple(xs[i].shape) != (B, H, W, 64) or tuple(outs[i].shape) != (B, H, W, 64):
            raise ValueError(f"bottleneck: input {tuple(xs[i].shape)} / output {tuple(outs[i].shape)} must both be {(B, H, W, 64)}")
        note_weight(p1s[i], "w")
        note_weight(p3s[i], "w")
        ios[i].x, ios[i].x_ld = _addr(xs[i]), _check_view(xs[i], "bottleneck input")
        ios[i].y, ios[i].y_ld = _addr(outs[i]), _check_view(outs[i], "bottleneck output")
        ios[i].w1, ios[i].b1 = _addr(p1s[i].w), _addr(p1s[i].bias)
        ios[i].w3, ios[i].b2 = _addr(p3s[i].w), _addr(p3s[i].bias)
    M = B * H * W
    patches = B * ((H + 3) // 4) * ((W + 31) // 32)          # 4 x 32 output pixels each, cv1 recomputed on a 6 x 34 halo
    work = {"tag": f"bottleneck M{M} C64 x{n}",
            "flops": 2.0 * 64 * (6 * 34 * 64 + 128 * 9 * 64) * patches * n,
            "bytes": 2.0 * n * (2 * M * 64 + 64 * 64 + 64 * 576)}
    _call("icaf_bottleneck_fwd", _lib.lib().icaf_bottleneck_fwd, (B, H, W, ios, n), work)
    return list(outs)


def pack_stem_weight(weight: torch.Tensor, bias: Optional[torch.Tensor], act: int, device=None) -> "PackedConv":
    """(Cout,3,6,6) stride-2 pad-2 stem filter (BN folded) -> the equivalent 3x3 / stride 1 / pad 1 filter over the
    space-to-depth image (16 channels: (dy*2+dx)*4 + c), packed for the implicit-GEMM kernel.  ky = 2*ty+dy, kx = 2*tx+dx."""
    cout, cin, kh, kw = weight.shape
    assert (cin, kh, kw) == (3, 6, 6)
    w = weight.detach().float()
    w4 = torch.cat([w, w.new_zeros(cout, 1, 6, 6)], 1)                       # (n, c4, ky, kx)
    w4 = w4.view(cout, 4, 3, 2, 3, 2)                                        # (n, c, ty, dy, tx, dx)
    ws = w4.permute(0, 3, 5, 1, 2, 4).reshape(cout, 16, 3, 3)                # (n, (dy,dx,c), ty, tx)
    return pack_conv_weight(ws, bias, 1, 1, act, device)


def pack_image(img: torch.Tensor, scale: float = 1.0, s2d: bool = False) -> torch.Tensor:
    """(B,3,H,W) fp16 / fp32 / uint8 planar image -> (B,H,W,4) fp16, or with `s2d` -> (B,H/2,W/2,16) space-to-depth."""
    if img.dim() != 4 or img.shape[1] != 3 or not on_device(img):
        raise ValueError(f"pack_image: expected a CUDA (B,3,H,W) tensor, got {tuple(img.shape)}")
    code = {torch.float16: 0, torch.float32: 1, torch.uint8: 2}.get(img.dtype)
    if code is None:
        raise ValueError(f"pack_image: unsupported dtype {img.dtype}")
    img = img.contiguous()
    B, _, H, W = img.shape
    if s2d:
        out = torch.empty(B, H // 2, W // 2, 16, dtype=torch.float16, device=img.device)
        _call("icaf_pack_image", _lib.lib().icaf_pack_image_s2d, (_ptr(img), code, float(scale), B, H, W, _ptr(out)),
              {"bytes": float(img.numel() * img.element_size() + out.numel() * 2)})
        return out
    out = torch.empty(B, H, W, 4, dtype=torch.float16, device=img.device)
    _call("icaf_pack_image", _lib.lib().icaf_pack_image, (_ptr(img), code, float(scale), B, H, W, _ptr(out)),
          {"bytes": float(img.numel() * img.element_size() + out.numel() * 2)})
    return out


def sppf_pool(x: torch.Tensor, y1: torch.Tensor, y2: torch.Tensor, y3: torch.Tensor) -> None:
    B, H, W, Cc = x.shape
    ld = _check_view(y1, "sppf y1")
    assert _check_view(y2, "sppf y2") == ld and _check_view(y3, "sppf y3") == ld
    _call("icaf_sppf_pool", _lib.lib().icaf_sppf_pool, (_ptr(x), _check_view(x, "sppf x"), _ptr(y1), _ptr(y2), _ptr(y3), ld, B, H, W, Cc),
          {"bytes": 8.0 * x.numel()})


def upsample2x(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    B, H, W, Cc = x.shape
    if out is None:
        out = torch.empty(B, 2 * H, 2 * W, Cc, dtype=torch.float16, device=x.device)
    elif tuple(out.shape) != (B, 2 * H, 2 * W, Cc):
        raise ValueError(f"upsample2x: output shape {tuple(out.shape)} != {(B, 2 * H, 2 * W, Cc)}")
    _call("icaf_upsample2x", _lib.lib().icaf_upsample2x, (_ptr(x), _check_view(x, "upsample x"), _ptr(out), _check_view(out, "upsample out"),
                                                        B, H, W, Cc), {"bytes": 10.0 * x.numel()})
    return out


def copy_channels(x: torch.Tensor, out: torch.Tensor) -> None:
    B, H, W, Cc = x.shape
    if tuple(out.shape) != tuple(x.shape):
        raise ValueError(f"copy_channels: output shape {tuple(out.shape)} != {tuple(x.shape)}")
    _call("icaf_copy_channels", _lib.lib().icaf_copy_channels, (_ptr(x), _check_view(x, "copy x"), _ptr(out), _check_view(out, "copy out"),
                                                              B * H * W, Cc), {"bytes": 4.0 * x.numel()})


def dmff_pool_tokens(x_vis, x_ir, pos_vis, pos_ir, mix, nh: int, nw: int, with_stats: bool = False):
    """-> (tok_vis, tok_ir) fp16 (B, Npad, C); with_stats: also (stats_vis, stats_ir) fp32 (B*Npad, C/32, 2) row statistics."""
    B, H, W, Cc = x_vis.shape
    n_pad = round_up(nh * nw, 8)
    tv = torch.empty(B, n_pad, Cc, dtype=torch.float16, device=x_vis.device)
    ti = torch.empty_like(tv)
    ld = _check_view(x_vis, "dmff x_vis")
    assert _check_view(x_ir, "dmff x_ir") == ld
    sv = si = None
    if with_stats:
        sv = torch.empty(B * n_pad, Cc // 32, 2, dtype=torch.float32, device=x_vis.device)
        si = torch.empty_like(sv)
    _call("icaf_dmff_pool_tokens", _lib.lib().icaf_dmff_pool_tokens,
          (_ptr(x_vis), _ptr(x_ir), ld, _ptr(pos_vis), _ptr(pos_ir), _ptr(mix), _ptr(tv), _ptr(ti), _ptr(sv), _ptr(si), B, H, W, Cc, nh, nw,
           n_pad), {"bytes": 4.0 * x_vis.numel() + 4.0 * tv.numel() + 4.0 * pos_vis.numel()})
    return (tv, ti, sv, si) if with_stats else (tv, ti)


def layernorm(x0, g0, b0, x1=None, g1=None, b1=None, eps: float = 1e-5):
    """LayerNorm over the last dim of (.., C) fp16 contiguous tensors; one or two problems per launch."""
    Cc = x0.shape[-1]
    rows = x0.numel() // Cc
    y0 = torch.empty_like(x0)
    y1 = torch.empty_like(x1) if x1 is not None else None
    assert x0.is_contiguous() and (x1 is None or (x1.is_contiguous() and x1.shape == x0.shape))
    _call("icaf_layernorm", _lib.lib().icaf_layernorm,
          (_ptr(x0), _ptr(x1), _ptr(g0), _ptr(b0), _ptr(g1), _ptr(b1), _ptr(y0), _ptr(y1), rows, Cc, float(eps)),
          {"bytes": 4.0 * x0.numel() * (2 if x1 is not None else 1)})
    return (y0, y1) if x1 is not None else y0


def cross_attention(qk_vis, qk_ir, vt_vis, vt_ir, B: int, N: int, n_pad: int, Cc: int, heads: int, simt: bool = False):
    """Both directions of the DMFF cross-attention.  Fused form: vt_vis = vt_ir = None and qk_* are (B, Npad, 3C) [q|k|v]
    rows; split form: qk_* (B, Npad, 2C) and vt_* (C, B*Npad)."""
    out_v = torch.empty(B, n_pad, Cc, dtype=torch.float16, device=qk_vis.device)
    out_i = torch.empty_like(out_v)
    fn = _lib.lib().icaf_cross_attention_simt if simt else _lib.lib().icaf_cross_attention
    fused = vt_vis is None
    if fused != (vt_ir is None):
        raise ValueError("cross_attention: pass both V^T tensors or neither")
    for t in (qk_vis, qk_ir) + (() if fused else (vt_vis, vt_ir)):
        assert t.is_contiguous() and t.dtype == torch.float16
    want = (B, n_pad, (3 if fused else 2) * Cc)
    if tuple(qk_vis.shape) != want or tuple(qk_ir.shape) != want:
        raise ValueError(f"cross_attention: projection tensors must be {want}, got {tuple(qk_vis.shape)}")
    _call("icaf_cross_attention_simt" if simt else "icaf_cross_attention", fn,
          (_ptr(qk_vis), _ptr(qk_ir), _ptr(vt_vis), _ptr(vt_ir), _ptr(out_v), _ptr(out_i), B, N, n_pad, Cc, heads),
          {"flops": 8.0 * B * N * N * Cc, "bytes": 2.0 * 2 * (3 * B * n_pad * Cc + B * n_pad * Cc), "N": N, "d": Cc // heads})
    return out_v, out_i


def cross_attention_train(qkv_vis, qkv_ir, B: int, N: int, n_pad: int, Cc: int, heads: int, p_drop: float = 0.0, seed: int = 0):
    """Training-mode forward of the fused cross-attention: dropout p_drop on the probabilities (common.py:677,680), mask keyed
    by `seed` so that cross_attention_bwd regenerates it."""
    want = (B, n_pad, 3 * Cc)
    for t in (qkv_vis, qkv_ir):
        assert t.is_contiguous() and t.dtype == torch.float16
        if tuple(t.shape) != want:
            raise ValueError(f"cross_attention_train: projection tensors must be {want}, got {tuple(t.shape)}")
    out_v = torch.empty(B, n_pad, Cc, dtype=torch.float16, device=qkv_vis.device)
    out_i = torch.empty_like(out_v)
    _call("icaf_cross_attention_train", _lib.lib().icaf_cross_attention_train,
          (_ptr(qkv_vis), _ptr(qkv_ir), _ptr(out_v), _ptr(out_i), B, N, n_pad, Cc, heads, float(p_drop), int(seed) & 0xffffffff),
          {"flops": 8.0 * B * N * N * Cc, "bytes": 2.0 * 2 * 4 * B * n_pad * Cc})
    return out_v, out_i


def cross_attention_bwd(qkv_vis, qkv_ir, out_vis, out_ir, dout_vis, dout_ir, B: int, N: int, n_pad: int, Cc: int, heads: int,
                        p_drop: float = 0.0, seed: int = 0):
    """Gradients of the fused cross-attention w.r.t. the two [q|k|v] projection tensors (probabilities recomputed)."""
    want = (B, n_pad, 3 * Cc)
    for t in (qkv_vis, qkv_ir):
        assert t.is_contiguous() and t.dtype == torch.float16
        if tuple(t.shape) != want:
            raise ValueError(f"cross_attention_bwd: projection tensors must be {want}, got {tuple(t.shape)}")
    for t in (out_vis, out_ir, dout_vis, dout_ir):
        assert t.is_contiguous() and t.dtype == torch.float16
        if tuple(t.shape) != (B, n_pad, Cc):
            raise ValueError(f"cross_attention_bwd: outputs / output gradients must be {(B, n_pad, Cc)}, got {tuple(t.shape)}")
    dq_v = torch.empty_like(qkv_vis)
    dq_i = torch.empty_like(qkv_ir)
    nb = _lib.lib().icaf_cross_attention_bwd_workspace_bytes(B, n_pad, heads)
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=qkv_vis.device)
    _call("icaf_cross_attention_bwd", _lib.lib().icaf_cross_attention_bwd,
          (_ptr(qkv_vis), _ptr(qkv_ir), _ptr(out_vis), _ptr(out_ir), _ptr(dout_vis), _ptr(dout_ir), _ptr(dq_v), _ptr(dq_i),
           B, N, n_pad, Cc, heads, float(p_drop), int(seed) & 0xffffffff, _ptr(ws), nb),
          {"flops": 20.0 * B * N * N * Cc, "bytes": 2.0 * 2 * 9 * B * n_pad * Cc})
    return dq_v, dq_i


def dmff_pool_tokens_bwd(x_vis, x_ir, dtok_vis, dtok_ir, mix, nh: int, nw: int):
    """Gradients of dmff_pool_tokens w.r.t. the two NHWC feature maps (dense fp16)."""
    B, H, W, Cc = x_vis.shape
    ld = _check_view(x_vis, "dmff x_vis")
    if tuple(x_ir.shape) != tuple(x_vis.shape) or _check_view(x_ir, "dmff x_ir") != ld:
        raise ValueError("dmff_pool_tokens_bwd: the two feature maps must share shape and pitch")
    n_pad = dtok_vis.shape[1]
    for t in (dtok_vis, dtok_ir):
        assert t.is_contiguous() and t.dtype == torch.float16 and tuple(t.shape) == (B, n_pad, Cc)
    dx_v = torch.empty(B, H, W, Cc, dtype=torch.float16, device=x_vis.device)
    dx_i = torch.empty_like(dx_v)
    ws = torch.empty((2 * B * nh * nw * Cc + 7) // 8, dtype=torch.int64, device=x_vis.device)
    _call("icaf_dmff_pool_tokens_bwd", _lib.lib().icaf_dmff_pool_tokens_bwd,
          (_ptr(x_vis), _ptr(x_ir), ld, _ptr(dtok_vis), _ptr(dtok_ir), _ptr(mix), _ptr(dx_v), _ptr(dx_i), B, H, W, Cc, nh, nw, n_pad, _ptr(ws),
           C.c_size_t(ws.numel() * 8)),
          {"bytes": 2.0 * 2 * (2 * x_vis.numel() + dtok_vis.numel())})
    return dx_v, dx_i


def dmff_upsample_cat_bwd(dcat: torch.Tensor, nh: int, nw: int, n_pad: int, mode: int = 1):
    """Token-stream gradients of dmff_upsample_cat in its training mode (nearest); dcat: (B,H,W,2C) NHWC view."""
    B, H, W, C2 = dcat.shape
    Cc = C2 // 2
    ld = _check_view(dcat, "dmff dcat")
    dt_v = torch.empty(B, n_pad, Cc, dtype=torch.float16, device=dcat.device)
    dt_i = torch.empty_like(dt_v)
    _call("icaf_dmff_upsample_cat_bwd", _lib.lib().icaf_dmff_upsample_cat_bwd,
          (_ptr(dcat), ld, _ptr(dt_v), _ptr(dt_i), B, H, W, Cc, nh, nw, n_pad, mode), {"bytes": 2.0 * (dcat.numel() + 2 * dt_v.numel())})
    return dt_v, dt_i


def dmff_upsample_cat(tok_vis, tok_ir, x_vis, x_ir, nh: int, nw: int, mode: int = 0) -> torch.Tensor:
    B, H, W, Cc = x_vis.shape
    out = torch.empty(B, H, W, 2 * Cc, dtype=torch.float16, device=x_vis.device)
    ld = _check_view(x_vis, "dmff x_vis")
    if tuple(x_ir.shape) != tuple(x_vis.shape) or _check_view(x_ir, "dmff x_ir") != ld:
        raise ValueError("dmff_upsample_cat: the two feature maps must share shape and pitch")
    n_pad = tok_vis.shape[1]
    if tuple(tok_vis.shape) != (B, n_pad, Cc) or tuple(tok_ir.shape) != (B, n_pad, Cc) or n_pad < nh * nw or \
            not (tok_vis.is_contiguous() and tok_ir.is_contiguous()):
        raise ValueError(f"dmff_upsample_cat: token tensors must be contiguous (B, >= {nh * nw}, {Cc})")
    _call("icaf_dmff_upsample_cat", _lib.lib().icaf_dmff_upsample_cat,
          (_ptr(tok_vis), _ptr(tok_ir), tok_vis.shape[1], _ptr(x_vis), _ptr(x_ir), ld, _ptr(out), 2 * Cc, B, H, W, Cc, nh, nw, mode),
          {"bytes": 2.0 * (2 * x_vis.numel() + out.numel() + 2 * tok_vis.numel())})
    return out


def detect_decode(p: torch.Tensor, na: int, no: int, z: torch.Tensor, logits: torch.Tensor, row_off: int, stride: float,
                  anchors_px: Sequence[float]) -> torch.Tensor:
    """p: (B,ny,nx,>=na*no) conv output. Fills rows [row_off, row_off+na*ny*nx) of z/logits; returns x (B,na,ny,nx,no)."""
    B, ny, nx, pc = p.shape
    if pc < na * no or z.shape[0] != B or logits.shape[:2] != z.shape[:2] or z.shape[2] != no or logits.shape[2] != no - 5 or \
            row_off < 0 or row_off + na * ny * nx > z.shape[1]:
        raise ValueError(f"detect_decode: level ({ny}x{nx}, {na} anchors) at row {row_off} does not fit z {tuple(z.shape)}")
    x_out = torch.empty(B, na, ny, nx, no, dtype=torch.float16, device=p.device)
    anch = (C.c_float * (2 * na))(*[float(a) for a in anchors_px])
    _call("icaf_detect_decode", _lib.lib().icaf_detect_decode,
          (_ptr(p), _check_view(p, "detect p"), _ptr(x_out), _ptr(z), _ptr(logits), B, ny, nx, na, no, z.shape[1], row_off, float(stride), anch),
          {"bytes": 2.0 * (p.numel() + 2.2 * x_out.numel())})
    return x_out


def axpby(x: torch.Tensor, a: torch.Tensor, y: Optional[torch.Tensor] = None, b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = a*x (+ b*y): fp16 tensors of one shape, `a` / `b` one-element fp32 device tensors (LearnableCoefficient /
    LearnableWeights called stand-alone, common.py:569-587)."""
    if x.dtype != torch.float16 or not on_device(x):
        raise ValueError("axpby: expected a CUDA fp16 tensor")
    x = x.contiguous()
    n = x.numel()
    if n % 8:
        raise ValueError("axpby: element count must be a multiple of 8")
    if y is not None:
        if y.shape != x.shape or y.dtype != torch.float16:
            raise ValueError("axpby: x and y must share shape and dtype")
        y = y.contiguous()
    out = torch.empty_like(x)
    _call("icaf_axpby", _lib.lib().icaf_axpby, (_ptr(x), _ptr(y), _ptr(a), _ptr(b), _ptr(out), n),
          {"bytes": 2.0 * n * (3 if y is not None else 2)})
    return out


# ------------------------------------------------------------------------------------------------
# fp32 DMFF token streams (training with TransformerFusionBlock.stream_dtype = float32): the reference's autocast makes its token
# streams fp32 from the pooling to the upsample-and-add.  Tokens and token gradients are fp32 here; maps, map gradients and
# GEMM operands stay fp16.  Every wrapper checks each operand's dtype: the C ABI takes untyped pointers.
def _need(t: torch.Tensor, dtype, what: str, shape=None) -> torch.Tensor:
    if not torch.is_tensor(t) or t.dtype != dtype or not on_device(t):
        raise ValueError(f"{what}: expected a CUDA {dtype} tensor, got "
                         f"{(t.dtype, t.device) if torch.is_tensor(t) else type(t).__name__}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{what}: expected shape {tuple(shape)}, got {tuple(t.shape)}")
    return t


def _need_contig(t: torch.Tensor, dtype, what: str, shape=None) -> torch.Tensor:
    _need(t, dtype, what, shape)
    if not t.is_contiguous():
        raise ValueError(f"{what}: must be contiguous")
    return t


def dmff_pool_tokens_f32(x_vis, x_ir, pos_vis, pos_ir, mix, nh: int, nw: int):
    """dmff_pool_tokens over an fp32 stream: fp16 maps, fp32 (N, C) position embeddings -> fp32 (B, Npad, C) tokens."""
    B, H, W, Cc = x_vis.shape
    ld = _check_view(x_vis, "dmff x_vis")
    if tuple(x_ir.shape) != tuple(x_vis.shape) or _check_view(x_ir, "dmff x_ir") != ld:
        raise ValueError("dmff_pool_tokens_f32: the two feature maps must share shape and pitch")
    for t, w in ((pos_vis, "pos_vis"), (pos_ir, "pos_ir")):
        _need_contig(t, torch.float32, f"dmff_pool_tokens_f32 {w}", (nh * nw, Cc))
    _need_contig(mix, torch.float32, "dmff_pool_tokens_f32 mix", (4,))
    n_pad = round_up(nh * nw, 8)
    tv = torch.empty(B, n_pad, Cc, dtype=torch.float32, device=x_vis.device)
    ti = torch.empty_like(tv)
    _call("icaf_dmff_pool_tokens_f32", _lib.lib().icaf_dmff_pool_tokens_f32,
          (_ptr(x_vis), _ptr(x_ir), ld, _ptr(pos_vis), _ptr(pos_ir), _ptr(mix), _ptr(tv), _ptr(ti), B, H, W, Cc, nh, nw, n_pad),
          {"bytes": 4.0 * x_vis.numel() + 8.0 * tv.numel() + 8.0 * pos_vis.numel()})
    return tv, ti


def dmff_pool_tokens_bwd_f32(x_vis, x_ir, dtok_vis, dtok_ir, mix, nh: int, nw: int):
    """Gradients of dmff_pool_tokens_f32 w.r.t. the two fp16 NHWC maps, from fp32 token gradients."""
    B, H, W, Cc = x_vis.shape
    ld = _check_view(x_vis, "dmff x_vis")
    if tuple(x_ir.shape) != tuple(x_vis.shape) or _check_view(x_ir, "dmff x_ir") != ld:
        raise ValueError("dmff_pool_tokens_bwd_f32: the two feature maps must share shape and pitch")
    n_pad = dtok_vis.shape[1]
    for t, w in ((dtok_vis, "dtok_vis"), (dtok_ir, "dtok_ir")):
        _need_contig(t, torch.float32, f"dmff_pool_tokens_bwd_f32 {w}", (B, n_pad, Cc))
    _need_contig(mix, torch.float32, "dmff_pool_tokens_bwd_f32 mix", (4,))
    dx_v = torch.empty(B, H, W, Cc, dtype=torch.float16, device=x_vis.device)
    dx_i = torch.empty_like(dx_v)
    ws = torch.empty((2 * B * nh * nw * Cc + 7) // 8, dtype=torch.int64, device=x_vis.device)
    _call("icaf_dmff_pool_tokens_bwd_f32", _lib.lib().icaf_dmff_pool_tokens_bwd_f32,
          (_ptr(x_vis), _ptr(x_ir), ld, _ptr(dtok_vis), _ptr(dtok_ir), _ptr(mix), _ptr(dx_v), _ptr(dx_i), B, H, W, Cc, nh, nw, n_pad, _ptr(ws),
           C.c_size_t(ws.numel() * 8)),
          {"bytes": 2.0 * 2 * 2 * x_vis.numel() + 4.0 * 2 * dtok_vis.numel()})
    return dx_v, dx_i


def dmff_upsample_cat_f32(tok_vis, tok_ir, x_vis, x_ir, nh: int, nw: int) -> torch.Tensor:
    """The training-mode (nearest) tail over fp32 tokens: fp16 (B, H, W, 2C) = [up(tok_vis) + x_vis | up(tok_ir) + x_ir], each sum
    formed in fp32 and rounded once."""
    B, H, W, Cc = x_vis.shape
    ld = _check_view(x_vis, "dmff x_vis")
    if tuple(x_ir.shape) != tuple(x_vis.shape) or _check_view(x_ir, "dmff x_ir") != ld:
        raise ValueError("dmff_upsample_cat_f32: the two feature maps must share shape and pitch")
    n_pad = tok_vis.shape[1]
    if n_pad < nh * nw:
        raise ValueError(f"dmff_upsample_cat_f32: {n_pad} token rows for a {nh}x{nw} grid")
    for t, w in ((tok_vis, "tok_vis"), (tok_ir, "tok_ir")):
        _need_contig(t, torch.float32, f"dmff_upsample_cat_f32 {w}", (B, n_pad, Cc))
    out = torch.empty(B, H, W, 2 * Cc, dtype=torch.float16, device=x_vis.device)
    _call("icaf_dmff_upsample_cat_f32", _lib.lib().icaf_dmff_upsample_cat_f32,
          (_ptr(tok_vis), _ptr(tok_ir), n_pad, _ptr(x_vis), _ptr(x_ir), ld, _ptr(out), 2 * Cc, B, H, W, Cc, nh, nw),
          {"bytes": 2.0 * (2 * x_vis.numel() + out.numel()) + 4.0 * 2 * tok_vis.numel()})
    return out


def dmff_upsample_cat_bwd_f32(dcat: torch.Tensor, nh: int, nw: int, n_pad: int):
    """fp32 token-stream gradients of dmff_upsample_cat_f32; dcat: fp16 (B,H,W,2C) NHWC view."""
    B, H, W, C2 = dcat.shape
    Cc = C2 // 2
    ld = _check_view(dcat, "dmff dcat")
    dt_v = torch.empty(B, n_pad, Cc, dtype=torch.float32, device=dcat.device)
    dt_i = torch.empty_like(dt_v)
    _call("icaf_dmff_upsample_cat_bwd_f32", _lib.lib().icaf_dmff_upsample_cat_bwd_f32,
          (_ptr(dcat), ld, _ptr(dt_v), _ptr(dt_i), B, H, W, Cc, nh, nw, n_pad), {"bytes": 2.0 * dcat.numel() + 8.0 * dt_v.numel()})
    return dt_v, dt_i


def layernorm_f32(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """LayerNorm over the last dim of an fp32 contiguous (.., C) tensor -> fp16 (the fp32 LayerNorm, rounded once)."""
    _need_contig(x, torch.float32, "layernorm_f32 x")
    Cc = x.shape[-1]
    for t, w in ((g, "gamma"), (b, "beta")):
        _need_contig(t, torch.float32, f"layernorm_f32 {w}", (Cc,))
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _call("icaf_layernorm_f32", _lib.lib().icaf_layernorm_f32,
          (_ptr(x), _ptr(None), _ptr(g), _ptr(b), _ptr(None), _ptr(None), _ptr(y), _ptr(None), x.numel() // Cc, Cc, float(eps)),
          {"bytes": 6.0 * x.numel()})
    return y


def layernorm_bwd_f32(x, dy, gamma, eps: float, dgamma=None, dbeta=None, grad_scale: float = 1.0, accumulate: bool = False):
    """LayerNorm backward with fp32 x, fp16 dy -> fp32 dx; dgamma / dbeta (fp32 [C]) when given."""
    _need_contig(x, torch.float32, "layernorm_bwd_f32 x")
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    dy = _need(dy, torch.float16, "layernorm_bwd_f32 dy", x.shape).contiguous()
    _need_contig(gamma, torch.float32, "layernorm_bwd_f32 gamma", (Cc,))
    for t, w in ((dgamma, "dgamma"), (dbeta, "dbeta")):
        if t is not None:
            _need_contig(t, torch.float32, f"layernorm_bwd_f32 {w}", (Cc,))
    dx = torch.empty_like(x)
    ws = _train_ws(Cc, 2 * rows, x.device)
    _call("icaf_layernorm_bwd_f32", _lib.lib().icaf_layernorm_bwd_f32,
          (_ptr(x), _ptr(dy), _ptr(gamma), _ptr(dx), _ptr(dgamma), _ptr(dbeta), rows, Cc, float(eps), float(grad_scale), int(accumulate), _ptr(ws),
           C.c_size_t(ws.numel() * 4)), {"bytes": 14.0 * x.numel()})
    return dx


def axpby_f32(x: torch.Tensor, a: torch.Tensor, y: Optional[torch.Tensor] = None, b: Optional[torch.Tensor] = None,
              out_dtype=torch.float32) -> torch.Tensor:
    """out = a*x (+ b*y) with x fp32, y fp16: torch's fp32 `a * x + b * y` bit for bit (a coefficient pair of an fp32 token
    stream, common.py:747-750); out fp32, or fp16 (the backward's gradient of an fp16 branch output)."""
    x = _need(x, torch.float32, "axpby_f32 x").contiguous()
    if out_dtype not in (torch.float32, torch.float16):
        raise ValueError(f"axpby_f32: output dtype float32 or float16, got {out_dtype}")
    n = x.numel()
    if n % 8:
        raise ValueError("axpby_f32: element count must be a multiple of 8")
    _need(a, torch.float32, "axpby_f32 a", (1,))
    if y is not None:
        y = _need(y, torch.float16, "axpby_f32 y", x.shape).contiguous()
        _need(b, torch.float32, "axpby_f32 b", (1,))
    out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    _call("icaf_axpby_f32", _lib.lib().icaf_axpby_f32, (_ptr(x), _ptr(y), _ptr(a), _ptr(b), _ptr(out), int(out_dtype == torch.float16), n),
          {"bytes": n * (4.0 + out.element_size() + (2.0 if y is not None else 0.0))})
    return out


def dot_f32(x: torch.Tensor, y: torch.Tensor, out: Optional[torch.Tensor] = None, scale: float = 1.0):
    """<x, y> (fp32, one element) with x fp32 and y fp16 or fp32 of x's shape; accumulates into `out` when given."""
    x = _need(x, torch.float32, "dot_f32 x").contiguous()
    if not torch.is_tensor(y) or y.dtype not in (torch.float16, torch.float32):
        raise ValueError("dot_f32: y must be an fp16 or fp32 tensor")
    y = _need(y, y.dtype, "dot_f32 y", x.shape).contiguous()
    Cc = x.shape[-1]
    acc = out is not None
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=x.device)
    _need(out, torch.float32, "dot_f32 out", (1,))
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_dot_f32", _lib.lib().icaf_dot_f32, (_ptr(x), _ptr(y), int(y.dtype == torch.float16), x.numel() // Cc, Cc, _ptr(out), float(scale),
                                                   int(acc), _ptr(ws), C.c_size_t(ws.numel() * 4)),
          {"bytes": (4.0 + y.element_size()) * x.numel()})
    return out


def colsum_f32(x: torch.Tensor, scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Column sums (fp32) of a dense fp32 (rows, C) matrix; accumulates into `out` when given."""
    _need_contig(x, torch.float32, "colsum_f32 x")
    rows, Cc = x.shape
    acc = out is not None
    if out is None:
        out = torch.empty(Cc, dtype=torch.float32, device=x.device)
    _need(out, torch.float32, "colsum_f32 out", (Cc,))
    ws = torch.empty(64 * Cc, dtype=torch.float32, device=x.device)
    _call("icaf_colsum_f32", _lib.lib().icaf_colsum_f32, (_ptr(x), rows, Cc, _ptr(out), float(scale), int(acc), _ptr(ws), C.c_size_t(ws.numel() * 4)),
          {"bytes": 4.0 * x.numel()})
    return out


def nms_workspace_bytes(B: int, R: int, no: int, multi_label: bool = False) -> int:
    """Device workspace :func:`nms` needs for a (B, R, no) prediction tensor (multi_label only counts when nc = no - 5 > 1)."""
    if multi_label and no - 5 > 1:
        return int(_lib.lib().icaf_nms_multi_label_workspace_bytes(B, R, no))
    return int(_lib.lib().icaf_nms_workspace_bytes(B, R))


def nms(z: torch.Tensor, conf_thres: float = 0.25, iou_thres: float = 0.45, agnostic: bool = False,
        classes: Optional[Sequence[int]] = None, max_det: int = 300, det: Optional[torch.Tensor] = None,
        count: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None, multi_label: bool = False):
    """Batched NMS on the device (utils/general.py:518-607).  z: fp16 (B, R, nc+5) decoded predictions.  `multi_label`
    (test.py's setting) keeps one candidate per (row, class) above the threshold; like the reference it only applies when
    nc > 1.  Returns (det fp32 (B, max_det, 6) rows [x1,y1,x2,y2,conf,cls] in confidence order, count int32 (B,)); no host
    sync.  `workspace` must hold :func:`nms_workspace_bytes` bytes."""
    if z.dim() != 3 or z.dtype != torch.float16 or not on_device(z) or not z.is_contiguous():
        raise ValueError(f"nms: expected a contiguous CUDA fp16 (B, R, nc+5) tensor, got {z.dtype} {tuple(z.shape)}")
    B, R, no = z.shape
    mask = 0
    if classes is not None:
        for c in classes:
            if not 0 <= int(c) < min(no - 5, 64):
                raise ValueError(f"nms: class {c} outside [0, {min(no - 5, 64)})")
            mask |= 1 << int(c)
        if mask == 0:
            raise ValueError("nms: empty class filter")
    if det is None:
        det = torch.zeros(B, max_det, 6, dtype=torch.float32, device=z.device)
    if count is None:
        count = torch.zeros(B, dtype=torch.int32, device=z.device)
    multi_label = bool(multi_label) and no - 5 > 1
    need = nms_workspace_bytes(B, R, no, multi_label)
    if workspace is None:
        workspace = torch.empty((need + 7) // 8, dtype=torch.int64, device=z.device)
    if tuple(det.shape) != (B, max_det, 6) or det.dtype != torch.float32 or tuple(count.shape) != (B,) or count.dtype != torch.int32:
        raise ValueError("nms: det must be fp32 (B, max_det, 6) and count int32 (B,)")
    name = "icaf_nms_multi_label" if multi_label else "icaf_nms"
    _call(name, getattr(_lib.lib(), name),
          (_ptr(z), B, R, no, float(conf_thres), float(iou_thres), int(bool(agnostic)), C.c_uint64(mask), int(max_det), _ptr(det), _ptr(count),
           _ptr(workspace), C.c_size_t(workspace.numel() * workspace.element_size())), {"bytes": 2.0 * z.numel()})
    return det, count


def confluence_workspace_bytes(B: int, R: int, no: int) -> int:
    """Device workspace :func:`confluence` needs for (B, R, no) predictions (no = 5 + the number of classes)."""
    return int(_lib.lib().icaf_confluence_workspace_bytes(B, R, no))


def confluence(z: torch.Tensor, conf_thres: float = 0.1, p_thres: float = 0.6, max_det: int = 300,
               det: Optional[torch.Tensor] = None, count: Optional[torch.Tensor] = None,
               workspace: Optional[torch.Tensor] = None, index: Optional[torch.Tensor] = None,
               class_num: Optional[int] = None):
    """Batched Confluence on the device (utils/confluence.py:50-193), the reference's alternative to NMS.  z: fp16 or fp32
    (B, R, nc+5) decoded predictions, read in their own dtype.  Returns (det fp32 (B, max_det, 6) rows
    [x1,y1,x2,y2,conf,cls] in ascending candidate order, count int32 (B,)): count is the true number kept, and rows past
    max_det are not written when it is larger.  No host sync.  `workspace` must hold :func:`confluence_workspace_bytes`
    bytes; `index` (int32 (B, max_det)), when given, receives the row of each written detection.
    `class_num`: z is instead fp32 detection rows (B, R, 6) [x1,y1,x2,y2,conf,cls], what confluence() takes, clustered
    per class 0 .. class_num-1 by their own cls and conf, without a threshold."""
    rows = class_num is not None
    if z.dim() != 3 or not on_device(z) or not z.is_contiguous() or \
            (z.dtype != torch.float32 if rows else z.dtype not in (torch.float16, torch.float32)) or (rows and z.shape[2] != 6):
        raise ValueError(f"confluence: expected a contiguous CUDA {'fp32 (B, R, 6)' if rows else 'fp16 or fp32 (B, R, nc+5)'} "
                         f"tensor, got {z.dtype} {tuple(z.shape)}")
    B, R = z.shape[:2]
    no = int(class_num) + 5 if rows else z.shape[2]
    if det is None:
        det = torch.zeros(B, max_det, 6, dtype=torch.float32, device=z.device)
    if count is None:
        count = torch.zeros(B, dtype=torch.int32, device=z.device)
    if workspace is None:
        workspace = torch.empty((confluence_workspace_bytes(B, R, no) + 15) // 16, 2, dtype=torch.int64, device=z.device)
    if det.dim() != 3 or (det.shape[0], det.shape[2]) != (B, 6) or det.dtype != torch.float32 or \
            tuple(count.shape) != (B,) or count.dtype != torch.int32:
        raise ValueError("confluence: det must be fp32 (B, max_det, 6) and count int32 (B,)")
    if index is not None and (tuple(index.shape) != tuple(det.shape[:2]) or index.dtype != torch.int32):
        raise ValueError("confluence: index must be int32 (B, max_det)")
    dtype = 2 if rows else (0 if z.dtype == torch.float16 else 1)
    _call("icaf_confluence", _lib.lib().icaf_confluence,
          (_ptr(z), dtype, B, R, no, float(conf_thres), float(p_thres), _ptr(det), _ptr(index), det.shape[1], _ptr(count),
           _ptr(workspace), C.c_size_t(workspace.numel() * workspace.element_size())),
          {"bytes": float(z.numel() * z.element_size())})
    return det, count


def match_detections(det: torch.Tensor, count: torch.Tensor, targets: torch.Tensor, ratio_pad: torch.Tensor, height: int,
                     width: int, iouv: torch.Tensor, single_cls: bool = False, correct: Optional[torch.Tensor] = None,
                     native: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None):
    """test.py:196-227 for one batch on the device: which NMS detections are true positives at each IoU threshold.
    det / count: what :func:`nms` returns.  targets: fp32 (T, 6) rows [image, cls, x, y, w, h] normalised to the
    (height, width) batch.  ratio_pad: fp32 (B, 5) rows [h0, w0, gain, padw, padh] (the loader's ``shapes``).  iouv: fp32
    (niou,) thresholds on the device.  Returns (correct uint8 (B, max_det, niou), native): ``native`` (fp32 (B, max_det, 4),
    the scale_coords boxes) is written only when passed in.  Rows at or past ``count`` are zero.  No host sync."""
    if det.dim() != 3 or det.shape[2] != 6 or det.dtype != torch.float32 or not det.is_contiguous() or not on_device(det):
        raise ValueError(f"match_detections: det must be contiguous CUDA fp32 (B, max_det, 6), got {det.dtype} {tuple(det.shape)}")
    B, max_det = det.shape[0], det.shape[1]
    niou = iouv.numel()
    if tuple(count.shape) != (B,) or count.dtype != torch.int32:
        raise ValueError("match_detections: count must be int32 (B,)")
    if targets.dim() != 2 or targets.shape[1] != 6 or targets.dtype != torch.float32 or not targets.is_contiguous():
        raise ValueError(f"match_detections: targets must be contiguous fp32 (T, 6), got {targets.dtype} {tuple(targets.shape)}")
    if tuple(ratio_pad.shape) != (B, 5) or ratio_pad.dtype != torch.float32 or not ratio_pad.is_contiguous():
        raise ValueError("match_detections: ratio_pad must be contiguous fp32 (B, 5)")
    if iouv.dtype != torch.float32 or iouv.dim() != 1 or not 1 <= niou <= 32:
        raise ValueError("match_detections: iouv must be fp32 (niou,) with 1 <= niou <= 32")
    for t, what in ((count, "count"), (targets, "targets"), (ratio_pad, "ratio_pad"), (iouv, "iouv")):
        if t.device != det.device:
            raise ValueError(f"match_detections: {what} is on {t.device}, det on {det.device}")
    if correct is None:
        correct = torch.empty(B, max_det, niou, dtype=torch.uint8, device=det.device)
    elif tuple(correct.shape) != (B, max_det, niou) or correct.dtype not in (torch.uint8, torch.bool) or not correct.is_contiguous():
        raise ValueError(f"match_detections: correct must be contiguous uint8 / bool {(B, max_det, niou)}")
    if native is not None and (tuple(native.shape) != (B, max_det, 4) or native.dtype != torch.float32 or not native.is_contiguous()):
        raise ValueError(f"match_detections: native must be contiguous fp32 {(B, max_det, 4)}")
    T = int(targets.shape[0])
    need = int(_lib.lib().icaf_match_detections_workspace_bytes(T))
    if workspace is None or workspace.numel() * workspace.element_size() < need:
        workspace = torch.empty(max((need + 3) // 4, 1), dtype=torch.int32, device=det.device)
    _call("icaf_match_detections", _lib.lib().icaf_match_detections,
          (_ptr(det), _ptr(count), B, max_det, _ptr(targets if T else None), T, _ptr(ratio_pad), int(height), int(width),
           _ptr(iouv), niou, int(bool(single_cls)), _ptr(correct), _ptr(native), _ptr(workspace),
           C.c_size_t(workspace.numel() * workspace.element_size())),
          {"bytes": float(det.numel() * 4 + B * max_det * niou + T * 24 * B)})
    return correct, native


KAIST_MAX_DET = 1000      # the reference's maxDets: beyond it its evaluateImg indexes past its IoU rows


def kaist_mr(gt, rows: torch.Tensor, span: torch.Tensor, max_per_image: int, day_images: int = 1455, curves: bool = False,
             workspace: Optional[torch.Tensor] = None):
    """The nine KAIST miss-rate evaluations of evaluation_script.evaluate on the device (icaf_kaist_mr).  gt: the device
    arrays of a :class:`~icafusion_b200.kaist_eval.KaistAnnotations` (attributes box, height, occlusion, ignore, id, offset).
    rows: float64 (N, 5) detections x, y, w, h, score; span: int32 (images, 2) (offset, count) per image, counts at most
    ``max_per_image`` (<= 1000).  Returns (ys float64 (9, 9), counts int32 (9, 3) [kept, tp, npig], curves float64
    (9, 2, N) fppi / miss rate or None); no host sync."""
    images = int(gt.offset.numel()) - 1
    if not 0 <= int(max_per_image) <= KAIST_MAX_DET:
        raise ValueError(f"kaist_mr: more than {KAIST_MAX_DET} detections in one image ({max_per_image}); the reference's "
                         "evaluateImg fails there")
    if rows.dim() != 2 or rows.shape[1] != 5 or rows.dtype != torch.float64 or not rows.is_contiguous() or not on_device(rows):
        raise ValueError(f"kaist_mr: rows must be contiguous CUDA float64 (N, 5), got {rows.dtype} {tuple(rows.shape)}")
    if tuple(span.shape) != (images, 2) or span.dtype != torch.int32 or not span.is_contiguous():
        raise ValueError(f"kaist_mr: span must be contiguous int32 {(images, 2)}")
    N, G = int(rows.shape[0]), int(gt.id.numel())
    dev = rows.device
    ys = torch.empty(9, 9, dtype=torch.float64, device=dev)
    counts = torch.empty(9, 3, dtype=torch.int32, device=dev)
    cv = torch.empty(9, 2, N, dtype=torch.float64, device=dev) if curves else None
    need = 256 if _DRY is not None else int(_lib.lib().icaf_kaist_mr_workspace_bytes(images, G, N))
    if need == 0:
        raise _lib.IcafError(f"icaf_kaist_mr_workspace_bytes failed: {_lib.lib().icaf_last_error().decode()}")
    if workspace is None or workspace.numel() < need + 256:
        workspace = torch.empty(need + 256, dtype=torch.uint8, device=dev)
    base = (-workspace.data_ptr()) % 256 if _DRY is None else 0     # the kernel wants a 256-byte aligned workspace
    ws = workspace[base:base + need]
    _call("icaf_kaist_mr", _lib.lib().icaf_kaist_mr,
          (_ptr(gt.box), _ptr(gt.height), _ptr(gt.occlusion), _ptr(gt.ignore), _ptr(gt.id), _ptr(gt.offset), images, G,
           int(day_images), _ptr(rows), _ptr(span), N, int(max_per_image), _ptr(ys), _ptr(counts), _ptr(cv), _ptr(ws),
           C.c_size_t(need)),
          {"bytes": float(N * 40 + G * 40)})
    return ys, counts, cv


def kaist_round_detections(native: torch.Tensor, det: torch.Tensor, count: torch.Tensor, image: torch.Tensor,
                           rows: torch.Tensor, span: torch.Tensor):
    """test.py's ``%g`` result lines of one batch, in memory (icaf_kaist_round_detections): for image b, p = image[b],
    rows (images * max_det, 5) float64 at p * max_det + i get float('%g' % v) of the fp32 x1, y1, w, h, score, and
    span[p] = (p * max_det, count[b]).  native: fp32 (B, max_det, 4); det / count: what :func:`nms` returns; image: int32
    (B,) dataset indices on the device.  No host sync."""
    B, max_det = int(det.shape[0]), int(det.shape[1])
    images = int(span.shape[0])
    if tuple(native.shape) != (B, max_det, 4) or native.dtype != torch.float32 or not native.is_contiguous():
        raise ValueError(f"kaist_round_detections: native must be contiguous fp32 {(B, max_det, 4)}")
    if det.dim() != 3 or det.shape[2] != 6 or det.dtype != torch.float32 or not det.is_contiguous():
        raise ValueError("kaist_round_detections: det must be contiguous fp32 (B, max_det, 6)")
    if tuple(count.shape) != (B,) or count.dtype != torch.int32 or tuple(image.shape) != (B,) or image.dtype != torch.int32:
        raise ValueError("kaist_round_detections: count and image must be int32 (B,)")
    if tuple(rows.shape) != (images * max_det, 5) or rows.dtype != torch.float64 or span.dtype != torch.int32 or \
            span.dim() != 2 or span.shape[1] != 2:
        raise ValueError(f"kaist_round_detections: rows must be float64 {(images * max_det, 5)} and span int32 (images, 2)")
    _call("icaf_kaist_round_detections", _lib.lib().icaf_kaist_round_detections,
          (_ptr(native), _ptr(det), _ptr(count), _ptr(image), B, max_det, images, _ptr(rows), _ptr(span)),
          {"bytes": float(B * max_det * (16 + 4 + 40))})


# ---------------------------------------------------------------------------------------------------------------
# Training-step building blocks (operator level; see include/icaf_b200.h).  Gradients of Conv2d / Linear layers.
def conv2d_wgrad(x: torch.Tensor, dy: torch.Tensor, kh: int, kw: int, stride: int, pad: int, scale: float = 1.0,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dW (Cout, Cin, kh, kw) fp32 = scale * sum_pixels dy x.  x (B,Hi,Wi,Cin), dy (B,Ho,Wo,Cout): fp16 NHWC views.  With
    `out` the gradient is ACCUMULATED into it (`.grad` semantics)."""
    B, Hi, Wi, Cin = x.shape
    _, Ho, Wo, Cout = dy.shape
    g = _lib.ConvGeom(B, Hi, Wi, Cin, Ho, Wo, Cout, kh, kw, stride, pad, round_up(kh * kw * Cin, 64), round_up(Cout, 32), 0, 0)
    need = int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g)))
    if need == 0:
        raise _lib.IcafError(f"conv2d_wgrad: unsupported geometry Cin={Cin} Cout={Cout} k={kh}x{kw} s={stride}")
    ws = torch.empty((need + 7) // 8, dtype=torch.int64, device=x.device)
    acc = out is not None
    if out is None:
        out = torch.empty(Cout, Cin, kh, kw, dtype=torch.float32, device=x.device)
    elif tuple(out.shape) != (Cout, Cin, kh, kw) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("conv2d_wgrad: `out` must be contiguous fp32 (Cout, Cin, kh, kw)")
    _call("icaf_conv2d_wgrad", _lib.lib().icaf_conv2d_wgrad,
          (C.byref(g), _ptr(x), _check_view(x, "wgrad x"), _ptr(dy), _check_view(dy, "wgrad dy"), _ptr(out), float(scale), int(acc), _ptr(ws),
           C.c_size_t(ws.numel() * 8)), {"flops": 2.0 * B * Ho * Wo * Cout * Cin * kh * kw, "bytes": 2.0 * (x.numel() + dy.numel())})
    return out


def linear_wgrad(x: torch.Tensor, dy: torch.Tensor, scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dW (N, K) fp32 of y = x W^T for (rows, K) x and (rows, N) dy."""
    o4 = None if out is None else out.view(out.shape[0], out.shape[1], 1, 1)
    return conv2d_wgrad(x.unflatten(0, (1, 1, x.shape[0])), dy.unflatten(0, (1, 1, dy.shape[0])), 1, 1, 1, 0, scale, o4).view(dy.shape[1], x.shape[1])


def pack_weight(weight: torch.Tensor, stride: int, pad: int, act: int = ACT_NONE, bias: Optional[torch.Tensor] = None,
                dgrad: bool = False) -> PackedConv:
    """fp32 master filter (Cout,Cin,kh,kw) on the device -> PackedConv through icaf_pack_weight (one launch; the training step
    re-packs every filter after each optimiser update).  dgrad: the flipped / transposed filter of the data-gradient
    convolution, W'[c][n][ky][kx] = W[n][c][kh-1-ky][kw-1-kx], its channel count (Cout) padded to a multiple of 8."""
    cout, cin, kh, kw = weight.shape
    w = weight.detach()
    if w.dtype != torch.float32 or not w.is_contiguous() or not on_device(w):
        raise ValueError("pack_weight: contiguous fp32 CUDA filter expected")
    if dgrad:
        chan, rows, pcin, pcout = round_up(cout, 8), round_up(cin, 32), round_up(cout, 8), cin
    else:
        if cin % 8:
            raise ValueError(f"pack_weight: input channels must be a multiple of 8, got {cin}")
        chan, rows, pcin, pcout = cin, round_up(cout, 32), cin, cout
    k_pad = round_up(kh * kw * chan, 64)
    out = torch.empty(rows, k_pad, dtype=torch.float16, device=w.device)
    _call("icaf_pack_weight", _lib.lib().icaf_pack_weight, (_ptr(w), cout, cin, kh, kw, chan, rows, k_pad, int(dgrad), _ptr(out)),
          {"bytes": 4.0 * w.numel() + 2.0 * out.numel()})
    b = None if bias is None else bias.detach().float().contiguous()
    return PackedConv(out, b, pcin, pcout, kh, kw, stride, pad, act)


def pack_weight_pair(weight: torch.Tensor, stride: int, pad: int, act: int = ACT_NONE, bias: Optional[torch.Tensor] = None):
    """-> (forward PackedConv, data-gradient PackedConv) of one fp32 master filter in ONE launch (see pack_weight)."""
    cout, cin, kh, kw = weight.shape
    w = weight.detach()
    if w.dtype != torch.float32 or not w.is_contiguous() or not on_device(w) or cin % 8:
        raise ValueError("pack_weight_pair: contiguous fp32 CUDA filter with input channels % 8 == 0 expected")
    rows_f, kpad_f = round_up(cout, 32), round_up(kh * kw * cin, 64)
    chan_d = round_up(cout, 8)
    rows_d, kpad_d = round_up(cin, 32), round_up(kh * kw * chan_d, 64)
    buf = torch.empty(rows_f * kpad_f + rows_d * kpad_d, dtype=torch.float16, device=w.device)
    of, od = buf[:rows_f * kpad_f].view(rows_f, kpad_f), buf[rows_f * kpad_f:].view(rows_d, kpad_d)
    _call("icaf_pack_weight_pair", _lib.lib().icaf_pack_weight_pair,
          (_ptr(w), cout, cin, kh, kw, rows_f, kpad_f, _ptr(of), chan_d, rows_d, kpad_d, _ptr(od)), {"bytes": 4.0 * w.numel() + 2.0 * buf.numel()})
    b = None if bias is None else bias.detach().float().contiguous()
    return PackedConv(of, b, cin, cout, kh, kw, stride, pad, act), PackedConv(od, None, chan_d, cin, kh, kw, 1, 0, ACT_NONE)


def pack_dgrad_weight(weight: torch.Tensor, device=None) -> PackedConv:
    """Filter of the data-gradient convolution (stride 1; pad k-1-p is set by conv2d_dgrad; no bias, no activation)."""
    w = weight.detach().float().contiguous()
    if device is not None:
        w = w.to(device)
    return pack_weight(w, 1, 0, ACT_NONE, None, dgrad=True)


def zero_stuff2(dy: torch.Tensor, H2: int, W2: int) -> torch.Tensor:
    B, H, W, Cc = dy.shape
    out = torch.empty(B, H2, W2, Cc, dtype=torch.float16, device=dy.device)
    _call("icaf_zero_stuff2", _lib.lib().icaf_zero_stuff2, (_ptr(dy.contiguous()), _ptr(out), B, H, W, Cc, H2, W2), {"bytes": 2.0 * (dy.numel() + out.numel())})
    return out


def conv2d_dgrad(dy: torch.Tensor, weight: torch.Tensor, stride: int, pad: int, in_hw, packed: Optional[PackedConv] = None) -> torch.Tensor:
    """dx (B,Hi,Wi,Cin) fp16 of y = conv2d(x, weight, stride, pad): the forward tensor-core kernel on the flipped / transposed
    filter (`packed`: that filter if the caller packed it already); a stride-2 layer first spreads dy over the input grid
    (icaf_zero_stuff2)."""
    k = weight.shape[2]
    Hi, Wi = in_hw
    pk = packed if packed is not None else pack_dgrad_weight(weight, dy.device)
    if stride == 2:
        dy = zero_stuff2(dy, Hi + 2 * pad - k + 1, Wi + 2 * pad - k + 1)
    elif stride != 1:
        raise NotImplementedError("conv2d_dgrad: stride 1 or 2")
    pk.pad = k - 1 - pad
    dx = conv2d([dy], [pk])[0]
    if tuple(dx.shape[1:3]) != (Hi, Wi):
        raise ValueError(f"conv2d_dgrad: got a {tuple(dx.shape[1:3])} gradient map for a {(Hi, Wi)} input")
    return dx


def colsum(x: torch.Tensor, scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Column sums (fp32) of a dense fp16 (rows, C) matrix -- bias gradients; accumulates into `out` when given."""
    rows, Cc = x.shape
    assert x.is_contiguous() and x.dtype == torch.float16
    acc = out is not None
    if out is None:
        out = torch.empty(Cc, dtype=torch.float32, device=x.device)
    ws = torch.empty(64 * Cc, dtype=torch.float32, device=x.device)
    _call("icaf_colsum", _lib.lib().icaf_colsum, (_ptr(x), rows, Cc, _ptr(out), float(scale), int(acc), _ptr(ws), C.c_size_t(ws.numel() * 4)),
          {"bytes": 2.0 * x.numel()})
    return out


def _train_ws(Cc: int, extra_floats: int, device) -> torch.Tensor:
    need = int(_lib.lib().icaf_train_workspace_bytes(Cc)) // 4 + extra_floats
    return torch.empty(need, dtype=torch.float32, device=device)


def bn_act_fwd(x: torch.Tensor, gamma, beta, run_mean, run_var, eps: float, momentum: float, act: int):
    """Training-mode BatchNorm2d + activation on a dense fp16 NHWC map: -> (y, save_mean, save_invstd)."""
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    assert x.is_contiguous() and x.dtype == torch.float16
    y = torch.empty_like(x)
    sm = torch.empty(Cc, dtype=torch.float32, device=x.device)
    si = torch.empty_like(sm)
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_bn_act_fwd", _lib.lib().icaf_bn_act_fwd,
          (_ptr(x), _ptr(gamma), _ptr(beta), _ptr(run_mean), _ptr(run_var), _ptr(y), _ptr(sm), _ptr(si), rows, Cc, float(eps), float(momentum), int(act),
           _ptr(ws), C.c_size_t(ws.numel() * 4)), {"bytes": 6.0 * x.numel()})
    return y, sm, si


def bn_act_bwd(x, dy, gamma, beta, sm, si, act: int, dgamma=None, dbeta=None, grad_scale: float = 1.0, accumulate: bool = False):
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    dy = dy.contiguous()
    dx = torch.empty_like(x)
    ws = _train_ws(Cc, 2 * Cc, x.device)
    _call("icaf_bn_act_bwd", _lib.lib().icaf_bn_act_bwd,
          (_ptr(x), _ptr(dy), _ptr(gamma), _ptr(beta), _ptr(sm), _ptr(si), _ptr(dx), _ptr(dgamma), _ptr(dbeta), rows, Cc, int(act), float(grad_scale),
           int(accumulate), _ptr(ws), C.c_size_t(ws.numel() * 4)), {"bytes": 10.0 * x.numel()})
    return dx


# Synchronised BatchNorm (torch.nn.SyncBatchNorm): bn_act_fwd / bn_act_bwd in two phases each, with the per-channel sums of
# phase 1 summed over the ranks (all_reduce_) before phase 2.  Fed phase 1's buffer unchanged, phase 2 equals the one-call form.
def bn_act_fwd_stats(x: torch.Tensor) -> torch.Tensor:
    """Phase 1 of the forward: -> fp32 [2C + 1] = (sum x, sum x^2 per channel, row count) of this rank's dense NHWC map."""
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    assert x.is_contiguous() and x.dtype == torch.float16
    stats = torch.empty(2 * Cc + 1, dtype=torch.float32, device=x.device)
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_bn_act_fwd_stats", _lib.lib().icaf_bn_act_fwd_stats, (_ptr(x), rows, Cc, _ptr(stats), _ptr(ws), C.c_size_t(ws.numel() * 4)),
          {"bytes": 2.0 * x.numel()})
    return stats


def bn_act_fwd_apply(x: torch.Tensor, gamma, beta, run_mean, run_var, stats, eps: float, momentum: float, act: int):
    """Phase 2 of the forward from the summed `stats`: -> (y, save_mean, save_invstd) over the rows of every rank."""
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    assert x.is_contiguous() and x.dtype == torch.float16 and stats.numel() == 2 * Cc + 1
    y = torch.empty_like(x)
    sm = torch.empty(Cc, dtype=torch.float32, device=x.device)
    si = torch.empty_like(sm)
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_bn_act_fwd_apply", _lib.lib().icaf_bn_act_fwd_apply,
          (_ptr(x), _ptr(gamma), _ptr(beta), _ptr(run_mean), _ptr(run_var), _ptr(stats), _ptr(y), _ptr(sm), _ptr(si), rows, Cc, float(eps),
           float(momentum), int(act), _ptr(ws), C.c_size_t(ws.numel() * 4)), {"bytes": 4.0 * x.numel()})
    return y, sm, si


def bn_act_bwd_sums(x, dy, gamma, beta, sm, si, act: int, dgamma=None, dbeta=None, grad_scale: float = 1.0, accumulate: bool = False):
    """Phase 1 of the backward: dgamma / dbeta of this rank's rows, -> fp32 [2C] = (sum dz, sum dz * xhat) to be summed.
    `dy` must be contiguous (phase 2 reads the same tensor)."""
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    assert dy.is_contiguous()
    sums = torch.empty(2 * Cc, dtype=torch.float32, device=x.device)
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_bn_act_bwd_sums", _lib.lib().icaf_bn_act_bwd_sums,
          (_ptr(x), _ptr(dy), _ptr(gamma), _ptr(beta), _ptr(sm), _ptr(si), _ptr(dgamma), _ptr(dbeta), _ptr(sums), rows, Cc, int(act), float(grad_scale),
           int(accumulate), _ptr(ws), C.c_size_t(ws.numel() * 4)), {"bytes": 4.0 * x.numel()})
    return sums


def bn_act_bwd_apply(x, dy, gamma, beta, sm, si, sums, count, act: int):
    """Phase 2 of the backward: dx from the summed `sums` and the forward's summed row count (`count`: fp32 [1] on the device)."""
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    assert dy.is_contiguous() and sums.numel() == 2 * Cc and count.numel() == 1
    dx = torch.empty_like(x)
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_bn_act_bwd_apply", _lib.lib().icaf_bn_act_bwd_apply,
          (_ptr(x), _ptr(dy), _ptr(gamma), _ptr(beta), _ptr(sm), _ptr(si), _ptr(sums), _ptr(count), _ptr(dx), rows, Cc, int(act), _ptr(ws),
           C.c_size_t(ws.numel() * 4)), {"bytes": 6.0 * x.numel()})
    return dx


def all_reduce_(buf: torch.Tensor, group=None) -> torch.Tensor:
    """Sum `buf` over the ranks of `group` in place: torch.distributed.all_reduce, ordered on the current stream (NCCL makes
    the stream wait, not the host, so it can be captured in a CUDA graph).  A dry run records it as ("all_reduce", (buf,),
    work) instead, so a walk counts exchanges as it counts launches."""
    if _DRY is not None:
        _DRY.append(("all_reduce", (buf,), {"bytes": 4.0 * buf.numel(), "group": group}))
        return buf
    torch.distributed.all_reduce(buf, group=group)
    return buf


def eltwise(mode: int, x, dy=None, p: float = 0.0, seed: int = 0):
    x = x.contiguous()
    y = torch.empty_like(x)
    _call("icaf_eltwise", _lib.lib().icaf_eltwise, (int(mode), _ptr(x), _ptr(None if dy is None else dy.contiguous()), _ptr(y), x.numel(), float(p), C.c_uint32(seed & 0xFFFFFFFF)),
          {"bytes": 4.0 * x.numel()})
    return y


def layernorm_bwd(x, dy, gamma, eps: float, dgamma=None, dbeta=None, grad_scale: float = 1.0, accumulate: bool = False):
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    x, dy = x.contiguous(), dy.contiguous()
    dx = torch.empty_like(x)
    ws = _train_ws(Cc, 2 * rows, x.device)
    _call("icaf_layernorm_bwd", _lib.lib().icaf_layernorm_bwd,
          (_ptr(x), _ptr(dy), _ptr(gamma), _ptr(dx), _ptr(dgamma), _ptr(dbeta), rows, Cc, float(eps), float(grad_scale), int(accumulate), _ptr(ws),
           C.c_size_t(ws.numel() * 4)), {"bytes": 8.0 * x.numel()})
    return dx


def dot(x, y, out: Optional[torch.Tensor] = None, scale: float = 1.0):
    """<x, y> (fp32, one element) of equally shaped fp16 tensors; accumulates into `out` when given."""
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    x, y = x.contiguous(), y.contiguous()
    acc = out is not None
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=x.device)
    ws = _train_ws(Cc, 0, x.device)
    _call("icaf_dot", _lib.lib().icaf_dot, (_ptr(x), _ptr(y), rows, Cc, _ptr(out), float(scale), int(acc), _ptr(ws), C.c_size_t(ws.numel() * 4)),
          {"bytes": 4.0 * x.numel()})
    return out


def upsample2x_bwd(dy):
    B, H2, W2, Cc = dy.shape
    dy = dy.contiguous()
    dx = torch.empty(B, H2 // 2, W2 // 2, Cc, dtype=torch.float16, device=dy.device)
    _call("icaf_upsample2x_bwd", _lib.lib().icaf_upsample2x_bwd, (_ptr(dy), _ptr(dx), B, H2 // 2, W2 // 2, Cc), {"bytes": 2.5 * dy.numel()})
    return dx


def maxpool5_bwd(x, dy):
    B, H, W, Cc = x.shape
    x, dy = x.contiguous(), dy.contiguous()
    dx = torch.empty_like(x)
    ws = torch.empty((x.numel() + 7) // 8, dtype=torch.int64, device=x.device)
    _call("icaf_maxpool5_bwd", _lib.lib().icaf_maxpool5_bwd, (_ptr(x), _ptr(dy), _ptr(dx), B, H, W, Cc, _ptr(ws), C.c_size_t(ws.numel() * 8)),
          {"bytes": 7.0 * x.numel()})
    return dx


class OptimTable:
    """A device table of icaf_optim_tensor entries (include/icaf_b200.h) for the optimiser-step kernels.  `rows` are tuples
    (p, g, m, v, step) of dense fp32 tensors of one size (None where a kernel does not read the field); `ranges` names
    consecutive row ranges (the parameter groups) that a launch may walk on their own.  The table holds the addresses of
    these very tensors: rebuild it when one of them is reallocated."""

    def __init__(self, rows, device, ranges=None):
        from .datasets import ParamBlock
        n = len(rows)
        if n < 1:
            raise ValueError("OptimTable: no tensors")
        structs = (_lib.OptimTensor * n)()
        self.chunk0, c = [], 0
        for i, row in enumerate(rows):
            p = row[0]
            for t in row:
                if t is None:
                    continue
                if t.dtype != torch.float32 or not t.is_contiguous() or not on_device(t) or (_DRY is None and t.device != p.device):
                    raise ValueError(f"OptimTable: row {i}: every tensor must be dense fp32 on the device, got {t.dtype} "
                                     f"{tuple(t.shape)} on {t.device}")
                if t is not row[4] and t.numel() != p.numel():
                    raise ValueError(f"OptimTable: row {i}: tensors of {t.numel()} and {p.numel()} elements")
            if row[4] is not None and row[4].numel() != 1:
                raise ValueError(f"OptimTable: row {i}: the step count must be one element")
            structs[i] = _lib.OptimTensor(*[_addr(t) or 0 for t in row[:5]], p.numel(), c)
            self.chunk0.append(c)
            c += -(-p.numel() // _lib.OPTIM_CHUNK)
        self.chunk0.append(c)
        self.rows = list(rows)              # keeps the tensors the table points at alive
        self.n = n
        self.ranges = dict(ranges or {})
        self.block = ParamBlock().upload(structs, [], int(_lib.lib().icaf_optim_table_bytes(n)), device)

    def span(self, name=None):
        """(table address, table bytes, tensors, chunks) of the named range, or of the whole table."""
        lo, hi = self.ranges[name] if name is not None else (0, self.n)
        entry = C.sizeof(_lib.OptimTensor)
        addr = (_addr(self.block) or 0) + lo * entry
        return C.c_void_p(addr), C.c_size_t(self.block.numel() - lo * entry), hi - lo, self.chunk0[hi] - self.chunk0[lo]


def _optim_bytes(tab: OptimTable, name, tensors_per_row: int) -> float:
    return 4.0 * tensors_per_row * sum(tab.rows[i][0].numel() for i in range(*(tab.ranges[name] if name is not None else (0, tab.n))))


def amp_unscale(tab: OptimTable, scale: torch.Tensor, found_inf: torch.Tensor) -> None:
    """GradScaler.unscale_ over the `g` tensors of the table; sets found_inf (fp32, one element) on a non-finite element."""
    _call("icaf_amp_unscale", _lib.lib().icaf_amp_unscale, (*tab.span(), _ptr(scale), _ptr(found_inf)), {"bytes": _optim_bytes(tab, None, 2)})


def sgd_step(tab: OptimTable, group: int, hyper: torch.Tensor, found_inf: torch.Tensor) -> None:
    """Nesterov SGD over the table range `group` with the scalars of row `group` of hyper (float64 (groups, OPTIM_HYPER))."""
    _call("icaf_sgd_step", _lib.lib().icaf_sgd_step, (*tab.span(group), _ptr(hyper), int(group), int(hyper.shape[0]), _ptr(found_inf)),
          {"bytes": _optim_bytes(tab, group, 5)})


def adam_step(tab: OptimTable, group: int, hyper: torch.Tensor, bias_corr: torch.Tensor, found_inf: torch.Tensor) -> None:
    """Adam over the table range `group`; bias_corr is float64 (groups, steps, 2) of torch's (bc1, bc2_sqrt) per step."""
    _call("icaf_adam_step", _lib.lib().icaf_adam_step,
          (*tab.span(group), _ptr(hyper), int(group), int(hyper.shape[0]), _ptr(bias_corr), int(bias_corr.shape[1]), _ptr(found_inf)),
          {"bytes": _optim_bytes(tab, group, 7)})


def amp_update_scale(scale: torch.Tensor, growth_tracker: torch.Tensor, found_inf: torch.Tensor, growth_factor: float,
                     backoff_factor: float, growth_interval: int) -> None:
    _call("icaf_amp_update_scale", _lib.lib().icaf_amp_update_scale,
          (_ptr(scale), _ptr(growth_tracker), _ptr(found_inf), float(growth_factor), float(backoff_factor), int(growth_interval)), {})


def ema_update(tab: OptimTable, decay: torch.Tensor) -> None:
    """ModelEMA.update over the table's (p = EMA entry, g = model entry) rows with d = decay[0] (device float64)."""
    _call("icaf_ema_update", _lib.lib().icaf_ema_update, (*tab.span(), _ptr(decay)), {"bytes": _optim_bytes(tab, None, 3)})


# ---------------------------------------------------------------------------------------------------------------
# Validation exchange buffers: a validation split over ranks packs its per-image results, the buffers cross ranks, and the
# merge puts them back in the one-process image order (include/icaf_b200.h, icaf_val_pack / icaf_val_merge).
def val_pack_bytes(n_images: int, max_det: int, native: bool) -> int:
    """Bytes of the exchange buffer of n_images images of at most max_det rows (a pure function of its arguments)."""
    return int(_lib.lib().icaf_val_pack_bytes(int(n_images), int(max_det), _lib.VAL_PACK_NATIVE if native else 0))


def val_pack(batches, niou: int, native: bool = False, positions=None) -> torch.Tensor:
    """Pack the per-image results of `batches` into one exchange buffer, in the given order.  batches: [(det fp32 (B, max_det,
    6), count int32 (B,), correct uint8 / bool (B, max_det, niou), native fp32 (B, max_det, 4) or None, image0)], image0 the
    global index of the batch's first image.  positions: the images' KAIST annotation positions (int32, one per image) or
    None.  Returns the int32 device buffer (its header's word 3 is the number of words written); no host sync."""
    if not batches:
        raise ValueError("val_pack: no batches")
    structs = (_lib.ValBatch * len(batches))()
    n_images, max_det, device = 0, 1, batches[0][0].device
    for k, (det, count, correct, nat, image0) in enumerate(batches):
        if det.dim() != 3 or det.shape[2] != 6 or det.dtype != torch.float32 or not det.is_contiguous() or not on_device(det):
            raise ValueError(f"val_pack: batch {k}: det must be contiguous CUDA fp32 (B, max_det, 6), got {det.dtype} {tuple(det.shape)}")
        B, md = int(det.shape[0]), int(det.shape[1])
        if tuple(count.shape) != (B,) or count.dtype != torch.int32 or not count.is_contiguous():
            raise ValueError(f"val_pack: batch {k}: count must be int32 ({B},)")
        if tuple(correct.shape) != (B, md, niou) or correct.dtype not in (torch.uint8, torch.bool) or not correct.is_contiguous():
            raise ValueError(f"val_pack: batch {k}: correct must be contiguous uint8 / bool {(B, md, niou)}")
        if native and (nat is None or tuple(nat.shape) != (B, md, 4) or nat.dtype != torch.float32 or not nat.is_contiguous()):
            raise ValueError(f"val_pack: batch {k}: native must be contiguous fp32 {(B, md, 4)}")
        for t in (count, correct) + ((nat,) if native else ()):
            if t.device != det.device or (_DRY is None and t.device != device):
                raise ValueError(f"val_pack: batch {k}: tensors on {t.device} and {det.device} (batch 0 on {device})")
        structs[k] = _lib.ValBatch(_addr(det), _addr(count), _addr(correct), _addr(nat) if native else None, int(image0), B, md,
                                   n_images)
        n_images += B
        max_det = max(max_det, md)
    flags = (_lib.VAL_PACK_NATIVE if native else 0) | (_lib.VAL_PACK_POS if positions is not None else 0)
    regions = ()
    if positions is not None:
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.int32).reshape(-1))
        if pos.size != n_images:
            raise ValueError(f"val_pack: {pos.size} positions for {n_images} images")
        regions = (pos,)
    from .datasets import ParamBlock
    nbytes = int(_lib.lib().icaf_val_pack_params_bytes(len(batches), n_images, flags))
    if nbytes == 0:
        raise ValueError(f"val_pack: unsupported sizes ({len(batches)} batches, {n_images} images)")
    params = ParamBlock().upload(structs, regions, nbytes, device)
    out_bytes = val_pack_bytes(n_images, max_det, native)
    if out_bytes == 0:
        raise ValueError(f"val_pack: {n_images} images of {max_det} rows do not fit an int32-indexed buffer")
    out = torch.empty(out_bytes // 4, dtype=torch.int32, device=device)
    _call("icaf_val_pack", _lib.lib().icaf_val_pack,
          (_ptr(params), C.c_size_t(nbytes), len(batches), n_images, int(niou), flags, _ptr(out), C.c_size_t(out_bytes)),
          {"bytes": float(out_bytes)})
    out._icaf_params = params                  # the block must outlive the launch
    return out


def val_merge(bufs: torch.Tensor, n_images: int, n_rows: int, niou: int, native: bool = False, mr=None) -> dict:
    """Merge exchange buffers (int32 (n_bufs, words), one per row, as val_pack wrote them) into flat arrays in global image
    order: correct uint8 (n_rows, niou), conf / pcls fp32 (n_rows,), native fp32 (n_rows, 4) or None, counts int32
    (n_images,), offsets int32 (n_images + 1,) and status int32 (4,) (see :func:`val_merge_check`).  mr: (images, max_det)
    to also write the icaf_kaist_round_detections rows / span of every image with a position ('mr_rows', 'mr_span').
    No host sync."""
    if bufs.dim() != 2 or bufs.dtype != torch.int32 or not bufs.is_contiguous() or not on_device(bufs):
        raise ValueError(f"val_merge: bufs must be contiguous CUDA int32 (n_bufs, words), got {bufs.dtype} {tuple(bufs.shape)}")
    if n_images < 1 or n_rows < 0:
        raise ValueError(f"val_merge: {n_images} images, {n_rows} rows")
    dev = bufs.device
    out = dict(correct=torch.empty(n_rows, niou, dtype=torch.uint8, device=dev), conf=torch.empty(n_rows, dtype=torch.float32, device=dev),
               pcls=torch.empty(n_rows, dtype=torch.float32, device=dev),
               native=torch.empty(n_rows, 4, dtype=torch.float32, device=dev) if native else None,
               counts=torch.empty(n_images, dtype=torch.int32, device=dev), offsets=torch.empty(n_images + 1, dtype=torch.int32, device=dev),
               status=torch.empty(4, dtype=torch.int32, device=dev), mr_rows=None, mr_span=None)
    mr_images = mr_max_det = 0
    if mr is not None:
        mr_images, mr_max_det = int(mr[0]), int(mr[1])
        out["mr_rows"] = torch.empty(mr_images * mr_max_det, 5, dtype=torch.float64, device=dev)
        out["mr_span"] = torch.zeros(mr_images, 2, dtype=torch.int32, device=dev)
    need = int(_lib.lib().icaf_val_merge_workspace_bytes(int(n_images)))
    ws = torch.empty(max(need // 16, 1), 4, dtype=torch.int32, device=dev)
    flags = _lib.VAL_PACK_NATIVE if native else 0
    _call("icaf_val_merge", _lib.lib().icaf_val_merge,
          (_ptr(bufs), int(bufs.shape[0]), int(bufs.shape[1]), int(n_images), int(n_rows), int(niou), flags, _ptr(out["correct"]),
           _ptr(out["conf"]), _ptr(out["pcls"]), _ptr(out["native"]), _ptr(out["counts"]), _ptr(out["offsets"]), _ptr(out["status"]),
           _ptr(out["mr_rows"]), _ptr(out["mr_span"]), mr_images, mr_max_det, _ptr(ws), C.c_size_t(ws.numel() * 4)),
          {"bytes": float(bufs.numel() * 4 + n_rows * (niou + 8 + (16 if native else 0)))})
    return out


def val_merge_check(status, n_rows: int) -> None:
    """Refuse a merge whose status (host copy of val_merge's 'status') shows a missing, duplicated or malformed image."""
    missing, dup, bad, rows = (int(v) for v in status)
    if missing or dup or bad or rows != n_rows:
        raise ValueError(f"val_merge: {missing} image(s) missing from every buffer, {dup} in more than one, {bad} malformed "
                         f"entries, {rows} rows for {n_rows} expected")
