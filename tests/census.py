"""Launch census (test helper): every C-ABI call the detectors make, replayed alone against a plain high-precision reference.

``walk`` runs the real inference or training forward (and backward) of a detector on ``meta`` tensors under
``ops.dry_run()`` and returns the recorded calls.  ``key`` reduces a record to its entry point plus every integer and float
argument (geometry, channel pitches, epilogue flags, scales; never pointers), which is what decides the kernel, tile shape,
staging mode and split count a launch gets.  ``REPLAYED`` maps each entry point to a builder that allocates random operands
of exactly the recorded shapes and pitches, issues the same call through ``ops``, and returns ``Check`` objects pairing the
device result with its reference.  ``NOT_REPLAYED`` lists the remaining entry points with the reason.

Builders also run on ``meta`` tensors under a dry run (tests/test_census_cpu.py): there they only issue the call, and the
references, which are lazy, are never evaluated.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
import zlib
from dataclasses import dataclass
from typing import Callable, List, Union

import numpy as np
import torch
import torch.nn.functional as F

from icafusion_b200 import _lib, ops


# ---------------------------------------------------------------------------------------------------------------
# Configurations and walks
@dataclass(frozen=True)
class Config:
    kind: str        # "infer" | "train"
    size: str        # n s m l x
    dataset: str     # "kaist" | "FLIR"
    B: int
    H: int
    W: int

    @property
    def id(self) -> str:
        return f"yolov5{self.size}-{self.dataset.lower()}-{self.H}x{self.W}-b{self.B}-{self.kind}"


CONFIGS = [Config("infer", s, ds, B, H, W) for s in "nsmlx" for ds, H, W in (("kaist", 512, 640), ("FLIR", 320, 320)) for B in (1, 16)] + \
          [Config("train", s, "kaist", B, 512, 640) for s in "nsl" for B in (2, 16)] + \
          [Config("infer", s, "FLIR", B, 512, 640) for s in "nsmlx" for B in (1, 16)] + \
          [Config("infer", s, ds, B, 544, 672) for s in "nsmlx" for ds in ("kaist", "FLIR") for B in (1, 32)] + \
          [Config("train", s, "kaist", B, 640, 640) for s in "nsl" for B in (8, 16, 3)] + \
          [Config("train", "s", "FLIR", 8, 640, 640)]
# Inference: detect.py letterboxes the 512x640 frames of both datasets to 512x640; test.py's rectangular batches
# (rect=True, pad=0.5) make them 544x672, at test.py's batch 32 and train.py's validation batch 1.  Training: train.py's mosaic
# batches are img_size x img_size = 640x640 at its default batch 8, at 16 and with a ragged last batch of 3.
# Training of yolov5m / yolov5x is not built: the attention backward has no head dim 24 / 48 / 96 / 160.

TARGETS_PER_IMAGE = 16      # a mosaic stitches four frames of a few pedestrians each


def walk(kind: str, cfg: str, B: int, H: int, W: int):
    """Records [(entry point, ctypes args, work)] of one dry-run walk of model `cfg` (e.g. 'yolov5s_Transfusion_kaist').
    A training walk is TrainStep's: forward, ComputeLoss with train.py's hyper-parameters as TrainStep scales them, and the
    backward from the loss."""
    from icafusion_b200 import Model
    rgb = torch.empty(B, 3, H, W, dtype=torch.uint8, device="meta")
    if kind == "infer":
        m = Model(cfg).eval().fuse().half()
        with torch.no_grad(), ops.dry_run() as dr:
            m(rgb, rgb)
    elif kind == "train":
        from icafusion_b200.trainer import TrainStep
        m = Model(cfg).train()
        step = TrainStep(m, imgsz=max(H, W), amp_scale=False)       # ComputeLoss reads the anchors before the move to meta
        m.to("meta")
        targets = torch.empty(TARGETS_PER_IMAGE * B, 6, device="meta")
        with ops.dry_run() as dr:
            loss, _ = step.compute_loss(m(rgb, rgb), targets)
            loss.backward()
    else:
        raise ValueError(kind)
    return dr.records


@functools.lru_cache(maxsize=None)
def walk_config(c: Config):
    return walk(c.kind, f"yolov5{c.size}_Transfusion_{c.dataset}", c.B, c.H, c.W)


# ---------------------------------------------------------------------------------------------------------------
# Dedupe key
# Arguments that are not geometry: the dropout probability and mask seed of the training attention, and the mask seed of the
# element-wise dropout.  The replay chooses them itself: each dropout record is replayed at p = 0 and at its recorded p, with
# a seed from its key, against the mask restated on the host (tests/dropout_mask.py).  A seed is drawn per call, so keying
# it would also make two walks of one configuration differ.
_NOT_KEYED = {"icaf_cross_attention_train": (9, 10), "icaf_cross_attention_bwd": (13, 14), "icaf_eltwise": (6,)}


def _value(v):
    """A struct field as a plain value: nested arrays (LossHyp.balance) as tuples, which compare by content."""
    return tuple(v) if isinstance(v, C.Array) else v


def _fields(s):
    """The non-pointer fields of a struct: ConvGeom; ConvIO / BottleneckIO channel pitches, ln_parts, ln_eps; LossHyp."""
    return tuple(_value(getattr(s, f)) for f, t in s._fields_ if t is not C.c_void_p)


def key(rec) -> tuple:
    name, args, _ = rec
    skip = _NOT_KEYED.get(name, ())
    out = [name]
    for i, a in enumerate(args):
        if i in skip or a is None or isinstance(a, C.c_void_p):
            continue
        if isinstance(a, (int, float)):
            out.append(a)
        elif isinstance(a, C._SimpleCData):
            out.append(a.value)
        elif isinstance(a, C.Array):
            if issubclass(a._type_, C.Structure):
                out.append(tuple(_fields(s) for s in a))
            elif a._type_ is C.c_void_p:                  # per-level pointers (compute_loss): not geometry
                continue
            else:
                out.append(tuple(a))
        elif type(a).__name__ == "CArgObject":           # byref(ConvGeom), byref(LossHyp)
            out.append(_fields(a._obj))
        else:
            raise TypeError(f"{name}: argument {i} of type {type(a).__name__} has no key form")
    return tuple(out)


def unique(records):
    """{key: record} in first-issue order."""
    out = {}
    for r in records:
        out.setdefault(key(r), r)
    return out


def describe(rec) -> str:
    """A short geometry line for failure tables."""
    name, args, _ = rec
    if name in ("icaf_conv2d_fwd", "icaf_conv2d_wgrad"):
        g = args[0]._obj
        s = f"B{g.B} {g.Hi}x{g.Wi}x{g.Cin}->{g.Ho}x{g.Wo}x{g.Cout} k{g.kh}s{g.stride}p{g.pad} act{g.act} epi{g.epi}"
        if name == "icaf_conv2d_fwd":
            s += f" n{args[2]} ld " + ",".join(f"{io.x_ld}/{io.y_ld}/{io.res_ld}" for io in args[1])
        else:
            s += f" ld {args[2]}/{args[4]} scale {args[6]:g} acc {args[7]}"
        return s
    return " ".join(str(v) for v in key(rec)[1:])


# ---------------------------------------------------------------------------------------------------------------
# Checks
Lazy = Union[torch.Tensor, Callable[[], torch.Tensor]]


@dataclass
class Check:
    """One comparison.  mode: 'norm' max|a-b|/max|b|; 'chan' the same per index of the last dim, each against
    max(max|b[..., c]|, 1e-2 max|b|); 'l2' ||a-b||/||b||; 'exact' bit-identical (error 0 or inf); 'close'
    max |a-b| / (atol + rtol |b|) with tol = 1 (atol, rtol in `arg`)."""
    what: str
    got: Lazy
    ref: Lazy
    tol: float
    mode: str = "norm"
    arg: tuple = ()

    def error(self) -> float:
        a = self.got() if callable(self.got) else self.got
        b = self.ref() if callable(self.ref) else self.ref
        assert tuple(a.shape) == tuple(b.shape), (self.what, tuple(a.shape), tuple(b.shape))
        if self.mode == "exact":
            if a.dtype != b.dtype:
                return math.inf
            if a.is_floating_point():          # compare bits, so that NaN patterns compare too
                it = {torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[a.dtype]
                a, b = a.contiguous().view(it), b.contiguous().view(it)
            return 0.0 if torch.equal(a, b) else math.inf
        a, b = a.double(), b.double()
        if not bool(torch.isfinite(a).all()):
            return math.inf
        d = (a - b).abs()
        if self.mode == "norm":
            return float(d.max() / b.abs().max().clamp_min(1e-30)) if d.numel() else 0.0
        if self.mode == "chan":
            c = a.shape[-1]
            dm = d.reshape(-1, c).amax(0)
            bm = b.abs().reshape(-1, c).amax(0)
            return float((dm / bm.clamp_min(1e-2 * float(bm.max())).clamp_min(1e-30)).max())
        if self.mode == "l2":
            return float(d.norm() / b.norm().clamp_min(1e-30))
        if self.mode == "close":
            atol, rtol = self.arg
            return float((d / (atol + rtol * b.abs())).max())
        raise ValueError(self.mode)


NAN16 = 0x7E00


class Operands:
    """Seeded operand factory: CUDA tensors from a CUDA generator, or bare ``meta`` tensors for a dry run."""

    def __init__(self, device, seed: int):
        self.dev = torch.device(device)
        self.meta = self.dev.type == "meta"
        self.seed = seed
        self.gen = None if self.meta else torch.Generator(device=self.dev).manual_seed(seed)

    def randn(self, *shape, dtype=torch.float16, scale=1.0):
        if self.meta:
            return torch.empty(*shape, dtype=dtype, device=self.dev)
        return (torch.randn(*shape, generator=self.gen, device=self.dev) * scale).to(dtype)

    def rand(self, *shape):
        if self.meta:
            return torch.empty(*shape, device=self.dev)
        return torch.rand(*shape, generator=self.gen, device=self.dev)

    def zeros(self, *shape, dtype=torch.float16):
        return torch.zeros(*shape, dtype=dtype, device=self.dev)

    def nan(self, *shape, dtype=torch.float16):
        """Buffer pre-filled with NaN (fp16 0x7E00 / fp32 NaN): an element the kernel does not write fails the finiteness check."""
        if dtype == torch.float16:
            return torch.full(shape, NAN16, dtype=torch.int16, device=self.dev).view(torch.float16)
        return torch.full(shape, float("nan"), dtype=dtype, device=self.dev)

    def view_in(self, buf, start: int, width: int):
        return buf[..., start:start + width]


def seed_of(k: tuple) -> int:
    return zlib.crc32(repr(k).encode())


def _slot(ld: int, width: int) -> int:
    """Channel offset of a `width`-channel view inside an `ld`-channel buffer: the last 16-byte aligned slot, so that a
    neighbour lies on both sides whenever the pitch leaves room."""
    return (ld - width) // 8 * 8


def _neighbours(buf, start: int, width: int):
    """The channels of `buf` outside [start, start + width), flattened (empty when there are none)."""
    parts = [buf[..., :start].reshape(-1), buf[..., start + width:].reshape(-1)]
    return torch.cat(parts)


def _untouched(what, buf, start, width) -> List[Check]:
    if buf.shape[-1] == width:
        return []
    def got():
        return _neighbours(buf, start, width)
    def ref():
        n = _neighbours(buf, start, width)
        if n.dtype == torch.float16:
            return torch.full(n.shape, NAN16, dtype=torch.int16, device=n.device).view(torch.float16)
        return torch.full(n.shape, float("nan"), dtype=n.dtype, device=n.device)
    return [Check(what + " neighbours unchanged", got, ref, 0.0, "exact")]


def _zero(what, got) -> Check:
    """Rows the kernel must write as zero (either sign)."""
    return Check(what, got, lambda: torch.zeros_like(got()), 0.0)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _act(y, act):
    return F.silu(y) if act == ops.ACT_SILU else F.gelu(y) if act == ops.ACT_GELU else y


# ---------------------------------------------------------------------------------------------------------------
# Builders: (record, Operands) -> [Check]
def _conv_fwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    g, ios, n = args[0]._obj, args[1], args[2]
    B, Hi, Wi, Cin, Ho, Wo, Cout = g.B, g.Hi, g.Wi, g.Cin, g.Ho, g.Wo, g.Cout
    K, M = g.kh * g.kw * Cin, B * Ho * Wo
    epi = g.epi
    bias_row, add_res, scaled = bool(epi & ops.EPI_BIAS_ROW), bool(epi & ops.EPI_ADD_RES), bool(epi & ops.EPI_SCALED_RES)
    ln, emit = bool(epi & ops.EPI_LN_FOLD), bool(epi & ops.EPI_EMIT_STATS)
    xs, packs, outs, ybufs, res, sc, lns, sos, probs = [], [], [], [], [], [], [], [], []
    for i in range(n):
        io = ios[i]
        w = R.zeros(g.w_rows, g.k_pad)
        w[:Cout, :K] = R.randn(Cout, K, scale=1.0 / math.sqrt(K))
        bias = R.randn(M if bias_row else Cout, dtype=torch.float32, scale=0.5)
        pk = ops.PackedConv(w, bias, Cin, Cout, g.kh, g.kw, g.stride, g.pad, g.act, is_weight=not bias_row)
        xbuf = R.randn(B, Hi, Wi, io.x_ld)
        xo = _slot(io.x_ld, Cin)
        if ln:
            rows = B * Hi * Wi
            xbuf = (xbuf.float() * (0.5 + R.rand(rows, 1).view(B, Hi, Wi, 1)) + 0.3 * R.randn(rows, 1, dtype=torch.float32).view(B, Hi, Wi, 1)).half()
        x = R.view_in(xbuf, xo, Cin)
        if ln:
            parts = io.ln_parts
            xd = x.reshape(M, parts, Cin // parts).double()
            st = torch.stack([xd.sum(2), (xd * xd).sum(2)], 2).float().contiguous()
            pk.colsum = w.float().sum(1).contiguous()
            pk.ln_eps = io.ln_eps
            lns.append(st)
        ybuf = R.nan(B, Ho, Wo, io.y_ld)
        yo = _slot(io.y_ld, Cout)
        r = None
        if add_res or scaled:
            rbuf = R.randn(B, Ho, Wo, io.res_ld)
            r = R.view_in(rbuf, _slot(io.res_ld, Cout), Cout)
            res.append(r)
        if scaled:
            ab = 0.5 + R.rand(2)
            sc.append((ab[0:1], ab[1:2]))
        if emit:
            sos.append(R.nan(M, (Cout + 31) // 32, 2, dtype=torch.float32))
        xs.append(x)
        packs.append(pk)
        ybufs.append((ybuf, yo))
        outs.append(R.view_in(ybuf, yo, Cout))
        probs.append((x, w, bias, r, sc[-1] if scaled else None))
    ops.conv2d(xs, packs, outs, res or None, sc or None, bias_row, ln_stats=lns or None, stats_out=sos or None)
    if R.meta:
        return []

    checks = []
    for i, (x, w, bias, r, ab) in enumerate(probs):
        def ref(x=x, w=w, bias=bias, r=r, ab=ab, eps=ios[i].ln_eps):
            xf = x.float()
            if ln:
                xd = x.double()
                mu = xd.mean(-1, keepdim=True)
                var = (xd * xd).mean(-1, keepdim=True) - mu * mu
                xf = ((xd - mu) / torch.sqrt(var + eps)).float()
            wf = w[:Cout, :K].float().view(Cout, g.kh, g.kw, Cin).permute(0, 3, 1, 2)
            y = F.conv2d(_nchw(xf), wf, None, stride=g.stride, padding=g.pad).permute(0, 2, 3, 1)
            y = y + (bias.view(B, Ho, Wo, 1) if bias_row else bias)
            y = _act(y, g.act)
            if scaled:
                y = ab[0] * r.float() + ab[1] * y
            elif add_res:
                y = y + r.float()
            return y
        ref = functools.lru_cache(None)(ref)
        tol = 1e-3 if ln else 1.5e-3
        y = outs[i]
        checks += [Check(f"y[{i}]", y, ref, tol), Check(f"y[{i}] per channel", y, ref, tol, "chan")]
        checks += _untouched(f"y[{i}]", *ybufs[i], Cout)
        if emit:
            so = sos[i]
            checks.append(Check(f"stats[{i}] row sums", lambda so=so: so.sum(1).double(),
                                lambda y=y: torch.stack([y.double().reshape(M, Cout).sum(1), (y.double().reshape(M, Cout) ** 2).sum(1)], 1),
                                1.0, "close", (1e-2, 1e-4)))
    return checks


def _bottleneck(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    B, H, W, ios, n = args
    xs, p1s, p3s, outs, bufs, ws = [], [], [], [], [], []
    for i in range(n):
        w1 = R.randn(64, 64, 1, 1, scale=1 / 8).float()
        w3 = R.randn(64, 64, 3, 3, scale=1 / 24).float()
        b1, b2 = R.randn(64, dtype=torch.float32, scale=0.5), R.randn(64, dtype=torch.float32, scale=0.5)
        p1s.append(ops.pack_conv_weight(w1, b1, 1, 0, ops.ACT_SILU, device=R.dev))
        p3s.append(ops.pack_conv_weight(w3, b2, 1, 1, ops.ACT_SILU, device=R.dev))
        xbuf = R.randn(B, H, W, ios[i].x_ld)
        xs.append(R.view_in(xbuf, _slot(ios[i].x_ld, 64), 64))
        ybuf = R.nan(B, H, W, ios[i].y_ld)
        yo = _slot(ios[i].y_ld, 64)
        bufs.append((ybuf, yo))
        outs.append(R.view_in(ybuf, yo, 64))
        ws.append((w1, b1, w3, b2))
    ops.bottleneck(xs, p1s, p3s, outs)
    if R.meta:
        return []
    checks = []
    for i in range(n):
        def ref(x=xs[i], w=ws[i]):
            w1, b1, w3, b2 = w
            xf = _nchw(x.float())
            h = F.silu(F.conv2d(xf, w1, b1))
            return (xf + F.silu(F.conv2d(h, w3, b2, padding=1))).permute(0, 2, 3, 1)
        checks.append(Check(f"y[{i}]", outs[i], functools.lru_cache(None)(ref), 1.5e-3))
        checks += _untouched(f"y[{i}]", *bufs[i], 64)
    return checks


def _wgrad_operands(rec, R: Operands):
    _, args, _ = rec
    g = args[0]._obj
    x = R.view_in(R.randn(g.B, g.Hi, g.Wi, args[2]), _slot(args[2], g.Cin), g.Cin)
    dy = R.view_in(R.randn(g.B, g.Ho, g.Wo, args[4], scale=0.1), _slot(args[4], g.Cout), g.Cout)
    return g, x, dy


def _wgrad(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    g, x, dy = _wgrad_operands(rec, R)
    scale, acc = args[6], args[7]
    shape = (g.Cout, g.Cin, g.kh, g.kw)
    pre = R.randn(*shape, dtype=torch.float32, scale=0.1 * math.sqrt(g.B * g.Ho * g.Wo) * abs(scale)) if acc else None
    dw = ops.conv2d_wgrad(x, dy, g.kh, g.kw, g.stride, g.pad, scale, pre.clone() if acc else None)
    dw2 = ops.conv2d_wgrad(x, dy, g.kh, g.kw, g.stride, g.pad, scale, pre.clone() if acc else None)
    if R.meta:
        return []
    checks = _dgrad(rec, R)

    @functools.lru_cache(None)
    def ref():
        r = torch.nn.grad.conv2d_weight(_nchw(x.float()), shape, _nchw(dy.float()), stride=g.stride, padding=g.pad) * scale
        return r + pre if acc else r
    rows = lambda t: t.reshape(g.Cout, -1).t()            # noqa: E731  (per Cout row)
    return [Check("dW", dw, ref, 1e-3), Check("dW per Cout row", lambda: rows(dw), lambda: rows(ref()), 1e-3, "chan"),
            Check("dW repeat", dw2, dw, 0.0, "exact")] + checks


def is_linear(g) -> bool:
    """Linear layers run as convolutions with rows as pixels: one image, one row, 1x1."""
    return g.B == 1 and g.Hi == 1 and g.kh == 1 and g.kw == 1


def _dgrad(rec, R: Operands) -> List[Check]:
    """Data gradient of the layer a weight-gradient record belongs to (the product issues it as a conv2d_fwd on the filter
    from pack_weight_pair, over a zero-stuffed map for stride 2)."""
    g = rec[1][0]._obj
    if is_linear(g) or g.Cin % 8:
        return []
    w = R.randn(g.Cout, g.Cin, g.kh, g.kw, dtype=torch.float32, scale=1 / math.sqrt(g.Cin * g.kh * g.kw)).half().float().contiguous()
    dy = R.randn(g.B, g.Ho, g.Wo, g.Cout, scale=0.1)
    _, pd = ops.pack_weight_pair(w, g.stride, g.pad)
    dx = ops.conv2d_dgrad(dy, w, g.stride, g.pad, (g.Hi, g.Wi), packed=pd)
    ref = lambda: torch.nn.grad.conv2d_input((g.B, g.Cin, g.Hi, g.Wi), w, _nchw(dy.float()), stride=g.stride,   # noqa: E731
                                             padding=g.pad).permute(0, 2, 3, 1)
    return [Check("dX", dx, ref, 1.5e-3)]


def _pack_pair(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    cout, cin, kh, kw, rows_f, kpad_f = args[1:7]
    chan_d, rows_d, kpad_d = args[8:11]
    w = R.randn(cout, cin, kh, kw, dtype=torch.float32).contiguous()
    of, od = R.nan(rows_f, kpad_f), R.nan(rows_d, kpad_d)
    L = _lib.lib()
    ops._call("icaf_pack_weight_pair", L.icaf_pack_weight_pair,
              (ops._ptr(w), cout, cin, kh, kw, rows_f, kpad_f, ops._ptr(of), chan_d, rows_d, kpad_d, ops._ptr(od)), {})
    if R.meta:
        return []

    def ref_f():
        r = torch.zeros(rows_f, kpad_f, dtype=torch.float16, device=w.device)
        r[:cout, :kh * kw * cin] = w.permute(0, 2, 3, 1).reshape(cout, -1).half()
        return r

    def ref_d():     # W'[c][ky][kx][n] = W[n][c][kh-1-ky][kw-1-kx], n padded to chan_d
        t = torch.zeros(cin, kh, kw, chan_d, device=w.device)
        t[..., :cout] = w.flip(2, 3).permute(1, 2, 3, 0)
        r = torch.zeros(rows_d, kpad_d, dtype=torch.float16, device=w.device)
        r[:cin, :kh * kw * chan_d] = t.reshape(cin, -1).half()
        return r
    return [Check("forward bank", of, ref_f, 0.0, "exact"), Check("dgrad bank", od, ref_d, 0.0, "exact")]


def _bn_input(R: Operands, rows, Cc):
    """Per-channel offsets up to +-4 sigma and scales from 1/4 to 4: probes the E[x^2] - mean^2 variance."""
    s = 2.0 ** (4 * R.rand(Cc) - 2)
    o = (8 * R.rand(Cc) - 4) * s
    return (R.randn(rows, Cc, dtype=torch.float32) * s + o).half()


def _bn_params(R: Operands, Cc):
    return 1 + 0.2 * R.randn(Cc, dtype=torch.float32), 0.2 * R.randn(Cc, dtype=torch.float32)


def _bn_fwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    rows, Cc, eps, mom, act = args[8:13]
    x = _bn_input(R, rows, Cc)
    gamma, beta = _bn_params(R, Cc)
    rm0, rv0 = R.randn(Cc, dtype=torch.float32, scale=0.3), 0.5 + R.rand(Cc)
    rm, rv = rm0.clone(), rv0.clone()
    y, sm, si = ops.bn_act_fwd(x, gamma, beta, rm, rv, eps, mom, act)
    rm2, rv2 = rm0.clone(), rv0.clone()
    y2, _, _ = ops.bn_act_fwd(x, gamma, beta, rm2, rv2, eps, mom, act)
    if R.meta:
        return []

    @functools.lru_cache(None)
    def ref():
        rmr, rvr = rm0.double().clone(), rv0.double().clone()
        yr = F.batch_norm(x.double(), rmr, rvr, gamma.double(), beta.double(), True, mom, eps)
        return _act(yr, act), rmr, rvr
    return [Check("y", y, lambda: ref()[0], 1e-3), Check("running mean", rm, lambda: ref()[1], 1e-4),
            Check("running var", rv, lambda: ref()[2], 1e-4), Check("y repeat", y2, y, 0.0, "exact"),
            Check("running var repeat", rv2, rv, 0.0, "exact")]


def _bn_bwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    rows, Cc, act, gs, acc = args[9:14]
    x = _bn_input(R, rows, Cc)
    gamma, beta = _bn_params(R, Cc)
    dy = R.randn(rows, Cc, scale=0.1)
    eps = 1e-3
    if R.meta:
        sm, si = R.zeros(Cc, dtype=torch.float32), R.zeros(Cc, dtype=torch.float32)
    else:
        xd = x.double()
        mu, var = xd.mean(0), xd.var(0, unbiased=False)
        sm, si = mu.float(), (1 / torch.sqrt(var + eps)).float()
    pg, pb = R.randn(Cc, dtype=torch.float32), R.randn(Cc, dtype=torch.float32)
    dg, db = pg.clone(), pb.clone()
    dx = ops.bn_act_bwd(x, dy, gamma, beta, sm, si, act, dg, db, gs, bool(acc))
    dg2, db2 = pg.clone(), pb.clone()
    dx2 = ops.bn_act_bwd(x, dy, gamma, beta, sm, si, act, dg2, db2, gs, bool(acc))
    if R.meta:
        return []

    @functools.lru_cache(None)
    def ref():
        xr = x.double().requires_grad_(True)
        gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        y = _act(F.batch_norm(xr, None, None, gr, br, True, 0.0, eps), act)
        y.backward(dy.double())
        k = 1.0 if acc else 0.0
        return xr.grad, k * pg.double() + gs * gr.grad, k * pb.double() + gs * br.grad
    return [Check("dx", dx, lambda: ref()[0], 2e-3), Check("dgamma", dg, lambda: ref()[1], 1e-3), Check("dbeta", db, lambda: ref()[2], 1e-3),
            Check("dx repeat", dx2, dx, 0.0, "exact"), Check("dgamma repeat", dg2, dg, 0.0, "exact"),
            Check("dbeta repeat", db2, db, 0.0, "exact")]


def _layernorm(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    rows, Cc, eps = args[8:11]
    x = (R.randn(rows, Cc, dtype=torch.float32) * (0.5 + R.rand(rows, 1)) + R.randn(rows, 1, dtype=torch.float32)).half()
    gamma, beta = _bn_params(R, Cc)
    y = ops.layernorm(x, gamma, beta, eps=eps)
    if R.meta:
        return []
    return [Check("y", y, lambda: F.layer_norm(x.double(), (Cc,), gamma.double(), beta.double(), eps), 1e-3)]


def _layernorm_bwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    rows, Cc, eps, gs, acc = args[6:11]
    x = (R.randn(rows, Cc, dtype=torch.float32) * (0.5 + R.rand(rows, 1)) + R.randn(rows, 1, dtype=torch.float32)).half()
    dy = R.randn(rows, Cc, scale=0.1)
    gamma, _ = _bn_params(R, Cc)
    pg, pb = R.randn(Cc, dtype=torch.float32), R.randn(Cc, dtype=torch.float32)
    dg, db, dg2, db2 = pg.clone(), pb.clone(), pg.clone(), pb.clone()
    dx = ops.layernorm_bwd(x, dy, gamma, eps, dg, db, gs, bool(acc))
    dx2 = ops.layernorm_bwd(x, dy, gamma, eps, dg2, db2, gs, bool(acc))
    if R.meta:
        return []

    @functools.lru_cache(None)
    def ref():
        xr, gr = x.double().requires_grad_(True), gamma.double().requires_grad_(True)
        br = torch.zeros(Cc, dtype=torch.float64, device=x.device, requires_grad=True)
        F.layer_norm(xr, (Cc,), gr, br, eps).backward(dy.double())
        k = 1.0 if acc else 0.0
        return xr.grad, k * pg.double() + gs * gr.grad, k * pb.double() + gs * br.grad
    return [Check("dx", dx, lambda: ref()[0], 1.5e-3), Check("dgamma", dg, lambda: ref()[1], 1e-3), Check("dbeta", db, lambda: ref()[2], 1e-3),
            Check("dx repeat", dx2, dx, 0.0, "exact"), Check("dgamma repeat", dg2, dg, 0.0, "exact"),
            Check("dbeta repeat", db2, db, 0.0, "exact")]


def _colsum(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    rows, Cc, scale, acc = args[1], args[2], args[4], args[5]
    x = R.randn(rows, Cc, scale=0.1)
    pre = R.randn(Cc, dtype=torch.float32)
    out = ops.colsum(x, scale, pre.clone() if acc else None)
    out2 = ops.colsum(x, scale, pre.clone() if acc else None)
    if R.meta:
        return []
    ref = lambda: (pre.double() if acc else 0) + scale * x.double().sum(0)      # noqa: E731
    return [Check("colsum", out, ref, 1e-4), Check("colsum repeat", out2, out, 0.0, "exact")]


def _dot(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    rows, Cc, scale, acc = args[2], args[3], args[5], args[6]
    x, y = R.randn(rows, Cc), R.randn(rows, Cc, scale=0.1)
    pre = R.randn(1, dtype=torch.float32)
    out = ops.dot(x, y, pre.clone() if acc else None, scale)
    out2 = ops.dot(x, y, pre.clone() if acc else None, scale)
    if R.meta:
        return []
    # against the sum of |x y|: the dot of random operands cancels, so its own magnitude is no yardstick
    mag = lambda: float((x.double() * y.double()).abs().sum() * abs(scale)) + 1e-30      # noqa: E731
    ref = lambda: (pre.double() if acc else 0) + scale * (x.double() * y.double()).sum().view(1)      # noqa: E731
    return [Check("dot", lambda: out.double() / mag(), lambda: ref() / mag(), 1.0, "close", (1e-5, 0.0)),
            Check("dot repeat", out2, out, 0.0, "exact")]


def _attn_ref(q_src, kv_src, N, Cc, h, mask=None, p=0.0):
    """One direction of the cross-attention (common.py:670-684) in fp32: queries of one modality on the other's keys/values;
    mask (B * h, N, N) = kept probabilities of the dropout with probability p."""
    B = q_src.shape[0]
    d = Cc // h
    q = q_src[:, :N, :Cc].reshape(B, N, h, d).permute(0, 2, 1, 3)
    k = kv_src[:, :N, Cc:2 * Cc].reshape(B, N, h, d).permute(0, 2, 1, 3)
    v = kv_src[:, :N, 2 * Cc:].reshape(B, N, h, d).permute(0, 2, 1, 3)
    att = torch.softmax(q @ k.transpose(-1, -2) / d ** 0.5, -1)
    if mask is not None:
        att = att * mask.view(B, h, N, N) / (1 - p)
    return (att @ v).permute(0, 2, 1, 3).reshape(B, N, Cc)


def _attn_checks(out_v, out_i, qv, qi, N, Cc, h, tol, mask=None, p=0.0, tag=""):
    """mask: lazy (2, B * h, N, N) keep mask, direction 0 the RGB output."""
    m = (lambda dir: mask()[dir]) if mask is not None else (lambda dir: None)      # noqa: E731
    ref_v = lambda: _attn_ref(qi.float(), qv.float(), N, Cc, h, m(0), p)      # noqa: E731  RGB output: IR queries on RGB keys / values
    ref_i = lambda: _attn_ref(qv.float(), qi.float(), N, Cc, h, m(1), p)      # noqa: E731
    checks = [Check(tag + "out_vis", lambda: out_v[:, :N], ref_v, tol), Check(tag + "out_ir", lambda: out_i[:, :N], ref_i, tol)]
    if out_v.shape[1] > N:
        checks.append(_zero(tag + "pad rows", lambda: torch.cat([out_v[:, N:], out_i[:, N:]])))
    return checks


def _qkv(R: Operands, B, n_pad, Cc):
    return R.randn(B, n_pad, 3 * Cc), R.randn(B, n_pad, 3 * Cc)


def _attention(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    B, N, n_pad, Cc, h = args[6:11]
    qv, qi = _qkv(R, B, n_pad, Cc)
    out_v, out_i = ops.cross_attention(qv, qi, None, None, B, N, n_pad, Cc, h)
    return [] if R.meta else _attn_checks(out_v, out_i, qv, qi, N, Cc, h, 1e-3)


def _attn_mask(R: Operands, B, h, N, p):
    """Lazy keep mask of a replay at dropout probability p, seeded by the replay's own seed."""
    from dropout_mask import attn_keep_mask
    return functools.lru_cache(None)(lambda: attn_keep_mask(R.seed, 0, B, h, N, p, R.dev))


def _attention_train(rec, R: Operands) -> List[Check]:
    """At p = 0 (the inference kernel) and, for a dropout record, at its recorded p (the dropout instantiation)."""
    _, args, _ = rec
    B, N, n_pad, Cc, h, p = args[4:10]
    qv, qi = _qkv(R, B, n_pad, Cc)
    out_v, out_i = ops.cross_attention_train(qv, qi, B, N, n_pad, Cc, h, 0.0, 0)
    if p > 0:
        dv, di = ops.cross_attention_train(qv, qi, B, N, n_pad, Cc, h, p, R.seed)
        dv2, di2 = ops.cross_attention_train(qv, qi, B, N, n_pad, Cc, h, p, R.seed)
    if R.meta:
        return []
    checks = _attn_checks(out_v, out_i, qv, qi, N, Cc, h, 1e-3)
    if p > 0:
        checks += _attn_checks(dv, di, qv, qi, N, Cc, h, 1.5e-3, _attn_mask(R, B, h, N, p), p, f"p {p:g}: ")
        checks += [Check(f"p {p:g}: out_vis repeat", dv2, dv, 0.0, "exact"), Check(f"p {p:g}: out_ir repeat", di2, di, 0.0, "exact")]
    return checks


def _attention_bwd_case(qv, qi, dov, doi, B, N, n_pad, Cc, h, p, R: Operands) -> List[Check]:
    seed = R.seed if p > 0 else 0
    if R.meta:
        out_v, out_i = (R.randn(B, n_pad, Cc) for _ in range(2))
    else:
        out_v, out_i = ops.cross_attention_train(qv, qi, B, N, n_pad, Cc, h, p, seed)
    dq_v, dq_i = ops.cross_attention_bwd(qv, qi, out_v, out_i, dov, doi, B, N, n_pad, Cc, h, p, seed)
    if p > 0:
        dq_v2, dq_i2 = ops.cross_attention_bwd(qv, qi, out_v, out_i, dov, doi, B, N, n_pad, Cc, h, p, seed)
    if R.meta:
        return []
    mask = _attn_mask(R, B, h, N, p) if p > 0 else None

    @functools.lru_cache(None)
    def ref():
        rv, ri = qv.float().requires_grad_(True), qi.float().requires_grad_(True)
        m = (lambda dir: mask()[dir]) if mask is not None else (lambda dir: None)      # noqa: E731
        (_attn_ref(ri, rv, N, Cc, h, m(0), p) * dov[:, :N].float()).sum().backward(retain_graph=True)
        (_attn_ref(rv, ri, N, Cc, h, m(1), p) * doi[:, :N].float()).sum().backward()
        return rv.grad[:, :N], ri.grad[:, :N]
    tag = f"p {p:g}: " if p > 0 else ""
    checks = [Check(tag + "dqkv_vis", lambda: dq_v[:, :N], lambda: ref()[0], 2e-3),
              Check(tag + "dqkv_ir", lambda: dq_i[:, :N], lambda: ref()[1], 2e-3)]
    if n_pad > N:
        pad = lambda: torch.cat([dq_v[:, N:], dq_i[:, N:]])      # noqa: E731
        checks.append(_zero(tag + "pad rows", pad))
    if p > 0:
        checks += [Check(tag + "dqkv_vis repeat", dq_v2, dq_v, 0.0, "exact"), Check(tag + "dqkv_ir repeat", dq_i2, dq_i, 0.0, "exact")]
    return checks


def _attention_bwd(rec, R: Operands) -> List[Check]:
    """At p = 0 and, for a dropout record, at its recorded p; each on the forward output of the same p and seed."""
    _, args, _ = rec
    B, N, n_pad, Cc, h, p = args[8:14]
    qv, qi = _qkv(R, B, n_pad, Cc)
    dov, doi = R.randn(B, n_pad, Cc, scale=0.1), R.randn(B, n_pad, Cc, scale=0.1)
    checks = _attention_bwd_case(qv, qi, dov, doi, B, N, n_pad, Cc, h, 0.0, R)
    if p > 0:
        checks += _attention_bwd_case(qv, qi, dov, doi, B, N, n_pad, Cc, h, p, R)
    return checks


ELTWISE_GUARD = 8          # NaN elements on each side of the output: a write past either end fails the check


def _eltwise(rec, R: Operands) -> List[Check]:
    """Mode 0 (GELU) against F.gelu and mode 1 (its gradient) against autograd, in fp32; mode 2 (dropout) bit-exact against
    the mask restated on the host: fp16(fp32(x) / (1 - fp32(p))) where kept, 0 where dropped."""
    _, args, _ = rec
    mode, n, p = args[0], args[4], args[5]
    x = R.randn(n, scale=2.0)
    dy = R.randn(n, scale=0.1) if mode == 1 else None
    ybuf = R.nan(n + 2 * ELTWISE_GUARD)
    y = ybuf[ELTWISE_GUARD:ELTWISE_GUARD + n]
    ops._call("icaf_eltwise", _lib.lib().icaf_eltwise,
              (mode, ops._ptr(x), ops._ptr(dy), ops._ptr(y), n, p, C.c_uint32(R.seed)), {})
    if R.meta:
        return []
    guard = lambda: torch.cat([ybuf[:ELTWISE_GUARD], ybuf[ELTWISE_GUARD + n:]])      # noqa: E731
    checks = [Check("y neighbours unchanged", guard, lambda: R.nan(2 * ELTWISE_GUARD), 0.0, "exact")]
    if mode == 0:
        return checks + [Check("gelu", y, lambda: F.gelu(x.float()), 1e-3)]
    if mode == 1:
        def ref():
            xr = x.float().requires_grad_(True)
            F.gelu(xr).backward(dy.float())
            return xr.grad
        return checks + [Check("gelu'", y, ref, 1e-3)]
    from dropout_mask import eltwise_dropout, eltwise_keep
    return checks + [Check(f"dropout p {p:g}", y, lambda: eltwise_dropout(x, eltwise_keep(n, R.seed, 0, p, R.dev), p), 0.0, "exact")]


def _pool_window(H, W, nh, nw):
    sh, sw = H // nh, W // nw
    return (H - (nh - 1) * sh, W - (nw - 1) * sw), (sh, sw)


def _ref_pool_tokens(x, pos, w1, w2, nh, nw):
    """AdaptivePool2d avg / max (common.py:868-891) mixed by LearnableWeights + positional embedding (common.py:817-819);
    x NCHW."""
    B, Cc, H, W = x.shape
    if H > nh or W > nw:
        k, s = _pool_window(H, W, nh, nw)
        a, m = F.avg_pool2d(x, k, s), F.max_pool2d(x, k, s)
    else:
        a = m = x
    return (w1 * a + w2 * m).flatten(2).permute(0, 2, 1) + pos


def _pool_operands(args, R: Operands):
    B, H, W, Cc, nh, nw, n_pad = args[10:17]
    ld = args[2]
    N = nh * nw
    xo = _slot(ld, Cc)
    xv = R.view_in(R.randn(B, H, W, ld), xo, Cc)
    xi = R.view_in(R.randn(B, H, W, ld), xo, Cc)
    pv, pi = R.randn(N, Cc, scale=0.1), R.randn(N, Cc, scale=0.1)
    mix = 0.2 + 0.8 * R.rand(4)
    return B, H, W, Cc, nh, nw, n_pad, N, xv, xi, pv, pi, mix


def _pool_tokens(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    B, H, W, Cc, nh, nw, n_pad, N, xv, xi, pv, pi, mix = _pool_operands(args, R)
    tv, ti, sv, si = ops.dmff_pool_tokens(xv, xi, pv, pi, mix, nh, nw, with_stats=Cc % 32 == 0)
    if R.meta:
        return []
    checks = []
    for nm, t, x, p, w1, w2, s in (("vis", tv, xv, pv, 0, 1, sv), ("ir", ti, xi, pi, 2, 3, si)):
        ref = lambda x=x, p=p, w1=w1, w2=w2: _ref_pool_tokens(_nchw(x.float()), p.float(), mix[w1], mix[w2], nh, nw)   # noqa: E731
        checks.append(Check(f"tok_{nm}", lambda t=t: t[:, :N], ref, 1e-3))
        if n_pad > N:
            checks.append(_zero(f"tok_{nm} pad rows", lambda t=t: t[:, N:]))
        if s is not None:
            def got(s=s):
                return s.view(B * n_pad, Cc // 32, 2).double()
            def want(t=t):
                tt = t.double().reshape(B * n_pad, Cc // 32, 32)
                return torch.stack([tt.sum(2), (tt * tt).sum(2)], 2)
            checks.append(Check(f"stats_{nm}", got, want, 1.0, "close", (1e-2, 1e-4)))
    return checks


def _pool_tokens_bwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    B, H, W, Cc, nh, nw = args[8:14]
    n_pad = args[14]
    ld = args[2]
    N = nh * nw
    xo = _slot(ld, Cc)
    xv = R.view_in(R.randn(B, H, W, ld), xo, Cc)
    xi = R.view_in(R.randn(B, H, W, ld), xo, Cc)
    mix = 0.2 + 0.8 * R.rand(4)
    dtv, dti = R.randn(B, n_pad, Cc, scale=0.1), R.randn(B, n_pad, Cc, scale=0.1)
    dx_v, dx_i = ops.dmff_pool_tokens_bwd(xv, xi, dtv, dti, mix, nh, nw)
    if R.meta:
        return []

    def ref(x, d, w1, w2):
        xr = _nchw(x.float()).requires_grad_(True)
        (_ref_pool_tokens(xr, 0.0, mix[w1], mix[w2], nh, nw) * d[:, :N].float()).sum().backward()
        return xr.grad.permute(0, 2, 3, 1)
    # L2: where two window elements tie for the maximum, kernel and reference may route the gradient differently
    return [Check("dx_vis", dx_v, lambda: ref(xv, dtv, 0, 1), 2e-3, "l2"), Check("dx_ir", dx_i, lambda: ref(xi, dti, 2, 3), 2e-3, "l2")]


def _upsample_cat(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    n_pad, x_ld, y_ld = args[2], args[5], args[7]
    B, H, W, Cc, nh, nw, mode = args[8:15]
    N = nh * nw
    tv, ti = R.randn(B, n_pad, Cc), R.randn(B, n_pad, Cc)
    xo = _slot(x_ld, Cc)
    xv = R.view_in(R.randn(B, H, W, x_ld), xo, Cc)
    xi = R.view_in(R.randn(B, H, W, x_ld), xo, Cc)
    ybuf = R.nan(B, H, W, y_ld)
    yo = _slot(y_ld, 2 * Cc)
    y = R.view_in(ybuf, yo, 2 * Cc)
    ops._call("icaf_dmff_upsample_cat", _lib.lib().icaf_dmff_upsample_cat,
              (ops._ptr(tv), ops._ptr(ti), n_pad, ops._ptr(xv), ops._ptr(xi), ops._check_view(xv, "x_vis"), ops._ptr(y),
               ops._check_view(y, "y"), B, H, W, Cc, nh, nw, mode), {})
    if R.meta:
        return []

    def up(t):   # common.py:827-837
        t = t[:, :N].float().reshape(B, nh, nw, Cc).permute(0, 3, 1, 2)
        return F.interpolate(t, size=(H, W), mode="nearest" if mode else "bilinear").permute(0, 2, 3, 1)
    ref = lambda: torch.cat([up(tv) + xv.float(), up(ti) + xi.float()], -1)      # noqa: E731
    return [Check("y", y, ref, 1e-3)] + _untouched("y", ybuf, yo, 2 * Cc)


def _upsample_cat_bwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    ld = args[1]
    B, H, W, Cc, nh, nw, n_pad, mode = args[4:12]
    N = nh * nw
    dcat = R.view_in(R.randn(B, H, W, ld, scale=0.1), _slot(ld, 2 * Cc), 2 * Cc)
    dt_v, dt_i = ops.dmff_upsample_cat_bwd(dcat, nh, nw, n_pad, mode)
    if R.meta:
        return []

    @functools.lru_cache(None)
    def ref():
        t = torch.zeros(2, B, N, Cc, device=dcat.device, requires_grad=True)
        up = F.interpolate(t.reshape(2 * B, nh, nw, Cc).permute(0, 3, 1, 2), size=(H, W), mode="nearest")
        d = torch.cat([dcat[..., :Cc], dcat[..., Cc:]]).float().permute(0, 3, 1, 2)
        (up * d).sum().backward()
        return t.grad
    checks = [Check("dtok_vis", lambda: dt_v[:, :N], lambda: ref()[0], 2e-3), Check("dtok_ir", lambda: dt_i[:, :N], lambda: ref()[1], 2e-3)]
    if n_pad > N:
        pad = lambda: torch.cat([dt_v[:, N:], dt_i[:, N:]])      # noqa: E731
        checks.append(_zero("pad rows", pad))
    return checks


def _sppf(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    x_ld, y_ld = args[1], args[5]
    B, H, W, Cc = args[6:10]
    x = R.view_in(R.randn(B, H, W, x_ld), _slot(x_ld, Cc), Cc)
    ybuf = R.nan(B, H, W, y_ld)
    y0 = _slot(y_ld, 3 * Cc)
    ys = [R.view_in(ybuf, y0 + j * Cc, Cc) for j in range(3)]
    ops.sppf_pool(x, *ys)
    if R.meta:
        return []

    @functools.lru_cache(None)
    def ref():
        y1 = F.max_pool2d(_nchw(x.float()), 5, 1, 2)
        y2 = F.max_pool2d(y1, 5, 1, 2)
        return torch.cat([y1, y2, F.max_pool2d(y2, 5, 1, 2)], 1).permute(0, 2, 3, 1).half()
    return [Check("y1,y2,y3", lambda: ybuf[..., y0:y0 + 3 * Cc], ref, 0.0, "exact")] + _untouched("y", ybuf, y0, 3 * Cc)


def _maxpool5_bwd(rec, R: Operands) -> List[Check]:
    _, args, _ = rec
    B, H, W, Cc = args[3:7]
    x, dy = R.randn(B, H, W, Cc), R.randn(B, H, W, Cc, scale=0.1)
    dx = ops.maxpool5_bwd(x, dy)
    if R.meta:
        return []

    def ref():
        xr = _nchw(x.float()).requires_grad_(True)
        F.max_pool2d(xr, 5, 1, 2).backward(_nchw(dy.float()))
        return xr.grad.permute(0, 2, 3, 1)
    return [Check("dx", dx, ref, 1e-3, "l2")]


def _f32_hit(f, x0: float, want: float, side: str) -> np.float32:
    """The fp32 x next to x0 at which the monotone fp32 function f reaches `want`: side 'at' f(x) == want exactly, 'below'
    the largest x with f(x) < want, 'above' the smallest x with f(x) > want."""
    up = lambda v: np.nextafter(v, np.float32(np.inf))        # noqa: E731
    down = lambda v: np.nextafter(v, np.float32(-np.inf))     # noqa: E731
    want = np.float32(want)
    x = np.float32(x0)
    while f(x) < want:
        x = up(x)
    while f(down(x)) >= want:
        x = down(x)
    if side == "at":
        assert f(x) == want, (x0, want)
        return x
    if side == "below":
        return down(x)
    while f(x) <= want:
        x = up(x)
    return x


def _grid(n: int):
    """fp32 normalised coordinate -> grid coordinate, as build_targets scales it (targets * gain, loss.py:425-426)."""
    n = np.float32(n)
    return lambda x: np.float32(x) * n


def _loss_targets(rng, nt: int, B: int, nc: int, ny, nx, anchors):
    """(nt, 6) fp32 targets [image, class, x, y, w, h] that hit the edges of build_targets (loss.py:405-463) on every level,
    then random boxes.  The last image of a batch of two or more gets none.  Rows 0-3: two pairs of targets contesting one
    (image, anchor, cell) of the coarsest level, the better-fitting one first in one pair and second in the other (their
    predictions are set by _contest_logits)."""
    rows = []
    L = len(ny) - 1
    aw, ah = anchors[L][0]
    for k, (gi, gj) in enumerate(((1, 1), (nx[L] - 3, ny[L] - 2))):
        fit = [gi + 0.3, gj + 0.3, 1.2 * aw, 1.2 * ah]
        off = [gi + 0.3, gj + 0.3, 2.0 * aw, 0.8 * ah]
        for box in ((fit, off) if k == 0 else (off, fit)):
            rows.append([0, 0, box[0] / nx[L], box[1] / ny[L], box[2] / nx[L], box[3] / ny[L]])
    edges = []                     # per kind, per level
    for lvl in range(len(ny)):
        gx, gy = _grid(nx[lvl]), _grid(ny[lvl])
        a_w, a_h = anchors[lvl][0]
        w, h = a_w / nx[lvl], a_h / ny[lvl]
        kx, ky = nx[lvl] // 3, ny[lvl] // 3
        sx, sy = (kx + 0.25) / nx[lvl], (ky + 0.25) / ny[lvl]            # a plain coordinate on the other axis
        kinds = []
        for n, f, safe, k, put in ((nx[lvl], gx, sy, kx, lambda v, s: (v, s)), (ny[lvl], gy, sx, ky, lambda v, s: (s, v))):
            for want, side in ((k + 0.5, "at"), (k + 0.5, "below"),               # fractional part at / just below 0.5
                               (1.0, "at"), (1.0, "above"),                          # g at / just above 1
                               (n - 1.0, "at"), (n - 1.0, "below"),                  # n - g at / just above 1
                               (n - k - 0.5, "above")):                              # n - g: fractional part just below 0.5
                kinds.append((*put(float(_f32_hit(f, want / n, want, side)), safe), w, h))
        kinds += [(1.0, sy, w, h), (sx, 1.0, w, h), (1.0, 1.0, w, h), (0.0, 0.0, w, h)]     # image border: gi / gj clamp
        ratio = lambda v, s=a_w, f=gx: np.float32(f(v) / np.float32(s))                   # noqa: E731  gw / anchor_w
        for side in ("at", "below", "above"):                                             # gw / aw at / around anchor_t = 4
            kinds.append((sx, sy, float(_f32_hit(ratio, 4 * w, 4.0, side)), h))
        hr = lambda v, s=a_h, f=gy: np.float32(f(v) / np.float32(s))                      # noqa: E731  gh / ah = 1 / 4
        kinds.append((sx, sy, w, float(_f32_hit(hr, h / 4, 0.25, "at"))))
        edges.append(kinds)
    for kind in zip(*edges):
        for x, y, w, h in kind:
            rows.append([0, 0, x, y, w, h])
    n_img = max(B - 1, 1)
    for i in range(4, len(rows)):
        rows[i][0] = i % n_img
        rows[i][1] = i % nc
    t = np.zeros((nt, 6), dtype=np.float32)
    t[:min(nt, len(rows))] = np.array(rows[:nt], dtype=np.float32)
    r = nt - len(rows)
    if r > 0:
        t[len(rows):, 0] = rng.integers(0, n_img, r)
        t[len(rows):, 1] = rng.integers(0, nc, r)
        t[len(rows):, 2:4] = rng.uniform(0.0, 1.0, (r, 2))
        t[len(rows):, 4:6] = np.exp(rng.uniform(np.log(0.005), np.log(0.4), (r, 2)))
    return t


def _contest_logits(buf, t, ny, nx, anchors):
    """Anchor 0's box logits of the coarsest level at the cell of the better-fitting target of each contested pair (rows 0
    and 3), decoding to that target's box, so that the two targets of a pair have clearly different IoUs there (loss.py:355-361
    decode, inverted)."""
    L = len(ny) - 1
    aw, ah = anchors[L][0]
    logit = lambda s: math.log(s / (1 - s))       # noqa: E731
    for row in (0, 3):
        if row >= len(t):
            break
        x, y, w, h = (float(v) for v in t[row, 2:6])
        gx, gy = x * nx[L], y * ny[L]
        gi, gj = int(gx), int(gy)
        sx, sy = (gx - gi + 0.5) / 2, (gy - gj + 0.5) / 2
        sw, sh = math.sqrt(w * nx[L] / aw) / 2, math.sqrt(h * ny[L] / ah) / 2
        v = torch.tensor([logit(sx), logit(sy), logit(sw), logit(sh)], dtype=buf.dtype)
        buf[int(t[row, 0]), gj, gi, 0:4] = v.to(buf.device)


def _loss(rec, R: Operands) -> List[Check]:
    """icaf_compute_loss_fwd and _bwd of one record (the builder issues both, like the training step): fp16 head maps in
    the record's NHWC layout with pitch p_ld (pad channels NaN: the kernels must not read them), targets on the edges of
    build_targets, against the oracle's ComputeLoss (oracle/focal_loss.py) in float64 on the fp16 predictions, with fp32
    targets and anchors so that candidate selection is the reference's fp32 arithmetic.  Replayed at the record's fl_gamma,
    at the other of 0 / 1.5, and once with no targets."""
    import types
    from icafusion_b200.loss import ComputeLoss
    _, args, _ = rec
    p_ld, ny, nx, nl, B, na, no, nt = args[2], list(args[3]), list(args[4]), args[5], args[6], args[7], args[8], args[10]
    nc = no - 5
    anchors = torch.tensor(list(args[11]), dtype=torch.float32).view(nl, na, 2)
    h = args[12]._obj
    hyp = dict(box=h.box, obj=h.obj, cls=h.cls, cls_pw=h.cls_pw, obj_pw=h.obj_pw, anchor_t=h.anchor_t, fl_gamma=h.fl_gamma,
               label_smoothing=2.0 * h.cn)
    rng = np.random.Generator(np.random.PCG64(R.seed))
    tg = _loss_targets(rng, nt, B, nc, ny, nx, anchors.tolist())
    bufs, views = [], []
    for lvl in range(nl):
        buf = R.nan(B, ny[lvl], nx[lvl], p_ld)
        logits = R.randn(B, ny[lvl], nx[lvl], na, no, dtype=torch.float32)
        if not R.meta:
            logits[..., 4] = 1.5 * logits[..., 4] - 4.0                    # objectness: mostly background
        buf[..., :na * no] = logits.view(B, ny[lvl], nx[lvl], na * no).half()
        bufs.append(buf)
        views.append(buf.as_strided((B, na, ny[lvl], nx[lvl], no), (ny[lvl] * nx[lvl] * p_ld, no, nx[lvl] * p_ld, p_ld, 1)))
    if not R.meta:
        _contest_logits(bufs[-1], tg, ny, nx, anchors.tolist())
    checks = []
    other = 1.5 if not h.fl_gamma > 0 else 0.0
    for gamma, t in ((h.fl_gamma, tg), (other, tg), (h.fl_gamma, tg[:0])):
        hp = dict(hyp, fl_gamma=gamma)
        det = types.SimpleNamespace(na=na, nc=nc, nl=nl, anchors=anchors)
        crit = ComputeLoss(types.SimpleNamespace(hyp=hp, gr=h.gr, model=[det]))
        checks += _loss_case(crit, R, views, bufs, p_ld, torch.from_numpy(t).to(R.dev), anchors, hp, h.gr,
                             f"fl_gamma {gamma:g} nt {len(t)}")
    return checks


LOSS_GRAD_OUT = 256.0      # d/d(loss * bs) fed to the backward: keeps the fp16 gradient of every level in the normal range


def _loss_case(crit, R: Operands, views, bufs, p_ld, tg, anchors, hyp, gr, tag) -> List[Check]:
    from oracle import focal_loss
    crit.with_backward = True
    ld, ps = crit._layout(views)
    assert ld == p_ld, (ld, p_ld)
    B = views[0].shape[0]
    na, no = views[0].shape[1], views[0].shape[4]
    out, out2 = R.nan(5, dtype=torch.float32), R.nan(5, dtype=torch.float32)
    ws = crit._launch(ps, p_ld, tg, out=out)
    crit._launch(ps, p_ld, tg, out=out2)
    dbufs, dps = [], []
    for v in views:
        _, _, ny, nx, _ = v.shape
        d = R.nan(B + 2, ny, nx, p_ld)                        # images 0 and B + 1: NaN neighbours the backward must not touch
        d[1:B + 1, ..., na * no:] = 0                         # pad channels zeroed, as _LossFn.backward allocates them
        dbufs.append(d)
        dps.append(d[1:B + 1].as_strided(v.shape, v.stride()))
    gout = torch.full((1,), LOSS_GRAD_OUT, dtype=torch.float32, device=R.dev)
    crit._launch(ps, p_ld, tg, ws=ws, grad_out=gout, dps=dps)
    if R.meta:
        return []

    @functools.lru_cache(None)
    def ref():
        pr = [v.detach().double().cpu().requires_grad_(True) for v in views]
        lo, items = focal_loss.compute_loss(pr, tg.cpu(), anchors, hyp, gr)
        (lo * LOSS_GRAD_OUT).backward()
        return torch.cat([lo.detach().view(1), items.detach()]), [p.grad for p in pr]

    checks = [Check(f"{tag}: loss, lbox, lobj, lcls", lambda: out.cpu(), lambda: ref()[0], 1.0, "close", (2e-6, 3e-5)),
              Check(f"{tag}: forward repeat", out2, out, 0.0, "exact")]
    for lvl, (dp, d) in enumerate(zip(dps, dbufs)):
        # 2e-5 of the level's largest gradient, plus the half ulp of the kernel's final rounding to fp16 (2^-11 of the value)
        scale = lambda lvl=lvl: float(ref()[1][lvl].abs().max())                              # noqa: E731
        checks.append(Check(f"{tag}: dp[{lvl}]", lambda dp=dp, s=scale: dp.double().cpu() / s(),
                            lambda lvl=lvl, s=scale: ref()[1][lvl] / s(), 1.0, "close", (2e-5, 2.0 ** -11)))
        if p_ld > na * no:
            checks.append(Check(f"{tag}: dp[{lvl}] pad channels", lambda d=d: d[1:B + 1, ..., na * no:],
                                lambda d=d: torch.zeros_like(d[1:B + 1, ..., na * no:]), 0.0, "exact"))
        nb = lambda d=d: torch.cat([d[0].reshape(-1), d[B + 1].reshape(-1)])                   # noqa: E731
        checks.append(Check(f"{tag}: dp[{lvl}] neighbours unchanged", nb,
                            lambda nb=nb: torch.full(nb().shape, NAN16, dtype=torch.int16, device=R.dev).view(torch.float16), 0.0, "exact"))
    return checks


REPLAYED = {
    "icaf_conv2d_fwd": _conv_fwd,
    "icaf_compute_loss_fwd": _loss,           # both builders issue the forward and the backward
    "icaf_compute_loss_bwd": _loss,
    "icaf_bottleneck_fwd": _bottleneck,
    "icaf_conv2d_wgrad": _wgrad,            # and the data gradient of the same layer
    "icaf_pack_weight_pair": _pack_pair,
    "icaf_bn_act_fwd": _bn_fwd,
    "icaf_bn_act_bwd": _bn_bwd,
    "icaf_layernorm": _layernorm,
    "icaf_layernorm_bwd": _layernorm_bwd,
    "icaf_colsum": _colsum,
    "icaf_dot": _dot,
    "icaf_cross_attention": _attention,
    "icaf_cross_attention_train": _attention_train,
    "icaf_cross_attention_bwd": _attention_bwd,
    "icaf_dmff_pool_tokens": _pool_tokens,
    "icaf_dmff_pool_tokens_bwd": _pool_tokens_bwd,
    "icaf_dmff_upsample_cat": _upsample_cat,
    "icaf_dmff_upsample_cat_bwd": _upsample_cat_bwd,
    "icaf_sppf_pool": _sppf,
    "icaf_maxpool5_bwd": _maxpool5_bwd,
    "icaf_eltwise": _eltwise,
}

_ELEMENTWISE = "pure element-wise kernel with no shape-dependent plan"
NOT_REPLAYED = {
    "icaf_axpby": _ELEMENTWISE,
    "icaf_copy_channels": _ELEMENTWISE,
    "icaf_upsample2x": _ELEMENTWISE,
    "icaf_upsample2x_bwd": _ELEMENTWISE,
    "icaf_pack_image": _ELEMENTWISE,
    "icaf_detect_decode": _ELEMENTWISE,
    "all_reduce": "host-side exchange between ranks, not a kernel",
    "icaf_zero_stuff2": "covered through the data gradient replayed with every icaf_conv2d_wgrad record",
}


def replay(rec, device) -> List[Check]:
    """Issue `rec` again on fresh seeded operands (seed from its key) and return the checks."""
    return REPLAYED[rec[0]](rec, Operands(device, seed_of(key(rec))))


def conv_plan(g, n_io: int, sms: int):
    pl = _lib.ConvPlan()
    rc = _lib.lib().icaf_conv2d_plan(C.byref(g), n_io, sms, 0, C.byref(pl))
    return pl if rc == 0 else None


def describe_plan(pl) -> str:
    if pl is None:
        return "no plan"
    persistent = pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z
    return (f"bn{pl.bn} a_mode{pl.a_mode} halo{pl.halo} {'persistent' if persistent else 'one-tile'} tile {pl.tile_h}x{pl.tile_w} "
            f"splits{pl.splits} stages{pl.stages} ctas{pl.ctas}")
