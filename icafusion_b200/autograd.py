"""Training-mode forward / backward of the hot path: ``torch.autograd.Function`` nodes over the C-ABI kernels.

``loss.backward()`` (train.py:344) on the output of ``Model.forward`` in training mode runs these nodes: every forward and
every backward computation is a kernel of libicaf_b200 (wgmma implicit-GEMM convolutions for the forward, data- and
weight-gradient passes; the BatchNorm / SiLU / LayerNorm / GELU / dropout / pooling / attention kernels of csrc/train.cu,
pool.cu, dmff.cu, attn_bwd.cu).  torch provides the graph walk, the gradient accumulation where a tensor has several consumers,
and the ``.grad`` buffers -- so the reference's optimiser, GradScaler, EMA and DDP (train.py:120-235) work unchanged.

Activations and activation gradients are fp16 NHWC (the reference trains under autocast, train.py:334); parameters stay
fp32 masters and are re-packed to the kernels' fp16 layout each step; parameter gradients are fp32.  A TransformerFusionBlock
whose ``stream_dtype`` is torch.float32 keeps its token streams and their gradients in fp32, from the pooling to the
upsample-and-add, where the reference's autocast makes them fp32 (an fp32 one-element parameter times an fp16 tensor promotes);
GEMM operands, attention and branch outputs stay fp16.  The nodes on the stream take their precision from the tensors they get.

Reference semantics reproduced here (training mode): BatchNorm with batch statistics and running-stat update
(common.py:56), dropout on attention probabilities, projection and MLP outputs (common.py:677-685, 716-721), nearest
resampling in the DMFF tail (common.py:828-829), Detect returning the raw (B,na,ny,nx,no) maps (yolo_test.py:49-51).
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn as nn
from torch.autograd import Function

from . import ops
from .common import C3, SPPF, Concat, Conv, TransformerFusionBlock
from .ops import ACT_NONE, ACT_SILU
from .yolo_test import Detect

_STATE = {"seed": 0x1234567, "count": 0, "defer_bn": False, "bn": []}


def manual_seed(seed: int) -> None:
    """Seed of the counter-based dropout masks (every dropout site draws next_seed())."""
    _STATE["seed"], _STATE["count"] = int(seed) & 0xFFFFFFFF, 0


def next_seed() -> int:
    _STATE["count"] += 1
    return (_STATE["seed"] * 0x9E3779B1 + _STATE["count"] * 0x85EBCA77) & 0xFFFFFFFF


def _f32(t: torch.Tensor) -> torch.Tensor:
    t = t.detach()
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous()


# ------------------------------------------------------------------------------------------------
# Conv2d (no bias) + BatchNorm2d (batch statistics) + activation            models/common.py:48-57
class ConvBnActFn(Function):
    """A SyncBatchNorm `bn` (train.py --sync-bn) takes the two-phase BatchNorm with one exchange per direction when sync_group
    says so.  The exchange is queued on the current stream, which is the one this node's kernels (and, by autograd, its
    backward's) run on, side streams included."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, bn: nn.BatchNorm2d, stride: int, pad: int, act: int, stem: bool):
        w = _f32(weight)
        ctx.pk_dgrad = None
        if stem:      # 6x6/s2/p2 over the image == 3x3/s1/p1 over its space-to-depth form (ops.pack_stem_weight)
            pk = ops.pack_stem_weight(w, None, ACT_NONE)
        elif ctx.needs_input_grad[0]:
            pk, ctx.pk_dgrad = ops.pack_weight_pair(w, stride, pad)      # the backward's flipped filter comes out of the same launch
        else:
            pk = ops.pack_weight(w, stride, pad)
        z = ops.conv2d([x], [pk])[0]
        mom = 0.1 if bn.momentum is None else bn.momentum
        ctx.group = sync_group(bn)
        count = None
        if ctx.group is None:
            y, sm, si = ops.bn_act_fwd(z, _f32(gamma), _f32(beta), bn.running_mean, bn.running_var, bn.eps, mom, act)
        else:         # SyncBatchNorm: statistics over the rows of every rank of the group
            stats = ops.all_reduce_(ops.bn_act_fwd_stats(z), ctx.group)
            y, sm, si = ops.bn_act_fwd_apply(z, _f32(gamma), _f32(beta), bn.running_mean, bn.running_var, stats, bn.eps, mom, act)
            count = stats[-1:]                      # the global row count, for the backward
        if bn.num_batches_tracked is not None:     # nn.BatchNorm2d's step counter: one fused increment per model forward
            _STATE["bn"].append(bn.num_batches_tracked)
            if not _STATE["defer_bn"]:
                _flush_bn_counters()
        ctx.save_for_backward(x, z, weight, gamma, beta, sm, si, count)
        ctx.cfg = (stride, pad, act, stem)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, z, weight, gamma, beta, sm, si, count = ctx.saved_tensors
        stride, pad, act, stem = ctx.cfg
        dgamma = torch.empty(gamma.shape, dtype=torch.float32, device=z.device)
        dbeta = torch.empty_like(dgamma)
        if ctx.group is None:
            dz = ops.bn_act_bwd(z, dy, _f32(gamma), _f32(beta), sm, si, act, dgamma, dbeta)
        else:         # SyncBatchNorm: dgamma / dbeta stay local (DDP averages them); the two sums dx needs are summed over ranks
            dy = dy.contiguous()
            g32, b32 = _f32(gamma), _f32(beta)
            sums = ops.all_reduce_(ops.bn_act_bwd_sums(z, dy, g32, b32, sm, si, act, dgamma, dbeta), ctx.group)
            dz = ops.bn_act_bwd_apply(z, dy, g32, b32, sm, si, sums, count, act)
        cout, cin, kh, kw = weight.shape
        if stem:
            d16 = ops.conv2d_wgrad(x, dz, 3, 3, 1, 1)                         # (Cout, 16 = (dy,dx,c4), ty, tx)
            dw = d16.view(cout, 2, 2, 4, 3, 3).permute(0, 3, 4, 1, 5, 2).reshape(cout, 4, 6, 6)[:, :3].contiguous()
            dx = None
        else:
            dw = ops.conv2d_wgrad(x, dz, kh, kw, stride, pad)
            dx = ops.conv2d_dgrad(dz, _f32(weight), stride, pad, (x.shape[1], x.shape[2]), ctx.pk_dgrad) if ctx.needs_input_grad[0] else None
        return dx, dw.to(weight.dtype), dgamma.to(gamma.dtype), dbeta.to(beta.dtype), None, None, None, None, None


def sync_group(bn: nn.Module):
    """The process group a BatchNorm's training statistics are summed over, or None for per-rank statistics: torch's own
    SyncBatchNorm rule -- an nn.SyncBatchNorm in training mode, torch.distributed initialised, and more than one rank in
    ``bn.process_group`` (WORLD when unset)."""
    if not (isinstance(bn, nn.SyncBatchNorm) and bn.training):
        return None
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = dist.group.WORLD if bn.process_group is None else bn.process_group
    return group if dist.get_world_size(group) > 1 else None


def _flush_bn_counters() -> None:
    if _STATE["bn"]:
        torch._foreach_add_(_STATE["bn"], 1)
        _STATE["bn"] = []


def conv_bn_act(m, x: torch.Tensor, stem: bool = False) -> torch.Tensor:
    """Training forward of a common.Conv module on an NHWC tensor."""
    conv, bn = m.conv, m.bn
    if conv.groups != 1 or conv.dilation != (1, 1) or conv.bias is not None:
        raise NotImplementedError("Conv (training): groups=1, dilation=1, bias-free convolutions only")
    if isinstance(m.act, nn.SiLU):
        act = ACT_SILU
    elif isinstance(m.act, nn.Identity):
        act = ACT_NONE
    else:
        raise NotImplementedError(f"Conv: activation {type(m.act).__name__} not supported")
    return ConvBnActFn.apply(x, conv.weight, bn.weight, bn.bias, bn, conv.stride[0], conv.padding[0], act, stem)


# ------------------------------------------------------------------------------------------------
# Detect's 1x1 convolution with bias; output handed over as the (B,na,ny,nx,no) view the reference returns
class HeadConvFn(Function):
    @staticmethod
    def forward(ctx, x, weight, bias, na: int, no: int):
        B, H, W, _ = x.shape
        cout = na * no
        ld = ops.round_up(cout, 8)
        buf = torch.zeros(B, H, W, ld, dtype=torch.float16, device=x.device) if ld > cout else \
            torch.empty(B, H, W, ld, dtype=torch.float16, device=x.device)
        pk, ctx.pk_dgrad = ops.pack_weight_pair(_f32(weight), 1, 0, ACT_NONE, _f32(bias))
        ops.conv2d([x], [pk], [buf[..., :cout]])
        ctx.save_for_backward(x, weight)
        ctx.cfg = (na, no, ld)
        return buf.as_strided((B, na, H, W, no), (H * W * ld, no, W * ld, ld, 1))

    @staticmethod
    def backward(ctx, dp):
        x, weight = ctx.saved_tensors
        na, no, ld = ctx.cfg
        B, H, W, cin = x.shape
        cout = na * no
        want = (H * W * ld, no, W * ld, ld, 1)
        if dp.dtype == torch.float16 and dp.stride() == want and dp.storage_offset() == 0 and \
                dp.untyped_storage().nbytes() >= B * H * W * ld * 2:
            dbuf = dp.as_strided((B, H, W, ld), (H * W * ld, W * ld, ld, 1))          # our own loss backward: already NHWC
        else:                                                                     # e.g. the reference's loss: (B,na,ny,nx,no)
            dbuf = torch.zeros(B, H, W, ld, dtype=torch.float16, device=x.device)
            dbuf[..., :cout] = dp.permute(0, 2, 3, 1, 4).reshape(B, H, W, cout)
        dw = ops.conv2d_wgrad(x, dbuf, 1, 1, 1, 0)[:cout]
        db = ops.colsum(dbuf.view(B * H * W, ld))[:cout]
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.conv2d([dbuf], [ctx.pk_dgrad])[0]
        return dx, dw.to(weight.dtype).contiguous(), db.contiguous(), None, None


# ------------------------------------------------------------------------------------------------
# nn.Linear on (rows, K) fp16 token matrices
class LinearFn(Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        pk, ctx.pk_dgrad = ops.pack_weight_pair(_f32(weight)[:, :, None, None], 1, 0, ACT_NONE, None if bias is None else _f32(bias))
        y = ops.linear([x], [pk])[0]
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous()
        dw = ops.linear_wgrad(x, dy)
        db = ops.colsum(dy) if ctx.has_bias else None
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.linear([dy], [ctx.pk_dgrad])[0]
        return dx, dw.to(weight.dtype), db


class LayerNormFn(Function):
    """fp16 output for either input: over an fp32 token stream it is autocast's fp32 LayerNorm followed by the fp16 cast at the
    Linear it feeds, and the backward adds an fp32 dx into the stream's gradient."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps: float):
        ln = ops.layernorm_f32 if x.dtype == torch.float32 else ops.layernorm
        y = ln(x.contiguous(), _f32(gamma), _f32(beta), eps=eps)
        ctx.save_for_backward(x, gamma)
        ctx.eps = eps
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma = ctx.saved_tensors
        dg = torch.empty(gamma.shape, dtype=torch.float32, device=x.device)
        db = torch.empty_like(dg)
        bwd = ops.layernorm_bwd_f32 if x.dtype == torch.float32 else ops.layernorm_bwd
        dx = bwd(x.contiguous(), dy, _f32(gamma), ctx.eps, dg, db)
        return dx, dg, db, None


class GeluFn(Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return ops.eltwise(0, x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return ops.eltwise(1, x, dy)


class DropoutFn(Function):
    @staticmethod
    def forward(ctx, x, p: float, seed: int):
        ctx.cfg = (p, seed)
        return ops.eltwise(2, x, p=p, seed=seed)

    @staticmethod
    def backward(ctx, dy):
        p, seed = ctx.cfg
        return ops.eltwise(2, dy, p=p, seed=seed), None, None


def dropout(x: torch.Tensor, p: float) -> torch.Tensor:
    return x if p <= 0.0 else DropoutFn.apply(x, float(p), next_seed())


class CoefPairFn(Function):
    """c_a * x + c_b * o with two LearnableCoefficient scalars (common.py:747-750).  With an fp32 stream x (and the fp16 branch
    output o) the result and dx are fp32 and do is fp16, each the reference's autocast value bit for bit."""

    @staticmethod
    def forward(ctx, x, o, ca, cb):
        ctx.save_for_backward(x, o, ca, cb)
        if x.dtype == torch.float32:
            return ops.axpby_f32(x, _f32(ca), o, _f32(cb))
        return ops.axpby(x, _f32(ca), o, _f32(cb))

    @staticmethod
    def backward(ctx, dy):
        x, o, ca, cb = ctx.saved_tensors
        dy = dy.contiguous()
        if x.dtype == torch.float32:
            dx = ops.axpby_f32(dy, _f32(ca)) if ctx.needs_input_grad[0] else None
            do = ops.axpby_f32(dy, _f32(cb), out_dtype=o.dtype) if ctx.needs_input_grad[1] else None
            return dx, do, ops.dot_f32(dy, x).to(ca.dtype), ops.dot_f32(dy, o).to(cb.dtype)
        dx = ops.axpby(dy, _f32(ca)) if ctx.needs_input_grad[0] else None
        do = ops.axpby(dy, _f32(cb)) if ctx.needs_input_grad[1] else None
        return dx, do, ops.dot(dy, x).to(ca.dtype), ops.dot(dy, o).to(cb.dtype)


class AddFn(Function):
    """Bottleneck shortcut (common.py:193)."""

    @staticmethod
    def forward(ctx, x, y):
        one = torch.ones(1, dtype=torch.float32, device=x.device)
        return ops.axpby(x, one, y, one)

    @staticmethod
    def backward(ctx, dy):
        return dy, dy


class CrossAttentionFn(Function):
    @staticmethod
    def forward(ctx, qkv_v, qkv_i, B: int, N: int, n_pad: int, C: int, heads: int, p: float, seed: int):
        o_v, o_i = ops.cross_attention_train(qkv_v.view(B, n_pad, 3 * C), qkv_i.view(B, n_pad, 3 * C), B, N, n_pad, C, heads, p, seed)
        ctx.save_for_backward(qkv_v, qkv_i, o_v, o_i)
        ctx.cfg = (B, N, n_pad, C, heads, p, seed)
        return o_v.view(B * n_pad, C), o_i.view(B * n_pad, C)

    @staticmethod
    def backward(ctx, do_v, do_i):
        qkv_v, qkv_i, o_v, o_i = ctx.saved_tensors
        B, N, n_pad, C, heads, p, seed = ctx.cfg
        dq_v, dq_i = ops.cross_attention_bwd(qkv_v.view(B, n_pad, 3 * C), qkv_i.view(B, n_pad, 3 * C), o_v, o_i,
                                             do_v.contiguous().view(B, n_pad, C), do_i.contiguous().view(B, n_pad, C),
                                             B, N, n_pad, C, heads, p, seed)
        return dq_v.view(B * n_pad, 3 * C), dq_i.view(B * n_pad, 3 * C), None, None, None, None, None, None, None


class PoolTokensFn(Function):
    """avg / max adaptive pooling mixed by LearnableWeights + positional embedding (common.py:817-823).  f32: fp32 tokens with
    the fp32 pos_emb, and fp32 token gradients in the backward (the reference's autocast regime); else fp16 tokens."""

    @staticmethod
    def forward(ctx, rgb, ir, pos_v, pos_i, w1v, w2v, w1i, w2i, nh: int, nw: int, f32: bool = False):
        mix = torch.cat([_f32(t).reshape(1) for t in (w1v, w2v, w1i, w2i)])
        if f32:
            tv, ti = ops.dmff_pool_tokens_f32(rgb, ir, _f32(pos_v[0]), _f32(pos_i[0]), mix, nh, nw)
        else:
            tv, ti = ops.dmff_pool_tokens(rgb, ir, pos_v.detach()[0].to(torch.float16).contiguous(),
                                          pos_i.detach()[0].to(torch.float16).contiguous(), mix, nh, nw)
        ctx.save_for_backward(rgb, ir, mix)
        ctx.cfg = (nh, nw, pos_v.dtype, w1v.dtype, f32)
        return tv, ti

    @staticmethod
    def backward(ctx, dtv, dti):
        rgb, ir, mix = ctx.saved_tensors
        nh, nw, pdt, wdt, f32 = ctx.cfg
        dtv, dti = dtv.contiguous(), dti.contiguous()
        B, n_pad, C = dtv.shape
        N = nh * nw
        pool_bwd, colsum, dot = (ops.dmff_pool_tokens_bwd_f32, ops.colsum_f32, ops.dot_f32) if f32 else \
            (ops.dmff_pool_tokens_bwd, ops.colsum, ops.dot)
        dx_v, dx_i = pool_bwd(rgb, ir, dtv, dti, mix, nh, nw)
        # positional embeddings: sum over the batch; mixing weights: <dtok, avg-pooled> and <dtok, max-pooled>, the pooled
        # tokens fp16 in both regimes (torch's fp16 pooling returns fp16)
        dpos = [colsum(t.view(B, n_pad * C))[:N * C].view(1, N, C).to(pdt) for t in (dtv, dti)]
        zero = torch.zeros(N, C, dtype=torch.float16, device=rgb.device)
        dev = rgb.device
        even = (torch.arange(4, device=dev) % 2 == 0).float()          # (1, 0, 1, 0), built on the device (graph-capture safe)
        avg = ops.dmff_pool_tokens(rgb, ir, zero, zero, even, nh, nw)
        mx = ops.dmff_pool_tokens(rgb, ir, zero, zero, 1.0 - even, nh, nw)
        dw = [dot(dtv, avg[0]), dot(dtv, mx[0]), dot(dti, avg[1]), dot(dti, mx[1])]
        return (dx_v if ctx.needs_input_grad[0] else None, dx_i if ctx.needs_input_grad[1] else None, dpos[0], dpos[1],
                dw[0].to(wdt), dw[1].to(wdt), dw[2].to(wdt), dw[3].to(wdt), None, None, None)


class UpsampleCatFn(Function):
    """tokens -> (nh,nw) map -> nearest resample to (H,W), + residual, concat over channels (common.py:827-840, training).
    fp32 tokens: each sum is formed in fp32 and rounded once to the fp16 concat, and the token gradients are fp32."""

    @staticmethod
    def forward(ctx, tok_v, tok_i, rgb, ir, nh: int, nw: int):
        f32 = tok_v.dtype == torch.float32
        ctx.cfg = (nh, nw, tok_v.shape[1], rgb.shape[3], f32)
        if f32:
            return ops.dmff_upsample_cat_f32(tok_v, tok_i, rgb, ir, nh, nw)
        return ops.dmff_upsample_cat(tok_v, tok_i, rgb, ir, nh, nw, mode=1)

    @staticmethod
    def backward(ctx, dcat):
        nh, nw, n_pad, C, f32 = ctx.cfg
        if f32:
            dt_v, dt_i = ops.dmff_upsample_cat_bwd_f32(dcat, nh, nw, n_pad)
        else:
            dt_v, dt_i = ops.dmff_upsample_cat_bwd(dcat, nh, nw, n_pad, mode=1)
        return dt_v, dt_i, dcat[..., :C], dcat[..., C:], None, None


class ConcatFn(Function):
    @staticmethod
    def forward(ctx, *xs):
        B, H, W, _ = xs[0].shape
        ctx.widths = [x.shape[3] for x in xs]
        out = torch.empty(B, H, W, sum(ctx.widths), dtype=torch.float16, device=xs[0].device)
        o = 0
        for x in xs:
            ops.copy_channels(x, out[..., o:o + x.shape[3]])
            o += x.shape[3]
        return out

    @staticmethod
    def backward(ctx, dy):
        outs, o = [], 0
        for w in ctx.widths:
            outs.append(dy[..., o:o + w])
            o += w
        return tuple(outs)


class Upsample2xFn(Function):
    @staticmethod
    def forward(ctx, x):
        return ops.upsample2x(x)

    @staticmethod
    def backward(ctx, dy):
        return ops.upsample2x_bwd(dy)


class SppfPoolFn(Function):
    """x -> [x | m(x) | m(m(x)) | m(m(m(x)))] with m = MaxPool2d(5, 1, 2) (common.py:262-267)."""

    @staticmethod
    def forward(ctx, x):
        B, H, W, c = x.shape
        cat = torch.empty(B, H, W, 4 * c, dtype=torch.float16, device=x.device)
        ops.copy_channels(x, cat[..., :c])
        ops.sppf_pool(cat[..., :c], cat[..., c:2 * c], cat[..., 2 * c:3 * c], cat[..., 3 * c:])
        ctx.save_for_backward(cat)
        return cat

    @staticmethod
    def backward(ctx, dcat):
        (cat,) = ctx.saved_tensors
        c = cat.shape[3] // 4
        one = torch.ones(1, dtype=torch.float32, device=cat.device)
        part = lambda t, k: t[..., k * c:(k + 1) * c].contiguous()     # noqa: E731
        d2 = ops.axpby(part(dcat, 2), one, ops.maxpool5_bwd(part(cat, 2), part(dcat, 3)), one)
        d1 = ops.axpby(part(dcat, 1), one, ops.maxpool5_bwd(part(cat, 1), d2), one)
        return ops.axpby(part(dcat, 0), one, ops.maxpool5_bwd(part(cat, 0), d1), one)


# ------------------------------------------------------------------------------------------------
# module-level training forwards (NHWC in, NHWC out)
def bottleneck(m, x):
    y = conv_bn_act(m.cv2, conv_bn_act(m.cv1, x))
    return AddFn.apply(x, y) if m.add else y


def c3(m, x):
    a = conv_bn_act(m.cv1, x)
    for b in m.m:
        a = bottleneck(b, a)
    return conv_bn_act(m.cv3, ConcatFn.apply(a, conv_bn_act(m.cv2, x)))                 # common.py:227


def sppf(m, x):
    if m.m.kernel_size != 5:
        raise NotImplementedError("SPPF: only k=5 is supported")
    return conv_bn_act(m.cv2, SppfPoolFn.apply(conv_bn_act(m.cv1, x)))


def _linear(lin: nn.Linear, x):
    return LinearFn.apply(x, lin.weight, lin.bias)


def _layernorm(ln: nn.LayerNorm, x):
    return LayerNormFn.apply(x, ln.weight, ln.bias, ln.eps)


# Head dims icaf_cross_attention_bwd is built for.  The forward runs every multiple of 8 up to 128, and 160, so a model can
# run in eval() with a head dim (yolov5m: 24 / 48 / 96, yolov5x: 40 / 80 / 160) that it cannot train with.
ATTN_BWD_HEAD_DIMS = (8, 16, 32, 64, 128)


def require_attention_backward(m):
    """Raise NotImplementedError if the CrossAttention module `m` has a head dim without a backward kernel."""
    d = m.d_model // m.h
    if d not in ATTN_BWD_HEAD_DIMS:
        raise NotImplementedError(f"training: cross-attention head dim {d} (d_model {m.d_model}, {m.h} heads) has no backward "
                                  f"kernel; head dims {'/'.join(map(str, ATTN_BWD_HEAD_DIMS))} train")


def cross_attention(m, r2, i2, B: int, N: int, n_pad: int):
    """common.py:641-687 on (B*n_pad, C) token matrices: LN -> one [q|k|v] GEMM per modality -> attention with dropout on the
    probabilities -> output projection -> dropout."""
    require_attention_backward(m)
    C = m.d_model
    outs = []
    qkv = []
    for x, ln, q, k, v in ((r2, m.LN1, m.que_proj_vis, m.key_proj_vis, m.val_proj_vis), (i2, m.LN2, m.que_proj_ir, m.key_proj_ir, m.val_proj_ir)):
        w = torch.cat([q.weight, k.weight, v.weight], 0)
        b = torch.cat([q.bias, k.bias, v.bias], 0)
        qkv.append(LinearFn.apply(_layernorm(ln, x), w, b))
    p_att = m.attn_drop.p if m.training else 0.0
    a_v, a_i = CrossAttentionFn.apply(qkv[0], qkv[1], B, N, n_pad, C, m.h, float(p_att), next_seed() if p_att > 0 else 0)
    p_res = m.resid_drop.p if m.training else 0.0
    outs.append(dropout(_linear(m.out_proj_vis, a_v), p_res))
    outs.append(dropout(_linear(m.out_proj_ir, a_i), p_res))
    return outs


def _mlp(mlp: nn.Sequential, x, training: bool):
    h = GeluFn.apply(_linear(mlp[0], x))
    return dropout(_linear(mlp[2], h), mlp[3].p if training else 0.0)


def cross_transformer_block(m, r2, i2, B: int, N: int, n_pad: int):
    """common.py:737-759.  r2 / i2 carry the stream's precision (fp16, or fp32): the LayerNorms and coefficient pairs follow it,
    and with loops > 1 the stream they return is fed back in the same precision."""
    c = [getattr(m, f"coefficient{j}").bias for j in range(1, 9)]
    for _ in range(m.loops):
        o_r, o_i = cross_attention(m.crossatt, r2, i2, B, N, n_pad)
        ra = CoefPairFn.apply(r2, o_r, c[0], c[1])
        ia = CoefPairFn.apply(i2, o_i, c[2], c[3])
        r2 = CoefPairFn.apply(ra, _mlp(m.mlp_vis, _layernorm(m.LN2, ra), m.training), c[4], c[5])
        i2 = CoefPairFn.apply(ia, _mlp(m.mlp_ir, _layernorm(m.LN2, ia), m.training), c[6], c[7])
    return r2, i2


def fusion_block(m, rgb, ir):
    """TransformerFusionBlock.forward in training mode (common.py:807-841), its token streams in ``m.stream_dtype``."""
    f32 = stream_is_f32(m)
    B, H, W, C = rgb.shape
    nh, nw = m.avgpool.out_size(H, W)
    N = nh * nw
    if N != m.pos_emb_vis.shape[1]:
        raise ValueError(f"TransformerFusionBlock: {nh}x{nw} tokens but pos_emb has {m.pos_emb_vis.shape[1]} rows")
    tv, ti = PoolTokensFn.apply(rgb, ir, m.pos_emb_vis, m.pos_emb_ir, m.vis_coefficient.w1, m.vis_coefficient.w2,
                                m.ir_coefficient.w1, m.ir_coefficient.w2, nh, nw, f32)
    n_pad = tv.shape[1]
    r2, i2 = tv.view(B * n_pad, C), ti.view(B * n_pad, C)
    for blk in m.crosstransformer:
        r2, i2 = cross_transformer_block(blk, r2, i2, B, N, n_pad)
    cat = UpsampleCatFn.apply(r2.view(B, n_pad, C), i2.view(B, n_pad, C), rgb, ir, nh, nw)
    return conv_bn_act(m.conv1x1_out, cat)


def stream_is_f32(m) -> bool:
    """True when the TransformerFusionBlock `m` trains with fp32 token streams (``stream_dtype``: torch.float16 or float32)."""
    dt = getattr(m, "stream_dtype", torch.float16)
    if dt not in (torch.float16, torch.float32):
        raise ValueError(f"TransformerFusionBlock.stream_dtype: torch.float16 or torch.float32, got {dt}")
    return dt == torch.float32


def detect(m, xs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """Detect.forward in training mode: the raw maps, (B, na, ny, nx, no) (yolo_test.py:49-51)."""
    return [HeadConvFn.apply(x, m.m[i].weight, m.m[i].bias, m.na, m.no) for i, x in enumerate(xs)]


def model_forward(model, rgb_img: torch.Tensor, ir_img: torch.Tensor, taps: list = None):
    """The layer walk of Model.forward_once (yolo_test.py:136-163) over the training-mode nodes.  `taps` (diagnostics): receives
    every layer's NHWC output."""
    from .common import CrossAttention
    for mod in model.modules():          # refuse before the backbone launches anything
        if isinstance(mod, CrossAttention):
            require_attention_backward(mod)
    _STATE["defer_bn"], _STATE["bn"] = True, []
    try:
        return _walk(model, rgb_img, ir_img, taps)
    finally:
        _STATE["defer_bn"] = False
        _flush_bn_counters()


def _walk(model, rgb_img, ir_img, taps):
    """The IR backbone (layers s .. 2s-1, fed by `f == -4`) is independent of the RGB one until the first DMFF block: it is
    issued on a side stream, so the two streams' kernels overlap -- and so do their backward nodes, which autograd runs on the
    stream each forward ran on.  Inside a CUDA-graph capture the fork / join become parallel branches of the graph.  Sources,
    the stream split and the side-stream DMFF blocks come from the model's layer plan (yolo_test.plan_layers)."""
    import contextlib
    import os
    plan = model._layer_plan()
    y: list = []
    x = None
    s_ir = plan.ir_start if os.environ.get("ICAF_TRAIN_STREAMS", "1") != "0" else None
    main = side = None
    if s_ir is not None and rgb_img.is_cuda:
        main = torch.cuda.current_stream(rgb_img.device)
        side = model._side_streams(rgb_img.device, 1)[0]
        side.wait_stream(main)                       # fork before any RGB work is queued: the IR branch only needs the input batch
    joined = side is None
    forked = {}                                      # layer index -> side stream a DMFF block is running on
    for m in model.model:
        srcs = plan.srcs[m.i]
        on_side = side is not None and s_ir <= m.i < 2 * s_ir
        if not joined and m.i >= 2 * s_ir:           # first consumer of both branches
            main.wait_stream(side)
            for t in y[s_ir:2 * s_ir]:
                if t is not None:
                    t.record_stream(main)            # produced in the side stream's pool, read (and saved for backward) on main
            joined = True
        st = side if on_side else None
        if side is not None and m.i in plan.side_dmff:
            # the DMFF blocks only read backbone maps and are independent of each other: one side stream each (they are chains
            # of small token-level kernels that leave most of the GPU idle when run one after the other)
            st = model._side_streams(rgb_img.device, 2 + len(forked))[1 + len(forked)]
            st.wait_stream(main)
            for j in srcs:
                if y[j] is not None:
                    y[j].record_stream(st)
            forked[m.i] = st
        elif forked:                                 # any other layer: join the DMFF streams it may read from
            for i, fs in forked.items():
                main.wait_stream(fs)
                if y[i] is not None:
                    y[i].record_stream(main)
            if torch.is_tensor(x):
                x.record_stream(main)                # the previous layer's output arrives as `-1` even when it is not in `save`
            forked = {}
        with (torch.cuda.stream(st) if st is not None else contextlib.nullcontext()):
            x = _layer(model, m, [x if j == m.i - 1 else y[j] for j in srcs], rgb_img, ir_img)
        y.append(x if m.i in model.save else None)
        if taps is not None:
            taps.append(x)
    return x


def _layer(model, m, xs, rgb_img, ir_img):
    """Layer `m` on the maps `xs` of its sources (none: an image stem, RGB is the first layer, IR enters at f == -4)."""
    stem = not xs
    if stem:
        xs = [model._stage(ir_img if m.f == -4 else rgb_img, m)]
        if not (isinstance(m, Conv) and m.is_s2d_stem()):
            raise NotImplementedError("training: the image stem must be the 6x6 / stride 2 Conv of the yolov5 YAMLs")
    if isinstance(m, Conv):
        return conv_bn_act(m, xs[0], stem)
    if isinstance(m, C3):
        return c3(m, xs[0])
    if isinstance(m, SPPF):
        return sppf(m, xs[0])
    if isinstance(m, nn.Upsample):
        if m.mode != "nearest" or m.scale_factor is None or float(m.scale_factor) != 2.0:
            raise NotImplementedError("Upsample: only nearest x2 is supported")
        return Upsample2xFn.apply(xs[0])
    if isinstance(m, Concat):
        return ConcatFn.apply(*xs)
    if isinstance(m, TransformerFusionBlock):
        return fusion_block(m, xs[0], xs[1])
    if isinstance(m, Detect):
        return detect(m, xs)
    raise NotImplementedError(type(m).__name__)
