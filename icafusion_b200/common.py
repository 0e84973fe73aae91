"""Host-side mirror of the reference operator library (models/common.py) for the ICAFusion hot path.

Same class names, constructor signatures, sub-module / parameter names and ``state_dict`` keys as the
reference, so reference checkpoints load with ``strict=True`` and ``models/yolo_test.py``-style graph
builders can ``eval()`` these names.  The ``forward`` bodies do not call PyTorch operators: they
marshal tensors into libicaf_b200.so (hand-written sm_90a kernels, see include/icaf_b200.h).

Data layout: modules accept logical (B,C,H,W) tensors like the reference; internally everything is
fp16 NHWC, which is exactly torch's ``channels_last`` memory format, so consecutive modules exchange
tensors without any layout conversion (outputs are returned as channels_last views).

Scope of this round: inference semantics (``eval()``: BatchNorm running statistics, dropout = identity,
bilinear DMFF up-sampling) with or without ``Model.fuse()``.  Training-mode forward (batch statistics,
dropout, autograd) raises NotImplementedError -- there is no silent PyTorch fallback.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch
import torch.nn as nn

from . import ops
from .ops import ACT_GELU, ACT_NONE, ACT_SILU, PackedConv

__all__ = ["autopad", "Conv", "Bottleneck", "C3", "SPPF", "Concat", "Upsample", "LearnableCoefficient",
           "LearnableWeights", "CrossAttention", "CrossTransformerBlock", "TransformerFusionBlock",
           "AdaptivePool2d", "to_nhwc", "to_nchw"]


def autopad(k, p=None):
    """reference: models/common.py:36-40"""
    if p is None:
        p = k // 2 if isinstance(k, int) else [x // 2 for x in k]
    return p


# ------------------------------------------------------------------------------------------------
# layout plumbing
def to_nhwc(x: torch.Tensor) -> torch.Tensor:
    """Logical (B,C,H,W) -> fp16 (B,H,W,C) contiguous view (zero-copy for channels_last fp16 input)."""
    if not ops.on_device(x):
        raise RuntimeError("icafusion_b200 operators run on CUDA tensors only (no CPU fallback)")
    v = x.permute(0, 2, 3, 1)
    if v.dtype != torch.float16 or not v.is_contiguous():
        v = v.to(torch.float16).contiguous()
    return v


def to_nchw(v: torch.Tensor) -> torch.Tensor:
    """(B,H,W,C) -> logical (B,C,H,W) channels_last view."""
    return v.permute(0, 3, 1, 2)


def _require_eval(m: nn.Module):
    if m.training:
        raise NotImplementedError(f"{type(m).__name__}: the NHWC `run` entry points are the inference path (folded BatchNorm, fused "
                                  "epilogues); in train() call the module itself (forward) or icafusion_b200.autograd")


def _train_nodes():
    from . import autograd
    return autograd


def _dev_half(t: torch.Tensor) -> torch.Tensor:
    if not ops.on_device(t):
        raise RuntimeError("icafusion_b200 operators run on CUDA tensors only (no CPU fallback)")
    return t if t.dtype == torch.float16 else t.to(torch.float16)


def _versions(*ts) -> tuple:
    return tuple((t.data_ptr(), t._version, t.device) if t is not None else None for t in ts)


# ------------------------------------------------------------------------------------------------
class Conv(nn.Module):
    """Conv2d + BatchNorm2d + SiLU (reference: models/common.py:48-60).  After ``Model.fuse()`` the BN is
    folded into ``self.conv`` (with bias) and ``forward`` is rebound to ``fuseforward`` exactly as the
    reference does; before that, eval-mode BN is folded on the fly into the packed filter."""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, autopad(k, p), groups=g, bias=False)
        self.bn = nn.BatchNorm2d(c2)
        self.act = nn.SiLU() if act is True else (act if isinstance(act, nn.Module) else nn.Identity())

    # -- packed filter cache -------------------------------------------------------------------
    def packed(self, in_place: bool = False) -> PackedConv:
        """The BN-folded filter in the kernel's layout, re-packed when a parameter or BN buffer changed.  `in_place`: copy a
        re-pack into the cached tensors instead of replacing them (engine.refresh_packed_)."""
        conv = self.conv
        bn = getattr(self, "bn", None)
        key = _versions(conv.weight, conv.bias, *( (bn.weight, bn.bias, bn.running_mean, bn.running_var) if bn is not None else ()))
        cache = self.__dict__.get("_icaf_pack")
        if cache is not None and cache[0] == key:
            return cache[1]
        if conv.groups != 1 or conv.dilation != (1, 1) or conv.kernel_size[0] != conv.kernel_size[1] or \
                conv.stride[0] != conv.stride[1] or conv.padding[0] != conv.padding[1]:
            raise NotImplementedError("Conv: only groups=1, dilation=1, square kernel/stride/padding are supported")
        if isinstance(self.act, nn.SiLU):
            act = ACT_SILU
        elif isinstance(self.act, nn.Identity):
            act = ACT_NONE
        else:
            raise NotImplementedError(f"Conv: activation {type(self.act).__name__} not supported")
        w = conv.weight.detach().float()
        b = conv.bias.detach().float() if conv.bias is not None else torch.zeros(w.shape[0], device=w.device)
        if bn is not None:   # fold eval-mode BN: utils/torch_utils.py:182-202
            scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
            w = w * scale.view(-1, 1, 1, 1)
            b = (b - bn.running_mean.detach().float()) * scale + bn.bias.detach().float()
        if self.is_s2d_stem():
            pk = ops.pack_stem_weight(w, b, act)          # 6x6/s2/p2 over the image == 3x3/s1/p1 over its space-to-depth form
        else:
            pk = ops.pack_conv_weight(w, b, conv.stride[0], conv.padding[0], act)
        if in_place and cache is not None:
            pk = ops.copy_packed_(cache[1], pk)
        self.__dict__["_icaf_pack"] = (key, pk)
        return pk

    def is_s2d_stem(self) -> bool:
        """The yolov5 image stem `Conv(3, c, 6, 2, 2)`: staged as a space-to-depth image (see ops.pack_stem_weight)."""
        c = self.conv
        return c.in_channels == 3 and c.kernel_size == (6, 6) and c.stride == (2, 2) and c.padding == (2, 2)

    def stage_image(self, img: torch.Tensor) -> torch.Tensor:
        """Planar (B,3,H,W) image -> the NHWC tensor this stem consumes (uint8 is scaled by 1/255 on the fly)."""
        if img.dtype not in (torch.float16, torch.float32, torch.uint8):
            img = img.float()
        scale = 1.0 / 255.0 if img.dtype == torch.uint8 else 1.0
        s2d = self.is_s2d_stem() and img.shape[2] % 2 == 0 and img.shape[3] % 2 == 0
        if self.is_s2d_stem() and not s2d:
            raise ValueError("the 6x6/s2 image stem needs even image height and width")
        return ops.pack_image(img, scale, s2d=s2d)

    @staticmethod
    def run(mods: Sequence["Conv"], xs: Sequence[torch.Tensor], outs=None, res=None) -> List[torch.Tensor]:
        """NHWC-level entry: 1 or 2 Conv modules of identical geometry in one grouped launch."""
        for m in mods:
            if hasattr(m, "bn"):
                _require_eval(m)
        return ops.conv2d(list(xs), [m.packed() for m in mods], outs, res)

    def forward(self, x):
        if x.shape[1] == 3 and self.conv.in_channels == 3:     # image stem: planar -> packed NHWC4 / space-to-depth
            if not ops.on_device(x):
                raise RuntimeError("icafusion_b200 operators run on CUDA tensors only (no CPU fallback)")
            v = self.stage_image(x)
        else:
            v = to_nhwc(x)
        if self.training and hasattr(self, "bn"):          # batch statistics + backward: the autograd node (common.py:56-57)
            return to_nchw(_train_nodes().conv_bn_act(self, v, stem=v.shape[3] == 16 and self.is_s2d_stem()))
        return to_nchw(Conv.run([self], [v])[0])

    def fuseforward(self, x):
        return Conv.forward(self, x)


class Bottleneck(nn.Module):
    """reference: models/common.py:184-194"""

    def __init__(self, c1, c2, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_, c2, 3, 1, g=g)
        self.add = shortcut and c1 == c2

    @staticmethod
    def fusable(mods, xs, outs=None) -> bool:
        """The one-launch form (ops.bottleneck) applies: shortcut, 64 channels throughout, 16-byte aligned views, outputs
        that share no storage with the inputs (its patches read x halos that neighbouring patches would overwrite), and
        enough 4 x 32-pixel patches to give both consumer warpgroups of every SM of an H100 SXM (132 SMs) one."""
        m0 = mods[0]
        if not m0.add or m0.cv1.conv.in_channels != 64 or m0.cv1.conv.out_channels != 64 or m0.cv2.conv.kernel_size != (3, 3):
            return False
        B, H, W, _ = xs[0].shape
        if len(xs) * B * ((H + 3) // 4) * ((W + 31) // 32) < 2 * 132:
            return False
        for m in mods:
            _require_eval(m)
        views = list(xs) + list(outs or [])
        if any(t.shape[3] != 64 or t.stride(2) % 8 or (ops._addr(t) or 0) % 16 for t in views):
            return False
        stores = {t.untyped_storage()._cdata for t in xs}
        return not any(t.untyped_storage()._cdata in stores for t in outs or [])

    @staticmethod
    def run(mods, xs, outs=None):
        if Bottleneck.fusable(mods, xs, outs):
            p1s, p3s = [m.cv1.packed() for m in mods], [m.cv2.packed() for m in mods]
            if all(p.act == ACT_SILU for p in p1s + p3s):
                return ops.bottleneck(list(xs), p1s, p3s, outs)
        h = Conv.run([m.cv1 for m in mods], xs)
        return Conv.run([m.cv2 for m in mods], h, outs, list(xs) if mods[0].add else None)   # residual fused in the epilogue

    def forward(self, x):
        if self.training:
            return to_nchw(_train_nodes().bottleneck(self, to_nhwc(x)))
        return to_nchw(Bottleneck.run([self], [to_nhwc(x)])[0])


class C3(nn.Module):
    """CSP bottleneck with 3 convolutions (reference: models/common.py:216-227).  The channel concat is
    never materialised as a copy: the last bottleneck and cv2 write straight into the two halves of the
    buffer cv3 reads."""

    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c1, c_, 1, 1)
        self.cv3 = Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*[Bottleneck(c_, c_, shortcut, g, e=1.0) for _ in range(n)])

    def packed_cv12(self, in_place: bool = False) -> PackedConv:
        """cv1 and cv2 read the same input: one GEMM with the two filter banks stacked ([cv1 | cv2] output channels)."""
        p1, p2 = self.cv1.packed(in_place), self.cv2.packed(in_place)
        keys = (self.cv1.__dict__["_icaf_pack"][0], self.cv2.__dict__["_icaf_pack"][0])    # in-place re-packs keep p1, p2
        cache = self.__dict__.get("_icaf_pack12")
        if cache is not None and cache[0] is p1 and cache[1] is p2 and cache[3] == keys:
            return cache[2]
        c_ = p1.cout
        w = torch.cat([p1.w[:c_], p2.w[:c_]], 0)
        rows = ops.round_up(2 * c_, 32)
        if rows != 2 * c_:
            w = torch.cat([w, w.new_zeros(rows - 2 * c_, w.shape[1])], 0)
        pk = PackedConv(w.contiguous(), torch.cat([p1.bias, p2.bias]).contiguous(), p1.cin, 2 * c_, 1, 1, 1, 0, p1.act)
        if in_place and cache is not None:
            pk = ops.copy_packed_(cache[2], pk)
        self.__dict__["_icaf_pack12"] = (p1, p2, pk, keys)
        return pk

    @staticmethod
    def run(mods, xs, outs=None):
        c_ = mods[0].cv1.conv.out_channels
        B, H, W, _ = xs[0].shape
        for m in mods:
            _require_eval(m)
        cats = [torch.empty(B, H, W, 2 * c_, dtype=torch.float16, device=xs[0].device) for _ in mods]
        left = [c[..., :c_] for c in cats]
        ops.conv2d(list(xs), [m.packed_cv12() for m in mods], cats)          # [cv1(x) | cv2(x)] in one launch
        a = left
        n = len(mods[0].m)
        for j in range(n):
            # the last bottleneck writes back into the left half: with n = 1 that is its own input, which only the
            # two-launch form allows (its residual read is element-wise, same thread); with n >= 2 it reads a scratch map
            # and runs fused like the others
            a = Bottleneck.run([m.m[j] for m in mods], a, left if j == n - 1 else None)
        return Conv.run([m.cv3 for m in mods], cats, outs)

    def forward(self, x):
        if self.training:
            return to_nchw(_train_nodes().c3(self, to_nhwc(x)))
        return to_nchw(C3.run([self], [to_nhwc(x)])[0])


class SPPF(nn.Module):
    """reference: models/common.py:252-267 (three chained 5x5 max pools, concatenated with the input)."""

    def __init__(self, c1, c2, k=5):
        super().__init__()
        c_ = c1 // 2
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_ * 4, c2, 1, 1)
        self.m = nn.MaxPool2d(kernel_size=k, stride=1, padding=k // 2)

    @staticmethod
    def run(mods, xs, outs=None):
        c_ = mods[0].cv1.conv.out_channels
        if mods[0].m.kernel_size != 5:
            raise NotImplementedError("SPPF: only k=5 is supported")
        B, H, W, _ = xs[0].shape
        cats = [torch.empty(B, H, W, 4 * c_, dtype=torch.float16, device=xs[0].device) for _ in mods]
        Conv.run([m.cv1 for m in mods], xs, [c[..., :c_] for c in cats])
        for c in cats:
            ops.sppf_pool(c[..., :c_], c[..., c_:2 * c_], c[..., 2 * c_:3 * c_], c[..., 3 * c_:])
        return Conv.run([m.cv2 for m in mods], cats, outs)

    def forward(self, x):
        if self.training:
            return to_nchw(_train_nodes().sppf(self, to_nhwc(x)))
        return to_nchw(SPPF.run([self], [to_nhwc(x)])[0])


class Concat(nn.Module):
    """reference: models/common.py:313-321 (channel concat of NCHW maps)."""

    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension

    @staticmethod
    def run(vs: Sequence[torch.Tensor]) -> torch.Tensor:
        B, H, W, _ = vs[0].shape
        out = torch.empty(B, H, W, sum(v.shape[3] for v in vs), dtype=torch.float16, device=vs[0].device)
        o = 0
        for v in vs:
            ops.copy_channels(v, out[..., o:o + v.shape[3]])
            o += v.shape[3]
        return out

    def forward(self, x):
        if self.d != 1:
            raise NotImplementedError("Concat: only the channel dimension is supported")
        return to_nchw(Concat.run([to_nhwc(t) for t in x]))


class Upsample(nn.Upsample):
    """`nn.Upsample(None, 2, 'nearest')` rows of the model YAML (yolov5l_Transfusion_kaist.yaml:48,53)."""

    def forward(self, x):
        if self.mode != "nearest" or float(self.scale_factor) != 2.0:
            raise NotImplementedError("Upsample: only nearest x2 is supported")
        return to_nchw(ops.upsample2x(to_nhwc(x)))


# ------------------------------------------------------------------------------------------------
# DMFF
class LearnableCoefficient(nn.Module):
    """reference: models/common.py:569-576 (scalar gain; consumed fused inside CrossTransformerBlock)."""

    def __init__(self):
        super().__init__()
        self.bias = nn.Parameter(torch.FloatTensor([1.0]), requires_grad=True)

    def forward(self, x):
        """Stand-alone call (inside CrossTransformerBlock the gain rides in the GEMM epilogues): x * bias."""
        return ops.axpby(_dev_half(x), self.bias.detach().float()).view(x.shape)


class LearnableWeights(nn.Module):
    """reference: models/common.py:579-587 (two scalar mixing weights; fused into the token pooling kernel)."""

    def __init__(self):
        super().__init__()
        self.w1 = nn.Parameter(torch.tensor([0.5]), requires_grad=True)
        self.w2 = nn.Parameter(torch.tensor([0.5]), requires_grad=True)

    def forward(self, x1, x2):
        """Stand-alone call (inside the DMFF block the mix rides in the token-pooling kernel): x1*w1 + x2*w2."""
        return ops.axpby(_dev_half(x1), self.w1.detach().float(), _dev_half(x2), self.w2.detach().float()).view(x1.shape)


class AdaptivePool2d(nn.Module):
    """reference: models/common.py:868-891.  Holds the geometry; the pooling itself runs fused with the
    avg/max mix and the positional embedding in icaf_dmff_pool_tokens."""

    def __init__(self, output_h, output_w, pool_type="avg"):
        super().__init__()
        self.output_h = output_h
        self.output_w = output_w
        self.pool_type = pool_type

    def out_size(self, H: int, W: int):
        if H > self.output_h or W > self.output_w:
            if H < self.output_h or W < self.output_w:
                raise ValueError(f"AdaptivePool2d: map {H}x{W} is smaller than the {self.output_h}x{self.output_w} grid in "
                                 "one dimension (the reference divides by zero here, common.py:880)")
            return self.output_h, self.output_w
        return H, W

    def forward(self, x):
        """Stand-alone call: (B,C,H,W) -> (B,C,output_h,output_w) with the reference's stride / kernel rule (common.py:874-888);
        runs the same pooling kernel as the fused block with the mix pinned to this module's pool type."""
        v = to_nhwc(x)
        B, H, W, C = v.shape
        nh, nw = self.out_size(H, W)
        if (nh, nw) == (H, W):
            return x
        if self.pool_type not in ("avg", "max"):
            raise NotImplementedError(f"AdaptivePool2d: pool_type {self.pool_type!r}")
        mix = torch.tensor([1.0, 0.0, 1.0, 0.0] if self.pool_type == "avg" else [0.0, 1.0, 0.0, 1.0], device=v.device)
        pos = torch.zeros(nh * nw, C, dtype=torch.float16, device=v.device)
        tok, _ = ops.dmff_pool_tokens(v, v, pos, pos, mix, nh, nw)
        return tok[:, :nh * nw].reshape(B, nh, nw, C).permute(0, 3, 1, 2)


class CrossAttention(nn.Module):
    """reference: models/common.py:590-687.  Parameters only; the computation (LN -> fused QK / V^T
    projections -> flash cross-attention -> out_proj) is driven by CrossTransformerBlock."""

    def __init__(self, d_model, d_k, d_v, h, attn_pdrop=.1, resid_pdrop=.1):
        super().__init__()
        assert d_k % h == 0
        self.d_model = d_model
        self.d_k = d_model // h
        self.d_v = d_model // h
        self.h = h
        self.que_proj_vis = nn.Linear(d_model, h * self.d_k)
        self.key_proj_vis = nn.Linear(d_model, h * self.d_k)
        self.val_proj_vis = nn.Linear(d_model, h * self.d_v)
        self.que_proj_ir = nn.Linear(d_model, h * self.d_k)
        self.key_proj_ir = nn.Linear(d_model, h * self.d_k)
        self.val_proj_ir = nn.Linear(d_model, h * self.d_v)
        self.out_proj_vis = nn.Linear(h * self.d_v, d_model)
        self.out_proj_ir = nn.Linear(h * self.d_v, d_model)
        self.attn_drop = nn.Dropout(attn_pdrop)
        self.resid_drop = nn.Dropout(resid_pdrop)
        self.LN1 = nn.LayerNorm(d_model)
        self.LN2 = nn.LayerNorm(d_model)
        for m in self.modules():          # reference init, common.py:626-639
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, std=0.001)
                nn.init.constant_(m.bias, 0)

    # -- packed parameters ---------------------------------------------------------------------
    def packed(self, in_place: bool = False):
        live = [self.que_proj_vis, self.key_proj_vis, self.val_proj_vis, self.que_proj_ir, self.key_proj_ir, self.val_proj_ir,
                self.out_proj_vis, self.out_proj_ir, self.LN1, self.LN2]
        key = _versions(*[p for m in live for p in (m.weight, m.bias)])
        cache = self.__dict__.get("_icaf_pack")
        if cache is not None and cache[0] == key:
            return cache[1]
        if self.d_model % 64:
            raise NotImplementedError("CrossAttention: d_model must be a multiple of 64")
        P = {}
        # one [Q|K|V] projection per modality with its LayerNorm folded in (LN1 -> rgb, LN2 -> ir: common.py:660,665)
        for mod, q, k, v, o, ln in (("vis", self.que_proj_vis, self.key_proj_vis, self.val_proj_vis, self.out_proj_vis, self.LN1),
                                    ("ir", self.que_proj_ir, self.key_proj_ir, self.val_proj_ir, self.out_proj_ir, self.LN2)):
            P[f"qkv_{mod}"] = ops.pack_linear_ln(torch.cat([q.weight, k.weight, v.weight], 0), torch.cat([q.bias, k.bias, v.bias], 0),
                                                 ln.weight, ln.bias, ln.eps)
            P[f"out_{mod}"] = ops.pack_linear(o.weight, o.bias)
        if in_place and cache is not None:
            P = ops.copy_packed_(cache[1], P)
        self.__dict__["_icaf_pack"] = (key, P)
        return P

    def attend(self, r2: torch.Tensor, i2: torch.Tensor, B: int, N: int, n_pad: int, stats=None):
        """[LN ->] fused Q|K|V projection -> flash cross-attention for both directions (common.py:660-682).
        r2, i2: fp16 (B*n_pad, C) token matrices; `stats`: their row statistics (fp32 (rows, parts, 2) x 2) if a producer
        already emitted them.  LayerNorm never runs as a kernel: it is folded into the projection GEMM's epilogue.
        Returns the merged-head attention outputs (B*n_pad, C) x 2 and the packs."""
        P = self.packed()
        rows, C = r2.shape
        if stats is None:
            stats = ops.row_stats(r2, i2)
        qkv_v, qkv_i = ops.linear([r2, i2], [P["qkv_vis"], P["qkv_ir"]], ln_stats=list(stats))   # common.py:660-668
        a_v, a_i = ops.cross_attention(qkv_v.view(B, n_pad, 3 * C), qkv_i.view(B, n_pad, 3 * C), None, None, B, N, n_pad, C, self.h)
        return a_v.view(rows, C), a_i.view(rows, C), P                                             # common.py:670-684

    def forward(self, x, attention_mask=None, attention_weights=None):
        """Stand-alone call: x = [rgb_tokens, ir_tokens] (B, N, C) -> [out_vis, out_ir] (common.py:641-687).  Inside
        CrossTransformerBlock the output projection additionally carries the coefficient pair in its epilogue."""
        if attention_mask is not None or attention_weights is not None:
            raise NotImplementedError("CrossAttention: attention_mask / attention_weights are unused by the reference forward")
        r, i = x
        B, N, C = r.shape
        r, i, n_pad = _pad_tokens(r, N), _pad_tokens(i, N), ops.round_up(N, 8)
        if self.training:                                  # dropout on probabilities / outputs, autograd nodes
            o_v, o_i = _train_nodes().cross_attention(self, r.view(B * n_pad, C), i.view(B * n_pad, C), B, N, n_pad)
            return [o_v.view(B, n_pad, C)[:, :N], o_i.view(B, n_pad, C)[:, :N]]
        a_v, a_i, P = self.attend(r.view(B * n_pad, C), i.view(B * n_pad, C), B, N, n_pad)
        o_v, o_i = ops.linear([a_v, a_i], [P["out_vis"], P["out_ir"]])                     # common.py:683,685
        return [o_v.view(B, n_pad, C)[:, :N], o_i.view(B, n_pad, C)[:, :N]]


def _pad_tokens(t: torch.Tensor, N: int) -> torch.Tensor:
    """(B, N, C) tokens -> contiguous fp16 (B, round_up(N, 8), C), pad rows zero."""
    t = _dev_half(t)
    B, _, C = t.shape
    n_pad = ops.round_up(N, 8)
    if n_pad == N:
        return t.contiguous()
    out = t.new_zeros(B, n_pad, C)
    out[:, :N] = t
    return out


def _mlp(d_model, block_exp, resid_pdrop):
    return nn.Sequential(nn.Linear(d_model, block_exp * d_model), nn.GELU(),
                         nn.Linear(block_exp * d_model, d_model), nn.Dropout(resid_pdrop))


class CrossTransformerBlock(nn.Module):
    """reference: models/common.py:690-759.  ``loops`` is mutable like in the reference.  Dead parameters
    (ln_input, ln_output, mlp, LN1) are kept so state_dicts match."""

    def __init__(self, d_model, d_k, d_v, h, block_exp, attn_pdrop, resid_pdrop, loops_num=1):
        super().__init__()
        self.loops = loops_num
        self.ln_input = nn.LayerNorm(d_model)
        self.ln_output = nn.LayerNorm(d_model)
        self.crossatt = CrossAttention(d_model, d_k, d_v, h, attn_pdrop, resid_pdrop)
        self.mlp_vis = _mlp(d_model, block_exp, resid_pdrop)
        self.mlp_ir = _mlp(d_model, block_exp, resid_pdrop)
        self.mlp = _mlp(d_model, block_exp, resid_pdrop)
        self.LN1 = nn.LayerNorm(d_model)
        self.LN2 = nn.LayerNorm(d_model)
        for j in range(1, 9):
            setattr(self, f"coefficient{j}", LearnableCoefficient())

    # -- packed parameters ---------------------------------------------------------------------
    def packed(self, in_place: bool = False):
        live = [self.mlp_vis[0], self.mlp_vis[2], self.mlp_ir[0], self.mlp_ir[2], self.LN2]
        ts = [p for m in live for p in (m.weight, m.bias)] + [getattr(self, f"coefficient{j}").bias for j in range(1, 9)]
        key = _versions(*ts)
        cache = self.__dict__.get("_icaf_pack")
        if cache is not None and cache[0] == key:
            return cache[1]
        P = {}
        for mod, mlp in (("vis", self.mlp_vis), ("ir", self.mlp_ir)):      # the SAME LN2 in front of both MLPs (common.py:749-750)
            P[f"fc1_{mod}"] = ops.pack_linear_ln(mlp[0].weight, mlp[0].bias, self.LN2.weight, self.LN2.bias, self.LN2.eps, ACT_GELU)
            P[f"fc2_{mod}"] = ops.pack_linear(mlp[2].weight, mlp[2].bias)
        P["coef"] = torch.cat([getattr(self, f"coefficient{j}").bias.detach().float().reshape(1) for j in range(1, 9)])
        if in_place and cache is not None:
            P = ops.copy_packed_(cache[1], P)
        self.__dict__["_icaf_pack"] = (key, P)
        return P

    def run(self, r: torch.Tensor, i: torch.Tensor, N: int, stats=None):
        """r, i: fp16 (B, Npad, C) token streams (pad rows finite); `stats`: their row statistics when the producer emitted
        them (the token-pooling kernel does).  Five launches per loop: [LN+QKV] -> attention -> [out_proj, coefficients, row
        statistics] -> [LN2+fc1+GELU] -> [fc2, coefficients, row statistics].  Returns the updated streams."""
        _require_eval(self)
        P = self.packed()
        B, n_pad, C = r.shape
        rows = B * n_pad
        c = P["coef"]
        co = lambda a, b: (c[a - 1:a], c[b - 1:b])   # noqa: E731  (alpha, beta) device scalars
        r2, i2 = r.view(rows, C), i.view(rows, C)
        new_stats = lambda: [torch.empty(rows, (C + 31) // 32, 2, dtype=torch.float32, device=r.device) for _ in range(2)]  # noqa: E731
        for loop in range(self.loops):
            a_v, a_i, A = self.crossatt.attend(r2, i2, B, N, n_pad, stats)                  # common.py:745 (660-682)
            # out_proj + coefficient pair: ra = c1*r + c2*o_r          common.py:683,685,747-748
            st_a = new_stats()
            ra, ia = ops.linear([a_v, a_i], [A["out_vis"], A["out_ir"]], res=[r2, i2], scaled=[co(1, 2), co(3, 4)], stats_out=st_a)
            # MLPs on LN2 (same LN2 for both), LayerNorm folded into fc1  common.py:749-750, 704-715
            hr, hi = ops.linear([ra, ia], [P["fc1_vis"], P["fc1_ir"]], ln_stats=st_a)
            stats = new_stats() if loop + 1 < self.loops else None                         # feeds the next loop's LN1 / LN2
            r2, i2 = ops.linear([hr, hi], [P["fc2_vis"], P["fc2_ir"]], res=[ra, ia], scaled=[co(5, 6), co(7, 8)], stats_out=stats)
        return r2.view(B, n_pad, C), i2.view(B, n_pad, C)

    def forward(self, x):
        """x = [rgb_tokens, ir_tokens], each (B, N, C) like the reference (common.py:737-759)."""
        r, i = x
        B, N, C = r.shape
        if self.training:
            n_pad = ops.round_up(N, 8)
            r2, i2 = _train_nodes().cross_transformer_block(self, _pad_tokens(r, N).view(B * n_pad, C), _pad_tokens(i, N).view(B * n_pad, C), B, N, n_pad)
            return [r2.view(B, n_pad, C)[:, :N], i2.view(B, n_pad, C)[:, :N]]
        r, i = self.run(_pad_tokens(r, N), _pad_tokens(i, N), N)
        return [r[:, :N], i[:, :N]]


class TransformerFusionBlock(nn.Module):
    """The DMFF block (reference: models/common.py:762-865)."""

    def __init__(self, d_model, vert_anchors=16, horz_anchors=16, h=8, block_exp=4, n_layer=1, embd_pdrop=0.1,
                 attn_pdrop=0.1, resid_pdrop=0.1):
        super().__init__()
        self.n_embd = d_model
        self.vert_anchors = vert_anchors
        self.horz_anchors = horz_anchors
        d_k = d_v = d_model
        self.pos_emb_vis = nn.Parameter(torch.zeros(1, vert_anchors * horz_anchors, self.n_embd))
        self.pos_emb_ir = nn.Parameter(torch.zeros(1, vert_anchors * horz_anchors, self.n_embd))
        self.avgpool = AdaptivePool2d(self.vert_anchors, self.horz_anchors, "avg")
        self.maxpool = AdaptivePool2d(self.vert_anchors, self.horz_anchors, "max")
        self.vis_coefficient = LearnableWeights()
        self.ir_coefficient = LearnableWeights()
        self.crosstransformer = nn.Sequential(*[CrossTransformerBlock(d_model, d_k, d_v, h, block_exp, attn_pdrop,
                                                                      resid_pdrop) for _ in range(n_layer)])
        # (the reference applies its _init_weights before these exist, common.py:787-790: the attention projections keep
        #  CrossAttention's std = 0.001 init, the MLPs the nn.Linear default -- same initial state here)
        self.concat = Concat(dimension=1)
        self.conv1x1_out = Conv(c1=d_model * 2, c2=d_model, k=1, s=1, p=0, g=1, act=True)

    def _front(self, in_place: bool = False):
        ts = (self.pos_emb_vis, self.pos_emb_ir, self.vis_coefficient.w1, self.vis_coefficient.w2,
              self.ir_coefficient.w1, self.ir_coefficient.w2)
        key = _versions(*ts)
        cache = self.__dict__.get("_icaf_pack")
        if cache is not None and cache[0] == key:
            return cache[1]
        pk = (self.pos_emb_vis.detach()[0].to(torch.float16).contiguous(),
              self.pos_emb_ir.detach()[0].to(torch.float16).contiguous(),
              torch.cat([t.detach().float().reshape(1) for t in ts[2:]]))
        if in_place and cache is not None:
            pk = ops.copy_packed_(cache[1], pk)
        self.__dict__["_icaf_pack"] = (key, pk)
        return pk

    def run(self, rgb: torch.Tensor, ir: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """rgb, ir: fp16 NHWC feature maps -> fused NHWC map (optionally written into the view `out`)."""
        _require_eval(self)
        B, H, W, C = rgb.shape
        nh, nw = self.avgpool.out_size(H, W)
        N = nh * nw
        if N != self.pos_emb_vis.shape[1]:
            raise ValueError(f"TransformerFusionBlock: {nh}x{nw} tokens but pos_emb has {self.pos_emb_vis.shape[1]} rows")
        pos_v, pos_i, mix = self._front()
        r, i, sv, si = ops.dmff_pool_tokens(rgb, ir, pos_v, pos_i, mix, nh, nw, with_stats=True)   # common.py:817-823
        stats = [sv, si]
        for blk in self.crosstransformer:
            r, i = blk.run(r, i, N, stats)                                         # common.py:825
            stats = None
        cat = ops.dmff_upsample_cat(r, i, rgb, ir, nh, nw, mode=0)                 # common.py:827-840 (eval: bilinear)
        return Conv.run([self.conv1x1_out], [cat], None if out is None else [out])[0]   # common.py:841

    def forward(self, x):
        rgb, ir = x
        assert rgb.shape[0] == ir.shape[0]
        if self.training:                                  # dropout, nearest tail, batch-statistics BN: the autograd nodes
            return to_nchw(_train_nodes().fusion_block(self, to_nhwc(rgb), to_nhwc(ir)))
        return to_nchw(self.run(to_nhwc(rgb), to_nhwc(ir)))
