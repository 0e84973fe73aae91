"""fp32 DMFF token streams on the device (TransformerFusionBlock.stream_dtype = float32, TrainStep(dmff_fp32=True)).

Each fp32-stream node against torch on the same inputs, at the token grids and widths yolov5n / s / l train with; the
coefficient pair bit for bit against torch's `c_a * x + c_b * o`; the CrossTransformerBlock chain (loops 1 and 2, with and
without dropout, masks from tests/dropout_mask.py) against fp32 autograd; the whole-model step's one-element gradients; the
graphed step against the eager one bit for bit over an accumulation window and a step, with PDL on and off; and the
default (fp16 streams) unchanged."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_mask as DM
from conftest import ROOT
from helpers import err

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (C, map H, W, token grid nh, nw): the P3 / P4 / P5 DMFF blocks of yolov5n (FLIR), s and l at 320 x 320, and P3 at 640
SHAPES = [(64, 40, 40, 20, 20), (128, 20, 20, 16, 16), (256, 10, 10, 10, 10),
          (128, 40, 40, 20, 20), (256, 20, 20, 16, 16), (512, 10, 10, 10, 10),
          (256, 40, 40, 20, 20), (512, 20, 20, 16, 16), (1024, 10, 10, 10, 10),
          (128, 80, 80, 20, 20)]


def _rel(a, b, floor=0.0) -> float:
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / max(float(b.norm()), floor, 1e-30))


@pytest.mark.parametrize("C,H,W,nh,nw", SHAPES)
def test_pool_tokens_and_tail_f32(cuda_device, C, H, W, nh, nw):
    from icafusion_b200 import autograd as A
    dev = cuda_device
    B, N = 2, nh * nw
    g = torch.Generator().manual_seed(C + H + nh)
    rgb, ir = (torch.randn(B, C, H, W, generator=g).half().to(dev) for _ in range(2))
    pos = [(0.1 * torch.randn(1, N, C, generator=g)).to(dev) for _ in range(2)]              # fp32, not fp16-representable
    wts = [torch.tensor([v], device=dev) for v in (0.6137, 0.3861, 0.2919, 0.7083)]
    dtok = [(0.1 * torch.randn(B, N, C, generator=g)).to(dev) for _ in range(2)]
    # the reference's own computation: torch's fp16 pooling, then fp32 LearnableWeights and pos_emb (type promotion)
    sh, sw = H // nh, W // nw
    k = (H - (nh - 1) * sh, W - (nw - 1) * sw)
    R = [t.clone().requires_grad_(True) for t in (rgb, ir)]
    P = [t.clone().requires_grad_(True) for t in pos]
    Wt = [t.clone().requires_grad_(True) for t in wts]

    def ref(x, p, w1, w2):
        a, m = (F.avg_pool2d(x, k, (sh, sw)), F.max_pool2d(x, k, (sh, sw))) if (H > nh or W > nw) else (x, x)
        return (a * w1 + m * w2).flatten(2).permute(0, 2, 1) + p, a, m
    tr = [ref(R[0], P[0], Wt[0], Wt[1]), ref(R[1], P[1], Wt[2], Wt[3])]
    assert tr[0][0].dtype == torch.float32
    ((tr[0][0] * dtok[0]).sum() + (tr[1][0] * dtok[1]).sum()).backward()
    Rd = [t.permute(0, 2, 3, 1).contiguous().requires_grad_(True) for t in (rgb, ir)]
    Pd = [t.clone().requires_grad_(True) for t in pos]
    Wd = [t.clone().requires_grad_(True) for t in wts]
    tv, ti = A.PoolTokensFn.apply(Rd[0], Rd[1], Pd[0], Pd[1], Wd[0], Wd[1], Wd[2], Wd[3], nh, nw, True)
    n_pad = tv.shape[1]
    assert tv.dtype == ti.dtype == torch.float32 and float(tv[:, N:].abs().max() if n_pad > N else 0) == 0
    pad = lambda t: torch.cat([t, t.new_zeros(B, n_pad - N, C)], 1)      # noqa: E731
    ((tv * pad(dtok[0])).sum() + (ti * pad(dtok[1])).sum()).backward()
    torch.cuda.synchronize()
    # forward: the same roundings in the same order; only the window sums' order differs (before the fp16 rounding)
    mism = sum(int((t[:, :N] != r[0].detach()).sum()) for t, r in zip((tv, ti), tr))
    e_f = max(err(tv[:, :N], tr[0][0]), err(ti[:, :N], tr[1][0]))
    # map gradients: the reference rounds d(avg) and d(max) to fp16 before its fp16 pool backwards; the device rounds once
    e_x = max(_rel(Rd[0].grad.permute(0, 3, 1, 2), R[0].grad), _rel(Rd[1].grad.permute(0, 3, 1, 2), R[1].grad))
    e_p = max(_rel(Pd[0].grad, P[0].grad), _rel(Pd[1].grad, P[1].grad))
    # the mixing weights: <dtok, pooled> over fp32 dtok and the fp16 pooled maps, against the float64 sum
    want = [(dtok[j // 2].double() * tr[j // 2][1 + j % 2].detach().flatten(2).permute(0, 2, 1).double()).sum() for j in range(4)]
    e_w = max(abs(float(Wd[j].grad) - float(want[j])) / max(abs(float(want[j])), 1e-3) for j in range(4))
    e_wt = max(abs(float(Wt[j].grad) - float(want[j])) / max(abs(float(want[j])), 1e-3) for j in range(4))
    print(f"\n[pool f32 {H}x{W}->{nh}x{nw} C{C}] fwd {e_f:.1e} ({mism} of {2 * B * N * C} differ)  dx {e_x:.1e}  dpos {e_p:.1e}  "
          f"dmix {e_w:.1e} (torch {e_wt:.1e})")
    assert e_f < 1e-6 and mism <= 1e-4 * 2 * B * N * C
    assert e_x < 2e-3 and e_p < 1e-6 and e_w < 1e-4
    # tail: nearest resample + residual + concat, one rounding of the fp32 sum
    tok = [torch.randn(B, N, C, generator=g).to(dev) for _ in range(2)]
    dcat = (0.1 * torch.randn(B, H, W, 2 * C, generator=g)).half().to(dev)
    T = [t.clone().requires_grad_(True) for t in tok]
    up = lambda t: F.interpolate(t.reshape(B, nh, nw, C).permute(0, 3, 1, 2), size=(H, W), mode="nearest")   # noqa: E731
    cat = torch.cat([up(T[0]) + rgb, up(T[1]) + ir], 1).half()
    (cat.float() * dcat.permute(0, 3, 1, 2).float()).sum().backward()
    Td = [pad(t).requires_grad_(True) for t in tok]
    Rd = [t.permute(0, 2, 3, 1).contiguous().requires_grad_(True) for t in (rgb, ir)]
    cd = A.UpsampleCatFn.apply(Td[0], Td[1], Rd[0], Rd[1], nh, nw)
    cd.backward(dcat)
    torch.cuda.synchronize()
    assert torch.equal(cd.permute(0, 3, 1, 2), cat)
    e_t = max(_rel(Td[0].grad[:, :N], T[0].grad), _rel(Td[1].grad[:, :N], T[1].grad))
    assert Td[0].grad.dtype == torch.float32 and Rd[0].grad.dtype == torch.float16
    assert torch.equal(Rd[0].grad, dcat[..., :C]) and torch.equal(Rd[1].grad, dcat[..., C:])
    print(f"[tail f32 {nh}x{nw}->{H}x{W}] fwd bit-exact  dtok {e_t:.1e}")
    assert e_t < 1e-6 and (n_pad == N or float(Td[0].grad[:, N:].abs().max()) == 0)


@pytest.mark.parametrize("C,N", [(64, 400), (256, 256), (1024, 100)])
def test_coef_pair_and_layernorm_f32(cuda_device, C, N):
    from icafusion_b200 import autograd as A
    dev = cuda_device
    B = 2
    n_pad = (N + 7) // 8 * 8
    g = torch.Generator().manual_seed(C + N)
    x = torch.randn(B * n_pad, C, generator=g).to(dev)
    o = torch.randn(B * n_pad, C, generator=g).half().to(dev)
    ca, cb = torch.tensor([0.9173], device=dev), torch.tensor([1.1311], device=dev)
    dy = torch.randn(B * n_pad, C, generator=g).to(dev)
    xr, orr, car, cbr = (t.clone().requires_grad_(True) for t in (x, o, ca, cb))
    y_ref = car * xr + cbr * orr                                # torch's promotion: fp32, two rounded products, a rounded sum
    assert y_ref.dtype == torch.float32
    y_ref.backward(dy)
    xd, od, cad, cbd = (t.clone().requires_grad_(True) for t in (x, o, ca, cb))
    y = A.CoefPairFn.apply(xd, od, cad, cbd)
    y.backward(dy)
    torch.cuda.synchronize()
    assert torch.equal(y, y_ref.detach()), "coefficient pair forward differs from torch's fp32 c_a * x + c_b * o"
    assert torch.equal(xd.grad, xr.grad) and xd.grad.dtype == torch.float32
    assert torch.equal(od.grad, orr.grad) and od.grad.dtype == torch.float16
    want = [(dy.double() * x.double()).sum(), (dy.double() * o.double()).sum()]
    e_c = max(abs(float(a.grad) - float(w)) / abs(float(w)) for a, w in zip((cad, cbd), want))
    print(f"\n[coef pair f32 C{C} N{N}] forward, dx, do bit-exact; dc {e_c:.1e}")
    assert e_c < 1e-4
    # LayerNorm: fp32 tokens -> fp16 operand; backward from the fp16 GEMM data gradient to an fp32 dx
    gam = (1 + 0.2 * torch.randn(C, generator=g)).to(dev)
    bet = (0.2 * torch.randn(C, generator=g)).to(dev)
    dl = (0.1 * torch.randn(B * n_pad, C, generator=g)).half().to(dev)
    xr, gr, br = (t.clone().requires_grad_(True) for t in (x, gam, bet))
    yl = F.layer_norm(xr, (C,), gr, br, 1e-5)
    yl.backward(dl.float())
    xd, gd, bd = (t.clone().requires_grad_(True) for t in (x, gam, bet))
    y = A.LayerNormFn.apply(xd, gd, bd, 1e-5)
    y.backward(dl)
    torch.cuda.synchronize()
    assert y.dtype == torch.float16 and xd.grad.dtype == torch.float32
    yh = yl.detach().half()
    same = (y.float() * yh.float() > 0) | ((y.float() == 0) & (yh.float() == 0))
    ulps = int((y.view(torch.int16).int() - yh.view(torch.int16).int()).abs()[same].max())            # fp16 units in the last place
    ulps = max(ulps, int(((y.float() - yh.float()).abs()[~same] > 6e-8).sum()) * 99)                   # a sign change: only at +-0
    e_y, e_dx = err(y, yl), _rel(xd.grad, xr.grad)
    e_g = max(_rel(gd.grad, gr.grad), _rel(bd.grad, br.grad))
    print(f"[layernorm f32 C{C}] fwd {e_y:.1e} (at most {ulps} fp16 ulp from torch's rounded output)  dx {e_dx:.1e}  dgamma/dbeta {e_g:.1e}")
    assert e_y < 1e-3 and ulps <= 1 and e_dx < 1e-5 and e_g < 1e-5


def _init_block(blk, g):
    with torch.no_grad():
        for k, p in blk.named_parameters():
            if p.dim() >= 2:
                p.copy_((torch.randn(p.shape, generator=g) / p.shape[1] ** 0.5).half().float())     # fp16-representable filters
            elif "coefficient" in k:
                p.copy_(1 + 0.3 * torch.randn(p.shape, generator=g))
            elif k.endswith("weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))


def _ref_block(m, r, i, B, N, n_pad, seeds, p_att, p_res):
    """common.py:737-759 in fp32 autograd, on the real (unpadded) tokens, with the device's dropout masks."""
    C, h = r.shape[-1], m.crossatt.h
    d = C // h
    c = [getattr(m, f"coefficient{j}").bias for j in range(1, 9)]
    seeds = list(seeds)

    def drop(t, p):
        if p <= 0:
            return t
        keep = DM.eltwise_keep(B * n_pad * C, seeds.pop(0), 0, p, t.device).view(B, n_pad, C)[:, :N]
        return t * keep / float(np.float32(1) - np.float32(p))

    heads = lambda t: t.reshape(B, N, h, d).permute(0, 2, 1, 3)      # noqa: E731
    for _ in range(m.loops):
        a = m.crossatt
        xr, xi = a.LN1(r), a.LN2(i)
        qv, kv, vv = heads(a.que_proj_vis(xr)), heads(a.key_proj_vis(xr)), heads(a.val_proj_vis(xr))
        qi, ki, vi = heads(a.que_proj_ir(xi)), heads(a.key_proj_ir(xi)), heads(a.val_proj_ir(xi))
        att_v = torch.softmax(qi @ kv.transpose(-1, -2) / d ** 0.5, -1)        # RGB output: IR queries on RGB keys
        att_i = torch.softmax(qv @ ki.transpose(-1, -2) / d ** 0.5, -1)
        if p_att > 0:
            mk = DM.attn_keep_mask(seeds.pop(0), 0, B, h, N, p_att, r.device).view(2, B, h, N, N)
            att_v, att_i = att_v * mk[0] / (1 - p_att), att_i * mk[1] / (1 - p_att)
        ov = drop(a.out_proj_vis((att_v @ vv).permute(0, 2, 1, 3).reshape(B, N, C)), p_res)
        oi = drop(a.out_proj_ir((att_i @ vi).permute(0, 2, 1, 3).reshape(B, N, C)), p_res)
        ra, ia = c[0] * r + c[1] * ov, c[2] * i + c[3] * oi
        mv = drop(m.mlp_vis[2](F.gelu(m.mlp_vis[0](m.LN2(ra)))), p_res)
        mi = drop(m.mlp_ir[2](F.gelu(m.mlp_ir[0](m.LN2(ia)))), p_res)
        r, i = c[4] * ra + c[5] * mv, c[6] * ia + c[7] * mi
    return r, i


@pytest.mark.parametrize("C,N,loops,p", [(64, 256, 1, 0.0), (64, 256, 2, 0.1), (256, 100, 2, 0.0), (256, 400, 1, 0.1),
                                         (1024, 100, 1, 0.1)])
def test_cross_transformer_block_chain_f32(cuda_device, C, N, loops, p):
    """The whole CrossTransformerBlock on fp32 streams -- LayerNorms, fp16 GEMMs, attention, GELU, dropout, coefficient pairs,
    the stream fed back for loops > 1 -- against fp32 autograd with the same masks; and the same block on fp16 streams from
    the same (fp16-representable) tokens: the fp32 streams must bring the block's worst one-element gradient closer to fp32
    (the median is printed; it moves either way)."""
    import copy
    from icafusion_b200 import autograd as A
    from icafusion_b200.common import CrossTransformerBlock
    dev = cuda_device
    B, h = 2, 8
    n_pad = (N + 7) // 8 * 8
    g = torch.Generator().manual_seed(C * loops + N)
    blk = CrossTransformerBlock(C, C, C, h, 4, p, p, loops)
    _init_block(blk, g)
    blk = blk.to(dev).train()
    ref = copy.deepcopy(blk)
    r0, i0 = (torch.randn(B, N, C, generator=g).half().float().to(dev) for _ in range(2))
    dr, di = (torch.randn(B, N, C, generator=g).to(dev) for _ in range(2))
    pad = lambda t: torch.cat([t, t.new_zeros(B, n_pad - N, C)], 1)      # noqa: E731
    res = {}
    for dtype in (torch.float32, torch.float16):
        dev_blk = copy.deepcopy(blk)
        rd, id_ = (pad(t).reshape(B * n_pad, C).to(dtype).clone().requires_grad_(True) for t in (r0, i0))
        A.manual_seed(4321)
        c0 = A._STATE["count"]
        r2, i2 = A.cross_transformer_block(dev_blk, rd, id_, B, N, n_pad)
        n_seeds = A._STATE["count"] - c0
        assert r2.dtype == i2.dtype == dtype
        dy = [pad(t).reshape(B * n_pad, C).to(dtype) for t in (dr, di)]
        torch.autograd.backward([r2, i2], dy)
        res[dtype] = (dev_blk, r2.detach().float(), i2.detach().float(), rd.grad.float(), id_.grad.float())
    A.manual_seed(4321)
    seeds = [A.next_seed() for _ in range(n_seeds)]
    assert n_seeds == (loops * 5 if p > 0 else 0)
    rr, ir_ = (t.clone().requires_grad_(True) for t in (r0, i0))
    yr, yi = _ref_block(ref, rr, ir_, B, N, n_pad, seeds, p, p)
    ((yr * dr).sum() + (yi * di).sum()).backward()
    torch.cuda.synchronize()
    pr = dict(ref.named_parameters())
    gmax = max(float(q.grad.norm()) for q in pr.values() if q.grad is not None)
    worst = {}
    for dtype, (dev_blk, r2, i2, gr, gi) in res.items():
        e_y = max(_rel(r2.view(B, n_pad, C)[:, :N], yr), _rel(i2.view(B, n_pad, C)[:, :N], yi))
        e_x = max(_rel(gr.view(B, n_pad, C)[:, :N], rr.grad), _rel(gi.view(B, n_pad, C)[:, :N], ir_.grad))
        multi, scal = [], []
        for k, q in dev_blk.named_parameters():
            if pr[k].grad is None:
                assert q.grad is None, k
                continue
            e = _rel(q.grad, pr[k].grad, 1e-3 * gmax)
            (multi if q.numel() > 1 else scal).append((e, k))
        worst[dtype] = (e_y, e_x, max(multi), max(scal), float(np.median([e for e, _ in scal])))
        print(f"\n[block {'fp32' if dtype == torch.float32 else 'fp16'} streams C{C} N{N} loops {loops} p {p}] out {e_y:.1e}  "
              f"dx {e_x:.1e}  worst parameter {max(multi)[0]:.1e} ({max(multi)[1]})  one-element: worst {max(scal)[0]:.1e} "
              f"({max(scal)[1]}), median {worst[dtype][4]:.1e}")
    e_y, e_x, wm, ws, med = worst[torch.float32]
    assert e_y < 5e-3 and e_x < 1e-2
    assert wm[0] < 3e-2, wm
    assert ws[0] < 5e-2, ws
    # the measured gain of the fp32 streams on the block's one-element gradients
    assert ws[0] < worst[torch.float16][3][0], (worst[torch.float32], worst[torch.float16])


# ------------------------------------------------------------------------------------------------ the whole step

# One-element gradients over the un-exempted bar with fp32 streams (measured on an H100 at both loss scales).  Every one of
# them is over it with fp16 streams as well, at nearly the same e_k (the test prints both columns): yolov5l's
# model.20.crosstransformer.0.coefficient3.bias is at 1.17 with fp32 streams and 1.10 with fp16 streams, against ea_k 1.3e-2.
# Their error does not come from the streams' precision, which the fp32 streams match to the reference's; what sets them
# apart from the scalars that pass is the autocast oracle's distance from fp32: their ea_k (1.8e-3 .. 1.8e-1) is small
# against their e_k, which lies inside the range of the passing e_k of the same case.  They stay held to EXEMPT's bar.
STILL_OVER = {
    "train_yolov5s_320": {"model.20.vis_coefficient.w2", "model.20.crosstransformer.0.coefficient2.bias",
                          "model.21.ir_coefficient.w1"},
    "train_yolov5s_640": {"model.20.ir_coefficient.w2", "model.20.crosstransformer.0.coefficient4.bias",
                          "model.20.crosstransformer.0.coefficient6.bias", "model.21.crosstransformer.0.coefficient2.bias",
                          "model.21.crosstransformer.0.coefficient8.bias", "model.22.crosstransformer.0.coefficient2.bias",
                          "model.22.crosstransformer.0.coefficient6.bias"},
    "train_yolov5l_320": {"model.20.crosstransformer.0.coefficient3.bias", "model.20.crosstransformer.0.coefficient5.bias",
                          "model.22.crosstransformer.0.coefficient8.bias"},
}

@pytest.mark.parametrize("case", ["train_yolov5n_flir_320", "train_yolov5s_320", "train_yolov5s_640", "train_yolov5l_320"])
def test_training_step_fp32_streams(cuda_device, case, monkeypatch):
    """The whole-model gradient check of tests/train_grads.py (loss scales 2^8 and 2^16), run with fp16 and with fp32 DMFF
    streams.  Prints every LearnableCoefficient / LearnableWeights gradient's e_k under both, side by side.  With fp32 streams
    every one of them but the ones STILL_OVER names meets the un-exempted bar max(BETA * ea_k, TAU), and none misses it
    that fp16 streams do not miss.  (The streams' precision moves these e_k by a few per cent: no gain is asserted.)"""
    import icafusion_b200
    import train_grads
    from icafusion_b200.trainer import set_dmff_stream_dtype
    real_model, real_check = icafusion_b200.Model, train_grads.tensor_check
    exempt = [pat for pat, _, _, _ in train_grads.EXEMPT]
    rows = {}

    for fp32 in (False, True):
        calls = rows[fp32] = []

        def model(*a, fp32=fp32, **k):
            m = real_model(*a, **k)
            set_dmff_stream_dtype(m, fp32)
            return m

        def check(got, ref, amp, *a, calls=calls, **k):
            out = real_check(got, ref, amp, *a, **k)
            calls.append({r[4]: r[:2] for r in out[0] if any(p.search(r[4]) for p in exempt)})
            return out
        monkeypatch.setattr(icafusion_b200, "Model", model)
        monkeypatch.setattr(train_grads, "tensor_check", check)
        train_grads.run_case(cuda_device, case)
    # the first check of a case is its 2^8 step (the mutations and the 2^16 step follow)
    s16, s32 = rows[False][0], rows[True][0]
    assert sorted(s16) == sorted(s32) and len(s16) == 36
    bar = lambda ea: max(train_grads.BETA * ea, train_grads.TAU)      # noqa: E731
    print(f"\n[{case} one-element gradients at 2^8] e_k with fp16 streams, e_k with fp32 streams, ea_k (fp16-autocast oracle)")
    for k in sorted(s16, key=lambda k: -s16[k][0]):
        (e16, ea), (e32, _) = s16[k], s32[k]
        print(f"    {e16:.2e} {e32:.2e} {ea:.2e}  {'over' if e16 > bar(ea) else '    '} {'over' if e32 > bar(ea) else '    '}  {k}")
    stats = {}
    for name, sc in (("fp16", s16), ("fp32", s32)):
        ratio = [e / max(ea, 1e-30) for e, ea in sc.values()]
        passing = [e for e, ea in sc.values() if e <= bar(ea)]
        stats[name] = dict(worst=max(ratio), median=float(np.median(ratio)), median_e=float(np.median([e for e, _ in sc.values()])),
                           over=sum(e > bar(ea) for e, ea in sc.values()), passing_e=(min(passing, default=0), max(passing, default=0)))
        print(f"[{case} {name} streams] e_k / ea_k worst {stats[name]['worst']:.2f}, median {stats[name]['median']:.2f}; median e_k "
              f"{stats[name]['median_e']:.2e}; {stats[name]['over']} of {len(sc)} over the un-exempted bar; passing e_k from "
              f"{stats[name]['passing_e'][0]:.1e} to {stats[name]['passing_e'][1]:.1e}")
    over = {}
    for calls in rows[True]:
        for k, (e, ea) in calls.items():
            if e > bar(ea):
                over[k] = (e, ea)
    unexpected = {k: v for k, v in over.items() if k not in STILL_OVER.get(case, ())}
    assert not unexpected, unexpected
    new = sorted(k for k, (e, ea) in s32.items() if e > bar(ea) and s16[k][0] <= bar(ea))
    assert not new, new                                  # fp32 streams add no miss at 2^8


# ------------------------------------------------------------------------------------------------ graph capture, PDL

def _child(out_path):
    """The train_yolov5s_320 batch for three calls (an accumulation window of two, then one step), eager and from
    GraphedTrainStep(dmff_fp32=...), with fp32 and with fp16 DMFF streams: losses, gradients and state after every call, to
    out_path."""
    sys.path[:0] = [ROOT, HERE]
    from conftest import load_golden
    from helpers import load_synth
    from icafusion_b200 import Model
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep
    from oracle import synth
    from oracle.gen_golden_train import synth_targets
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    m, _ = load_golden("train_yolov5s_320")
    B, H, W = m["B"], m["H"], m["W"]
    data = []
    for s in range(3):
        rgb, ir = synth.synth_images(B, H, W, m["seed"] + s)
        data.append(((rgb * 255).to(torch.uint8).to(dev), (ir * 255).to(torch.uint8).to(dev),
                     torch.from_numpy(synth_targets(m["nt"], B, m["seed"] + s)).to(dev)))
    flags = (False, True, True)
    res = {}
    for graphed, fp32 in ((False, True), (True, True), (False, False), (True, False)):
        model = Model("yolov5s_Transfusion_kaist")
        load_synth(model, m["seed"])
        model = model.to(dev).train()
        for mod in model.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
        ts = TrainStep(model, None, total_batch_size=B, imgsz=H, dmff_fp32=fp32 and not graphed)   # the graphed one sets it itself
        step = GraphedTrainStep(ts, B, H, W, 16, dev, dmff_fp32=fp32) if graphed else None
        tag = ("graphed" if graphed else "eager") + ("" if fp32 else "16")
        for n, (batch, flag) in enumerate(zip(data, flags)):
            if graphed:
                loss = step(*batch, optimizer_step=flag)[0]
            else:
                loss = ts(*batch, optimizer_step=False)[0]
            if flag and not graphed:                       # the optimizer_step=True branch of TrainStep.__call__, with the
                ts.scaler.unscale_(ts.optimizer)           # unscaled gradients read before SGD runs: torch's foreach nesterov
            torch.cuda.synchronize()                       # adds momentum * buf into .grad in place where weight_decay is 0,
            res[f"{tag} {n} loss"] = loss.detach().clone()     # the device step leaves .grad the gradient
            res.update({f"{tag} {n} grad {k}": v.grad.detach().clone() for k, v in model.named_parameters() if v.grad is not None})
            if flag and not graphed:
                ts.scaler.step(ts.optimizer)
                ts.scaler.update()
                ts.zero_grad()
            res.update({f"{tag} {n} state {k}": v.detach().clone() for k, v in model.state_dict().items()})
        if graphed:
            assert step.acc_graph is not None
            step.close()
        torch.cuda.synchronize()
        res[f"{tag} scale"] = torch.tensor([float(ts.scaler.get_scale())])
        del model, ts, step
    torch.save({k: v.cpu() for k, v in res.items()}, out_path)


def test_graphed_fp32_streams_equal_eager_pdl_on_and_off(tmp_path):
    """Three calls -- a fresh micro-batch, the accumulating one that steps, and a fresh one that steps -- from
    GraphedTrainStep equal the eager TrainStep's bit for bit (losses, unscaled gradients, parameters, buffers, GradScaler's
    scale), with fp32 and with fp16 DMFF streams, with PDL on and off."""
    raw = lambda x: x.contiguous().reshape(-1).view(torch.uint8)                # noqa: E731  (bits, so NaNs compare too)
    runs = {}
    for pdl in ("0", "1"):
        out = tmp_path / f"pdl{pdl}.pt"
        p = subprocess.run([sys.executable, os.path.abspath(__file__), str(out)], env=dict(os.environ, ICAF_PDL=pdl), cwd=ROOT,
                           capture_output=True, text=True, timeout=1500)
        assert p.returncode == 0, f"ICAF_PDL={pdl} child failed:\n{p.stdout[-4000:]}\n{p.stderr[-4000:]}"
        r = torch.load(out)
        for sfx in ("", "16"):
            eager = {k[len("eager" + sfx) + 1:]: v for k, v in r.items() if k.startswith(f"eager{sfx} ")}
            graphed = {k[len("graphed" + sfx) + 1:]: v for k, v in r.items() if k.startswith(f"graphed{sfx} ")}
            assert sorted(eager) == sorted(graphed) and any(" grad " in k for k in eager)
            diff = [k for k in eager if eager[k].dtype != graphed[k].dtype or not torch.equal(raw(eager[k]), raw(graphed[k]))]
            worst = max([float((graphed[k].double() - eager[k].double()).abs().max() / max(float(eager[k].double().abs().max()), 1e-6))
                         for k in diff if eager[k].is_floating_point()] + [0.0])
            by_call = {n: sum(k.startswith(f"{n} ") for k in diff) for n in range(3)}
            print(f"\n[{'fp32' if not sfx else 'fp16'} streams, ICAF_PDL={pdl}] {len(eager)} tensors, graphed against eager: "
                  f"{len(diff)} differ (per call {by_call}), worst relative {worst:.2e}: {diff[:6]}")
            assert not diff, diff[:20]
        runs[pdl] = r
    diff = [k for k in runs["0"] if not torch.equal(raw(runs["0"][k]), raw(runs["1"][k]))]
    assert not diff, diff[:20]


def test_default_streams_unchanged(cuda_device):
    """dmff_fp32=False gives the gradients of a step that never mentions the flag, bit for bit; fp32 streams change them."""
    from helpers import load_synth
    from icafusion_b200 import Model
    from icafusion_b200.trainer import TrainStep
    from oracle import synth
    from oracle.gen_golden_train import synth_targets
    B, H = 2, 320
    rgb, ir = synth.synth_images(B, H, H, 11)
    batch = ((rgb * 255).to(torch.uint8).to(cuda_device), (ir * 255).to(torch.uint8).to(cuda_device),
             torch.from_numpy(synth_targets(8, B, 11)).to(cuda_device))
    grads = []
    for kw in ({}, {"dmff_fp32": False}, {"dmff_fp32": True}):
        model = Model("yolov5s_Transfusion_kaist")
        load_synth(model, 11)
        model = model.to(cuda_device).train()
        for mod in model.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
        ts = TrainStep(model, None, total_batch_size=B, imgsz=H, **kw)
        ts(*batch, optimizer_step=False)
        torch.cuda.synchronize()
        grads.append({k: v.grad.clone() for k, v in model.named_parameters() if v.grad is not None})
        del model, ts
    assert sorted(grads[0]) == sorted(grads[1]) == sorted(grads[2])
    assert all(torch.equal(grads[0][k], grads[1][k]) for k in grads[0])
    changed = [k for k in grads[0] if not torch.equal(grads[0][k], grads[2][k])]
    print(f"\n[default streams] flag off == flag never mentioned; fp32 streams change {len(changed)} of {len(grads[0])} gradients")
    assert any("coefficient" in k for k in changed)


if __name__ == "__main__":
    _child(sys.argv[1])
