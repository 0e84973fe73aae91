"""Training-step building blocks (operator level): weight / data / bias gradients of the Conv2d and Linear layers of the
hot path against torch autograd (CPU, fp32, on the same fp16-rounded operands)."""
import pytest
import torch
import torch.nn.functional as F

import dropout_mask as DM
from helpers import err, nhwc

pytestmark = pytest.mark.gpu


def _grads(x, w, dy, s, p):
    x = x.float().requires_grad_(True)
    w = w.float().requires_grad_(True)
    y = F.conv2d(x, w, None, stride=s, padding=p)
    y.backward(dy.float())
    return x.grad, w.grad


@pytest.mark.parametrize("B,Cin,H,W,Cout,k,s,p", [
    (2, 64, 16, 20, 64, 1, 1, 0), (2, 64, 32, 40, 128, 3, 1, 1), (3, 128, 16, 20, 256, 3, 2, 1), (1, 256, 16, 20, 128, 1, 1, 0),
    (4, 64, 33, 47, 64, 3, 1, 1), (2, 192, 16, 24, 64, 3, 1, 1), (8, 16, 64, 80, 32, 3, 1, 1), (2, 32, 32, 40, 64, 3, 2, 1),
    (16, 128, 64, 80, 128, 3, 1, 1), (2, 512, 16, 20, 24, 1, 1, 0)])
def test_conv_weight_and_data_gradients(cuda_device, B, Cin, H, W, Cout, k, s, p):
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(B * 100 + Cin + k)
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x = torch.randn(B, Cin, H, W, generator=g).half()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).half()
    dy = (torch.randn(B, Cout, Ho, Wo, generator=g) * 0.1).half()
    dx_ref, dw_ref = _grads(x, w, dy, s, p)
    xv, dyv = nhwc(x).to(cuda_device), nhwc(dy).to(cuda_device)
    dw = ops.conv2d_wgrad(xv, dyv, k, k, s, p)
    acc = dw.clone()
    ops.conv2d_wgrad(xv, dyv, k, k, s, p, scale=0.5, out=acc)            # accumulate with a scale: .grad += 0.5 dW
    dx = ops.conv2d_dgrad(dyv, w.float().to(cuda_device), s, p, (H, W))
    torch.cuda.synchronize()
    e_w = err(dw, dw_ref)
    print(f"\n[grads B{B} {Cin}->{Cout} {H}x{W} k{k}s{s}] dW {e_w:.2e}" + ("" if dx is None else f"  dX {err(dx.permute(0, 3, 1, 2), dx_ref):.2e}"))
    assert e_w < 1e-3
    assert err(acc, dw_ref * 1.5) < 1e-3
    if dx is not None:
        assert err(dx.permute(0, 3, 1, 2), dx_ref) < 1.5e-3          # fp16 output
    dw2 = ops.conv2d_wgrad(xv, dyv, k, k, s, p)
    assert torch.equal(dw, dw2), "wgrad is not deterministic"


def test_linear_and_bias_gradients(cuda_device):
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(9)
    for rows, K, N in ((400, 256, 768), (6400, 256, 1024), (1664, 1024, 64), (104, 4096, 1024)):
        x = torch.randn(rows, K, generator=g).half()
        dy = (torch.randn(rows, N, generator=g) * 0.1).half()
        dw = ops.linear_wgrad(x.to(cuda_device), dy.to(cuda_device))
        db = ops.colsum(dy.to(cuda_device))
        torch.cuda.synchronize()
        assert err(dw, dy.float().t() @ x.float()) < 1e-3, (rows, K, N)
        assert err(db, dy.float().sum(0)) < 1e-4


def test_batchnorm_silu_training_forward_backward(cuda_device):
    """Conv.forward in training mode after the convolution (models/common.py:56-57): BatchNorm2d with batch statistics + SiLU,
    forward (incl. the running-statistics update) and backward vs torch autograd."""
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(4)
    for B, C, H, W, act in ((4, 64, 32, 40, 1), (2, 256, 16, 20, 1), (16, 128, 64, 80, 1), (3, 64, 9, 11, 0)):
        x = (torch.randn(B, C, H, W, generator=g) * 1.3 + 0.2).half()
        dy = (torch.randn(B, C, H, W, generator=g) * 0.1).half()
        gamma, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
        bn = torch.nn.BatchNorm2d(C, eps=1e-3, momentum=0.03)
        with torch.no_grad():
            bn.weight.copy_(gamma); bn.bias.copy_(beta)
        xr = x.float().requires_grad_(True)
        yr = bn(xr)
        yr = F.silu(yr) if act else yr
        yr.backward(dy.float())
        rm, rv = torch.zeros(C, device=cuda_device), torch.ones(C, device=cuda_device)
        gd, bd = gamma.to(cuda_device), beta.to(cuda_device)
        xv = nhwc(x).to(cuda_device)
        y, sm, si = ops.bn_act_fwd(xv, gd, bd, rm, rv, 1e-3, 0.03, act)
        dg, db = torch.zeros(C, device=cuda_device), torch.zeros(C, device=cuda_device)
        dx = ops.bn_act_bwd(xv, nhwc(dy).to(cuda_device), gd, bd, sm, si, act, dg, db)
        torch.cuda.synchronize()
        assert err(y.permute(0, 3, 1, 2), yr) < 1e-3
        assert err(rm, bn.running_mean) < 1e-4 and err(rv, bn.running_var) < 1e-4
        assert err(dx.permute(0, 3, 1, 2), xr.grad) < 2e-3
        assert err(dg, bn.weight.grad) < 1e-3 and err(db, bn.bias.grad) < 1e-3


def test_small_training_kernels(cuda_device):
    """GELU forward/backward, LayerNorm backward, dot products, nearest-upsample and SPPF max-pool backward, dropout."""
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(6)
    x = torch.randn(400, 256, generator=g).half()
    dy = (torch.randn(400, 256, generator=g) * 0.1).half()
    xr = x.float().requires_grad_(True)
    F.gelu(xr).backward(dy.float())
    xd, dyd = x.to(cuda_device), dy.to(cuda_device)
    assert err(ops.eltwise(0, xd), F.gelu(x.float())) < 1e-3
    assert err(ops.eltwise(1, xd, dyd), xr.grad) < 1e-3
    gamma, beta = 1 + 0.2 * torch.randn(256, generator=g), 0.2 * torch.randn(256, generator=g)
    xr = x.float().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    F.layer_norm(xr, (256,), gr, br, 1e-5).backward(dy.float())
    dg, db = torch.zeros(256, device=cuda_device), torch.zeros(256, device=cuda_device)
    dx = ops.layernorm_bwd(xd, dyd, gamma.to(cuda_device), 1e-5, dg, db)
    torch.cuda.synchronize()
    assert err(dx, xr.grad) < 1.5e-3 and err(dg, gr.grad) < 1e-3 and err(db, br.grad) < 1e-3
    assert abs(float(ops.dot(xd, dyd)) - float((x.float() * dy.float()).sum())) < 1e-2
    # nearest 2x up-sampling and one SPPF pool stage
    m = torch.randn(2, 64, 16, 20, generator=g).half()
    d2 = torch.randn(2, 64, 32, 40, generator=g).half()
    mr = m.float().requires_grad_(True)
    F.interpolate(mr, scale_factor=2, mode="nearest").backward(d2.float())
    assert err(ops.upsample2x_bwd(nhwc(d2).to(cuda_device)).permute(0, 3, 1, 2), mr.grad) < 1e-3
    d1 = torch.randn(2, 64, 16, 20, generator=g).half()
    mr = m.float().requires_grad_(True)
    F.max_pool2d(mr, 5, 1, 2).backward(d1.float())
    assert err(ops.maxpool5_bwd(nhwc(m).to(cuda_device), nhwc(d1).to(cuda_device)).permute(0, 3, 1, 2), mr.grad) < 1e-3
    # dropout: keeps ~ (1 - p), scales by 1 / (1 - p), same mask for the same seed; bit for bit the restated mask and scale
    ones = torch.ones(1 << 16, dtype=torch.float16, device=cuda_device)
    a, b2, c2 = ops.eltwise(2, ones, p=0.1, seed=7), ops.eltwise(2, ones, p=0.1, seed=7), ops.eltwise(2, ones, p=0.1, seed=8)
    keep = float((a > 0).float().mean())
    assert torch.equal(a, b2) and not torch.equal(a, c2) and abs(keep - 0.9) < 0.01 and abs(float(a.max()) - 1 / 0.9) < 1e-3
    for y, seed in ((a, 7), (c2, 8)):
        want = DM.eltwise_dropout(ones, DM.eltwise_keep(ones.numel(), seed, 0, 0.1, cuda_device), 0.1)
        assert torch.equal(y.view(torch.int16), want.view(torch.int16)), seed


def _attn_ref(qkv_q, qkv_kv, N, C, h, mask=None, p=0.0):
    """One direction of the cross-attention (common.py:670-684) with autograd; mask (B, h, N, N) = kept probabilities."""
    B = qkv_q.shape[0]
    d = C // h
    q = qkv_q[:, :N, :C].reshape(B, N, h, d).permute(0, 2, 1, 3)
    k = qkv_kv[:, :N, C:2 * C].reshape(B, N, h, d).permute(0, 2, 1, 3)
    v = qkv_kv[:, :N, 2 * C:].reshape(B, N, h, d).permute(0, 2, 1, 3)
    att = torch.softmax(q @ k.transpose(-1, -2) / d ** 0.5, -1)
    if mask is not None:
        att = att * mask / (1 - p)
    return (att @ v).permute(0, 2, 1, 3).reshape(B, N, C)


@pytest.mark.parametrize("B,N,C,h", [(2, 100, 128, 8), (1, 333, 256, 8), (1, 200, 512, 8), (1, 150, 1024, 8), (2, 77, 64, 4)])
def test_cross_attention_backward(cuda_device, B, N, C, h):
    """dq, dk, dv of both directions against torch autograd (fp32 on the same fp16 operands), eval (no dropout)."""
    from icafusion_b200 import ops
    n_pad = ops.round_up(N, 8)
    g = torch.Generator().manual_seed(N + C)
    qv, qi = torch.randn(B, n_pad, 3 * C, generator=g).half(), torch.randn(B, n_pad, 3 * C, generator=g).half()
    dov, doi = (torch.randn(B, n_pad, C, generator=g) * 0.1).half(), (torch.randn(B, n_pad, C, generator=g) * 0.1).half()
    rv, ri = qv.float().requires_grad_(True), qi.float().requires_grad_(True)
    o_v, o_i = _attn_ref(ri, rv, N, C, h), _attn_ref(rv, ri, N, C, h)     # RGB output: IR queries on RGB keys/values
    (o_v * dov[:, :N].float()).sum().backward(retain_graph=True)
    (o_i * doi[:, :N].float()).sum().backward()
    dev = [t.to(cuda_device) for t in (qv, qi)]
    out_v, out_i = ops.cross_attention_train(*dev, B, N, n_pad, C, h)
    dq_v, dq_i = ops.cross_attention_bwd(*dev, out_v, out_i, dov.to(cuda_device), doi.to(cuda_device), B, N, n_pad, C, h)
    torch.cuda.synchronize()
    e_o = max(err(out_v[:, :N], o_v.detach()), err(out_i[:, :N], o_i.detach()))
    e_g = max(err(dq_v[:, :N], rv.grad[:, :N]), err(dq_i[:, :N], ri.grad[:, :N]))
    print(f"\n[attention bwd B{B} N{N} C{C} d{C // h}] out {e_o:.2e}  dqkv {e_g:.2e}")
    assert e_o < 1e-3 and e_g < 2e-3
    if n_pad > N:
        assert float(dq_v[:, N:].abs().max()) == 0 and float(dq_i[:, N:].abs().max()) == 0


def test_cross_attention_dropout(cuda_device):
    """Attention dropout: the mask is read back through identity values, then the dropped forward and its backward are checked
    against autograd with that mask; the keep rate and seed behaviour are checked too."""
    from icafusion_b200 import ops
    B, N, C, h, p, seed = 2, 64, 256, 4, 0.25, 1234
    d, n_pad = C // h, 64
    g = torch.Generator().manual_seed(3)
    qv, qi = torch.randn(B, n_pad, 3 * C, generator=g).half(), torch.randn(B, n_pad, 3 * C, generator=g).half()
    qv[:, :, :2 * C] *= 0.3
    qi[:, :, :2 * C] *= 0.3                                   # flat-ish rows: every probability stays well above fp16 zero
    eye = torch.eye(N).reshape(1, N, 1, d).expand(B, N, h, d).reshape(B, N, C).half()     # v[key, head, c] = (key == c)
    pv, pi = qv.clone(), qi.clone()
    pv[:, :, 2 * C:], pi[:, :, 2 * C:] = eye, eye
    m_v, m_i = ops.cross_attention_train(pv.to(cuda_device), pi.to(cuda_device), B, N, n_pad, C, h, p, seed)
    mask_v = (m_v.cpu().reshape(B, N, h, d).permute(0, 2, 1, 3) > 0).float()              # (B, h, q, key)
    mask_i = (m_i.cpu().reshape(B, N, h, d).permute(0, 2, 1, 3) > 0).float()
    keep = float(torch.cat([mask_v, mask_i]).mean())
    assert abs(keep - (1 - p)) < 0.02 and not torch.equal(mask_v, mask_i)
    want = DM.attn_keep_mask(seed, 0, B, h, N, p).view(2, B, h, N, N)
    assert torch.equal(mask_v.bool(), want[0]) and torch.equal(mask_i.bool(), want[1])
    m2, _ = ops.cross_attention_train(pv.to(cuda_device), pi.to(cuda_device), B, N, n_pad, C, h, p, seed + 1)
    assert not torch.equal(m2, m_v)
    dov, doi = (torch.randn(B, n_pad, C, generator=g) * 0.1).half(), (torch.randn(B, n_pad, C, generator=g) * 0.1).half()
    rv, ri = qv.float().requires_grad_(True), qi.float().requires_grad_(True)
    o_v, o_i = _attn_ref(ri, rv, N, C, h, mask_v, p), _attn_ref(rv, ri, N, C, h, mask_i, p)
    (o_v * dov.float()).sum().backward(retain_graph=True)
    (o_i * doi.float()).sum().backward()
    dev = [t.to(cuda_device) for t in (qv, qi)]
    out_v, out_i = ops.cross_attention_train(*dev, B, N, n_pad, C, h, p, seed)
    dq_v, dq_i = ops.cross_attention_bwd(*dev, out_v, out_i, dov.to(cuda_device), doi.to(cuda_device), B, N, n_pad, C, h, p, seed)
    torch.cuda.synchronize()
    e_o = max(err(out_v, o_v.detach()), err(out_i, o_i.detach()))
    e_g = max(err(dq_v, rv.grad), err(dq_i, ri.grad))
    print(f"\n[attention dropout p{p}] keep {keep:.3f}  out {e_o:.2e}  dqkv {e_g:.2e}")
    assert e_o < 1.5e-3 and e_g < 2e-3


def _ref_pool_tokens(x, pos, w1, w2, nh, nw):
    """AdaptivePool2d avg / max (common.py:868-891) mixed by LearnableWeights + positional embedding (common.py:817-819)."""
    B, C, H, W = x.shape
    if H > nh or W > nw:
        sh, sw = H // nh, W // nw
        k = (H - (nh - 1) * sh, W - (nw - 1) * sw)
        a, m = F.avg_pool2d(x, k, (sh, sw)), F.max_pool2d(x, k, (sh, sw))
    else:
        a = m = x
    return (w1 * a + w2 * m).flatten(2).permute(0, 2, 1) + pos


@pytest.mark.parametrize("B,C,H,W,va,ha", [(2, 64, 40, 40, 20, 20), (2, 128, 20, 20, 16, 16), (1, 64, 64, 80, 20, 20), (2, 64, 10, 10, 10, 10)])
def test_dmff_pool_and_tail_nodes(cuda_device, B, C, H, W, va, ha):
    """PoolTokensFn / UpsampleCatFn (token pooling with overlapping windows, nearest tail) forward + backward vs torch autograd."""
    from icafusion_b200 import autograd as A
    g = torch.Generator().manual_seed(H * W + va)
    nh, nw = (va, ha) if (H > va or W > ha) else (H, W)
    N = nh * nw
    rgb, ir = torch.randn(B, C, H, W, generator=g).half(), torch.randn(B, C, H, W, generator=g).half()
    rgb[0, :, 0:3, 0:3] = rgb[0, :, 0:1, 0:1]                     # ties inside a window: the first maximum takes the gradient
    pos = [(0.1 * torch.randn(1, N, C, generator=g)).half().float() for _ in range(2)]
    wts = [torch.tensor([v]) for v in (0.6, 0.4, 0.3, 0.7)]
    dtok = [(0.1 * torch.randn(B, N, C, generator=g)).half() for _ in range(2)]
    dcat = (0.1 * torch.randn(B, 2 * C, H, W, generator=g)).half()
    # reference (fp32 autograd on the same fp16-rounded operands)
    R = [t.float().requires_grad_(True) for t in (rgb, ir)]
    P = [t.clone().requires_grad_(True) for t in pos]
    Wt = [t.clone().requires_grad_(True) for t in wts]
    tr = [_ref_pool_tokens(R[0], P[0], Wt[0], Wt[1], nh, nw), _ref_pool_tokens(R[1], P[1], Wt[2], Wt[3], nh, nw)]
    (tr[0] * dtok[0].float()).sum().backward(retain_graph=True)
    (tr[1] * dtok[1].float()).sum().backward()
    # device
    dev = cuda_device
    Rd = [nhwc(t).to(dev).requires_grad_(True) for t in (rgb, ir)]
    Pd = [t.clone().to(dev).requires_grad_(True) for t in pos]
    Wd = [t.clone().to(dev).requires_grad_(True) for t in wts]
    tv, ti = A.PoolTokensFn.apply(Rd[0], Rd[1], Pd[0], Pd[1], Wd[0], Wd[1], Wd[2], Wd[3], nh, nw)
    n_pad = tv.shape[1]
    pad = lambda t: torch.cat([t, t.new_zeros(B, n_pad - N, C)], 1).to(dev)      # noqa: E731
    ((tv.float() * pad(dtok[0]).float()).sum() + (ti.float() * pad(dtok[1]).float()).sum()).backward()
    e_f = max(err(tv[:, :N], tr[0]), err(ti[:, :N], tr[1]))
    e_x = max(err(Rd[0].grad.permute(0, 3, 1, 2), R[0].grad), err(Rd[1].grad.permute(0, 3, 1, 2), R[1].grad))
    e_p = max(err(Pd[0].grad, P[0].grad), err(Pd[1].grad, P[1].grad))
    e_w = max(err(Wd[k].grad, Wt[k].grad) for k in range(4))
    print(f"\n[pool tokens {H}x{W}->{nh}x{nw} C{C}] fwd {e_f:.2e}  dx {e_x:.2e}  dpos {e_p:.2e}  dmix {e_w:.2e}")
    assert e_f < 1e-3 and e_x < 2e-3 and e_p < 1e-3 and e_w < 5e-3     # dmix: a cancelling sum of fp16-rounded token products
    # tail: nearest resample + residual + concat
    tok = [(torch.randn(B, N, C, generator=g)).half() for _ in range(2)]
    T = [t.float().requires_grad_(True) for t in tok]
    R = [t.float().requires_grad_(True) for t in (rgb, ir)]
    up = lambda t: F.interpolate(t.reshape(B, nh, nw, C).permute(0, 3, 1, 2), size=(H, W), mode="nearest")   # noqa: E731
    cat = torch.cat([up(T[0]) + R[0], up(T[1]) + R[1]], 1)
    (cat * dcat.float()).sum().backward()
    Td = [pad(t).requires_grad_(True) for t in tok]
    Rd = [nhwc(t).to(dev).requires_grad_(True) for t in (rgb, ir)]
    cd = A.UpsampleCatFn.apply(Td[0], Td[1], Rd[0], Rd[1], nh, nw)
    (cd.float() * nhwc(dcat).to(dev).float()).sum().backward()
    e_f = err(cd.permute(0, 3, 1, 2), cat)
    e_t = max(err(Td[0].grad[:, :N], T[0].grad), err(Td[1].grad[:, :N], T[1].grad))
    e_x = max(err(Rd[0].grad.permute(0, 3, 1, 2), R[0].grad), err(Rd[1].grad.permute(0, 3, 1, 2), R[1].grad))
    print(f"[tail {nh}x{nw}->{H}x{W}] fwd {e_f:.2e}  dtok {e_t:.2e}  dx {e_x:.2e}")
    assert e_f < 1e-3 and e_t < 2e-3 and e_x < 1e-3
    assert float(Td[0].grad[:, N:].abs().max() if n_pad > N else 0.0) == 0.0


def test_conv_bn_act_node(cuda_device):
    """ConvBnActFn (common.Conv in train()): forward, running statistics, and all four gradients vs torch autograd; also the
    6x6 / stride-2 image stem through its space-to-depth form."""
    import torch.nn as nn
    from icafusion_b200 import autograd as A
    from icafusion_b200 import common
    g = torch.Generator().manual_seed(21)
    for (cin, cout, k, s, H, W, stem) in [(64, 128, 3, 2, 32, 40, False), (128, 64, 1, 1, 16, 20, False), (3, 32, 6, 2, 64, 96, True)]:
        m = common.Conv(cin, cout, k, s, 2 if stem else None)
        with torch.no_grad():
            m.conv.weight.copy_((torch.randn(m.conv.weight.shape, generator=g) / (cin * k * k) ** 0.5).half().float())
            m.bn.weight.copy_(1 + 0.2 * torch.randn(cout, generator=g))
            m.bn.bias.copy_(0.2 * torch.randn(cout, generator=g))
        m.bn.eps, m.bn.momentum = 1e-3, 0.03
        ref = nn.Sequential(nn.Conv2d(cin, cout, k, s, m.conv.padding, bias=False), nn.BatchNorm2d(cout, eps=1e-3, momentum=0.03), nn.SiLU())
        ref[0].weight.data.copy_(m.conv.weight.data)
        ref[1].load_state_dict(m.bn.state_dict())
        ref.train()
        x = torch.rand(2, cin, H, W, generator=g).half() if stem else torch.randn(2, cin, H, W, generator=g).half()
        xr = x.float().requires_grad_(True)
        y = ref(xr)
        dy = (0.1 * torch.randn(y.shape, generator=g)).half()
        y.backward(dy.float())
        m = m.to(cuda_device).train()
        if stem:
            xd = m.stage_image(x.to(cuda_device))
        else:
            xd = nhwc(x).to(cuda_device).requires_grad_(True)
        yd = A.conv_bn_act(m, xd, stem)
        yd.backward(nhwc(dy).to(cuda_device))
        torch.cuda.synchronize()
        e = dict(y=err(yd.permute(0, 3, 1, 2), y), dw=err(m.conv.weight.grad, ref[0].weight.grad), dg=err(m.bn.weight.grad, ref[1].weight.grad),
                 db=err(m.bn.bias.grad, ref[1].bias.grad), rm=err(m.bn.running_mean, ref[1].running_mean), rv=err(m.bn.running_var, ref[1].running_var))
        if not stem:
            e["dx"] = err(xd.grad.permute(0, 3, 1, 2), xr.grad)
        print(f"\n[conv node {cin}->{cout} k{k}s{s}{' stem' if stem else ''}] " + "  ".join(f"{k2} {v:.2e}" for k2, v in e.items()))
        assert max(e.values()) < 2.5e-3, e
        assert int(m.bn.num_batches_tracked) == 1
