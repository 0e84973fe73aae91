"""yolov5n / yolov5m on the GPU: the cross-attention at the padded head dims 8 / 24 / 48 / 96 (forward, dropout forward, and
the head-dim-8 backward), both detectors against the reference's goldens (oracle/gen_golden_sizes.py), yolov5m at batch 16
through the CUDA graph, and one yolov5n training step."""
import math

import pytest
import torch

import dropout_mask as DM
import train_grads
from conftest import load_golden
from helpers import err, load_synth
from oracle import icaf_oracle as O
from oracle import synth
from test_gpu_attn import TOL, _oracle
from test_gpu_train_ops import _attn_ref

pytestmark = pytest.mark.gpu
TOL_MODEL = 3e-3          # as tests/test_gpu_model.py
PADDED = [8, 24, 48, 96]  # DMFF head dims of yolov5n P3 and yolov5m P3 / P4 / P5 (C / 8 heads)


@pytest.mark.parametrize("d", PADDED)
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("N", [100, 256, 400, 77])
@pytest.mark.parametrize("B", [1, 2])
def test_cross_attention_padded_head_dims(cuda_device, d, fused, N, B):
    """The wgmma kernel at the next power-of-two width with zero-filled columns vs the CPU oracle and the CUDA-core kernel."""
    from icafusion_b200 import ops
    h = 8
    C, n_pad = h * d, ops.round_up(N, 8)
    g = torch.Generator().manual_seed(d * 1000 + N + B)
    if fused:
        qkv_v, qkv_i = torch.randn(B, n_pad, 3 * C, generator=g).half(), torch.randn(B, n_pad, 3 * C, generator=g).half()
        args = [qkv_v.to(cuda_device), qkv_i.to(cuda_device), None, None]
        vt = lambda t: t[:, :, 2 * C:].permute(2, 0, 1).reshape(C, B * n_pad).contiguous()       # noqa: E731
        qk_v, qk_i, vt_v, vt_i = qkv_v[:, :, :2 * C], qkv_i[:, :, :2 * C], vt(qkv_v), vt(qkv_i)
    else:
        qk_v, qk_i = torch.randn(B, n_pad, 2 * C, generator=g).half(), torch.randn(B, n_pad, 2 * C, generator=g).half()
        vt_v, vt_i = torch.randn(C, B * n_pad, generator=g).half(), torch.randn(C, B * n_pad, generator=g).half()
        args = [t.to(cuda_device) for t in (qk_v, qk_i, vt_v, vt_i)]
    o_v, o_i = ops.cross_attention(*args, B, N, n_pad, C, h)
    s_v, s_i = ops.cross_attention(*args, B, N, n_pad, C, h, simt=True)
    torch.cuda.synchronize()
    r_v = _oracle(qk_i, qk_v, vt_v, B, N, n_pad, C, h)      # RGB output: IR queries on RGB keys/values
    r_i = _oracle(qk_v, qk_i, vt_i, B, N, n_pad, C, h)
    es, eo = max(err(s_v[:, :N], r_v), err(s_i[:, :N], r_i)), max(err(o_v[:, :N], r_v), err(o_i[:, :N], r_i))
    print(f"\n[attention d{d} {'fused' if fused else 'split'} B{B} N{N}] wgmma {eo:.2e}  cuda-core {es:.2e}  (tol {TOL:.0e})")
    assert es < TOL and eo < TOL
    if n_pad > N:
        assert float(o_v[:, N:].abs().max()) == 0 and float(o_i[:, N:].abs().max()) == 0
    if fused:
        t_v, t_i = ops.cross_attention_train(args[0], args[1], B, N, n_pad, C, h)        # dropout 0: the inference kernel
        assert torch.equal(t_v, o_v) and torch.equal(t_i, o_i)


@pytest.mark.parametrize("d", PADDED)
def test_cross_attention_dropout_padded(cuda_device, d):
    """The padded dropout kernel: the mask is read back through identity values (N = d keys, v[key, head, c] = (key == c)),
    then the dropped forward on random values is checked against the reference with that mask."""
    from icafusion_b200 import ops
    B, h, p, seed = 2, 8, 0.25, 99
    N = n_pad = d
    C = h * d
    g = torch.Generator().manual_seed(d)
    qv, qi = torch.randn(B, n_pad, 3 * C, generator=g).half(), torch.randn(B, n_pad, 3 * C, generator=g).half()
    qv[:, :, :2 * C] *= 0.3
    qi[:, :, :2 * C] *= 0.3
    eye = torch.eye(N).reshape(1, N, 1, d).expand(B, N, h, d).reshape(B, N, C).half()
    pv, pi = qv.clone(), qi.clone()
    pv[:, :, 2 * C:], pi[:, :, 2 * C:] = eye, eye
    m_v, m_i = ops.cross_attention_train(pv.to(cuda_device), pi.to(cuda_device), B, N, n_pad, C, h, p, seed)
    mask_v = (m_v.cpu().reshape(B, N, h, d).permute(0, 2, 1, 3) > 0).float()
    mask_i = (m_i.cpu().reshape(B, N, h, d).permute(0, 2, 1, 3) > 0).float()
    n = 2 * mask_v.numel()
    keep = float(torch.cat([mask_v, mask_i]).mean())
    assert abs(keep - (1 - p)) < 5 * math.sqrt(p * (1 - p) / n)
    want = DM.attn_keep_mask(seed, 0, B, h, N, p).view(2, B, h, N, N)
    assert torch.equal(mask_v.bool(), want[0]) and torch.equal(mask_i.bool(), want[1])
    out_v, out_i = ops.cross_attention_train(qv.to(cuda_device), qi.to(cuda_device), B, N, n_pad, C, h, p, seed)
    torch.cuda.synchronize()
    o_v, o_i = _attn_ref(qi.float(), qv.float(), N, C, h, mask_v, p), _attn_ref(qv.float(), qi.float(), N, C, h, mask_i, p)
    e_o = max(err(out_v, o_v), err(out_i, o_i))
    print(f"\n[attention dropout d{d} p{p}] keep {keep:.3f}  out {e_o:.2e}")
    assert e_o < 1.5e-3


@pytest.mark.parametrize("B,N", [(2, 100), (1, 400), (2, 77), (1, 256)])
def test_cross_attention_backward_head_dim_8(cuda_device, B, N):
    """yolov5n's P3 block: dq, dk, dv of both directions against autograd (fp32 on the same fp16 operands)."""
    from icafusion_b200 import ops
    C, h = 64, 8
    n_pad = ops.round_up(N, 8)
    g = torch.Generator().manual_seed(N + B)
    qv, qi = torch.randn(B, n_pad, 3 * C, generator=g).half(), torch.randn(B, n_pad, 3 * C, generator=g).half()
    dov, doi = (torch.randn(B, n_pad, C, generator=g) * 0.1).half(), (torch.randn(B, n_pad, C, generator=g) * 0.1).half()
    rv, ri = qv.float().requires_grad_(True), qi.float().requires_grad_(True)
    o_v, o_i = _attn_ref(ri, rv, N, C, h), _attn_ref(rv, ri, N, C, h)
    (o_v * dov[:, :N].float()).sum().backward(retain_graph=True)
    (o_i * doi[:, :N].float()).sum().backward()
    dev = [t.to(cuda_device) for t in (qv, qi)]
    out_v, out_i = ops.cross_attention_train(*dev, B, N, n_pad, C, h)
    dq_v, dq_i = ops.cross_attention_bwd(*dev, out_v, out_i, dov.to(cuda_device), doi.to(cuda_device), B, N, n_pad, C, h)
    torch.cuda.synchronize()
    e_o = max(err(out_v[:, :N], o_v.detach()), err(out_i[:, :N], o_i.detach()))
    e_g = max(err(dq_v[:, :N], rv.grad[:, :N]), err(dq_i[:, :N], ri.grad[:, :N]))
    print(f"\n[attention bwd d8 B{B} N{N}] out {e_o:.2e}  dqkv {e_g:.2e}")
    assert e_o < TOL and e_g < 2e-3
    if n_pad > N:
        assert float(dq_v[:, N:].abs().max()) == 0 and float(dq_i[:, N:].abs().max()) == 0


def test_standalone_attention_modules_at_new_widths(cuda_device):
    """Eval-mode CrossAttention / TransformerFusionBlock at C = 64 / 192 / 384 / 768 (head dims 8 / 24 / 48 / 96) vs the oracle."""
    from icafusion_b200 import CrossAttention, TransformerFusionBlock
    g = torch.Generator().manual_seed(2)
    for C in (64, 192, 384, 768):
        blk = TransformerFusionBlock(C, 10, 10).eval()
        sd = load_synth(blk, C, "blk.")
        rgb, ir = synth.synth_features(1, C, 16, 20, C)
        with torch.no_grad():
            out = blk.to(cuda_device)([rgb.to(cuda_device).half(), ir.to(cuda_device).half()])
            ref = O.dmff_block(rgb.half().float(), ir.half().float(), sd, "blk", 10, 10, 1, bn_eps=1e-5)
        e = err(out, ref)
        att = CrossAttention(C, C, C, 8).eval().to(cuda_device)
        r, i = torch.randn(2, 100, C, generator=g).to(cuda_device), torch.randn(2, 100, C, generator=g).to(cuda_device)
        with torch.no_grad():
            a_r, a_i = att([r, i])
        print(f"\n[DMFF block C{C} d{C // 8}] {e:.2e}")
        assert e < 2e-3
        assert tuple(a_r.shape) == (2, 100, C) and torch.isfinite(a_r).all() and torch.isfinite(a_i).all()


@pytest.mark.parametrize("name", ["yolov5n_flir_320", "yolov5m_flir_320", "yolov5m_flir_512x640"])
@pytest.mark.parametrize("fused", [False, True])
def test_model_matches_reference_golden(cuda_device, name, fused):
    """z against the reference's (stored in fp16; the fused and unfused reference differ by ~1e-6, meta 'fused_dev'); logits
    and the three head maps against the fp32 oracle, which tests/test_model_sizes_cpu.py pins to the reference's fingerprints."""
    from icafusion_b200 import Model
    from icafusion_b200.cfg import load_cfg
    m, d = load_golden(name)
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_FLIR")
    model = Model(cfg).eval()
    sd = load_synth(model, m["seed"])
    if fused:
        model.fuse()
    model = model.to(cuda_device)
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    with torch.no_grad():
        z, logits, xs = model(rgb.to(cuda_device), ir.to(cuda_device))
        _, lr, xr = O.model_forward(O.fold_bn(sd) if fused else sd, cfg, rgb, ir)
    torch.cuda.synchronize()
    ez = err(z, d["z16"].astype("float32"))
    el = err(logits, lr)
    ex = max(err(xs[j], xr[j]) for j in range(3))
    print(f"\n[{name} fused={fused}] z {ez:.2e} logits {el:.2e} x {ex:.2e}  (reference fp16 self-dev: {m.get('ref_fp16_self_dev')})")
    assert tuple(z.shape) == d["z16"].shape and len(xs) == 3
    assert ez < TOL_MODEL and el < TOL_MODEL and ex < TOL_MODEL


def test_yolov5m_b16_through_graph(cuda_device):
    """yolov5m, batch 16, 512x640 uint8 frames through GraphedDetector: pairs 0 and 15 against the fp32 CPU oracle, and the
    single-label NMS on the result returns finite rows."""
    from icafusion_b200 import Model
    from icafusion_b200.cfg import load_cfg
    from icafusion_b200.engine import GraphedDetector
    from icafusion_b200.general import non_max_suppression
    cfg = load_cfg("yolov5m_Transfusion_FLIR")
    model = Model(cfg).eval()
    sd = load_synth(model, 0)
    model = model.fuse().half().to(cuda_device)
    B = 16
    rgb, ir = synth.synth_images(B, 512, 640, 0)
    rgb_u8, ir_u8 = (rgb * 255).to(torch.uint8), (ir * 255).to(torch.uint8)
    eng = GraphedDetector(model, B, 512, 640, in_dtype=torch.uint8, device=cuda_device)
    z = eng.infer_to_host(rgb_u8.pin_memory(), ir_u8.pin_memory()).clone()
    assert tuple(z.shape) == (B, 20160, 8) and torch.isfinite(z.float()).all()
    with torch.no_grad():
        for j in (0, 15):
            a, b = rgb_u8[j:j + 1].float() / 255.0, ir_u8[j:j + 1].float() / 255.0
            zr = O.model_forward(O.fold_bn(sd), cfg, a, b)[0]
            e = err(z[j:j + 1], zr)
            print(f"\n[yolov5m b16 graph, pair {j}] z vs fp32 oracle {e:.2e}")
            assert e < TOL_MODEL
    dets = non_max_suppression(z.to(cuda_device), 0.001, 0.6)
    assert len(dets) == B
    for o in dets:
        assert o.shape[1] == 6 and torch.isfinite(o).all()
        assert bool(((o[:, 5] >= 0) & (o[:, 5] < 3)).all())
    print(f"[yolov5m b16 graph] NMS rows per image: {[int(o.shape[0]) for o in dets]}")


def test_training_step_yolov5n_320(cuda_device):
    """One yolov5n training step (P3 attention at head dim 8) against fp32 autograd through the oracle and the reference's own
    step (tests/golden/train_yolov5n_flir_320.npz), one gradient tensor at a time (tests/train_grads.py)."""
    train_grads.run_case(cuda_device, "train_yolov5n_flir_320")
