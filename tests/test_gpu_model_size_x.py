"""yolov5x on the GPU: the exact-width cross-attention at head dim 160 (yolov5x's P5 block), the detector against the
reference's goldens (oracle/gen_golden_sizes_x.py), and yolov5x at batch 16 through the CUDA graph."""
import pytest
import torch

from conftest import load_golden
from helpers import err, load_synth
from oracle import icaf_oracle as O
from oracle import synth
from test_gpu_attn import TOL, _oracle

pytestmark = pytest.mark.gpu
TOL_MODEL = 3e-3          # as tests/test_gpu_model.py


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("N", [100, 77, 256, 400])
@pytest.mark.parametrize("B", [1, 2])
def test_cross_attention_head_dim_160(cuda_device, fused, N, B):
    """The D = 160 wgmma kernel (five 32-column boxes, N = 160 PV) against fp32 torch on the same fp16 operands; pad rows
    are zero."""
    from icafusion_b200 import ops
    d, h = 160, 8
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
    torch.cuda.synchronize()
    r_v = _oracle(qk_i, qk_v, vt_v, B, N, n_pad, C, h)      # RGB output: IR queries on RGB keys/values
    r_i = _oracle(qk_v, qk_i, vt_i, B, N, n_pad, C, h)
    eo = max(err(o_v[:, :N], r_v), err(o_i[:, :N], r_i))
    print(f"\n[attention d160 {'fused' if fused else 'split'} B{B} N{N}] wgmma {eo:.2e}  (tol {TOL:.0e})")
    assert eo < TOL
    if n_pad > N:
        assert float(o_v[:, N:].abs().max()) == 0 and float(o_i[:, N:].abs().max()) == 0


def test_standalone_attention_modules_at_head_dim_160(cuda_device):
    """Eval-mode TransformerFusionBlock at C = 1280 (yolov5x's P5 block, 10 x 10 tokens) against the oracle."""
    from icafusion_b200 import TransformerFusionBlock
    C = 1280
    blk = TransformerFusionBlock(C, 10, 10).eval()
    sd = load_synth(blk, C, "blk.")
    rgb, ir = synth.synth_features(1, C, 16, 20, C)
    with torch.no_grad():
        out = blk.to(cuda_device)([rgb.to(cuda_device).half(), ir.to(cuda_device).half()])
        ref = O.dmff_block(rgb.half().float(), ir.half().float(), sd, "blk", 10, 10, 1, bn_eps=1e-5)
    e = err(out, ref)
    print(f"\n[DMFF block C{C} d160] {e:.2e}")
    assert e < 2e-3


@pytest.mark.parametrize("name", ["yolov5x_flir_320", "yolov5x_flir_512x640"])
@pytest.mark.parametrize("fused", [False, True])
def test_yolov5x_matches_reference_golden(cuda_device, name, fused):
    """z against the reference's (stored in fp16); logits and the three head maps against the fp32 oracle, which
    tests/test_model_size_x_cpu.py pins to the reference's fingerprints."""
    from icafusion_b200 import Model
    from icafusion_b200.cfg import load_cfg
    m, d = load_golden(name)
    cfg = load_cfg("yolov5x_Transfusion_FLIR")
    model = Model("yolov5x_Transfusion_FLIR").eval()
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


def test_yolov5x_b16_through_graph(cuda_device):
    """yolov5x, batch 16, 512x640 uint8 frames through GraphedDetector: exactly the eager forward of the same model and
    batch, and pairs 0 and 15 against the fp32 CPU oracle."""
    from icafusion_b200 import Model
    from icafusion_b200.cfg import load_cfg
    from icafusion_b200.engine import GraphedDetector
    cfg = load_cfg("yolov5x_Transfusion_FLIR")
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
        z_eager = model(rgb_u8.to(cuda_device), ir_u8.to(cuda_device))[0].cpu()
        print(f"\n[yolov5x b16 graph] vs the eager forward {err(z, z_eager):.2e}")
        assert torch.equal(z, z_eager)
        for j in (0, 15):
            a, b = rgb_u8[j:j + 1].float() / 255.0, ir_u8[j:j + 1].float() / 255.0
            zr = O.model_forward(O.fold_bn(sd), cfg, a, b)[0]
            e = err(z[j:j + 1], zr)
            print(f"[yolov5x b16 graph, pair {j}] z vs fp32 oracle {e:.2e}")
            assert e < TOL_MODEL
