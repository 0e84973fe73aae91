"""Stride-1 3x3 launches of the persistent conv kernel: one input halo per 64-channel block feeds all nine taps (wgmma RS
with A fragments read from the halo by ldmatrix).  Every case checks through its plan that it runs on the persistent
kernel with 4-D TMA tiles of the expected shape, then compares against the CPU oracle (torch fp32 conv on the same
fp16-rounded operands) and the on-device CUDA-core reference."""
import pytest
import torch
import torch.nn.functional as F

from helpers import conv_plan, err, nchw, nhwc

pytestmark = pytest.mark.gpu

TOL = 1.5e-3   # fp16 output rounding (2^-11) + fp32 accumulation-order noise, norm-wise

CASES = [
    # B, Cin, H,  W,  Cout, problems, residual, x_ld, tile (tw, th)
    (4, 128, 64, 80, 128, 1, False, 128, (16, 8)),    # yolov5l P3 geometry
    (4, 128, 64, 80, 128, 2, True, 256, (16, 8)),     # two problems, residual, input in a channel slice of a wider map
    (8, 256, 32, 40, 256, 1, False, 256, (8, 16)),    # P4
    (8, 256, 32, 40, 256, 2, True, 384, (8, 16)),     # ... grouped with residual, sliced input
    (12, 512, 16, 20, 512, 1, False, 512, (20, 6)),   # P5: the last tile row of each image hangs over the map (rows 16, 17)
    (8, 512, 16, 20, 512, 2, True, 1024, (20, 6)),    # ... grouped with residual, sliced input
    (12, 128, 29, 48, 128, 1, True, 192, (24, 5)),    # 29 rows: the bottom edge cuts the last tile row, 26 x 7 halo
]


@pytest.mark.parametrize("case", CASES)
def test_halo_path_matches_oracle(cuda_device, case):
    from icafusion_b200 import ops
    B, Cin, H, W, Cout, n, with_res, x_ld, tile = case
    g = torch.Generator().manual_seed(B * 1000 + Cin + n)
    xs, packs, ress, refs = [], [], [], []
    for i in range(n):
        x = torch.randn(B, Cin, H, W, generator=g).half()
        w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5).half()
        b = torch.randn(Cout, generator=g) * 0.5
        wide = torch.randn(B, H, W, x_ld, generator=g).half().to(cuda_device)
        wide[..., x_ld - Cin:] = nhwc(x).to(cuda_device)
        xs.append(wide[..., x_ld - Cin:])
        packs.append(ops.pack_conv_weight(w.float(), b, 1, 1, 1, device=cuda_device))
        ref = F.silu(F.conv2d(x.float(), w.float(), b, stride=1, padding=1))
        if with_res:
            r = torch.randn(B, Cout, H, W, generator=g).half()
            ress.append(nhwc(r).to(cuda_device))
            ref = ref + r.float()
        refs.append(ref)
    res = ress if with_res else None
    pl = conv_plan(lambda: ops.conv2d(xs, packs, None, res))
    assert pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z, "expected a persistent launch"
    assert pl.a_mode == 2 and (pl.tile_w, pl.tile_h) == tile and pl.halo == 0, (pl.a_mode, pl.tile_w, pl.tile_h, pl.halo)
    assert pl.stages >= 2 and pl.smem_bytes <= 227 * 1024, (pl.stages, pl.smem_bytes)
    ys = ops.conv2d(xs, packs, None, res)
    ys_simt = ops.conv2d(xs, packs, None, res, simt=True)
    torch.cuda.synchronize()
    for i in range(n):
        e_tc, e_simt = err(nchw(ys[i]), refs[i]), err(nchw(ys_simt[i]), refs[i])
        print(f"\n[halo {case} problem {i}] wgmma {e_tc:.2e}  cuda-core {e_simt:.2e}")
        assert e_simt < TOL, "CUDA-core reference kernel disagrees with the oracle"
        assert e_tc < TOL
        assert err(ys[i], ys_simt[i]) < TOL
