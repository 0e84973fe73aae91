"""The image-stem conv kernel (conv_stem_kernel): 16-channel stride-1 3x3 launches at BN = 64 gather one input halo per
tile and feed all nine taps from it (wgmma RS with A fragments read by ldmatrix).  Every case checks through its plan that
the launch runs on it (one tile per CTA, BN 64, cp.async gather, a single stage), then compares against the CPU oracle
(torch fp32 6x6 / stride-2 conv of the image) and the on-device CUDA-core reference; one case compares it element for
element with the one-tile kernel, which runs the same geometry when TMA cannot store the output."""
import pytest
import torch

from helpers import conv_plan, err, nchw
from test_gpu_conv import TOL, _mk, _ref

pytestmark = pytest.mark.gpu


def _on_stem_kernel(pl):
    return pl.ctas == pl.grid_x * pl.grid_y * pl.grid_z and pl.bn == 64 and pl.a_mode == 0 and pl.cluster == 1 and \
        pl.stages == 1


CASES = {
    # name: (B, image H, W, Cout, act, bias, problems, input channel pitch, zero images)
    "flagship_frame_grouped": (1, 512, 640, 64, 1, True, 2, 16, False),
    "odd_tile_count": (1, 264, 264, 64, 1, True, 1, 16, False),             # 132 x 132 map: 137 tiles, the last one ragged
    "image_boundary_sliced_input": (4, 260, 300, 64, 1, True, 1, 32, False),   # 130 x 150 maps: tiles span two images
    "narrow_map": (12, 100, 72, 64, 1, True, 1, 16, False),                  # 50 x 36 map: up to five runs per tile
    "n48_no_activation": (2, 256, 320, 48, 0, False, 2, 16, False),          # the training stem's epilogue, ragged N
    "zeros": (2, 256, 320, 64, 1, True, 1, 16, True),                        # output = SiLU(bias): the padding is zero
}


@pytest.mark.parametrize("name", list(CASES))
def test_stem_kernel_matches_oracle(cuda_device, name):
    from icafusion_b200 import ops
    B, H, W, Cout, act, bias, n_io, x_ld, zeros = CASES[name]
    xs, packs, refs = [], [], []
    for i in range(n_io):
        x, w, b = _mk(B, 3, H, W, Cout, 6, 2, 2, seed=140 + i, bias=bias)
        if zeros:
            x.zero_()
        packs.append(ops.pack_stem_weight(w.float(), b, act, device=cuda_device))
        s2d = ops.pack_image(x.to(cuda_device), s2d=True)
        if x_ld != 16:
            wide = torch.full((B, H // 2, W // 2, x_ld), 9.0, dtype=torch.float16, device=cuda_device)
            wide[..., x_ld - 16:] = s2d
            s2d = wide[..., x_ld - 16:]
        xs.append(s2d)
        refs.append(_ref(x, w, b, 2, 2, act))
    pl = conv_plan(lambda: ops.conv2d(xs, packs))
    assert _on_stem_kernel(pl), (pl.bn, pl.a_mode, pl.stages, pl.ctas, pl.cluster)
    if name == "odd_tile_count":
        assert pl.grid_x == 137
    ys = ops.conv2d(xs, packs)
    ys_simt = ops.conv2d(xs, packs, simt=True)
    torch.cuda.synchronize()
    for y, y_simt, ref in zip(ys, ys_simt, refs):
        e_tc, e_simt = err(nchw(y), ref), err(nchw(y_simt), ref)
        print(f"\n[stem {name}] wgmma {e_tc:.2e}  cuda-core {e_simt:.2e}")
        assert e_simt < TOL and e_tc < TOL
        assert err(y, y_simt) < TOL
        if zeros:
            assert bool((y == y[:1, :1, :1]).all())


@pytest.mark.parametrize("act,bias", [(1, True), (0, False)])
def test_stem_kernel_equals_one_tile_kernel(cuda_device, act, bias):
    """Same nine products summed in the same order as the one-tile kernel's gather path (whose three padded K steps add
    +0), and the same epilogue expression: the outputs are equal element for element.  An output whose row pitch is
    not a multiple of 8 halfs cannot be stored by TMA, so that launch runs on the one-tile kernel (staged rows)."""
    from icafusion_b200 import ops
    B, H, W, Cout = 4, 260, 300, 64
    x, w, b = _mk(B, 3, H, W, Cout, 6, 2, 2, seed=150, bias=bias)
    pk = ops.pack_stem_weight(w.float(), b, act, device=cuda_device)
    s2d = ops.pack_image(x.to(cuda_device), s2d=True)
    assert _on_stem_kernel(conv_plan(lambda: ops.conv2d([s2d], [pk])))
    y = ops.conv2d([s2d], [pk])[0]
    wide = torch.zeros(B, H // 2, W // 2, Cout + 4, dtype=torch.float16, device=cuda_device)
    ops.conv2d([s2d], [pk], [wide[..., 4:]])
    torch.cuda.synchronize()
    assert bool((y == wide[..., 4:]).all())
