"""The persistent conv kernel's epilogue on the accumulator registers with TMA-stored output tiles (and TMA-loaded residual
tiles), vs the CPU oracle and the on-device CUDA-core reference: 2-D and 4-D output maps, stride 2, a partial last n-tile,
channel-slice outputs, both residual forms, the per-row bias, every activation and grouped problems.  Every case asserts
through icaf_conv2d_plan that it runs on the persistent kernel."""
import pytest
import torch

from helpers import conv_plan, err, nchw, nhwc
from test_gpu_conv import TOL, _mk, _ref

pytestmark = pytest.mark.gpu


def _persistent(pl):
    return pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z


CASES = {
    # name: (B, Cin, H, W, Cout, k, s, p, act, residual, problems, a_mode)
    "1x1_none": (8, 64, 32, 40, 256, 1, 1, 0, 0, None, 1, 1),
    "1x1_silu": (8, 64, 32, 40, 256, 1, 1, 0, 1, None, 1, 1),
    "1x1_gelu": (8, 64, 32, 40, 256, 1, 1, 0, 2, None, 1, 1),
    "3x3_tiles_20x6_over_Ho": (16, 64, 16, 20, 512, 3, 1, 1, 1, None, 1, 2),
    "3x3_stride2": (8, 64, 64, 80, 256, 3, 2, 1, 1, None, 1, 2),
    "1x1_N192": (8, 64, 32, 40, 192, 1, 1, 0, 1, None, 1, 1),
    "3x3_add_res": (16, 64, 16, 20, 512, 3, 1, 1, 1, "add", 1, 2),
    "1x1_add_res_grouped": (8, 64, 32, 40, 256, 1, 1, 0, 1, "add", 2, 1),
    "1x1_scaled_res_gelu": (8, 128, 32, 40, 256, 1, 1, 0, 2, "scaled", 1, 1),
    "3x3_grouped": (16, 64, 16, 20, 256, 3, 1, 1, 1, None, 2, 2),
}


@pytest.mark.parametrize("name", list(CASES))
def test_persistent_tma_epilogue(cuda_device, name):
    from icafusion_b200 import ops
    B, Cin, H, W, Cout, k, s, p, act, resid, n_io, a_mode = CASES[name]
    coef = torch.tensor([0.7, 1.25], device=cuda_device)
    xs, packs, ress, refs = [], [], [], []
    for i in range(n_io):
        x, w, b = _mk(B, Cin, H, W, Cout, k, s, p, seed=40 + i)
        ref = _ref(x, w, b, s, p, act)
        xs.append(nhwc(x).to(cuda_device))
        packs.append(ops.pack_conv_weight(w.float(), b, s, p, act, device=cuda_device))
        if resid is not None:
            r = torch.randn(ref.shape, generator=torch.Generator().manual_seed(50 + i)).half()
            ress.append(nhwc(r).to(cuda_device))
            ref = ref + r.float() if resid == "add" else 0.7 * r.float() + 1.25 * ref
        refs.append(ref)
    kw = dict(res=ress or None, scaled=[(coef[0:1], coef[1:2])] * n_io if resid == "scaled" else None)
    pl = conv_plan(lambda: ops.conv2d(xs, packs, **kw))
    assert _persistent(pl) and pl.a_mode == a_mode, f"expected a persistent launch with a_mode {a_mode}"
    ys = ops.conv2d(xs, packs, **kw)
    ys_simt = ops.conv2d(xs, packs, simt=True, **kw)
    torch.cuda.synchronize()
    for y, y_simt, ref in zip(ys, ys_simt, refs):
        e_tc, e_simt = err(nchw(y), ref), err(nchw(y_simt), ref)
        print(f"\n[{name}] wgmma {e_tc:.2e}  cuda-core {e_simt:.2e}")
        assert e_simt < TOL and e_tc < TOL
        assert err(y, y_simt) < TOL


def test_persistent_tma_epilogue_channel_slice(cuda_device):
    """Input read from and output written into channel slices of wider buffers (the concat of a C3 block): the output map
    spans the slice's channels only, so its neighbours stay untouched."""
    from icafusion_b200 import ops
    B, C, H, W = 16, 128, 32, 40
    x, w, b = _mk(B, C, H, W, C, 1, 1, 0, seed=60)
    wide_in = torch.randn(B, H, W, 2 * C, generator=torch.Generator().manual_seed(61)).half().to(cuda_device)
    wide_in[..., C:] = nhwc(x).to(cuda_device)
    out_wide = torch.zeros(B, H, W, 3 * C, dtype=torch.float16, device=cuda_device)
    pk = ops.pack_conv_weight(w.float(), b, 1, 0, 1, device=cuda_device)
    xin, y = wide_in[..., C:], out_wide[..., C:2 * C]
    assert _persistent(conv_plan(lambda: ops.conv2d([xin], [pk], [y])))
    ops.conv2d([xin], [pk], [y])
    y_simt = ops.conv2d([xin], [pk], simt=True)[0]
    torch.cuda.synchronize()
    assert err(nchw(y), _ref(x, w, b, 1, 0, 1)) < TOL
    assert err(y, y_simt) < TOL
    assert float(out_wide[..., :C].abs().max()) == 0 and float(out_wide[..., 2 * C:].abs().max()) == 0


def test_persistent_tma_epilogue_bias_row(cuda_device):
    """Swap-AB linear with a per-row bias (BIAS_ROW): out[c, t] = Wv[c] . x[t] + bv[c]."""
    import torch.nn.functional as F
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(7)
    rows, K, C = 1024, 128, 4096
    x = torch.randn(rows, K, generator=g).half()
    wv = (torch.randn(C, K, generator=g) / K ** 0.5).half()
    bv = torch.randn(C, generator=g)
    tok = ops.PackedConv(x.to(cuda_device), bv.to(cuda_device), K, rows, 1, 1, 1, 0, ops.ACT_NONE, is_weight=False)
    wd = wv.to(cuda_device)
    assert _persistent(conv_plan(lambda: ops.linear([wd], [tok], bias_row=True)))
    vt = ops.linear([wd], [tok], bias_row=True)[0]
    vt_simt = ops.linear([wd], [tok], bias_row=True, simt=True)[0]
    torch.cuda.synchronize()
    assert err(vt, F.linear(x.float(), wv.float(), bv).t()) < TOL
    assert err(vt, vt_simt) < TOL


def test_misaligned_output_pitch_takes_one_tile_kernel(cuda_device):
    """An output pitch that is not a multiple of 8 channels cannot be written by TMA (16-byte row pitch): the launch
    is eligible for the persistent kernel by its geometry but runs on the one-tile kernel (encoding the persistent
    kernel's output map for this pitch would fail the call), and the result is right."""
    from icafusion_b200 import ops
    B, C, H, W, N = 8, 64, 32, 40, 256
    x, w, b = _mk(B, C, H, W, N, 1, 1, 0, seed=70)
    out_wide = torch.zeros(B, H, W, N + 4, dtype=torch.float16, device=cuda_device)
    pk = ops.pack_conv_weight(w.float(), b, 1, 0, 1, device=cuda_device)
    xd, y = nhwc(x).to(cuda_device), out_wide[..., :N]
    assert _persistent(conv_plan(lambda: ops.conv2d([xd], [pk], [y])))
    ops.conv2d([xd], [pk], [y])
    torch.cuda.synchronize()
    assert err(nchw(y), _ref(x, w, b, 1, 0, 1)) < TOL
    assert float(out_wide[..., N:].abs().max()) == 0
