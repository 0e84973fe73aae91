"""The one-tile conv kernel's epilogue on the accumulator registers with TMA-stored output tiles (and a TMA-loaded residual
tile in the ring stage after the last K block), vs the CPU oracle and the on-device CUDA-core reference: 2-D, 4-D and
gather launches at BN = 64 and 128, ragged M tails, channel-slice outputs with a residual, and the launches that keep
the staged-row epilogue (BN = 32, split-K, the row-statistics epilogue).  Every case asserts through icaf_conv2d_plan
that it runs one tile per CTA."""
import pytest
import torch

from helpers import conv_plan, err, nchw, nhwc, sm_count
from test_gpu_conv import TOL, _mk, _ref

pytestmark = pytest.mark.gpu


def _one_tile(pl):
    return pl.ctas == pl.grid_x * pl.grid_y * pl.grid_z


def _run(dev, B, Cin, H, W, Cout, k, s, p, act, resid, n_io, seed):
    """Conv of n_io problems (inputs, outputs and residuals NHWC); returns (outputs, CUDA-core outputs, oracle, plan)."""
    from icafusion_b200 import ops
    coef = torch.tensor([0.7, 1.25], device=dev)
    xs, packs, ress, refs = [], [], [], []
    for i in range(n_io):
        x, w, b = _mk(B, Cin, H, W, Cout, k, s, p, seed=seed + i)
        ref = _ref(x, w, b, s, p, act)
        xs.append(nhwc(x).to(dev))
        packs.append(ops.pack_conv_weight(w.float(), b, s, p, act, device=dev))
        if resid is not None:
            r = torch.randn(ref.shape, generator=torch.Generator().manual_seed(seed + 50 + i)).half()
            ress.append(nhwc(r).to(dev))
            ref = ref + r.float() if resid == "add" else 0.7 * r.float() + 1.25 * ref
        refs.append(ref)
    kw = dict(res=ress or None, scaled=[(coef[0:1], coef[1:2])] * n_io if resid == "scaled" else None)
    pl = conv_plan(lambda: ops.conv2d(xs, packs, **kw))
    ys = ops.conv2d(xs, packs, **kw)
    ys_simt = ops.conv2d(xs, packs, simt=True, **kw)
    torch.cuda.synchronize()
    return ys, ys_simt, refs, pl


def _check(name, ys, ys_simt, refs):
    for y, y_simt, ref in zip(ys, ys_simt, refs):
        e_tc, e_simt = err(nchw(y), ref), err(nchw(y_simt), ref)
        print(f"\n[{name}] wgmma {e_tc:.2e}  cuda-core {e_simt:.2e}")
        assert e_simt < TOL and e_tc < TOL
        assert err(y, y_simt) < TOL


CASES = {
    # name: (B, Cin, H, W, Cout, k, s, p, act, residual, problems, bn, a_mode)
    "bn64_2d_ragged_m": (3, 64, 100, 84, 64, 1, 1, 0, 1, None, 1, 64, 1),          # 25200 rows: 197 tiles, the last one ragged
    "bn64_2d_gelu_scaled_res_grouped": (3, 64, 100, 84, 64, 1, 1, 0, 2, "scaled", 2, 64, 1),
    "bn64_4d_add_res": (8, 64, 64, 80, 64, 3, 1, 1, 1, "add", 1, 64, 2),
    "bn64_4d_stride2_grouped": (8, 64, 128, 160, 64, 3, 2, 1, 1, None, 2, 64, 2),
    "bn64_4d_over_ho_none": (48, 64, 20, 20, 64, 3, 1, 1, 0, None, 1, 64, 2),     # 6 x 20 tiles, the last tile row hangs over
    "bn64_gather_cin32": (8, 32, 64, 80, 64, 3, 1, 1, 1, "add", 2, 64, 0),
    "bn32_detect_n18": (1, 128, 16, 20, 18, 1, 1, 0, 0, None, 1, 32, 1),          # staged-row epilogue
    "bn32_detect_n18_grouped": (4, 128, 32, 40, 18, 1, 1, 0, 0, None, 2, 32, 1),
}


@pytest.mark.parametrize("name", list(CASES))
def test_one_tile_epilogue(cuda_device, name):
    B, Cin, H, W, Cout, k, s, p, act, resid, n_io, bn, a_mode = CASES[name]
    ys, ys_simt, refs, pl = _run(cuda_device, B, Cin, H, W, Cout, k, s, p, act, resid, n_io, seed=80)
    assert _one_tile(pl) and pl.bn == bn and pl.a_mode == a_mode and pl.cluster == 1, (pl.bn, pl.a_mode, pl.cluster)
    _check(name, ys, ys_simt, refs)


@pytest.mark.parametrize("resid", [None, "add"])
def test_one_tile_epilogue_bn128_single_wave(cuda_device, resid):
    """BN = 128 tiles that fit in one wave stay on the one-tile kernel: N = 192 (the last n-tile stores one 64-column half),
    a ragged M tail, both problems: m-tiles x 2 n-tiles x 2 problems = the SM count."""
    mt = sm_count() // 4
    ys, ys_simt, refs, pl = _run(cuda_device, 1, 64, 1, mt * 128 - 40, 192, 1, 1, 0, 1, resid, 2, seed=90)
    assert _one_tile(pl) and pl.bn == 128 and pl.cluster == 1, (pl.bn, pl.ctas, pl.cluster)
    _check(f"bn128_single_wave_{resid}", ys, ys_simt, refs)


def test_one_tile_epilogue_split_k(cuda_device):
    """A split-K cluster launch keeps the staged rows (the leader reduces the cluster's partial tiles through DSMEM)."""
    ys, ys_simt, refs, pl = _run(cuda_device, 1, 512, 16, 20, 512, 3, 1, 1, 1, "add", 1, seed=100)
    assert _one_tile(pl) and pl.cluster > 1
    _check("split_k", ys, ys_simt, refs)


@pytest.mark.parametrize("H,W,n_io", [(512, 640, 2), (264, 264, 1)])
def test_one_tile_epilogue_stem(cuda_device, H, W, n_io):
    """The image stem (cp.async gather over the 16-channel space-to-depth frame, N = 64) at the flagship frame size and at
    an odd tile count (132 x 132 outputs: 137 tiles, the last one ragged)."""
    from icafusion_b200 import ops
    xs, packs, refs = [], [], []
    for i in range(n_io):
        x, w, b = _mk(1, 3, H, W, 64, 6, 2, 2, seed=110 + i)
        packs.append(ops.pack_stem_weight(w.float(), b, 1, device=cuda_device))
        xs.append(ops.pack_image(x.to(cuda_device), s2d=True))
        refs.append(_ref(x, w, b, 2, 2, 1))
    pl = conv_plan(lambda: ops.conv2d(xs, packs))
    assert _one_tile(pl) and pl.bn == 64 and pl.a_mode == 0 and pl.cluster == 1
    if (H, W) == (264, 264):
        assert pl.grid_x == 137
    ys = ops.conv2d(xs, packs)
    ys_simt = ops.conv2d(xs, packs, simt=True)
    torch.cuda.synchronize()
    _check(f"stem_{H}x{W}", ys, ys_simt, refs)


def test_one_tile_epilogue_channel_slice_residual(cuda_device):
    """4-D launch with a residual, output written into a channel slice of a wider buffer: the output map spans the slice's
    channels only, so its neighbours stay untouched."""
    from icafusion_b200 import ops
    B, C, H, W = 8, 64, 64, 80
    x, w, b = _mk(B, C, H, W, C, 3, 1, 1, seed=120)
    r = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(121)).half()
    wide = torch.full((B, H, W, 3 * C), 7.0, dtype=torch.float16, device=cuda_device)
    pk = ops.pack_conv_weight(w.float(), b, 1, 1, 1, device=cuda_device)
    xd, rd, y = nhwc(x).to(cuda_device), nhwc(r).to(cuda_device), wide[..., C:2 * C]
    pl = conv_plan(lambda: ops.conv2d([xd], [pk], [y], [rd]))
    assert _one_tile(pl) and pl.bn == 64 and pl.a_mode == 2
    ops.conv2d([xd], [pk], [y], [rd])
    y_simt = ops.conv2d([xd], [pk], None, [rd], simt=True)[0]
    torch.cuda.synchronize()
    assert err(nchw(y), _ref(x, w, b, 1, 1, 1) + r.float()) < TOL
    assert err(y, y_simt) < TOL
    assert bool((wide[..., :C] == 7).all()) and bool((wide[..., 2 * C:] == 7).all())


def test_one_tile_epilogue_row_statistics(cuda_device):
    """The row-statistics instantiation (XM) at BN = 64 keeps the staged rows; its output matches the CUDA-core reference."""
    from icafusion_b200 import ops
    M, K, N, n_io = 20000, 256, 64, 2
    g = torch.Generator().manual_seed(130)
    al = torch.tensor([0.8, 1.3], device=cuda_device)
    xs, rs, packs = [], [], []
    for _ in range(n_io):
        xs.append(torch.randn(M, K, generator=g).half().to(cuda_device))
        rs.append(torch.randn(M, N, generator=g).half().to(cuda_device))
        packs.append(ops.pack_linear(torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g) * 0.3,
                                     device=cuda_device))
    so = [torch.zeros(M, (N + 31) // 32, 2, device=cuda_device) for _ in range(n_io)]
    kw = dict(res=rs, scaled=[(al[0:1], al[1:2])] * n_io)
    pl = conv_plan(lambda: ops.linear(xs, packs, stats_out=so, **kw))
    assert _one_tile(pl) and pl.bn == 64
    ys = ops.linear(xs, packs, stats_out=so, **kw)
    ys_simt = ops.linear(xs, packs, simt=True, **kw)
    torch.cuda.synchronize()
    for y, y_simt in zip(ys, ys_simt):
        assert err(y, y_simt) < TOL
