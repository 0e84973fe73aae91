"""wgmma implicit-GEMM conv / linear kernel vs the CPU oracle (torch fp32 conv on the same fp16-rounded
operands) and vs the on-device CUDA-core reference.  All calls go through the C ABI."""
import pytest
import torch
import torch.nn.functional as F

from helpers import conv_plan, err, nchw, nhwc

pytestmark = pytest.mark.gpu

TOL = 1.5e-3   # fp16 output rounding (2^-11) + fp32 accumulation-order noise, norm-wise


def _mk(B, Cin, H, W, Cout, k, s, p, seed=0, bias=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g).half()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).half()
    b = torch.randn(Cout, generator=g) * 0.5 if bias else None
    return x, w, b


def _ref(x, w, b, s, p, act):
    y = F.conv2d(x.float(), w.float(), b, stride=s, padding=p)
    if act == 1:
        y = F.silu(y)
    elif act == 2:
        y = F.gelu(y)
    return y


CASES = [
    # B, Cin, H,  W,  Cout, k, s, p, act
    (1, 64, 16, 20, 64, 1, 1, 0, 1),      # 1x1, partial last M tile
    (1, 64, 16, 20, 128, 3, 1, 1, 1),     # 3x3 same
    (1, 32, 32, 40, 64, 3, 2, 1, 1),      # stride 2, Cin < 64: one K block spans two taps
    (2, 3, 64, 80, 32, 6, 2, 2, 1),       # image stem (packed NHWC4 input)
    (1, 128, 16, 20, 18, 1, 1, 0, 0),     # Detect head: N=18, no activation
    (1, 128, 64, 80, 128, 3, 1, 1, 1),    # M=5120
    (2, 64, 128, 160, 256, 1, 1, 0, 1),   # many tiles -> BN=128 path
    (1, 256, 16, 20, 256, 3, 1, 1, 1),    # deep K (36 K blocks), few tiles -> BN=32 path
    (1, 8, 9, 11, 40, 3, 1, 1, 2),        # odd sizes, Cin=8, GELU (gather path)
    (1, 32, 16, 20, 96, 1, 1, 0, 1),      # 1x1 via 2-D TMA with Cin < 64 and N not a multiple of the tile (TMA zero fill)
    (2, 64, 32, 40, 128, 3, 2, 1, 1),     # 3x3 stride 2 via 4-D TMA (traversal stride 2, negative start coordinate)
    (2, 128, 32, 40, 64, 3, 1, 1, 1),     # 3x3 stride 1 via 4-D TMA, tile 16 rows x 8 cols, two K blocks per tap
    (16, 64, 32, 40, 512, 1, 1, 0, 1),    # BN=128 tiles, one CTA per SM (128 accumulator registers per consumer thread)
    (1, 64, 16, 20, 64, 3, 1, 1, 1),      # 20-wide map: 6x20 tiles (120 of 128 MMA rows, last tile hangs over the map), split-K
    (2, 128, 16, 20, 128, 3, 2, 1, 1),    # stride 2 onto an 8x10 map: 10-wide tiles
    (1, 512, 16, 20, 512, 3, 1, 1, 1),    # P5 of yolov5l at batch 1: 72 K blocks over an 8-CTA cluster (DSMEM split-K reduction)
    (1, 2048, 1, 104, 512, 1, 1, 0, 0),   # MLP fc2 shape (rows as pixels): K=2048, split-K over clusters, 2-D TMA
    (8, 64, 64, 80, 64, 3, 1, 1, 1),      # 3x3/s1 on 64 channels, 640 4-D TMA tiles, BN=64 (two CTAs per SM)
    (8, 3, 128, 160, 32, 6, 2, 2, 1),     # 320 tiles, cp.async gather (6x6 image stem on the packed NHWC4 image), BN=32
    (4, 128, 64, 80, 256, 3, 2, 1, 1),    # 4-D TMA stride 2, BN=128, 18 K blocks per tile
    (3, 64, 100, 84, 96, 1, 1, 0, 2),     # 2-D TMA, ragged M (25200 rows) and N (96), GELU
    (8, 32, 64, 80, 64, 3, 1, 1, 1),      # 32 channels: cp.async gather, one K block spans two taps
    (8, 32, 128, 160, 64, 3, 2, 1, 1),    # ... stride 2 (yolov5s layer 1 geometry)
    (8, 16, 64, 80, 32, 3, 1, 1, 1),      # ... 16 channels, K = 144 (tail K block holds one tap)
    (1, 16, 16, 20, 32, 3, 1, 1, 1),      # 16 channels on a small grid: cp.async gather path
    (16, 256, 32, 40, 256, 3, 1, 1, 1),   # 640 BN=128 tiles on 132 SMs (ragged last wave), 36 K blocks
    (19, 1024, 32, 64, 256, 1, 1, 0, 0),  # 2-D TMA, K=1024, no activation
    (32, 128, 32, 40, 256, 3, 1, 1, 1),   # 4-D TMA (16x8 tiles), 320 M tiles
    (1, 64, 301, 128, 512, 1, 1, 0, 1),   # odd M-tile count (301)
    (99, 64, 16, 24, 256, 3, 1, 1, 1),    # 4-D TMA, 297 M tiles
    (16, 512, 16, 20, 512, 3, 1, 1, 1),   # yolov5l P5 at batch 16: 6x20 tiles, the last tile row of each image hangs over
    (4, 16, 128, 160, 64, 3, 1, 1, 1),    # image stem over the space-to-depth frame (16 channels, gather), N = 64
    (12, 16, 50, 36, 48, 3, 1, 1, 0),     # stem geometry, ragged: 36-wide map, 50 rows, N = 48, no activation
    (2, 16, 256, 320, 32, 3, 1, 1, 1),    # stem geometry at the yolov5s frame size, N = 32
]


@pytest.mark.parametrize("case", CASES)
def test_conv_matches_oracle(cuda_device, case):
    from icafusion_b200 import ops
    B, Cin, H, W, Cout, k, s, p, act = case
    x, w, b = _mk(B, Cin, H, W, Cout, k, s, p)
    pk = ops.pack_conv_weight(w.float(), b, s, p, act, device=cuda_device)
    xv = ops.pack_image(x.to(cuda_device)) if Cin == 3 else nhwc(x).to(cuda_device)
    y = ops.conv2d([xv], [pk])[0]
    y_simt = ops.conv2d([xv], [pk], simt=True)[0]
    torch.cuda.synchronize()
    ref = _ref(x, w, b, s, p, act)
    e_simt, e_tc = err(nchw(y_simt), ref), err(nchw(y), ref)
    print(f"\n[conv {case}] wgmma {e_tc:.2e}  cuda-core {e_simt:.2e}")
    assert e_simt < TOL, "CUDA-core reference kernel disagrees with the oracle"
    assert e_tc < TOL
    assert err(y, y_simt) < TOL


def test_grouped_residual_and_slices(cuda_device):
    """Two problems per launch, fused residual add, input read from / output written into channel slices."""
    from icafusion_b200 import ops
    B, C, H, W = 2, 64, 16, 20
    xs, ws, bs, refs, packs, outs, ress, xin = [], [], [], [], [], [], [], []
    for i in range(2):
        x, w, b = _mk(B, C, H, W, C, 3, 1, 1, seed=10 + i)
        wide = torch.randn(B, H, W, 2 * C).half().to(cuda_device)          # input lives in a slice of a wider buffer
        wide[..., C:] = nhwc(x).to(cuda_device)
        res = torch.randn(B, C, H, W).half()
        out_wide = torch.zeros(B, H, W, 3 * C, dtype=torch.float16, device=cuda_device)
        xin.append(wide[..., C:]); ress.append(nhwc(res).to(cuda_device)); outs.append(out_wide[..., C:2 * C])
        packs.append(ops.pack_conv_weight(w.float(), b, 1, 1, 1, device=cuda_device))
        refs.append(_ref(x, w, b, 1, 1, 1) + res.float())
        xs.append(out_wide)
    ops.conv2d(xin, packs, outs, ress)
    torch.cuda.synchronize()
    for i in range(2):
        assert err(nchw(outs[i]), refs[i]) < TOL
        assert float(xs[i][..., :C].abs().max()) == 0 and float(xs[i][..., 2 * C:].abs().max()) == 0   # neighbours untouched


def test_persistent_kernel_grouped_residual(cuda_device):
    """Wide-tile (BN = 128) launch with two problems (RGB / IR streams) and the fused Bottleneck residual: more tiles than
    SMs, so it runs on the persistent kernel."""
    from icafusion_b200 import ops
    B, C, H, W = 16, 256, 32, 40
    xs, packs, ress, refs = [], [], [], []
    for i in range(2):
        x, w, b = _mk(B, C, H, W, C, 3, 1, 1, seed=20 + i)
        res = torch.randn(B, C, H, W).half()
        xs.append(nhwc(x).to(cuda_device)); ress.append(nhwc(res).to(cuda_device))
        packs.append(ops.pack_conv_weight(w.float(), b, 1, 1, 1, device=cuda_device))
        refs.append(_ref(x, w, b, 1, 1, 1) + res.float())
    pl = conv_plan(lambda: ops.conv2d(xs, packs, None, ress))
    assert pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z, "expected a persistent launch"
    ys = ops.conv2d(xs, packs, None, ress)
    torch.cuda.synchronize()
    for i in range(2):
        assert err(nchw(ys[i]), refs[i]) < TOL


@pytest.mark.parametrize("B,H,W,Cout", [(1, 64, 80, 32), (8, 256, 320, 32), (2, 128, 160, 64)])
def test_stem_space_to_depth(cuda_device, B, H, W, Cout):
    """Image stem Conv(3, c, 6, 2, 2) run as a 3x3/s1/p1 conv over the 16-channel space-to-depth image (cp.async gather
    path) vs the plain 6x6 stride-2 convolution on the CPU."""
    from icafusion_b200 import ops
    x, w, b = _mk(B, 3, H, W, Cout, 6, 2, 2, seed=5)
    pk = ops.pack_stem_weight(w.float(), b, 1, device=cuda_device)
    assert (pk.cin, pk.kh, pk.stride, pk.pad) == (16, 3, 1, 1)
    xv = ops.pack_image(x.to(cuda_device), s2d=True)
    assert tuple(xv.shape) == (B, H // 2, W // 2, 16)
    y = ops.conv2d([xv], [pk])[0]
    torch.cuda.synchronize()
    assert err(nchw(y), _ref(x, w, b, 2, 2, 1)) < TOL


def test_one_tile_kernel_grouped_residual(cuda_device):
    """Many tiles (640) with two problems per launch, fused residual and channel-slice output: 64 output channels give
    BN = 64 tiles, so it runs on the one-tile-per-CTA kernel."""
    from icafusion_b200 import ops
    B, C, H, W = 8, 64, 64, 80
    packs, xin, ress, outs, refs = [], [], [], [], []
    for i in range(2):
        x, w, b = _mk(B, C, H, W, C, 3, 1, 1, seed=20 + i)
        res = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(30 + i)).half()
        wide = torch.zeros(B, H, W, 2 * C, dtype=torch.float16, device=cuda_device)
        xin.append(nhwc(x).to(cuda_device)); ress.append(nhwc(res).to(cuda_device)); outs.append(wide[..., C:])
        packs.append(ops.pack_conv_weight(w.float(), b, 1, 1, 1, device=cuda_device))
        refs.append(_ref(x, w, b, 1, 1, 1) + res.float())
    pl = conv_plan(lambda: ops.conv2d(xin, packs, outs, ress))
    assert pl.bn == 64 and pl.ctas == pl.grid_x * pl.grid_y * pl.grid_z, "expected a one-tile-per-CTA launch"
    ops.conv2d(xin, packs, outs, ress)
    torch.cuda.synchronize()
    for i in range(2):
        assert err(nchw(outs[i]), refs[i]) < TOL


def test_linear_epilogues(cuda_device):
    """GELU linear; scaled residual (alpha*res + beta*(xW^T+b)); swap-AB with per-row bias."""
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(3)
    rows, K, N = 208, 128, 512
    x = torch.randn(rows, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    b = torch.randn(N, generator=g)
    xd = x.to(cuda_device)
    y = ops.linear([xd], [ops.pack_linear(w.float(), b, ops.ACT_GELU, device=cuda_device)])[0]
    assert err(y, F.gelu(F.linear(x.float(), w.float(), b))) < TOL
    # scaled residual
    w2 = (torch.randn(K, N, generator=g) / N ** 0.5).half()
    b2 = torch.randn(K, generator=g)
    res = torch.randn(rows, K, generator=g).half()
    coef = torch.tensor([0.8, 1.3], device=cuda_device)
    h = torch.randn(rows, N, generator=g).half()
    y2 = ops.linear([h.to(cuda_device)], [ops.pack_linear(w2.float(), b2, device=cuda_device)], res=[res.to(cuda_device)],
                    scaled=[(coef[0:1], coef[1:2])])[0]
    assert err(y2, 0.8 * res.float() + 1.3 * F.linear(h.float(), w2.float(), b2)) < TOL
    # swap-AB: out[C, rows] = Wv . x^T + bv[:, None]
    wv = (torch.randn(K, K, generator=g) / K ** 0.5).half()
    bv = torch.randn(K, generator=g)
    tok = ops.PackedConv(xd, bv.to(cuda_device), K, rows, 1, 1, 1, 0, ops.ACT_NONE)
    vt = ops.linear([wv.to(cuda_device)], [tok], bias_row=True)[0]
    torch.cuda.synchronize()
    assert err(vt, (F.linear(x.float(), wv.float(), bv)).t()) < TOL


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm folded into the consuming linear layer (ICAF_EPI_LN_FOLD) and row statistics emitted by the producing one
# (ICAF_EPI_EMIT_STATS): the DMFF loop's LN1/LN2 (common.py:660,665,749-750) without a LayerNorm launch.
@pytest.mark.parametrize("M,K,N,n_io,act", [(400, 256, 768, 2, 0), (104, 1024, 4096, 2, 2), (6400, 256, 768, 2, 0), (6400, 256, 1024, 2, 2),
                                            (20480, 512, 1536, 1, 0), (1664, 1024, 3072, 2, 0), (77 * 8, 128, 384, 1, 2)])
def test_linear_with_folded_layernorm(cuda_device, M, K, N, n_io, act):
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(M + N)
    xs, packs, refs = [], [], []
    for _ in range(n_io):
        x = (torch.randn(M, K, generator=g) * (0.5 + torch.rand(M, 1, generator=g)) + 0.3 * torch.randn(M, 1, generator=g)).half()
        w = torch.randn(N, K, generator=g) / K ** 0.5
        b = torch.randn(N, generator=g) * 0.3
        gamma, beta = 1 + 0.2 * torch.randn(K, generator=g), 0.2 * torch.randn(K, generator=g)
        y = F.layer_norm(x.float(), (K,), gamma, beta, 1e-5) @ w.t() + b
        refs.append(F.gelu(y) if act == 2 else y)
        xs.append(x.to(cuda_device))
        packs.append(ops.pack_linear_ln(w, b, gamma, beta, 1e-5, act, device=cuda_device))
    stats = ops.row_stats(*xs) if n_io == 2 else [ops.row_stats(xs[0])]
    ys = ops.linear(xs, packs, ln_stats=list(stats))
    torch.cuda.synchronize()
    e = max(err(y, r) for y, r in zip(ys, refs))
    print(f"\n[LN-folded linear M{M} K{K} N{N} x{n_io} act{act}] {e:.2e}")
    assert e < 1e-3


@pytest.mark.parametrize("M,K,N,n_io", [(400, 256, 256, 2), (104, 4096, 1024, 2), (6400, 1024, 256, 2), (20480, 512, 512, 1), (4096, 512, 2048, 2)])
def test_scaled_residual_emits_row_statistics(cuda_device, M, K, N, n_io):
    """y = alpha*res + beta*(x W^T + b) with EMIT_STATS: the partials of every row sum to (sum y, sum y^2) of the fp16 output,
    and feeding them to an LN-folded linear reproduces LayerNorm(y) W2^T."""
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(M + K)
    al = torch.tensor([0.8, 1.3], device=cuda_device)
    xs, rs, packs, packs2, outs_ref = [], [], [], [], []
    for _ in range(n_io):
        x = torch.randn(M, K, generator=g).half()
        r = torch.randn(M, N, generator=g).half()
        w = torch.randn(N, K, generator=g) / K ** 0.5
        b = torch.randn(N, generator=g) * 0.3
        xs.append(x.to(cuda_device)); rs.append(r.to(cuda_device))
        packs.append(ops.pack_linear(w, b, device=cuda_device))
        w2 = torch.randn(64, N, generator=g) / N ** 0.5
        gamma, beta = 1 + 0.2 * torch.randn(N, generator=g), 0.2 * torch.randn(N, generator=g)
        packs2.append(ops.pack_linear_ln(w2, None, gamma, beta, 1e-5, device=cuda_device))
        outs_ref.append((0.8 * r.float() + 1.3 * (x.float() @ w.t() + b), w2, gamma, beta))
    so = [torch.full((M, (N + 31) // 32, 2), float("nan"), device=cuda_device) for _ in range(n_io)]
    ys = ops.linear(xs, packs, res=rs, scaled=[(al[0:1], al[1:2])] * n_io, stats_out=so)
    zs = ops.linear(ys, packs2, ln_stats=so)
    torch.cuda.synchronize()
    for y, st, z, (ref, w2, gamma, beta) in zip(ys, so, zs, outs_ref):
        assert err(y, ref) < 1e-3
        tot = st.sum(1).double().cpu()
        yf = y.double().cpu()
        assert torch.allclose(tot[:, 0], yf.sum(1), rtol=1e-4, atol=1e-2) and torch.allclose(tot[:, 1], (yf * yf).sum(1), rtol=1e-4, atol=1e-2)
        zr = F.layer_norm(y.float().cpu(), (N,), gamma, beta, 1e-5) @ w2.t()
        assert err(z, zr) < 1e-3


def test_full_size_linearity(cuda_device):
    """Size-independent property at a BASELINE-size layer (yolov5l P3 bottleneck, batch 16: M = 81920, K = 1152; too big for
    the CPU oracle in a test): without bias and activation the convolution is linear, conv(x1 + x2) == conv(x1) + conv(x2)
    up to the fp16 rounding of the three outputs, and conv(0) == 0 exactly."""
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(5)
    B, C, H, W = 16, 128, 64, 80
    x1 = (torch.randn(B, H, W, C, generator=g) * 0.5).half().to(cuda_device)
    x2 = (torch.randn(B, H, W, C, generator=g) * 0.5).half().to(cuda_device)
    w = torch.randn(C, C, 3, 3, generator=g) / (C * 9) ** 0.5
    pk = ops.pack_conv_weight(w, None, 1, 1, ops.ACT_NONE, device=cuda_device)
    xs = (x1.float() + x2.float()).half()
    y1, y2, ys = (ops.conv2d([t], [pk])[0].float() for t in (x1, x2, xs))
    y0 = ops.conv2d([torch.zeros_like(x1)], [pk])[0]
    torch.cuda.synchronize()
    assert float(y0.abs().max()) == 0.0
    e = float((ys - (y1 + y2)).abs().max() / ys.abs().max())
    print(f"\n[linearity M{B * H * W} K{C * 9}] {e:.2e}")
    assert e < 2e-3            # three fp16 output roundings + the fp16 rounding of x1 + x2 carried through K = 1152
