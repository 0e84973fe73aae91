"""The fused Bottleneck (icaf_bottleneck_fwd) against the two-launch path it replaces (cv1, then cv2 with the residual:
bit-identical, the MMAs and roundings are the same) and against an fp32 oracle that rounds h to fp16 as both paths do:
the flagship P2 geometry, maps whose edges cut the 4 x 32 patches, channel-slice input and output, and a large b1 on a
zero-bordered input (the 3x3 pads h with zeros, not with SiLU(b1))."""
import pytest
import torch
import torch.nn.functional as F

from helpers import conv_plan, err, nchw, nhwc
from test_gpu_conv import TOL

pytestmark = pytest.mark.gpu


def _problem(dev, B, H, W, seed, b1_shift=0.0, zero_border=False):
    from icafusion_b200 import ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 64, H, W, generator=g).half()
    if zero_border:
        x[:, :, 0], x[:, :, -1], x[:, :, :, 0], x[:, :, :, -1] = 0, 0, 0, 0
    w1 = (torch.randn(64, 64, 1, 1, generator=g) / 8).half()
    b1 = torch.randn(64, generator=g) * 0.5 + b1_shift
    w3 = (torch.randn(64, 64, 3, 3, generator=g) / 24).half()
    b2 = torch.randn(64, generator=g) * 0.5
    p1 = ops.pack_conv_weight(w1.float(), b1, 1, 0, ops.ACT_SILU, device=dev)
    p3 = ops.pack_conv_weight(w3.float(), b2, 1, 1, ops.ACT_SILU, device=dev)
    xd = x.to(dev)
    h = F.silu(F.conv2d(xd.float(), w1.to(dev).float(), b1.to(dev))).half().float()
    ref = F.silu(F.conv2d(h, w3.to(dev).float(), b2.to(dev), padding=1)) + xd.float()
    return nhwc(xd), p1, p3, ref


def _two_launch(xs, p1s, p3s):
    from icafusion_b200 import ops
    hs = ops.conv2d(xs, p1s)
    return ops.conv2d(hs, p3s, res=xs)


def _check(name, ys, xs, p1s, p3s, refs):
    from icafusion_b200 import ops
    y2 = _two_launch(xs, p1s, p3s)
    # a small map's cv2 splits K over a cluster, which sums in another order: equal within the tolerance only
    exact = conv_plan(lambda: ops.conv2d(y2, p3s, res=xs)).splits == 1
    torch.cuda.synchronize()
    for y, yt, ref in zip(ys, y2, refs):
        e = err(nchw(y), ref)
        print(f"\n[{name}] fused vs oracle {e:.2e}, identical to the two-launch path: {torch.equal(y, yt)}")
        assert e < TOL
        assert torch.equal(y, yt) if exact else err(y, yt) < TOL


@pytest.fixture(autouse=True)
def _fp32_oracle():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("B,H,W,n_io", [(16, 128, 160, 2), (3, 37, 45, 1), (3, 37, 45, 2), (2, 5, 33, 1)])
def test_fused_bottleneck(cuda_device, B, H, W, n_io):
    from icafusion_b200 import ops
    probs = [_problem(cuda_device, B, H, W, seed=10 + i) for i in range(n_io)]
    xs, p1s, p3s, refs = (list(t) for t in zip(*probs))
    ys = ops.bottleneck(xs, p1s, p3s)
    _check(f"{B}x64x{H}x{W} x{n_io}", ys, xs, p1s, p3s, refs)


def test_fused_bottleneck_channel_slices(cuda_device):
    """Input and output are 64-channel slices of 128-channel buffers (x_ld = y_ld = 128, as C3.run passes them); the
    output's neighbouring channels stay untouched."""
    from icafusion_b200 import ops
    B, H, W = 4, 40, 96
    xs, wides, ys, p1s, p3s, refs = [], [], [], [], [], []
    for i in range(2):
        x, p1, p3, ref = _problem(cuda_device, B, H, W, seed=30 + i)
        src = torch.randn(B, H, W, 128, dtype=torch.float16, device=cuda_device)
        src[..., 64:] = x
        wide = torch.full((B, H, W, 128), 7.0, dtype=torch.float16, device=cuda_device)
        xs.append(src[..., 64:])
        wides.append(wide)
        ys.append(wide[..., :64])
        p1s.append(p1)
        p3s.append(p3)
        refs.append(ref)
    ops.bottleneck(xs, p1s, p3s, ys)
    _check("channel slices", ys, xs, p1s, p3s, refs)
    for wide in wides:
        assert bool((wide[..., 64:] == 7).all())


def test_fused_bottleneck_pads_the_hidden_map_with_zeros(cuda_device):
    """b1 = 4 + noise: SiLU(b1) is far from zero, so a halo pixel outside the image that were not zeroed would shift every
    border output; the zero border of x makes that shift the only difference at the edges."""
    from icafusion_b200 import ops
    x, p1, p3, ref = _problem(cuda_device, 2, 36, 70, seed=50, b1_shift=4.0, zero_border=True)
    ys = ops.bottleneck([x], [p1], [p3])
    _check("large b1", ys, [x], [p1], [p3], [ref])


def test_c3_runs_its_bottlenecks_fused(cuda_device):
    """C3 with n = 3 at 64 hidden channels: the fused launches (scratch maps in between, the last one writes the left half
    of the concat buffer) give the result of the two-launch path, bit for bit."""
    from icafusion_b200 import common, ops
    torch.manual_seed(0)
    m = common.C3(128, 128, n=3).eval()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.uniform_(-0.2, 0.2)
            mod.running_var.uniform_(0.5, 1.5)
    m = m.to(cuda_device)
    x = torch.randn(2, 128, 128, 160, device=cuda_device).half().permute(0, 2, 3, 1).contiguous()
    with torch.no_grad(), ops.dry_run() as dr:
        common.C3.run([m, m], [x, x])
    assert sum(n == "icaf_bottleneck_fwd" for n, _, _ in dr.records) == 3
    with torch.no_grad():
        y = common.C3.run([m, m], [x, x])[0]
        orig = common.Bottleneck.fusable
        try:
            common.Bottleneck.fusable = staticmethod(lambda mods, xs, outs=None: False)
            y2 = common.C3.run([m, m], [x, x])[0]
        finally:
            common.Bottleneck.fusable = orig
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
