"""Dropout masks read back from the device and compared with the host restatement (tests/dropout_mask.py) for equality: the
attention forward and the backward's key/value kernel at every (N, head dim) pair training issues, and the device-side seed
offset that gives each CUDA-graph replay new masks.

Read-back: with the q columns of both projections zero, every score is 0 and every unnormalised probability is exactly 1, so
the dropped probability of (query i, key j) is keep / (N (1 - p)), non-zero exactly when kept.  One-hot values
v[key, head, c] = (key == blk d + c) bring keys blk d .. blk d + d - 1 out to the forward's channels; one-hot output gradients
dO[query, head, c] = (query == blk d + c) bring queries blk d .. out to the backward's dv rows (dv = Pd^T dO)."""
import pytest
import torch

import dropout_mask as DM

pytestmark = pytest.mark.gpu

B, HEADS, P = 3, 8, 0.1
# (N, n_pad, head dim) of training's dropout launches (640x640 and 512x640 batches): every pair, at a ragged batch of 3
GEOMS = [(100, 104, 32), (100, 104, 64), (100, 104, 128), (256, 256, 16), (256, 256, 32), (256, 256, 64),
         (400, 400, 8), (400, 400, 16), (400, 400, 32)]
ATTN_QT, ATTN_KV = 128, 64          # forward kernel: queries per CTA, keys per tile (for the failure report)


def _qkv(N, n_pad, d, seed):
    """Both [q|k|v] projections with zero q columns and random k columns."""
    C = HEADS * d
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for _ in range(2):
        t = torch.zeros(B, n_pad, 3 * C, dtype=torch.float16, device="cuda")
        t[:, :N, C:2 * C] = torch.randn(B, N, C, generator=g, device="cuda").half()
        out.append(t)
    return out


def _one_hot(t, N, d, blk):
    """t (B, n_pad, HEADS * d): row blk d + c of every head gets a 1 in channel c; returns the rows covered."""
    t.zero_()
    rows = min(d, N - blk * d)
    r = torch.arange(rows, device="cuda")
    t.view(B, -1, HEADS, d)[:, blk * d + r, :, r] = 1.0
    return rows


def forward_mask(N, n_pad, d, p, seed):
    """The forward's keep mask, bool (2, B * HEADS, N queries, N keys)."""
    from icafusion_b200 import ops
    C = HEADS * d
    qv, qi = _qkv(N, n_pad, d, seed)
    mask = torch.zeros(2, B * HEADS, N, N, dtype=torch.bool, device="cuda")
    for blk in range((N + d - 1) // d):
        for t in (qv, qi):
            rows = _one_hot(t[..., 2 * C:], N, d, blk)
        outs = ops.cross_attention_train(qv, qi, B, N, n_pad, C, HEADS, p, seed)
        for dir, o in enumerate(outs):          # o[b, q, head, c] -> mask[dir, b * HEADS + head, q, blk d + c]
            m = o[:, :N].reshape(B, N, HEADS, d)[..., :rows] != 0
            mask[dir, :, :, blk * d:blk * d + rows] = m.permute(0, 2, 1, 3).reshape(B * HEADS, N, rows)
    return mask


def kv_mask(N, n_pad, d, p, seed):
    """The backward key/value kernel's keep mask, bool (2, B * HEADS, N queries, N keys), from its dv."""
    from icafusion_b200 import ops
    C = HEADS * d
    qv, qi = _qkv(N, n_pad, d, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    for t in (qv, qi):
        t[:, :N, 2 * C:] = torch.randn(B, N, C, generator=g, device="cuda").half()
    o_v, o_i = ops.cross_attention_train(qv, qi, B, N, n_pad, C, HEADS, p, seed)
    dov, doi = torch.zeros_like(o_v), torch.zeros_like(o_i)
    mask = torch.zeros(2, B * HEADS, N, N, dtype=torch.bool, device="cuda")
    for blk in range((N + d - 1) // d):
        for t in (dov, doi):
            rows = _one_hot(t, N, d, blk)
        dq = ops.cross_attention_bwd(qv, qi, o_v, o_i, dov, doi, B, N, n_pad, C, HEADS, p, seed)
        for dir, t in enumerate(dq):            # dv[b, key, head, c] -> mask[dir, b * HEADS + head, blk d + c, key]
            dv = t[:, :N, 2 * C:].reshape(B, N, HEADS, d)[..., :rows] != 0
            mask[dir, :, blk * d:blk * d + rows, :] = dv.permute(0, 2, 3, 1).reshape(B * HEADS, rows, N)
    return mask


def assert_masks_equal(got, want, what):
    bad = (got != want).nonzero()
    if len(bad):
        lines = [f"dir {int(r[0])} bh {int(r[1])} query {int(r[2])} (tile {int(r[2]) // ATTN_QT}) key {int(r[3])} "
                 f"(tile {int(r[3]) // ATTN_KV}): device {bool(got[tuple(r)])}" for r in bad[:12]]
        dirs = sorted({int(r[0]) for r in bad})
        pytest.fail(f"{what}: {len(bad)} of {got.numel()} mask bits differ (directions {dirs}):\n" + "\n".join(lines), pytrace=False)


@pytest.mark.parametrize("N,n_pad,d", GEOMS, ids=[f"N{n}-d{d}" for n, _, d in GEOMS])
def test_forward_mask(cuda_device, N, n_pad, d):
    seed = 0x9E3779B9 ^ (N * 131 + d)
    got = forward_mask(N, n_pad, d, P, seed)
    want = DM.attn_keep_mask(seed, 0, B, HEADS, N, P, "cuda")
    keep = float(got.float().mean())
    print(f"\n[dropout forward N{N} d{d}] keep {keep:.4f}")
    assert_masks_equal(got, want, f"forward N{N} d{d}")


@pytest.mark.parametrize("N,n_pad,d", GEOMS, ids=[f"N{n}-d{d}" for n, _, d in GEOMS])
def test_backward_kv_mask(cuda_device, N, n_pad, d):
    seed = 0x85EBCA77 ^ (N * 131 + d)
    assert_masks_equal(kv_mask(N, n_pad, d, P, seed), DM.attn_keep_mask(seed, 0, B, HEADS, N, P, "cuda"), f"backward kv N{N} d{d}")


@pytest.fixture
def seed_offset(cuda_device):
    """A device int32 counter as the library's seed offset; the process-global pointer is cleared again on exit."""
    from icafusion_b200 import _lib
    ctr = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    _lib.check(_lib.lib().icaf_set_seed_offset(ctr.data_ptr()), "icaf_set_seed_offset")
    try:
        yield ctr
    finally:
        torch.cuda.synchronize()
        _lib.lib().icaf_set_seed_offset(None)


def _set(ctr, t: int):
    ctr.fill_(t - 2 ** 32 if t >= 2 ** 31 else t)          # the kernels read the counter as uint32


# one key block covers every key, so one launch reads a whole mask back
ONE_BLOCK = (100, 104, 128)
ELT_N = 65536 + 8


@pytest.mark.parametrize("seed,t", [(0x1234567, 5), (0xFFFFFFF0, 0x25), (0x70000123, 0x90000000)])
def test_seed_offset_eager(seed_offset, seed, t):
    """Forward, backward and element-wise dropout draw their masks at seed + offset (mod 2^32)."""
    from icafusion_b200 import ops
    N, n_pad, d = ONE_BLOCK
    _set(seed_offset, t)
    want = DM.attn_keep_mask(seed, t, B, HEADS, N, P, "cuda")
    assert_masks_equal(forward_mask(N, n_pad, d, P, seed), want, f"forward at offset {t:#x}")
    assert_masks_equal(kv_mask(N, n_pad, d, P, seed), want, f"backward kv at offset {t:#x}")
    x = torch.randn(ELT_N, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda").half()
    y = ops.eltwise(2, x, p=P, seed=seed)
    assert torch.equal(y.view(torch.int16), DM.eltwise_dropout(x, DM.eltwise_keep(ELT_N, seed, t, P, "cuda"), P).view(torch.int16))
    assert not torch.equal(want, DM.attn_keep_mask(seed, 0, B, HEADS, N, P, "cuda"))


@pytest.mark.parametrize("N,n_pad,d", [ONE_BLOCK, (256, 256, 64), (400, 400, 8)], ids=["N100-d128", "N256-d64", "N400-d8"])
def test_seed_offset_reaches_every_kernel(seed_offset, N, n_pad, d):
    """Forward and backward values at (seed, offset t) are bit for bit those at (seed + t, offset 0): every kernel of the
    call, the backward's query kernel included, adds the offset (the census checks the values at offset 0)."""
    from icafusion_b200 import ops
    C = HEADS * d
    g = torch.Generator(device="cuda").manual_seed(N + d)
    qv, qi = (torch.randn(B, n_pad, 3 * C, generator=g, device="cuda").half() for _ in range(2))
    dov, doi = (0.1 * torch.randn(B, n_pad, C, generator=g, device="cuda")).half(), (0.1 * torch.randn(B, n_pad, C, generator=g, device="cuda")).half()
    runs = []
    for s, t in ((0xFFFFFF00, 0x345), ((0xFFFFFF00 + 0x345) & DM.M32, 0)):
        _set(seed_offset, t)
        o_v, o_i = ops.cross_attention_train(qv, qi, B, N, n_pad, C, HEADS, P, s)
        runs.append((o_v, o_i) + ops.cross_attention_bwd(qv, qi, o_v, o_i, dov, doi, B, N, n_pad, C, HEADS, P, s))
    torch.cuda.synchronize()
    for what, a, b in zip(("out_vis", "out_ir", "dqkv_vis", "dqkv_ir"), *runs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), what


def test_seed_offset_graph_replays(seed_offset):
    """ctr += 1; attention forward; element-wise dropout -- captured once: replay r draws the masks at seed + r."""
    from icafusion_b200 import ops
    N, n_pad, d = ONE_BLOCK
    C = HEADS * d
    seed = 0xDEADBEEF
    qv, qi = _qkv(N, n_pad, d, 7)
    for t in (qv, qi):
        _one_hot(t[..., 2 * C:], N, d, 0)
    x = torch.randn(ELT_N, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda").half()

    def body():
        seed_offset.add_(1)
        o_v, o_i = ops.cross_attention_train(qv, qi, B, N, n_pad, C, HEADS, P, seed)
        return o_v, o_i, ops.eltwise(2, x, p=P, seed=seed)
    body()                                              # first launches configure the kernels outside the capture
    torch.cuda.synchronize()
    seed_offset.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = body()
    for r in (1, 2):
        graph.replay()
        torch.cuda.synchronize()
        assert int(seed_offset) == r
        mask = torch.stack([o[:, :N].reshape(B, N, HEADS, d).permute(0, 2, 1, 3).reshape(B * HEADS, N, d)[..., :N] != 0 for o in outs[:2]])
        assert_masks_equal(mask, DM.attn_keep_mask(seed, r, B, HEADS, N, P, "cuda"), f"graph replay {r}")
        want = DM.eltwise_dropout(x, DM.eltwise_keep(ELT_N, seed, r, P, "cuda"), P)
        assert torch.equal(outs[2].view(torch.int16), want.view(torch.int16)), f"element-wise dropout, graph replay {r}"
