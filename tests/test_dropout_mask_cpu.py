"""The host restatement of the dropout masks (tests/dropout_mask.py) is the kernels' own function: dropout_hash and attn_keep
cut out of csrc/ptx.cuh and the element-wise dropout step cut out of csrc/train.cu, compiled as host C++ with g++ (the host
compiler nvcc uses), against the restatement on grids that reach every term of the hash."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dropout_mask as DM
from conftest import ROOT

CSRC = os.path.join(ROOT, "icafusion_b200", "csrc")


def _cut(path: str, pattern: str) -> str:
    src = open(os.path.join(CSRC, path)).read()
    m = re.search(pattern, src, re.S)
    assert m, f"{pattern!r} not found in {path}"
    return m.group(0)


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    """The source's functions as a host library: hash_n, attn_keep_n and eltwise_dropout_n loop over arrays."""
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("g++ not found")
    fns = [_cut("ptx.cuh", r"__device__ __forceinline__ uint32_t dropout_hash\(.*?\n}\n"),
           _cut("ptx.cuh", r"__device__ __forceinline__ bool attn_keep\(.*?\n}\n")]
    fns = [f.replace("__device__ __forceinline__", "static inline") for f in fns]
    # the MODE == 2 branch of eltwise_kernel: element index, seed (+ device-side offset), keep test and scale
    body = _cut("train.cu", r"if \(MODE == 2\) \{\n(.*?)\n    \}\n")
    body = re.match(r"if \(MODE == 2\) \{\n(.*)\n    \}\n", body, re.S).group(1)
    assert "dropout_hash(" in body and "idx" in body, body
    src = "#include <cstdint>\n#define __ldg(p) (*(p))\n" + "".join(fns) + """
extern "C" void hash_n(const uint32_t* a, const uint32_t* b, const uint32_t* c, uint32_t* out, long n) {
  for (long t = 0; t < n; ++t) out[t] = dropout_hash(a[t], b[t], c[t]);
}
extern "C" void attn_keep_n(const uint32_t* seed, const int* dir, const int* bh, const int* q, const int* k, float p, uint8_t* out, long n) {
  for (long t = 0; t < n; ++t) out[t] = attn_keep(seed[t], dir[t], bh[t], q[t], k[t], p);
}
extern "C" void eltwise_dropout_n(const long long* index, const float* x, uint32_t seed, const uint32_t* seed_off, float p, float* out, long n) {
  for (long t = 0; t < n; ++t) {
    const long long i = index[t] / 8;
    const int e = int(index[t] % 8);
    float xv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    xv[e] = x[t];
""" + body + """
    out[t] = xv[e];
  }
}
"""
    d = tmp_path_factory.mktemp("dropout_host")
    cpp, so = d / "dropout.cpp", d / "dropout.so"
    cpp.write_text(src)
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(so), str(cpp)])
    L = ctypes.CDLL(str(so))
    L.attn_keep_n.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_float, ctypes.c_void_p, ctypes.c_long]
    L.eltwise_dropout_n.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_float,
                                    ctypes.c_void_p, ctypes.c_long]
    L.hash_n.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_long]
    return L


def _p(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def _host_keep(L, seed, dir, bh, q, k, p):
    seed, dir, bh, q, k = (np.ascontiguousarray(v) for v in np.broadcast_arrays(
        np.asarray(seed, np.uint32), np.asarray(dir, np.int32), np.asarray(bh, np.int32), np.asarray(q, np.int32), np.asarray(k, np.int32)))
    out = np.zeros(seed.shape, np.uint8)
    L.attn_keep_n(_p(seed), _p(dir), _p(bh), _p(q), _p(k), p, _p(out), out.size)
    return torch.from_numpy(out.astype(bool))


# seed + offset pairs: plain, and sums that wrap past 2^32
SEEDS = [(0x1234567, 0), (0xFFFFFFF0, 0x25), (0x80000001, 0xFFFFFFFF), (3020855033, 0x7FFFFFFF)]


def test_hash_is_the_sources(host):
    rng = np.random.default_rng(1)
    a, b, c = (np.concatenate([np.array([0, 1, 0xFFFFFFFF, 0x80000000], np.uint32), rng.integers(0, 2 ** 32, 4096, dtype=np.uint32)])
               for _ in range(3))
    out = np.zeros_like(a)
    host.hash_n(_p(a), _p(b), _p(c), _p(out), out.size)
    got = DM.dropout_hash(torch.from_numpy(a.astype(np.int64)), torch.from_numpy(b.astype(np.int64)), torch.from_numpy(c.astype(np.int64)))
    assert torch.equal(got, torch.from_numpy(out.astype(np.int64)))


@pytest.mark.parametrize("p", [0.0, 0.1, 0.25, 0.5])
@pytest.mark.parametrize("seed,offset", SEEDS)
def test_attention_mask_is_the_sources(host, seed, offset, p):
    """A query x key grid with keys past 65536 (the k >> 16 term), several batch * head rows and both directions."""
    q = np.concatenate([np.arange(0, 130), [255, 256, 399, 4095, 65535]]).astype(np.int64)
    k = np.concatenate([np.arange(0, 130), [399, 65535, 65536, 65537, 131071, 131072, 200000]]).astype(np.int64)
    s = (seed + offset) & DM.M32
    for dir in (0, 1):
        for bh in (0, 1, 7, 47, 127):
            want = _host_keep(host, s, dir, bh, q[:, None], k[None, :], p)
            got = DM.attn_keep(s, dir, bh, torch.from_numpy(q)[:, None], torch.from_numpy(k)[None, :], p)
            assert torch.equal(got, want), (dir, bh, int((got != want).sum()))
    # the mask builder: (dir, b * heads + head, q, k) at seed + offset
    B, heads, N = 2, 3, 70
    m = DM.attn_keep_mask(seed, offset, B, heads, N, p)
    r = np.arange(N)
    want = _host_keep(host, s, np.arange(2)[:, None, None, None], np.arange(B * heads)[None, :, None, None], r[None, None, :, None],
                      r[None, None, None, :], p)
    assert m.shape == (2, B * heads, N, N) and torch.equal(m, want)
    if p == 0.0:
        assert bool(m.all())
    else:
        assert abs(float(m.float().mean()) - (1 - p)) < 0.02


def test_keep_threshold_is_inclusive(host):
    """p exactly at one hash's threshold: (h >> 8) * 2^-24 == p keeps (>=), one fp32 step above drops."""
    h = int(DM.dropout_hash(torch.tensor(5 * 65536 + 9), torch.tensor(2 * 3 + 1), torch.tensor(0xABCDEF)))
    p = (h >> 8) * 2.0 ** -24
    assert p == DM.f32(p) and 0 < p < 1
    above = float(np.nextafter(np.float32(p), np.float32(1)))
    for pp, kept in ((p, True), (above, False)):
        assert bool(_host_keep(host, 0xABCDEF, 1, 3, 5, 9, pp)[()]) is kept
        assert bool(DM.attn_keep(0xABCDEF, 1, 3, 5, 9, pp)) is kept


@pytest.mark.parametrize("p", [0.1, 0.25, 0.5])
@pytest.mark.parametrize("seed,offset", SEEDS)
def test_eltwise_dropout_is_the_sources(host, seed, offset, p):
    """Element indices from 0 through 2^32 and past it (the idx >> 32 term), with the offset read through the seed_off
    pointer as the kernel reads it; kept values scaled by 1 / (1 - p) in fp32."""
    firsts = [0, 12345 * 8, 2 ** 32 - 64, 2 ** 32, 3 * 2 ** 32 + 8, 2 ** 40]
    rng = np.random.default_rng(2)
    for first in firsts:
        n = 512
        idx = np.arange(first, first + n, dtype=np.int64)
        x = rng.standard_normal(n).astype(np.float16).astype(np.float32)
        off = np.array([offset], np.uint32)
        out = np.full(n, np.nan, np.float32)
        host.eltwise_dropout_n(_p(idx), _p(x), seed, _p(off), p, _p(out), n)
        km = DM.eltwise_keep(n, seed, offset, p, first=first)
        assert torch.equal(km, torch.from_numpy(out != 0)), first
        want = DM.eltwise_dropout(torch.from_numpy(x).half(), km, p)
        assert torch.equal(torch.from_numpy(out).half().view(torch.int16), want.view(torch.int16)), first
