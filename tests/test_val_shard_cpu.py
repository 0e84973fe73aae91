"""Sharded validation without a GPU: the exchange-buffer layout of icaf_val_pack / icaf_val_merge restated in numpy on
ragged inputs, the entry points' host-side refusals and pure size queries, batch ownership over the ranks, the dry-run
record of the pack and merge launches, and a spill-free ptxas report."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from test_conv_ptxas_cpu import _nvcc

NIOU = 10


# ---------------------------------------------------------------------------------------------- numpy restatement
def pack_reference(batches, niou, native, positions=None):
    """icaf_val_pack in numpy.  batches: [(det (B, max_det, 6), count (B,), correct (B, max_det, niou), native or None, image0)]."""
    rw = 3 + 4 * native
    heads, rows, first, k = [], [], 0, 0
    for det, count, correct, nat, image0 in batches:
        for b in range(det.shape[0]):
            c = int(min(max(count[b], 0), det.shape[1]))
            heads.append([image0 + b, c, first, -1 if positions is None else positions[k]])
            for i in range(c):
                bits = int(sum(1 << j for j in range(niou) if correct[b, i, j]))
                r = [det[b, i, 4:5].view(np.int32)[0], det[b, i, 5:6].view(np.int32)[0], np.uint32(bits).view(np.int32)]
                if native:
                    r += list(nat[b, i].view(np.int32))
                rows.append(r)
            first += c
            k += 1
    n = len(heads)
    head = [n, first, rw, 4 + 4 * n + first * rw]
    body = np.array(heads, np.int32).reshape(-1)
    return np.concatenate([np.array(head, np.int32), body, np.array(rows, np.int32).reshape(-1)])


def merge_reference(bufs, n_images, niou, native):
    """icaf_val_merge in numpy: the flat arrays in global image order; refuses missing and duplicated images."""
    rw = 3 + 4 * native
    where = {}
    for b, buf in enumerate(bufs):
        n = int(buf[0])
        assert buf[2] == rw and buf[3] == 4 + 4 * n + buf[1] * rw
        for e in range(n):
            img = int(buf[4 + 4 * e])
            if img in where:
                raise ValueError(f"image {img} in more than one buffer")
            where[img] = (b, e)
    missing = sorted(set(range(n_images)) - set(where))
    if missing:
        raise ValueError(f"images {missing} missing from every buffer")
    counts, offsets, correct, conf, pcls, nat = [], [0], [], [], [], []
    for img in range(n_images):
        b, e = where[img]
        buf = bufs[b]
        _, c, first, _ = buf[4 + 4 * e:8 + 4 * e]
        base = 4 + 4 * int(buf[0]) + first * rw
        r = buf[base:base + c * rw].reshape(c, rw)
        counts.append(c)
        offsets.append(offsets[-1] + c)
        conf.append(r[:, 0].view(np.float32))
        pcls.append(r[:, 1].view(np.float32))
        correct.append(((r[:, 2:3].view(np.uint32) >> np.arange(niou, dtype=np.uint32)) & 1).astype(np.uint8))
        if native:
            nat.append(r[:, 3:7].view(np.float32))
    out = dict(counts=np.array(counts, np.int32), offsets=np.array(offsets, np.int32),
               conf=np.concatenate(conf), pcls=np.concatenate(pcls), correct=np.concatenate(correct).reshape(-1, niou))
    out["native"] = np.concatenate(nat).reshape(-1, 4) if native else None
    return out


def host_loop(batches):
    """What test.test's host loop appends per image: (correct bool, conf, pcls, native) slices, in batch order."""
    out = []
    for det, count, correct, nat, _ in batches:
        for b in range(det.shape[0]):
            n = int(count[b])
            out.append((correct[b, :n].astype(bool), det[b, :n, 4], det[b, :n, 5], None if nat is None else nat[b, :n]))
    return out


def ragged_batches(seed, sizes, max_det=300, niou=NIOU, native=True):
    """Random NMS-shaped batches with image counts per batch `sizes`; rows include zero and max_det kept detections."""
    g = np.random.Generator(np.random.PCG64(seed))
    out, image0 = [], 0
    for B in sizes:
        det = g.standard_normal((B, max_det, 6)).astype(np.float32)
        det[..., 5] = g.integers(0, 3, (B, max_det))
        count = g.integers(0, max_det + 1, B).astype(np.int32)
        count[g.random(B) < 0.2] = 0
        count[g.random(B) < 0.2] = max_det
        if len(out) == 1:
            count[0], count[-1] = 0, max_det
        correct = (g.random((B, max_det, niou)) < 0.3).astype(np.uint8)
        nat = g.standard_normal((B, max_det, 4)).astype(np.float32) * 300 if native else None
        out.append((det, count, correct, nat, image0))
        image0 += B
    return out, image0


def shard(batches, world):
    from icafusion_b200.test import owned_batches
    return [[batches[j] for j in owned_batches(len(batches), r, world)] for r in range(world)]


def pad(bufs, native):
    width = max([len(b) for b in bufs if b is not None] + [4])
    out = np.zeros((len(bufs), width), np.int32)
    for r, b in enumerate(bufs):
        out[r, :len(b) if b is not None else 4] = b if b is not None else [0, 0, 3 + 4 * native, 4]
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 7])
@pytest.mark.parametrize("native", [False, True])
def test_reference_pack_and_merge_give_the_host_loop_slices(world, native):
    """Ragged batches (B = 1 and 4 with a partial last batch; images with 0 and all 300 rows; W = 7 leaves ranks without a
    batch): packing each rank's batches and merging the buffers gives exactly the slices of the one-process loop."""
    batches, n = ragged_batches(world + 10 * native, [1, 4, 4, 2, 1, 3])
    bufs = [pack_reference(b, NIOU, native) if b else None for b in shard(batches, world)]
    m = merge_reference(pad(bufs, native), n, NIOU, native)
    want = host_loop(batches)
    assert len(m["counts"]) == n == len(want)
    assert {0, 300} <= set(m["counts"].tolist())
    for k, (cor, conf, pcls, nat) in enumerate(want):
        o, c = m["offsets"][k], m["counts"][k]
        assert np.array_equal(m["correct"][o:o + c].astype(bool), cor) and np.array_equal(m["conf"][o:o + c], conf)
        assert np.array_equal(m["pcls"][o:o + c], pcls)
        if native:
            assert np.array_equal(m["native"][o:o + c], nat)


def test_reference_merge_refuses_missing_and_duplicated_images():
    batches, n = ragged_batches(3, [2, 2, 1])
    parts = shard(batches, 2)
    bufs = [pack_reference(p, NIOU, False) for p in parts]
    with pytest.raises(ValueError, match="missing"):
        merge_reference(pad(bufs[:1], False), n, NIOU, False)
    with pytest.raises(ValueError, match="more than one"):
        merge_reference(pad(bufs + bufs[1:], False), n, NIOU, False)


def test_batch_ownership_covers_every_batch_once():
    from icafusion_b200.test import owned_batches
    for nb in (1, 2, 3, 4, 7, 2252):
        for world in range(1, 9):
            got = sorted(j for r in range(world) for j in owned_batches(nb, r, world))
            assert got == list(range(nb)), (nb, world)
            sizes = [len(owned_batches(nb, r, world)) for r in range(world)]
            assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        owned_batches(4, 2, 2)


def test_val_batches_shard_owns_the_same_batches():
    from icafusion_b200.test import owned_batches
    from icafusion_b200.valdata import ValBatches
    vb = ValBatches([np.zeros((0, 5), np.float32)] * 7, lambda i: None, [(512, 640)] * 7, 640, batch_size=2, device="meta")
    vb.batch = lambda j: ("batch", j)                              # no staging: only the ownership is checked here
    for world in (1, 2, 3, 5):
        for r in range(world):
            got = list(vb.shard(r, world))
            assert [g[0] for g in got] == list(owned_batches(len(vb), r, world))
            assert all(g[1] == 2 * g[0] and g[2] == ("batch", g[0]) for g in got)


# ---------------------------------------------------------------------------------------------- the C ABI
def test_entries_declared_exported_and_sizes_are_pure():
    from test_abi_cpu import _header_symbols
    from icafusion_b200 import _lib
    L = _lib.lib()
    for s in ("icaf_val_pack", "icaf_val_pack_bytes", "icaf_val_pack_params_bytes", "icaf_val_merge",
              "icaf_val_merge_workspace_bytes"):
        assert s in _header_symbols() and s in _lib.SIGNATURES and hasattr(L, s)
    assert ctypes.sizeof(_lib.ValBatch) == 64
    assert L.icaf_val_pack_bytes(2252, 300, 1) == 4 * (4 + 2252 * (4 + 300 * 7)) == L.icaf_val_pack_bytes(2252, 300, 1)
    assert L.icaf_val_pack_bytes(10, 300, 0) == 4 * (4 + 10 * (4 + 900))
    assert L.icaf_val_pack_bytes(-1, 300, 0) == 0 and L.icaf_val_pack_bytes(1, 0, 0) == 0 and L.icaf_val_pack_bytes(1, 1, 4) == 0
    assert L.icaf_val_pack_bytes(1 << 30, 300, 1) == 0                              # past int32 word indices
    assert L.icaf_val_pack_params_bytes(3, 7, 0) == 3 * 64 and L.icaf_val_pack_params_bytes(3, 7, 2) == 3 * 64 + 32
    assert L.icaf_val_pack_params_bytes(0, 7, 0) == 0 and L.icaf_val_pack_params_bytes(3, 2, 0) == 0
    assert L.icaf_val_merge_workspace_bytes(2252) == 2252 * 16 and L.icaf_val_merge_workspace_bytes(0) == 0


def test_entries_refuse_bad_arguments_before_any_launch():
    from icafusion_b200 import _lib
    L = _lib.lib()
    fake, n0 = 1 << 20, L.icaf_kernel_launches()                   # never dereferenced: refused on the host
    need = L.icaf_val_pack_params_bytes(2, 5, 0)
    out = L.icaf_val_pack_bytes(5, 300, 0)

    def pack(params=fake, nbytes=need, nb=2, n=5, niou=NIOU, flags=0, o=fake, ob=out):
        return L.icaf_val_pack(params, nbytes, nb, n, niou, flags, o, ob, None)

    assert pack(params=None) == 1 and pack(o=None) == 1 and b"null" in L.icaf_last_error()
    assert pack(nbytes=need - 1) == 1 and b"icaf_val_pack_params_bytes" in L.icaf_last_error()
    assert pack(nb=3) == 1 and pack(flags=2) == 1                                    # the table does not match its size
    assert pack(params=fake + 4) == 1 and pack(o=fake + 8) == 1                     # misaligned
    assert pack(niou=0) == 1 and pack(niou=33) == 1 and pack(ob=4 * (4 + 4 * 5) - 1) == 1
    ws = L.icaf_val_merge_workspace_bytes(5)

    def merge(bufs=fake, n_bufs=2, words=64, n=5, rows=10, flags=0, correct=fake, conf=fake, pcls=fake, native=None,
              counts=fake, offsets=fake, status=fake, mr_rows=None, mr_span=None, mr_images=0, mr_max=0, w=fake, wb=ws):
        return L.icaf_val_merge(bufs, n_bufs, words, n, rows, NIOU, flags, correct, conf, pcls, native, counts, offsets, status,
                                mr_rows, mr_span, mr_images, mr_max, w, wb, None)

    assert merge(bufs=None) == 1 and merge(status=None) == 1 and merge(counts=None) == 1 and merge(conf=None) == 1
    assert merge(flags=1) == 1                                                       # native rows without a native output
    assert merge(wb=ws - 1) == 1 and b"icaf_val_merge_workspace_bytes" in L.icaf_last_error()
    assert merge(n_bufs=0) == 1 and merge(n=0) == 1 and merge(words=3) == 1 and merge(bufs=fake + 4) == 1
    assert merge(mr_rows=fake) == 1 and merge(mr_rows=fake, mr_span=fake, mr_images=4, mr_max=300) == 1   # KAIST needs native
    assert merge(flags=8) == 1
    assert L.icaf_kernel_launches() == n0


def test_python_wrappers_refuse_bad_input_and_merge_status():
    from icafusion_b200 import ops
    with ops.dry_run():
        det = torch.empty(2, 300, 6, device="meta")
        with pytest.raises(ValueError, match="count"):
            ops.val_pack([(det, torch.empty(3, dtype=torch.int32, device="meta"), torch.empty(2, 300, NIOU, dtype=torch.uint8,
                                                                                                    device="meta"), None, 0)], NIOU)
        with pytest.raises(ValueError, match="native"):
            ops.val_pack([(det, torch.empty(2, dtype=torch.int32, device="meta"),
                           torch.empty(2, 300, NIOU, dtype=torch.uint8, device="meta"), None, 0)], NIOU, native=True)
    ops.val_merge_check([0, 0, 0, 12], 12)
    for st in ([1, 0, 0, 12], [0, 1, 0, 12], [0, 0, 1, 12], [0, 0, 0, 11]):
        with pytest.raises(ValueError):
            ops.val_merge_check(st, 12)


def test_dry_run_records_pack_and_merge_of_a_yolov5s_flir_shard():
    """The exchange of a sharded yolov5s FLIR call (nc = 3, 544 x 672 at B = 4, save_txt): rank 1 of 2 packs its two
    batches in one launch group, rank 0 merges the two buffers in another."""
    from icafusion_b200 import ops
    from icafusion_b200.test import owned_batches
    z = torch.empty(4, 3 * (68 * 84 + 34 * 42 + 17 * 21), 8, dtype=torch.float16, device="meta")     # Detect's rows at 544 x 672
    with torch.no_grad(), ops.dry_run() as d:
        batches = []
        for j in owned_batches(4, 1, 2):
            det, count = ops.nms(z, 0.001, 0.6, multi_label=True)
            native = torch.empty(4, 300, 4, device="meta")
            correct, _ = ops.match_detections(det, count, torch.empty(0, 6, device="meta"), torch.empty(4, 5, device="meta"),
                                              544, 672, torch.empty(NIOU, device="meta"), native=native)
            batches.append((det, count, correct, native, 4 * j))
        buf = ops.val_pack(batches, NIOU, native=True)
        m = ops.val_merge(torch.empty(2, buf.numel(), dtype=torch.int32, device="meta"), 16, 100, NIOU, native=True)
    names = [r[0] for r in d.records]
    assert names.count("icaf_val_pack") == 1 and names.count("icaf_val_merge") == 1
    assert names.count("icaf_nms_multi_label") == 2 and names[-2:] == ["icaf_val_pack", "icaf_val_merge"]
    pack = d.records[-2][1]
    assert pack[2:6] == (2, 8, NIOU, 1) and pack[1].value == 2 * 64
    assert buf.numel() * 4 == ops.val_pack_bytes(8, 300, True)
    merge = d.records[-1][1]
    assert merge[1:7] == (2, buf.numel(), 16, 100, NIOU, 1)
    assert tuple(m["correct"].shape) == (100, NIOU) and tuple(m["offsets"].shape) == (17,) and m["mr_rows"] is None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_val_exchange_kernels_spill_free(tmp_path):
    """ptxas report of metrics.cu: none of the pack and merge kernels spills."""
    from icafusion_b200 import build as B
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, "metrics.cu"), "-o", str(tmp_path / "m.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    log = out.stdout + out.stderr
    found = re.findall(r"Compiling entry function '(\w*val_(?:pack|merge)_\w+_kernel\w*)' for 'sm_90a'\n"
                       r"ptxas info\s*: Function properties for \w+\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    assert len(found) == 6, log
    assert all(f[1:] == ("0", "0", "0") for f in found), found
