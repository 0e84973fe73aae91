"""datasets.ParamBlock, the host builder of the icaf_val_stage and icaf_augment parameter blocks: table interning, 16-byte
aligned regions, and block sizes equal to what the library computes for the same layout."""
import ctypes as C

import numpy as np
import pytest


def test_param_block_layout_matches_the_library():
    from icafusion_b200 import _lib, ops
    from icafusion_b200.datasets import ParamBlock, resize_taps
    L = _lib.lib()

    # validation: int32 tables of any length, each padded to a 16-byte boundary
    blk = ParamBlock()
    tabs = {k: np.arange(1, n + 1, dtype=np.int32) * (k + 1) for k, n in enumerate((6, 8, 3, 12))}
    offs = [blk.table(("t", k), lambda k=k: tabs[k]) for k in tabs]
    assert offs == [0, 8, 16, 20] and blk.n_words == 32
    assert blk.table(("t", 1), lambda: pytest.fail("a repeated key builds its table again")) == 8 and blk.n_words == 32
    samples = (_lib.ValSample * 3)()
    samples[1].mode = 7
    nbytes = int(L.icaf_val_stage_params_bytes(3, blk.n_words))
    with ops.dry_run():
        got = blk.upload(samples, (), nbytes, "cpu").numpy()
        with pytest.raises(ValueError):
            blk.upload(samples, (), nbytes + 16, "cpu")
    assert got.size == nbytes
    assert got[:C.sizeof(samples)].tobytes() == bytes(samples)
    base = (C.sizeof(samples) + 15) // 16 * 16
    words = got[base:].view(np.int32)
    for k, o in zip(tabs, offs):
        assert (base + 4 * o) % 16 == 0
        n = tabs[k].size
        assert np.array_equal(words[o:o + n], tabs[k]) and not words[o + n:(o + n + 3) // 4 * 4].any()

    # augmentation: the warp region, then resize_taps tables addressed in int4 rows
    blk = ParamBlock()
    B, s = 2, 40
    warp = np.arange(B * 4 * s, dtype=np.int32).reshape(B, 4, s)
    rows = [blk.table(key, lambda key=key: resize_taps(*key)) // 4 for key in ((640, 40, False), (512, 32, True), (640, 40, False))]
    assert rows == [0, 40, 0] and blk.n_words == 4 * 72
    samples = (_lib.AugSample * B)()
    nbytes = int(L.icaf_augment_params_bytes(B, s, blk.n_words // 4))
    with ops.dry_run():
        got = blk.upload(samples, (warp,), nbytes, "cpu").numpy()
    assert got.size == nbytes
    base = (C.sizeof(samples) + 15) // 16 * 16
    assert np.array_equal(got[base:base + warp.nbytes].view(np.int32).reshape(B, 4, s), warp)
    taps = got[base + warp.nbytes:].view(np.int32).reshape(-1, 4)
    assert np.array_equal(taps[:40], resize_taps(640, 40)) and np.array_equal(taps[40:], resize_taps(512, 32, True))
