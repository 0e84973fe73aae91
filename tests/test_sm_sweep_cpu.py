"""The SM-count target without a GPU: its semantics in the library (icaf_set_sm_count_target, ops.sm_count_target), and the
sweep's selection (tests/sm_sweep.py) covering every plan the targets produce for the census launches."""
import collections
import ctypes as C

import pytest

import census
import sm_sweep


def _probe():
    """A 3x3 64 -> 128 weight gradient on a 160 x 160 map: 9 work items and 200 M tiles, so that its split count,
    2 * sms // 9, moves with every SM count up to 288."""
    from icafusion_b200 import _lib
    return _lib.ConvGeom(1, 160, 160, 64, 160, 160, 128, 3, 3, 1, 1, 576, 128, 0, 0)


def test_target_is_clamped_restored_and_validated():
    from icafusion_b200 import _lib, ops
    L, g = _lib.lib(), _probe()
    per = sm_sweep.wgrad_split_bytes(g)
    ws = lambda: int(L.icaf_conv2d_wgrad_workspace_bytes(C.byref(g)))      # noqa: E731
    own, sms = ws(), L.icaf_sm_count()
    assert own > 0 and own % per == 0
    for t in (1, 4, 8, 16, 32, 60, 64, 78, 114, 132):
        with ops.sm_count_target(t):
            assert ws() == per * max(1, min(2 * t // 9, 64)), t
            assert L.icaf_sm_count() == sms                    # the device's count, whatever the target
    # a target above the count the library sees plans for that count; 0 restores it
    with ops.sm_count_target(1 << 20):
        assert ws() == own
    assert L.icaf_set_sm_count_target(8) == 0 and ws() == per
    assert L.icaf_set_sm_count_target(0) == 0 and ws() == own
    # a negative target is refused and leaves the target as it was
    with ops.sm_count_target(16):
        assert L.icaf_set_sm_count_target(-1) == 1 and b"positive" in L.icaf_last_error()
        with pytest.raises(_lib.IcafError):
            with ops.sm_count_target(-8):
                pass
        assert ws() == per * 3
    assert ws() == own


def test_target_is_restored_when_the_body_raises():
    from icafusion_b200 import _lib, ops
    g = _probe()
    own = int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g)))
    with ops.sm_count_target(32):
        with pytest.raises(RuntimeError):
            with ops.sm_count_target(8):
                raise RuntimeError("replay failed")
        assert sm_sweep.wgrad_signature(("icaf_conv2d_wgrad", (C.byref(g),), {}), 32) == 7
        assert int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g))) == sm_sweep.wgrad_split_bytes(g) * 7
    assert int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g))) == own


@pytest.fixture(scope="module")
def selection():
    """(pairs at 132 SMs, {pair the targets add: target it is replayed under}); a pair is ((geometry), signature)."""
    base = sm_sweep.CPU_SMS
    table = sm_sweep.coverage(base)
    cov_of = {id(r): cov for r, cov in table}
    at_base = {cov[base] for _, cov in table}
    picked = {}
    for t in sm_sweep.TARGETS:
        for rec in sm_sweep.select(t, base):
            pair = cov_of[id(rec)][t]
            assert pair not in at_base and pair not in picked, (t, census.describe(rec))
            picked[pair] = t
    return at_base, picked


def _conv_sigs(pairs):
    return [p[1] for p in pairs if p[0][0] == "icaf_conv2d_fwd"]


def test_selection_covers_every_plan_the_targets_produce(selection):
    at_base, picked = selection
    table = sm_sweep.coverage(sm_sweep.CPU_SMS)
    everything = {cov[s] for _, cov in table for s in (sm_sweep.CPU_SMS,) + sm_sweep.TARGETS}
    assert at_base | set(picked) == everything
    per_target = collections.defaultdict(collections.Counter)
    for pair, t in picked.items():
        per_target[pair[0][0]][t] += 1
    base_pairs = collections.Counter(p[0][0] for p in at_base)
    print(f"\n(geometry, plan) pairs at {sm_sweep.CPU_SMS} SMs: " + ", ".join(f"{n} {c}" for n, c in sorted(base_pairs.items())))
    print("extra pairs the targets add: " + ", ".join(f"{n} {sum(c.values())}" for n, c in sorted(per_target.items())))
    for name, c in sorted(per_target.items()):
        print(f"  {name:22s} " + "  ".join(f"{t}: {c[t]}" for t in sm_sweep.TARGETS))
    assert set(per_target) == set(sm_sweep.SIGNATURES)

    # plans 132 SMs never gives: a split-K cluster of 7, and persistent CTAs that walk two, three and four or more tiles
    assert 7 not in {s[6] for s in _conv_sigs(at_base)}
    new = _conv_sigs(picked)
    assert 7 in {s[6] for s in new}
    walks = collections.Counter(s[8:] for s in new if s[7])
    print("persistent plans the targets add, by (min(floor, 4), min(ceil, 4), parities) tiles per CTA: " +
          ", ".join(f"{w}: {n}" for w, n in sorted(walks.items())))
    assert {(1, 2), (2, 3), (3, 4), (4, 4)} <= {w[:2] for w in walks}


def test_targets_send_yolov5s_at_batch_1_to_the_persistent_kernel(selection):
    """At 132 SMs no yolov5s batch-1 512x640 launch is persistent (tests/test_persist_plan_cpu.py); smaller counts send some
    there, and the selection replays each of those plans."""
    _, picked = selection
    cfg = census.Config("infer", "s", "kaist", 1, 512, 640)
    assert cfg in census.CONFIGS
    convs = [r for k, r in census.unique(census.walk_config(cfg)).items() if k[0] == "icaf_conv2d_fwd"]
    assert not any(sm_sweep.conv_signature(r, sm_sweep.CPU_SMS)[7] for r in convs)
    counts = {}
    for t in sm_sweep.TARGETS:
        persistent = [r for r in convs if sm_sweep.conv_signature(r, t)[7]]
        counts[t] = len(persistent)
        for r in persistent:
            pair = (sm_sweep.geometry(r), sm_sweep.conv_signature(r, t))
            assert picked.get(pair, 0) >= t, (t, census.describe(r))          # replayed under t or a larger target
    print("\nyolov5s b1 512x640 persistent launches per target: " + ", ".join(f"{t}: {n}" for t, n in counts.items()))
    assert counts[8] > 0
