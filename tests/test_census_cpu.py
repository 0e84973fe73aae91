"""The launch census without a GPU: every entry point the detectors issue is either replayed or listed with a reason, the
census spans every conv plan family, and each replay builder re-issues exactly the launch it replays (tests/census.py)."""
import collections

import pytest

import census


@pytest.fixture(scope="module")
def walks():
    return {c.id: census.walk_config(c) for c in census.CONFIGS}


@pytest.fixture(scope="module")
def records(walks):
    """Unique records over all configurations, {key: record}."""
    out = {}
    for recs in walks.values():
        for k, r in census.unique(recs).items():
            out.setdefault(k, r)
    return out


def test_configurations():
    ids = [c.id for c in census.CONFIGS]
    assert len(ids) == len(set(ids)) == 5 * 2 * 2 + 3 * 2 + 5 * 2 + 5 * 2 * 2 + 3 * 3 + 1
    assert "yolov5x-kaist-512x640-b16-infer" in ids and "yolov5l-kaist-512x640-b16-train" in ids
    # train.py's mosaic batches (640x640, batch 8 by default) and test.py's rectangular validation batches (544x672)
    for s in "nsl":
        assert {f"yolov5{s}-kaist-640x640-b{B}-train" for B in (8, 16, 3)} <= set(ids)
    assert "yolov5s-flir-640x640-b8-train" in ids
    assert {f"yolov5{s}-{ds}-544x672-b{B}-infer" for s in "nsmlx" for ds in ("kaist", "flir") for B in (1, 32)} <= set(ids)
    assert {f"yolov5{s}-flir-512x640-b{B}-infer" for s in "nsmlx" for B in (1, 16)} <= set(ids)


def test_keys_are_pointer_free():
    """Two walks of one configuration give the same key set: no pointer, seed or per-call object reaches a key (the loss
    records pass per-level pointer arrays and byref(LossHyp))."""
    c = census.Config("train", "n", "kaist", 3, 640, 640)
    a, b = (census.walk(c.kind, f"yolov5{c.size}_Transfusion_{c.dataset}", c.B, c.H, c.W) for _ in range(2))
    ka, kb = set(census.unique(a)), set(census.unique(b))
    assert ka == kb
    assert {"icaf_compute_loss_fwd", "icaf_compute_loss_bwd"} <= {k[0] for k in ka}


def test_every_entry_point_is_accounted_for(walks):
    """A C-ABI call a detector issues is replayed or listed with a reason, and neither map names a call no walk issues."""
    assert not set(census.REPLAYED) & set(census.NOT_REPLAYED)
    issued = {name for recs in walks.values() for name, _, _ in recs}
    accounted = set(census.REPLAYED) | set(census.NOT_REPLAYED)
    assert issued - accounted == set(), f"entry points the census neither replays nor excuses: {sorted(issued - accounted)}"
    # all_reduce is issued only when SyncBatchNorm runs under a process group
    assert accounted - issued <= {"all_reduce"}, f"entry points no walk issues: {sorted(accounted - issued)}"


def test_census_covers_every_conv_plan_family(records):
    from icafusion_b200 import _lib
    convs = [r for k, r in records.items() if k[0] == "icaf_conv2d_fwd"]
    wgrads = [r for k, r in records.items() if k[0] == "icaf_conv2d_wgrad"]
    slices = [r for r in convs if any(io.x_ld > r[1][0]._obj.Cin or io.y_ld > r[1][0]._obj.Cout for io in r[1][1])]
    bns, modes, kinds, splits = collections.Counter(), collections.Counter(), collections.Counter(), collections.Counter()
    for _, args, _ in convs:
        pl = census.conv_plan(args[0]._obj, args[2], 132)
        assert pl is not None and pl.kernel == _lib.KERNEL_TC, census.describe((None, args, None))
        bns[pl.bn] += 1
        modes[pl.a_mode] += 1
        kinds["persistent" if pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z else "one-tile"] += 1
        splits[pl.splits] += 1
    print(f"\n{len(convs)} conv, {len(wgrads)} wgrad, {len(slices)} slice launches; bn {dict(bns)} a_mode {dict(modes)} {dict(kinds)} "
          f"splits {dict(sorted(splits.items()))}")
    assert len(convs) >= 2450 and len(wgrads) >= 525 and len(slices) >= 625
    assert {32, 64, 128} <= set(bns) and {0, 1, 2} <= set(modes) and {"persistent", "one-tile"} <= set(kinds)
    assert {2, 3, 4, 5, 6, 8} <= set(splits)


DROPOUT_P = {"icaf_cross_attention_train": 9, "icaf_cross_attention_bwd": 13, "icaf_eltwise": 5}     # argument index of p


def test_builders_reissue_the_recorded_launch(records):
    """Each builder, run on meta tensors under a dry run, issues a call with the same key as the record it replays: the replay
    hits the product's geometry, channel pitches, epilogue flags and scales.  A dropout record (p > 0) is also replayed at its
    recorded p, which the key leaves out."""
    from icafusion_b200 import ops
    done, dropout = collections.Counter(), collections.Counter()
    for k, rec in records.items():
        if k[0] not in census.REPLAYED:
            continue
        with ops.dry_run() as dr:
            assert census.replay(rec, "meta") == []
        issued = {census.key(r) for r in dr.records}
        assert k in issued, f"{census.describe(rec)}: the replay issued {sorted(issued, key=str)[:4]}"
        done[k[0]] += 1
        if k[0] in DROPOUT_P and rec[1][DROPOUT_P[k[0]]] > 0:
            i = DROPOUT_P[k[0]]
            ps = {r[1][i] for r in dr.records if census.key(r) == k}
            assert rec[1][i] in ps, f"{census.describe(rec)}: recorded p {rec[1][i]}, replayed at {sorted(ps)}"
            dropout[k[0]] += 1
    print("\ndistinct launches replayed per entry point: " + ", ".join(f"{n} {c}" for n, c in sorted(done.items())))
    print("of which replayed at their dropout probability: " + ", ".join(f"{n} {c}" for n, c in sorted(dropout.items())))
    assert set(done) == set(census.REPLAYED)
    # training's dropout launches: 36 attention geometries (forward and backward) and 27 element-wise sizes, all at p = 0.1
    assert dropout == {"icaf_cross_attention_train": 36, "icaf_cross_attention_bwd": 36, "icaf_eltwise": 27}, dropout
    assert done["icaf_eltwise"] == 81
