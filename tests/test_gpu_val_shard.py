"""test.test(..., group=) on the device: the pack / merge kernels against the numpy layout and the one-process host loop,
then two and three gloo ranks on one GPU (and two NCCL ranks when there are two GPUs) against one process running the
whole loader, compared with == on the results, maps, MRresult, loss and every save_txt file."""
import functools
import os
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist

from test_gpu_sync_bn import _spawn
from test_gpu_val_graphs import HYP, _batches, _labels_list, _Loader, _model
from test_val_shard_cpu import NIOU, host_loop, pack_reference, pad, ragged_batches, shard

pytestmark = pytest.mark.gpu


def _to_dev(batches, dev):
    return [(torch.from_numpy(d).to(dev), torch.from_numpy(c).to(dev), torch.from_numpy(k).to(dev),
             None if n is None else torch.from_numpy(n).to(dev), i0) for d, c, k, n, i0 in batches]


@pytest.mark.parametrize("native", [False, True])
def test_pack_and_merge_equal_the_host_loop(cuda_device, native):
    """Ragged B = 1 / 4 batches with images of 0 and 300 rows, packed per rank for W = 1, 3 and 8 (ranks without a batch),
    merged on the device: every flat array equals the host loop's slices; the packed words equal the numpy layout.  At the
    device's SM count the row kernels give each image its own block; planned for one SM their grids are 8 blocks, so that
    the merge of the 15 images and the pack of W = 1 walk two images per block."""
    from icafusion_b200 import ops
    batches, n = ragged_batches(7 + native, [1, 4, 4, 2, 1, 3], native=native)
    assert n > 8
    want = host_loop(batches)
    for target in (0, 1):
        with ops.sm_count_target(target):
            _pack_and_merge(cuda_device, batches, n, want, native)


def _pack_and_merge(cuda_device, batches, n, want, native):
    from icafusion_b200 import ops
    for world in (1, 3, 8):
        bufs = []
        for part_h, part_d in zip(shard(batches, world), shard(_to_dev(batches, cuda_device), world)):
            if not part_d:
                bufs.append(None)
                continue
            buf = ops.val_pack(part_d, NIOU, native=native)
            ref = pack_reference(part_h, NIOU, native)
            got = buf.cpu().numpy()
            assert got[3] == len(ref) and np.array_equal(got[:len(ref)], ref)
            bufs.append(ref)
        m = ops.val_merge(torch.from_numpy(pad(bufs, native)).to(cuda_device), n, sum(len(w[1]) for w in want), NIOU, native)
        ops.val_merge_check(m["status"].cpu().tolist(), sum(len(w[1]) for w in want))
        counts, offsets = m["counts"].cpu().tolist(), m["offsets"].cpu().tolist()
        correct, conf, pcls = m["correct"].cpu().numpy().astype(bool), m["conf"].cpu().numpy(), m["pcls"].cpu().numpy()
        assert {0, 300} <= set(counts)
        for k, (cor, cf, pc, nat) in enumerate(want):
            o, c = offsets[k], counts[k]
            assert np.array_equal(correct[o:o + c], cor) and np.array_equal(conf[o:o + c], cf) and np.array_equal(pcls[o:o + c], pc)
            if native:
                assert np.array_equal(m["native"][o:o + c].cpu().numpy(), nat)


def test_merge_writes_the_kaist_rows_and_refuses_missing_or_duplicated_images(cuda_device):
    from icafusion_b200 import ops
    batches, n = ragged_batches(11, [1, 4, 3, 2])
    for d, *_ in batches:
        d[..., :4] = np.abs(d[..., :4]) * 100                  # scores and boxes in the range test.py writes
    dev = _to_dev(batches, cuda_device)
    perm = np.random.Generator(np.random.PCG64(1)).permutation(n + 5).astype(np.int32)[:n]      # KAIST positions
    images = n + 5
    rows = torch.empty(images * 300, 5, dtype=torch.float64, device=cuda_device)
    span = torch.zeros(images, 2, dtype=torch.int32, device=cuda_device)
    for (d, c, _, nat, i0) in dev:
        ops.kaist_round_detections(nat, d, c, torch.from_numpy(perm[i0:i0 + d.shape[0]]).to(cuda_device), rows, span)
    parts = shard(dev, 2)
    pos = [np.concatenate([perm[b[4]:b[4] + b[0].shape[0]] for b in p]) for p in parts]
    bufs = [ops.val_pack(p, NIOU, native=True, positions=q) for p, q in zip(parts, pos)]
    w = max(int(b[3]) for b in bufs)
    stacked = torch.stack([torch.cat([b[:int(b[3])], b.new_zeros(w - int(b[3]))]) for b in bufs])
    n_rows = sum(int(b[1]) for b in bufs)
    m = ops.val_merge(stacked, n, n_rows, NIOU, native=True, mr=(images, 300))
    ops.val_merge_check(m["status"].cpu().tolist(), n_rows)
    assert torch.equal(m["mr_span"], span)
    for p in range(images):
        o, c = span[p].tolist()
        assert torch.equal(m["mr_rows"][o:o + c], rows[o:o + c])
    for bad in (stacked[:1], torch.cat([stacked, stacked[1:]])):            # image missing, image twice
        m = ops.val_merge(bad.contiguous(), n, n_rows, NIOU, native=True)
        with pytest.raises(ValueError):
            ops.val_merge_check(m["status"].cpu().tolist(), n_rows)


# ------------------------------------------------------------------------------------------------------------------------
# ranks against one process
def _call(model, loader, save_dir, graphs=None, group=None, **kw):
    from icafusion_b200 import test as T
    nc = model.model[-1].nc
    res, maps, mr, t = T.test({"nc": nc, "names": [str(i) for i in range(nc)]}, model=model, dataloader=loader,
                              save_dir=save_dir, graphs=graphs, group=group, **kw)
    files = None
    if kw.get("save_txt") and (group is None or dist.get_rank(group) == 0):
        d = Path(save_dir) / "labels" / "pred"
        files = {p.name: p.read_bytes() for p in sorted(d.iterdir())}
    return [float(x) for x in res], np.asarray(maps), list(mr), files


def _same(a, b, where):
    assert a[0] == b[0], (where, a[0], b[0])
    assert np.array_equal(a[1], b[1]), where
    assert a[2] == b[2], where
    if a[3] is not None and b[3] is not None:
        assert a[3] == b[3], where


def _flir_batches(kind):
    if kind == "b1":
        return _batches([(1, 544, 672, 5)] * 4, 3, 5)
    return None


def _val_batches(nc, dev):
    """A B = 4 ValBatches over 7 synthetic pairs: batches of 4 and 3 (the partial last batch)."""
    from icafusion_b200.valdata import ValBatches
    g = np.random.Generator(np.random.PCG64(3))
    hw0 = [(512, 640)] * 4 + [(480, 640)] * 3
    frames = {i: (g.integers(0, 256, hw + (3,), dtype=np.uint8), g.integers(0, 256, hw + (3,), dtype=np.uint8)) for i, hw in enumerate(hw0)}
    labels = []
    for _ in hw0:
        lab = np.concatenate([g.integers(0, nc, (5, 1)), g.uniform(0.2, 0.8, (5, 2)), g.uniform(0.05, 0.2, (5, 2))], 1)
        labels.append(lab.astype(np.float32))
    return ValBatches(labels, frames.__getitem__, hw0, 640, batch_size=4, paths=[f"/d/vb{i}.jpg" for i in range(7)], device=dev)


def _flir_case(rank, dev, cfg="yolov5l_Transfusion_FLIR", world=2):
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.loss import ComputeLoss
    model = _model(cfg, 21, dev)
    group = dist.group.WORLD
    tmp = Path(tempfile.mkdtemp())
    out = {}
    batches = _flir_batches("b1")
    vb = _val_batches(3, dev)
    loaders = {"b1": (lambda strict=(): _Loader(batches, strict), _labels_list(batches)),
               "b4": (lambda strict=(): vb, sorted(Path(p).stem + ".txt" for p in vb.paths))}
    for name, (make, labels_list) in loaders.items():
        kw = dict(compute_loss=ComputeLoss(model), save_txt=True, labels_list=labels_list)
        graphs = ValidationGraphs(model)
        strict = range(world, len(batches)) if name == "b1" else ()
        out[name, "graphed"] = _call(model, make(strict), tmp / f"{name}g", graphs, group, **kw)
        out[name, "graphed again"] = _call(model, make(strict and range(len(batches))), tmp / f"{name}g2", graphs, group, **kw)
        out[name, "captures"] = graphs.captures
        out[name, "eager"] = _call(model, make(), tmp / f"{name}e", None, group, **kw)
        if rank == 0:
            out[name, "one"] = _call(model, make(), tmp / f"{name}1", None, None, **kw)
    return out


def _check_flir(res, names=("b1", "b4")):
    one = res[0]
    for rank, out in enumerate(res):
        for name in names:
            for mode in ("graphed", "graphed again", "eager"):
                _same(out[name, mode], one[name, "one"], (rank, name, mode))
            assert out[name, "captures"] == (rank < {"b1": 4, "b4": 2}[name])     # a rank without a batch captures nothing
    for name in names:
        assert one[name, "one"][3] and one[name, "one"][0][8:] != [0.0] * 4     # files written, a loss accumulated


def test_flir_two_gloo_ranks_equal_one_process(cuda_device):
    """yolov5l FLIR at B = 1 (four batches) and a B = 4 ValBatches with a partial last batch, graphed (twice: the second
    call replays only, with no synchronising call in the loop) and eager, on both ranks."""
    res = _spawn(_flir_case, timeout=900)
    _check_flir(res)                                              # one capture per rank: the second call reused the graphs


def test_flir_three_ranks_over_four_batches(cuda_device):
    """W = 3 over four B = 1 batches (rank 0 runs two, ranks 1 and 2 one each) and over the two ValBatches batches (rank 2
    runs none)."""
    res = _spawn(functools.partial(_flir_case, cfg="yolov5n_Transfusion_FLIR", world=3), world=3, timeout=900)
    _check_flir(res)


def _kaist_case(rank, dev):
    from oracle.gen_golden_kaist_mr import SMALL_ANN, build_small, gunzip_to
    from oracle import synth
    from icafusion_b200 import kaist_eval as K
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.loss import ComputeLoss
    small, labels_list, _ = build_small()
    model = _model("yolov5s_Transfusion_kaist", 41, dev)
    batches = []
    for k, (_, tg, shapes, paths) in enumerate(small):
        rgb, ir = synth.synth_images(len(paths), 544, 672, 60 + k)
        img = (torch.cat([rgb, ir], 1) * 255).to(torch.uint8)
        batches.append((img.pin_memory(), torch.from_numpy(tg.copy()).pin_memory(), list(paths), list(shapes)))
    tmp = Path(tempfile.mkdtemp())
    ann = K.KaistAnnotations(gunzip_to(SMALL_ANN, tmp), dev)
    kw = dict(labels_list=labels_list, mr_annotations=ann, save_txt=True, compute_loss=ComputeLoss(model))
    group = dist.group.WORLD
    out = {"graphed": _call(model, _Loader(batches), tmp / "g", ValidationGraphs(model), group, **kw),
           "eager": _call(model, _Loader(batches), tmp / "e", None, group, **kw)}
    if rank == 0:
        out["one"] = _call(model, _Loader(batches), tmp / "1", None, None, **kw)
    return out


def test_kaist_miss_rate_two_gloo_ranks_equal_one_process(cuda_device):
    """yolov5s KAIST (nc = 1) with mr_annotations: MRresult, the loss and the files equal one process's."""
    res = _spawn(_kaist_case, timeout=900)
    one = res[0]["one"]
    assert one[2] != [0.0] * 10
    for rank, out in enumerate(res):
        for mode in ("graphed", "eager"):
            _same(out[mode], one, (rank, mode))


def _broadcast_case(rank, dev):
    from icafusion_b200.engine import ValidationGraphs, broadcast_model_
    from icafusion_b200.loss import ComputeLoss
    from icafusion_b200.trainer import ModelEMA
    ema = ModelEMA(_model("yolov5s_Transfusion_kaist", 32 + 7 * rank, dev))      # rank 1 starts from other weights
    model = ema.ema
    model.hyp, model.gr = dict(HYP), 1.0
    batches = _batches([(1, 512, 640, 4)] * 4, 1, 9)
    kw = dict(compute_loss=ComputeLoss(model), save_txt=True, labels_list=_labels_list(batches))
    group = dist.group.WORLD
    tmp = Path(tempfile.mkdtemp())
    graphs = ValidationGraphs(model)
    broadcast_model_(model, 0, group)
    out = {"first": _call(model, _Loader(batches), tmp / "g1", graphs, group, **kw)}
    if rank == 0:
        out["first one"] = _call(model, _Loader(batches), tmp / "o1", None, None, **kw)
        train = _model("yolov5s_Transfusion_kaist", 31, dev)
        anchors = model.model[-1].anchor_grid.clone()
        ema.updates = 500
        ema.update(train)
        model.model[-1].anchor_grid.copy_(anchors)
    broadcast_model_(model, 0, group)
    out["second"] = _call(model, _Loader(batches, strict=range(2, 4)), tmp / "g2", graphs, group, **kw)
    out["captures"] = graphs.captures
    if rank == 0:
        out["second one"] = _call(model, _Loader(batches), tmp / "o2", None, None, **kw)
    return out


def test_broadcast_model_then_graphed_sharded_call_equals_rank0(cuda_device):
    """broadcast_model_ gives rank 1 rank 0's EMA weights in place: after an EMA update on rank 0 and a second broadcast, the
    graphed sharded call equals rank 0's one-process call, from the graphs captured by the first call."""
    res = _spawn(_broadcast_case, timeout=900)
    for rank, out in enumerate(res):
        _same(out["first"], res[0]["first one"], (rank, "first"))
        _same(out["second"], res[0]["second one"], (rank, "second"))
        assert out["captures"] == 1
    assert res[0]["second one"][0] != res[0]["first one"][0]


def _refusal_case(rank, dev):
    from icafusion_b200 import test as T
    model = _model("yolov5n_Transfusion_FLIR", 5, dev)
    batches = _flir_batches("b1")
    msgs = []
    for loader in (_Loader(batches[:4 - rank]),):
        try:
            T.test({"nc": 3, "names": ["0", "1", "2"]}, model=model, dataloader=loader, save_dir=tempfile.mkdtemp(),
                   group=dist.group.WORLD)
        except ValueError as e:
            msgs.append(str(e))
    return msgs


def test_loaders_of_different_lengths_are_refused_on_every_rank(cuda_device):
    res = _spawn(_refusal_case)
    assert all(len(m) == 1 and "batches" in m[0] for m in res)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (NCCL)")
def test_flir_two_nccl_ranks_equal_one_process(cuda_device):
    res = _spawn(functools.partial(_flir_case, cfg="yolov5n_Transfusion_FLIR"), backend="nccl", timeout=900)
    _check_flir(res)
