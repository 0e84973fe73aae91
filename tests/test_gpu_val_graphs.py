"""test.test(..., graphs=ValidationGraphs(model)): the batch loop replayed from CUDA graphs gives exactly what the eager call
gives (results, maps, loss, MRresult and the save_txt files), across weight updates, shapes, partial batches and target
counts past the captured capacity, with no synchronising call once a shape is captured."""
import numpy as np
import pytest
import torch

from helpers import load_synth
from oracle import synth
from oracle.gen_golden_kaist_mr import SMALL_ANN, build_small, gunzip_to
from oracle.gen_golden_val import _image

pytestmark = pytest.mark.gpu

SHAPES = [((512, 640), ((1.0, 1.0), (16.0, 16.0))), ((590, 758), ((0.85, 0.85), (13.7, 21.3)))]
HYP = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


class _Loader:
    """Pinned batches.  `strict`: indices of batches whose consumer loop body must not synchronise (any such call raises)."""

    def __init__(self, batches, strict=()):
        self.batches, self.strict = batches, set(strict)

    def __len__(self):
        return len(self.batches)

    def __iter__(self):
        try:
            for i, b in enumerate(self.batches):
                torch.cuda.set_sync_debug_mode("error" if i in self.strict else 0)
                yield b
        finally:
            torch.cuda.set_sync_debug_mode(0)


def _model(cfg, seed, dev):
    from icafusion_b200 import Model
    m = Model(cfg).eval()
    load_synth(m, seed)
    m = m.to(dev)
    m.hyp, m.gr = dict(HYP), 1.0
    return m


def _batches(specs, nc, seed, names="img"):
    """specs: [(B, H, W, labels per image)] -> pinned (img uint8 (B, 6, H, W), targets, paths, shapes) batches."""
    g = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k, (B, H, W, n) in enumerate(specs):
        rgb, ir = synth.synth_images(B, H, W, 100 + k)
        img = (torch.cat([rgb, ir], 1) * 255).to(torch.uint8)
        lab = [np.concatenate([np.full((n, 1), i), _image(g, nc, n)[0]], 1) for i in range(B)]
        tg = torch.from_numpy(np.concatenate(lab).astype(np.float32))
        if nc == 1:
            tg[:, 1] = 0
        out.append((img.pin_memory(), tg.pin_memory(), [f"/d/{names}{k}_{i}.jpg" for i in range(B)],
                    [SHAPES[(k + i) % 2] for i in range(B)]))
    return out


def _labels_list(batches):
    from pathlib import Path
    return sorted([Path(p).stem + ".txt" for b in batches for p in b[2]] + ["zz_other.txt"])


def _run(model, batches, tmp, graphs=None, strict=(), **kw):
    from icafusion_b200 import test as T
    nc = model.model[-1].nc
    res, maps, mr, t = T.test({"nc": nc, "names": [str(i) for i in range(nc)]}, model=model,
                              dataloader=_Loader(batches, strict), save_dir=tmp, graphs=graphs, **kw)
    txt = (tmp / "labels" / "pred" / "result.txt").read_bytes() if kw.get("save_txt") else None
    return [float(x) for x in res], maps, mr, txt, t


def _same(a, b, where):
    assert a[0] == b[0], (where, a[0], b[0])
    assert np.array_equal(a[1], b[1]), where
    assert a[2] == b[2], where
    assert a[3] == b[3], where


def test_graphed_flir_detector_equals_eager_without_sync(cuda_device, tmp_path):
    """yolov5n FLIR through test.test at 544 x 672, B = 2, with compute_loss and save_txt: the graphed call equals the eager
    call, and once the shape is captured its batches make no synchronising call."""
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.loss import ComputeLoss
    model = _model("yolov5n_Transfusion_FLIR", 21, cuda_device)
    batches = _batches([(2, 544, 672, 5)] * 4, 3, 5)
    kw = dict(compute_loss=ComputeLoss(model), save_txt=True, labels_list=_labels_list(batches))
    eager = _run(model, batches, tmp_path / "eager", **kw)
    graphs = ValidationGraphs(model)
    got = _run(model, batches, tmp_path / "graphed", graphs, strict=(1, 2, 3), **kw)
    _same(got, eager, "first call")
    assert graphs.captures == 1 and len(graphs.entries) == 1
    assert eager[0][8:] != [0.0] * 4 and eager[0][6] >= 0 and len(got[4]) == 6
    again = _run(model, batches, tmp_path / "again", graphs, strict=(0, 1, 2, 3), **kw)
    _same(again, eager, "second call")
    assert graphs.captures == 1


def test_refresh_carries_ema_updates_into_the_graphs(cuda_device, tmp_path):
    """yolov5s KAIST with synthetic weights, one ValidationGraphs over three calls with ModelEMA.update between them; each
    graphed call equals an eager call on the same weights bit for bit.  In the second the anchors are put back after the
    update, so the new filters reach the graphs by the in-place refresh alone (nothing is captured again); in the third the
    eager call runs first and re-packs into new tensors, which the graphs must notice."""
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.loss import ComputeLoss
    from icafusion_b200.trainer import ModelEMA
    train = _model("yolov5s_Transfusion_kaist", 31, cuda_device)
    ema = ModelEMA(_model("yolov5s_Transfusion_kaist", 32, cuda_device))
    model = ema.ema
    model.hyp, model.gr = dict(HYP), 1.0
    batches = _batches([(1, 512, 640, 4)] * 3, 1, 9)
    kw = dict(compute_loss=ComputeLoss(model), save_txt=True, labels_list=_labels_list(batches))
    graphs = ValidationGraphs(model)
    first = _run(model, batches, tmp_path / "g1", graphs, **kw)
    _same(first, _run(model, batches, tmp_path / "e1", **kw), "before the update")
    assert graphs.captures == 1
    det = model.model[-1]
    anchors = det.anchor_grid.clone()
    ema.updates = 500
    ema.update(train)
    det.anchor_grid.copy_(anchors)
    second = _run(model, batches, tmp_path / "g2", graphs, strict=(0, 1, 2), **kw)
    _same(second, _run(model, batches, tmp_path / "e2", **kw), "after an update, refreshed in place")
    assert graphs.captures == 1 and second[0] != first[0]
    ema.update(train)
    eager = _run(model, batches, tmp_path / "e3", **kw)
    third = _run(model, batches, tmp_path / "g3", graphs, **kw)
    _same(third, eager, "after an update, eager first")
    assert graphs.captures == 2 and third[0] != second[0]


def test_shapes_partial_batch_and_target_capacity(cuda_device, tmp_path):
    """Two rect shapes, a partial last batch and a batch with more labels than the shape's captured capacity (64 rows),
    with at most two shapes held (the partial batch's shape runs eagerly): the results equal the eager call's."""
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.loss import ComputeLoss
    model = _model("yolov5n_Transfusion_FLIR", 23, cuda_device)
    batches = _batches([(2, 544, 672, 5), (2, 512, 672, 3), (2, 544, 672, 6), (2, 544, 672, 40), (2, 512, 672, 2),
                        (2, 544, 672, 4), (1, 512, 672, 3)], 3, 11)
    kw = dict(compute_loss=ComputeLoss(model), save_txt=True, labels_list=_labels_list(batches))
    eager = _run(model, batches, tmp_path / "eager", **kw)
    graphs = ValidationGraphs(model)
    graphs.max_shapes = 2
    got = _run(model, batches, tmp_path / "graphed", graphs, strict=(2, 4, 5, 6), **kw)
    _same(got, eager, "mixed shapes")
    assert graphs.captures == 3                                 # two shapes, one of them again at 128 target rows
    assert sorted(e.capacity for e in graphs.entries.values()) == [64, 128]


def test_kaist_miss_rate_equals_eager(cuda_device, tmp_path):
    """The KAIST mr_annotations path (icaf_kaist_round_detections captured behind the matching) gives the eager MRresult."""
    from icafusion_b200 import kaist_eval as K
    from icafusion_b200.engine import ValidationGraphs
    small, labels_list, _ = build_small()
    model = _model("yolov5n_Transfusion_kaist", 41, cuda_device)
    batches = []
    for k, (_, tg, shapes, paths) in enumerate(small):
        rgb, ir = synth.synth_images(len(paths), 544, 672, 60 + k)
        img = (torch.cat([rgb, ir], 1) * 255).to(torch.uint8)
        batches.append((img.pin_memory(), torch.from_numpy(tg.copy()).pin_memory(), list(paths), list(shapes)))
    ann = K.KaistAnnotations(gunzip_to(SMALL_ANN, tmp_path), cuda_device)
    kw = dict(labels_list=labels_list, mr_annotations=ann)
    eager = _run(model, batches, tmp_path / "eager", **kw)
    graphs = ValidationGraphs(model)
    got = _run(model, batches, tmp_path / "graphed", graphs, strict=range(1, len(batches)), **kw)
    _same(got, eager, "KAIST")
    again = _run(model, batches, tmp_path / "again", graphs, **dict(kw, save_txt=True))
    _same(again[:3] + (None,), eager[:3] + (None,), "KAIST with save_txt")
    assert eager[2] != [0.0] * 10 and graphs.captures == 1             # save_txt alone changes nothing captured
