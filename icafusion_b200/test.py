"""Validation with the reference's name, signature and return value (test.py:23-367), for ``train.py``'s per-epoch call.

``test(data, model=ema.ema, dataloader=testloader, ...)`` returns ``(tp, fp, fn, f1, mp, mr, map50, map, *loss), maps,
MRresult, t`` like the reference.  Per batch everything stays on the device and nothing waits for it: the forward on the
uint8 halves, the optional validation loss (accumulated on the device), the multi-label NMS (icaf_nms_multi_label) and the
matching of detections to labels (icaf_match_detections, one launch per batch).  The host synchronises once, after the last
batch, to gather the statistics in the order the reference appends them and to compute the metrics (metrics.py).

Not built: the command-line path (``weights=`` without ``model=``: attempt_load and a loader made from ``opt``), the
pycocotools JSON (``save_json`` / ``is_coco``), autolabelling (``save_hybrid``), augmented inference, plots and the
confusion matrix (``plots=True`` logs a warning and draws nothing; it never changes the metrics) and W&B media.

The KAIST miss rate, which the reference comments out (``MRresult`` is its ten zeros), runs on the device when
``mr_annotations=`` names the annotation file (or a :class:`~icafusion_b200.kaist_eval.KaistAnnotations`): one rounding
launch per batch turns the detections into the doubles the reference reads back from its ``result.txt`` (icaf_kaist_round_
detections), and one icaf_kaist_mr after the last batch evaluates them.  ``MRresult`` is then [MR_all, ..., MR_heavy,
recall_all] as the commented reference code computes them from evaluate() on that ``result.txt``.
"""
from __future__ import annotations

import glob
import logging
import os
import re
from pathlib import Path

import numpy as np
import torch
import yaml

from . import ops
from .metrics import ap_per_class

logger = logging.getLogger(__name__)

NIOU = 10


def increment_path(path, exist_ok=False, sep="", mkdir=False):
    """reference: utils/general.py:705-719 -- runs/exp -> runs/exp2, runs/exp3, ... when the path exists."""
    path = Path(path)
    if path.exists() and not exist_ok:
        suffix = path.suffix
        path = path.with_suffix("")
        found = [re.search(rf"%s{sep}(\d+)" % path.stem, d) for d in glob.glob(f"{path}{sep}*")]
        idx = [int(m.groups()[0]) for m in found if m]
        path = Path(f"{path}{sep}{max(idx) + 1 if idx else 2}{suffix}")
    d = path if path.suffix == "" else path.parent
    if not d.exists() and mkdir:
        d.mkdir(parents=True, exist_ok=True)
    return path


def ratio_pad_rows(shapes):
    """The loader's shapes[i] = ((h0, w0), ((gain, _), (padw, padh))) -> fp32 (B, 5) rows [h0, w0, gain, padw, padh]."""
    return torch.tensor([[s[0][0], s[0][1], s[1][0][0], s[1][1][0], s[1][1][1]] for s in shapes], dtype=torch.float32)


def label_classes(targets, nb):
    """tcls of test.py:147 for each image of a batch, from host-side targets [image, cls, ...]."""
    t = targets.detach().cpu()
    return [t[t[:, 0] == si, 1].tolist() for si in range(nb)]


def append_txt(labels_dir, stem, index, native, conf, save_conf=True):
    """test.py:163-170 for one image: one line (index + 1, x1, y1, w, h[, conf]) per detection in %g format."""
    xywh = native.copy()
    xywh[:, 2] = native[:, 2] - native[:, 0]            # xyxy2xywh2 in fp32, general.py:312-319
    xywh[:, 3] = native[:, 3] - native[:, 1]
    with open(Path(labels_dir) / (stem + ".txt"), "a") as f:
        for box, c in zip(xywh.tolist(), conf.tolist()):
            line = (index + 1, *box, c) if save_conf else (index + 1, *box)
            f.write(("%g," * len(line)).rstrip(",") % line + "\n")


def write_result_txt(labels_dir):
    """test.py:248-258: every per-image file of labels_dir, in sorted name order, concatenated into result.txt."""
    lines = []
    for name in sorted(os.listdir(labels_dir)):
        with open(Path(labels_dir) / name, "r") as f:
            lines.extend(f)
    with open(Path(labels_dir) / "result.txt", "a") as f:
        f.writelines(lines)


def mr_positions(kaist, labels_list, paths, seen):
    """int32 (B,) annotation-image positions of a batch's images (image id = the label file's index in labels_list, as
    test.py's result lines number them); each image may come once."""
    pos = []
    for p in paths:
        i = labels_list.index(Path(p).stem + ".txt")
        if i not in kaist.position:
            raise ValueError(f"test: image {Path(p).name} (id {i}) is not in the KAIST annotations {kaist.path}")
        if i in seen:
            raise ValueError(f"test: image {Path(p).name} (id {i}) is validated twice; the miss rate takes each image once")
        seen.add(i)
        pos.append(kaist.position[i])
    return torch.tensor(pos, dtype=torch.int32)


def kaist_mr_result(ys, counts):
    """MRresult of the reference's commented KAIST code: [MR_all, ..., MR_heavy, recall_all], recall_all 0.0 where `all`
    keeps no detection (the reference's line raises there)."""
    from .kaist_eval import SETUP_OF, log_average, recall_all
    mrs = [float(log_average(ys[e])) for e in range(len(SETUP_OF))]
    r = recall_all(ys, counts)
    return mrs + [0.0 if r is None else r]


def summarise(stats, nc, names, seen, verbose=False, mr_result=(0.0,) * 10):
    """test.py:287-312 on the gathered statistics [(correct bool (n, niou), conf fp32 (n), pcls fp32 (n), tcls list)] of the
    images the reference appends.  Returns (tp, fp, fn, f1, mp, mr, map50, map, maps) as the reference computes them.
    mr_result: the ten MRresult values the log line prints (x 100)."""
    p = r = f1 = mp = mr = map50 = map75 = 0.0
    mean_ap = 0
    tp, fp, fn = 0, 0, 0
    ap_class = []
    stats = [np.concatenate(x, 0) for x in zip(*stats)]
    if len(stats) and stats[0].any():
        tp, fp, fn, p, r, ap, f1, ap_class = ap_per_class(*stats)
        ap50, ap75, ap = ap[:, 0], ap[:, 5], ap.mean(1)
        mp, mr, map50, map75, mean_ap = p.mean(), r.mean(), ap50.mean(), ap75.mean(), ap.mean()
        nt = np.bincount(stats[3].astype(np.int64), minlength=nc)
    else:
        nt = np.zeros(1)
    if not isinstance(tp, int):            # the reference returns (and with nc == 1 prints) the first class's values
        tp, fp, fn, f1 = tp[0], fp[0], fn[0], f1[0]
    if nc > 1:
        pf = "%20s" + "%12i" * 2 + "%12.3g" * 5
        logger.info(pf % ("all", seen, nt.sum(), mp, mr, map50, map75, mean_ap))
    else:
        pf = "%20s" + "%12i" * 2 + "%12.4g" * 8
        logger.info(pf % ("all", seen, nt.sum(), tp, fp, fn, f1, mp, mr, map50, mean_ap))
    logger.info(("%20s" + "%11s" * 9) % ("MR-all", "MR-day", "MR-night", "MR-near", "MR-medium", "MR-far", "MR-none",
                                         "MR-partial", "MR-heavy", "Recall-all"))
    logger.info(("%20.2f" + "%11.2f" * 9) % tuple(v * 100 for v in mr_result))
    if verbose and nc > 1 and len(stats):
        for i, c in enumerate(ap_class):
            logger.info(pf % (names[c], seen, nt[c], p[i], r[i], ap50[i], ap75[i], ap[i]))
    maps = np.zeros(nc) + mean_ap
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    return (tp, fp, fn, f1, mp, mr, map50, mean_ap), maps


def test(data,
         weights=None,
         batch_size=32,
         imgsz=640,
         conf_thres=0.001,
         iou_thres=0.5,
         save_json=False,
         single_cls=False,
         augment=False,
         verbose=False,
         model=None,
         dataloader=None,
         save_dir=Path(""),
         save_txt=False,
         save_hybrid=False,
         save_conf=True,
         plots=False,
         wandb_logger=None,
         compute_loss=None,
         half_precision=True,
         is_coco=False,
         opt=None,
         labels_list=None,
         mr_annotations=None,
         graphs=None,
         group=None):
    """reference: test.py:23-367, the path train.py takes (``model=`` an eval-mode CUDA Model, ``dataloader=`` batches of
    (img uint8 (B, 6, H, W), targets (T, 6), paths, shapes)).  The model is not cast: it runs in the precision it has.
    mr_annotations: a KAIST annotation file or KaistAnnotations; image i of labels_list is the file's image id i.
    graphs: an :class:`~icafusion_b200.engine.ValidationGraphs` of ``model``, kept for the whole run: the batch loop then
    replays CUDA graphs, with the filters refreshed in place from the model's current weights.  The results are the same;
    ``t``'s inference time then includes the validation loss.
    group: a torch.distributed process group of W > 1 ranks, every one calling test.test with the same arguments (each with
    ``graphs=`` of its own model copy, if any): the batches are split over the ranks (see :func:`owned_batches`), their
    per-image results are exchanged and merged on the device, and every rank returns exactly what one process returns,
    except the times in ``t``, which sum every rank's batches.  A :class:`~icafusion_b200.valdata.ValBatches` loader
    stages only the rank's own batches; any other iterable is iterated in full on every rank (each rank pays the loader's
    cost of every batch) and the other ranks' batches are skipped."""
    if model is None or dataloader is None:
        raise NotImplementedError("test: only the train.py path (model= and dataloader=) is built; the command-line path "
                                  "(weights=, attempt_load, a loader made from opt) is not")
    if save_json or is_coco:
        raise NotImplementedError("test: the pycocotools JSON evaluation (save_json / is_coco) is not built")
    if save_hybrid:
        raise NotImplementedError("test: autolabelling (save_hybrid, NMS labels=) is not built")
    if augment:
        raise NotImplementedError("test: augmented inference is not built")
    if plots:
        logger.warning("test: plots=True draws nothing here (no plots, no confusion matrix); the metrics are unaffected")
    if group is not None and _world(group) > 1:
        return _test_sharded(group, data, batch_size, imgsz, conf_thres, iou_thres, single_cls, verbose, model, dataloader,
                             save_dir, save_txt, save_conf, compute_loss, labels_list, mr_annotations, graphs)
    device = next(model.parameters()).device
    if graphs is not None:
        graphs.check(model, device)
    if device.type != "cuda" and not (ops.dry_running() and device.type == "meta"):
        raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
    kaist = None
    if mr_annotations is not None:
        from .kaist_eval import KaistAnnotations
        if labels_list is None:
            raise ValueError("test: mr_annotations= needs labels_list (a detection's image id is its label file's index)")
        kaist = mr_annotations if isinstance(mr_annotations, KaistAnnotations) else KaistAnnotations(mr_annotations, device)
        if kaist.device != device:
            raise ValueError(f"test: mr_annotations are on {kaist.device}, the model on {device}")
        mr_rows = mr_span = None
        mr_seen = set()
    save_dir = Path(save_dir)
    (save_dir / "labels" if save_txt else save_dir).mkdir(parents=True, exist_ok=True)
    labels_dir = increment_path(save_dir / "labels" / "pred", exist_ok=False, mkdir=True) if save_txt else None

    model.eval()
    if isinstance(data, str):
        with open(data) as f:
            data = yaml.safe_load(f)
    nc = 1 if single_cls else int(data["nc"])
    iouv = torch.linspace(0.5, 0.95, NIOU).to(device)          # made on the CPU, as test.py:85 does
    names = {k: v for k, v in enumerate(model.names if hasattr(model, "names") else model.module.names)}

    loss = torch.zeros(4, device=device)
    if graphs is not None:
        loss = graphs.begin(iouv, (conf_thres, iou_thres, single_cls, compute_loss, save_txt or kaist is not None, kaist))
    batches, timers = [], []
    for img, targets, paths, shapes in dataloader:
        entry = graphs.entry(img, targets.shape[0]) if graphs is not None else None
        if entry is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            image = None
            if kaist is not None:
                if mr_rows is None:
                    mr_rows, mr_span = graphs.kaist_buffers(kaist)
                image = mr_positions(kaist, labels_list, paths, mr_seen)
            det, count, correct, native = entry.run(img, targets, ratio_pad_rows(shapes), image, ev)
            timers.append(ev)
            batches.append((det, count, correct, native if save_txt else None, [Path(p) for p in paths],
                            label_classes(targets, img.shape[0])))
            continue
        img = img.to(device, non_blocking=True)
        targets_dev = targets.to(device, torch.float32, non_blocking=True).contiguous()
        nb, _, height, width = img.shape
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.no_grad():
            ev[0].record()
            out, _, train_out = model(img[:, :3], img[:, 3:])
            ev[1].record()
            if compute_loss:
                loss += compute_loss([x.float() for x in train_out], targets_dev)[1][:4]
            ev[2].record()
            z = out if out.dtype == torch.float16 else out.half()
            det, count = ops.nms(z.contiguous(), conf_thres, iou_thres, agnostic=single_cls, multi_label=True)
            ev[3].record()
            ratio_pad = ratio_pad_rows(shapes).pin_memory().to(device, non_blocking=True)
            need_native = save_txt or kaist is not None
            native = torch.empty(nb, det.shape[1], 4, dtype=torch.float32, device=device) if need_native else None
            correct, _ = ops.match_detections(det, count, targets_dev, ratio_pad, height, width, iouv, single_cls,
                                              native=native)
            if kaist is not None:
                if mr_rows is None and graphs is not None:      # the buffers the captured batches write
                    mr_rows, mr_span = graphs.kaist_buffers(kaist)
                elif mr_rows is None:
                    mr_rows = torch.empty(kaist.images * det.shape[1], 5, dtype=torch.float64, device=device)
                    mr_span = torch.zeros(kaist.images, 2, dtype=torch.int32, device=device)
                image = mr_positions(kaist, labels_list, paths, mr_seen)
                ops.kaist_round_detections(native, det, count, image.pin_memory().to(device, non_blocking=True), mr_rows,
                                           mr_span)
        timers.append(ev)
        batches.append((det, count, correct, native if save_txt else None, [Path(p) for p in paths],
                        label_classes(targets, nb)))
    mr_out = None
    if kaist is not None and mr_rows is not None:
        from .kaist_eval import DAY_IMAGES
        mr_out = ops.kaist_mr(kaist, mr_rows, mr_span, int(mr_rows.shape[0] // kaist.images), DAY_IMAGES)

    torch.cuda.synchronize()
    t0 = sum(e[0].elapsed_time(e[1]) for e in timers) / 1e3
    t1 = sum(e[2].elapsed_time(e[3]) for e in timers) / 1e3
    stats, seen = [], 0
    for det, count, correct, native, paths, tcls in batches:
        det, count, correct = det.cpu().numpy(), count.cpu().tolist(), correct.cpu().numpy().astype(bool)
        native = native.cpu().numpy() if native is not None else None
        for si, n in enumerate(count):
            seen += 1
            if n == 0:
                if tcls[si]:
                    stats.append((np.zeros((0, NIOU), dtype=bool), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls[si]))
                continue
            pcls = np.zeros(n, np.float32) if single_cls else det[si, :n, 5]
            if save_txt:
                append_txt(labels_dir, paths[si].stem, labels_list.index(paths[si].stem + ".txt"), native[si, :n],
                           det[si, :n, 4], save_conf)
            stats.append((correct[si, :n], det[si, :n, 4], pcls, tcls[si]))
    if save_txt:
        write_result_txt(labels_dir)

    mr_result = [0.0] * 10
    if mr_out is not None:
        mr_result = kaist_mr_result(mr_out[0].cpu().numpy(), mr_out[1].cpu().numpy())
    results, maps = summarise(stats, nc, names, seen, verbose, mr_result)
    t = tuple(x / max(seen, 1) * 1e3 for x in (t0, t1, t0 + t1)) + (imgsz, imgsz, batch_size)
    return (*results, *(loss.cpu() / len(dataloader)).tolist()), maps, mr_result, t


# ------------------------------------------------------------------------------------------------------------------------
# Validation sharded over the ranks of a process group
def _world(group) -> int:
    import torch.distributed as dist
    return dist.get_world_size(group)


def owned_batches(n_batches: int, rank: int, world: int) -> range:
    """The global batches rank `rank` of `world` runs: j = rank (mod world), which spreads the rect batch shapes evenly."""
    if not 0 <= rank < world:
        raise ValueError(f"test: rank {rank} outside a world of {world}")
    return range(rank, n_batches, world)


def _owned(dataloader, rank, world, total):
    """(j, global index of the batch's first image, batch) of this rank's batches; total[0] gets the loader's image count."""
    from .valdata import ValBatches
    if isinstance(dataloader, ValBatches):
        total[0] = len(dataloader.order)
        yield from dataloader.shard(rank, world)
        return
    n = 0
    for j, batch in enumerate(dataloader):
        if j % world == rank:
            yield j, n, batch
        n += int(batch[0].shape[0])
    total[0] = n


def _gather_objects(obj, group) -> list:
    import torch.distributed as dist
    out = [None] * dist.get_world_size(group)
    dist.all_gather_object(out, obj, group=group)
    return out


def _test_sharded(group, data, batch_size, imgsz, conf_thres, iou_thres, single_cls, verbose, model, dataloader, save_dir,
                  save_txt, save_conf, compute_loss, labels_list, mr_annotations, graphs):
    """test() over the ranks of `group`: each rank runs its own batches, packs their per-image results (icaf_val_pack), the
    buffers are all-gathered, and rank 0 merges them in global image order (icaf_val_merge) and runs the one-process tail
    on the same arrays, so every metric, the loss and the files are those of one process.  The result is broadcast."""
    import torch.distributed as dist
    from .engine import ValidationGraphs
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    device = next(model.parameters()).device
    problem = None
    if graphs is not None:
        try:
            graphs.check(model, device)
        except ValueError as e:
            problem = str(e)
    got = _gather_objects((len(dataloader), problem), group)      # before any launch: every rank refuses together
    for _, p in got:
        if p:
            raise ValueError(p)
    if len({n for n, _ in got}) != 1:
        raise ValueError(f"test: the dataloader holds {[n for n, _ in got]} batches on ranks 0..{world - 1}; a sharded call "
                         "needs the same loader on every rank")
    if device.type != "cuda":
        raise RuntimeError("icafusion_b200 runs on CUDA tensors only (no CPU fallback)")
    kaist = None
    if mr_annotations is not None:
        from .kaist_eval import KaistAnnotations
        if labels_list is None:
            raise ValueError("test: mr_annotations= needs labels_list (a detection's image id is its label file's index)")
        kaist = mr_annotations if isinstance(mr_annotations, KaistAnnotations) else KaistAnnotations(mr_annotations, device)
        if kaist.device != device:
            raise ValueError(f"test: mr_annotations are on {kaist.device}, the model on {device}")
    labels_dir = None
    if rank == 0:
        save_dir = Path(save_dir)
        (save_dir / "labels" if save_txt else save_dir).mkdir(parents=True, exist_ok=True)
        labels_dir = increment_path(save_dir / "labels" / "pred", exist_ok=False, mkdir=True) if save_txt else None

    model.eval()
    if isinstance(data, str):
        with open(data) as f:
            data = yaml.safe_load(f)
    nc = 1 if single_cls else int(data["nc"])
    iouv = torch.linspace(0.5, 0.95, NIOU).to(device)
    names = {k: v for k, v in enumerate(model.names if hasattr(model, "names") else model.module.names)}
    need_native = save_txt or kaist is not None
    max_det = ValidationGraphs.max_det

    n_batches = len(dataloader)
    own = owned_batches(n_batches, rank, world)
    rows = torch.zeros(len(own), 4, device=device) if compute_loss else None       # loss items per batch this rank runs
    if graphs is not None:
        graphs.begin(iouv, (conf_thres, iou_thres, single_cls, compute_loss, need_native, kaist), per_batch=True)
    batches, timers, images, positions, js = [], [], [], [], []
    total, mr_seen, mr_rows = [0], set(), None
    try:
        for k, (j, image0, (img, targets, paths, shapes)) in enumerate(_owned(dataloader, rank, world, total)):
            image = mr_positions(kaist, labels_list, paths, mr_seen) if kaist is not None else None
            entry = graphs.entry(img, targets.shape[0]) if graphs is not None else None
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            nb = img.shape[0]
            if entry is not None:
                if kaist is not None and mr_rows is None:
                    mr_rows = graphs.kaist_buffers(kaist)
                det, count, correct, native = entry.run(img, targets, ratio_pad_rows(shapes), image, ev,
                                                        loss_row=rows[k] if rows is not None else None)
            else:
                img = img.to(device, non_blocking=True)
                targets_dev = targets.to(device, torch.float32, non_blocking=True).contiguous()
                _, _, height, width = img.shape
                with torch.no_grad():
                    ev[0].record()
                    out, _, train_out = model(img[:, :3], img[:, 3:])
                    if compute_loss:
                        rows[k].copy_(compute_loss([x.float() for x in train_out], targets_dev)[1][:4])
                    ev[1].record()
                    ev[2].record()
                    z = out if out.dtype == torch.float16 else out.half()
                    det, count = ops.nms(z.contiguous(), conf_thres, iou_thres, agnostic=single_cls, multi_label=True,
                                         max_det=max_det)
                    ev[3].record()
                    ratio_pad = ratio_pad_rows(shapes).pin_memory().to(device, non_blocking=True)
                    native = torch.empty(nb, det.shape[1], 4, dtype=torch.float32, device=device) if need_native else None
                    correct, _ = ops.match_detections(det, count, targets_dev, ratio_pad, height, width, iouv, single_cls,
                                                      native=native)
            timers.append(ev)
            batches.append((det, count, correct, native if need_native else None, image0))
            tcls = label_classes(targets, nb)
            images += [(image0 + si, Path(p).stem, tcls[si]) for si, p in enumerate(paths)]
            if image is not None:
                positions += image.tolist()
            js.append(j)
    except ValueError as e:                         # e.g. an image outside the KAIST annotations: refused on every rank
        problem = str(e)
    payload = None
    if problem is None and batches:
        payload = ops.val_pack(batches, NIOU, native=need_native, positions=positions if kaist is not None else None)
    torch.cuda.synchronize()
    head = payload[:4].cpu().tolist() if payload is not None else [0, 0, 3 + 4 * need_native, 4]
    t0 = sum(e[0].elapsed_time(e[1]) for e in timers) / 1e3
    t1 = sum(e[2].elapsed_time(e[3]) for e in timers) / 1e3
    loss_rows = list(zip(js, rows.cpu().numpy())) if rows is not None else []
    info = _gather_objects(dict(problem=problem, head=head, images=images, positions=positions, loss=loss_rows, t=(t0, t1),
                                total=total[0]), group)
    for i in info:
        if i["problem"]:
            raise ValueError(i["problem"])

    width = max(i["head"][3] for i in info)
    buf = torch.zeros(width, dtype=torch.int32, device=device)
    if payload is not None:
        buf[:head[3]].copy_(payload[:head[3]])
    else:
        buf[:4].copy_(torch.tensor(head, dtype=torch.int32))
    gathered = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(gathered, buf, group=group)

    result = None
    if rank == 0:
        try:
            result = _sharded_tail(torch.stack(gathered), info, nc, names, single_cls, verbose, need_native, kaist, labels_list,
                                   labels_dir, save_txt, save_conf, imgsz, batch_size, n_batches, max_det)
        except ValueError as e:
            result = e
    box = [result]
    dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not dist.group.WORLD else 0, group=group)
    if isinstance(box[0], Exception):
        raise box[0]
    return box[0]


def _sharded_tail(bufs, info, nc, names, single_cls, verbose, need_native, kaist, labels_list, labels_dir, save_txt, save_conf,
                  imgsz, batch_size, n_batches, max_det):
    """Rank 0's part of a sharded test(): merge the ranks' buffers and run the one-process tail on the merged arrays."""
    n_images = info[0]["total"]
    meta = {}
    for i in info:
        for g, stem, tc in i["images"]:
            meta[g] = (stem, tc)
    if kaist is not None:
        pos = [p for i in info for p in i["positions"]]
        if len(set(pos)) != len(pos):
            dup = sorted({p for p in pos if pos.count(p) > 1})[0]
            raise ValueError(f"test: an image at KAIST position {dup} is validated twice; the miss rate takes each image once")
    n_rows = sum(i["head"][1] for i in info)
    stats, seen, mr_result = [], 0, [0.0] * 10
    if n_images:
        m = ops.val_merge(bufs, n_images, n_rows, NIOU, native=need_native,
                          mr=(kaist.images, max_det) if kaist is not None and meta else None)
        mr_out = None
        if m["mr_rows"] is not None:
            from .kaist_eval import DAY_IMAGES
            mr_out = ops.kaist_mr(kaist, m["mr_rows"], m["mr_span"], max_det, DAY_IMAGES)
        status = m["status"].cpu().tolist()
        ops.val_merge_check(status, n_rows)
        counts, offsets = m["counts"].cpu().tolist(), m["offsets"].cpu().tolist()
        correct, conf, pcls = m["correct"].cpu().numpy().astype(bool), m["conf"].cpu().numpy(), m["pcls"].cpu().numpy()
        native = m["native"].cpu().numpy() if m["native"] is not None else None
        for k in range(n_images):
            n, o = counts[k], offsets[k]
            stem, tc = meta[k]
            seen += 1
            if n == 0:
                if tc:
                    stats.append((np.zeros((0, NIOU), dtype=bool), np.zeros(0, np.float32), np.zeros(0, np.float32), tc))
                continue
            pc = np.zeros(n, np.float32) if single_cls else pcls[o:o + n]
            if save_txt:
                append_txt(labels_dir, stem, labels_list.index(stem + ".txt"), native[o:o + n], conf[o:o + n], save_conf)
            stats.append((correct[o:o + n], conf[o:o + n], pc, tc))
        if mr_out is not None:
            mr_result = kaist_mr_result(mr_out[0].cpu().numpy(), mr_out[1].cpu().numpy())
    if save_txt:
        write_result_txt(labels_dir)
    results, maps = summarise(stats, nc, names, seen, verbose, mr_result)
    loss = np.zeros(4, np.float32)
    for _, row in sorted(r for i in info for r in i["loss"]):    # the one-process call's fp32 adds, in batch order
        loss = loss + row
    t0, t1 = (sum(i["t"][0] for i in info), sum(i["t"][1] for i in info))
    t = tuple(x / max(seen, 1) * 1e3 for x in (t0, t1, t0 + t1)) + (imgsz, imgsz, batch_size)
    return (*results, *(torch.from_numpy(loss) / n_batches).tolist()), maps, mr_result, t
