"""KAIST log-average miss rate on the device: a drop-in for the reference's ``evaluation_script.evaluation_script``.

``evaluate(test_annotation_file, user_submission_file)`` returns what the reference's ``evaluate`` returns: a dict of the
nine evaluations (all, day, night, near, medium, far, none, partial, heavy), each with ``summarize(id_setup)`` and ``eval``
(``'TP'`` of shape (1, 9, 1, 1), the fppi / miss-rate curves ``'xx'`` / ``'yy'``, ``'counts'``, ``'params'``), with the
reference's numbers bit for bit.  The per-image matching and the accumulation run in one ``icaf_kaist_mr`` call; the host
only parses the file and takes the log-average of 81 numbers.  ``KaistAnnotations`` keeps the annotation arrays on the
device, so a training run loads them once (``test.test(..., mr_annotations=...)``).

Not built: the miss-rate plots (``draw_all``, ``KAISTPedEval.draw_figure``) need matplotlib.  A file with more than 1,000
detections in one image is refused: the reference's evaluateImg indexes past its IoU rows there.
"""
from __future__ import annotations

import datetime
import gzip
import json
import os
from typing import Optional

import numpy as np
import torch

from . import ops

EVALS = ("all", "day", "night", "near", "medium", "far", "none", "partial", "heavy")
SETUP_OF = (0, 0, 0, 1, 2, 3, 4, 5, 6)
DAY_IMAGES = 1455              # evaluate(): imgIds[:1455] is `day`, the rest `night`


class KAISTParams:
    """The reference's KAISTParams for bbox evaluation (the values its summarize and accumulate read)."""

    def __init__(self, img_ids=()):
        self.imgIds = list(img_ids)
        self.catIds = [1]
        self.iouThrs = np.array([0.5])
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1000]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'small', 'medium', 'large']
        self.useCats = 1
        self.fppiThrs = np.array([0.0100, 0.0178, 0.0316, 0.0562, 0.1000, 0.1778, 0.3162, 0.5623, 1.0000])
        self.HtRng = [[55, 1e5 ** 2], [115, 1e5 ** 2], [45, 115], [1, 45], [1, 1e5 ** 2], [1, 1e5 ** 2], [1, 1e5 ** 2]]
        self.OccRng = [[0, 1], [0], [0], [0], [0], [1], [2]]
        self.SetupLbl = ['Reasonable', 'scale=near', 'scale=medium', 'scale=far', 'occ=none', 'occ=partial', 'occ=heavy', 'All']
        self.bndRng = [5, 5, 635, 507]
        self.iouType = 'bbox'
        self.useSegm = None


def _open(path):
    path = os.fspath(path)
    return gzip.open(path, "rt") if path.endswith(".gz") else open(path)


class KaistAnnotations:
    """The gts of a KAIST annotation file (category 1, as the reference evaluates them) on `device`: per image (images in
    ascending id order) in file order, box float64 (G, 4), height float64 (G,), occlusion int32 (-1 for a value outside
    0..2), ignore int32 (the file's flag), id int64, offset int32 (images + 1)."""

    def __init__(self, path, device=None):
        with _open(path) as f:
            data = json.load(f)
        self.path = os.fspath(path)
        self.image_ids = sorted(int(im["id"]) for im in data["images"])
        self.position = {i: p for p, i in enumerate(self.image_ids)}
        anns = [a for a in data["annotations"] if a["category_id"] == 1 and a["image_id"] in self.position]
        pos = np.array([self.position[a["image_id"]] for a in anns], dtype=np.int64)
        order = np.argsort(pos, kind="stable")
        anns = [anns[i] for i in order]

        def occ(v):
            v = float(v)
            return int(v) if v in (0.0, 1.0, 2.0) else -1
        box = np.array([a["bbox"] for a in anns], dtype=np.float64).reshape(-1, 4)
        height = np.array([a["height"] for a in anns], dtype=np.float64)
        occlusion = np.array([occ(a["occlusion"]) for a in anns], dtype=np.int32)
        ignore = np.array([int(bool(a.get("ignore", 0))) for a in anns], dtype=np.int32)
        ids = np.array([a["id"] for a in anns], dtype=np.int64)
        offset = np.zeros(len(self.image_ids) + 1, dtype=np.int32)
        np.cumsum(np.bincount(pos[order], minlength=len(self.image_ids)), out=offset[1:])
        self.host = dict(box=box, height=height, occlusion=occlusion, ignore=ignore, id=ids, offset=offset)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        for k, v in self.host.items():
            setattr(self, k, torch.from_numpy(v).to(self.device))

    @property
    def images(self) -> int:
        return len(self.image_ids)


def load_detections(path, ann: KaistAnnotations):
    """Parse a result file as the reference's KAIST.loadRes does (.txt lines `image_index + 1,x,y,w,h,score`, read with
    float(); .json: COCO results, category 1) -> (rows float64 (N, 5) grouped by image in image order and in file order
    within an image, span int32 (images, 2), the largest per-image count)."""
    path = os.fspath(path)
    name = path[:-3] if path.endswith(".gz") else path
    if name.endswith(".txt"):
        with _open(path) as f:
            data = np.loadtxt(f, delimiter=",", dtype=np.float64, ndmin=2)
        if data.size and data.shape[1] < 6:
            raise ValueError(f"{path}: a line has fewer than 6 values (image, x, y, w, h, score)")
        data = data.reshape(-1, data.shape[1] if data.size else 6)
        img = data[:, 0] - 1
        rows = np.ascontiguousarray(data[:, 1:6])
    elif name.endswith(".json"):
        with _open(path) as f:
            res = json.load(f)
        if not isinstance(res, list):
            raise ValueError(f"{path}: results in not an array of objects")
        res_ids = [r["image_id"] for r in res]
        res = [r for r in res if r["category_id"] == 1]
        img = np.array(res_ids, dtype=np.float64)
        rows = np.array([[*r["bbox"], r["score"]] for r in res], dtype=np.float64).reshape(-1, 5)
    else:
        raise ValueError(f"[Error] Exception extension : {name.split('.')[-1]}")
    bad = [v for v in np.unique(img) if v not in ann.position]
    if bad:
        raise ValueError(f"{path}: results do not correspond to the annotation set (image ids {bad[:5]} are not in it)")
    if name.endswith(".json"):
        img = np.array([r["image_id"] for r in res], dtype=np.float64)
    pos = np.array([ann.position[v] for v in img.tolist()], dtype=np.int64) if len(img) else np.zeros(0, np.int64)
    order = np.argsort(pos, kind="stable")
    counts = np.bincount(pos, minlength=ann.images)
    if counts.size and counts.max() > ops.KAIST_MAX_DET:
        p = int(np.argmax(counts))
        raise ValueError(f"{path}: image {ann.image_ids[p]} has {int(counts[p])} detections; the evaluation takes at most "
                         f"{ops.KAIST_MAX_DET} per image (the reference's evaluateImg fails past its maxDets)")
    span = np.zeros((ann.images, 2), dtype=np.int32)
    span[1:, 0] = np.cumsum(counts)[:-1]
    span[:, 1] = counts
    return np.ascontiguousarray(rows[order]), span, int(counts.max()) if counts.size else 0


def log_average(ys_row: np.ndarray) -> float:
    """KAISTPedEval.summarize for one evaluation: exp(mean(log(mrs + 1e-5))) over mrs = 1 - ys where ys != -1; -1 if none."""
    s = np.asarray(ys_row, dtype=np.float64).reshape(1, -1, 1, 1)
    mrs = 1 - s[:, :, :, [0]]
    if len(mrs[mrs < 2]) == 0:
        return -1
    return np.exp(np.mean(np.log(mrs[mrs < 2] + 1e-5)))


def recall_all(ys: np.ndarray, counts: np.ndarray) -> Optional[float]:
    """1 - eval['all'].eval['yy'][0][-1] of the reference, or None where its curve is missing or empty."""
    kept, tp, npig = (int(v) for v in counts[0])
    if ys[0][0] == -1 or kept == 0:
        return None
    yy_last = 1 - np.array([tp], dtype=np.float64) / npig
    return float(1 - yy_last[-1])


class KAISTPedEval:
    """One evaluation's result in the shape of the reference's KAISTPedEval after evaluate / accumulate."""

    def __init__(self, params: KAISTParams, ys_row, xx, yy, method="unknown"):
        self.params = params
        self.method = method
        self.eval = {'params': params, 'counts': [1, 9, 1, 1],
                     'date': datetime.datetime.now().strftime('%Y-%m-%d %H:%M:%S'),
                     'TP': np.asarray(ys_row, dtype=np.float64).reshape(1, 9, 1, 1).copy(), 'xx': xx, 'yy': yy}

    @staticmethod
    def draw_figure(ax, eval_results, methods, colors):
        raise NotImplementedError("KAISTPedEval.draw_figure: the miss-rate plots need matplotlib and are not built")

    def summarize(self, id_setup, res_file=None):
        p = self.params
        s = self.eval['TP'][np.where(.5 == p.iouThrs)[0]]
        mrs = 1 - s[:, :, :, [i for i, m in enumerate(p.maxDets) if m == 1000]]
        if len(mrs[mrs < 2]) == 0:
            mean_s = -1
        else:
            mean_s = np.exp(np.mean(np.log(mrs[mrs < 2] + 1e-5)))
        if res_file:
            occ = ['none', 'partial_occ', 'heavy_occ']
            res_file.write(' {:<18} {} @ {:<18} [ IoU={:<9} | height={:>6s} | visibility={:>6s} ] = {:0.2f}%'.format(
                'Average Miss Rate', '(MR)', p.SetupLbl[id_setup], '{:0.2f}'.format(0.5),
                '[{:0.0f}:{:0.0f}]'.format(p.HtRng[id_setup][0], p.HtRng[id_setup][1]),
                '[' + '+'.join(occ[o] for o in p.OccRng[id_setup]) + ']', mean_s * 100))
            res_file.write('\n')
        return mean_s


def evaluate_device(ann: KaistAnnotations, rows: torch.Tensor, span: torch.Tensor, max_per_image: int,
                    method="unknown") -> dict:
    """The nine evaluations of the detections (rows, span on ann's device; see ops.kaist_mr) -> {name: KAISTPedEval}."""
    ys, counts, curves = ops.kaist_mr(ann, rows, span, max_per_image, DAY_IMAGES, curves=True)
    ys, counts = ys.cpu().numpy(), counts.cpu().numpy()
    out = {}
    for e, name in enumerate(EVALS):
        ids = ann.image_ids[:DAY_IMAGES] if name == "day" else ann.image_ids[DAY_IMAGES:] if name == "night" else ann.image_ids
        xx, yy = [], []
        if ys[e][0] != -1:
            n = int(counts[e][0])
            c = curves[e, :, :n].cpu().numpy()
            xx, yy = [c[0].copy()], [c[1].copy()]
        out[name] = KAISTPedEval(KAISTParams(ids), ys[e], xx, yy, method)
    return out


def evaluate(test_annotation_file, user_submission_file: str, phase_codename: str = 'Multispectral', plot=False):
    """reference: evaluation_script.py:546-646.  test_annotation_file: a path (or a KaistAnnotations); the submission a
    .txt or .json result file (optionally .gz).  Returns {all, day, night, near, medium, far, none, partial, heavy}."""
    ann = test_annotation_file if isinstance(test_annotation_file, KaistAnnotations) else KaistAnnotations(test_annotation_file)
    rows, span, mx = load_detections(user_submission_file, ann)
    method = os.path.basename(os.fspath(user_submission_file)).split('_')[0]
    res = evaluate_device(ann, torch.from_numpy(rows).to(ann.device), torch.from_numpy(span).to(ann.device), mx, method)
    recall = 1 - res['all'].eval['yy'][0][-1]            # the reference's line: IndexError when nothing is kept in `all`
    if plot:
        mr = {k: res[k].summarize(s) for k, s in zip(EVALS, SETUP_OF)}
        print(f'\n########## Method: {method} ##########\n' + ''.join(f'MR_{k}: {mr[k] * 100:.2f}\n' for k in EVALS) +
              f'recall_all: {recall * 100:.2f}\n' + '######################################\n\n')
    return res


def draw_all(eval_results, filename='figure.jpg'):
    raise NotImplementedError("draw_all: the miss-rate plots need matplotlib and are not built")
