"""Generate the KAIST miss-rate goldens by executing the REAL reference's evaluation_script.evaluate (build container only;
needs /root/reference).

    python -m oracle.gen_golden_kaist_mr

Writes, under tests/golden/:
  kaist_annotation.json.gz         the reference's KAIST_annotation.json (2,252 test images, 4,254 person boxes)
  kaist_mr_<case>.txt.gz / .json.gz the detection files of every case (see CASES)
  kaist_mr_small_annotation.json.gz a 40-image KAIST-like annotation file for the test.test case (night is empty there)
  kaist_mr_cases.npz               per case: ys (9 evaluations x 9 fppi thresholds), the nine MRs, recall_all, and the
                                   length and sums of every fppi / miss-rate curve; the per-setup ignore flags that the
                                   reference's _prepare gives the real annotations; the small test.test case's MRresult and
                                   result.txt bytes.

The shipped competitor files are MLPD, MBNet and MSDS-RCNN (.txt) and MLPD (.json), whole, and ARCNN's lines with a score
of at least 0.001 (validation's default conf_thres: 19,951 of its 76,743 detections; the whole file is 1.9 MB gzip'd, too
large to keep in the repository).  The synthetic ones are seeded
(PCG64) and sit on the real annotations: MLPD with its lines shuffled (the reference's double permutation of the IoU rows
makes the result depend on the line order), a detection exactly on annotation id 0 in the `medium` setup (matched, yet a
false positive: dtMatches stores the id 0), score ties across images, only false positives, only hits on ignored regions
(no evaluation keeps a detection: the reference's recall_all line raises IndexError, so that case is recorded per
evaluation) and detections on day images only (night has no evaluated image: MR_night is -1).
"""
from __future__ import annotations

import copy
import gzip
import importlib
import json
import os
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden")
EVALS = ["all", "day", "night", "near", "medium", "far", "none", "partial", "heavy"]
SETUP_OF = [0, 0, 0, 1, 2, 3, 4, 5, 6]
ANN = "kaist_annotation.json.gz"
SMALL_ANN = "kaist_mr_small_annotation.json.gz"
SMALL_IMAGES = 40
# case -> (annotation file, detection file); the .gz detection files are written by this script
CASES = {
    "MLPD": (ANN, "kaist_mr_MLPD.txt.gz"),
    "MBNet": (ANN, "kaist_mr_MBNet.txt.gz"),
    "MSDS-RCNN": (ANN, "kaist_mr_MSDS-RCNN.txt.gz"),
    "ARCNN_conf0.001": (ANN, "kaist_mr_ARCNN_conf0.001.txt.gz"),
    "MLPD_json": (ANN, "kaist_mr_MLPD.json.gz"),
    "MLPD_shuffled": (ANN, "kaist_mr_MLPD_shuffled.txt.gz"),
    "id0_medium": (ANN, "kaist_mr_id0_medium.txt.gz"),
    "score_ties": (ANN, "kaist_mr_score_ties.txt.gz"),
    "only_fp": (ANN, "kaist_mr_only_fp.txt.gz"),
    "ignored_only": (ANN, "kaist_mr_ignored_only.txt.gz"),
    "day_only": (ANN, "kaist_mr_day_only.txt.gz"),
    "small_first_fp": (SMALL_ANN, "kaist_mr_small_first_fp.txt.gz"),
}
SHIPPED = {"MLPD": "MLPD_result.txt", "MBNet": "MBNet_result.txt", "MSDS-RCNN": "MSDS-RCNN_result.txt",
           "ARCNN_conf0.001": "ARCNN_result.txt", "MLPD_json": "MLPD_result.json"}
ARCNN_MIN_SCORE = 0.001


def golden_path(name):
    return os.path.join(OUT, name)


def read_gz(name) -> bytes:
    with gzip.open(golden_path(name), "rb") as f:
        return f.read()


def gunzip_to(name, directory) -> str:
    """Decompress a golden file into `directory` (same name without .gz) and return the path."""
    path = os.path.join(str(directory), name[:-3])
    with open(path, "wb") as f:
        f.write(read_gz(name))
    return path


def _line(img, box, score):
    return "%d,%.4f,%.4f,%.4f,%.4f,%.6f\n" % (img + 1, *box, score)


def _by_image(anns):
    out = {}
    for a in anns:
        out.setdefault(a["image_id"], []).append(a)
    return out


def _overlaps_any(box, gts):
    x, y, w, h = box
    for a in gts:
        gx, gy, gw, gh = a["bbox"]
        if min(x + w, gx + gw) > max(x, gx) and min(y + h, gy + gh) > max(y, gy):
            return True
    return False


def synthetic_files(ann):
    """{case: file text} of the synthetic cases on the real annotations (seeded)."""
    g = np.random.Generator(np.random.PCG64(31))
    by_img = _by_image(ann["annotations"])
    n_img = len(ann["images"])
    jitter = lambda b, s: [b[0] + g.normal(0, s * b[2]), b[1] + g.normal(0, s * b[3]), b[2] * np.exp(g.normal(0, s)),
                           b[3] * np.exp(g.normal(0, s))]
    out = {}
    # a detection exactly on annotation 0 (regular in `medium`: height 50, occlusion 0), among ordinary hits and misses
    lines = [_line(0, ann["annotations"][0]["bbox"], 0.95)]
    for a in ann["annotations"][1:600]:
        if g.uniform() < 0.8:
            lines.append(_line(a["image_id"], jitter(a["bbox"], 0.08), g.uniform(0.05, 0.99)))
    for i in range(0, n_img, 7):
        lines.append(_line(i, [g.uniform(0, 600), g.uniform(0, 460), 20, 45], g.uniform(0.0, 0.6)))
    out["id0_medium"] = lines
    # scores from a set of five values: ties inside and across images, hits and misses alike
    lines = []
    for i in range(0, n_img, 3):
        for a in by_img.get(i, []):
            lines.append(_line(i, jitter(a["bbox"], 0.1), g.choice([0.3, 0.5, 0.7, 0.8, 0.9])))
        for _ in range(int(g.integers(0, 3))):
            lines.append(_line(i, [g.uniform(0, 600), g.uniform(0, 460), 22, 50], g.choice([0.3, 0.5, 0.7, 0.8, 0.9])))
    out["score_ties"] = lines
    # boxes that touch no annotation at all: every kept detection is a false positive
    lines = []
    for i in range(0, n_img, 2):
        for _ in range(int(g.integers(1, 4))):
            for _try in range(50):
                b = [g.uniform(0, 600), g.uniform(0, 460), g.uniform(8, 40), g.uniform(16, 80)]
                if not _overlaps_any(b, by_img.get(i, [])):
                    lines.append(_line(i, b, g.uniform(0.01, 0.99)))
                    break
    out["only_fp"] = lines
    # exactly on the boxes the annotation file marks ignore = 1 (ignored in every setup): nothing is ever kept
    out["ignored_only"] = [_line(a["image_id"], a["bbox"], g.uniform(0.1, 0.9)) for a in ann["annotations"] if a["ignore"]]
    # day images only (ids < 1455): the night evaluation has no image with a detection
    lines = []
    for a in ann["annotations"]:
        if a["image_id"] < 1455 and g.uniform() < 0.7:
            lines.append(_line(a["image_id"], jitter(a["bbox"], 0.1), g.uniform(0.05, 0.99)))
    for i in range(0, 1455, 5):
        lines.append(_line(i, [g.uniform(0, 600), g.uniform(0, 460), 20, 45], g.uniform(0.0, 0.5)))
    out["day_only"] = lines
    return {k: "".join(v) for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------------------------
# The small KAIST-like set for the test.test case: 40 images (fewer than 1,455, so `night` evaluates no image), 24 of them
# in six batches of four through the reference's test.test with a stub detector; the other 16 have annotations only.
def build_small(seed=37):
    """(batches [(z16, targets, shapes, paths)], labels_list, annotation dict) for the small test.test case."""
    from oracle.gen_golden_val import H, W, _batch
    g = np.random.Generator(np.random.PCG64(seed))
    plain = ((512, 640), ((1.0, 1.0), (16.0, 16.0)))
    batches = []
    for k in range(6):
        z, tg = _batch(g, 1, 4, 256, special=(k == 2))
        batches.append((z, tg, [plain] * 4, [f"/data/kaist/images/set_{k:02d}_{i}.jpg" for i in range(4)]))
    stems = [Path(p).stem + ".txt" for _, _, _, paths in batches for p in paths]
    labels_list = sorted(stems + [f"other_{k:03d}.txt" for k in range(SMALL_IMAGES - len(stems))])
    anns = []

    def add(img, x1, y1, w, h):
        anns.append({"id": len(anns), "image_id": img, "category_id": 1, "bbox": [x1, y1, w, h], "height": h,
                     "occlusion": int(g.integers(0, 3)), "ignore": int(g.uniform() < 0.15)})
    for z, tg, shapes, paths in batches:
        for si, p in enumerate(paths):
            img = labels_list.index(Path(p).stem + ".txt")
            for r in tg[tg[:, 0] == si]:
                cx, cy, w, h = float(r[2]) * W - 16, float(r[3]) * H - 16, float(r[4]) * W, float(r[5]) * H
                add(img, round(cx - w / 2, 3), round(cy - h / 2, 3), round(w, 3), round(h, 3))
    for img, name in enumerate(labels_list):
        if name.startswith("other_"):
            for _ in range(int(g.integers(0, 3))):
                add(img, round(g.uniform(10, 560), 3), round(g.uniform(10, 380), 3), 30.0, round(g.uniform(20, 110), 3))
    ann = {"images": [{"id": i, "im_name": n[:-4], "height": 512, "width": 640} for i, n in enumerate(labels_list)],
           "annotations": anns, "categories": [{"id": 0, "name": "__ignore__"}, {"id": 1, "name": "person"}]}
    return batches, labels_list, ann


def small_first_fp(ann):
    """On the small set: the best-scoring kept detection is a false positive, so at fppi thresholds below 1/40 the
    reference's searchsorted index is -1 and it reads the LAST recall."""
    g = np.random.Generator(np.random.PCG64(41))
    lines = [_line(0, [600.0, 2.0, 10.0, 20.0], 0.999)]
    for a in ann["annotations"]:
        if not a["ignore"] and g.uniform() < 0.8:
            b = a["bbox"]
            lines.append(_line(a["image_id"], [b[0] + 0.5, b[1] + 0.5, b[2], b[3]], g.uniform(0.1, 0.9)))
    return "".join(lines)


# ---------------------------------------------------------------------------------------------------------------------
def load_reference_eval():
    """The reference's evaluation_script.evaluation_script (matplotlib stubbed, rc included)."""
    from oracle.gen_golden_val import load_reference_test
    load_reference_test()
    return importlib.import_module("evaluation_script.evaluation_script")


def run_reference(E, ann_path, det_path):
    """{ys (9, 9), mr (9,), recall_all, xx_len, xx_sum, yy_sum, raises} from the reference's evaluate().  When evaluate()
    raises at its recall_all line (no kept detection in `all`), the nine evaluations are run one by one as evaluate() runs
    them, and recall_all is NaN."""
    try:
        res = E.evaluate(ann_path, det_path)
        raises = ""
        recall_all = 1 - res["all"].eval["yy"][0][-1]
    except IndexError as e:
        raises = "IndexError"
        kaistGt = E.KAIST(ann_path)
        kaistDt = kaistGt.loadRes(det_path)
        imgIds = sorted(kaistGt.getImgIds())
        ev = E.KAISTPedEval(kaistGt, kaistDt, "bbox", "x")
        ev.params.catIds = [1]
        res = {k: copy.deepcopy(ev) for k in EVALS}
        for k, s in zip(EVALS, SETUP_OF):
            res[k].params.imgIds = imgIds[:1455] if k == "day" else imgIds[1455:] if k == "night" else imgIds
            res[k].evaluate(s)
            res[k].accumulate()
        recall_all = float("nan")
        print("   (evaluate raised", type(e).__name__, e, ")")
    ys = np.stack([res[k].eval["TP"].reshape(9) for k in EVALS])
    mr = np.array([res[k].summarize(s) for k, s in zip(EVALS, SETUP_OF)], dtype=np.float64)
    xx_len = np.array([len(res[k].eval["xx"][0]) if res[k].eval["xx"] else -1 for k in EVALS])
    xx_sum = np.array([float(np.sum(res[k].eval["xx"][0])) if res[k].eval["xx"] else 0.0 for k in EVALS])
    yy_sum = np.array([float(np.sum(res[k].eval["yy"][0])) if res[k].eval["yy"] else 0.0 for k in EVALS])
    return dict(ys=ys, mr=mr, recall_all=np.float64(recall_all), xx_len=xx_len, xx_sum=xx_sum, yy_sum=yy_sum), raises


def ignore_flags(E, ann_path):
    """(7, n_annotations) uint8: the `ignore` flag _prepare(setup) gives each annotation (by annotation id)."""
    kaistGt = E.KAIST(ann_path)
    n = len(kaistGt.dataset["annotations"])
    out = np.zeros((7, n), np.uint8)
    for s in range(7):
        ev = E.KAISTPedEval(copy.deepcopy(kaistGt), copy.deepcopy(kaistGt), "bbox", "x")
        ev.params.catIds = [1]
        ev.params.imgIds = sorted(kaistGt.getImgIds())
        ev._prepare(s)
        for gts in ev._gts.values():
            for gt in gts:
                out[s, gt["id"]] = gt["ignore"]
    return out


def write_gz(name, data: bytes):
    with open(golden_path(name), "wb") as f:
        with gzip.GzipFile(fileobj=f, mode="wb", compresslevel=9, mtime=0) as z:
            z.write(data)


def main():
    from oracle.ref_shim import REF_ROOT
    E = load_reference_eval()
    sota = os.path.join(REF_ROOT, "evaluation_script", "state_of_arts")
    ann_bytes = open(os.path.join(REF_ROOT, "evaluation_script", "KAIST_annotation.json"), "rb").read()
    write_gz(ANN, ann_bytes)
    ann = json.loads(ann_bytes)
    for case, fname in SHIPPED.items():
        data = open(os.path.join(sota, fname), "rb").read()
        if case.startswith("ARCNN"):
            data = b"".join(ln for ln in data.splitlines(keepends=True) if float(ln.split(b",")[5]) >= ARCNN_MIN_SCORE)
        write_gz(CASES[case][1], data)
    lines = open(os.path.join(sota, "MLPD_result.txt")).readlines()
    perm = np.random.Generator(np.random.PCG64(29)).permutation(len(lines))
    write_gz(CASES["MLPD_shuffled"][1], "".join(lines[i] for i in perm).encode())
    for case, text in synthetic_files(ann).items():
        write_gz(CASES[case][1], text.encode())
    batches, labels_list, small = build_small()
    write_gz(SMALL_ANN, json.dumps(small).encode())
    write_gz(CASES["small_first_fp"][1], small_first_fp(small).encode())

    arrays, meta = {}, {"cases": {}, "evals": EVALS, "numpy": np.__version__, "torch": torch.__version__,
                        "reference": "evaluation_script/evaluation_script.py evaluate() on the CPU"}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                        # loadRes writes its temporary json into the working directory
        try:
            arrays["ignore_flags"] = ignore_flags(E, gunzip_to(ANN, tmp))
            for case, (a, d) in CASES.items():
                r, raises = run_reference(E, gunzip_to(a, tmp), gunzip_to(d, tmp))
                for k, v in r.items():
                    arrays[f"{case}_{k}"] = v
                meta["cases"][case] = {"annotations": a, "detections": d, "raises": raises}
                print(case, "MR x 100:", np.round(r["mr"] * 100, 2).tolist(), "recall", round(float(r["recall_all"]) * 100, 2))
            # the reference's test.test(save_txt=True) on the small KAIST-like loader, then evaluate() on its result.txt
            from oracle.gen_golden_val import StubDetector, digest, load_reference_test, loader
            ref = load_reference_test()
            save = Path(tmp) / "run"
            ref.test({"nc": 1, "names": ["person"]}, model=StubDetector([b[0] for b in batches], 1), dataloader=loader(batches),
                     save_dir=save, save_txt=True, half_precision=False, labels_list=labels_list)
            txt = save / "labels" / "pred" / "result.txt"
            arrays["test_result_txt"] = np.frombuffer(txt.read_bytes(), dtype=np.uint8)
            r, raises = run_reference(E, gunzip_to(SMALL_ANN, tmp), str(txt))
            assert not raises
            for k, v in r.items():
                arrays[f"test_{k}"] = v
            arrays["test_mr_result"] = np.array([*r["mr"], r["recall_all"]], dtype=np.float64)
            meta["test"] = {"inputs": [digest(z, tg) for z, tg, _, _ in batches], "labels_list": labels_list}
            print("test.test MRresult x 100:", np.round(arrays["test_mr_result"] * 100, 2).tolist())
        finally:
            os.chdir(cwd)
    path = golden_path("kaist_mr_cases.npz")
    np.savez_compressed(path, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
