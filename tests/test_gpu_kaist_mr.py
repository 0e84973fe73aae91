"""KAIST miss rate on the device: evaluate() against the real reference's evaluate() on every golden case (== on ys, the nine
MRs and recall_all), the rounding kernel against its numpy mirror, test.test(mr_annotations=...) against the reference's
test.test + evaluate() and against evaluate() on the result.txt the same call writes, and the dense and packed layouts."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden
from oracle.gen_golden_kaist_mr import ANN, CASES, EVALS, SETUP_OF, SMALL_ANN, build_small, gunzip_to
from test_kaist_mr_cpu import round_g6

pytestmark = pytest.mark.gpu


def _check(res, d, prefix, where):
    ys = np.stack([res[k].eval["TP"].reshape(9) for k in EVALS])
    assert np.array_equal(ys, d[f"{prefix}_ys"]), (where, ys, d[f"{prefix}_ys"])
    mr = np.array([res[k].summarize(s) for k, s in zip(EVALS, SETUP_OF)], dtype=np.float64)
    assert np.array_equal(mr, d[f"{prefix}_mr"]), (where, mr * 100, d[f"{prefix}_mr"] * 100)
    xx_len = np.array([len(res[k].eval["xx"][0]) if res[k].eval["xx"] else -1 for k in EVALS])
    assert np.array_equal(xx_len, d[f"{prefix}_xx_len"]), where
    for k in ("xx", "yy"):
        sums = np.array([float(np.sum(res[n].eval[k][0])) if res[n].eval[k] else 0.0 for n in EVALS])
        assert np.array_equal(sums, d[f"{prefix}_{k}_sum"]), (where, k)


@pytest.mark.parametrize("case", list(CASES))
def test_evaluate_equals_reference_golden(cuda_device, case):
    from icafusion_b200 import kaist_eval as K
    meta, d = load_golden("kaist_mr_cases")
    a, f = CASES[case]
    ann = K.KaistAnnotations(os.path.join(GOLDEN, a), cuda_device)
    if meta["cases"][case]["raises"]:           # nothing kept in `all`: the reference's recall_all line raises
        with pytest.raises(IndexError):
            K.evaluate(ann, os.path.join(GOLDEN, f))
        rows, span, mx = K.load_detections(os.path.join(GOLDEN, f), ann)
        res = K.evaluate_device(ann, torch.from_numpy(rows).to(cuda_device), torch.from_numpy(span).to(cuda_device), mx)
    else:
        res = K.evaluate(ann, os.path.join(GOLDEN, f))
        assert 1 - res["all"].eval["yy"][0][-1] == d[f"{case}_recall_all"], case
    _check(res, d, case, case)
    if case == "MLPD":
        mr = [round(float(res[k].summarize(s)) * 100, 2) for k, s in zip(EVALS, SETUP_OF)]
        assert mr == [7.58, 7.96, 6.95, 0.04, 11.93, 50.86, 24.15, 28.75, 53.97]


def test_evaluate_from_a_path_and_plot_message(cuda_device, tmp_path, capsys):
    from icafusion_b200 import kaist_eval as K
    meta, d = load_golden("kaist_mr_cases")
    res = K.evaluate(gunzip_to(ANN, tmp_path), gunzip_to(CASES["MLPD"][1], tmp_path), plot=True)
    assert "MR_all: 7.58" in capsys.readouterr().out and res["all"].method == "kaist"
    _check(res, d, "MLPD", "path")
    with pytest.raises(NotImplementedError, match="matplotlib"):
        K.draw_all([res])


def test_rounding_kernel_equals_numpy_mirror(cuda_device):
    from icafusion_b200 import ops
    g = np.random.Generator(np.random.PCG64(8))
    B, max_det, images = 6, 300, 20
    native = np.exp(g.uniform(np.log(1e-3), np.log(640), (B, max_det, 4))).astype(np.float32)
    native[..., 2:] += native[..., :2]
    native[0, :5] = np.array([[0, 0, 640, 512], [0.5, 1.5, 2.5, 1234.5], [12.34565, 100, 100.00001, 511.99997],
                              [1e-7, 3e-6, 639.99994, 7], [5.5, 6.5, 7.5, 8.5]], np.float32)
    det = np.zeros((B, max_det, 6), np.float32)
    det[..., 4] = np.exp(g.uniform(np.log(1e-6), 0, (B, max_det))).astype(np.float32)
    det[0, :3, 4] = [0.001, 1.0, 0.5]
    count = np.array([300, 0, 17, 299, 1, 300], np.int32)
    image = np.array([3, 0, 19, 7, 8, 11], np.int32)
    rows = torch.full((images * max_det, 5), -7.0, dtype=torch.float64, device=cuda_device)
    span = torch.zeros(images, 2, dtype=torch.int32, device=cuda_device)
    t = lambda a: torch.from_numpy(a).to(cuda_device)
    ops.kaist_round_detections(t(native), t(det), t(count), t(image), rows, span)
    rows, span = rows.cpu().numpy(), span.cpu().numpy()
    for b in range(B):
        p, n = image[b], count[b]
        assert tuple(span[p]) == (p * max_det, n)
        nb = native[b, :n]
        want = np.stack([round_g6(nb[:, 0]), round_g6(nb[:, 1]), round_g6(nb[:, 2] - nb[:, 0]), round_g6(nb[:, 3] - nb[:, 1]),
                         round_g6(det[b, :n, 4])], 1)
        assert np.array_equal(rows[p * max_det:p * max_det + n], want), b
        assert (rows[p * max_det + n:(p + 1) * max_det] == -7.0).all()
        line = [float("%g" % v) for v in (nb[:1, 0].tolist() + (nb[:1, 2] - nb[:1, 0]).tolist())] if n else []
        assert not n or (rows[p * max_det, 0], rows[p * max_det, 2]) == tuple(line)


def test_dropin_test_mr_annotations_equals_reference(cuda_device, tmp_path):
    from icafusion_b200 import kaist_eval as K
    from icafusion_b200 import test as T
    from oracle.gen_golden_val import StubDetector, digest, loader
    meta, d = load_golden("kaist_mr_cases")
    batches, labels_list, _ = build_small()
    assert [digest(z, tg) for z, tg, _, _ in batches] == meta["test"]["inputs"] and labels_list == meta["test"]["labels_list"]
    ann_path = gunzip_to(SMALL_ANN, tmp_path)
    want = d["test_mr_result"].tolist()
    for save_txt, ann in ((True, ann_path), (False, K.KaistAnnotations(ann_path, cuda_device))):
        stub = StubDetector([b[0] for b in batches], 1).to(cuda_device)
        run = tmp_path / f"run_{save_txt}"
        res, maps, mr, t = T.test({"nc": 1, "names": ["person"]}, model=stub, dataloader=loader(batches, pin=True),
                                  save_dir=run, save_txt=save_txt, labels_list=labels_list, mr_annotations=ann)
        assert mr == want, (save_txt, np.array(mr) * 100, np.array(want) * 100)
        if save_txt:
            txt = run / "labels" / "pred" / "result.txt"
            assert txt.read_bytes() == d["test_result_txt"].tobytes()
            res_txt = K.evaluate(ann_path, str(txt))
            assert [res_txt[k].summarize(s) for k, s in zip(EVALS, SETUP_OF)] + \
                [1 - res_txt["all"].eval["yy"][0][-1]] == mr
            _check(res_txt, d, "test", "result.txt")
    assert want[2] == -1                         # night: no image of the 40


def test_dense_and_packed_layouts_agree(cuda_device):
    from icafusion_b200 import kaist_eval as K
    from icafusion_b200 import ops
    ann = K.KaistAnnotations(os.path.join(GOLDEN, ANN), cuda_device)
    rows, span, mx = K.load_detections(os.path.join(GOLDEN, CASES["MBNet"][1]), ann)
    ys_p, counts_p, cv_p = ops.kaist_mr(ann, torch.from_numpy(rows).to(cuda_device), torch.from_numpy(span).to(cuda_device),
                                        mx, curves=True)
    per = mx + 3                                 # a dense layout with gaps, as test.test's max_det rows per image
    dense = np.full((ann.images * per, 5), np.nan)
    dspan = np.zeros_like(span)
    for p, (o, n) in enumerate(span):
        dense[p * per:p * per + n] = rows[o:o + n]
        dspan[p] = (p * per, n)
    ys_d, counts_d, cv_d = ops.kaist_mr(ann, torch.from_numpy(dense).to(cuda_device), torch.from_numpy(dspan).to(cuda_device),
                                        per, curves=True)
    assert torch.equal(ys_p, ys_d) and torch.equal(counts_p, counts_d)
    for e in range(9):
        n = int(counts_p[e, 0])
        assert torch.equal(cv_p[e, :, :n], cv_d[e, :, :n])
