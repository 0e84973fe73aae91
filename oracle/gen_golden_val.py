"""Generate tests/golden/val_cases.npz by executing the REAL reference's test.test (build container only; needs
/root/reference).

    python -m oracle.gen_golden_val

The detector is a stub module whose forward returns fixed decoded predictions, so test.test runs on the CPU with the
reference's own NMS, matching loop, ap_per_class and save_txt code.  `build_inputs()` (seeded PCG64) makes the batches:
predictions seeded around the labels (IoU spread over 0.3-0.98, a duplicate pair on one label whose second hit is a false
positive, wrong-class overlaps, two identical same-class labels whose IoU tie goes to the first, low-confidence noise), an
image with labels and no candidates, an image with candidates and no labels, and target rows shuffled across the batch.
Settings: FLIR-like nc = 3 at test.py's rect shape 544 x 672 (gain 1), the same data with gain != 1, non-integer pads and
boxes clipped at the border, KAIST-like nc = 1 (best-class NMS, the TP/FP/FN print path), single_cls (label classes 0, as
the loader makes them), and save_txt with a labels_list.  Recorded per setting: the results tuple, maps, the iouv used, the inputs ap_per_class received and the
result.txt bytes.  The inputs are not stored: the tests rebuild them and check the SHA-256 stored per batch.
"""
from __future__ import annotations

import hashlib
import importlib.util
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
H, W = 544, 672
# name -> (dataset, single_cls, save_txt)
SETTINGS = {
    "flir": ("flir", False, False),
    "flir_scaled": ("flir_scaled", False, False),
    "kaist": ("kaist", False, False),
    "single_cls": ("flir_single", True, False),
    "save_txt": ("flir", False, True),
}


def _image(g, nc, n_labels, candidates=True, tie=False, dup=True):
    """One image: labels [cls, x, y, w, h] normalised to (H, W), and fp32 prediction rows [x, y, w, h, obj, cls...] in pixels."""
    labels, rows = [], []
    for k in range(n_labels):
        w, h = g.uniform(12, 160), g.uniform(12, 160)
        x, y = g.uniform(-0.1 * w, W + 0.1 * w), g.uniform(-0.1 * h, H + 0.1 * h)      # some cross the border
        labels.append([int(g.integers(nc)), x, y, w, h])
    if tie and labels:
        labels.append(list(labels[-1]))                      # identical same-class label right after the original
    for k, (c, x, y, w, h) in enumerate(labels):
        for _ in range(int(g.integers(1, 3))):
            s = g.uniform(0.0, 0.45)                         # box noise: IoU from ~0.98 down to ~0.3
            bx, by = x + g.normal(0, s * w / 3), y + g.normal(0, s * h / 3)
            bw, bh = w * np.exp(g.normal(0, s / 1.5)), h * np.exp(g.normal(0, s / 1.5))
            cls = np.full(nc, 0.0)
            cls[:] = g.uniform(0.0, 0.25, nc)
            cc = c if g.uniform() > 0.15 else int(g.integers(nc))      # sometimes a wrong class
            cls[cc] = g.uniform(0.5, 0.99)
            rows.append([bx, by, bw, bh, g.uniform(0.2, 0.95), *cls])
        if dup and k == 0:                                    # two halves of one label: both kept, the second one an FP
            for dy in (-0.15 * h, 0.15 * h):
                cls = np.zeros(nc)
                cls[c] = 0.9
                rows.append([x, y + dy, w, 0.7 * h, g.uniform(0.4, 0.9), *cls])
    for _ in range(25):                                       # low-confidence noise
        cls = g.uniform(0.0, 1.0, nc)
        rows.append([g.uniform(0, W), g.uniform(0, H), g.uniform(8, 120), g.uniform(8, 120), g.uniform(0.0, 0.05), *cls])
    rows = np.array(rows, dtype=np.float32).reshape(-1, 5 + nc)
    if not candidates:
        rows[:, 4] = 0.0
    lab = np.array(labels, dtype=np.float64).reshape(-1, 5)
    lab[:, 1:] /= [W, H, W, H]
    return lab, rows


def _batch(g, nc, B, R, special=False):
    z = np.zeros((B, R, 5 + nc), dtype=np.float32)
    tg = []
    for i in range(B):
        n_labels = int(g.integers(2, 9))
        cand, tie = True, i == 1
        if special and i == 2:
            cand = False                                     # labels, no candidates
        if special and i == 3:
            n_labels = 0                                     # candidates, no labels
        lab, rows = _image(g, nc, n_labels, cand, tie)
        rows = rows[g.permutation(rows.shape[0])]
        z[i, :rows.shape[0]] = rows
        tg += [[i, *r] for r in lab]
    tg = np.array(tg, dtype=np.float32).reshape(-1, 6)
    return z.astype(np.float16), tg[g.permutation(tg.shape[0])]


def build_inputs(seed=23):
    """{dataset: [(z16 (B, R, 5+nc), targets fp32 (T, 6), shapes, paths)]}: 4 images per batch at 544 x 672."""
    g = np.random.Generator(np.random.PCG64(seed))
    out = {}
    flir = [_batch(g, 3, 4, 256, special=(k == 0)) for k in range(3)]
    kaist = [_batch(g, 1, 4, 256, special=(k == 1)) for k in range(2)]
    plain = ((512, 640), ((1.0, 1.0), (16.0, 16.0)))                 # FLIR / KAIST 512 x 640 in test.py's rect batch
    scaled = [((590, 758), ((0.85, 0.85), (13.7, 21.3))), ((600, 770), ((0.84375, 0.84375), (11.25, 18.875))),
              ((590, 758), ((0.85, 0.85), (13.7, 21.3))), ((480, 600), ((1.1, 1.1), (5.9, 8.1)))]
    for name, data, shapes in (("flir", flir, [plain] * 4), ("flir_scaled", flir, scaled), ("kaist", kaist, [plain] * 4)):
        out[name] = [(z, tg, list(shapes), [f"/data/{name}/images/{name}_{k:02d}_{i}.jpg" for i in range(4)])
                     for k, (z, tg) in enumerate(data)]
    # single_cls: the loader makes every label class 0 (the reference's nc == 1 print fails on more label classes)
    out["flir_single"] = [(z, tg * np.array([1, 0, 1, 1, 1, 1], np.float32), shapes, paths) for z, tg, shapes, paths in out["flir"]]
    return out


def labels_list_for(batches):
    """A sorted label-file list in which the batch images sit among other names (test.py:397-399)."""
    stems = [Path(p).stem + ".txt" for _, _, _, paths in batches for p in paths]
    return sorted(stems + [f"other_{k:03d}.txt" for k in range(7)])


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def checked_inputs(meta) -> dict:
    """build_inputs(), each batch asserted byte-identical to the one the golden was generated from."""
    inputs = build_inputs()
    for name, shas in meta["inputs"].items():
        assert [digest(z, tg) for z, tg, _, _ in inputs[name]] == shas, \
            f"rebuilt input {name} differs from the golden's (numpy {np.__version__}, golden made with {meta['numpy']})"
    return inputs


class StubDetector(torch.nn.Module):
    """A detector whose forward returns the next batch's fixed decoded predictions (fp32 on the CPU, fp16 on CUDA)."""

    def __init__(self, zs, nc):
        super().__init__()
        self.zs, self.k = zs, 0
        self.names = [f"c{i}" for i in range(nc)]
        self.anchor = torch.nn.Parameter(torch.zeros(1))

    def forward(self, x, x2, augment=False):
        z = torch.from_numpy(self.zs[self.k % len(self.zs)])
        self.k += 1
        z = z.to(x.device, torch.float16 if x.is_cuda else torch.float32)
        return z, None, []


def loader(batches, device="cpu", pin=False):
    """[(img uint8 (B, 6, H, W), targets fp32 (T, 6), paths, shapes)] as the reference's collate_fn gives them."""
    out = []
    for z, tg, shapes, paths in batches:
        img, t = torch.zeros(z.shape[0], 6, H, W, dtype=torch.uint8), torch.from_numpy(tg.copy())
        if pin:
            img, t = img.pin_memory(), t.pin_memory()
        out.append((img.to(device) if device != "cpu" and not pin else img, t, list(paths), list(shapes)))
    return out


def load_reference_test():
    """The reference's test.py as a module named ref_test (`test` would be the stdlib package)."""
    from oracle.ref_shim import REF_ROOT, _lenient, _stub, load_reference
    load_reference()
    for name in ("matplotlib.collections", "matplotlib.patches"):      # evaluation_script/coco.py imports these
        if name not in sys.modules:
            _lenient(_stub(name))
    spec = importlib.util.spec_from_file_location("ref_test", os.path.join(REF_ROOT, "test.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_test"] = mod
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = load_reference_test()
    captured = {}
    real_ap = ref.ap_per_class

    def ap_spy(tp, conf, pred_cls, target_cls, **kw):
        captured["args"] = (tp.copy(), conf.copy(), pred_cls.copy(), target_cls.copy())
        return real_ap(tp, conf, pred_cls, target_cls, **kw)
    ref.ap_per_class = ap_spy
    inputs = build_inputs()
    iouv = torch.linspace(0.5, 0.95, 10)
    arrays = {"iouv": iouv.numpy()}
    meta = {"inputs": {k: [digest(z, tg) for z, tg, _, _ in v] for k, v in inputs.items()}, "settings": {}, "H": H, "W": W}
    for name, (ds, single_cls, save_txt) in SETTINGS.items():
        batches = inputs[ds]
        nc = batches[0][0].shape[2] - 5
        captured.clear()
        with tempfile.TemporaryDirectory() as tmp:
            labels_list = labels_list_for(batches) if save_txt else None
            res, maps, mr, _ = ref.test({"nc": nc, "names": [f"c{i}" for i in range(nc)]}, model=StubDetector([b[0] for b in batches], nc),
                                        dataloader=loader(batches), save_dir=Path(tmp), save_txt=save_txt,
                                        single_cls=single_cls, half_precision=False, labels_list=labels_list, verbose=True)
            if save_txt:
                txt = open(os.path.join(tmp, "labels", "pred", "result.txt"), "rb").read()
                arrays[f"{name}_result_txt"] = np.frombuffer(txt, dtype=np.uint8)
        tp, conf, pcls, tcls = captured["args"]
        assert tp.dtype == bool and conf.dtype == np.float32 and pcls.dtype == np.float32 and tcls.dtype == np.float64
        arrays.update({f"{name}_tp": tp, f"{name}_conf": conf, f"{name}_pcls": pcls, f"{name}_tcls": tcls,
                       f"{name}_maps": np.asarray(maps, dtype=np.float64)})
        meta["settings"][name] = dict(dataset=ds, single_cls=single_cls, save_txt=save_txt, nc=nc,
                                      results=[float(x) for x in res], mr=[float(x) for x in mr],
                                      n_pred=int(tp.shape[0]), tp50=int(tp[:, 0].sum()), n_labels=int(tcls.shape[0]))
        print(name, "results", [round(float(x), 4) for x in res], "preds", tp.shape[0], "TP@.5", int(tp[:, 0].sum()))
    meta["reference"] = "test.py:23-367 test.test(model=stub, dataloader=..., half_precision=False) on the CPU"
    meta["torch"] = torch.__version__
    meta["numpy"] = np.__version__
    path = os.path.join(OUT, "val_cases.npz")
    np.savez_compressed(path, meta=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8), **arrays)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
