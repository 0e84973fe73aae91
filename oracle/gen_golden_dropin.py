"""Golden data of tests/test_dropin_cpu.py, produced with the REAL reference (run where the reference tree exists):

    python -m oracle.gen_golden_dropin

tests/golden/dropin_ckpt.pt.gz : a gzip-compressed full-object checkpoint written by the reference's own classes
                                (``torch.save({'model': model})``, train.py:424-435) of yolov5s_Transfusion_kaist.  Every
                                tensor is one constant broadcast to its shape (stride 0), so the file stays below 100 KB
                                while each tensor still carries a distinct value (dropin_value).
tests/golden/dropin_reference.json : the reference's state_dict layout (key -> shape), the class names of models/common.py
                                and the constructor signatures of the operator classes the YAMLs and pickles name.
tests/golden/reference_yaml.json   : models/transformer/yolov5{s,l}_Transfusion_kaist.yaml as parsed by yaml.safe_load
                                (tests/test_host_logic_cpu.py compares the generated configs with them).
"""
import gzip
import inspect
import io
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
CLASSES = ("Conv", "Bottleneck", "C3", "SPPF", "Concat", "TransformerFusionBlock", "CrossTransformerBlock", "CrossAttention",
           "LearnableCoefficient", "LearnableWeights", "AdaptivePool2d")
SIGNED = ("Conv", "Bottleneck", "C3", "SPPF", "Concat", "TransformerFusionBlock", "CrossTransformerBlock", "CrossAttention", "AdaptivePool2d")


def dropin_value(i: int, key: str) -> float:
    """The constant stored for the i-th state_dict entry (sorted keys); variances stay positive."""
    v = 0.05 + 0.01 * (i % 37)
    return 1.0 + v if key.endswith("running_var") else (v if i % 2 else -v)


def _compact_json(d: dict) -> str:
    """One line per top-level entry, and per element of a top-level list: small, yet readable in a diff."""
    parts = []
    for k, v in d.items():
        if isinstance(v, list):
            body = "[\n  " + ",\n  ".join(json.dumps(x, separators=(",", ":")) for x in v) + "\n ]"
        else:
            body = json.dumps(v, separators=(",", ":"))
        parts.append(f" {json.dumps(k)}: {body}")
    return "{\n" + ",\n".join(parts) + "\n}\n"


def main():
    from oracle.ref_shim import REF_ROOT, load_reference
    common, yolo = load_reference()
    model = yolo.Model(os.path.join(REF_ROOT, "models", "transformer", "yolov5s_Transfusion_kaist.yaml"), ch=3, nc=1)
    model.half()                                   # train.py:427 saves the half() model object
    sd = model.state_dict()
    keys = sorted(sd)
    tensors = dict(model.named_parameters())
    tensors.update(dict(model.named_buffers()))
    with torch.no_grad():
        for i, k in enumerate(keys):
            t = tensors[k]
            if t.is_floating_point():
                t.data = torch.full((1,), dropin_value(i, k), dtype=t.dtype).expand(t.shape)
    buf = io.BytesIO()
    torch.save({"epoch": 3, "model": model, "optimizer": None}, buf)
    with open(os.path.join(GOLDEN, "dropin_ckpt.pt.gz"), "wb") as f:
        f.write(gzip.compress(buf.getvalue(), 9, mtime=0))
    src = open(os.path.join(REF_ROOT, "models", "common.py")).read()
    sig = lambda f: [[p.name, repr(p.default)] for p in inspect.signature(f).parameters.values()]
    meta = {"state_dict": [[k, list(sd[k].shape), str(sd[k].dtype)] for k in keys],
            "model_module": type(model).__module__,
            "common_classes": [n for n in CLASSES if f"class {n}(" in src],
            "signatures": {n: sig(getattr(common, n).__init__) for n in SIGNED},
            "detect_params": [p.name for p in inspect.signature(yolo.Detect.__init__).parameters.values()]}
    with open(os.path.join(GOLDEN, "dropin_reference.json"), "w") as f:
        f.write(_compact_json(meta))
    import yaml
    cfgs = {}
    for size in ("s", "l"):
        with open(os.path.join(REF_ROOT, "models", "transformer", f"yolov5{size}_Transfusion_kaist.yaml")) as f:
            cfgs[size] = yaml.safe_load(f)
    with open(os.path.join(GOLDEN, "reference_yaml.json"), "w") as f:
        f.write(_compact_json(cfgs))


if __name__ == "__main__":
    main()
