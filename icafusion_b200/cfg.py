"""Model descriptions for the two-stream ICAFusion ("Transfusion") detectors.

The reference describes its networks with YAML rows ``[from, number, module, args]``
(models/transformer/yolov5{s,l}_Transfusion_kaist.yaml, consumed by parse_model,
models/yolo_test.py:216-302).  We keep that row format as the interchange format -- a user
YAML written for the reference loads unchanged through :func:`load_cfg` -- but the stock
KAIST configurations are generated here rather than stored as files.
"""
from __future__ import annotations

import copy
from typing import Dict, Union

KAIST_ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]
_MULT = {"n": (0.33, 0.25), "s": (0.33, 0.50), "m": (0.67, 0.75), "l": (1.00, 1.00), "x": (1.33, 1.25)}
# DMFF token grids at P3 / P4 / P5 (vert_anchors, horz_anchors), yolov5l_Transfusion_kaist.yaml:39-41
DMFF_GRIDS = ((20, 20), (16, 16), (10, 10))


def _stream(first_from: int):
    """One CSPDarknet stream: stem, then (downsample conv, C3) x4, then SPPF."""
    rows = [[first_from, 1, "Conv", [64, 6, 2, 2]]]
    for width, depth in ((128, 3), (256, 6), (512, 9), (1024, 3)):
        rows.append([-1, 1, "Conv", [width, 3, 2]])
        rows.append([-1, depth, "C3", [width]])
    rows.append([-1, 1, "SPPF", [1024, 5]])
    return rows


def transfusion_kaist_cfg(size: str = "s", nc: int = 1) -> Dict:
    """Config dict equivalent to models/transformer/yolov5<size>_Transfusion_kaist.yaml."""
    gd, gw = _MULT[size]
    rgb = _stream(-1)            # layers 0-9
    ir = _stream(-4)             # layers 10-19; -4 routes the IR image (yolo_test.py:154-155)
    taps = ((4, 14, 256), (6, 16, 512), (9, 19, 1024))   # P3, P4, P5 outputs of each stream
    fusion = [[[a, b], 1, "TransformerFusionBlock", [c, va, ha]]
              for (a, b, c), (va, ha) in zip(taps, DMFF_GRIDS)]          # layers 20-22
    up = ["None", 2, "nearest"]          # the YAML literal `None` is a string (eval-ed by parse_model)
    head = [
        [-1, 1, "Conv", [512, 1, 1]],              # 23
        [-1, 1, "nn.Upsample", list(up)],          # 24
        [[-1, 21], 1, "Concat", [1]],              # 25
        [-1, 3, "C3", [512, False]],               # 26
        [-1, 1, "Conv", [256, 1, 1]],              # 27
        [-1, 1, "nn.Upsample", list(up)],          # 28
        [[-1, 20], 1, "Concat", [1]],              # 29
        [-1, 3, "C3", [256, False]],               # 30  P3 out
        [-1, 1, "Conv", [256, 3, 2]],              # 31
        [[-1, 27], 1, "Concat", [1]],              # 32
        [-1, 3, "C3", [512, False]],               # 33  P4 out
        [-1, 1, "Conv", [512, 3, 2]],              # 34
        [[-1, 23], 1, "Concat", [1]],              # 35
        [-1, 3, "C3", [1024, False]],              # 36  P5 out
        [[30, 33, 36], 1, "Detect", ["nc", "anchors"]],
    ]
    return {"nc": nc, "depth_multiple": gd, "width_multiple": gw,
            "anchors": copy.deepcopy(KAIST_ANCHORS), "backbone": rgb + ir + fusion, "head": head}


# Stock dataset suffixes and their class counts: the reference's FLIR YAMLs differ from the KAIST ones only in nc.
_DATASET_NC = {"_Transfusion_kaist": 1, "_Transfusion_FLIR": 3}


def load_cfg(cfg: Union[str, Dict]) -> Dict:
    """Accepts a config dict, a YAML path in the reference's row format, or a stock name
    ('yolov5{n,s,m,l,x}_Transfusion_kaist' or '..._Transfusion_FLIR', with or without '.yaml').  Other datasets' YAMLs
    load by path; ``Model(cfg, nc=...)`` overrides the class count of any of them."""
    if isinstance(cfg, dict):
        out = copy.deepcopy(cfg)
    else:
        import os
        stem = os.path.basename(str(cfg))
        stem = stem[:-5] if stem.endswith(".yaml") else stem
        if os.path.isfile(str(cfg)):
            import yaml
            with open(cfg) as f:
                out = yaml.safe_load(f)
        elif stem.startswith("yolov5") and len(stem) > 6 and stem[6] in _MULT and stem[7:] in _DATASET_NC:
            out = transfusion_kaist_cfg(stem[6], nc=_DATASET_NC[stem[7:]])
        else:
            raise FileNotFoundError(cfg)
    # resolve the two symbolic Detect args like parse_model's eval() does (yolo_test.py:225-229)
    for row in out["backbone"] + out["head"]:
        row[3] = [out["nc"] if a == "nc" else out["anchors"] if a == "anchors" else a for a in row[3]]
    return out
