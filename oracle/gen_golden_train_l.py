"""Generate tests/golden/train_yolov5l_320.npz by executing the REAL reference's training step (build container only).

    python -m oracle.gen_golden_train_l          # needs the reference checkout (oracle/ref_shim.py REF_ROOT)

gen_golden_sizes.train_step on yolov5l_Transfusion_kaist: the one trained size with head dim 128 in the attention backward
and up to nine Bottlenecks per C3.  Batch 2 at 320x320, 12 targets, seed 1234, dropout p = 0, fp32 CPU.  Stored, as for the
other training goldens: the loss, a fingerprint (L2 norm + two seeded projections, float64) of every parameter gradient and
of the three Detect outputs, the dead parameters and the updated running statistics of the BN probe layers.
"""
from __future__ import annotations

import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.gen_golden_sizes import train_step  # noqa: E402
from oracle.ref_shim import load_reference  # noqa: E402

TRAIN_CASE = dict(name="train_yolov5l_320", size="l", dataset="kaist", nc=1, B=2, H=320, W=320, nt=12, seed=1234)


def main():
    warnings.filterwarnings("ignore")
    _, yolo = load_reference()
    train_step(yolo, TRAIN_CASE)


if __name__ == "__main__":
    main()
