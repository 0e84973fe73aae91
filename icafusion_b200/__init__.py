"""icafusion_b200 -- H100 (sm_90a) native implementation of the ICAFusion hot path:
two-stream CSPDarknet Conv+BN+SiLU backbone + DMFF cross-attention fusion + Detect head.

    from icafusion_b200 import Model
    model = Model("yolov5s_Transfusion_kaist").cuda().eval().fuse()
    z, logits, xs = model(rgb, ir)            # (B,3,H,W) images, like the reference's model(img_rgb, img_ir)

The operator classes in :mod:`icafusion_b200.common` mirror models/common.py of the reference (same names,
constructor signatures and state_dict keys); their forwards run hand-written CUDA kernels from
``libicaf_b200.so`` through the C ABI in ``include/icaf_b200.h``.
"""
from ._lib import IcafError, LIB_PATH  # noqa: F401
from .cfg import load_cfg, transfusion_kaist_cfg  # noqa: F401
from .common import (C3, SPPF, AdaptivePool2d, Bottleneck, Concat, Conv, CrossAttention, CrossTransformerBlock,  # noqa: F401
                     LearnableCoefficient, LearnableWeights, TransformerFusionBlock, Upsample)
from .yolo_test import Detect, Model, parse_model  # noqa: F401

__version__ = "0.1.0"
