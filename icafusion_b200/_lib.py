"""ctypes binding of libicaf_b200.so (the C ABI declared in include/icaf_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, the
product path raises.  Build it with ``python -m icafusion_b200.build`` (or
``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libicaf_b200.so")

ACT_NONE, ACT_SILU, ACT_GELU = 0, 1, 2
EPI_BIAS_ROW, EPI_ADD_RES, EPI_SCALED_RES, EPI_LN_FOLD, EPI_EMIT_STATS = 1, 2, 4, 8, 16


class ConvGeom(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("B", "Hi", "Wi", "Cin", "Ho", "Wo", "Cout", "kh", "kw", "stride", "pad",
                                       "k_pad", "w_rows", "act", "epi")]


class ConvIO(C.Structure):
    _fields_ = [("x", C.c_void_p), ("x_ld", C.c_int64), ("w", C.c_void_p), ("bias", C.c_void_p),
                ("res", C.c_void_p), ("res_ld", C.c_int64), ("y", C.c_void_p), ("y_ld", C.c_int64),
                ("alpha", C.c_void_p), ("beta", C.c_void_p),
                ("ln_stats", C.c_void_p), ("ln_colsum", C.c_void_p), ("ln_parts", C.c_int), ("ln_eps", C.c_float),
                ("stats_out", C.c_void_p)]


class ConvPlan(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("kernel", "bn", "a_mode", "tile_w", "tile_h", "tiles_x", "tiles_y", "cblk", "halo",
                                       "stages", "splits", "grid_x", "grid_y", "grid_z", "cluster", "smem_bytes",
                                       "work_items", "ctas")]


class BottleneckIO(C.Structure):
    _fields_ = [("x", C.c_void_p), ("x_ld", C.c_int64), ("w1", C.c_void_p), ("b1", C.c_void_p), ("w3", C.c_void_p),
                ("b2", C.c_void_p), ("y", C.c_void_p), ("y_ld", C.c_int64)]


class LossHyp(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("box", "obj", "cls", "cls_pw", "obj_pw", "anchor_t", "fl_gamma", "gr", "cp", "cn")] + \
               [("balance", C.c_float * 5)]


class AugTile(C.Structure):
    _fields_ = [("rgb", C.c_void_p), ("ir", C.c_void_p)] + \
               [(n, C.c_int) for n in ("H0", "W0", "h", "w", "x1a", "y1a", "x2a", "y2a", "x1b", "y1b", "xtab", "ytab")]


class AugSample(C.Structure):
    _fields_ = [("tile", AugTile * 4)] + [(n, C.c_int) for n in ("ntiles", "canvas", "warp", "flipud", "fliplr", "reserved")] + \
               [("lut", C.c_uint8 * (2 * 3 * 256))]


class ValSample(C.Structure):
    _fields_ = [("rgb", C.c_void_p), ("ir", C.c_void_p)] + \
               [(n, C.c_int) for n in ("H0", "W0", "h", "w", "top", "left", "mode", "xtab", "ytab", "sx", "sy", "reserved")]


KERNEL_TC = 0

OPTIM_CHUNK, OPTIM_HYPER = 2048, 8        # ICAF_OPTIM_CHUNK, ICAF_OPTIM_HYPER


class ValBatch(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("det", "count", "correct", "native")] + [("image0", C.c_int64)] + \
               [(n, C.c_int) for n in ("B", "max_det", "local0")] + [("reserved", C.c_int * 3)]


VAL_PACK_NATIVE, VAL_PACK_POS = 1, 2       # ICAF_VAL_PACK_NATIVE, ICAF_VAL_PACK_POS


class OptimTensor(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("p", "g", "m", "v", "step")] + [("numel", C.c_int64), ("chunk0", C.c_int64), ("reserved", C.c_int64)]

_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float
# name -> argtypes; every symbol include/icaf_b200.h declares (tests check the .so exports them all)
SIGNATURES = {
    "icaf_version": [],
    "icaf_last_error": [],
    "icaf_sm_count": [],
    "icaf_set_sm_count_target": [_i],
    "icaf_kernel_launches": [],
    "icaf_conv2d_fwd": [C.POINTER(ConvGeom), C.POINTER(ConvIO), _i, _vp],
    "icaf_conv2d_plan": [C.POINTER(ConvGeom), _i, _i, _i, C.POINTER(ConvPlan)],
    "icaf_conv2d_fwd_simt": [C.POINTER(ConvGeom), C.POINTER(ConvIO), _i, _vp],
    "icaf_bottleneck_fwd": [_i, _i, _i, C.POINTER(BottleneckIO), _i, _vp],
    "icaf_pack_image": [_vp, _i, _f, _i, _i, _i, _vp, _vp],
    "icaf_pack_image_s2d": [_vp, _i, _f, _i, _i, _i, _vp, _vp],
    "icaf_letterbox": [_vp, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp],
    "icaf_sppf_pool": [_vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp],
    "icaf_upsample2x": [_vp, _i64, _vp, _i64, _i, _i, _i, _i, _vp],
    "icaf_copy_channels": [_vp, _i64, _vp, _i64, _i64, _i, _vp],
    "icaf_prefetch_l2": [_vp, C.c_size_t, _vp],
    "icaf_dmff_pool_tokens": [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_row_stats": [_vp, _vp, _vp, _vp, _i64, _i, _vp],
    "icaf_layernorm": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _vp],
    "icaf_cross_attention": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp],
    "icaf_cross_attention_simt": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp],
    "icaf_dmff_upsample_cat": [_vp, _vp, _i, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_nms_workspace_bytes": [_i, _i],
    "icaf_nms": [_vp, _i, _i, _i, _f, _f, _i, C.c_uint64, _i, _vp, _vp, _vp, C.c_size_t, _vp],
    "icaf_nms_multi_label_workspace_bytes": [_i, _i, _i],
    "icaf_nms_multi_label": [_vp, _i, _i, _i, _f, _f, _i, C.c_uint64, _i, _vp, _vp, _vp, C.c_size_t, _vp],
    "icaf_confluence_workspace_bytes": [_i, _i, _i],
    "icaf_confluence": [_vp, _i, _i, _i, _i, _f, C.c_double, _vp, _vp, _i, _vp, _vp, C.c_size_t, _vp],
    "icaf_match_detections_workspace_bytes": [_i],
    "icaf_match_detections": [_vp, _vp, _i, _i, _vp, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, C.c_size_t, _vp],
    "icaf_kaist_mr_workspace_bytes": [_i, _i, _i],
    "icaf_kaist_mr": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, C.c_size_t, _vp],
    "icaf_kaist_round_detections": [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp],
    "icaf_loss_workspace_bytes": [_i, _i, _i, C.POINTER(C.c_int), C.POINTER(C.c_int), _i, _i],
    "icaf_compute_loss_fwd": [C.POINTER(C.c_void_p), _i, _i, C.POINTER(C.c_int), C.POINTER(C.c_int), _i, _i, _i, _i, _vp, _i,
                              C.POINTER(C.c_float), C.POINTER(LossHyp), _vp, _vp, C.c_size_t, _vp],
    "icaf_compute_loss_bwd": [C.POINTER(C.c_void_p), _i, _i, C.POINTER(C.c_int), C.POINTER(C.c_int), _i, _i, _i, _i, _vp, _i,
                              C.POINTER(C.c_float), C.POINTER(LossHyp), _vp, C.POINTER(C.c_void_p), _vp, C.c_size_t, _vp],
    "icaf_conv2d_wgrad_workspace_bytes": [C.POINTER(ConvGeom)],
    "icaf_conv2d_wgrad": [C.POINTER(ConvGeom), _vp, _i64, _vp, _i64, _vp, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_zero_stuff2": [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_colsum": [_vp, _i64, _i, _vp, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_train_workspace_bytes": [_i],
    "icaf_bn_act_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_bn_act_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_bn_act_fwd_stats": [_vp, _i64, _i, _vp, _vp, C.c_size_t, _vp],
    "icaf_bn_act_fwd_apply": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_bn_act_bwd_sums": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_bn_act_bwd_apply": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp, C.c_size_t, _vp],
    "icaf_eltwise": [_i, _vp, _vp, _vp, _i64, _f, C.c_uint32, _vp],
    "icaf_layernorm_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_dot": [_vp, _vp, _i64, _i, _vp, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_upsample2x_bwd": [_vp, _vp, _i, _i, _i, _i, _vp],
    "icaf_maxpool5_bwd": [_vp, _vp, _vp, _i, _i, _i, _i, _vp, C.c_size_t, _vp],
    "icaf_dmff_pool_tokens_bwd": [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, C.c_size_t, _vp],
    "icaf_dmff_upsample_cat_bwd": [_vp, _i64, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_pack_weight": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp],
    "icaf_pack_weight_pair": [_vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp],
    "icaf_set_seed_offset": [_vp],
    "icaf_cross_attention_train": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, C.c_uint32, _vp],
    "icaf_cross_attention_bwd_workspace_bytes": [_i, _i, _i],
    "icaf_cross_attention_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, C.c_uint32, _vp, C.c_size_t, _vp],
    "icaf_axpby": [_vp, _vp, _vp, _vp, _vp, _i64, _vp],
    "icaf_dmff_pool_tokens_f32": [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_dmff_pool_tokens_bwd_f32": [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, C.c_size_t, _vp],
    "icaf_dmff_upsample_cat_f32": [_vp, _vp, _i, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_dmff_upsample_cat_bwd_f32": [_vp, _i64, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp],
    "icaf_layernorm_f32": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _vp],
    "icaf_layernorm_bwd_f32": [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_axpby_f32": [_vp, _vp, _vp, _vp, _vp, _i, _i64, _vp],
    "icaf_dot_f32": [_vp, _vp, _i, _i64, _i, _vp, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_colsum_f32": [_vp, _i64, _i, _vp, _f, _i, _vp, C.c_size_t, _vp],
    "icaf_detect_decode": [_vp, _i64, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, C.POINTER(C.c_float), _vp],
    "icaf_augment_params_bytes": [_i, _i, _i],
    "icaf_augment": [_vp, C.c_size_t, _i, _i, _i, _vp, _vp, _vp],
    "icaf_val_stage_params_bytes": [_i, _i],
    "icaf_val_stage": [_vp, C.c_size_t, _i, _i, _i, _i, _vp, _vp],
    "icaf_optim_table_bytes": [_i],
    "icaf_amp_unscale": [_vp, C.c_size_t, _i, _i64, _vp, _vp, _vp],
    "icaf_sgd_step": [_vp, C.c_size_t, _i, _i64, _vp, _i, _i, _vp, _vp],
    "icaf_adam_step": [_vp, C.c_size_t, _i, _i64, _vp, _i, _i, _vp, _i, _vp, _vp],
    "icaf_amp_update_scale": [_vp, _vp, _vp, C.c_double, C.c_double, _i, _vp],
    "icaf_ema_update": [_vp, C.c_size_t, _i, _i64, _vp, _vp],
    "icaf_val_pack_params_bytes": [_i, _i, _i],
    "icaf_val_pack_bytes": [_i, _i, _i],
    "icaf_val_pack": [_vp, C.c_size_t, _i, _i, _i, _i, _vp, C.c_size_t, _vp],
    "icaf_val_merge_workspace_bytes": [_i],
    "icaf_val_merge": [_vp, _i, _i64, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, C.c_size_t, _vp],
}

_lib = None


class IcafError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise IcafError(f"{LIB_PATH} not found -- build it with `python -m icafusion_b200.build`; "
                            "icafusion_b200 has no non-CUDA fallback")
        L = C.CDLL(LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(L, name)            # AttributeError here = header/.so drift
            fn.argtypes = argtypes
            fn.restype = {"icaf_last_error": C.c_char_p, "icaf_kernel_launches": C.c_longlong,
                          "icaf_nms_workspace_bytes": C.c_size_t, "icaf_loss_workspace_bytes": C.c_size_t,
                          "icaf_nms_multi_label_workspace_bytes": C.c_size_t,
                          "icaf_confluence_workspace_bytes": C.c_size_t,
                          "icaf_match_detections_workspace_bytes": C.c_size_t,
                          "icaf_kaist_mr_workspace_bytes": C.c_size_t,
                          "icaf_conv2d_wgrad_workspace_bytes": C.c_size_t, "icaf_train_workspace_bytes": C.c_size_t,
                          "icaf_cross_attention_bwd_workspace_bytes": C.c_size_t,
                          "icaf_augment_params_bytes": C.c_size_t, "icaf_val_stage_params_bytes": C.c_size_t,
                          "icaf_optim_table_bytes": C.c_size_t, "icaf_val_pack_params_bytes": C.c_size_t,
                          "icaf_val_pack_bytes": C.c_size_t, "icaf_val_merge_workspace_bytes": C.c_size_t}.get(name, C.c_int)
        _lib = L
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().icaf_last_error()
        raise IcafError(f"{what or 'icaf call'} failed (code {rc}): {msg.decode() if msg else '?'}")
