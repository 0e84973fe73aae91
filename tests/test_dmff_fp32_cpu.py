"""fp32 DMFF token streams (TransformerFusionBlock.stream_dtype = float32, TrainStep(dmff_fp32=True)) without a GPU: the training
step's launches on `meta` tensors, the host-side refusals of the new entry points, and the ptxas report of their kernels."""
import collections
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from icafusion_b200 import build as B

# fp16 entry point -> its fp32-stream form; every DMFF token-stream call switches, nothing else does
F32_FORM = {
    "icaf_dmff_pool_tokens": "icaf_dmff_pool_tokens_f32",
    "icaf_dmff_pool_tokens_bwd": "icaf_dmff_pool_tokens_bwd_f32",
    "icaf_dmff_upsample_cat": "icaf_dmff_upsample_cat_f32",
    "icaf_dmff_upsample_cat_bwd": "icaf_dmff_upsample_cat_bwd_f32",
    "icaf_layernorm": "icaf_layernorm_f32",
    "icaf_layernorm_bwd": "icaf_layernorm_bwd_f32",
    "icaf_axpby": "icaf_axpby_f32",
    "icaf_dot": "icaf_dot_f32",
    "icaf_colsum": "icaf_colsum_f32",
}


def _train_step_records(fp32):
    from icafusion_b200 import Model, ops
    from icafusion_b200.trainer import set_dmff_stream_dtype
    m = Model("yolov5s_Transfusion_kaist").to("meta").train()
    if fp32 is not None:
        set_dmff_stream_dtype(m, fp32)
    rgb = torch.empty(2, 3, 320, 320, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        pred = m(rgb, rgb)
        torch.autograd.backward(pred, [torch.empty_like(p) for p in pred])
    live = sorted(k for k, p in m.named_parameters() if p.grad is not None)
    dead = sorted(k for k, p in m.named_parameters() if p.grad is None)
    return [name for name, _, _ in dr.records], live, dead, m


def test_train_step_dry_run_switches_exactly_the_token_stream_calls():
    """yolov5s kaist in train() on `meta`, forward + backward: with fp32 streams every DMFF token-stream call is its fp32 form,
    every other launch is unchanged, and the same parameters (all but the 30 dead ones) receive a gradient."""
    from icafusion_b200.trainer import dead_parameters
    base, live0, dead0, _ = _train_step_records(None)
    f16, live16, _, _ = _train_step_records(False)
    f32, live32, dead32, m = _train_step_records(True)
    assert f16 == base and live16 == live0
    assert live32 == live0 and dead32 == dead0 == sorted(dead_parameters(m)) and len(dead32) == 30
    back = {v: k for k, v in F32_FORM.items()}
    # one for one: the fp32 run's calls with the fp32 forms mapped back are the fp16 run's calls, in the same order
    assert [back.get(n, n) for n in f32] == base
    c16, c32 = collections.Counter(base), collections.Counter(f32)
    n_blk = sum(type(x).__name__ == "TransformerFusionBlock" for x in m.modules())
    n_ctb = sum(type(x).__name__ == "CrossTransformerBlock" for x in m.modules())
    n_add = sum(getattr(x, "add", False) for x in m.modules() if type(x).__name__ == "Bottleneck")
    assert n_blk == 3 and n_ctb == 3
    # every stream call is fp32: LayerNorms (LN1 x2, LN2 x2 per loop), coefficient pairs (4 per loop + 2 per pair backward),
    # the pooling, tail, their backwards and the scalar reductions; the fp16 forms left are the backbone's and the two pooled
    # operands of the mixing-weight dots
    for k in ("icaf_layernorm", "icaf_layernorm_bwd", "icaf_dmff_pool_tokens_bwd", "icaf_dmff_upsample_cat", "icaf_dmff_upsample_cat_bwd",
              "icaf_dot", "icaf_colsum"):
        assert c32[F32_FORM[k]] == c16[k] - (c32[k] if k == "icaf_colsum" else 0), k
    assert c32["icaf_layernorm"] == c32["icaf_layernorm_bwd"] == c32["icaf_dot"] == 0
    assert c32["icaf_layernorm_f32"] == 4 * n_ctb and c32["icaf_dot_f32"] == 4 * n_blk + 8 * n_ctb
    assert c32["icaf_dmff_pool_tokens_f32"] == n_blk and c32["icaf_dmff_pool_tokens"] == 2 * n_blk
    assert c32["icaf_colsum_f32"] == 2 * n_blk
    assert c32["icaf_axpby_f32"] == 4 * n_ctb * 3                 # forward + dx + do of every coefficient pair
    assert c32["icaf_axpby"] == c16["icaf_axpby"] - 12 * n_ctb >= n_add


def test_flag_sets_and_eval_ignores_the_stream_dtype():
    from icafusion_b200 import Model, TransformerFusionBlock
    from icafusion_b200.trainer import TrainStep
    m = Model("yolov5s_Transfusion_kaist")
    blocks = [x for x in m.modules() if isinstance(x, TransformerFusionBlock)]
    assert all(b.stream_dtype == torch.float16 for b in blocks)
    keys = list(m.state_dict())
    ts = TrainStep(m, dmff_fp32=True)
    assert len(blocks) == 3 and all(b.stream_dtype == torch.float32 for b in blocks)
    assert list(m.state_dict()) == keys                               # no state_dict entry added
    TrainStep(m)                                                      # None keeps what is set
    assert all(b.stream_dtype == torch.float32 for b in blocks)
    TrainStep(m, dmff_fp32=False)
    assert all(b.stream_dtype == torch.float16 for b in blocks)
    blocks[1].stream_dtype = torch.float32                            # set by hand on a plain model, then wrapped
    TrainStep(m)
    assert [b.stream_dtype for b in blocks] == [torch.float16, torch.float32, torch.float16]
    del ts
    blocks[0].stream_dtype = torch.bfloat16
    from icafusion_b200 import ops
    with ops.dry_run(), pytest.raises(ValueError, match="stream_dtype"):
        m.to("meta").train()(torch.empty(1, 3, 320, 320, dtype=torch.uint8, device="meta"),
                             torch.empty(1, 3, 320, 320, dtype=torch.uint8, device="meta"))


def test_wrappers_refuse_wrong_dtypes_and_shapes():
    """Each fp32-stream wrapper checks its operands' dtypes (the C ABI takes untyped pointers) and shapes before any call."""
    from icafusion_b200 import ops
    meta = dict(device="meta")
    B, H, W, C, nh, nw = 2, 20, 20, 64, 10, 10
    N, n_pad = nh * nw, 104
    x16 = torch.empty(B, H, W, C, dtype=torch.float16, **meta)
    pos32 = torch.empty(N, C, dtype=torch.float32, **meta)
    mix = torch.empty(4, dtype=torch.float32, **meta)
    tok32 = torch.empty(B, n_pad, C, dtype=torch.float32, **meta)
    one = torch.empty(1, dtype=torch.float32, **meta)
    with ops.dry_run() as dr:
        ops.dmff_pool_tokens_f32(x16, x16, pos32, pos32, mix, nh, nw)
        ops.dmff_pool_tokens_bwd_f32(x16, x16, tok32, tok32, mix, nh, nw)
        ops.dmff_upsample_cat_f32(tok32, tok32, x16, x16, nh, nw)
        ops.dmff_upsample_cat_bwd_f32(torch.empty(B, H, W, 2 * C, dtype=torch.float16, **meta), nh, nw, n_pad)
        ops.layernorm_f32(tok32, pos32[0], pos32[0])
        ops.layernorm_bwd_f32(tok32, tok32.half(), pos32[0], 1e-5)
        ops.axpby_f32(tok32, one, tok32.half(), one)
        ops.axpby_f32(tok32, one, out_dtype=torch.float16)
        ops.dot_f32(tok32, tok32.half())
        ops.dot_f32(tok32, tok32)
        ops.colsum_f32(tok32.view(B, n_pad * C))
        assert len(dr.records) == 11
        bad = [
            lambda: ops.dmff_pool_tokens_f32(x16, x16, pos32.half(), pos32, mix, nh, nw),          # fp16 pos_emb
            lambda: ops.dmff_pool_tokens_f32(x16, x16, pos32[:50], pos32, mix, nh, nw),           # wrong token count
            lambda: ops.dmff_pool_tokens_f32(x16.float(), x16, pos32, pos32, mix, nh, nw),        # fp32 map
            lambda: ops.dmff_pool_tokens_bwd_f32(x16, x16, tok32.half(), tok32, mix, nh, nw),     # fp16 token gradients
            lambda: ops.dmff_upsample_cat_f32(tok32.half(), tok32, x16, x16, nh, nw),             # fp16 tokens
            lambda: ops.dmff_upsample_cat_f32(tok32[:, :96], tok32[:, :96], x16, x16, nh, nw),   # fewer rows than tokens
            lambda: ops.dmff_upsample_cat_bwd_f32(torch.empty(B, H, W, 2 * C, dtype=torch.float32, **meta), nh, nw, n_pad),
            lambda: ops.layernorm_f32(tok32.half(), pos32[0], pos32[0]),
            lambda: ops.layernorm_f32(tok32, pos32[0, :32], pos32[0]),                            # gamma of the wrong width
            lambda: ops.layernorm_bwd_f32(tok32, tok32, pos32[0], 1e-5),                          # fp32 dy
            lambda: ops.layernorm_bwd_f32(tok32.half(), tok32.half(), pos32[0], 1e-5),
            lambda: ops.axpby_f32(tok32.half(), one, tok32.half(), one),                          # fp16 stream
            lambda: ops.axpby_f32(tok32, one, tok32, one),                                        # fp32 branch
            lambda: ops.axpby_f32(tok32, one.half(), tok32.half(), one),
            lambda: ops.axpby_f32(tok32, one, out_dtype=torch.bfloat16),
            lambda: ops.dot_f32(tok32.half(), tok32.half()),
            lambda: ops.dot_f32(tok32, tok32[:, :8].half()),
            lambda: ops.colsum_f32(tok32.half().view(B, n_pad * C)),
        ]
        for i, f in enumerate(bad):
            with pytest.raises(ValueError):
                f()
                pytest.fail(f"case {i} accepted")
        assert len(dr.records) == 11


def test_entry_points_refuse_bad_shapes_and_workspaces_on_the_host():
    """The C entry points reject bad shapes and short workspaces before any CUDA call (code 1 / 2, readable error)."""
    from icafusion_b200 import _lib
    L = _lib.lib()
    one = ctypes.c_void_p(16)                     # a non-null pointer that is never dereferenced: validation fails first
    n0 = L.icaf_kernel_launches()
    ws = 2 * 1 * 8 * 8 * 128
    # pooling: C % 8, grid larger than the map, n_pad < tokens; backward: short / misaligned workspace, windows > 255 pixels
    assert L.icaf_dmff_pool_tokens_f32(one, one, 128, one, one, one, one, one, 1, 16, 16, 124, 8, 8, 64, None) == 1
    assert L.icaf_dmff_pool_tokens_f32(one, one, 128, one, one, one, one, one, 1, 16, 16, 128, 20, 8, 160, None) == 1
    assert L.icaf_dmff_pool_tokens_f32(one, one, 128, one, one, one, one, one, 1, 16, 16, 128, 8, 8, 56, None) == 1
    assert L.icaf_dmff_pool_tokens_f32(None, one, 128, one, one, one, one, one, 1, 16, 16, 128, 8, 8, 64, None) == 1
    assert L.icaf_dmff_pool_tokens_bwd_f32(one, one, 128, one, one, one, one, one, 1, 16, 16, 128, 8, 8, 64, one, ws - 1, None) == 1
    assert b"workspace" in L.icaf_last_error()
    assert L.icaf_dmff_pool_tokens_bwd_f32(one, one, 128, one, one, one, one, one, 1, 16, 16, 128, 8, 8, 64, ctypes.c_void_p(20), ws, None) == 1
    assert L.icaf_dmff_pool_tokens_bwd_f32(one, one, 128, one, one, one, one, one, 1, 320, 320, 128, 2, 2, 8, one, 1 << 20, None) == 2
    # tail: concat pitch narrower than 2C, grid larger than the map
    assert L.icaf_dmff_upsample_cat_f32(one, one, 64, one, one, 128, one, 128, 1, 16, 16, 128, 8, 8, None) == 1
    assert L.icaf_dmff_upsample_cat_f32(one, one, 64, one, one, 128, one, 256, 1, 4, 4, 128, 8, 8, None) == 1
    assert L.icaf_dmff_upsample_cat_bwd_f32(one, 256, one, one, 1, 16, 16, 128, 8, 8, 60, None) == 1
    # LayerNorm: C > 2048 / C % 8; backward workspace without the row statistics
    assert L.icaf_layernorm_f32(one, None, one, one, None, None, one, None, 10, 4096, 1e-5, None) == 2
    assert L.icaf_layernorm_f32(one, one, one, one, None, None, one, one, 10, 64, 1e-5, None) == 1
    tw = L.icaf_train_workspace_bytes(64)
    assert L.icaf_layernorm_bwd_f32(one, one, one, one, one, one, 10, 64, 1e-5, 1.0, 0, one, tw, None) == 1
    assert b"workspace" in L.icaf_last_error()
    assert L.icaf_layernorm_bwd_f32(one, one, one, one, one, one, 10, 60, 1e-5, 1.0, 0, one, 1 << 30, None) == 1
    # axpby: n % 8, y without b; dot: short workspace, C % 8; colsum: short workspace
    assert L.icaf_axpby_f32(one, None, one, None, one, 0, 12, None) == 1
    assert L.icaf_axpby_f32(one, one, one, None, one, 1, 16, None) == 1
    assert L.icaf_dot_f32(one, one, 1, 10, 64, one, 1.0, 0, one, tw - 4, None) == 1
    assert L.icaf_dot_f32(one, one, 0, 10, 60, one, 1.0, 0, one, 1 << 30, None) == 1
    assert L.icaf_colsum_f32(one, 10, 64, one, 1.0, 0, one, 64 * 64 * 4 - 4, None) == 1
    assert L.icaf_kernel_launches() == n0


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


# the fp32-stream instantiations (mangled-name fragments, with their count)
NEW_KERNELS = {"axpby_f32_kernel": 2, "layernorm_kernelIf": 1, "dmff_upsample_cat_kernelIf": 1, "dmff_upsample_cat_bwd_kernelIf": 1,
               "dmff_pool_tokens_bwd_kernelIf": 1, "dmff_pool_tokens_f32_kernel": 1, "chan_partial_kernelILi2Ef": 1,
               "chan_partial_kernelILi3Ef": 2, "ln_bwd_kernelIf": 1, "colsum_partial_kernelIf": 1}


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_fp32_stream_kernels_are_spill_free(tmp_path):
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    procs = [(s, subprocess.Popen([_nvcc(), *flags, "-Xptxas", "-v", "-c", os.path.join(B.CSRC, s), "-o", str(tmp_path / (s + ".o"))],
                                  stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)) for s in ("dmff.cu", "train.cu", "wgrad.cu")]
    found = collections.Counter()
    spills = []
    for s, p in procs:
        log, _ = p.communicate(timeout=900)
        assert p.returncode == 0, log
        entry = None
        for line in log.splitlines():
            m = re.search(r"Compiling entry function '(\w+)'", line)
            if m:
                entry = m.group(1)
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and entry:
                keys = [k for k in NEW_KERNELS if k in entry]
                found.update(keys)
                if keys and (int(m.group(1)) or int(m.group(2))):
                    spills.append((entry, m.group(1), m.group(2)))
                entry = None
    assert dict(found) == NEW_KERNELS, found
    assert not spills, spills
