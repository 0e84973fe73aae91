"""The device optimiser step on the host (no GPU): the C ABI of icaf_amp_unscale / icaf_sgd_step / icaf_adam_step /
icaf_amp_update_scale / icaf_ema_update and its argument checks, the tensor tables DeviceOptimizerStep builds for train.py's
parameter groups and the EMA, Adam's bias-correction rows, and the fixed launch list of the step graph (ops.dry_run)."""
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

from conftest import ROOT

ENTRY_POINTS = ["icaf_optim_table_bytes", "icaf_amp_unscale", "icaf_sgd_step", "icaf_adam_step", "icaf_amp_update_scale",
                "icaf_ema_update"]


def test_entry_points_declared_exported_and_bound():
    from icafusion_b200 import _lib
    src = open(os.path.join(ROOT, "include", "icaf_b200.h")).read()
    L = _lib.lib()
    for name in ENTRY_POINTS:
        assert re.search(rf"\b{name}\s*\(", src), name
        assert hasattr(L, name) and name in _lib.SIGNATURES, name
    assert int(re.search(r"#define ICAF_OPTIM_CHUNK (\d+)", src).group(1)) == _lib.OPTIM_CHUNK
    assert int(re.search(r"#define ICAF_OPTIM_HYPER (\d+)", src).group(1)) == _lib.OPTIM_HYPER
    assert ctypes.sizeof(_lib.OptimTensor) == 64
    assert L.icaf_optim_table_bytes(0) == 0 and L.icaf_optim_table_bytes(3) == 3 * 64


def test_entry_points_refuse_bad_arguments_before_any_launch():
    from icafusion_b200 import _lib
    L = _lib.lib()
    P = ctypes.c_void_p
    one = P(256)                              # non-null, 16-byte aligned, never dereferenced: validation fails first
    n0 = L.icaf_kernel_launches()
    nb = L.icaf_optim_table_bytes(4)
    # null pointers
    assert L.icaf_amp_unscale(None, nb, 4, 8, one, one, None) == 1 and b"null" in L.icaf_last_error()
    assert L.icaf_amp_unscale(one, nb, 4, 8, None, one, None) == 1
    assert L.icaf_sgd_step(one, nb, 4, 8, None, 0, 3, one, None) == 1
    assert L.icaf_sgd_step(one, nb, 4, 8, one, 0, 3, None, None) == 1
    assert L.icaf_adam_step(one, nb, 4, 8, one, 0, 3, None, 16, one, None) == 1
    assert L.icaf_amp_update_scale(None, one, one, 2.0, 0.5, 2000, None) == 1
    assert L.icaf_ema_update(one, nb, 4, 8, None, None) == 1
    # a table that does not match its sizes (or is misaligned)
    assert L.icaf_amp_unscale(one, nb - 1, 4, 8, one, one, None) == 1 and b"icaf_optim_table_bytes" in L.icaf_last_error()
    assert L.icaf_sgd_step(one, nb, 0, 8, one, 0, 3, one, None) == 1
    assert L.icaf_ema_update(one, nb, 4, -1, one, None) == 1
    assert L.icaf_adam_step(P(264), nb, 4, 8, one, 0, 3, one, 16, one, None) == 1 and b"aligned" in L.icaf_last_error()
    # a bad group index
    for g, n in ((3, 3), (-1, 3), (0, 0)):
        assert L.icaf_sgd_step(one, nb, 4, 8, one, g, n, one, None) == 1 and b"group" in L.icaf_last_error()
        assert L.icaf_adam_step(one, nb, 4, 8, one, g, n, one, 16, one, None) == 1
    assert L.icaf_adam_step(one, nb, 4, 8, one, 0, 3, one, 1, one, None) == 1       # bias-correction table too short
    assert L.icaf_amp_update_scale(one, one, one, 2.0, 0.5, 0, None) == 1
    assert L.icaf_amp_update_scale(one, one, one, 1.0, 0.5, 2000, None) == 1
    assert L.icaf_kernel_launches() == n0


def test_adam_bias_corrections_equal_torch_expressions():
    """Row s is what torch's _multi_tensor_adam computes in Python for a float32 step tensor holding s, bit for bit."""
    from icafusion_b200.trainer import adam_bias_corrections
    for b1, b2 in ((0.937, 0.999), (0.9, 0.999), (0.8, 0.99)):
        tab = adam_bias_corrections(b1, b2, 3000)
        for s in list(range(1, 40)) + [999, 1000, 2047, 2999]:
            step = torch.tensor(float(s), dtype=torch.float32).item()          # torch.optim.adam._get_value
            bc1 = 1 - b1 ** step
            bc2_sqrt = (1 - b2 ** step) ** 0.5
            assert tab[s, 0] == bc1 and tab[s, 1] == bc2_sqrt, s
            assert (lr := 0.01) / tab[s, 0] * -1 == (lr / bc1) * -1


def _meta_train_step(size: str, adam: bool):
    from icafusion_b200 import Model
    from icafusion_b200.trainer import TrainStep
    model = Model(f"yolov5{size}_Transfusion_kaist").train()          # host tensors; the step's own buffers go to `meta`
    ts = TrainStep(model, None, total_batch_size=16, imgsz=640, ema=True, adam=adam)
    for g in ts.optimizer.param_groups:
        for p in g["params"]:
            p.grad = torch.empty_like(p)
    ts.scaler = types.SimpleNamespace(is_enabled=lambda: True, _scale=torch.empty(1, device="meta"),
                                      _growth_tracker=torch.empty(1, dtype=torch.int32, device="meta"), _growth_factor=2.0,
                                      _backoff_factor=0.5, _growth_interval=2000)
    return model, ts


def _device_step(ts, model):
    from icafusion_b200 import ops
    from icafusion_b200.trainer import DeviceOptimizerStep
    with ops.dry_run() as dr:
        opt = DeviceOptimizerStep(ts.optimizer, ts.scaler, ts.ema, model, "meta")
        assert not dr.records                                   # building the tables launches nothing
        opt.enqueue()
    return opt, dr.records


def test_tables_hold_the_eager_tensors():
    """yolov5s: the table lists pg0 / pg1 / pg2 in group order with the 30 dead and the 18 group-less parameters left out, each
    row (param, .grad, momentum buffer) of the eager optimiser; the EMA table pairs every floating EMA entry with the model's."""
    from icafusion_b200 import _lib
    from icafusion_b200.trainer import dead_parameters, param_groups
    model, ts = _meta_train_step("s", adam=False)
    opt, _ = _device_step(ts, model)
    pg = param_groups(model)
    assert [len(g) for g in pg] == [len(g["params"]) for g in ts.optimizer.param_groups]
    flat = [p for g in pg for p in g]
    grouped = {id(p) for p in flat}
    named = dict(model.named_parameters())
    loose = [k for k, p in named.items() if id(p) not in grouped]
    assert len(dead_parameters(model)) == 30 and len(loose) == 30 + 18
    assert set(dead_parameters(model)) <= set(loose)
    rows = opt.table.rows
    assert len(rows) == len(flat) == opt.table.n
    lo = 0
    for gi, g in enumerate(pg):
        assert opt.table.ranges[gi] == (lo, lo + len(g))
        lo += len(g)
    chunks = 0
    for r, p in zip(rows, flat):
        assert r[0] is p and r[1] is p.grad and r[2] is ts.optimizer.state[p]["momentum_buffer"] and r[3] is None and r[4] is None
        assert r[2].shape == p.shape
        chunks += -(-p.numel() // _lib.OPTIM_CHUNK)
    assert opt.table.chunk0[-1] == chunks
    assert opt.table.block.numel() == 64 * len(rows)
    esd, msd = ts.ema.ema.state_dict(), model.state_dict()
    want = [k for k, v in esd.items() if v.dtype.is_floating_point]
    assert not any(k.endswith("num_batches_tracked") for k in want)
    assert any(k.endswith("running_var") for k in want)
    assert len(opt.ema_table.rows) == len(want)
    for (v, src, *_), k in zip(opt.ema_table.rows, want):
        assert v.shape == esd[k].shape and src.shape == msd[k].shape
    # a group's span covers exactly its rows and chunks
    addr0 = opt.table.span()[0].value or 0
    for gi in range(3):
        a, nbytes, n, c = opt.table.span(gi)
        lo, hi = opt.table.ranges[gi]
        assert (a.value or 0) - addr0 == 64 * lo and n == hi - lo and c == opt.table.chunk0[hi] - opt.table.chunk0[lo]
        assert nbytes.value >= _lib.lib().icaf_optim_table_bytes(n)


def test_adam_state_moves_to_the_device_rows():
    model, ts = _meta_train_step("s", adam=True)
    opt, _ = _device_step(ts, model)
    for r in opt.table.rows:
        st = ts.optimizer.state[r[0]]
        assert r[2] is st["exp_avg"] and r[3] is st["exp_avg_sq"] and r[4] is st["step"]
        assert st["step"].device.type == "meta" and st["step"].dtype == torch.float32 and st["step"].numel() == 1
    assert tuple(opt.bias_corr.shape) == (3, opt.BIAS_STEPS, 2)


@pytest.mark.parametrize("adam", [False, True])
def test_step_launch_list_is_fixed(adam):
    """The step graph is unscale, one optimiser launch per group, the scale update and the EMA update, for yolov5s and
    yolov5l alike (hundreds of tensors more)."""
    lists = []
    for size in ("s", "l"):
        model, ts = _meta_train_step(size, adam)
        opt, records = _device_step(ts, model)
        lists.append(([(name, args[5] if name in ("icaf_sgd_step", "icaf_adam_step") else None) for name, args, _ in records],
                      opt.table.n))
    (l0, n0), (l1, n1) = lists
    step = "icaf_adam_step" if adam else "icaf_sgd_step"
    assert l0 == l1 == [("icaf_amp_unscale", None), (step, 0), (step, 1), (step, 2), ("icaf_amp_update_scale", None),
                        ("icaf_ema_update", None)]
    assert n1 > n0 + 200
