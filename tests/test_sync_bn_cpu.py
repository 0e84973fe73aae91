"""Synchronised BatchNorm (train.py --sync-bn) on the host: argument refusals of the two-phase entry points, the conversion
TrainStep(sync_bn=True) makes and the optimiser groups around it, and -- in a gloo world of two processes, on `meta`
tensors -- which launches and exchanges a converted model's training step issues."""
import ctypes
import os
import socket
import traceback

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

CFG = "yolov5s_Transfusion_kaist"
N_BN = 93


def test_two_phase_entry_points_refuse_bad_arguments():
    from icafusion_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(256)                     # never dereferenced: every call below is refused on the host
    ws = int(L.icaf_train_workspace_bytes(64))
    cases = [
        ("icaf_bn_act_fwd_stats", lambda rows, C, w, x=p: L.icaf_bn_act_fwd_stats(x, rows, C, p, p, w, None)),
        ("icaf_bn_act_fwd_apply", lambda rows, C, w, x=p: L.icaf_bn_act_fwd_apply(x, p, p, None, None, p, p, p, p, rows, C, 1e-3, 0.03, 1, p, w, None)),
        ("icaf_bn_act_bwd_sums", lambda rows, C, w, x=p: L.icaf_bn_act_bwd_sums(x, p, p, p, p, p, None, None, p, rows, C, 1, 1.0, 0, p, w, None)),
        ("icaf_bn_act_bwd_apply", lambda rows, C, w, x=p: L.icaf_bn_act_bwd_apply(x, p, p, p, p, p, p, p, p, rows, C, 1, p, w, None)),
    ]
    n0 = L.icaf_kernel_launches()
    for name, call in cases:
        short = name[len("icaf_"):].encode()
        for args, what in (((10, 64, ws, None), b"bad argument"), ((10, 60, ws), b"bad argument"), ((0, 64, ws), b"bad argument"),
                           ((10, 64, ws - 4), b"workspace too small")):
            rc = call(*args)
            msg = L.icaf_last_error()
            assert rc == 1 and short in msg and what in msg, (name, args, rc, msg)
    assert L.icaf_kernel_launches() == n0
    # the backward's phase 2 needs the summed count as well
    assert L.icaf_bn_act_bwd_apply(p, p, p, p, p, p, p, None, p, 10, 64, 1, p, ws, None) == 1


def _bn_weights(model):
    return [m.weight for m in model.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]


def test_param_groups_of_a_converted_model_equal_the_unconverted_groups():
    from icafusion_b200 import Model
    from icafusion_b200.trainer import freeze_dead_parameters, param_groups
    model = Model(CFG)
    freeze_dead_parameters(model)
    before = [[id(p) for p in g] for g in param_groups(model)]
    assert len(before[0]) == N_BN
    model = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert sum(isinstance(m, nn.SyncBatchNorm) for m in model.modules()) == N_BN
    assert [[id(p) for p in g] for g in param_groups(model)] == before


def test_world_size_1_leaves_the_model_unconverted():
    from icafusion_b200 import Model
    from icafusion_b200.trainer import TrainStep
    model = Model(CFG)
    ts = TrainStep(model, None, total_batch_size=4, world_size=1, imgsz=320, sync_bn=True)
    assert ts.raw_model is model
    assert sum(type(m) is nn.BatchNorm2d for m in model.modules()) == N_BN
    assert not any(isinstance(m, nn.SyncBatchNorm) for m in model.modules())


def _dry_step(model):
    from icafusion_b200 import ops
    rgb = torch.empty(2, 3, 320, 320, dtype=torch.uint8, device="meta")
    with ops.dry_run() as dr:
        pred = model(rgb, rgb)
        torch.autograd.backward(pred, [torch.empty_like(p) for p in pred])
    return [(name, args, work) for name, args, work in dr.records]


def _scenario(rank):
    from icafusion_b200 import Model
    from icafusion_b200.trainer import TrainStep
    out = {}
    # TrainStep(sync_bn=True): groups first, then the conversion, then DDP (train.py:124-131, 195-198, 233)
    model = Model(CFG)
    keys = list(model.state_dict().keys())
    bn_w = _bn_weights(model)
    wrapped = []

    class StandInDDP(nn.Module):                 # torch's DDP refuses SyncBatchNorm on CPU modules: record what it is handed
        def __init__(self, module, **kw):
            super().__init__()
            wrapped.append(sum(isinstance(m, nn.SyncBatchNorm) for m in module.modules()))
            self.module = module

    keep = torch.nn.parallel.DistributedDataParallel
    torch.nn.parallel.DistributedDataParallel = StandInDDP
    try:
        ts = TrainStep(model, None, total_batch_size=4, world_size=2, imgsz=320, sync_bn=True)
    finally:
        torch.nn.parallel.DistributedDataParallel = keep
    out["wrapped"] = wrapped
    out["n_sync"] = sum(isinstance(m, nn.SyncBatchNorm) for m in ts.raw_model.modules())
    out["n_plain"] = sum(type(m) is nn.BatchNorm2d for m in ts.raw_model.modules())
    out["group0_same"] = [id(p) for p in ts.optimizer.param_groups[0]["params"]] == [id(p) for p in bn_w]
    out["keys_same"] = list(ts.raw_model.state_dict().keys()) == keys
    # dry-run walks of the training step: converted (world-2 group), converted over a one-rank group, unconverted
    plain = _dry_step(Model(CFG).to("meta").train())
    conv = _dry_step(nn.SyncBatchNorm.convert_sync_batchnorm(Model(CFG).to("meta").train()))
    solo = [dist.new_group([0]), dist.new_group([1])][rank]            # every rank takes part in creating each group
    one = _dry_step(nn.SyncBatchNorm.convert_sync_batchnorm(Model(CFG).to("meta").train(), solo))
    out["plain"] = [n for n, _, _ in plain]
    out["one"] = [n for n, _, _ in one]
    out["plain_bytes"] = [w.get("bytes") for _, _, w in plain]
    out["one_bytes"] = [w.get("bytes") for _, _, w in one]
    seq = []
    for i, (name, args, work) in enumerate(conv):
        if name in ("icaf_bn_act_fwd_stats", "icaf_bn_act_bwd_sums"):
            C = int(args[2]) if name == "icaf_bn_act_fwd_stats" else int(args[10])
            n2, a2, w2 = conv[i + 1]
            n3 = conv[i + 2][0]
            seq.append((name, C, n2, a2[0].numel(), w2["group"] is dist.group.WORLD or w2["group"] is None, n3))
    out["conv_names"] = [n for n, _, _ in conv]
    out["seq"] = seq
    return out


def _worker(rank, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        q.put((rank, _scenario(rank)))
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def test_sync_bn_world2_conversion_and_dry_run_exchanges():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        got = dict(q.get(timeout=600) for _ in procs)
        for p in procs:
            p.join(120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
    assert all(isinstance(v, dict) for v in got.values()), got
    res = got[0]
    assert res["n_sync"] == N_BN and res["n_plain"] == 0 and res["wrapped"] == [N_BN]
    assert res["group0_same"] and res["keys_same"]
    # a one-rank group: exactly the unconverted model's launches
    assert res["one"] == res["plain"] and res["one_bytes"] == res["plain_bytes"]
    # world 2: every BatchNorm layer runs both phases in each direction with one exchange in between, and nothing else changes
    names = res["conv_names"]
    n_fwd = res["plain"].count("icaf_bn_act_fwd")
    assert n_fwd == res["plain"].count("icaf_bn_act_bwd") == N_BN
    assert "icaf_bn_act_fwd" not in names and "icaf_bn_act_bwd" not in names
    for n in ("icaf_bn_act_fwd_stats", "icaf_bn_act_fwd_apply", "icaf_bn_act_bwd_sums", "icaf_bn_act_bwd_apply"):
        assert names.count(n) == N_BN, n
    assert names.count("all_reduce") == 2 * N_BN
    assert len(res["seq"]) == 2 * N_BN
    for phase1, C, n2, numel, world, n3 in res["seq"]:
        assert n2 == "all_reduce" and world
        if phase1 == "icaf_bn_act_fwd_stats":
            assert numel == 2 * C + 1 and n3 == "icaf_bn_act_fwd_apply"
        else:
            assert numel == 2 * C and n3 == "icaf_bn_act_bwd_apply"
    strip = {"icaf_bn_act_fwd_stats": "icaf_bn_act_fwd", "icaf_bn_act_bwd_sums": "icaf_bn_act_bwd"}
    rest = [strip.get(n, n) for n in names if n not in ("all_reduce", "icaf_bn_act_fwd_apply", "icaf_bn_act_bwd_apply")]
    assert rest == res["plain"]
