"""TrainStep's train.py options on CPU: gradient accumulation over the nominal batch (train.py:123-125, 314-320, 344-352),
--adam (train.py:133-141), and the oracle's focal loss and accumulating loop against goldens of the real reference.  The
step runs a stand-in forward here (the CUDA kernels cannot run without a GPU): what is under test is when the optimiser,
GradScaler and EMA move, what .grad holds, and DDP's all-reduce over accumulated gradients at world size 2 over gloo."""
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from conftest import load_golden


class _Detect(nn.Module):
    nl, nc, na = 3, 1, 3

    def __init__(self):
        super().__init__()
        self.register_buffer("anchors", torch.ones(3, 3, 2))


class _Tiny(nn.Module):
    """What TrainStep reads from a detector (model.model[-1], BatchNorm / weight / bias groups), with a stand-in forward that
    touches every parameter nonlinearly and depends on the batch."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.model = nn.ModuleList([nn.Conv2d(3, 4, 1), nn.BatchNorm2d(4), nn.Linear(4, 2), _Detect()])

    def forward(self, rgb, ir):
        return sum(torch.tanh(p * rgb + ir).square().sum() for p in self.parameters())


def _step(world_size=1, total_batch_size=16, **kw):
    from icafusion_b200.trainer import TrainStep
    model = _Tiny()
    ts = TrainStep(model, None, total_batch_size=total_batch_size, world_size=world_size, imgsz=320, **kw)
    ts.compute_loss = lambda pred, targets: (pred, torch.zeros(4))
    return model, ts


def _data(i, rank=0):
    return torch.tensor(0.3 + 0.1 * i + 0.05 * rank), torch.tensor(0.2 - 0.03 * i + 0.07 * rank)


def _transcription(model, batches, accumulate, world=1):
    """train.py:117-141 and 344-352 written out on the stand-in: SGD groups, then per batch backward and, when
    ni % accumulate == 0, step + zero_grad + EMA update.  batches[ni - 1] is a list of one (rgb, ir) per rank; the gradient DDP
    forms from `loss * world_size` on each rank is the sum of the ranks' gradients."""
    from icafusion_b200.trainer import HYP_SCRATCH, ModelEMA, param_groups
    hyp = dict(HYP_SCRATCH)
    hyp["weight_decay"] *= 16 * accumulate / 64
    pg0, pg1, pg2 = param_groups(model)
    opt = torch.optim.SGD(pg0, lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)
    opt.add_param_group({"params": pg1, "weight_decay": hyp["weight_decay"]})
    opt.add_param_group({"params": pg2})
    ema = ModelEMA(model)
    opt.zero_grad()
    for ni, per_rank in enumerate(batches, 1):
        loss = sum(model(rgb, ir) for rgb, ir in per_rank)
        loss.backward()
        if ni % accumulate == 0:
            opt.step()
            opt.zero_grad()
            ema.update(model)
    return {k: v.detach().clone() for k, v in model.state_dict().items()}, ema


@pytest.mark.parametrize("tbs", [4, 8, 16, 64, 128])
def test_accumulate_at_is_train_py_warmup_ramp(tbs):
    _, ts = _step(total_batch_size=tbs)
    nbs = 64
    assert ts.accumulate == max(round(nbs / tbs), 1)
    for nw in (0, 1, 7, 1000):
        for ni in sorted({0, 1, 2, 3, nw // 3, nw // 2, nw - 1, nw, nw + 1, 5 * nw + 3} - {-1}):
            want = max(1, np.interp(ni, [0, nw], [1, nbs / tbs]).round()) if ni <= nw else ts.accumulate     # train.py:317
            assert ts.accumulate_at(ni, nw) == want, (tbs, nw, ni)


def test_accumulating_calls_add_up_and_only_stepping_calls_move_the_optimiser():
    from icafusion_b200.trainer import ModelEMA
    model, ts = _step(ema=True)
    live = [p for p in model.parameters() if p.requires_grad]
    calls = []

    class Scaler:               # GradScaler (disabled on CPU) with a record of what the step asked of it
        def __init__(self, inner):
            self.inner = inner

        def scale(self, x):
            return self.inner.scale(x)

        def step(self, opt):
            calls.append("step")
            return self.inner.step(opt)

        def update(self):
            calls.append("update")
            return self.inner.update()
    ts.scaler = Scaler(ts.scaler)
    before = [p.detach().clone() for p in live]
    want = [torch.zeros_like(p) for p in live]
    for i in range(3):
        rgb, ir = _data(i)
        ref = _Tiny()
        ref.load_state_dict(model.state_dict())
        for w, g in zip(want, torch.autograd.grad(ref(rgb, ir), [p for p in ref.parameters() if p.requires_grad])):
            w += g
        ts(rgb, ir, None, optimizer_step=False)
        assert calls == [] and ts.ema.updates == 0 and not ts.optimizer.state
        assert all(torch.equal(p, b) for p, b in zip(live, before))
        assert all(torch.allclose(p.grad, w, rtol=1e-6, atol=1e-7) for p, w in zip(live, want))
    ts(*_data(3), None)
    assert calls == ["step", "update"] and ts.ema.updates == 1
    assert all(p.grad is None for p in live)
    assert not all(torch.equal(p, b) for p, b in zip(live, before))
    assert isinstance(ts.ema, ModelEMA)


def test_two_windows_of_four_equal_train_py():
    """total batch 16 -> accumulate 4: eight calls stepping at ni % 4 == 0 leave the parameters and the EMA of train.py's loop."""
    model, ts = _step(ema=True)
    assert ts.accumulate == 4
    ref_model = _Tiny()
    ref_model.load_state_dict(model.state_dict())
    for ni in range(1, 9):
        ts(*_data(ni), None, optimizer_step=(ni % ts.accumulate_at(ni, 0) == 0))
    want, ema = _transcription(ref_model, [[_data(ni)] for ni in range(1, 9)], 4)
    got = model.state_dict()
    for k in want:
        assert torch.allclose(got[k], want[k], rtol=1e-6, atol=1e-7), k
    for k, v in ema.ema.state_dict().items():
        assert torch.allclose(ts.ema.ema.state_dict()[k], v, rtol=1e-6, atol=1e-7), k
    assert ts.ema.updates == ema.updates == 2
    # a partial window discarded by zero_grad() (train.py:291) leaves no trace in the next step
    ts(*_data(9), None, optimizer_step=False)
    ts.zero_grad()
    assert all(p.grad is None for p in model.parameters())


def _ddp_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        model, ts = _step(world_size=world)
        for ni in range(1, 9):
            ts(*_data(ni, rank), None, optimizer_step=(ni % ts.accumulate == 0))
        q.put((rank, {k: v.detach().numpy().copy() for k, v in model.state_dict().items()}))     # (numpy: outlives the process)
    finally:
        dist.destroy_process_group()


def test_ddp_world2_accumulation_all_reduces_every_micro_step():
    """Two gloo ranks, DDP all-reducing on every backward (no no_sync): after two windows of four both ranks hold the
    parameters of train.py's loop on the sum of the ranks' gradients."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=400) for _ in procs)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    want, _ = _transcription(_Tiny(), [[_data(ni, r) for r in range(2)] for ni in range(1, 9)], 4, world=2)
    for r in range(2):
        for k in want:
            assert torch.allclose(torch.from_numpy(res[r][k]), want[k], rtol=1e-5, atol=1e-6), (r, k)


def test_adam_optimiser_is_train_py_133_141():
    from icafusion_b200.trainer import HYP_SCRATCH, param_groups
    model, ts = _step(adam=True)
    hyp = dict(HYP_SCRATCH)
    hyp["weight_decay"] *= 16 * 4 / 64
    pg0, pg1, pg2 = param_groups(model)
    ref = torch.optim.Adam(pg0, lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))          # train.py:133-134
    ref.add_param_group({"params": pg1, "weight_decay": hyp["weight_decay"]})
    ref.add_param_group({"params": pg2})
    assert type(ts.optimizer) is torch.optim.Adam
    assert len(ts.optimizer.param_groups) == len(ref.param_groups) == 3
    for g, r in zip(ts.optimizer.param_groups, ref.param_groups):
        assert [id(p) for p in g["params"]] == [id(p) for p in r["params"]]
        assert {k: v for k, v in g.items() if k != "params"} == {k: v for k, v in r.items() if k != "params"}
    assert ts.optimizer.param_groups[0]["betas"] == (0.937, 0.999)
    assert [g["weight_decay"] for g in ts.optimizer.param_groups] == [0, hyp["weight_decay"], 0]
    _, sgd = _step()
    assert type(sgd.optimizer) is torch.optim.SGD and sgd.optimizer.param_groups[0]["nesterov"]


def test_focal_loss_oracle_matches_reference_golden():
    """oracle.focal_loss.compute_loss reproduces the REAL reference's ComputeLoss with fl_gamma 1.5 and 2.0
    (tests/golden/loss_focal_cases.npz, oracle/gen_golden_loss_focal.py): outputs and loss.backward()."""
    from oracle import focal_loss as FL
    from oracle.gen_golden_loss import grad_fingerprint, synth_case
    m, d = load_golden("loss_focal_cases")
    assert {cs["hyp"]["fl_gamma"] for cs in m["cases"]} == {1.5, 2.0} and len(m["cases"]) == 8
    for cs in m["cases"]:
        key = cs["key"]
        p, t = synth_case(cs["name"], cs["nc"], cs["B"], cs["nt"])
        assert np.array_equal(t, d[f"{key}_targets"])
        pt = [torch.from_numpy(x).requires_grad_(True) for x in p]
        loss, items = FL.compute_loss(pt, torch.from_numpy(t), torch.from_numpy(d[f"{key}_anchors"]), cs["hyp"], cs["gr"])
        got = np.concatenate([loss.detach().numpy().reshape(1), items.detach().numpy()])
        assert np.allclose(got, d[f"{key}_out"], rtol=2e-5, atol=1e-6), (key, got, d[f"{key}_out"])
        loss.sum().backward()
        g2 = d[f"{key}_grad2"]
        assert np.abs(pt[2].grad.numpy() - g2).max() <= 2e-5 * np.abs(g2).max(), key
        for lvl, x in enumerate(pt):
            want = d[f"{key}_gproj{lvl}"]
            assert np.allclose(grad_fingerprint(x.grad.numpy(), lvl), want, rtol=1e-4, atol=1e-6 * want[0]), (key, lvl)
    # fl_gamma = 0 is the plain-BCE oracle, unchanged
    from oracle import icaf_oracle as O
    p, t = synth_case("kaist_nc1", 1, 4, 37)
    cs = m["cases"][0]
    hyp = dict(cs["hyp"], fl_gamma=0.0)
    a = FL.compute_loss([torch.from_numpy(x) for x in p], torch.from_numpy(t), torch.from_numpy(d["kaist_nc1_g1.5_anchors"]), hyp)
    b = O.compute_loss([torch.from_numpy(x) for x in p], torch.from_numpy(t), torch.from_numpy(d["kaist_nc1_g1.5_anchors"]), hyp)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_accumulation_golden_is_reproduced_by_the_oracle():
    """The oracle's accumulating loop (two optimiser steps over two micro-batches each) reproduces the REAL reference's
    (tests/golden/train_accumulate_yolov5s_320.npz, oracle/gen_golden_train_accumulate.py)."""
    from icafusion_b200.cfg import load_cfg
    from oracle import synth
    from oracle.gen_golden_train import fingerprint
    from oracle.gen_golden_train_accumulate import batches, oracle_loop
    m, d = load_golden("train_accumulate_yolov5s_320")
    assert m["accumulate"] == 2 and m["micro_batches"] == 4
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_kaist")
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    upd, state, ema, losses = oracle_loop(sd, cfg, m, batches())
    assert np.allclose(losses, d["losses"], rtol=1e-4), (losses, d["losses"])
    grouped = sorted(k for g in m["groups"] for k in g)
    assert sorted(upd) == grouped
    # floor: parameters whose gradient is mathematically zero (key-projection biases, the dead parameters) move by rounding
    # noise only, on both sides.  fp32 on both sides; the first window's update agrees to 2e-5 (relative L2), the second
    # window's gradients are taken at the stepped weights and agree less closely: 1.0e-3 over all fingerprints, 6.1e-3 for
    # the worst tensor (observed)
    floor = 1e-3 * max(float(d["u:" + k][0]) for k in grouped)
    fp = {k: fingerprint(upd[k].numpy(), "u:" + k) for k in grouped}
    worst = max(float(np.abs(fp[k] - d["u:" + k]).max() / max(d["u:" + k][0], floor)) for k in grouped)
    rel = math.sqrt(sum(float(((fp[k] - d["u:" + k]) ** 2).sum()) for k in grouped) / sum(float((d["u:" + k] ** 2).sum()) for k in grouped))
    assert rel < 3e-3 and worst < 2e-2, (rel, worst)
    norm = math.sqrt(sum(float(d["e:" + k][0]) ** 2 for k in ema if "e:" + k in d))
    worst_e = max(float(np.abs(fingerprint((ema[k].double() - sd[k].double()).numpy(), "e:" + k) - d["e:" + k]).max())
                  for k in ema if "e:" + k in d) / norm
    assert worst_e < 1e-4, worst_e
    for k in m["bn_probes"]:
        assert np.allclose(state[k + ".running_mean"].numpy(), d["rm:" + k], rtol=1e-4, atol=1e-6), k
        assert np.allclose(state[k + ".running_var"].numpy(), d["rv:" + k], rtol=1e-4, atol=1e-6), k
    assert {k: int(v) for k, v in state.items() if k.endswith("num_batches_tracked")} == m["num_batches_tracked"]
