"""The device optimiser step against torch on the GPU: GradScaler's unscale + nesterov SGD / Adam, the EMA update and the
scale update bit for bit; non-finite gradients; GraphedTrainStep's step graph against the eager TrainStep over a train.py-shaped
loop; no host synchronisation in a stepping call; two ranks under NCCL."""
import copy
import warnings

import numpy as np
import pytest
import torch

from helpers import load_synth
from oracle import synth
from oracle.gen_golden_train import synth_targets

pytestmark = pytest.mark.gpu


def _group_shapes():
    """yolov5s's three train.py groups (BatchNorm weights, other weights, biases), as shapes."""
    from icafusion_b200 import Model
    from icafusion_b200.trainer import freeze_dead_parameters, param_groups
    m = Model("yolov5s_Transfusion_kaist")
    freeze_dead_parameters(m)
    return [[tuple(p.shape) for p in g] for g in param_groups(m)]


def _twin_params(dev, seed):
    """Two identical sets of yolov5s-shaped parameters (three groups) with random values and gradients."""
    g = torch.Generator(device=dev).manual_seed(seed)
    sets = ([], [])
    for shapes in _group_shapes():
        grp = ([], [])
        for s in shapes:
            p = torch.randn(s, device=dev, generator=g) * 0.05
            gr = torch.randn(s, device=dev, generator=g) * 3000.0
            for k in (0, 1):
                q = torch.nn.Parameter(p.clone())
                q.grad = gr.clone()
                grp[k].append(q)
        for k in (0, 1):
            sets[k].append(grp[k])
    return sets


def _scaler(dev, **kw):
    sc = torch.amp.GradScaler("cuda", **kw)
    sc.scale(torch.ones((), device=dev))              # creates _scale / _growth_tracker
    return sc


def _sgd(groups, lrs, moms, wd):
    opt = torch.optim.SGD(groups[0], lr=lrs[0], momentum=moms[0], nesterov=True)
    opt.add_param_group({"params": groups[1], "weight_decay": wd, "lr": lrs[1], "momentum": moms[1]})
    opt.add_param_group({"params": groups[2], "lr": lrs[2], "momentum": moms[2]})
    return opt


def _new_grads(groups_pair, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    for ga, gb in zip(*groups_pair):
        for a, b in zip(ga, gb):
            x = torch.randn(a.shape, device=dev, generator=g) * 3000.0
            a.grad.copy_(x)
            b.grad.copy_(x)


def test_sgd_step_equals_torch(cuda_device):
    """One unscale + nesterov SGD step over yolov5s's groups (weight decay on pg1, random momentum buffers): parameters and
    momentum buffers torch.equal torch's GradScaler.unscale_ + SGD (foreach)."""
    from icafusion_b200.trainer import DeviceOptimizerStep
    dev = cuda_device
    ref, mine = _twin_params(dev, 1)
    lrs, moms = (0.00731, 0.0123, 0.0911), (0.8423, 0.905, 0.937)
    opts = [_sgd(x, lrs, moms, 0.0005 * 16 * 4 / 64) for x in (ref, mine)]
    g = torch.Generator(device=dev).manual_seed(2)
    for pr, pm in zip((p for grp in ref for p in grp), (p for grp in mine for p in grp)):
        b = torch.randn(pr.shape, device=dev, generator=g)
        opts[0].state[pr]["momentum_buffer"] = b.clone()
        opts[1].state[pm]["momentum_buffer"] = b.clone()
    sc_ref, sc_dev = _scaler(dev, init_scale=4096.0), _scaler(dev, init_scale=4096.0)
    step = DeviceOptimizerStep(opts[1], sc_dev, None, None, dev)
    for it in range(3):
        if it:
            _new_grads((ref, mine), dev, 10 + it)
            for o in opts:
                for j, grp in enumerate(o.param_groups):
                    grp["lr"] *= 0.9
                    grp["momentum"] = moms[j] - 0.01 * it
        sc_ref.unscale_(opts[0])
        sc_ref.step(opts[0])
        sc_ref.update()
        step.stage()
        step.enqueue()
        torch.cuda.synchronize()
        for pr, pm in zip((p for grp in ref for p in grp), (p for grp in mine for p in grp)):
            assert torch.equal(pr, pm), f"step {it}: parameter {tuple(pr.shape)}"
            assert torch.equal(opts[0].state[pr]["momentum_buffer"], opts[1].state[pm]["momentum_buffer"])
        assert sc_ref.state_dict() == sc_dev.state_dict()


def test_adam_steps_equal_torch(cuda_device):
    """Adam (train.py --adam) over steps 1..5, with the lerp's two branches (1 - beta1 below and above 0.5) and weight decay:
    parameters, exp_avg, exp_avg_sq and step torch.equal torch's."""
    from icafusion_b200.trainer import DeviceOptimizerStep
    dev = cuda_device
    ref, mine = _twin_params(dev, 3)
    opts = []
    for x in (ref, mine):
        o = torch.optim.Adam(x[0], lr=0.001, betas=(0.937, 0.999))
        o.add_param_group({"params": x[1], "weight_decay": 0.0005, "betas": (0.3, 0.99)})
        o.add_param_group({"params": x[2], "lr": 0.0031})
        opts.append(o)
    sc_ref, sc_dev = _scaler(dev, init_scale=1024.0), _scaler(dev, init_scale=1024.0)
    step = DeviceOptimizerStep(opts[1], sc_dev, None, None, dev)
    for it in range(5):
        if it:
            _new_grads((ref, mine), dev, 20 + it)
            for o in opts:
                o.param_groups[0]["lr"] = 0.001 * (it + 1)
        sc_ref.step(opts[0])
        sc_ref.update()
        step.stage()
        step.enqueue()
        torch.cuda.synchronize()
        for pr, pm in zip((p for grp in ref for p in grp), (p for grp in mine for p in grp)):
            sr, sm = opts[0].state[pr], opts[1].state[pm]
            assert torch.equal(pr, pm), f"step {it + 1}: parameter {tuple(pr.shape)}"
            assert torch.equal(sr["exp_avg"], sm["exp_avg"]) and torch.equal(sr["exp_avg_sq"], sm["exp_avg_sq"])
            assert float(sr["step"]) == float(sm["step"]) == it + 1 and sm["step"].is_cuda
        assert sc_ref.state_dict() == sc_dev.state_dict()


def _model(dev, seed=1234):
    from icafusion_b200 import Model
    model = Model("yolov5s_Transfusion_kaist")
    load_synth(model, seed)
    model = model.to(dev).train()
    for mod in model.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    return model


def test_ema_update_equals_model_ema(cuda_device):
    """icaf_ema_update against ModelEMA.update at several update counts, BatchNorm running statistics included."""
    from icafusion_b200 import ops
    from icafusion_b200.trainer import ModelEMA
    model = _model(cuda_device)
    ref = ModelEMA(model)
    dev_ema = copy.deepcopy(ref)
    decay = torch.zeros(1, dtype=torch.float64, device=cuda_device)
    msd = model.state_dict()
    tab = ops.OptimTable([(v, msd[k], None, None, None) for k, v in dev_ema.ema.state_dict().items() if v.dtype.is_floating_point],
                         cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(5)
    for updates in (0, 1, 17, 1999, 40000):
        with torch.no_grad():
            for v in msd.values():
                if v.dtype.is_floating_point:
                    v.add_(torch.randn(v.shape, device=cuda_device, generator=g) * 0.01)
        ref.updates = dev_ema.updates = updates
        ref.update(model)
        dev_ema.updates += 1
        decay.fill_(dev_ema.decay(dev_ema.updates))
        ops.ema_update(tab, decay)
        torch.cuda.synchronize()
        for (k, a), b in zip(ref.ema.state_dict().items(), dev_ema.ema.state_dict().values()):
            assert torch.equal(a, b), (updates, k)


def test_scale_update_equals_torch(cuda_device):
    """icaf_amp_update_scale against torch._amp_update_scale_ through growth, backoff and a growth past fp32's range."""
    from icafusion_b200 import ops
    dev = cuda_device
    for start, flags in ((65536.0, [0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0]), (3.0e38, [0, 0, 0, 0, 1, 0])):
        s_ref = torch.full((1,), start, device=dev)
        t_ref = torch.zeros(1, dtype=torch.int32, device=dev)
        s_dev, t_dev = s_ref.clone(), t_ref.clone()
        for f in flags:
            fi = torch.full((1,), float(f), device=dev)
            fd = fi.clone()
            torch._amp_update_scale_(s_ref, t_ref, fi, 2.0, 0.5, 3)
            ops.amp_update_scale(s_dev, t_dev, fd, 2.0, 0.5, 3)
            torch.cuda.synchronize()
            assert torch.equal(s_ref, s_dev) and torch.equal(t_ref, t_dev), (start, flags)
            assert float(fd) == 0.0


def test_non_finite_gradients_skip_the_step_but_not_the_ema(cuda_device):
    """An inf in one gradient and a NaN in another: parameters, momentum buffers and Adam's step stay put, the scale halves and
    the tracker resets, the EMA still moves."""
    from icafusion_b200.trainer import DeviceOptimizerStep, TrainStep
    for adam in (False, True):
        model = _model(cuda_device)
        ts = TrainStep(model, None, total_batch_size=16, imgsz=320, ema=True, adam=adam)
        ts.scaler.scale(torch.ones((), device=cuda_device))
        ts.scaler._growth_tracker.fill_(7)
        live = [p for g in ts.optimizer.param_groups for p in g["params"]]
        for i, p in enumerate(live):
            p.grad = torch.randn_like(p)
        live[3].grad.view(-1)[5] = float("inf")
        live[-2].grad.view(-1)[0] = float("nan")
        step = DeviceOptimizerStep(ts.optimizer, ts.scaler, ts.ema, model, cuda_device)
        with torch.no_grad():
            for p in model.parameters():
                p.add_(0.01)                               # the EMA has something to move towards
        before = {k: v.clone() for k, v in model.state_dict().items()}
        state = {id(p): {k: v.clone() for k, v in ts.optimizer.state[p].items()} for p in live}
        ema_before = {k: v.clone() for k, v in ts.ema.ema.state_dict().items()}
        scale = float(ts.scaler.get_scale())
        step.stage()
        step.enqueue()
        torch.cuda.synchronize()
        assert all(torch.equal(v, before[k]) for k, v in model.state_dict().items())
        for p in live:
            for k, v in ts.optimizer.state[p].items():
                assert torch.equal(v, state[id(p)][k]), k
        assert float(ts.scaler.get_scale()) == scale / 2 and ts.scaler._get_growth_tracker() == 0
        assert float(step.found_inf) == 0.0
        moved = [k for k, v in ts.ema.ema.state_dict().items() if v.dtype.is_floating_point and not torch.equal(v, ema_before[k])]
        assert len(moved) > 100 and ts.ema.updates == 1


def _train_loop(dev, graphed: bool, adam: bool):
    """train.py:296-352 on yolov5s 320: warm-up lr / momentum written every batch, accumulate ramping 1 -> 2 -> 4, LambdaLR, EMA;
    GradScaler starting at 2**36 so the first window overflows and is skipped, then growing every two clean steps."""
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep
    B, H, nw = 2, 320, 6
    model = _model(dev)
    ts = TrainStep(model, None, total_batch_size=16, imgsz=H, ema=True, adam=adam)
    ts.scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 36, backoff_factor=2.0 ** -22, growth_interval=2)
    lf = lambda x: (1 - x / 300) * (1.0 - 0.2) + 0.2          # noqa: E731 (train.py:148)
    scheduler = torch.optim.lr_scheduler.LambdaLR(ts.optimizer, lr_lambda=lf)
    step = GraphedTrainStep(ts, B, H, H, 16, dev) if graphed else ts
    data = []
    for s in range(4):
        rgb, ir = synth.synth_images(B, H, H, 500 + s)
        t = torch.from_numpy(synth_targets(6 + s, B, 500 + s))
        data.append(((rgb * 255).to(torch.uint8).to(dev), (ir * 255).to(torch.uint8).to(dev), t.to(dev)))
    hyp = ts.hyp
    losses, scales, epoch, ni = [], [], 0, 0
    caught = []
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        for epoch in range(2):
            step.zero_grad()
            for i in range(7):
                ni = i + 7 * epoch
                accumulate = ts.accumulate_at(ni, nw)
                if ni <= nw:
                    for j, x in enumerate(ts.optimizer.param_groups):
                        x["lr"] = np.interp(ni, [0, nw], [0.1 if j == 2 else 0.0, x["initial_lr"] * lf(epoch)])
                        if "momentum" in x:
                            x["momentum"] = np.interp(ni, [0, nw], [0.8, hyp["momentum"]])
                flag = ni % accumulate == 0
                losses.append(float(step(*data[ni % 4], optimizer_step=flag)[0]))
                if flag:
                    scales.append(float(ts.scaler.get_scale()))
            scheduler.step()
    if graphed:
        step.close()
    torch.cuda.synchronize()
    sched_warn = [w for w in caught if "lr_scheduler.step()" in str(w.message)]
    return dict(losses=losses, scales=scales, model=model, ts=ts, sched_warn=sched_warn, step=step)


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / max(float(b.float().abs().max()), 1e-6))


def _check_graphed_equals_eager(e, g, adam):
    print(f"\n[device step {'adam' if adam else 'sgd'}] scales eager {e['scales']}\n  graphed {g['scales']}")
    assert e["scales"] == g["scales"]
    assert e["scales"][0] < 2.0 ** 36 and max(e["scales"]) > min(e["scales"])          # a skip, then growth
    assert np.allclose(e["losses"], g["losses"], rtol=1e-4)
    assert not g["sched_warn"], g["sched_warn"]
    se, sg = e["model"].state_dict(), g["model"].state_dict()
    worst = max(_rel(sg[k], se[k]) for k in se if se[k].is_floating_point())
    ee, eg = e["ts"].ema.ema.state_dict(), g["ts"].ema.ema.state_dict()
    worst_ema = max(_rel(eg[k], ee[k]) for k in ee if ee[k].is_floating_point())
    print(f"[device step] worst relative difference: parameters / buffers {worst:.2e}, EMA {worst_ema:.2e}")
    assert worst < 1e-3 and worst_ema < 1e-3
    assert all(torch.equal(sg[k], se[k]) for k in se if not se[k].is_floating_point())
    assert e["ts"].ema.updates == g["ts"].ema.updates
    oe, og = e["ts"].optimizer.state_dict(), g["ts"].optimizer.state_dict()
    assert oe["param_groups"] == og["param_groups"]
    assert oe["state"].keys() == og["state"].keys()
    for i, st in oe["state"].items():
        assert st.keys() == og["state"][i].keys()
        for k, v in st.items():
            if k == "step":
                assert float(v) == float(og["state"][i][k])
            else:
                assert _rel(og["state"][i][k], v) < 1e-3 or float(v.abs().max()) < 1e-6, (i, k)
    assert e["ts"].scaler.state_dict() == g["ts"].scaler.state_dict()


@pytest.mark.parametrize("adam", [False, True])
def test_graphed_step_equals_eager_train_loop(cuda_device, adam):
    _check_graphed_equals_eager(_train_loop(cuda_device, False, adam), _train_loop(cuda_device, True, adam), adam)


def test_adam_bias_table_growth_equals_eager(cuda_device, monkeypatch):
    """Adam's bias-correction table starting at 2 rows: the loop's stepping calls outgrow it twice (2 -> 4 -> 8 rows), each
    time reallocating it and capturing the step graph again, and the run still equals the eager one."""
    from icafusion_b200.trainer import DeviceOptimizerStep
    monkeypatch.setattr(DeviceOptimizerStep, "BIAS_STEPS", 2)
    e = _train_loop(cuda_device, False, True)
    g = _train_loop(cuda_device, True, True)
    assert g["step"].opt.bias_corr.shape[1] == 8 and g["step"].opt.max_step == 4
    _check_graphed_equals_eager(e, g, True)
    steps = [float(st["step"]) for st in g["ts"].optimizer.state.values()]
    assert set(steps) == {3.0}                      # four stepping calls, the first one skipped


def test_stepping_call_does_not_synchronise(cuda_device):
    """A stepping call reads nothing back: no synchronising call under set_sync_debug_mode("error"), and it returns while
    work queued ahead of it (torch.cuda._sleep) still runs."""
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep
    B, H = 2, 320
    model = _model(cuda_device)
    ts = TrainStep(model, None, total_batch_size=16, imgsz=H, ema=True)
    step = GraphedTrainStep(ts, B, H, H, 16, cuda_device)
    rgb, ir = synth.synth_images(B, H, H, 7)
    batch = ((rgb * 255).to(torch.uint8).to(cuda_device), (ir * 255).to(torch.uint8).to(cuda_device),
             torch.from_numpy(synth_targets(6, B, 7)).to(cuda_device))
    try:
        step(*batch)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for flag in (False, True, True):
                for g in ts.optimizer.param_groups:
                    g["lr"] *= 0.99
                step(*batch, optimizer_step=flag)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        torch.cuda._sleep(2_000_000_000)                 # about a second of GPU time ahead of the call
        step(*batch)
        done = torch.cuda.Event()
        done.record()
        assert not done.query()
        torch.cuda.synchronize()
    finally:
        step.close()


def _nccl_case(rank, dev):
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep
    B, H = 2, 320
    t = torch.tensor([[0, 0, 0.5, 0.5, 0.2, 0.3], [1, 0, 0.3, 0.6, 0.1, 0.2]], device=dev)
    model = _model(dev, 3)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        ts = TrainStep(model, None, total_batch_size=2 * B * 8, world_size=2, imgsz=H, ema=True)
        ts.scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 36, backoff_factor=2.0 ** -22)
    torch.cuda.current_stream(dev).wait_stream(side)
    step = GraphedTrainStep(ts, B, H, H, 16, dev)
    scales = []
    for s in range(4):
        g = torch.Generator().manual_seed(600 + 10 * s + rank)
        rgb, ir = (torch.randint(0, 256, (B, 3, H, H), generator=g).to(torch.uint8).to(dev) for _ in range(2))
        step(rgb, ir, t, optimizer_step=s % 2 == 1)
        if s % 2:
            scales.append(float(ts.scaler.get_scale()))
    step.close()
    torch.cuda.synchronize()
    return scales, {k: v.detach().cpu().numpy() for k, v in ts.raw_model.state_dict().items()}


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (NCCL)")
def test_ranks_stay_identical_across_a_skipped_step(cuda_device):
    from test_gpu_sync_bn import _spawn
    (sc0, s0), (sc1, s1) = _spawn(_nccl_case, backend="nccl")
    assert sc0 == sc1 and sc0[0] < 2.0 ** 36
    assert all(np.array_equal(s0[k], s1[k]) for k in s0)
