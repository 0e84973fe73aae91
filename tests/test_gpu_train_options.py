"""train.py's training options on the device: focal loss in icaf_compute_loss_fwd / _bwd against the real reference, and
gradient accumulation in TrainStep and GraphedTrainStep (with SGD, --adam and focal loss) against sums of single-batch
gradients, the eager step and the oracle's accumulating loop (itself pinned to tests/golden/train_accumulate_yolov5s_320.npz)."""
import types

import numpy as np
import pytest
import torch

from conftest import load_golden
from helpers import load_synth
from oracle import focal_loss as FL
from oracle import synth
from oracle.gen_golden_loss import synth_case
from oracle.gen_golden_train import synth_targets

pytestmark = pytest.mark.gpu


def _model_stub(nc, anchors, hyp, gr, device):
    det = types.SimpleNamespace(na=anchors.shape[1], nc=nc, nl=anchors.shape[0], anchors=torch.from_numpy(anchors).to(device))
    return types.SimpleNamespace(hyp=hyp, gr=gr, model=[det])


@pytest.mark.parametrize("layout", ["reference", "nhwc_padded"])
def test_focal_loss_matches_reference_and_autograd(cuda_device, layout):
    """fl_gamma 1.5 and 2.0 on every case of loss_focal_cases.npz: forward against the REAL reference within the plain loss's
    bar, d loss / d predictions against autograd through the oracle's FocalLoss, fp16 predictions against the oracle."""
    from icafusion_b200.loss import ComputeLoss
    m, d = load_golden("loss_focal_cases")
    for cs in m["cases"]:
        key = cs["key"]
        p, t = synth_case(cs["name"], cs["nc"], cs["B"], cs["nt"])
        anchors = d[f"{key}_anchors"]
        fn = ComputeLoss(_model_stub(cs["nc"], anchors, cs["hyp"], cs["gr"], cuda_device))
        ref = [torch.from_numpy(x).requires_grad_(True) for x in p]
        lo, _ = FL.compute_loss(ref, torch.from_numpy(t), torch.from_numpy(anchors), cs["hyp"], cs["gr"])
        (lo.sum() * 3.0).backward()
        dev = []
        for x in p:
            x = torch.from_numpy(x).to(cuda_device)
            if layout == "nhwc_padded":
                B, na, ny, nx, no = x.shape
                ld = (na * no + 7) // 8 * 8 + 8
                buf = torch.zeros(B, ny, nx, ld, device=cuda_device)
                buf[..., :na * no] = x.permute(0, 2, 3, 1, 4).reshape(B, ny, nx, na * no)
                x = buf.as_strided((B, na, ny, nx, no), (ny * nx * ld, no, nx * ld, ld, 1))
            dev.append(x.requires_grad_(True))
        loss, items = fn(dev, torch.from_numpy(t).to(cuda_device))
        got = torch.cat([loss.detach(), items]).cpu().numpy()
        print(f"\n[focal loss {key} {layout}] device {got}  reference {d[f'{key}_out']}")
        assert np.allclose(got, d[f"{key}_out"], rtol=3e-5, atol=2e-6), key
        (loss.sum() * 3.0).backward()
        for lvl, (g, r) in enumerate(zip(dev, ref)):
            e = float((g.grad.cpu() - r.grad).abs().max() / r.grad.abs().max())
            print(f"[focal loss bwd {key} {layout} level {lvl}] rel err {e:.2e}")
            assert e < 2e-5, (key, lvl, e)
        g2 = d[f"{key}_grad2"] * 3.0                          # the REAL reference's loss.backward(), coarsest level
        assert np.abs(dev[2].grad.cpu().numpy() - g2).max() <= 2e-5 * np.abs(g2).max(), key
        p16 = [torch.from_numpy(x).half() for x in p]
        l16, i16 = fn([x.to(cuda_device) for x in p16], torch.from_numpy(t).to(cuda_device))
        lo16, io16 = FL.compute_loss([x.float() for x in p16], torch.from_numpy(t), torch.from_numpy(anchors), cs["hyp"], cs["gr"])
        assert np.allclose(torch.cat([l16, i16]).cpu().numpy(), np.concatenate([lo16.numpy().reshape(1), io16.numpy()]), rtol=3e-5, atol=2e-6)


def _model(cuda_device, seed=1234):
    from icafusion_b200 import Model
    model = Model("yolov5s_Transfusion_kaist")
    load_synth(model, seed)
    model = model.to(cuda_device).train()
    for mod in model.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    return model


def _batches(cuda_device, n, B=2, H=320):
    out = []
    for s in range(n):
        rgb, ir = synth.synth_images(B, H, H, 300 + s)
        t = torch.from_numpy(synth_targets(6 + s, B, 300 + s))
        out.append(((rgb * 255).to(torch.uint8).to(cuda_device), (ir * 255).to(torch.uint8).to(cuda_device), t.to(cuda_device)))
    return out


def test_accumulated_grad_is_the_sum_of_single_batch_grads(cuda_device):
    from icafusion_b200.trainer import TrainStep
    model = _model(cuda_device)
    ts = TrainStep(model, None, total_batch_size=8, imgsz=320)
    ts.scaler = torch.amp.GradScaler("cuda", init_scale=256.0)     # keeps every fp16 gradient finite
    data = _batches(cuda_device, 3)
    live = [p for p in model.parameters() if p.requires_grad]
    want = [torch.zeros_like(p) for p in live]
    for b in data:
        ts.zero_grad()
        ts(*b, optimizer_step=False)
        for w, p in zip(want, live):
            if p.grad is not None:
                w += p.grad
    ts.zero_grad()
    before = [p.detach().clone() for p in live]
    for b in data:
        ts(*b, optimizer_step=False)
    torch.cuda.synchronize()
    assert all(torch.equal(p, q) for p, q in zip(live, before)) and not ts.optimizer.state
    num = sum(float(((p.grad - w) ** 2).sum()) if p.grad is not None else float((w ** 2).sum()) for p, w in zip(live, want))
    den = sum(float((w ** 2).sum()) for w in want)
    print(f"\n[accumulate] relative L2 of 3 accumulated micro-batches against the sum of single ones: {(num / den) ** 0.5:.2e}")
    assert (num / den) ** 0.5 <= 1e-5


# train.py:314-320 with nw = 6 and accumulate 4 (total batch 16): accumulate_at ramps 1, 2, 2, 2, 3, 4, 4, then 4.  ni 9 opens
# a window that zero_grad() (train.py:291) discards; ni 10 .. 12 form the next one.
def _schedule(ts):
    flags = [(ni, ni % ts.accumulate_at(ni, 6) == 0) for ni in range(10)]
    return flags + [("zero_grad", None)] + [(ni, ni % ts.accumulate_at(ni, 6) == 0) for ni in range(10, 13)]


@pytest.mark.parametrize("option", ["sgd", "adam", "focal"])
def test_graphed_accumulation_equals_eager(cuda_device, option):
    from icafusion_b200.trainer import HYP_SCRATCH, GraphedTrainStep, TrainStep
    B, H = 2, 320
    data = _batches(cuda_device, 4, B, H)
    hyp = dict(HYP_SCRATCH, fl_gamma=1.5) if option == "focal" else None
    runs = []
    for graphed in (False, True):
        model = _model(cuda_device)
        ts = TrainStep(model, hyp, total_batch_size=16, imgsz=H, adam=option == "adam")
        step = GraphedTrainStep(ts, B, H, H, 16, cuda_device) if graphed else ts
        sched = _schedule(ts)
        assert [ts.accumulate_at(ni, 6) for ni in range(9)] == [1, 2, 2, 2, 3, 4, 4, 4, 4]
        losses, steps = [], 0
        for ni, flag in sched:
            if ni == "zero_grad":
                step.zero_grad()
                continue
            losses.append(float(step(*data[ni % len(data)], optimizer_step=flag)[0]))
            steps += flag
        if graphed:
            assert step.acc_graph is not None
            step.close()
        torch.cuda.synchronize()
        runs.append((losses, {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}, float(ts.scaler.get_scale()), steps))
    (l0, s0, sc0, n0), (l1, s1, sc1, n1) = runs
    print(f"\n[graphed accumulation {option}] {n0} optimiser steps; losses eager {l0}\n  graphed {l1}  scale {sc0} / {sc1}")
    assert n0 == n1 == 4 and sc0 == sc1
    assert np.allclose(l0, l1, rtol=1e-4)
    worst = max(float((s1[k] - s0[k]).abs().max() / max(float(s0[k].abs().max()), 1e-6)) for k in s0 if s0[k].is_floating_point())
    print(f"[graphed accumulation {option}] worst relative parameter / buffer difference: {worst:.2e}")
    assert worst < 1e-3
    assert all(torch.equal(s0[k], s1[k]) for k in s0 if not s0[k].is_floating_point())      # num_batches_tracked


def test_accumulated_step_against_the_oracle(cuda_device):
    """Two optimiser steps over two micro-batches each (tests/golden/train_accumulate_yolov5s_320.npz): the device's parameter
    updates against the oracle's accumulating loop in fp32, with the reference's own fp16-autocast regime as the yardstick."""
    from icafusion_b200.cfg import load_cfg
    from icafusion_b200.trainer import TrainStep
    from oracle.gen_golden_train_accumulate import HYP, batches, oracle_loop
    scale = 256.0
    m, _ = load_golden("train_accumulate_yolov5s_320")
    model = _model(cuda_device, m["seed"])
    ts = TrainStep(model, dict(HYP), total_batch_size=m["total_batch_size"], imgsz=m["H"])
    assert ts.accumulate == m["accumulate"] == 2
    ts.scaler = torch.amp.GradScaler("cuda", init_scale=scale, growth_interval=10 ** 9)     # a static loss scale, as the oracle's
    before = {k: v.detach().clone() for k, v in model.named_parameters()}
    data = batches()
    for ni, (rgb, ir, t) in enumerate(data, 1):
        ts(rgb.to(cuda_device), ir.to(cuda_device), t.to(cuda_device), optimizer_step=(ni % ts.accumulate == 0))
    torch.cuda.synchronize()
    assert float(ts.scaler.get_scale()) == scale                # no step was skipped
    params = dict(model.named_parameters())
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_kaist")
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    ref, *_ = oracle_loop(sd, cfg, m, data)
    amp, *_ = oracle_loop(sd, cfg, m, data, autocast_device=cuda_device, loss_scale=scale)
    num = num_a = den = 0.0
    for k, r in ref.items():
        u = (params[k].detach() - before[k]).float().cpu() if k in params and params[k].requires_grad else torch.zeros_like(r)
        num += float(((u - r) ** 2).sum())
        num_a += float(((amp[k].float().cpu() - r) ** 2).sum())
        den += float((r ** 2).sum())
    rel, rel_a = (num / den) ** 0.5, (num_a / den) ** 0.5
    print(f"\n[accumulated step] parameter updates: relative L2 {rel:.2e} (fp16-autocast oracle: {rel_a:.2e})")
    assert rel <= max(1.5 * rel_a, 2e-3), (rel, rel_a)


# ------------------------------------------------------------------------------------------------------------------------
# two GPUs, NCCL
def _nccl_accumulate_case(rank, dev):
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep
    B, H = 2, 320
    t = torch.tensor([[0, 0, 0.5, 0.5, 0.2, 0.3], [1, 0, 0.3, 0.6, 0.1, 0.2]], device=dev)
    batches = []
    for s in range(4):
        g = torch.Generator().manual_seed(400 + 10 * s + rank)
        batches.append(tuple(torch.randint(0, 256, (B, 3, H, H), generator=g).to(torch.uint8).to(dev) for _ in range(2)) + (t,))
    runs = []
    for graphed in (False, True):
        model = _model(dev, 3)
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            ts = TrainStep(model, None, total_batch_size=2 * B * 8, world_size=2, imgsz=H)     # accumulate 2
        torch.cuda.current_stream(dev).wait_stream(side)
        step = GraphedTrainStep(ts, B, H, H, 16, dev) if graphed else ts
        losses = [float(step(*b, optimizer_step=(ni % ts.accumulate == 0))[0]) for ni, b in enumerate(batches, 1)]
        if graphed:
            step.close()
        torch.cuda.synchronize()
        runs.append((losses, {k: v.detach().float().cpu().numpy() for k, v in ts.raw_model.state_dict().items()}))
    return runs


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs (NCCL)")
def test_graphed_accumulation_over_nccl_equals_eager(cuda_device):
    """The accumulating graph under NCCL DDP (every micro-batch all-reduced) against the eager step, on two GPUs."""
    from test_gpu_sync_bn import _spawn
    for (l0, s0), (l1, s1) in _spawn(_nccl_accumulate_case, backend="nccl"):
        assert np.allclose(l0, l1, rtol=1e-4)
        worst = max(float(np.abs(s1[k] - s0[k]).max() / max(float(np.abs(s0[k]).max()), 1e-6)) for k in s0)
        assert worst < 1e-3, worst
