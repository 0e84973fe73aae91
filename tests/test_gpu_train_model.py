"""One training step of the whole two-stream model (train.py:334-344): train-mode forward, ComputeLoss, backward -- the CUDA
path against autograd through the CPU oracle (itself pinned to the reference's own step by tests/golden/train_yolov5s_320.npz)."""
import numpy as np
import pytest
import torch

import train_grads
from conftest import load_golden
from helpers import load_synth
from oracle import icaf_oracle as O
from oracle import synth
from oracle.gen_golden_train import synth_targets

pytestmark = pytest.mark.gpu


def test_training_step_yolov5s_320(cuda_device):
    """One step against fp32 autograd through the oracle and the reference's own step, one gradient tensor at a time, at loss
    scales 2^8 and 2^16 (tests/train_grads.py)."""
    train_grads.run_case(cuda_device, "train_yolov5s_320")


def _module_case(cuda_device, mod, pre, fwd_ref, fwd_dev, inputs, tol, l2=False):
    """Forward + every gradient of one module in train(): device nodes vs fp32 autograd through the oracle's restatement.
    Short chains, so the bar is tight (the whole-model step above can only be held to the fp16 regime's noise floor)."""
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for k, p in mod.named_parameters():
            if p.dim() >= 2:
                p.copy_((torch.randn(p.shape, generator=g) * (1.5 / max(p[0].numel(), 1) ** 0.5)).half().float())
            elif "bn.weight" in k or k.endswith("weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.2 * torch.randn(p.shape, generator=g))
    sd = {f"{pre}.{k}": v.clone() for k, v in mod.state_dict().items()}
    leaves = {k: v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    xs = [t.float().requires_grad_(True) for t in inputs]
    O._BN_TRAIN[0] = True
    try:
        y = fwd_ref(sd, *xs)
    finally:
        O._BN_TRAIN[0] = False
    dy = (0.1 * torch.randn(y.shape, generator=g)).half()
    y.backward(dy.float())
    mod = mod.to(cuda_device).train()
    for mm in mod.modules():
        if isinstance(mm, torch.nn.Dropout):
            mm.p = 0.0
    xd = [t.permute(0, 2, 3, 1).contiguous().to(cuda_device).requires_grad_(True) for t in inputs]
    yd = fwd_dev(mod, *xd)
    yd.backward(dy.permute(0, 2, 3, 1).contiguous().to(cuda_device))
    torch.cuda.synchronize()
    if l2:      # arg-max routing (max pools): an fp16 tie moves a whole gradient element, so the bar is the L2 norm
        rel = lambda a, b: float((a.detach().float().cpu() - b).norm() / max(float(b.norm()), 1e-6))            # noqa: E731
    else:
        rel = lambda a, b: float((a.detach().float().cpu() - b).abs().max() / max(float(b.abs().max()), 1e-6))  # noqa: E731
    errs = {"y": rel(yd.permute(0, 3, 1, 2), y.detach())}
    for i, (a, b) in enumerate(zip(xd, xs)):
        errs[f"dx{i}"] = rel(a.grad.permute(0, 3, 1, 2), b.grad)
    worst_p, worst_s = ("", 0.0), ("", 0.0)
    for k, p in mod.named_parameters():
        r = leaves[f"{pre}.{k}"].grad
        if r is None:
            assert p.grad is None, k
            continue
        floor = 1e-3 * float(max(v.grad.abs().max() for v in leaves.values() if v.grad is not None))
        e = float((p.grad.detach().float().cpu() - r).norm() / max(float(r.norm()), floor)) if l2 else \
            float((p.grad.detach().float().cpu() - r).abs().max() / max(float(r.abs().max()), floor))
        if p.numel() == 1:          # LearnableCoefficient / LearnableWeights: one cancelling sum over a whole fp16 tensor
            worst_s = max(worst_s, (k, e), key=lambda t: t[1])
        elif e > worst_p[1]:
            worst_p = (k, e)
    errs["dparam"] = worst_p[1]
    print(f"\n[{type(mod).__name__} node] " + "  ".join(f"{k} {v:.2e}" for k, v in errs.items()) + f"   (worst parameter: {worst_p[0]})"
          + (f"   scalar parameters: {worst_s[1]:.2e} ({worst_s[0]})" if worst_s[0] else ""))
    assert max(errs.values()) < tol, errs
    assert worst_s[1] < 1e-1, worst_s


def test_c3_sppf_fusion_block_nodes(cuda_device):
    from icafusion_b200 import autograd as A
    from icafusion_b200 import common
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 64, 24, 32, generator=g).half()
    for mod in (common.C3(64, 64, 2, True), common.C3(64, 128, 1, False)):
        for mm in mod.modules():
            if isinstance(mm, torch.nn.BatchNorm2d):
                mm.eps, mm.momentum = 1e-3, 0.03
        n, sc = len(mod.m), mod.m[0].add
        _module_case(cuda_device, mod, "m", lambda sd, t, n=n, sc=sc: O.c3(t, sd, "m", n, sc), A.c3, [x], 4e-3)
    mod = common.SPPF(64, 64)
    for mm in mod.modules():
        if isinstance(mm, torch.nn.BatchNorm2d):
            mm.eps, mm.momentum = 1e-3, 0.03
    _module_case(cuda_device, mod, "m", lambda sd, t: O.sppf(t, sd, "m"), A.sppf, [x], 1.5e-1, l2=True)
    # the pool chain alone on fp16-exact inputs: same ties on both sides, so the arg-max routing must agree element for element
    import torch.nn.functional as F
    xp = torch.randn(2, 32, 20, 28, generator=g).half()
    xp[0, :, 3:9, 3:9] = 1.0                                   # a plateau: every window inside it is one big tie
    xr = xp.float().requires_grad_(True)
    y1 = F.max_pool2d(xr, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    cat = torch.cat([xr, y1, y2, F.max_pool2d(y2, 5, 1, 2)], 1)
    dcat = (0.1 * torch.randn(cat.shape, generator=g)).half()
    cat.backward(dcat.float())
    xd = xp.permute(0, 2, 3, 1).contiguous().to(cuda_device).requires_grad_(True)
    cd = A.SppfPoolFn.apply(xd)
    cd.backward(dcat.permute(0, 2, 3, 1).contiguous().to(cuda_device))
    assert torch.equal(cd.permute(0, 3, 1, 2).float().cpu(), cat.detach())
    e = float((xd.grad.permute(0, 3, 1, 2).float().cpu() - xr.grad).abs().max() / xr.grad.abs().max())
    print(f"[SPPF pool chain, exact inputs] dx {e:.2e}")
    assert e < 2e-3
    # DMFF block in train(): pooled with overlapping windows (20x24 -> 16x16), two loops
    rgb, ir = torch.randn(2, 128, 20, 24, generator=g).half(), torch.randn(2, 128, 20, 24, generator=g).half()
    mod = common.TransformerFusionBlock(128, 16, 16)
    mod.crosstransformer[0].loops = 2
    _module_case(cuda_device, mod, "b", lambda sd, a, b: O.dmff_block(a, b, sd, "b", 16, 16, 2, training=True, bn_eps=1e-5),
                 lambda m, a, b: A.fusion_block(m, a, b), [rgb, ir], 6e-3)


def test_graphed_train_step_equals_eager(cuda_device, monkeypatch):
    """GraphedTrainStep (forward + loss + backward replayed from a CUDA graph) takes the same optimiser steps as the eager
    TrainStep: same losses and the same parameters / BatchNorm buffers after three steps on changing batches, dropout off."""
    check_graphed_train_step(cuda_device, monkeypatch, dropout=False)


def test_graphed_train_step_with_dropout_equals_eager(cuda_device, monkeypatch):
    """As above with the model's own dropout (p = 0.1).  Both runs draw the same per-site seeds (autograd.manual_seed before
    each eager step and before the capture), and eager step r runs with the seed offset at r, as graph replay r does after
    its in-graph increment: the masks then agree only if every replay draws new masks and every kernel adds the offset."""
    check_graphed_train_step(cuda_device, monkeypatch, dropout=True)


def check_graphed_train_step(cuda_device, monkeypatch, dropout: bool):
    from icafusion_b200 import Model, _lib
    from icafusion_b200 import autograd as A
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep, dead_parameters
    m, d = load_golden("train_yolov5s_320")
    B, H, W = 2, 320, 320
    S = 0x5EED
    batches = []
    for s in range(3):
        rgb, ir = synth.synth_images(B, H, W, 100 + s)
        t = torch.from_numpy(synth_targets(8 + s, B, 100 + s))
        batches.append(((rgb * 255).to(torch.uint8).to(cuda_device), (ir * 255).to(torch.uint8).to(cuda_device), t.to(cuda_device)))
    for k in ("seed", "count"):                        # restored on exit: the mask seed state is process-global
        monkeypatch.setitem(A._STATE, k, A._STATE[k])
    capture = GraphedTrainStep._capture

    def seeded_capture(self, graph, pool=None):
        A.manual_seed(S)
        return capture(self, graph, pool)
    monkeypatch.setattr(GraphedTrainStep, "_capture", seeded_capture)
    runs = []
    for graphed in (False, True):
        model = Model("yolov5s_Transfusion_kaist")
        load_synth(model, m["seed"])
        model = model.to(cuda_device).train()
        n_drop = 0
        for mod in model.modules():
            if isinstance(mod, torch.nn.Dropout):
                n_drop += mod.p > 0
                if not dropout:
                    mod.p = 0.0
        assert n_drop > 0
        ts = TrainStep(model, None, total_batch_size=B, imgsz=320)
        assert sorted(ts.dead) == sorted(m["dead_params"]) == sorted(dead_parameters(model))
        if graphed:
            step = GraphedTrainStep(ts, B, H, W, 16, cuda_device)
            try:
                losses = [float(step(*b)[0]) for b in batches]
            finally:
                step.close()
        else:
            ctr = torch.zeros(1, dtype=torch.int32, device=cuda_device)
            _lib.check(_lib.lib().icaf_set_seed_offset(ctr.data_ptr()), "icaf_set_seed_offset")
            losses = []
            try:
                for r, b in enumerate(batches, 1):
                    A.manual_seed(S)
                    ctr.fill_(r)
                    losses.append(float(ts(*b)[0]))
            finally:
                torch.cuda.synchronize()
                _lib.lib().icaf_set_seed_offset(None)
        torch.cuda.synchronize()
        runs.append((losses, {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}, float(ts.scaler.get_scale())))
    (l0, s0, sc0), (l1, s1, sc1) = runs
    print(f"\n[graphed step] losses eager {l0}  graphed {l1}  scale {sc0} / {sc1}")
    assert sc0 == sc1
    assert np.allclose(l0, l1, rtol=1e-4)
    worst = max(float((s1[k] - s0[k]).abs().max() / max(float(s0[k].abs().max()), 1e-6)) for k in s0 if s0[k].is_floating_point())
    print(f"[graphed step] worst relative parameter / buffer difference after 3 steps: {worst:.2e}")
    assert worst < 1e-3
    assert all(torch.equal(s0[k], s1[k]) for k in s0 if not s0[k].is_floating_point())      # num_batches_tracked


def test_standalone_module_forwards_in_train_mode(cuda_device):
    """The reference-shaped entry points (NCHW tensors / (B,N,C) token lists) of the operator classes in train(): same values as
    the NHWC autograd nodes they wrap, and gradients reach the caller's tensors and the parameters."""
    from icafusion_b200 import autograd as A
    from icafusion_b200 import common
    g = torch.Generator().manual_seed(4)
    m = common.C3(64, 64, 1).to(cuda_device).train()
    x = torch.randn(2, 64, 16, 24, generator=g).to(cuda_device).requires_grad_(True)
    y = m(x)
    assert tuple(y.shape) == (2, 64, 16, 24)
    y.float().square().mean().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all() and float(x.grad.abs().max()) > 0
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    m2 = common.C3(64, 64, 1).to(cuda_device).train()
    m2.load_state_dict(m.state_dict())
    y2 = A.c3(m2, x.detach().permute(0, 2, 3, 1).contiguous().half())
    assert torch.equal(y2.permute(0, 3, 1, 2), y.detach())
    # token-level classes, N not a multiple of 8 (padded internally), dropout active
    blk = common.CrossTransformerBlock(128, 128, 128, 8, 4, 0.1, 0.1).to(cuda_device).train()
    r = torch.randn(2, 100, 128, generator=g).to(cuda_device).requires_grad_(True)
    i = torch.randn(2, 100, 128, generator=g).to(cuda_device).requires_grad_(True)
    o_r, o_i = blk([r, i])
    assert tuple(o_r.shape) == (2, 100, 128) and tuple(o_i.shape) == (2, 100, 128)
    (o_r.float().sum() + o_i.float().square().sum()).backward()
    assert torch.isfinite(r.grad).all() and torch.isfinite(i.grad).all() and float(i.grad.abs().max()) > 0
    live = [k for k, p in blk.named_parameters() if p.grad is not None]
    dead = [k for k, p in blk.named_parameters() if p.grad is None]
    assert dead and all(k.split(".")[0] in ("ln_input", "ln_output", "mlp", "LN1") for k in dead), dead
    assert all(torch.isfinite(dict(blk.named_parameters())[k].grad).all() for k in live)
    att = common.CrossAttention(128, 128, 128, 8).to(cuda_device).train()
    a_r, a_i = att([r.detach(), i.detach()])
    assert tuple(a_r.shape) == (2, 100, 128) and torch.isfinite(a_r).all() and torch.isfinite(a_i).all()
    det_in = [torch.randn(2, c, h, w, generator=g).to(cuda_device) for c, h, w in ((128, 8, 8), (256, 4, 4), (512, 2, 2))]
    from icafusion_b200.yolo_test import Detect
    det = Detect(1, ((10, 13, 16, 30, 33, 23), (30, 61, 62, 45, 59, 119), (116, 90, 156, 198, 373, 326)), (128, 256, 512)).to(cuda_device).train()
    outs = det(det_in)
    assert [tuple(o.shape) for o in outs] == [(2, 3, 8, 8, 6), (2, 3, 4, 4, 6), (2, 3, 2, 2, 6)]
