"""Scheduling independence on the device.

Contested cells: several build_targets candidates of different targets on one (image, anchor, cell), at every level, with
gradients several orders of magnitude apart.  Their sum in icaf_compute_loss_bwd is taken in a fixed order (ascending
candidate index), so the gradient equals the float64 oracle at the census's bar, two launches agree bit for bit, and a
launch replayed from a CUDA graph equals the eager one bit for bit.  (That no kernel has a floating-point atomic at all is
checked on the PTX by test_launch_order_cpu.py.)

PDL off equals PDL on: inference, one eager training step (forward, loss, backward, GradScaler unscale, SGD step, EMA), the
same step replayed from the TrainStep graph and one graphed test.test batch, each in a child process with ICAF_PDL=0 and
one with programmatic dependent launch on, give the same bits.
"""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# yolov5s anchors in pixels (P3, P4, P5), strides 8 / 16 / 32
ANCHORS_PX = [[(10, 13), (16, 30), (33, 23)], [(30, 61), (62, 45), (59, 119)], [(116, 90), (156, 198), (373, 326)]]
HYP = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0, label_smoothing=0.0)
GRAD_OUT = 256.0


def _contested_targets():
    """Image 0: clusters of 3, 5 and 12 targets on one centre (duplicated boxes of different classes and sizes), plus targets
    whose half-cell neighbour offsets land on the 12-cluster's cell at the finest level; image 1: a few ordinary targets."""
    rows = []
    for (x, y, w, h), n in (((0.30, 0.30, 0.25, 0.25), 3), ((0.70, 0.30, 0.20, 0.30), 5), ((0.5, 0.72, 0.22, 0.22), 12)):
        for i in range(n):
            s = 1.0 + 0.15 * (i % 4) - 0.1 * (i % 3)
            rows.append([0, i % 4, x, y, w * s, h / s])
    # finest grid 32 x 32 (256 x 256 input): the 12-cluster sits in cell (16, 23); left / right / upper / lower neighbours
    for x, y in ((15.7 / 32, 23.5 / 32), (17.2 / 32, 23.5 / 32), (16.5 / 32, 22.8 / 32), (16.5 / 32, 24.3 / 32)):
        rows.append([0, 3, x, y, 0.2, 0.24])
    rows += [[1, 1, 0.2, 0.6, 0.1, 0.3], [1, 2, 0.8, 0.8, 0.3, 0.2], [1, 0, 0.45, 0.15, 0.5, 0.4]]
    return np.array(rows, dtype=np.float32)


def _candidates_per_cell(t, ny, nx, anchors):
    """{(level, image, anchor, gj, gi): count} of build_targets' candidates (loss.py:405-463 in fp32, as cand_setup)."""
    f = np.float32
    cells = {}
    for lvl in range(len(ny)):
        for row in t:
            gx, gy, gw, gh = f(row[2]) * f(nx[lvl]), f(row[3]) * f(ny[lvl]), f(row[4]) * f(nx[lvl]), f(row[5]) * f(ny[lvl])
            for a, (aw, ah) in enumerate(anchors[lvl]):
                r = max(gw / f(aw), f(aw) / gw, gh / f(ah), f(ah) / gh)
                if not r < 4.0:
                    continue
                offs = [(0, 0)]
                if gx % 1 < 0.5 and gx > 1: offs.append((0.5, 0))                                    # noqa: E701
                if gy % 1 < 0.5 and gy > 1: offs.append((0, 0.5))                                    # noqa: E701
                if (nx[lvl] - gx) % 1 < 0.5 and nx[lvl] - gx > 1: offs.append((-0.5, 0))             # noqa: E701
                if (ny[lvl] - gy) % 1 < 0.5 and ny[lvl] - gy > 1: offs.append((0, -0.5))             # noqa: E701
                for ox, oy in offs:
                    gi = min(max(int(gx - f(ox)), 0), nx[lvl] - 1)
                    gj = min(max(int(gy - f(oy)), 0), ny[lvl] - 1)
                    k = (lvl, int(row[0]), a, gj, gi)
                    cells[k] = cells.get(k, 0) + 1
    return cells


def _logits(B, na, ny, nx, no, gen):
    """Predictions whose per-candidate gradients span several orders of magnitude: class logits from -12 to +6 (sigmoid
    gradients from ~6e-6 to ~1), box logits spread so that the CIoU derivatives differ between cells."""
    x = torch.randn(B, na, ny, nx, no, generator=gen, dtype=torch.float64)
    x[..., 0:4] *= 1.5
    x[..., 4] = 1.5 * x[..., 4] - 4.0
    x[..., 5:] = torch.tensor([-12.0, -4.0, 0.5, 6.0], dtype=torch.float64)[: no - 5] + 0.5 * x[..., 5:]
    return x


def _case(dev, dtype):
    from icafusion_b200.loss import ComputeLoss
    B, na, nc, H, W = 2, 3, 4, 256, 256
    ny, nx = [H // 8, H // 16, H // 32], [W // 8, W // 16, W // 32]
    anchors = torch.tensor(ANCHORS_PX, dtype=torch.float32) / torch.tensor([8.0, 16.0, 32.0]).view(3, 1, 1)
    t = _contested_targets()
    counts = _candidates_per_cell(t, ny, nx, anchors.tolist())
    for lvl in range(3):                       # the case exercises what it claims to, at every level
        per = sorted({v for k, v in counts.items() if k[0] == lvl})
        assert {3, 5}.issubset(per) and max(per) >= 12, (lvl, per)
    gen = torch.Generator().manual_seed(11)
    p = [_logits(B, na, ny[i], nx[i], 5 + nc, gen).to(dtype) for i in range(3)]
    det = types.SimpleNamespace(na=na, nc=nc, nl=3, anchors=anchors)
    crit = ComputeLoss(types.SimpleNamespace(hyp=HYP, gr=1.0, model=[det]))
    crit.with_backward = True
    ps = [x.to(dev) for x in p]
    tg = torch.from_numpy(t).to(dev)
    return crit, p, ps, tg, anchors


def _launch(crit, ps, tg, ws, out, gout, dps):
    crit._launch(ps, 0, tg, out=out, ws=ws)
    crit._launch(ps, 0, tg, ws=ws, grad_out=gout, dps=dps)


def _bits(x):
    return x.contiguous().view({torch.float16: torch.int16, torch.float32: torch.int32}[x.dtype])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["p_fp32", "p_fp16"])
def test_contested_cells_gradient_is_fixed_order(cuda_device, dtype):
    from oracle import focal_loss
    crit, p, ps, tg, anchors = _case(cuda_device, dtype)
    ws = crit._launch(ps, 0, tg, out=torch.empty(5, device=cuda_device))
    gout = torch.full((1,), GRAD_OUT, dtype=torch.float32, device=cuda_device)
    outs = [torch.empty(5, device=cuda_device) for _ in range(3)]
    dps = [[torch.full_like(x, float("nan")) for x in ps] for _ in range(3)]
    _launch(crit, ps, tg, ws, outs[0], gout, dps[0])
    _launch(crit, ps, tg, ws, outs[1], gout, dps[1])
    # the same forward + backward captured in a CUDA graph, replayed once
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            _launch(crit, ps, tg, ws, outs[2], gout, dps[2])
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()

    pr = [x.double().requires_grad_(True) for x in p]
    lo, items = focal_loss.compute_loss(pr, tg.cpu(), anchors, HYP, 1.0)
    (lo * GRAD_OUT).backward()
    ref_out = torch.cat([lo.detach().view(1), items.detach()])
    got = outs[0].double().cpu()
    assert ((got - ref_out).abs() / (2e-6 + 3e-5 * ref_out.abs())).max() <= 1.0, (got, ref_out)
    for lvl in range(3):
        r = pr[lvl].grad
        s = float(r.abs().max())
        g = dps[0][lvl].double().cpu()
        assert torch.isfinite(g).all(), lvl
        # the census's bar: 2e-5 of the level's largest gradient plus the half ulp of the final rounding to fp16
        e = float(((g - r).abs() / s / (2e-5 + 2.0 ** -11 * (r.abs() / s))).max())
        print(f"\n[contested cells {dtype}] level {lvl}: error {e:.3f} of the bar, largest gradient {s:.3e}")
        assert e <= 1.0, (lvl, e)
        assert torch.equal(_bits(dps[1][lvl]), _bits(dps[0][lvl])), f"level {lvl}: second launch differs"
        assert torch.equal(_bits(dps[2][lvl]), _bits(dps[0][lvl])), f"level {lvl}: graph replay differs from eager"
    assert torch.equal(_bits(outs[1]), _bits(outs[0])) and torch.equal(_bits(outs[2]), _bits(outs[0]))


# ------------------------------------------------------------------------------------------------ PDL off equals PDL on

def _child(out_path):
    """Inference, an eager and a graphed training step and a graphed validation batch on cuda:0; every output to out_path."""
    sys.path[:0] = [ROOT, HERE]
    from conftest import load_golden
    from helpers import load_synth
    from icafusion_b200 import Model
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.trainer import GraphedTrainStep, TrainStep
    from oracle import synth
    from oracle.gen_golden_train import synth_targets
    from test_gpu_val_graphs import _batches, _labels_list, _model, _run
    from icafusion_b200.loss import ComputeLoss
    import pathlib
    import tempfile
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {}
    # (a) yolov5s inference, 512 x 640, batch 2
    with torch.no_grad():
        model = Model("yolov5s_Transfusion_kaist").eval()
        load_synth(model, 7)
        model = model.fuse().to(dev)
        a, b = synth.synth_images(2, 512, 640, 7)
        res["infer"] = model(a.to(dev), b.to(dev))[0].cpu()
    del model
    # (b), (c) one training step of the train_yolov5s_320 case, eager and from the TrainStep graph
    m, _ = load_golden("train_yolov5s_320")
    B, H, W = m["B"], m["H"], m["W"]
    rgb, ir = synth.synth_images(B, H, W, m["seed"])
    batch = ((rgb * 255).to(torch.uint8).to(dev), (ir * 255).to(torch.uint8).to(dev),
             torch.from_numpy(synth_targets(m["nt"], B, m["seed"])).to(dev))
    for graphed in (False, True):
        model = Model("yolov5s_Transfusion_kaist")
        load_synth(model, m["seed"])
        model = model.to(dev).train()
        for mod in model.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
        ts = TrainStep(model, None, total_batch_size=B, imgsz=H, ema=True)
        tag = "graphed" if graphed else "eager"
        if graphed:
            step = GraphedTrainStep(ts, B, H, W, 16, dev)
            try:
                res[f"{tag} loss"] = step(*batch)[0].clone()
            finally:
                step.close()
        else:
            res[f"{tag} loss"] = ts(*batch, optimizer_step=False)[0]
            for k, v in model.named_parameters():
                if v.grad is not None:
                    res[f"{tag} grad {k}"] = v.grad.clone()
            ts.scaler.step(ts.optimizer)                     # the optimizer_step=True branch of TrainStep.__call__
            ts.scaler.update()
            ts.zero_grad()
            ts.ema.update(ts.raw_model)
        torch.cuda.synchronize()
        res[f"{tag} scale"] = torch.tensor([float(ts.scaler.get_scale())])
        res.update({f"{tag} state {k}": v.detach().clone() for k, v in model.state_dict().items()})
        res.update({f"{tag} ema {k}": v.detach().clone() for k, v in ts.ema.ema.state_dict().items()})
        del model, ts
    # (d) one graphed test.test batch
    model = _model("yolov5s_Transfusion_kaist", 21, dev)
    batches = _batches([(2, 512, 640, 5)], 1, 5)
    with tempfile.TemporaryDirectory() as tmp:
        got = _run(model, batches, pathlib.Path(tmp), ValidationGraphs(model), compute_loss=ComputeLoss(model),
                   save_txt=True, labels_list=_labels_list(batches))
    res["val results"] = torch.tensor(got[0], dtype=torch.float64)
    res["val maps"] = torch.from_numpy(np.asarray(got[1]))
    res["val txt"] = torch.frombuffer(bytearray(got[3]), dtype=torch.uint8)
    torch.cuda.synchronize()
    torch.save({k: v.cpu() for k, v in res.items()}, out_path)


def test_pdl_off_equals_pdl_on(tmp_path):
    runs = {}
    for pdl in ("0", "1"):
        out = tmp_path / f"pdl{pdl}.pt"
        env = dict(os.environ, ICAF_PDL=pdl)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), str(out)], env=env, cwd=ROOT, capture_output=True,
                           text=True, timeout=1500)
        assert p.returncode == 0, f"ICAF_PDL={pdl} child failed:\n{p.stdout[-4000:]}\n{p.stderr[-4000:]}"
        runs[pdl] = torch.load(out)
    off, on = runs["0"], runs["1"]
    assert sorted(off) == sorted(on)
    assert any(k.startswith("eager grad ") for k in off) and "val txt" in off and len(off["val txt"]) > 0
    raw = lambda x: x.contiguous().reshape(-1).view(torch.uint8)                # noqa: E731  (bits, so NaNs compare too)
    diff = [k for k in off if off[k].dtype != on[k].dtype or not torch.equal(raw(off[k]), raw(on[k]))]
    print(f"\n[PDL off / on] {len(off)} tensors compared, {len(diff)} differ")
    assert not diff, diff[:20]


if __name__ == "__main__":
    _child(sys.argv[1])
