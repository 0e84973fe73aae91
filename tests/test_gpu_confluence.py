"""icaf_confluence on the device against the real reference's rows (tests/golden/confluence_cases.npz) and the fp64
restatement (oracle/confluence.py): bit for bit, in the reference's order, with its None pattern."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.confluence import confluence_process as oracle_process
from oracle.gen_golden_confluence import checked_inputs

pytestmark = pytest.mark.gpu


def _same(got, want):
    assert len(got) == len(want)
    for b, (g, w) in enumerate(zip(got, want)):
        assert (g is None) == (w is None), b
        if w is not None:
            g = g.cpu().numpy() if torch.is_tensor(g) else g
            assert g.shape == w.shape and np.array_equal(g, w), (b, g.shape, w.shape)


def _clustered(n, no, seed, spread=False):
    """One (1, R, no) fp32 image with n candidates: jittered copies around ~n/12 centres, or n spread boxes."""
    g = np.random.Generator(np.random.PCG64(seed))
    R = max(2 * n, 1000)
    x = np.zeros((R, no), np.float32)
    rows = np.sort(g.choice(R, n, replace=False))
    if spread:
        ctr = g.uniform(0, 640, size=(n, 2))
        wh = g.uniform(4, 40, size=(n, 2))
    else:
        k = max(1, n // 12)
        c = g.uniform(0, 640, size=(k, 2)); s = g.uniform(8, 120, size=(k, 2))
        pick = g.integers(0, k, size=n)
        ctr = c[pick] + g.normal(0, 2, size=(n, 2)); wh = s[pick] * g.uniform(0.9, 1.1, size=(n, 2))
    x[rows, :2] = ctr; x[rows, 2:4] = wh
    x[rows, 4] = g.uniform(0.2, 1.0, size=n)
    x[rows, 5:] = g.uniform(0.6, 1.0, size=(n, no - 5))
    return x[None]


def test_golden_cases_bit_exact(cuda_device):
    from icafusion_b200.confluence import confluence_process
    m, d = load_golden("confluence_cases")
    inputs = checked_inputs(m)
    for inp in m["inputs"]:
        pred = torch.from_numpy(inputs[inp["name"]]).to(cuda_device)
        for st in inp["settings"]:
            want = [None if n is None else d[f"{inp['name']}_{st['name']}_{b}"] for b, n in enumerate(st["counts"])]
            _same(confluence_process(pred, st["conf"], st["p_thres"]), want)


def test_detection_rows_entry_matches_reference_indices(cuda_device):
    from icafusion_b200.confluence import confluence
    from oracle.confluence import candidates, confluence as oracle_confluence
    m, _ = load_golden("confluence_cases")
    inputs = checked_inputs(m)
    for name in ("kaist", "flir"):
        for p_thres in (0.6, 0.5):
            dets = candidates(inputs[name][0].astype(np.float32), 0.1)
            nc = inputs[name].shape[2] - 5
            assert np.array_equal(confluence(dets, nc, p_thres), oracle_confluence(dets, nc, p_thres))


def test_past_shared_memory_equals_oracle(cuda_device):
    """5000 clustered candidates of one class (in shared memory), and 6500 (past its 6144: in the workspace)."""
    from icafusion_b200.confluence import confluence_process
    x = _clustered(5000, 6, 1)
    _same(confluence_process(torch.from_numpy(x).to(cuda_device), 0.1, 0.6), oracle_process(x, 0.1, 0.6))
    big = np.concatenate([_clustered(3250, 6, 2), _clustered(3250, 6, 3)], 1)        # 6500 candidates of one class
    _same(confluence_process(torch.from_numpy(big).to(cuda_device), 0.1, 0.5), oracle_process(big, 0.1, 0.5))


def test_batch_equals_per_image_calls(cuda_device):
    from icafusion_b200 import ops
    imgs = [_clustered(300, 8, 10 + i, spread=i % 2 == 1)[0] for i in range(4)]
    imgs.append(np.zeros_like(imgs[0]))
    z = torch.from_numpy(np.stack(imgs)).to(cuda_device).half()
    det, count = ops.confluence(z, 0.1, 0.6, max_det=3000)
    for b in range(len(imgs)):
        d1, c1 = ops.confluence(z[b:b + 1].contiguous(), 0.1, 0.6, max_det=3000)
        assert int(count[b]) == int(c1[0])
        assert torch.equal(det[b, :int(count[b])], d1[0, :int(c1[0])])
    assert int(count[-1]) == 0
    want = oracle_process(z.float().cpu().numpy(), 0.1, 0.6)
    _same([det[b, :int(count[b])] if int(count[b]) else None for b in range(len(imgs))], want)


def test_graph_replay_equals_eager(cuda_device):
    from icafusion_b200 import ops
    z = torch.from_numpy(np.concatenate([_clustered(400, 8, 20), _clustered(400, 8, 21, spread=True)])).to(cuda_device)
    det0, count0 = ops.confluence(z, 0.1, 0.5, max_det=1200)
    det = torch.full_like(det0, float("nan"))
    count = torch.zeros_like(count0)
    ws = torch.empty((ops.confluence_workspace_bytes(*z.shape) + 15) // 16, 2, dtype=torch.int64, device=cuda_device)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ops.confluence(z, 0.1, 0.5, det=det, count=count, workspace=ws)               # configure outside the capture
        s.synchronize()
        det.fill_(float("nan"))
        count.zero_()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.confluence(z, 0.1, 0.5, det=det, count=count, workspace=ws)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(count, count0)
    for b in range(2):
        n = int(count0[b])
        assert torch.equal(det[b, :n], det0[b, :n]) and bool(det[b, n:].isnan().all())


def test_max_det_overflow_reports_true_count(cuda_device):
    from icafusion_b200 import ops
    z = torch.from_numpy(_clustered(600, 6, 30, spread=True)).to(cuda_device)
    full, n_full = ops.confluence(z, 0.1, 0.6, max_det=600)
    n = int(n_full[0])
    assert n > 50
    det = torch.full((1, 50, 6), float("nan"), device=cuda_device)
    index = torch.full((1, 50), -1, dtype=torch.int32, device=cuda_device)
    _, count = ops.confluence(z, 0.1, 0.6, det=det, index=index)
    assert int(count[0]) == n
    assert torch.equal(det[0], full[0, :50])
    rows = torch.nonzero(z[0, :, 4] > 0.1).flatten()
    assert torch.equal(full[0, :50, 4], z[0, index[0].long(), 5] * z[0, index[0].long(), 4])
    assert bool(torch.isin(index[0].long(), rows).all())


def test_graphed_detector_with_confluence(cuda_device):
    from helpers import load_synth
    from icafusion_b200 import Model
    from icafusion_b200.engine import GraphedDetector
    from icafusion_b200.confluence import confluence_process
    model = Model("yolov5s_Transfusion_kaist").eval()
    load_synth(model, 6)
    model = model.fuse().half().to(cuda_device)
    gd = GraphedDetector(model, 1, 320, 320, device=cuda_device, confluence=dict(conf_thres=0.3, p_thres=0.5, max_det=4000))
    rgb = torch.rand(1, 3, 320, 320, device=cuda_device).half()
    ir = torch.rand(1, 3, 320, 320, device=cuda_device).half()
    det, count = gd.infer_detections(rgb, ir)
    want = confluence_process(gd.z, 0.3, 0.5)[0]
    n = int(count[0])
    k = min(n, 4000)
    assert (want is None and n == 0) or (n == want.shape[0] and torch.equal(det[0, :k], want[:k].cpu()))
