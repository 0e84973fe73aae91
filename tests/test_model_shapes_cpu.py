"""The oracle against the real reference at the shapes training and validation run (oracle/gen_golden_shapes.py), without a
GPU: test.py's rectangular 544x672 validation batches, where the DMFF token pooling runs windows up to 11 taps tall and 12
wide, and a train.py mosaic batch of 640x640, where build_targets assigns on 80x80 / 40x40 / 20x20 grids."""
import numpy as np
import pytest
import torch

from conftest import load_golden, normwise
from icafusion_b200.cfg import load_cfg
from oracle import icaf_oracle as O
from oracle import synth
from oracle.gen_golden_train import fingerprint, synth_targets

TOL_FP32 = 2e-5


@pytest.mark.parametrize("name", ["yolov5s_544x672", "yolov5l_flir_544x672"])
def test_model_oracle_matches_reference_at_544x672(name):
    """Every fp32 output (z, z of the fused model, logits, the three head maps) against the reference's fingerprint to 2e-5 of
    its norm, and z element by element to the fp16 rounding of the stored copy."""
    m, d = load_golden(name)
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_{m['dataset']}")
    assert cfg["nc"] == m["nc"]
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    with torch.no_grad():
        z, lg, xs = O.model_forward(sd, cfg, rgb, ir)
        zf = O.model_forward(O.fold_bn(sd), cfg, rgb, ir)[0]
    outs = dict(z=z, z_fused=zf, logits=lg, x0=xs[0], x1=xs[1], x2=xs[2])
    assert [list(xs[j].shape[2:4]) for j in range(3)] == [[68, 84], [34, 42], [17, 21]]
    for k, v in outs.items():
        assert list(v.shape) == m["shapes"][k], k
        want = d["fp:" + k]
        assert np.abs(fingerprint(v.numpy(), k) - want).max() < TOL_FP32 * want[0], k
    assert tuple(z.shape) == (1, 22491, m["nc"] + 5) and d["z16"].shape == z.shape
    assert normwise(z.numpy(), d["z16"].astype(np.float32)) < 1e-3          # stored as fp16: rounding <= 2^-11 of max|z|
    assert m["fused_dev"] < 1e-5


def test_training_step_oracle_matches_reference_at_640():
    """oracle.train_step at train.py's 640x640 mosaic shape: loss, every parameter gradient's fingerprint, the 30 parameters
    without a gradient, the Detect maps and BN running statistics against the reference's own step."""
    m, d = load_golden("train_yolov5s_640")
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_kaist")
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    t = synth_targets(m["nt"], m["B"], m["seed"])
    assert np.array_equal(t, d["targets"])
    loss, items, grads, pred, state = O.train_step(sd, cfg, rgb, ir, torch.from_numpy(t), m["hyp"], m["gr"])
    got = np.concatenate([loss.numpy().reshape(1), items.numpy()])
    assert np.allclose(got, d["out"], rtol=1e-4, atol=1e-6), (got, d["out"])
    assert sorted(grads) == sorted(m["params"]) and len(m["dead_params"]) == 30
    worst = max(float(np.abs(fingerprint(grads[k].numpy(), k) - d["g:" + k]).max() / max(d["g:" + k][0], 1e-3)) for k in m["params"])
    assert worst < 2e-4, worst
    for i in range(3):
        want = d[f"pred{i}"]
        assert np.abs(fingerprint(pred[i].numpy(), f"pred{i}") - want).max() < 1e-4 * want[0]
    for k in m["bn_probes"]:
        assert np.allclose(state[k + ".running_mean"].numpy(), d["rm:" + k], rtol=1e-4, atol=1e-6)
        assert np.allclose(state[k + ".running_var"].numpy(), d["rv:" + k], rtol=1e-4, atol=1e-6)
