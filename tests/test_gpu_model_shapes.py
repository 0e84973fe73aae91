"""The device at the shapes training and validation run, against the real reference (tests/golden, oracle/gen_golden_shapes.py):
test.py's rectangular 544x672 validation batches, eval forward unfused and fused, and one train.py step on a 640x640 mosaic
batch.  tests/test_model_shapes_cpu.py pins the oracle used here to the same goldens."""
import pytest
import torch

from conftest import load_golden
from helpers import err, load_synth
from oracle import icaf_oracle as O
from oracle import synth
from test_gpu_model import TOL_MODEL
from test_gpu_train_model import check_training_step

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["yolov5s_544x672", "yolov5l_flir_544x672"])
@pytest.mark.parametrize("fused", [False, True])
def test_model_matches_reference_golden_at_544x672(cuda_device, name, fused):
    """z against the reference's (stored in fp16; fused and unfused reference differ by ~1e-6, meta 'fused_dev'); logits and
    the three head maps against the fp32 oracle; at the bar of the other whole-model goldens."""
    from icafusion_b200 import Model
    from icafusion_b200.cfg import load_cfg
    m, d = load_golden(name)
    cfg = load_cfg(f"yolov5{m['size']}_Transfusion_{m['dataset']}")
    model = Model(cfg).eval()
    sd = load_synth(model, m["seed"])
    if fused:
        model.fuse()
    model = model.to(cuda_device)
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    with torch.no_grad():
        z, logits, xs = model(rgb.to(cuda_device), ir.to(cuda_device))
        _, lr, xr = O.model_forward(O.fold_bn(sd) if fused else sd, cfg, rgb, ir)
    torch.cuda.synchronize()
    ez = err(z, d["z16"].astype("float32"))
    el = err(logits, lr)
    ex = max(err(xs[j], xr[j]) for j in range(3))
    print(f"\n[{name} fused={fused}] z {ez:.2e} logits {el:.2e} x {ex:.2e}  (reference fp16 self-dev: {m.get('ref_fp16_self_dev')})")
    assert tuple(z.shape) == d["z16"].shape and len(xs) == 3
    assert ez < TOL_MODEL and el < TOL_MODEL and ex < TOL_MODEL


def test_training_step_yolov5s_640(cuda_device):
    check_training_step(cuda_device, "train_yolov5s_640")
