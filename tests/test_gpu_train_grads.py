"""yolov5l's training step -- the one trained size with head dim 128 in the attention backward and C3 stacks of up to nine
Bottlenecks -- against fp32 autograd through the oracle and the reference's own step (tests/golden/train_yolov5l_320.npz,
oracle/gen_golden_train_l.py), one gradient tensor at a time at loss scales 2^8 and 2^16, and the two perturbed copies of
its gradients that the per-tensor check must name (tests/train_grads.py)."""
import pytest

import train_grads

pytestmark = pytest.mark.gpu


def test_training_step_yolov5l_320(cuda_device):
    train_grads.run_case(cuda_device, "train_yolov5l_320")
