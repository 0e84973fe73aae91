"""Launch census on the device: every distinct launch the detectors issue (tests/census.py), replayed alone on random operands
of exactly the recorded shapes and pitches and compared with a plain fp32 / float64 reference, at the bars the operator tests
hold.  A launch shared by several configurations is replayed once per session, under the first configuration that issues it."""
import collections
import math
import time

import pytest
import torch

import census
from helpers import sm_count

pytestmark = pytest.mark.gpu

_DONE = set()            # keys replayed so far in this session


@pytest.fixture
def no_tf32():
    """TF32 convolutions and matmuls are ~1e-3 off, the size of the bars: the references run in full fp32."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("config", census.CONFIGS, ids=[c.id for c in census.CONFIGS])
def test_every_launch_matches_its_reference(cuda_device, no_tf32, config):
    props = torch.cuda.get_device_properties(cuda_device)
    sms = sm_count()
    t0 = time.perf_counter()
    todo = {k: r for k, r in census.unique(census.walk_config(config)).items() if k[0] in census.REPLAYED and k not in _DONE}
    t_walk = time.perf_counter() - t0
    stats = collections.defaultdict(lambda: [0, 0.0, 0.0])       # entry point -> [records, worst error / bar, seconds]
    failures = []
    for k, rec in todo.items():
        _DONE.add(k)
        t = time.perf_counter()
        worst, checks = 0.0, None
        try:
            checks = census.replay(rec, cuda_device)
            torch.cuda.synchronize()
            for c in checks:
                e = c.error()
                ratio = (0.0 if e == 0 else math.inf) if c.tol == 0 else e / c.tol
                worst = max(worst, ratio)
                if not ratio <= 1.0:
                    failures.append((rec, f"{c.what}: {e:.3e} (bar {c.tol:g})"))
        except Exception as ex:                                  # noqa: BLE001  (collected; the table below reports it)
            worst = math.inf
            failures.append((rec, f"{type(ex).__name__}: {ex}"))
        del checks
        s = stats[k[0]]
        s[0] += 1
        s[1] = max(s[1], worst)
        s[2] += time.perf_counter() - t
    print(f"\n[{config.id}] {props.name}, {sms} SMs: {len(todo)} new launches (walk {t_walk:.1f} s, total {time.perf_counter() - t0:.1f} s)")
    for name, (n, worst, secs) in sorted(stats.items()):
        print(f"  {name:32s} {n:5d} replayed  worst {worst:.2f} of the bar  {secs:7.1f} s")
    if failures:
        lines = []
        for rec, what in failures[:60]:
            plan = ""
            if rec[0] == "icaf_conv2d_fwd":
                plan = " | " + census.describe_plan(census.conv_plan(rec[1][0]._obj, rec[1][2], sms))
            lines.append(f"{rec[0]} {census.describe(rec)}{plan} | {what}")
        pytest.fail(f"{len(failures)} failing checks in {config.id}:\n" + "\n".join(lines), pytrace=False)
