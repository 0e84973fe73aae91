"""The launch census under the plans smaller Hopper parts and MIG slices get: for each SM-count target (tests/sm_sweep.py),
every conv, weight-gradient (with its data gradient) and fused Bottleneck launch whose plan the census has not run yet is
replayed under ops.sm_count_target and compared with its fp32 / float64 reference at the census's bars."""
import collections
import ctypes as C
import math
import time

import pytest
import torch

import census
import sm_sweep
from test_gpu_census import no_tf32          # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _probe():
    """A 3x3 64 -> 128 weight gradient with 9 work items and 200 M tiles: 2 * sms // 9 splits at every count below 288."""
    from icafusion_b200 import _lib
    return _lib.ConvGeom(1, 160, 160, 64, 160, 160, 128, 3, 3, 1, 1, 576, 128, 0, 0)


@pytest.mark.parametrize("target", sm_sweep.TARGETS)
def test_every_plan_the_target_adds_matches_its_reference(cuda_device, no_tf32, target):      # noqa: F811
    from icafusion_b200 import _lib, ops
    props = torch.cuda.get_device_properties(cuda_device)
    sms = sm_sweep.device_sms()
    # the target reaches the library: the probe's workspace holds fewer splits than at the device's count
    g = _probe()
    per = sm_sweep.wgrad_split_bytes(g)
    own = int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g)))
    assert own == per * min(2 * sms // 9, 64)
    assert sm_sweep.wgrad_workspace(g, target) == per * min(2 * min(target, sms) // 9, 64) < own

    t0 = time.perf_counter()
    todo = sm_sweep.select(target)
    t_select = time.perf_counter() - t0
    stats = collections.defaultdict(lambda: [0, 0.0, 0.0])       # entry point -> [records, worst error / bar, seconds]
    failures = []
    with ops.sm_count_target(target):
        for rec in todo:
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
            except Exception as ex:                              # noqa: BLE001  (collected; the table below reports it)
                worst = math.inf
                failures.append((rec, f"{type(ex).__name__}: {ex}"))
            del checks
            s = stats[rec[0]]
            s[0] += 1
            s[1] = max(s[1], worst)
            s[2] += time.perf_counter() - t
    assert int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g))) == own        # the target is restored
    print(f"\n[{target} of {sms} SMs] {props.name}: {len(todo)} launches with plans the census has not run "
          f"(selection {t_select:.1f} s, total {time.perf_counter() - t0:.1f} s)")
    for name, (n, worst, secs) in sorted(stats.items()):
        print(f"  {name:32s} {n:5d} replayed  worst {worst:.2f} of the bar  {secs:7.1f} s")
    assert set(stats) == set(sm_sweep.SIGNATURES)
    if failures:
        lines = []
        for rec, what in failures[:60]:
            plan = ""
            if rec[0] == "icaf_conv2d_fwd":
                plan = " | " + census.describe_plan(census.conv_plan(rec[1][0]._obj, rec[1][2], target))
            lines.append(f"{rec[0]} {census.describe(rec)}{plan} | {what}")
        pytest.fail(f"{len(failures)} failing checks under {target} SMs:\n" + "\n".join(lines), pytrace=False)
