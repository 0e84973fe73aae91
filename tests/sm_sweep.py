"""SM-count sweep (test helper): the census launches (tests/census.py) whose plan changes when the planners size for fewer SMs
than the device has, as on a smaller part or a MIG slice running the same sm_90a binary.

The planners read the SM count for the conv tile width, split-K factor (the cluster size), ring depth and persistent CTA
count, the weight-gradient M splits and the fused Bottleneck's CTAs per problem.  ``ops.sm_count_target(t)`` makes them
plan for t SMs.  Each swept entry point has a plan signature, computed on the host:

- ``icaf_conv2d_fwd``: icaf_conv2d_plan's (kernel, bn, a_mode, tile_w, tile_h, stages, splits, persistent); a persistent
  plan adds the tiles its CTAs walk, floor and ceiling of tiles / CTAs each capped at 4, and the parity of each (the
  kernel's ping-pong halves and halo slots alternate per tile);
- ``icaf_conv2d_wgrad``: the M split count, icaf_conv2d_wgrad_workspace_bytes under the target over the bytes of one split;
- ``icaf_bottleneck_fwd``: the CTAs per problem.

``select(t)`` returns the records whose (entry point, geometry, n_io, signature) no larger target and not the device's
own count (which the census covers) already gives: replaying them under target t covers every plan the sweep reaches.
A conv or Bottleneck launch is keyed by its geometry and n_io alone; a weight gradient as the census keys it (pitches,
scale and accumulation too).
"""
from __future__ import annotations

import ctypes as C
import functools

import torch

import census
from icafusion_b200 import _lib, ops

# The H100 PCIe (114 SMs), the H20 (78) and the 4g / 3g / 2g / 1g MIG slices of an H100 (64, 60, 32, 16), per NVIDIA's
# published figures; 8 sends every persistent CTA through long tile sequences.
TARGETS = (114, 78, 64, 60, 32, 16, 8)
CPU_SMS = 132           # without a GPU: an H100 SXM's count, as tests/test_persist_plan_cpu.py plans for


def device_sms() -> int:
    """SM count the census runs at: the device's, or CPU_SMS without one."""
    if torch.cuda.is_available():
        from helpers import sm_count
        return sm_count()
    return CPU_SMS


def conv_signature(rec, sms: int) -> tuple:
    _, args, _ = rec
    pl = census.conv_plan(args[0]._obj, args[2], sms)
    assert pl is not None, f"{census.describe(rec)}: no plan at {sms} SMs: {_lib.lib().icaf_last_error().decode()}"
    persistent = pl.ctas < pl.grid_x * pl.grid_y * pl.grid_z
    sig = (pl.kernel, pl.bn, pl.a_mode, pl.tile_w, pl.tile_h, pl.stages, pl.splits, persistent)
    if persistent:
        lo, hi = pl.work_items // pl.ctas, -(-pl.work_items // pl.ctas)
        sig += (min(lo, 4), min(hi, 4), lo % 2, hi % 2)
    return sig


def wgrad_split_bytes(g) -> int:
    """Workspace bytes of one M split of the weight gradient (wgrad.cu, plan_wgrad): fp32 [n_pad][taps][c_pad]."""
    c_tile = 128 if g.Cin % 64 == 0 else g.Cin
    return -(-g.Cout // 128) * 128 * g.kh * g.kw * -(-g.Cin // c_tile) * c_tile * 4


def wgrad_workspace(g, sms: int) -> int:
    with ops.sm_count_target(sms):
        return int(_lib.lib().icaf_conv2d_wgrad_workspace_bytes(C.byref(g)))


def wgrad_signature(rec, sms: int) -> int:
    g = rec[1][0]._obj
    ws, per = wgrad_workspace(g, sms), wgrad_split_bytes(g)
    assert ws > 0 and ws % per == 0, (census.describe(rec), ws, per)
    return ws // per


def bottleneck_signature(rec, sms: int) -> int:
    """CTAs per problem (bottleneck.cu): one per SM split between the problems, at most one per two 32 x 4 output patches."""
    B, H, W, _, n_io = rec[1]
    patches = B * -(-W // 32) * -(-H // 4)
    return max(1, min(sms // n_io, (patches + 1) // 2))


SIGNATURES = {"icaf_conv2d_fwd": conv_signature, "icaf_conv2d_wgrad": wgrad_signature, "icaf_bottleneck_fwd": bottleneck_signature}


def geometry(rec) -> tuple:
    """What a plan signature is paired with: entry point, geometry and n_io (a weight gradient: its census key)."""
    name, args, _ = rec
    if name == "icaf_conv2d_fwd":
        return (name, census._fields(args[0]._obj), args[2])
    if name == "icaf_bottleneck_fwd":
        return (name,) + tuple(args[:3]) + (args[4],)
    return census.key(rec)


@functools.lru_cache(maxsize=None)
def records() -> tuple:
    """The census records of the swept entry points over every configuration, one per census key, in first-issue order."""
    out = {}
    for c in census.CONFIGS:
        for k, r in census.unique(census.walk_config(c)).items():
            if k[0] in SIGNATURES:
                out.setdefault(k, r)
    return tuple(out.values())


@functools.lru_cache(maxsize=None)
def coverage(base: int) -> tuple:
    """[(record, {count: (geometry, signature)})] over the device's count `base` and every target (clamped to `base`, as
    the library clamps them)."""
    return tuple((r, {s: (geometry(r), SIGNATURES[r[0]](r, min(s, base))) for s in (base,) + TARGETS}) for r in records())


def select(target: int, base: int = 0) -> list:
    """The records to replay under `target`: the first record of each (geometry, signature) pair that `target` gives and
    neither `base` (default: the device's count) nor a larger target does."""
    assert target in TARGETS, target
    base = base or device_sms()
    table = coverage(base)
    covered = {cov[s] for _, cov in table for s in (base,) + tuple(t for t in TARGETS if t > target)}
    out = []
    for rec, cov in table:
        if cov[target] not in covered:
            covered.add(cov[target])
            out.append(rec)
    return out
