"""One whole-model training step (train.py:334-344), held one gradient tensor at a time.

The device's train-mode forward, ComputeLoss and scaled backward run against the fp32 oracle (oracle.icaf_oracle.train_step,
itself pinned to the reference's own step by the training goldens) and against the same oracle under fp16 autocast at the
same loss scale -- the reference's training regime, whose distance from fp32 sets each bar.  For every live parameter k,
with g_k the device's gradient divided by the scale, r_k the fp32 oracle's and a_k the autocast oracle's:

    e_k   = |g_k - r_k| / max(|r_k|, floor)         ea_k = |a_k - r_k| / max(|r_k|, floor)
    bar_k = max(BETA * ea_k, TAU)                   and   e_k <= bar_k
    |<g_k, w_j> - golden_j| <= C_PROJ * bar_k * max(|r_k|, floor)       for the golden's two seeded projections j = 1, 2

floor is 1e-2 of the median gradient norm of the reference: it keeps the mathematically zero gradients (key-projection
biases, the last MLP biases) on an absolute bar.  The projections (oracle.gen_golden_train.fingerprint) are of the REAL
reference's gradients, so they pin each tensor's direction to the reference itself: an error vector's projection on a
Gaussian w has a standard deviation equal to its norm, and 5 sigma leaves margin over the ~1,300 projections of a case.
A norm alone does not see a sign flip or two same-shape gradients swapped, and an L2 over all gradients together is
dominated by the large conv weights; the per-tensor bar sees both (tests/test_gpu_train_grads.py shows it on the device).

One-element parameters (LearnableCoefficient / LearnableWeights) follow the same rule, with the floor of their entry in
EXEMPT.  Each is one cancelling sum over a whole token stream, so ea_k reaches ~100 % on some and their bar is loose by
construction; the report lists them apart, and _module_case in tests/test_gpu_train_model.py holds them at 1e-1 on short
chains.

Each case runs at the static loss scale 2^8 the suite always used and at 2^16, GradScaler's init_scale (train.py:282).
Where the autocast oracle's gradients are finite the device's must be too.  Where the autocast oracle overflows (on an
H100 it does at 2^16 in every case: the Detect biases' or the stem's fp16 weight gradients), the case reports it and, if
the device's gradients are finite, holds them to the bars of the autocast oracle at 2^8; if they are not, or there is no
smaller finite scale, it skips the per-tensor check, as GradScaler would skip that step.
"""
from __future__ import annotations

import re
import warnings
import zlib

import numpy as np
import torch

BETA = 4.0
TAU = 1e-2
C_PROJ = 5.0
SCALES = (2.0 ** 8, 2.0 ** 16)
SENSITIVE = 5e-2          # a tensor whose bar is at or below this is one a gross error in it cannot hide from

# Tensors the device cannot hold to the common bar: (name pattern, their bar, why, the module test that holds them).
EXEMPT = [
    (re.compile(r"(\.coefficient\d\.bias|_coefficient\.w[12])$"), 1.5,
     "LearnableCoefficient / LearnableWeights: each gradient is one cancelling sum over a DMFF token stream.  Under the "
     "reference's autocast a one-element fp32 parameter times an fp16 tensor promotes to fp32, so the autocast oracle's token "
     "streams and their gradients are fp32; the device keeps them in fp16.  Measured on an H100: up to 86 x the autocast "
     "oracle's error (yolov5l model.20.crosstransformer.0.coefficient3.bias: 1.10 against 1.3e-2); multi-element gradients "
     "fed by the same stream gradients (the MLP output biases) stay within 1.2 x.  1.5 still fails a sign flip (2.0)",
     "tests/test_gpu_train_model.py::test_c3_sppf_fusion_block_nodes (every one-element gradient of a DMFF block, 1e-1)"),
]


def exempt_bar(k: str) -> float:
    return max((bar for pat, bar, _, _ in EXEMPT if pat.search(k)), default=0.0)


def floor_of(golden, live) -> float:
    return 1e-2 * float(np.median([golden["g:" + k][0] for k in live]))


def _norm(t: torch.Tensor) -> float:
    return float(t.double().norm())


def first_nonfinite(grads: dict):
    return next((k for k, g in grads.items() if not bool(torch.isfinite(g).all())), None)


def overflow(got: dict, amp: dict):
    """None when both sides are finite.  When the autocast oracle overflows: the reason the per-tensor check is skipped.
    When only the device overflows: fails, naming the device's first tensor that is not finite."""
    ka, kd = first_nonfinite(amp), first_nonfinite(got)
    if ka is not None:
        return f"the fp16-autocast oracle overflows (first non-finite gradient {ka}; device: {kd or 'finite'})"
    assert kd is None, f"device gradient not finite where the fp16-autocast oracle's is: {kd}"
    return None


class Projections:
    """<g, w_1>, <g, w_2> with the seeded Gaussian vectors of fingerprint(), drawn once per tensor and kept on g's device."""

    def __init__(self):
        self.w = {}

    def __call__(self, k: str, g: torch.Tensor) -> np.ndarray:
        w = self.w.get(k)
        if w is None:
            r = np.random.Generator(np.random.PCG64([23, zlib.crc32(k.encode())]))
            w = self.w[k] = torch.from_numpy(np.stack([r.standard_normal(g.numel()), r.standard_normal(g.numel())])).to(g.device)
        return (w @ g.reshape(-1).double()).cpu().numpy()


def tensor_check(got: dict, ref: dict, amp: dict, golden, proj: Projections, floor: float):
    """-> (rows, failures): rows (e_k, ea_k, bar_k, projection deviation in units of its bar, k) for every tensor of `ref`;
    failures the tensors over either bar, each with its reason."""
    rows, failures = [], []
    for k, r in ref.items():
        den = max(_norm(r), floor)
        e, ea = _norm(got[k] - r) / den, _norm(amp[k] - r) / den
        bar = max(BETA * ea, TAU, exempt_bar(k))
        dp = float(np.abs(proj(k, got[k]) - golden["g:" + k][1:]).max()) / (C_PROJ * bar * den)
        rows.append((e, ea, bar, dp, k))
        if e > bar:
            failures.append((k, f"error {e:.2e} > bar {bar:.2e} (fp16-autocast oracle {ea:.2e})"))
        elif dp > 1:
            failures.append((k, f"projection on the reference's gradient off by {dp:.2f} x its bar {C_PROJ:g} x {bar:.2e}"))
    return rows, failures


def global_l2(got: dict, ref: dict, amp: dict):
    """Relative L2 error over all gradients together, device and autocast oracle."""
    num = sum(_norm(got[k] - r) ** 2 for k, r in ref.items())
    num_a = sum(_norm(amp[k] - r) ** 2 for k, r in ref.items())
    den = sum(_norm(r) ** 2 for r in ref.values())
    return (num / den) ** 0.5, (num_a / den) ** 0.5


def norm_deviation(got: dict, amp: dict, golden, floor: float):
    """Worst relative difference of a multi-element gradient's norm from the reference's, device and autocast oracle."""
    dev = lambda g, k: abs(_norm(g) - golden["g:" + k][0]) / max(golden["g:" + k][0], floor)     # noqa: E731
    keys = [k for k, g in got.items() if g.numel() > 1]
    return max(dev(got[k], k) for k in keys), max(dev(amp[k], k) for k in keys)


def aggregate_checks(got: dict, ref: dict, amp: dict, golden, floor: float):
    """The whole-gradient assertions the suite held before the per-tensor check: -> (passes, description)."""
    l2, l2a = global_l2(got, ref, amp)
    nd, nda = norm_deviation(got, amp, golden, floor)
    ok = l2 < max(1.5 * l2a, 2e-3) and nd < max(1.5 * nda, 2e-2)
    return ok, f"global L2 {l2:.2e} (fp16-autocast {l2a:.2e}), worst norm deviation {nd:.2e} (fp16-autocast {nda:.2e})"


def bn_check(state: dict, ref_state: dict, amp_state: dict):
    """Every BatchNorm's running_mean and running_var after the step: relative L2 error against the fp32 oracle's, held to
    max(BETA x the autocast oracle's, TAU).  -> (worst (e, ea, key), failures)."""
    worst, failures = (0.0, 0.0, ""), []
    for k, r in ref_state.items():
        if not k.endswith(("running_mean", "running_var")):
            continue
        r = r.to(state[k].device)
        den = _norm(r)
        e, ea = _norm(state[k].float() - r) / den, _norm(amp_state[k].to(r.device).float() - r) / den
        worst = max(worst, (e, ea, k))
        if e > max(BETA * ea, TAU):
            failures.append((k, f"error {e:.2e} (fp16-autocast oracle {ea:.2e})"))
    return worst, failures


def report(tag: str, rows, scalars, l2, l2a) -> dict:
    """Print the worst ten tensors, the one-element parameters and the share of tight bars; -> the summary numbers."""
    multi = [r for r in rows if r[4] not in scalars]
    multi.sort(key=lambda r: r[0] / r[2], reverse=True)
    ratio = max(rows, key=lambda r: r[0] / max(r[1], 1e-30))
    share = sum(r[2] <= SENSITIVE for r in rows) / len(rows)
    over_tau = [r for r in rows if r[0] > TAU]
    need_beta = max((r[0] / r[1] for r in over_tau), default=0.0)          # the least BETA that would pass, given TAU
    need_tau = max((r[0] for r in rows if r[0] > BETA * r[1]), default=0.0)  # the least TAU that would pass, given BETA
    print(f"{tag} all {len(rows)} gradients: global relative L2 {l2:.2e} (fp16-autocast oracle {l2a:.2e}); "
          f"bars <= {SENSITIVE:g}: {100 * share:.1f} %; worst e/ea {ratio[0] / max(ratio[1], 1e-30):.2f} ({ratio[4]}); "
          f"least BETA at TAU {TAU:g}: {need_beta:.2f}; least TAU at BETA {BETA:g}: {need_tau:.2e}")
    print(f"{tag} worst tensors (e_k, ea_k, e_k / ea_k, bar_k, projection / its bar):")
    for e, ea, bar, dp, k in multi[:10]:
        print(f"    {e:.2e} {ea:.2e} {e / max(ea, 1e-30):7.2f} {bar:.2e} {dp:.2f} {k}")
    print(f"{tag} one-element parameters, loose by construction (e_k, ea_k, e_k / ea_k, bar_k):")
    for e, ea, bar, dp, k in sorted((r for r in rows if r[4] in scalars), reverse=True):
        print(f"    {e:.2e} {ea:.2e} {e / max(ea, 1e-30):7.2f} {bar:.2e} {dp:.2f} {k}")
    return dict(l2=l2, l2a=l2a, share=share, ratio=ratio[0] / max(ratio[1], 1e-30), ratio_k=ratio[4])


def hidden_from_global_l2(ref: dict) -> str:
    """The largest multi-element tensor whose negation moves the all-gradient relative L2 by less than 2e-3."""
    total = sum(_norm(r) ** 2 for r in ref.values()) ** 0.5
    hidden = [k for k, r in ref.items() if r.numel() > 1 and 2 * _norm(r) < 2e-3 * total]
    return max(hidden, key=lambda k: (ref[k].numel(), _norm(ref[k])))


def closest_pos_emb_pair(ref: dict):
    """The DMFF whose RGB and IR positional-embedding gradients are closest: the swap the norms and the L2 see least."""
    pairs = [(k, k[:-3] + "ir") for k in ref if k.endswith("pos_emb_vis")]
    return min(pairs, key=lambda p: _norm(ref[p[0]] - ref[p[1]]))


# ---- the device step and its oracles ---------------------------------------------------------------------------------------

def _cfg_name(m) -> str:
    return f"yolov5{m['size']}_Transfusion_{m.get('dataset') or 'kaist'}"


def device_step(cuda_device, m, d, scale: float):
    from helpers import load_synth
    from icafusion_b200 import Model
    from icafusion_b200.loss import ComputeLoss
    from oracle import synth
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    model = Model(_cfg_name(m))
    load_synth(model, m["seed"])
    model = model.to(cuda_device).train()
    for mod in model.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0                                   # the golden / oracle graph is dropout free
    model.hyp, model.gr = dict(m["hyp"]), m["gr"]
    pred = model(rgb.to(cuda_device), ir.to(cuda_device))
    loss, items = ComputeLoss(model)(pred, torch.from_numpy(d["targets"]).to(cuda_device))
    (loss * scale).sum().backward()
    torch.cuda.synchronize()
    return model, pred, loss, items


def oracle_step(m, d, autocast_device=None, scale: float = 1.0):
    from icafusion_b200.cfg import load_cfg
    from oracle import icaf_oracle as O
    from oracle import synth
    cfg = load_cfg(_cfg_name(m))
    sd = synth.synth_state_dict(synth.model_param_shapes(cfg), m["seed"])
    rgb, ir = synth.synth_images(m["B"], m["H"], m["W"], m["seed"])
    return O.train_step(sd, cfg, rgb, ir, torch.from_numpy(d["targets"]), m["hyp"], m["gr"], autocast_device=autocast_device,
                        loss_scale=scale)


def check_step(model, pred, loss, items, ref, amp, m, d, scale: float, proj: Projections, tag: str, held=None):
    """Every assertion on one scaled step; -> (failures, summary, device gradients / scale, fp32 and autocast gradients, floor)
    with the per-tensor and BatchNorm failures collected rather than raised, so that a case reports all its scales first.
    held: the autocast oracle's gradients at a smaller scale, whose bars hold the device's finite gradients where the
    autocast oracle overflows at this one; without it the per-tensor check is skipped there."""
    rl, ri, rg, rp, rstate = ref
    _, _, ag, ap, astate = amp
    got = torch.cat([loss.detach(), items]).cpu().numpy()
    want = np.concatenate([rl.numpy().reshape(1), ri.numpy()])
    print(f"\n{tag} loss device {got}  oracle {want}  reference {d['out']}")
    assert np.allclose(got, want, rtol=3e-3, atol=1e-4) and np.allclose(got, d["out"], rtol=3e-3, atol=1e-4)
    for i in range(3):
        e = float((pred[i].detach().float().cpu() - rp[i]).abs().max() / rp[i].abs().max())
        ea = float((ap[i].detach().float().cpu() - rp[i]).abs().max() / rp[i].abs().max())
        print(f"{tag} Detect map {i}: {e:.2e}   (fp16-autocast oracle: {ea:.2e})")
        # fp16 activations through ~60 batch-statistics BatchNorms: the bar is the reference regime's own distance from fp32
        assert e < max(1.5 * ea, 5e-3)
    params = dict(model.named_parameters())
    live = [k for k, p in params.items() if p.grad is not None]
    assert sorted(live) == sorted(m["params"]) == sorted(rg)        # the reference's 30 dead parameters stay without gradient
    dev = params[live[0]].device
    g = {k: params[k].grad.detach().float() / scale for k in live}
    r = {k: rg[k].to(dev) for k in live}
    a = {k: ag[k].float() for k in live}
    state = model.state_dict()
    failures, probes = [], []
    for k in m["bn_probes"]:
        for stat, key in (("running_mean", "rm:"), ("running_var", "rv:")):
            # against the reference itself, element by element: within rtol 5e-3 / atol 2e-4, or, where the reference's own
            # fp16 regime lands further off than that, within 1.5 x the autocast oracle's distance
            q, qa = (_allclose_ratio(st[f"{k}.{stat}"], d[key + k]) for st in (state, astate))
            probes.append((q, qa, f"{k}.{stat}"))
            if q > max(1.0, 1.5 * qa):
                failures.append((f"{k}.{stat}", f"{q:.2f} x the probe tolerance (fp16-autocast oracle {qa:.2f} x)"))
    q, qa, kp = max(probes)
    print(f"{tag} BN probes against the reference: worst {q:.2f} x rtol 5e-3 / atol 2e-4 (fp16-autocast oracle {qa:.2f} x) {kp}")
    (e, ea, kb), fb = bn_check(state, rstate, astate)
    failures += fb
    print(f"{tag} running statistics of every BatchNorm: worst {e:.2e} (fp16-autocast oracle {ea:.2e}) {kb}")
    floor = floor_of(d, live)
    skip = overflow(g, a)
    if skip is not None:
        if held is None or first_nonfinite(g) is not None:
            print(f"{tag} per-tensor check skipped: {skip}")
            warnings.warn(f"{tag} per-tensor check skipped: {skip}")
            return failures, dict(overflow=skip), g, r, a, floor
        print(f"{tag} {skip}: the device's finite gradients are held to the bars of the autocast oracle at the smaller scale")
        a = held
    rows, tf = tensor_check(g, r, a, d, proj, floor)
    summary = report(tag, rows, {k for k in live if params[k].numel() == 1}, *global_l2(g, r, a))
    summary["overflow"] = skip
    ok, desc = aggregate_checks(g, r, a, d, floor)
    print(f"{tag} {desc}")
    assert ok, desc
    return failures + tf, summary, g, r, a, floor


def _allclose_ratio(x: torch.Tensor, want: np.ndarray) -> float:
    """max |x - want| / (2e-4 + 5e-3 |want|): at most 1 where np.allclose(x, want, rtol=5e-3, atol=2e-4) holds."""
    return float((np.abs(x.float().cpu().numpy() - want) / (2e-4 + 5e-3 * np.abs(want))).max())


def check_mutations(g, r, a, d, proj, floor, tag, failing=()):
    """Perturbed copies of the device's gradients, no launches: (a) the largest multi-element tensor an all-gradient L2 bar
    of 2e-3 cannot see, negated -- the aggregate assertions pass it, the per-tensor check names it; (b) one DMFF's RGB and
    IR positional-embedding gradients swapped -- the per-tensor check fails, naming only them.  `failing`: the tensors the unperturbed
    gradients already fail on."""
    def caught(grads):
        return sorted({n for n, _ in tensor_check(grads, r, a, d, proj, floor)[1]} - set(failing))
    k = hidden_from_global_l2(r)
    neg = dict(g, **{k: -g[k]})
    ok, desc = aggregate_checks(neg, r, a, d, floor)
    c = caught(neg)
    print(f"{tag} mutation (a) {k} negated: aggregate assertions {'pass' if ok else 'FAIL'} ({desc}); per-tensor check fails {c}")
    assert ok, desc
    assert c == [k], c
    kv, ki = closest_pos_emb_pair(r)
    swap = dict(g, **{kv: g[ki], ki: g[kv]})
    c = caught(swap)
    print(f"{tag} mutation (b) {kv} <-> {ki}: global L2 {global_l2(swap, r, a)[0]:.2e}; per-tensor check fails {c}")
    # both, unless the autocast oracle's own error on one of them is as large as the swap (yolov5l's model.20.pos_emb_ir)
    assert c and set(c) <= {kv, ki}, c


def run_case(cuda_device, name: str):
    """The golden's case at every scale of SCALES, then the two mutations on the 2^8 gradients; fails at the end, listing
    every tensor over its bar at every scale."""
    from conftest import load_golden
    m, d = load_golden(name)
    ref = oracle_step(m, d)
    proj = Projections()
    failures, held = [], None
    for scale in SCALES:
        tag = f"[{name} scale 2^{int(np.log2(scale))}]"
        model, pred, loss, items = device_step(cuda_device, m, d, scale)
        amp = oracle_step(m, d, autocast_device=cuda_device, scale=scale)
        fails, summary, g, r, a, floor = check_step(model, pred, loss, items, ref, amp, m, d, scale, proj, tag, held)
        failures += [(tag, k, why) for k, why in fails]
        if summary["overflow"] is None:
            held = a
            if scale == SCALES[0]:
                check_mutations(g, r, a, d, proj, floor, tag, [k for k, _ in fails])
        del model, pred, loss, items, amp, g, r, a
    assert not failures, "\n".join(f"{t} {k}: {why}" for t, k, why in failures)
