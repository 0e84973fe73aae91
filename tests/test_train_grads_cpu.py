"""The per-tensor gradient checker of tests/train_grads.py on synthetic tensors, without a GPU: the floor, the one-element
path, the projection bar against the reference's fingerprints, the overflow rule and the two mutations."""
import pytest
import torch

import train_grads as T
from oracle.gen_golden_train import fingerprint


def _golden(ref):
    return {"g:" + k: fingerprint(r.numpy(), k) for k, r in ref.items()}


def _grads(seed=0):
    g = torch.Generator().manual_seed(seed)
    return {
        "model.0.conv.weight": torch.randn(32, 3, 3, 3, generator=g),
        "model.20.pos_emb_vis": torch.randn(1, 64, 32, generator=g) * 0.1,
        "model.20.pos_emb_ir": torch.randn(1, 64, 32, generator=g) * 0.1,
        "model.20.crossatt.key_proj_vis.bias": torch.zeros(32),           # mathematically zero
        "model.20.crossatt.val_proj_vis.bias": torch.randn(32, generator=g) * 1e-3,
        "model.20.crosstransformer.0.coefficient1.bias": torch.tensor([0.2]),
        "model.21.ln.weight": torch.randn(32, generator=g) * 0.5,
    }


def _noisy(ref, rel, seed):
    g = torch.Generator().manual_seed(seed)
    return {k: r + rel * r.norm() / r.numel() ** 0.5 * torch.randn(r.shape, generator=g) for k, r in ref.items()}


def _check(got, ref, amp, golden=None):
    golden = _golden(ref) if golden is None else golden
    floor = T.floor_of(golden, list(ref))
    rows, failures = T.tensor_check(got, ref, amp, golden, T.Projections(), floor)
    return {r[4]: r for r in rows}, dict(failures), floor


def test_clean_gradients_pass_and_rows_cover_every_tensor():
    ref = _grads()
    rows, failures, _ = _check(_noisy(ref, 1e-3, 1), ref, _noisy(ref, 1e-3, 2))
    assert failures == {} and set(rows) == set(ref)


def test_floor_holds_zero_gradients_on_an_absolute_bar():
    ref = _grads()
    golden = _golden(ref)
    floor = T.floor_of(golden, list(ref))
    norms = sorted(float(r.norm()) for r in ref.values())
    assert floor == pytest.approx(1e-2 * norms[len(norms) // 2])
    k = "model.20.crossatt.key_proj_vis.bias"
    for size, fails in ((0.5 * T.TAU, False), (2 * T.TAU, True)):
        got = dict(ref, **{k: torch.full((32,), size * floor / 32 ** 0.5)})
        rows, failures, _ = _check(got, ref, ref, golden)
        assert rows[k][0] == pytest.approx(size, rel=1e-5)                   # |g - 0| / floor, not a division by zero
        assert (k in failures) == fails and len(failures) == fails


def test_bar_follows_the_autocast_oracle_per_tensor():
    ref = _grads()
    k = "model.21.ln.weight"
    amp = dict(ref, **{k: ref[k] * 1.05})                                     # the autocast oracle 5 % off on this tensor
    for rel, fails in ((0.19, False), (0.21, True)):                          # bar = BETA x 5 % = 20 %
        rows, failures, _ = _check(dict(ref, **{k: ref[k] * (1 + rel)}), ref, amp)
        assert rows[k][2] == pytest.approx(T.BETA * 0.05)
        assert (k in failures) == fails and len(failures) == fails


def test_one_element_parameters_follow_the_same_rule_under_their_exemption():
    ref = _grads()
    k = "model.20.crosstransformer.0.coefficient1.bias"
    assert T.exempt_bar(k) > T.TAU and T.exempt_bar("model.21.ln.weight") == 0.0
    assert T.exempt_bar("model.20.vis_coefficient.w2") == T.exempt_bar(k)
    bar = T.exempt_bar(k)
    for rel, fails in ((0.9 * bar, False), (1.1 * bar, True), (-2.0, True)):  # -2: the sign flipped
        rows, failures, _ = _check(dict(ref, **{k: ref[k] * (1 + rel)}), ref, ref)
        assert (k in failures) == fails and len(failures) == fails
    amp = dict(ref, **{k: ref[k] * 1.5})                                      # the autocast oracle 50 % off: BETA x 50 %
    rows, failures, _ = _check(dict(ref, **{k: ref[k] * 3.1}), ref, amp)
    assert rows[k][2] == pytest.approx(T.BETA * 0.5) and k in failures


def test_projection_bar_pins_direction_to_the_reference():
    """The oracle and the device agree exactly, but the reference's gradient differs from the oracle's: only the projections
    on the reference's fingerprint can see it."""
    ref = _grads()
    k = "model.0.conv.weight"
    g = torch.Generator().manual_seed(9)
    off = dict(ref, **{k: ref[k] + 0.05 * ref[k].norm() / ref[k].numel() ** 0.5 * torch.randn(ref[k].shape, generator=g)})
    rows, failures, _ = _check(ref, ref, ref, _golden(off))
    assert rows[k][0] == 0 and set(failures) == {k} and "projection" in failures[k]
    # within the bar: an error of a fifth of TAU in the reference passes
    near = dict(ref, **{k: ref[k] + 2e-3 * ref[k].norm() / ref[k].numel() ** 0.5 * torch.randn(ref[k].shape, generator=g)})
    assert _check(ref, ref, ref, _golden(near))[1] == {}


def test_projections_equal_the_fingerprint():
    ref = _grads()
    p = T.Projections()
    for k, r in ref.items():
        assert p(k, r) == pytest.approx(fingerprint(r.numpy(), k)[1:], rel=1e-12, abs=1e-12)


def test_overflow_rule():
    ref = _grads()
    assert T.overflow(ref, ref) is None
    bad = dict(ref, **{"model.20.pos_emb_ir": ref["model.20.pos_emb_ir"] * float("inf"),
                       "model.21.ln.weight": ref["model.21.ln.weight"] * float("nan")})
    with pytest.raises(AssertionError, match="model.20.pos_emb_ir"):          # the first non-finite tensor, in order
        T.overflow(bad, ref)
    why = T.overflow(ref, bad)
    assert "model.20.pos_emb_ir" in why and "device: finite" in why
    assert "device: model.20.pos_emb_ir" in T.overflow(bad, bad)


def test_mutations_are_caught_by_name():
    ref = _grads()
    ref["model.1.conv.weight"] = torch.randn(256, 128, 3, 3, generator=torch.Generator().manual_seed(3))  # dominates the L2
    got, amp = _noisy(ref, 1e-3, 1), _noisy(ref, 1e-3, 2)
    golden = _golden(ref)
    floor = T.floor_of(golden, list(ref))
    assert T.hidden_from_global_l2(ref) == "model.20.crossatt.val_proj_vis.bias"      # of the two 32-element ones, the larger
    assert T.closest_pos_emb_pair(ref) == ("model.20.pos_emb_vis", "model.20.pos_emb_ir")
    T.check_mutations(got, ref, amp, golden, T.Projections(), floor, "[synthetic]")
