"""The row-wise, RoPE, loss and argmax checkers have teeth (CPU only).

Each test emulates in torch one kernel bug the GPU tests in test_rowwise_exact_gpu.py and test_loss_exact_gpu.py exist
to catch and requires the same reference and checker to reject it; the clean emulation must pass. Nothing here builds
or runs a kernel.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.exact import assert_between, assert_equal, assert_rounds_within, assert_within, round_bf16_from_fp64
from tests.test_loss_exact_gpu import argmax_ref, ce_dlogits_ref, ce_lse_bound, ce_rows
from tests.test_rowwise_exact_gpu import rms_inputs, rmsnorm_interval, rope_ref

CPU = torch.device("cpu")


# ------------------------------------------------------------------------------------------------ the helpers
def test_round_bf16_from_fp64_rounds_once():
    x = torch.tensor([1 + 2.0 ** -8 + 2.0 ** -30], dtype=torch.float64)
    assert float(x.to(torch.bfloat16)) == 1.0                          # torch: fp64 -> fp32 -> bf16, twice rounded
    assert float(round_bf16_from_fp64(x)) == 1 + 2.0 ** -7
    ties = torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8 - 2.0 ** -40), 3.5e38, -1e-50, math.inf,
                         math.nan], dtype=torch.float64)
    got = round_bf16_from_fp64(ties).double()
    assert got[:6].tolist() == [1.0, 1 + 2.0 ** -6, -1.0, math.inf, -0.0, math.inf]   # ties to even; overflow; -0
    assert math.isnan(float(got[6]))
    # agrees with the single rounding of numpy's float32 wherever the fp32 step is exact
    r = torch.randn(10000, dtype=torch.float64).float().double()
    assert torch.equal(round_bf16_from_fp64(r), r.float().to(torch.bfloat16))


def test_rounds_within_admits_both_neighbours_at_a_tie_and_nothing_else():
    ref = torch.tensor([1 + 2.0 ** -8], dtype=torch.float64)            # halfway between 1 and 1 + 2^-7
    err = torch.tensor([2.0 ** -20])
    for v in (1.0, 1 + 2.0 ** -7):
        assert_rounds_within(torch.tensor([v]).bfloat16(), ref, err, "neighbour")
    for v in (1 - 2.0 ** -8, 1 + 2.0 ** -6):
        with pytest.raises(AssertionError):
            assert_rounds_within(torch.tensor([v]).bfloat16(), ref, err, "one further")
    off = torch.tensor([1 + 2.0 ** -9], dtype=torch.float64)            # far from a tie: only round(ref)
    assert_rounds_within(torch.tensor([1.0]).bfloat16(), off, err, "exact")
    with pytest.raises(AssertionError):
        assert_rounds_within(torch.tensor([1 + 2.0 ** -7]).bfloat16(), off, err, "the other neighbour")
    with pytest.raises(AssertionError):
        assert_rounds_within(torch.tensor([math.nan]).bfloat16(), off, err, "NaN")


# ------------------------------------------------------------------------------------------------ RMSNorm
def _rms_emulate(x, w, eps, rstd_rows=None, drop_slot=None):
    """The kernel's arithmetic in fp32: rstd from (optionally) another row, or without one 256-vector slot."""
    xf = x.float()
    sq = xf * xf
    if drop_slot is not None:
        sq[:, drop_slot * 2048:(drop_slot + 1) * 2048] = 0
    rstd = torch.rsqrt(sq.sum(1, keepdim=True) / x.shape[1] + eps)
    if rstd_rows is not None:
        rstd = rstd[rstd_rows]
    n = (xf * rstd).bfloat16().float()
    return (w.float() * n).bfloat16()


@pytest.mark.parametrize("bug", ["previous_row_rstd", "dropped_last_vpt_slot"])
def test_rmsnorm_check_rejects(bug):
    H, M = 4104 if bug == "dropped_last_vpt_slot" else 2056, 40
    x, w = rms_inputs(M, H, CPU, seed=3)
    lo, hi = rmsnorm_interval(x, w, 1e-5)
    assert_between(_rms_emulate(x, w, 1e-5), lo, hi, "clean")
    kw = {"rstd_rows": torch.arange(M) - 1} if bug == "previous_row_rstd" else {"drop_slot": 2}
    with pytest.raises(AssertionError) as e:
        assert_between(_rms_emulate(x, w, 1e-5, **kw), lo, hi, bug)
    print(f"rejected: {e.value}")


# ------------------------------------------------------------------------------------------------ cross-entropy
def _ce_emulate(x, V, drop_tail):
    """lse as the kernel's two passes would produce it, in fp64, optionally without the pass-1 scalar tail."""
    n = V & ~3 if drop_tail else V
    return torch.logsumexp(x[:, :n].double(), 1)


def test_ce_lse_check_rejects_a_dropped_pass1_tail():
    V = 2047
    x = ce_rows(8, V, torch.Generator().manual_seed(1))
    x[1, V - 1] += 80                                                  # a maximum in the tail (V mod 4 = 3)
    lse64, err = ce_lse_bound(x, V)
    assert_within(_ce_emulate(x, V, False), lse64, err, "clean")
    with pytest.raises(AssertionError) as e:
        assert_within(_ce_emulate(x, V, True), lse64, err, "pass-1 tail dropped")
    print(f"rejected: {e.value}")


def test_ce_dlogits_check_rejects_a_onehot_missed_in_the_pass2_tail():
    V = 2047                                                           # V8 = 2040: labels 2044 and 2046 in the tail
    x = ce_rows(4, V, torch.Generator().manual_seed(2))
    labels = torch.tensor([2044, 2046, 5, -100], dtype=torch.int32)
    lse64, _ = ce_lse_bound(x, V)
    lse = lse64.float()
    ref, err = ce_dlogits_ref(x, lse, lse64, labels, 0.25)
    p = torch.exp(x.double() - lse.double()[:, None]).float()
    good = ((p - F.one_hot(labels.clamp(min=0).long(), V).float()) * 0.25 * (labels != -100)[:, None]).bfloat16()
    assert_rounds_within(good, ref, err, "clean")
    bad = good.clone()
    bad[:2] = (p[:2] * 0.25).bfloat16()                                # the tail never compares j == label
    with pytest.raises(AssertionError) as e:
        assert_rounds_within(bad, ref, err, "onehot missed in the pass-2 tail")
    print(f"rejected: {e.value}")


# ------------------------------------------------------------------------------------------------ RoPE
def test_rope_check_rejects_swapped_halves():
    d, M, n = 128, 64, 4
    g = torch.Generator().manual_seed(4)
    x = torch.randn(M, n, d, generator=g).bfloat16()
    ang = torch.rand(M, 1, d // 2, generator=g) * 6
    c, s = ang.cos().bfloat16().float(), ang.sin().bfloat16().float()
    ref, err = rope_ref(x, c, s, d)
    a, b = x.float()[..., :d // 2], x.float()[..., d // 2:]
    good = torch.cat([a * c - b * s, b * c + a * s], -1).bfloat16()
    assert_rounds_within(good, ref, err, "clean")
    bad = torch.cat([b * c + a * s, a * c - b * s], -1).bfloat16()
    with pytest.raises(AssertionError) as e:
        assert_rounds_within(bad, ref, err, "halves swapped")
    print(f"rejected: {e.value}")


# ------------------------------------------------------------------------------------------------ bilinear
def test_bilinear_check_rejects_a_tap_off_by_one():
    S, T, C = 27, 8, 16
    x = torch.randn(1, C, S, S).bfloat16().float()
    ref = F.interpolate(x, size=(T, T), mode="bilinear", align_corners=False).bfloat16()
    bad = F.interpolate(torch.roll(x, 1, dims=3), size=(T, T), mode="bilinear", align_corners=False).bfloat16()
    assert_equal(ref, ref, "clean")
    with pytest.raises(AssertionError) as e:
        assert_equal(bad, ref, "x tap off by one")
    print(f"rejected: {e.value}")


# ------------------------------------------------------------------------------------------------ argmax
def test_argmax_reference_rejects_the_unset_index():
    x = torch.full((3, 65), -math.inf)
    x[1] = math.nan
    x[2, ::2] = math.nan
    want = argmax_ref(x)
    assert want.tolist() == [0, 0, 0]
    assert int(torch.argmax(torch.tensor([1.0, math.nan]))) == 1       # torch.argmax picks NaN: not this rule
    unset = torch.full((3,), 0x7fffffff, dtype=torch.int32)
    with pytest.raises(AssertionError) as e:
        assert_equal(unset, want, "argmax returning 0x7fffffff")
    print(f"rejected: {e.value}")
    y = torch.tensor([[1.0, math.nan, 3.0, 3.0, math.inf, math.inf]])
    assert argmax_ref(y).tolist() == [4]
