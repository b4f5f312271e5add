"""CPU tests of decode log-probabilities: the C ABI's argument checks, the `logprobs=` validation of every entry point,
the fp64 restatement (oracle/logprobs.py) pinned by hand-computed rows, and its checkers rejecting emulated kernel bugs."""
import math

import numpy as np
import pytest
import torch

import oracle.logprobs as O

NAN = float("nan")
INF = float("inf")


def test_decode_logprobs_rejects_bad_arguments_without_gpu():
    from ctypes import c_int, c_void_p
    from metamorph_b200 import _build
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    _build.build(verbose=False)
    a = c_void_p(256)    # never dereferenced: the argument checks reject the call first
    z = c_void_p(0)

    def args(ld, R, V, max_ids=4, ptrs=None):
        p = ptrs or [a] * 8
        return (p[0], ll(ld), ll(R), c_int(V), p[1], p[2], p[3], p[4], c_int(max_ids), p[5], p[6], p[7], c_void_p(0))

    with pytest.raises(MetaMorphB200Error, match="bad shape"):
        call("mm_decode_logprobs", *args(100, 4, 128))             # ld < V
    with pytest.raises(MetaMorphB200Error, match="bad shape"):
        call("mm_decode_logprobs", *args(128, 0, 128))
    with pytest.raises(MetaMorphB200Error, match="bad shape"):
        call("mm_decode_logprobs", *args(128, 1, 0))
    with pytest.raises(MetaMorphB200Error, match="bad shape"):
        call("mm_decode_logprobs", *args(128, 1, 128, max_ids=0))
    with pytest.raises(MetaMorphB200Error, match="too many rows"):
        call("mm_decode_logprobs", *args(128, 1 << 29, 128))
    with pytest.raises(MetaMorphB200Error, match="shared-memory budget"):
        call("mm_decode_logprobs", *args(400000, 1, 393217))     # one element past 8 x 48K fp32 per CTA
    for k in range(8):
        p = [a] * 8
        p[k] = z
        with pytest.raises(MetaMorphB200Error, match="null pointer"):
            call("mm_decode_logprobs", *args(128, 1, 128, ptrs=p))


BAD = [-1, 21, True, 2.0, "5", np.float32(3)]


@pytest.mark.parametrize("bad", BAD)
def test_logprobs_argument_is_validated_before_device_work(bad):
    """A DecodeEngine without a model and a server without a device: the check comes first, so nothing else runs."""
    from metamorph_b200.engine.decode import DecodeEngine
    from metamorph_b200.engine.serve import ContinuousBatcher
    from metamorph_b200.model.metamorph_llama import MetaMorphLlamaForCausalLM
    with pytest.raises(ValueError, match="logprobs"):
        DecodeEngine(None).generate(torch.zeros(1, 2, 8), logprobs=bad)
    with pytest.raises(ValueError, match="logprobs"):
        ContinuousBatcher.__new__(ContinuousBatcher).submit(torch.zeros(2, 8), logprobs=bad)
    with pytest.raises(ValueError, match="logprobs"):
        MetaMorphLlamaForCausalLM.generate(None, torch.zeros(1, 2, dtype=torch.long), logprobs=bad)


def test_logprobs_accepts_every_count_in_range():
    from metamorph_b200.engine.logprobs import check_logprobs
    for n in [None, 0, 1, 5, 20, np.int64(7)]:
        check_logprobs(n)


# ---------------------------------------------------------------- the restatement, by hand
def test_oracle_plain_row():
    row = np.array([0.0, math.log(3.0), 0.0], dtype=np.float32)      # probabilities 1/5, 3/5, 1/5
    lp, ids, lps = O.report(row, 0, 3)
    assert ids.tolist() == [1, 0, 2]                                  # the tie 0 / 2 goes to the lower index
    np.testing.assert_allclose(lps, [math.log(3 / 5), math.log(1 / 5), math.log(1 / 5)], rtol=0, atol=1e-7)
    assert abs(lp - math.log(1 / 5)) < 1e-7


def test_oracle_ties_nan_and_short_vocabulary():
    row = np.array([-INF, NAN, 2.0, 2.0, -0.0, 0.0], dtype=np.float32)
    lp, ids, lps = O.report(row, 1, 8)
    # 2.0 twice, then -0 == +0 (lower index first), then -inf and NaN (= -inf) by index, then past V
    assert ids.tolist() == [2, 3, 4, 5, 0, 1, -1, -1]
    S = 2 + 2 * math.exp(-2.0)
    np.testing.assert_allclose(lps[:4], [-math.log(S)] * 2 + [-2 - math.log(S)] * 2, rtol=0, atol=1e-12)
    assert lps[4:].tolist() == [-INF] * 4
    assert lp == -INF                                                  # NaN logit = -inf
    _, ids, _ = O.report(row, 2, 0)
    assert ids.size == 0


def test_oracle_special_rows():
    row = np.array([1.0, INF, -INF, INF, NAN], dtype=np.float32)
    lp, ids, lps = O.report(row, 3, 3)
    assert ids.tolist() == [1, 3, 0] and lps.tolist() == [-math.log(2), -math.log(2), -INF]
    assert lp == -math.log(2)
    assert O.report(row, 0, 1)[0] == -INF
    dead = np.array([-INF, NAN, -INF], dtype=np.float32)
    lp, ids, lps = O.report(dead, 1, 5)
    assert math.isnan(lp) and ids.tolist() == [0, 1, 2, -1, -1]
    assert all(math.isnan(v) for v in lps[:3]) and lps[3:].tolist() == [-INF, -INF]
    assert math.isnan(O.report(row, 5, 1)[0]) and math.isnan(O.report(row, -1, 1)[0])    # token outside [0, V)


def test_oracle_store_rule():
    r = [np.array([0.0, float(k)], dtype=np.float32) for k in range(5)]
    trace = [(r[0], 1, 0, 1), (r[1], 0, 1, 1), (r[2], 0, 0, 2), (r[3], 1, -1, 2), (r[4], 1, 0, 3)]
    lp, ids, _ = O.store(trace, 2, 1)                                # the third id falls past max_ids = 2
    assert lp[0] == O.report(r[0], 1, 1)[0] and lp[1] == O.report(r[2], 0, 1)[0]
    assert ids[:, 0].tolist() == [0, 1]                               # [0, 0]: the tie goes to 0; [0, 2]: 1


def test_bound_is_below_two_to_minus_twenty_for_practical_logprobs():
    for x in (0.0, -1e-3, -3.0, -20.0, -1e4, -2.0 ** 29):
        assert O.bound(x) - 0.5 * O.ulp32(x) <= 2.0 ** -20


# ---------------------------------------------------------------- the checkers reject emulated bugs
SLICES = 8


def emulate(row, token, n, bug=None):
    """A numpy kernel: the contract evaluated in fp64 and rounded to fp32, with one bug switched on."""
    r = O.clean(row)
    V = r.size
    m = r.max()
    terms = np.exp(r - m)
    if bug == "drop_last_slice":
        S = (V + SLICES - 1) // SLICES
        terms = terms[:(SLICES - 1) * S]
    lnS = math.log(float(terms.sum()))
    f = lambda v: np.float32((float(v) - m) - lnS)                     # noqa: E731
    key = r.copy()
    if bug == "nan_above_neg_inf":
        key[np.isnan(np.asarray(row, dtype=np.float32))] = -1e300
    idx = np.arange(V)
    order = np.lexsort((-idx, -key)) if bug == "ties_high" else np.lexsort((idx, -key))
    order = order[:n]
    t = int(np.argmax(r)) if bug == "argmax_for_forced" else token
    return f(r[t]), order, np.array([f(r[i]) for i in order])


def _rows():
    rng = np.random.default_rng(3)
    row = (rng.standard_normal(1000) * 2).astype(np.float32)
    row[[10, 500, 990]] = row.max() + 1.0                              # a three-way tie at the top, across slices
    row[[20, 21]] = NAN
    row[[30]] = -INF
    return row


def test_emulated_kernel_without_bugs_passes():
    row = _rows()
    for tok in (10, 5, 20, 999):
        lp, ids, lps = emulate(row, tok, 20)
        assert O.check_report(lp, ids, lps, row, tok, 20) <= 1.0


@pytest.mark.parametrize("bug,tok,n", [("drop_last_slice", 5, 5), ("ties_high", 10, 5), ("argmax_for_forced", 7, 1)])
def test_checker_rejects_row_bugs(bug, tok, n):
    row = _rows()
    lp, ids, lps = emulate(row, tok, n, bug)
    with pytest.raises(AssertionError):
        O.check_report(lp, ids, lps, row, tok, n)


def test_checker_rejects_nan_ranked_above_neg_inf():
    row = np.array([-INF, NAN, 1.0, -INF], dtype=np.float32)
    lp, ids, lps = emulate(row, 2, 4, "nan_above_neg_inf")
    assert ids.tolist() == [2, 1, 0, 3]
    with pytest.raises(AssertionError):
        O.check_report(lp, ids, lps, row, 2, 4)
    lp, ids, lps = emulate(row, 2, 4)
    O.check_report(lp, ids, lps, row, 2, 4)


def _trace():
    rng = np.random.default_rng(9)
    rows = [(rng.standard_normal(64) * 3).astype(np.float32) for _ in range(6)]
    # (row, chosen token, append_kind, n_ids after the step): text, <image_start>, two image steps, <image_end>, text
    kinds = [0, 0, 1, 1, 0, 0]
    trace, n_ids = [], 0
    for row, kind in zip(rows, kinds):
        n_ids += kind == 0
        trace.append((row, int(np.argmax(row)), kind, n_ids))
    return trace


def _store_like_kernel(trace, max_ids, n, bug=None):
    lp = np.full(max_ids, np.float32(NAN))
    ids = np.full((max_ids, n), -2)
    lps = np.full((max_ids, n), np.float32(NAN))
    for row, tok, kind, n_ids in trace:
        slot = n_ids if bug == "slot_n_ids" else n_ids - 1
        if (kind != 0 and bug != "image_step") or not 0 <= slot < max_ids:
            continue
        lp[slot], ids[slot], lps[slot] = emulate(row, tok, n)
    return lp, ids, lps


def test_store_checker_accepts_the_rule_and_rejects_emulated_bugs():
    trace = _trace()
    O.check_stored(*_store_like_kernel(trace, 8, 3), trace, 8, 3, poison_id=-2)
    O.check_stored(*_store_like_kernel(trace, 3, 3), trace, 3, 3, poison_id=-2)      # ids past max_ids: not stored
    for bug in ("slot_n_ids", "image_step"):
        with pytest.raises(AssertionError):
            O.check_stored(*_store_like_kernel(trace, 8, 3, bug), trace, 8, 3, poison_id=-2)
