"""The decode sampler (csrc/sampling.cu) on the H100 at its slice and value edges, against the fp64 restatement in
oracle/sampling.py at the vocabulary under test.

A row is split over 8 CTAs in slices of S = ceil4(ceil(V / 8)) logits, so the vocabularies here are chosen from that
rule: CTAs with an empty slice, a last slice shorter than a Philox block, one element in the last CTA, and the largest
V the shared-memory budget takes. The kept set is probed by value (ties across the top-k threshold and across two
slices, the extreme k and p, -0 against +0, denormals, NaN at slice boundaries) and the rows without a finite scaled
maximum (+inf logits, a temperature whose reciprocal overflows) are held to the argmax rule of DESIGN.md §1.
Draws the oracle marks too close to call (perturbed-value gap < 1e-4, top-p margin < 1e-6) are skipped and counted.
tests/test_decode_checkers.py shows on the CPU that `check_draws` rejects emulated sampler bugs.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CTAS, MAX_V = 8, 8 * 48 * 1024
PAD = 5                                                    # ld = V + PAD, NaN in the padding
I32_MAX = 2 ** 31 - 1


def slice_len(V):
    return (-(-V // CTAS) + 3) // 4 * 4


def slice_sizes(V):
    S = slice_len(V)
    return [max(0, min(S, V - q * S)) for q in range(CTAS)]


def device_params(R, T, k, p, seed, counter, dev):
    f = lambda v, dt: torch.from_numpy(np.broadcast_to(np.asarray(v, dtype=np.float64), (R,)).copy()).to(dt).to(dev)  # noqa: E731
    seeds = [int(s) - (1 << 64) if int(s) >= 1 << 63 else int(s)
             for s in np.broadcast_to(np.asarray(seed, dtype=object), (R,))]
    return (f(T, torch.float32), f(k, torch.int32), f(p, torch.float32),
            torch.tensor(seeds, dtype=torch.int64, device=dev), f(counter, torch.int32))


def sample(dev, rows, T, k, p, seed, counter):
    """rows [R, V] fp32 (numpy) -> the kernel's tokens, drawn from a buffer with ld = V + PAD and NaN padding."""
    from metamorph_b200 import ops
    rows = np.asarray(rows, dtype=np.float32)
    R, V = rows.shape
    buf = torch.full((R, V + PAD), float("nan"), dtype=torch.float32)
    buf[:, :V] = torch.from_numpy(rows)
    out = ops.sample_rows(buf.to(dev), V, *device_params(R, T, k, p, seed, counter, dev))
    return out.cpu().numpy()


def check_draws(got, rows, T, k, p, seed, counter, what, max_skipped=0.02):
    """Every token equals the oracle's draw, except where the oracle says the row is too close to call. Returns
    (checked, skipped) and bounds the skipped share."""
    from oracle.sampling import draw
    rows = np.asarray(rows, dtype=np.float32)
    R = rows.shape[0]
    b = lambda v: np.broadcast_to(np.asarray(v, dtype=object), (R,))                                    # noqa: E731
    T, k, p, seed, counter = b(T), b(k), b(p), b(seed), b(counter)
    skipped = 0
    for i in range(R):
        tok, gap, margin = draw(rows[i], np.float32(T[i]), int(k[i]), float(np.float32(p[i])), int(seed[i]),
                                int(counter[i]))
        if gap < 1e-4 or margin < 1e-6:
            skipped += 1
            continue
        assert int(got[i]) == tok, f"{what}: row {i} (T={T[i]}, k={k[i]}, p={p[i]}, seed={seed[i]}, " \
                                   f"counter={counter[i]}): kernel {int(got[i])}, oracle {tok}"
    assert skipped <= max_skipped * R + 1, f"{what}: {skipped} of {R} draws too close to call"
    print(f"draws: {what}: {R - skipped} checked, {skipped} too close to call")
    return R - skipped, skipped


def _mixes(rng, R, V):
    T = rng.uniform(0.4, 1.6, R).astype(np.float32)
    k = np.where(np.arange(R) % 4 % 2 == 1, rng.integers(1, max(2, min(V, 300)), R), 0)
    p = np.where(np.arange(R) % 4 >= 2, rng.uniform(0.05, 0.97, R), 1.0).astype(np.float32)
    seed = [int(s) for s in rng.integers(0, 1 << 64, R, dtype=np.uint64)]
    counter = rng.integers(0, 5000, R)
    return T, k, p, seed, counter


# ------------------------------------------------------------------------------------------------ vocabulary
VOCABS = {
    1: "seven empty slices", 3: "seven empty slices, a slice shorter than a Philox block", 4: "seven empty slices",
    5: "six empty slices, one element in the second", 8: "six empty slices", 9: "one element in the third slice",
    31: "a last slice of 3", 32: "every slice one Philox block", 33: "four empty slices, one element in the fifth",
    57: "one element in the last CTA", 225: "one element in the last CTA",
    2047: "a last slice of 255", 2048: "every slice full", 2049: "a last slice of 229",
    MAX_V: "the shared-memory budget, every slice full",
}


@pytest.mark.parametrize("V", list(VOCABS))
def test_vocabulary_edges(cuda_device, V):
    n = slice_sizes(V)
    assert sum(n) == V
    if V in (1, 3, 4):
        assert n[1:] == [0] * 7
    if V in (5, 9, 33):
        assert 1 in n and n[-1] == 0
    if V in (57, 225):
        assert n[-1] == 1
    if V in (3, 31, 2047, 2049):
        assert any(x % 4 for x in n)
    if V in (32, 2048, MAX_V):
        assert all(x == slice_len(V) for x in n) and (V != MAX_V or n[0] == 48 * 1024)
    rng = np.random.default_rng(V)
    R = 16 if V == MAX_V else 64
    rows = (rng.standard_normal((R, V)) * 2).astype(np.float32)
    if V >= 64:                                             # LLM-like: a few tokens well above a broad background
        for r in range(R):
            rows[r, rng.choice(V, 20, replace=False)] += 8 + rng.random(20).astype(np.float32) * 4
    mix = _mixes(rng, R, V)
    check_draws(sample(cuda_device, rows, *mix), rows, *mix, f"V={V} ({VOCABS[V]})", max_skipped=0.05)


def test_a_vocabulary_above_the_budget_is_rejected_before_any_launch(cuda_device):
    from metamorph_b200 import ops
    from metamorph_b200._lib import MetaMorphB200Error
    V = MAX_V + 1
    buf = torch.zeros((1, V + 7), dtype=torch.float32, device=cuda_device)
    out = torch.full((1,), -77, dtype=torch.int32, device=cuda_device)
    with pytest.raises(MetaMorphB200Error, match="shared-memory budget"):
        ops.sample_rows(buf, V, *device_params(1, 1.0, 0, 1.0, 0, 0, cuda_device), out=out)
    torch.cuda.synchronize()
    assert int(out[0]) == -77


# ------------------------------------------------------------------------------------------------ the kept set
def _seeds(R, base=0):
    return [base + i for i in range(R)]


def test_ties_across_the_top_k_threshold_and_two_slices_are_all_kept(cuda_device):
    from oracle.sampling import warped_probs
    V, R = 64, 3000                                          # S = 8: tokens 7 and 8 sit in different CTAs
    assert slice_len(V) == 8
    row = np.full(V, -4.0, dtype=np.float32)
    row[40] = 5.0
    row[[7, 8, 23, 63]] = 3.0                                 # four exact ties at the k = 2 threshold
    rows = np.broadcast_to(row, (R, V))
    got = sample(cuda_device, rows, 1.0, 2, 1.0, _seeds(R), 3)
    check_draws(got, rows, 1.0, 2, 1.0, _seeds(R), 3, "top-k ties")
    kept = np.flatnonzero(warped_probs(row, np.float32(1.0), 2, 1.0) > 0)
    assert kept.tolist() == [7, 8, 23, 40, 63]
    assert sorted(set(got.tolist())) == kept.tolist(), "a tied token was dropped, or one outside the kept set drawn"
    # the tie frequencies follow the warped softmax: each 3.0 has e^-2 of the mass of the 5.0
    from scipy.stats import chisquare
    probs = warped_probs(row, np.float32(1.0), 2, 1.0)[kept]
    assert chisquare([(got == t).sum() for t in kept], probs * R).pvalue > 1e-4


@pytest.mark.parametrize("V", [9, 2049])
def test_top_k_extremes(cuda_device, V):
    rng = np.random.default_rng(V + 1)
    R = 400
    rows = (rng.standard_normal((R, V)) * 1.5).astype(np.float32)
    ks = np.asarray([1, V - 1, V, V + 1, I32_MAX])[np.arange(R) % 5]
    got = sample(cuda_device, rows, 1.0, ks, 1.0, _seeds(R, 10), 1)
    check_draws(got, rows, 1.0, ks, 1.0, _seeds(R, 10), 1, f"top-k extremes V={V}")
    assert np.array_equal(got[ks == 1], rows[ks == 1].argmax(1)), "top_k = 1 with a single maximum is the argmax"
    # k >= V is top-k off; V - 1 drops exactly the minimum
    off = sample(cuda_device, rows, 1.0, 0, 1.0, _seeds(R, 10), 1)
    assert np.array_equal(got[ks >= V], off[ks >= V])
    assert not (got[ks == V - 1] == rows[ks == V - 1].argmin(1)).any()


def test_top_p_extremes(cuda_device):
    rng = np.random.default_rng(11)
    V, R = 2049, 400
    rows = (rng.standard_normal((R, V)) * 1.5).astype(np.float32)
    tiny, under_one = float(np.float32(1e-45)), float(np.nextafter(np.float32(1), np.float32(0)))
    assert tiny > 0 and under_one < 1
    for p in (0.0, tiny):                                   # only the maximum survives, whatever the seed
        got = sample(cuda_device, rows, 0.9, 0, p, _seeds(R, 20), 2)
        assert np.array_equal(got, rows.argmax(1)), f"top_p = {p}"
    off = sample(cuda_device, rows, 0.9, 0, 1.0, _seeds(R, 20), 2)
    check_draws(off, rows, 0.9, 0, 1.0, _seeds(R, 20), 2, "top_p = 1")
    # just under 1 drops at most a tail of 2^-24 of the mass (too near the boundary for the fp64 oracle to call)
    got = sample(cuda_device, rows, 0.9, 0, under_one, _seeds(R, 20), 2)
    assert (got != off).sum() <= 0.01 * R


def test_top_p_on_either_side_of_a_cumulative_mass(cuda_device):
    """Masses 1, e^-1, e^-2 ...: p a relative 1e-5 below / above the mass of the first two tokens keeps two / three.
    (At exact equality the fixed-point masses and the fp64 oracle may round differently, so neither side is claimed.)"""
    from oracle.sampling import warped_probs
    V, R = 33, 1500
    row = -np.arange(V, dtype=np.float32)
    rows = np.broadcast_to(row, (R, V))
    mass = np.exp(-np.arange(V, dtype=np.float64))
    boundary = mass[:2].sum() / mass.sum()
    for p, n_kept in ((np.float32(boundary * (1 - 1e-5)), 2), (np.float32(boundary * (1 + 1e-5)), 3)):
        assert (warped_probs(row, np.float32(1.0), 0, float(p)) > 0).sum() == n_kept
        got = sample(cuda_device, rows, 1.0, 0, p, _seeds(R, 30), 4)
        check_draws(got, rows, 1.0, 0, p, _seeds(R, 30), 4, f"top_p {'below' if n_kept == 2 else 'above'} the boundary")
        assert sorted(set(got.tolist())) == list(range(n_kept))


def test_tied_maxima_under_top_k_1_and_top_p_0_follow_the_contract(cuda_device):
    """Ties are kept by value: with several maxima, k = 1 and p = 0 keep all of them and the draw picks among them."""
    V, R = 225, 600
    row = np.zeros(V, dtype=np.float32)
    row[[3, 28, 224]] = 2.0                                  # three maxima, the last one alone in the last CTA
    rows = np.broadcast_to(row, (R, V))
    for k, p in ((1, 1.0), (0, 0.0), (1, 0.0)):
        got = sample(cuda_device, rows, 0.7, k, p, _seeds(R, 40), 0)
        check_draws(got, rows, 0.7, k, p, _seeds(R, 40), 0, f"tied maxima k={k} p={p}")
        assert sorted(set(got.tolist())) == [3, 28, 224]
        assert min((got == t).sum() for t in (3, 28, 224)) > R / 5


# ------------------------------------------------------------------------------------------------ values
def test_negative_zero_ties_positive_zero(cuda_device):
    V, R = 33, 400
    row = np.full(V, -3.0, dtype=np.float32)
    row[2], row[17] = -0.0, 0.0
    assert np.signbit(row[2]) and not np.signbit(row[17])
    rows = np.broadcast_to(row, (R, V))
    for T in (1.0, 0.5):
        got = sample(cuda_device, rows, T, 1, 1.0, _seeds(R, 50), 0)
        check_draws(got, rows, T, 1, 1.0, _seeds(R, 50), 0, f"-0 against +0 at T={T}")
        assert sorted(set(got.tolist())) == [2, 17] and min((got == 2).sum(), (got == 17).sum()) > R / 3


def test_denormal_logits_and_a_lone_peak(cuda_device):
    rng = np.random.default_rng(13)
    V, R = 2047, 300
    rows = (rng.standard_normal((R, V)) * 1e-40).astype(np.float32)
    assert (np.abs(rows[rows != 0]) < np.finfo(np.float32).tiny).all() and len(np.unique(rows[0])) > V // 2
    ks = np.asarray([0, 7, 301])[np.arange(R) % 3]           # equal masses: keep 0.9 k off an integer
    for T in (1.0, 0.25):
        got = sample(cuda_device, rows, T, ks, 0.9, _seeds(R, 60), 6)
        check_draws(got, rows, T, ks, 0.9, _seeds(R, 60), 6, f"denormal logits at T={T}", max_skipped=0.1)
    # a maximum so far above the rest that every other mass rounds to 0 in the 2^-40 fixed point
    rows = (rng.standard_normal((R, V))).astype(np.float32)
    peak = rng.integers(0, V, R)
    rows[np.arange(R), peak] = 100.0
    assert np.exp(np.float64(rows[0, peak[0] - 1]) - 100.0) * 2.0 ** 40 < 0.5
    for k, p in ((0, 1.0), (0, 0.9), (5, 0.999)):
        got = sample(cuda_device, rows, 1.0, k, p, _seeds(R, 70), 6)
        check_draws(got, rows, 1.0, k, p, _seeds(R, 70), 6, f"lone peak k={k} p={p}")
        assert np.array_equal(got, peak)


def test_nan_at_slice_boundaries_and_a_single_live_element(cuda_device):
    rng = np.random.default_rng(17)
    V, R = 2049, 300
    S = slice_len(V)
    rows = (rng.standard_normal((R, V)) * 2).astype(np.float32)
    edges = [q * S + d for q in range(1, CTAS) for d in (-1, 0) if q * S + d < V] + [0, V - 1]
    rows[:, edges] = np.nan
    mix = _mixes(rng, R, V)
    got = sample(cuda_device, rows, *mix)
    check_draws(got, rows, *mix, "NaN at slice boundaries", max_skipped=0.05)
    assert not np.isin(got, edges).any()
    # -inf everywhere but one element: that element, for every parameter mix
    rows = np.full((R, V), -np.inf, dtype=np.float32)
    live = rng.integers(0, V, R)
    live[:3] = (0, V - 1, 7 * S)
    rows[np.arange(R), live] = rng.standard_normal(R).astype(np.float32)
    got = sample(cuda_device, rows, *mix)
    assert np.array_equal(got, live)
    check_draws(got, rows, *mix, "one live element")


# ------------------------------------------------------------------------------------------------ max z = +-inf
def test_rows_without_a_finite_scaled_maximum_return_the_argmax(cuda_device):
    """A +inf logit, several of them, and temperatures so small that max l / T overflows fp32 (to +inf for a positive
    maximum, to -inf for a negative one): the argmax of the logits, lowest index among the maxima, for every k, p and
    seed. The overflow rows are built so that the lowest index whose quotient overflows is NOT the argmax."""
    rng = np.random.default_rng(19)
    V = 2049
    S = slice_len(V)
    inf = np.float32(np.inf)
    cases = []
    base = (rng.standard_normal(V) * 2).astype(np.float32)
    a = base.copy(); a[1500] = inf; cases.append(("one +inf", a, 1.0, 1500))
    a = base.copy(); a[[1999, S, S - 1, 40]] = inf; cases.append(("several +inf", a, 0.8, 40))
    a = base.copy(); a[7] = np.nan; a[9] = inf; a[3] = -inf; cases.append(("+inf beside NaN and -inf", a, 1.3, 9))
    a = np.abs(base) + 1; a[5] = 50.0; a[1200] = 60.0
    cases.append(("T = 1e-39, every quotient overflows", a, 1e-39, 1200))
    a = np.abs(base) + 1; a[1200] = 60.0
    cases.append(("T = 1e-45", a, 1e-45, 1200))
    a = base.copy() * 1e30; a[2] = 3e38; a[2048] = 3.3e38
    cases.append(("T = 0.5, only the largest logits overflow", a, 0.5, 2048))
    a = -np.abs(base) - 1; a[800] = -0.5
    cases.append(("T = 1e-39, negative maximum: max z = -inf", a, 1e-39, 800))
    for what, row, T, want in cases:
        with np.errstate(over="ignore", divide="ignore"):
            zmax = np.float32(np.nanmax(row)) / np.float32(T)
        assert np.isinf(zmax), f"{what}: max z = {zmax} is finite"
        R = 30
        rows = np.broadcast_to(row, (R, V))
        ks = np.asarray([0, 1, 5, V])[np.arange(R) % 4]
        ps = np.asarray([1.0, 0.5, 0.0], dtype=np.float32)[np.arange(R) % 3]
        got = sample(cuda_device, rows, T, ks, ps, _seeds(R, 80), np.arange(R))
        assert (got == want).all(), f"{what}: drew {sorted(set(got.tolist()))}, the argmax is {want}"
        check_draws(got, rows, T, ks, ps, _seeds(R, 80), np.arange(R), what)


# ------------------------------------------------------------------------------------------------ counter and seed
def test_counter_and_seed_extremes_in_the_last_philox_block(cuda_device):
    """Only the four elements of the last Philox block of the largest V are live and they tie, so the token is decided
    by words 0..3 of block V / 4 - 1 alone. Seeds travel through SamplingArrays: 2^63 and 2^64 - 1 wrap to negative."""
    from metamorph_b200 import ops
    from metamorph_b200.engine.sampling import SamplingArrays, SamplingParams
    V = MAX_V
    pairs = [(s, c) for s in (0, 1 << 63, (1 << 64) - 1, 12345) for c in (0, I32_MAX)] * 4
    seeds, counters = [s for s, _ in pairs], [c for _, c in pairs]
    R = len(pairs)
    row = np.full(V, -np.inf, dtype=np.float32)
    row[V - 4:] = 1.0
    arrs = SamplingArrays.of([SamplingParams(temperature=1.0, top_k=0, top_p=1.0, seed=s) for s in seeds], cuda_device)
    assert arrs.seed.cpu().tolist()[:6:2] == [0, -(1 << 63), -1]
    one = SamplingArrays(1, cuda_device)
    one.set(0, SamplingParams(temperature=1.0, seed=(1 << 64) - 1))
    assert int(one.seed[0]) == -1
    buf = torch.from_numpy(row).to(cuda_device).expand(R, V).contiguous()
    counter = torch.tensor(counters, dtype=torch.int32, device=cuda_device)
    got = ops.sample_rows(buf, V, arrs.temperature, arrs.top_k, arrs.top_p, arrs.seed, counter).cpu().numpy()
    rows = np.broadcast_to(row, (R, V))
    check_draws(got, rows, 1.0, 0, 1.0, seeds, counters, "last Philox block", max_skipped=0.1)
    assert got.min() >= V - 4 and len(set(zip(seeds, counters, got.tolist()))) == 8
    assert len(set(got.tolist())) >= 2, "eight (seed, counter) pairs all drew the same word"


@pytest.mark.parametrize("R", [1, 2, 129])
def test_rows_are_independent(cuda_device, R):
    rng = np.random.default_rng(R)
    V = 2049
    rows = (rng.standard_normal((R, V)) * 2).astype(np.float32)
    mix = _mixes(rng, R, V)
    together = sample(cuda_device, rows, *mix)
    for r in range(R):
        alone = sample(cuda_device, rows[r:r + 1], *(np.asarray(m, dtype=object)[r:r + 1] for m in mix))
        assert int(alone[0]) == int(together[r]), f"row {r} of {R}"
    check_draws(together, rows, *mix, f"{R} rows together", max_skipped=0.05)
