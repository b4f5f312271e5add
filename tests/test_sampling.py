"""CPU tests of the decode sampler's host side: SamplingParams validation and seeding, the numpy Philox4x32-10 and
fp64 kept-set restatement (oracle/sampling.py) against known answers and HF's warpers, and the C ABI's argument checks."""
import numpy as np
import pytest
import torch


def test_sampling_params_validation():
    from metamorph_b200.engine.sampling import SamplingParams
    for bad in (dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")),
                dict(top_k=-1), dict(top_k=2.5), dict(top_p=-0.01), dict(top_p=1.01), dict(top_p=float("nan")),
                dict(seed=-1), dict(seed=1 << 64)):
        with pytest.raises(ValueError):
            SamplingParams(**bad)
    sp = SamplingParams(temperature=0.7, top_k=5, top_p=0.9, seed=(1 << 64) - 1)
    assert (sp.temperature, sp.top_k, sp.top_p, sp.seed) == (0.7, 5, 0.9, (1 << 64) - 1)
    assert SamplingParams().greedy and not sp.greedy
    assert SamplingParams(top_p=0.0).top_p == 0.0 and SamplingParams(top_p=1.0).top_p == 1.0


def test_seed_comes_from_torch_manual_seed():
    from metamorph_b200.engine.sampling import SamplingParams
    torch.manual_seed(1234)
    a = [SamplingParams(temperature=1.0).seed for _ in range(3)]
    torch.manual_seed(1234)
    b = [SamplingParams(temperature=1.0).seed for _ in range(3)]
    assert a == b and len(set(a)) == 3 and all(0 <= s < 1 << 63 for s in a)


def test_per_sequence_seeds_and_greedy_shortcut():
    from metamorph_b200.engine.sampling import SamplingParams, per_sequence
    assert per_sequence(None, 4) is None
    assert per_sequence(SamplingParams(temperature=0.0, seed=3), 4) is None          # all greedy: the argmax path
    ps = per_sequence(SamplingParams(temperature=1.0, top_k=3, seed=(1 << 64) - 2), 4)
    assert [p.seed for p in ps] == [(1 << 64) - 2, (1 << 64) - 1, 0, 1]
    assert all(p.top_k == 3 and p.temperature == 1.0 for p in ps)
    with pytest.raises(ValueError):
        per_sequence([SamplingParams(temperature=1.0)], 2)


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    from oracle.sampling import philox4x32_10
    assert tuple(int(w) for w in philox4x32_10(np.array(ctr), key)) == want


def test_uniform_words_layout():
    """Word i & 3 of the block with counter (i >> 2, c, 0, 0) and key (seed low, seed high)."""
    from oracle.sampling import philox4x32_10, uniform_words
    seed, c = 0x0123456789abcdef, 17
    w = uniform_words(10, seed, c)
    blk = philox4x32_10(np.array([2, c, 0, 0]), (seed & 0xffffffff, seed >> 32))
    assert np.array_equal(w[8:10], blk[:2])


@pytest.mark.parametrize("T,k,p", [(0.7, 0, 1.0), (1.0, 5, 1.0), (1.3, 0, 0.9), (1.0, 40, 0.5), (0.5, 0, 0.3),
                                   (2.0, 100, 0.95)])
def test_oracle_kept_set_equals_hf_warpers(T, k, p):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    from oracle.sampling import kept_set, scaled
    rng = np.random.default_rng(7)
    checked = 0
    for _ in range(20):
        row = (rng.standard_normal(1000) * 3).astype(np.float32)
        scores = torch.from_numpy(row.copy())[None]
        for w in [TemperatureLogitsWarper(T)] + ([TopKLogitsWarper(k)] if k else []) + \
                 ([TopPLogitsWarper(p)] if p < 1 else []):
            scores = w(None, scores)
        hf = torch.isfinite(scores[0]).numpy()
        keep, margin = kept_set(scaled(row, T), k, p)
        if margin < 1e-5:            # HF decides in fp32: a token this close to the top-p boundary may flip
            continue
        assert np.array_equal(keep, hf)
        checked += 1
    assert checked >= 18


def test_oracle_ties_at_the_boundaries_are_kept():
    from oracle.sampling import kept_set
    z = np.array([3.0, 1.0, 2.0, 2.0, 0.0, 2.0])
    keep, _ = kept_set(z, 2, 1.0)                 # count(z_j > 2) = 1 < 2 for every 2.0
    assert keep.tolist() == [True, False, True, True, False, True]
    keep, _ = kept_set(z, 0, 0.0)                 # p = 0: only the maximum
    assert keep.tolist() == [True, False, False, False, False, False]
    keep, _ = kept_set(z, 0, 0.5)                 # mass above 2.0 = e^0 < 0.5 M: all three 2.0 kept
    assert keep.tolist() == [True, False, True, True, False, True]


def test_sample_rows_rejects_bad_arguments_without_gpu():
    from ctypes import c_int, c_void_p
    from metamorph_b200 import _build
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    _build.build(verbose=False)
    a = c_void_p(256)    # never dereferenced: the argument checks reject the call first
    args = lambda ld, R, V: (a, ll(ld), ll(R), c_int(V), a, a, a, a, a, a, c_void_p(0))  # noqa: E731
    with pytest.raises(MetaMorphB200Error, match="bad shape"):
        call("mm_sample_rows", *args(100, 4, 128))          # ld < V
    with pytest.raises(MetaMorphB200Error, match="bad shape"):
        call("mm_sample_rows", *args(128, 0, 128))
    with pytest.raises(MetaMorphB200Error, match="shared-memory budget"):
        call("mm_sample_rows", *args(400000, 1, 393217))    # one element past 8 x 48K fp32 per CTA
