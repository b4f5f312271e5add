"""The decode control-path references have teeth, and the restatement itself is pinned (CPU only).

Hand-written traces hold oracle/decode_state.py to the reference loop body (metamorph_llama.py:547-582), the two quirk
shapes of tests/golden/greedy_decode_quirks.pt included, and to oracle/restatement.py::greedy_decode_nocache where the
two overlap. Then each test emulates in Python one bug of `decode_state_kernel` or of the sampler that
tests/test_decode_state_gpu.py and tests/test_sampling_edges_gpu.py exist to catch, and requires the same comparison
to reject it; the clean emulation must pass. The host-side rejections of forced ids and the temperature rule are here
too. Nothing here builds or runs a kernel.
"""
import types

import numpy as np
import pytest
import torch

from oracle.decode_state import HIDDEN as H_, TOKEN as T_, DecodeConfig, DecodeState, run, run_forced, step
from tests.test_decode_state_gpu import (ALPHABET, END, EOS0, EOS1, GUARD_BITS, START, _pattern, assert_state_equal,
                                         eos_pair, expected_arrays, expected_img_bits, reachable_regimes, stream_tree)
from tests.test_sampling_edges_gpu import check_draws, slice_len

S, E, X = 128256, 128257, 128009


# ------------------------------------------------------------------------------------------------ the restatement
def test_q1_eos_inside_an_image_ends_the_run_mid_block():
    s = run([S, 5, X, 6, 7], DecodeConfig(4, 12, S, E, (X,)))
    assert s.broke and s.total_output == 3 and s.ids == [S]                 # the EOS token itself is never emitted
    assert s.kept_steps == [1, 2] and s.appended == [T_, H_, H_]              # ... but its step's embedding is kept
    assert s.in_image_mode and s.total_image_tokens == 2


def test_q2_second_start_without_end_is_text_in_image_mode():
    cfg = DecodeConfig(2, 9, S, E, ())
    s = run([S, 1, 2, S, 3, 4, E, 5, S, 6], cfg)
    assert s.ids == [S, S, 3, 4, E, 5, S] and s.kept_steps == [1, 2, 9]
    assert s.appended == [T_, H_, H_, T_, T_, T_, T_, T_, T_, H_]
    assert s.broke and s.total_output == 10 and s.in_image_mode and s.total_image_tokens == 1
    mid = run([S, 1, 2, S, 3], cfg)                                            # counter still full, mode set again
    assert mid.in_image_mode and mid.total_image_tokens == 2 and not mid.broke


def test_zero_image_tokens_only_end_leaves_image_mode():
    s = run([S, 4, S, X, E, 4], DecodeConfig(0, 20, S, E, ()))
    assert s.ids == [S, 4, S, X, E, 4] and s.kept_steps == [] and not s.in_image_mode
    assert run([S, 4, S], DecodeConfig(0, 20, S, E, ())).in_image_mode


def test_limit_schedule_and_empty_eos():
    assert run([1, 2, 3], DecodeConfig(4, 0, S, E, (X,))).tokens == [1]       # `>`: max_new_tokens + 1 steps
    assert run([1, 2, 3, 4], DecodeConfig(4, 2, S, E, (X,))).tokens == [1, 2, 3]
    assert run([1, X, 3], DecodeConfig(4, 9, S, E, ())).tokens == [1, X, 3]   # an empty EOS list never matches
    s = run([1, 2, 3, 4, 5], DecodeConfig(4, 9, S, E, (X,)), forced=[9, -1, 8])
    assert s.tokens == [9, 2, 8, 4, 5]                                         # a hole, then the schedule ends
    assert run_forced([S, 1, X, 3], DecodeConfig(1, 3, S, E, (X,))).ids == [S, X]
    with pytest.raises(AssertionError):
        step(run([X], DecodeConfig(1, 3, S, E, (X,))), 1, DecodeConfig(1, 3, S, E, (X,)))


def test_agrees_with_the_whole_model_restatement_where_they_overlap():
    from oracle import restatement as R
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    W, live = with_sparse_lm_head(make_weights(TINY), 16)
    cfg = dict(TINY, image_tokens=2)
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(0, 128000, (6,), generator=g)
    emb = W["model.embed_tokens.weight"][prompt].float()[None]
    trace = []
    R.greedy_decode_nocache(W, cfg, emb, 9, start_id=-1, end_id=-2, eos=(), trace=trace)
    toks = [t["tok"] for t in trace]
    start, eos = toks[1], toks[-2]                   # ids the free run is known to emit play <image_start> and EOS
    trace = []
    ids, imgs = R.greedy_decode_nocache(W, cfg, emb, 9, start_id=start, end_id=-2, eos=(eos,), trace=trace)
    s = run([t["tok"] for t in trace], DecodeConfig(2, 9, start, -2, (eos,)))
    assert s.ids == ids and len(s.kept_steps) == imgs.shape[0] and s.total_output == len(trace)
    assert len(s.kept_steps) >= 1


# ------------------------------------------------------------------------------------------------ emulated kernel bugs
def _emu_launch(seqs, free, forced, forced_ld, cfg, max_ids, bug):
    """`decode_state_kernel` in Python over per-sequence dicts, with one bug switched on. Returns the img_out slot each
    sequence stored to (or None)."""
    e0, e1 = eos_pair(list(cfg.eos))
    slots = []
    for b, a in enumerate(seqs):
        kind, slot = -1, None
        if not a["finished"]:
            fidx = a["total_output"]
            if bug == "repeated_last_forced_token":
                fidx = min(fidx, forced_ld - 1)
            ftok = forced[b][fidx] if forced is not None and fidx < forced_ld else -1
            tok = ftok if ftok >= 0 else int(free[b])
            mode = a["in_image_mode"]
            if not mode and tok == cfg.start_id:
                a["in_image_mode"] = 1; a["ids"].append(tok); kind = 0
            elif mode and a["total_image_tokens"] < cfg.num_image_tokens:
                a["total_image_tokens"] += 1
                slot = a["n_img"] + (1 if bug == "img_slot_after_increment" else 0)
                a["n_img"] += 1
                kind = 1
                if a["total_image_tokens"] == cfg.num_image_tokens:
                    a["in_image_mode"] = 0
                    if bug == "counter_reset_when_block_completes":
                        a["total_image_tokens"] = 0
            elif tok == cfg.end_id:
                a["in_image_mode"] = 0; a["total_image_tokens"] = 0; a["ids"].append(tok); kind = 0
            else:
                a["ids"].append(tok); kind = 0
            a["total_output"] += 1
            a["next_token"] = tok
            over = a["total_output"] >= cfg.max_new_tokens if bug == "ge_at_the_limit" else \
                a["total_output"] > cfg.max_new_tokens
            if (tok == e0 or tok == e1) and not (bug == "eos_skipped_in_image_mode" and kind == 1):
                a["finished"] = 1
            elif over:
                a["finished"] = 1
            a["pos"] += 1
        elif bug == "finished_does_not_freeze_pos":
            a["pos"] += 1
        a["append_kind"] = kind
        slots.append(slot)
    return slots


def _emu_arrays(seqs, max_ids):
    out = {k: np.asarray([a[k] for a in seqs], dtype=np.int32) for k in
           ("in_image_mode", "total_image_tokens", "total_output", "finished", "pos", "n_img", "append_kind",
            "next_token")}
    out["n_ids"] = np.asarray([len(a["ids"]) for a in seqs], dtype=np.int32)
    ids = np.full((len(seqs), max_ids), -1, dtype=np.int32)
    for b, a in enumerate(seqs):
        ids[b, :min(len(a["ids"]), max_ids)] = a["ids"][:max_ids]
    out["ids_out"] = ids
    return out


def _compare(bug, cfg, free, forced=None, C=9, max_img=8):
    """The loop of the GPU tests with the emulation in the kernel's place: oracle and emulation side by side, all ten
    arrays after every step, then img_out."""
    B, L = free.shape
    max_ids, pad = L + 1, 5
    seqs = [dict(in_image_mode=0, total_image_tokens=0, total_output=0, finished=0, pos=3, n_img=0, append_kind=0,
                 next_token=0, ids=[]) for _ in range(B)]
    states = [DecodeState() for _ in range(B)]
    img = np.full(B * max_img * C + pad, GUARD_BITS, dtype=np.int16)
    rows = [list(map(int, r)) for r in forced] if forced is not None else None
    for l in range(L):
        nodes = []
        for b, s in enumerate(states):
            live = not s.broke
            if live:
                step(s, int(free[b, l]), cfg, rows[b] if rows else None)
            nodes.append((s, live))
        slots = _emu_launch(seqs, free[:, l], rows, forced.shape[1] if forced is not None else 0, cfg, max_ids, bug)
        for b, slot in enumerate(slots):
            if slot is not None and slot < max_img:
                img[(b * max_img + slot) * C:(b * max_img + slot + 1) * C] = _pattern(l, b, C)
        assert_state_equal(_emu_arrays(seqs, max_ids), expected_arrays(nodes, np.full(B, 3), max_ids), f"step {l}")
    want, _ = expected_img_bits(states, max_img, C, pad)
    assert np.array_equal(img, want), "img_out differs"


def _all_streams(L):
    letters = np.asarray(ALPHABET, dtype=np.int32)
    n = len(letters)
    idx = np.arange(n ** L)
    return np.stack([letters[(idx // n ** (L - 1 - l)) % n] for l in range(L)], 1)


BUGS = {
    "counter_reset_when_block_completes": "total_image_tokens",
    "eos_skipped_in_image_mode": "finished",
    "ge_at_the_limit": "finished",
    "repeated_last_forced_token": "differs",
    "finished_does_not_freeze_pos": "pos",
    "img_slot_after_increment": "img_out",
}


@pytest.mark.parametrize("bug", [None] + list(BUGS))
def test_state_comparison_rejects(bug):
    cfg = DecodeConfig(2, 4, START, END, (EOS0, EOS1))
    free = _all_streams(5)
    rng = np.random.default_rng(1)
    forced = np.asarray(ALPHABET, dtype=np.int32)[rng.integers(0, 6, (free.shape[0], 3))]
    forced[rng.random(forced.shape) < 0.4] = -1
    if bug is None:
        _compare(None, cfg, free)
        _compare(None, cfg, free, forced)
        return
    with pytest.raises(AssertionError, match=BUGS[bug]):
        _compare(bug, cfg, free, forced if bug == "repeated_last_forced_token" else None)


def test_stream_tree_reaches_what_the_loop_body_allows():
    for k, m, L in ((0, 3, 4), (1, 11, 5), (2, 1, 4), (1, 0, 3)):
        cfg = DecodeConfig(k, m, START, END, (EOS0, EOS1))
        levels, regimes = stream_tree(ALPHABET, L, cfg)
        assert regimes == reachable_regimes(cfg, L), (k, m, L, regimes)
        assert [len(x) for x in levels] == [6 ** l for l in range(L + 1)]
    assert reachable_regimes(DecodeConfig(1, 11, START, END, (EOS0,)), 5) == \
        {"eos_in_image", "second_start", "two_blocks"}
    # a frozen prefix keeps its parent's state object
    levels, _ = stream_tree(ALPHABET, 2, DecodeConfig(1, 5, START, END, (EOS0, EOS1)))
    assert levels[2][2 * 6][0] is levels[1][2][0] and not levels[2][2 * 6][1]


# ------------------------------------------------------------------------------------------------ emulated sampler bugs
def _emu_draw(row, T, k, seed, counter, bug):
    from oracle.sampling import gumbel_noise, kept_set, scaled, uniform_words
    z = scaled(row, T)
    V = z.shape[0]
    keep, _ = kept_set(z, k, 1.0)
    if bug == "top_k_drops_ties":
        keep = np.zeros(V, dtype=bool)
        keep[np.argsort(-z, kind="stable")[:k]] = True
    noise = gumbel_noise(V, seed, counter)
    if bug == "philox_block_from_the_slice_start":
        Sl = slice_len(V)
        w = np.concatenate([uniform_words(Sl, seed, counter)] * 8)[:V]
        noise = -np.log(-np.log((w.astype(np.float64) + 0.5) * 2.0 ** -32))
    return int(np.argmax(np.where(keep, z + noise, -np.inf)))


@pytest.mark.parametrize("bug", [None, "top_k_drops_ties", "philox_block_from_the_slice_start"])
def test_draw_comparison_rejects(bug):
    V, R = 64, 300
    row = np.full(V, -4.0, dtype=np.float32)
    row[40] = 5.0
    row[[7, 8, 23, 63]] = 3.0
    rows = np.broadcast_to(row, (R, V))
    seeds = list(range(R))
    got = np.asarray([_emu_draw(row, np.float32(1.0), 2, s, 3, bug) for s in seeds])
    if bug is None:
        checked, skipped = check_draws(got, rows, 1.0, 2, 1.0, seeds, 3, "clean")
        assert checked + skipped == R and checked > 0.95 * R
        assert sorted(set(got.tolist())) == [7, 8, 23, 40, 63]
        return
    with pytest.raises(AssertionError, match="kernel"):
        check_draws(got, rows, 1.0, 2, 1.0, seeds, 3, bug)


def test_oracle_rule_for_a_scaled_maximum_that_is_not_finite():
    from oracle.sampling import draw
    inf = np.float32(np.inf)
    row = np.asarray([1.0, 2.0, 7.0, 3.0, 7.0], dtype=np.float32)
    for T in (1e-39, 1e-45):                                                    # 7 / T overflows, and so does 1 / T
        assert draw(row, np.float32(T), 0, 1.0, 5, 0)[0] == 2
    assert draw(-row, np.float32(1e-39), 3, 0.5, 5, 0)[0] == 0                  # max z = -inf
    row[[3, 1]] = inf
    assert all(draw(row, np.float32(1.0), k, p, s, 0)[0] == 1 for k in (0, 1, 2) for p in (1.0, 0.3, 0.0)
               for s in range(5))
    assert draw(np.full(4, -inf), np.float32(1.0), 0, 1.0, 0, 0)[0] == 0        # no logit above -inf: still 0
    assert draw(np.asarray([np.nan, -inf], dtype=np.float32), np.float32(1e-39), 0, 1.0, 0, 0)[0] == 0


# ------------------------------------------------------------------------------------------------ host-side rules
def test_sampling_params_accept_any_positive_temperature():
    """A temperature whose reciprocal overflows fp32 is not an error: the row's scaled maximum is then not finite and
    the kernel returns the argmax (the limit T -> 0). One that rounds to 0 in fp32 is greedy on the device."""
    from metamorph_b200.engine.sampling import SamplingArrays, SamplingParams
    for t in (1e-38, 1e-39, 1e-45, 1e-50, 5e-324):
        sp = SamplingParams(temperature=t, seed=1)
        assert sp.temperature == t and not sp.greedy
    a = SamplingArrays.of([SamplingParams(temperature=1e-39, seed=1), SamplingParams(temperature=1e-50, seed=1)], "cpu")
    assert float(a.temperature[0]) > 0 and float(a.temperature[1]) == 0.0


def _fake_model(rows):
    inner = types.SimpleNamespace(embed_tokens=types.SimpleNamespace(weight=torch.empty(rows, 8)))
    return types.SimpleNamespace(get_model=lambda: inner), inner


@pytest.mark.parametrize("bad", [[[5, 10]], [[-2, 3]], [[0, 2 ** 31 - 1]], [[1.0, 2.0]]])
def test_generate_rejects_forced_ids_outside_the_embedding_table_on_the_host(bad):
    """The check runs before the engine touches a device: the model here has no stack, no layers and no CUDA tensor."""
    from metamorph_b200.engine.decode import DecodeEngine
    model, _ = _fake_model(10)
    emb = torch.zeros((1, 3, 8), dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="forced_tokens"):
        DecodeEngine(model).generate(emb, forced_tokens=torch.tensor(bad), max_new_tokens=4)
    with pytest.raises(ValueError, match=r"\[B=1, n\]"):
        DecodeEngine(model).generate(emb, forced_tokens=torch.tensor([1, 2]), max_new_tokens=4)
    with pytest.raises(AttributeError):                      # ids -1 and 9 pass the check; the fake has nothing beyond it
        DecodeEngine(model).generate(emb, forced_tokens=torch.tensor([[-1, 9]]), max_new_tokens=4)


@pytest.mark.parametrize("bad", [[10], [-2], [3, 4, 128258]])
def test_submit_rejects_forced_ids_outside_the_embedding_table_on_the_host(bad):
    from metamorph_b200.engine.serve import ContinuousBatcher
    srv = ContinuousBatcher.__new__(ContinuousBatcher)      # no device: only what submit reads before the check
    srv.inner = _fake_model(10)[1]
    srv.queue, srv.next_rid = [], 0
    with pytest.raises(ValueError, match="forced_tokens"):
        srv.submit(torch.zeros((3, 8)), max_new_tokens=2, forced_tokens=torch.tensor(bad))
    assert srv.queue == [] and srv.next_rid == 0
