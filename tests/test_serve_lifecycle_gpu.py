"""`DecodeEngine.generate` at its limits and the slot lifecycle of `ContinuousBatcher` on the H100 (TINY model).

A fully forced request needs no model to know its ids and how many visual embeddings it returns: both follow from
oracle/decode_state.py, the restatement of the reference loop body, and are asserted against it, not only against the
product's own `greedy_decode`. Slot reuse is probed through the batcher's own tensors: before a slot is handed to its
next request its stale cache, embeddings and ids are overwritten with NaN / a sentinel.
"""
import os

import pytest
import torch

from oracle.decode_state import DecodeConfig, run, run_forced

pytestmark = pytest.mark.gpu

START, END, EOS = 128256, 128257, (128001, 128009)
NTOK = 4


def _model(weights=None, ntok=NTOK):
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, weights if weights is not None else make_weights(TINY), num_image_tokens=ntok)
    model.eval()
    return model


def _emb(model, g, P, B=1):
    return model.get_model().embed_tokens(torch.randint(0, 128000, (B, P), generator=g).cuda())


def _schedule(g, n, **at):
    """n random ordinary ids with the given positions overwritten, e.g. _schedule(g, 9, **{"0": START})."""
    f = torch.randint(0, 128000, (n,), generator=g).to(torch.int32)
    for i, t in at.items():
        f[int(i)] = t
    return f


def _want(forced, max_new, ntok=NTOK):
    return run_forced(forced.tolist(), DecodeConfig(ntok, max_new, START, END, EOS))


def _server(model, **kw):
    from metamorph_b200.engine.serve import ContinuousBatcher
    args = dict(max_slots=2, max_context=64, max_new_tokens=24, poll_every=3)
    args.update(kw)
    return ContinuousBatcher(model, **args)


def _same_payload(a, b, what):
    assert a[0].cpu().tolist() == b[0].cpu().tolist(), f"{what}: ids differ"
    assert a[1].shape == b[1].shape and torch.equal(a[1], b[1]), f"{what}: visual embeddings differ"


# ------------------------------------------------------------------------------------------------ engine limits
@pytest.mark.parametrize("max_new", [0, 1, 2, 9])
def test_engine_limits_follow_the_restatement(cuda_device, max_new):
    model = _model()
    g = torch.Generator().manual_seed(100 + max_new)
    B, P = 3, 6
    lens = torch.tensor([6, 1, 4], dtype=torch.int32)          # a one-position prompt beside a full-length one
    forced = torch.stack([_schedule(g, max_new + 1) for _ in range(B)])
    forced[0, 0] = START                                        # images from the first step
    if max_new >= 2:
        forced[2, 1] = EOS[1]
    emb = _emb(model, g, P, B)
    for b in range(B):
        emb[b, int(lens[b]):] = 0
    want = [_want(forced[b], max_new) for b in range(B)]
    assert len(want[0].kept_steps) == min(max_new, NTOK) and want[1].total_output == max_new + 1
    assert max_new < 2 or want[2].total_output == 2
    for poll in (1, 16, 100):
        ids, imgs = model._decode.generate(emb, prompt_lens=lens, max_new_tokens=max_new, forced_tokens=forced,
                                           poll_every=poll)
        assert model._decode.last_timing["cuda_graph"] == (max_new + 1 > 2)     # steps_cap <= 2 has no graph path
        for b in range(B):
            assert ids[b].cpu().tolist() == want[b].ids, f"max_new={max_new} poll={poll} sequence {b}"
            assert imgs[b].shape[0] == len(want[b].kept_steps)
    # one sequence, and a run cut short by max_steps: the first max_steps passes of the loop
    if max_new == 9:
        ids, imgs = model._decode.generate(emb[:1], max_new_tokens=max_new, forced_tokens=forced[:1])
        assert ids[0].cpu().tolist() == want[0].ids and imgs[0].shape[0] == NTOK
        ids, imgs = model._decode.generate(emb[:1], max_new_tokens=max_new, forced_tokens=forced[:1], max_steps=4)
        cut = run([-1] * 4, DecodeConfig(NTOK, max_new, START, END, EOS), forced[0].tolist())
        assert not cut.broke and ids[0].cpu().tolist() == cut.ids and imgs[0].shape[0] == len(cut.kept_steps) == 3


@pytest.mark.parametrize("quirk", ["q1", "q2"])
def test_a_schedule_shorter_than_the_run_free_runs_in_engine_and_server(cuda_device, quirk):
    """The schedule holds one token, the one the reference's own free run emits first, so ending the schedule must give
    the reference's trajectory (tests/golden/greedy_decode_quirks.pt) in the engine and in the server alike. Repeating
    the last forced token instead would emit that token at every step."""
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "greedy_decode_quirks.pt"), weights_only=False)[quirk]
    model = _model(with_sparse_lm_head(make_weights(TINY), d["live_rows"])[0], d["num_image_tokens"])
    golden = [int(t) for t in d["ids"]]
    forced = torch.tensor([golden[0]], dtype=torch.int32)
    n_img = d["image_embeds"].shape[0]
    assert len(golden) + n_img > 1, "the schedule does not end before the run"
    repeated = run([golden[0]] * (d["max_new_tokens"] + 1),
                   DecodeConfig(d["num_image_tokens"], d["max_new_tokens"], d["start_image_token_id"],
                                d["end_image_token_id"], tuple(d["eos_token_id"])))
    assert (repeated.ids, len(repeated.kept_steps)) != (golden, n_img), "repeating the token would pass as well"
    kw = dict(start_image_token_id=d["start_image_token_id"], end_image_token_id=d["end_image_token_id"],
              eos_token_id=list(d["eos_token_id"]))
    emb = model.get_model().embed_tokens(d["prompt"].cuda())
    ids, imgs = model._decode.generate(emb.reshape(1, -1, emb.shape[-1]), max_new_tokens=d["max_new_tokens"],
                                       forced_tokens=forced.reshape(1, -1), **kw)
    assert ids[0].cpu().tolist() == golden, "engine"
    torch.testing.assert_close(imgs[0].float().cpu(), d["image_embeds"], rtol=0, atol=1e-2)
    srv = _server(model, **kw)
    rid = srv.submit(emb, max_new_tokens=d["max_new_tokens"], forced_tokens=forced)
    sids, simg = srv.run_until_idle()[rid]
    assert sids.cpu().tolist() == golden, "server"
    torch.testing.assert_close(simg.float().cpu(), d["image_embeds"], rtol=0, atol=1e-2)


def test_forced_ids_outside_the_embedding_table_are_rejected_before_any_step(cuda_device):
    model = _model()
    g = torch.Generator().manual_seed(7)
    emb = _emb(model, g, 5)
    rows = model.get_model().embed_tokens.weight.shape[0]
    srv = _server(model)
    for bad in (rows, rows + 1000, -2):
        with pytest.raises(ValueError, match="forced_tokens"):
            model.greedy_decode(None, None, emb, max_new_tokens=3, forced_tokens=torch.tensor([[1, bad, 2, 3]]))
        with pytest.raises(ValueError, match="forced_tokens"):
            srv.submit(emb, max_new_tokens=3, forced_tokens=torch.tensor([1, bad, 2, 3]))
    assert not srv.queue and srv.steps_run == 0
    last = torch.tensor([[rows - 1, -1, 0, 5]], dtype=torch.int32)             # the table's last row is a legal id
    ids, _ = model.greedy_decode(None, None, emb, max_new_tokens=0, forced_tokens=last, output_image=True)
    assert ids[0].cpu().tolist() == [rows - 1]


# ------------------------------------------------------------------------------------------------ slot reuse
def _reuse_cases():
    from metamorph_b200.engine.sampling import SamplingParams
    g = torch.Generator().manual_seed(50)
    long_forced = _schedule(g, 20, **{"1": START, "8": END, "10": START})
    return {
        "forced_then_free": (dict(max_new_tokens=18, forced_tokens=long_forced), dict(max_new_tokens=6)),
        "sampled_then_greedy": (dict(max_new_tokens=18, forced_tokens=torch.where(long_forced > 128000, long_forced, -1),
                                     sampling=SamplingParams(temperature=1.0, top_k=30, seed=5)),
                                dict(max_new_tokens=6)),
        "greedy_then_sampled": (dict(max_new_tokens=18, forced_tokens=long_forced),
                                dict(max_new_tokens=6, sampling=SamplingParams(temperature=0.9, top_p=0.9, seed=11))),
    }


@pytest.mark.parametrize("case", ["forced_then_free", "sampled_then_greedy", "greedy_then_sampled"])
def test_a_reused_slot_serves_its_next_request_as_a_fresh_server_would(cuda_device, case):
    first_kw, second_kw = _reuse_cases()[case]
    model = _model()
    g = torch.Generator().manual_seed(51)
    long_emb, short_emb = _emb(model, g, 12), _emb(model, g, 4)
    fresh = _server(model, max_slots=1)
    rid = fresh.submit(short_emb, **second_kw)
    alone = fresh.run_until_idle()[rid]

    srv = _server(model, max_slots=1)
    r1 = srv.submit(long_emb, **first_kw)
    r2 = srv.submit(short_emb, **second_kw)
    results = {}
    for rid, kind, payload in srv.run():
        if kind != "done":
            continue
        results[rid] = payload
        if rid == r1:                                           # the slot is free and its next request not yet admitted
            assert srv.slots[0] is None and len(srv.queue) == 1
            assert payload[1].shape[0] >= NTOK, "the first request left no visual embeddings behind"
            assert int(srv.st["n_ids"][0]) > 3 and int(srv.st["pos"][0]) > 4 + 6
            P = short_emb.shape[1]
            srv.kc[:, 0, :, P:, :] = float("nan")               # stale cache beyond the new prompt
            srv.vc[:, 0, :, P:, :] = float("nan")
            srv.img_out[0] = float("nan")
            srv.st["ids_out"][0] = -12345
            assert torch.isnan(srv.kc[:, 0, :, P:]).all() and torch.isnan(srv.img_out[0]).all()
    assert set(results) == {r1, r2}
    _same_payload(results[r2], alone, case)
    assert not torch.isnan(results[r2][1].float()).any() and (results[r2][0] >= 0).all()
    if case == "forced_then_free":                              # the second request did not inherit the schedule
        assert (srv.forced[0] == -1).all()
    if case == "greedy_then_sampled":
        assert srv.sampled_graph is not None or srv._warm_sampled


# ------------------------------------------------------------------------------------------------ frozen slots, bounds
def test_a_finished_slot_stays_frozen_while_its_neighbour_runs(cuda_device):
    model = _model()
    g = torch.Generator().manual_seed(60)
    short = (_emb(model, g, 5), dict(max_new_tokens=6, forced_tokens=_schedule(g, 8, **{"0": START, "2": EOS[0]})))
    long_ = (_emb(model, g, 9), dict(max_new_tokens=20, forced_tokens=_schedule(g, 22, **{"3": START, "9": END})))
    want_short, want_long = _want(short[1]["forced_tokens"], 6), _want(long_[1]["forced_tokens"], 20)
    assert want_short.total_output == 3 and want_short.in_image_mode and want_long.total_output == 21
    out = {}
    for poll in (1, 50):                                        # 50: the short request sits finished for 47 steps
        srv = _server(model, poll_every=poll)
        rids = [srv.submit(e, **kw) for e, kw in (short, long_)]
        res = srv.run_until_idle()
        out[poll] = [res[r] for r in rids]
        assert srv.steps_run >= (21 if poll == 1 else 50)
    for i, want in enumerate((want_short, want_long)):
        _same_payload(out[1][i], out[50][i], f"request {i}")
        assert out[1][i][0].cpu().tolist() == want.ids and out[1][i][1].shape[0] == len(want.kept_steps)
    srv = _server(model, poll_every=50)
    rid = srv.submit(long_[0], **long_[1])
    _same_payload(srv.run_until_idle()[rid], out[50][1], "the neighbour alone")


def test_admission_bounds(cuda_device):
    model = _model()
    g = torch.Generator().manual_seed(70)
    cap, ctx = 10, 24
    srv = _server(model, max_context=ctx, max_new_tokens=cap, poll_every=2)
    with pytest.raises(ValueError, match="max_context"):
        srv.submit(_emb(model, g, ctx - cap - 1), max_new_tokens=cap)           # one position too many
    with pytest.raises(ValueError, match="limit"):
        srv.submit(_emb(model, g, 3), max_new_tokens=cap + 1)
    reqs = {
        "fits_exactly": (_emb(model, g, ctx - cap - 2), cap, _schedule(g, cap + 1, **{"1": START})),
        "one_position_prompt": (_emb(model, g, 1), 5, _schedule(g, 6, **{"0": START})),   # nothing to prefill
        "no_new_tokens": (_emb(model, g, 4), 0, _schedule(g, 1)),
    }
    assert reqs["fits_exactly"][0].shape[1] + cap + 2 == ctx
    sentinel = 7.0
    srv.kc[:, 1, :, 1:] = sentinel                              # the idle slot only ever rewrites its own position 0
    srv.vc[:, 1, :, 1:] = sentinel
    for name, (emb, n_new, forced) in reqs.items():
        rid = srv.submit(emb, max_new_tokens=n_new, forced_tokens=forced)
        ids, img = srv.run_until_idle()[rid]
        want = _want(forced, n_new)
        assert want.total_output == n_new + 1, f"{name} did not run to its limit"
        assert ids.cpu().tolist() == want.ids and img.shape[0] == len(want.kept_steps), name
        assert int(srv.st["pos"][0]) == emb.shape[1] + n_new + 1 <= ctx - 1
    assert (srv.kc[:, 1, :, 1:] == sentinel).all() and (srv.vc[:, 1, :, 1:] == sentinel).all()
    # more requests than slots, all finishing in the same step
    batch = [(_emb(model, g, 3 + i), _schedule(g, 5, **{"3": EOS[1]})) for i in range(5)]
    rids = [srv.submit(e, max_new_tokens=8, forced_tokens=f) for e, f in batch]
    res = srv.run_until_idle()
    for rid, (_, f) in zip(rids, batch):
        assert res[rid][0].cpu().tolist() == _want(torch.cat([f, f]), 8).ids == f[:4].tolist()
    assert all(s is None for s in srv.slots) and not srv.queue


# ------------------------------------------------------------------------------------------------ run() and streaming
def _traffic(model):
    g = torch.Generator().manual_seed(80)
    return [(_emb(model, g, 4 + i), dict(max_new_tokens=6 + 3 * i,
                                         forced_tokens=_schedule(g, 20, **{str(i): START, str(i + 6): END})))
            for i in range(4)]


def _flat(events):
    return [(rid, kind, tuple(t.cpu().flatten().tolist() for t in (payload if kind == "done" else (payload,))))
            for rid, kind, payload in events]


def test_run_resumes_after_max_steps_and_streams_what_done_returns(cuda_device):
    model = _model()
    srv = _server(model)
    for e, kw in _traffic(model):
        srv.submit(e, **kw)
    whole, live_ok = [], True
    for ev in srv.run():
        if ev[1] != "done":                                     # a streamed event names a request that holds a slot
            live_ok &= ev[0] in {r.rid for r in srv.slots if r is not None}
        whole.append(ev)
    assert live_ok, "an event named an idle slot"
    srv2 = _server(model)
    for e, kw in _traffic(model):
        srv2.submit(e, **kw)
    first = list(srv2.run(max_steps=6))
    assert srv2.steps_run == 6 and any(s is not None for s in srv2.slots), "the first run() did not return mid-flight"
    assert not any(kind == "done" for _, kind, _ in first)
    rest = list(srv2.run())
    assert _flat(first + rest) == _flat(whole)
    # per request: the streamed chunks, concatenated, are the done payload
    for rid in range(4):
        ids = [p for r, k, p in whole if r == rid and k == "ids"]
        img = [p for r, k, p in whole if r == rid and k == "image_embeds"]
        done = [p for r, k, p in whole if r == rid and k == "done"]
        assert len(done) == 1 and torch.equal(torch.cat(ids), done[0][0]) and torch.equal(torch.cat(img), done[0][1])
        want = _want(_traffic(model)[rid][1]["forced_tokens"], 6 + 3 * rid)
        assert done[0][0].cpu().tolist() == want.ids and done[0][1].shape[0] == len(want.kept_steps) == NTOK
