"""Decode log-probabilities on the GPU: mm_decode_logprobs held to the fp64 restatement (oracle/logprobs.py) at the
vocabulary, tie, special-value and skip edges, and the engine / server / model API held to it along real decodes."""
import math
import os

import numpy as np
import pytest
import torch

import oracle.logprobs as O

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")
NAN, INF = float("nan"), float("inf")
WORST = {"fraction": 0.0, "values": 0}


def run(logits, V, tok, n_top, kind=None, n_ids=None, max_ids=3, graph=False):
    """One launch; outputs poisoned with NaN / -7 and a guard row past the last one. -> (lp, ids, lps) on the CPU."""
    from metamorph_b200 import ops
    R, dev = logits.shape[0], logits.device
    i32 = lambda v: torch.as_tensor(v, dtype=torch.int32).reshape(-1).expand(R).contiguous().to(dev)   # noqa: E731
    kind = i32(0 if kind is None else kind)
    n_ids = i32(1 if n_ids is None else n_ids)
    tok, n_top = i32(tok), i32(n_top)
    lp = torch.full((R + 1, max_ids), NAN, device=dev)
    ids = torch.full((R + 1, max_ids, 20), -7, dtype=torch.int32, device=dev)
    lps = torch.full((R + 1, max_ids, 20), NAN, device=dev)
    call = lambda: ops.decode_logprobs(logits, V, kind, tok, n_ids, n_top, lp, ids, lps)   # noqa: E731
    if graph:
        call()
        torch.cuda.synchronize()
        lp.fill_(NAN), ids.fill_(-7), lps.fill_(NAN)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call()
        g.replay()
    else:
        call()
    torch.cuda.synchronize()
    assert torch.isnan(lp[R]).all() and (ids[R] == -7).all() and torch.isnan(lps[R]).all(), "guard row written"
    return lp.cpu()[:R], ids.cpu()[:R], lps.cpu()[:R]


def check_rows(logits, V, tok, n, out, slot=0):
    lp, ids, lps = out
    x = logits[:, :V].cpu().numpy()
    nn = min(n, 20)
    for r in range(x.shape[0]):
        t = int(tok[r]) if hasattr(tok, "__len__") else int(tok)
        f = O.check_report(float(lp[r, slot]), ids[r, slot, :nn].numpy(), lps[r, slot, :nn].numpy().astype(np.float64),
                           x[r], t, nn, f"V={V} row {r}")
        WORST["fraction"] = max(WORST["fraction"], f)
        WORST["values"] += 1 + nn
        assert (ids[r, slot, nn:] == -7).all() and torch.isnan(lps[r, slot, nn:]).all(), "entry past n_top written"
        for s in range(lp.shape[1]):
            if s != slot:
                assert torch.isnan(lp[r, s]) and (ids[r, s] == -7).all(), "another slot written"
        # the emitted token's entry in the list has its bits
        hit = (ids[r, slot, :nn] == t).nonzero()
        if hit.numel():
            assert lps[r, slot, int(hit[0])].view(torch.int32) == lp[r, slot].view(torch.int32)


def rows(R, V, seed, scale=4.0, ld=None, dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    x = torch.full((R, ld or V), NAN)
    x[:, :V] = torch.randn(R, V, generator=g) * scale
    return x.to(dev)


# slice rule S = roundup4(ceil(V / 8)): empty trailing CTAs (V <= 24), a one-element last CTA (V = 7 S + 1), exact
# multiples, the LLaMA-3 vocabulary and the full shared-memory budget
VOCABS = [1, 2, 3, 5, 8, 29, 33, 64, 1000, 4097, 28673, 128258, 131072, 393216]


@pytest.mark.parametrize("V", VOCABS)
def test_kernel_matches_restatement_over_vocabularies(cuda_device, V):
    x = rows(3, V, V)
    if V > 40:
        x[0, V // 3] = x[0, V - 1] = x[0].max() + 2.0              # exact top tie across CTA slices
        x[1, 5] = NAN
    g = torch.Generator().manual_seed(1)
    tok = torch.randint(0, V, (3,), generator=g).tolist()
    tok[0] = int(torch.argmax(torch.nan_to_num(x[0, :V], nan=-INF)))
    check_rows(x, V, tok, 20, run(x, V, tok, 20))


def test_ld_wider_than_V_with_nan_padding(cuda_device):
    V = 128258
    x = rows(4, V, 7, ld=V + 38)
    x[:, V + 19:] = INF                                                # NaN, then +inf: never read as logits
    check_rows(x, V, [0, 1, V - 1, 77], 5, run(x, V, [0, 1, V - 1, 77], 5))


def test_exact_ties_across_slices_and_the_top_n_boundary(cuda_device):
    V = 128258
    x = torch.zeros(2, V, device="cuda")
    live = torch.tensor(np.sort(np.random.default_rng(5).choice(128000, 16, replace=False)))
    x[0, live.cuda()] = torch.randn(16, generator=torch.Generator().manual_seed(2)).cuda()   # sparse lm_head: 16 live rows
    x[1, ::16033] = 3.0                                               # 8 equal maxima, one per CTA slice
    x[1, 5:40] = 1.0                                                  # ties straddling entry 20
    for n in (0, 1, 5, 20):
        check_rows(x, V, [int(live[3]), 16033], n, run(x, V, [int(live[3]), 16033], n))


@pytest.mark.parametrize("n_top", [0, 1, 5, 20, 25])
def test_n_top_and_short_vocabularies(cuda_device, n_top):
    for V in (3, 17, 50000):
        x = rows(2, V, n_top + V)
        out = run(x, V, [0, V - 1], n_top)
        check_rows(x, V, [0, V - 1], n_top, out)                        # n_top 25 is 20 on the device


def test_special_values(cuda_device):
    V = 40000
    x = rows(8, V, 11)
    x[0, :] = 0.0
    x[0, 1::2] = -0.0                                                   # +-0 only: uniform, ties by index
    x[1, :] = torch.tensor(1e-40)                                       # denormals
    x[1, 123] = -1e-45
    x[2, 9] = 3.0e38
    x[2, 10] = -3.0e38                                                  # l - m overflows fp32
    x[3, 17] = x[3, 39000] = INF                                        # point mass on two entries
    x[4, :] = -INF                                                      # no distribution
    x[5, :] = NAN
    x[6, :5000] = NAN                                                   # NaN across a slice
    x[6, 4999] = 50.0
    x[7, 1] = INF
    x[7, 2] = NAN
    tok = [1, 123, 10, 39000, 3, 0, 4999, 2]
    out = run(x, V, tok, 20)
    check_rows(x, V, tok, 20, out)
    lp = out[0][:, 0]
    assert lp[3] == -math.log(2) and torch.isnan(lp[4]) and torch.isnan(lp[5]) and lp[7] == -INF
    assert out[1][4, 0].tolist() == list(range(20))
    assert torch.isnan(run(x, V, [V, -1, 5, 5, 5, 5, 5, 5], 1)[0][:2, 0]).all()    # tokens outside [0, V)


def test_skipped_rows_leave_outputs_untouched(cuda_device):
    V = 5000
    x = rows(6, V, 3)
    #            n_top -1    image step  nothing    n_ids > max_ids  n_ids == max_ids + 1  n_ids == 0
    n_top, kind, n_ids = [-1, 5, 5, 5, 5, 5], [0, 1, -1, 0, 0, 0], [1, 1, 1, 9, 4, 0]
    lp, ids, lps = run(x, V, [0] * 6, n_top, kind, n_ids, max_ids=3)
    assert torch.isnan(lp).all() and (ids == -7).all() and torch.isnan(lps).all()
    out = run(x, V, [4] * 6, 5, 0, 3, max_ids=3)                         # the last slot itself is written
    check_rows(x, V, [4] * 6, 5, out, slot=2)


def test_rows_are_independent_and_graph_replay_equals_stream(cuda_device):
    V = 128258
    x = rows(129, V, 21)
    tok = torch.randint(0, V, (129,), generator=torch.Generator().manual_seed(3)).tolist()
    n_top = [r % 21 for r in range(129)]
    full = run(x, V, tok, n_top)
    graph = run(x, V, tok, n_top, graph=True)
    for a, b in zip(full, graph):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for sel in ([0], [5, 77], list(range(128, 129))):
        sub = run(x[sel].contiguous(), V, [tok[i] for i in sel], [n_top[i] for i in sel])
        for a, b in zip(full, sub):
            assert torch.equal(a[sel].view(torch.int32), b.view(torch.int32))
    one = run(x[7:8].contiguous(), V, [tok[7]], 20)                       # n_top does not change the bits
    assert one[0][0, 0].view(torch.int32) == full[0][7, 0].view(torch.int32)
    assert one[2][0, 0, :n_top[7]].view(torch.int32).equal(full[2][7, 0, :n_top[7]].view(torch.int32))


def test_report_worst_fraction_of_the_bound(cuda_device):
    """Runs last in this file's kernel group: prints the largest fraction of eps reached over every value checked."""
    print(f"\nlogprob values checked {WORST['values']}, largest excess over 0.5 ulp = "
          f"{WORST['fraction']:.3g} of eps (2^-21 + 2^-51 |x|)")
    assert WORST["fraction"] <= 1.0


# ---------------------------------------------------------------- engine, server and model API
def _model(sparse=False, num_image_tokens=4):
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    from tests.helpers import build_product_model
    W = make_weights(TINY)
    if sparse:
        W = with_sparse_lm_head(W, 16)[0]
    m = build_product_model(TINY, W, num_image_tokens=num_image_tokens)
    m.eval()
    return m, W


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int16) \
        if t.dtype == torch.bfloat16 else t


def _prompts(m, B, P, seed):
    g = torch.Generator().manual_seed(seed)
    return m.get_model().embed_tokens(torch.randint(0, 128000, (B, P), generator=g).cuda())


@pytest.mark.parametrize("B", [1, 8, 40])
def test_engine_outputs_unchanged_and_logprobs_follow_ids(cuda_device, B):
    from metamorph_b200.engine.decode import DecodeEngine
    m, _ = _model(sparse=True)
    eng = DecodeEngine(m)
    x = _prompts(m, B, 9, B)
    ids0, img0 = eng.generate(x, max_new_tokens=12, start_image_token_id=1000)
    ids1, img1, lps = eng.generate(x, max_new_tokens=12, start_image_token_id=1000, logprobs=3)
    for b in range(B):
        assert torch.equal(ids0[b], ids1[b]) and torch.equal(_bits(img0[b]), _bits(img1[b]))
        k = ids1[b].numel()
        assert lps[b].logprob.shape == (k,) and lps[b].top_ids.shape == (k, 3) and lps[b].top_logprobs.shape == (k, 3)
        assert torch.equal(lps[b].top_ids[:, 0], ids1[b])              # unforced greedy: the emitted id is entry 0
        assert torch.equal(_bits(lps[b].top_logprobs[:, 0]), _bits(lps[b].logprob))


def _server(m, **kw):
    from metamorph_b200.engine.serve import ContinuousBatcher
    args = dict(max_slots=4, max_context=64, max_new_tokens=16, poll_every=4)
    args.update(kw)
    return ContinuousBatcher(m, **args)


def _serve(srv, reqs):
    """reqs: list of submit kwargs -> list of done payloads (in submission order) and the streamed events per rid."""
    rids = [srv.submit(**r) for r in reqs]
    done, stream = {}, {}
    for rid, kind, payload in srv.run():
        if kind == "done":
            done[rid] = payload
        else:
            stream.setdefault(rid, []).append((kind, payload))
    return [done[r] for r in rids], [stream.get(r, []) for r in rids]


def test_server_outputs_unchanged_for_requester_and_neighbours(cuda_device):
    from metamorph_b200.engine.sampling import SamplingParams
    m, _ = _model(sparse=True)
    x = _prompts(m, 4, 10, 1)
    forced = torch.tensor([5, 1000, 7, 7, 7, -1, 9])
    base = [dict(inputs_embeds=x[0]), dict(inputs_embeds=x[1], sampling=SamplingParams(temperature=0.9, seed=4)),
            dict(inputs_embeds=x[2], forced_tokens=forced), dict(inputs_embeds=x[3])]
    off, _ = _serve(_server(m, start_image_token_id=1000), base)
    for asker in range(4):
        reqs = [dict(r) for r in base]
        reqs[asker]["logprobs"] = 2
        on, _ = _serve(_server(m, start_image_token_id=1000), reqs)
        for i in range(4):
            assert torch.equal(off[i][0], on[i][0]) and torch.equal(_bits(off[i][1]), _bits(on[i][1]))
            assert len(on[i]) == (3 if i == asker else 2)
        assert on[asker][2].logprob.shape[0] == on[asker][0].numel()


def test_eager_server_reports_the_restatement_of_each_steps_logits(cuda_device):
    from metamorph_b200.engine.sampling import SamplingParams
    m, _ = _model(sparse=False)
    srv = _server(m, use_cuda_graph=False, poll_every=1, start_image_token_id=1000)
    x = _prompts(m, 3, 8, 2)
    reqs = [dict(inputs_embeds=x[0], logprobs=5), dict(inputs_embeds=x[1], logprobs=20, forced_tokens=torch.tensor(
            [3, 1000, -1, -1, -1, -1, 17, 128257])), dict(inputs_embeds=x[2], logprobs=0,
                                                          sampling=SamplingParams(temperature=1.3, top_k=50, seed=9))]
    trace = {}
    step = srv._device_step

    def snap():
        step()
        lg = srv.logits[:, :srv.V].cpu().numpy()
        st = {k: srv.st[k].cpu().tolist() for k in ("append_kind", "next_token", "n_ids")}
        for b, r in enumerate(srv.slots):
            if r is not None:
                trace.setdefault(r.rid, []).append((lg[b].copy(), st["next_token"][b], st["append_kind"][b],
                                                    st["n_ids"][b]))
    srv._device_step = snap
    done, _ = _serve(srv, reqs)
    worst = 0.0
    for rid, ((ids, img, lps), r) in enumerate(zip(done, reqs)):
        n = r["logprobs"]
        k = ids.numel()
        lp = np.full(k + 1, np.nan)
        lp[:k] = lps.logprob.cpu().numpy()
        top = np.full((k + 1, 20), -2)
        top[:k, :n] = lps.top_ids.cpu().numpy()
        tlp = np.full((k + 1, 20), np.nan)
        tlp[:k, :n] = lps.top_logprobs.cpu().numpy()
        worst = max(worst, O.check_stored(lp, top, tlp, trace[rid], k + 1, n, poison_id=-2, what=f"request {rid}"))
        assert [t for _, t, kind, _ in trace[rid] if kind == 0] == ids.cpu().tolist()
    print(f"\neager server: largest excess over 0.5 ulp = {worst:.3g} of eps")


def test_logprob_bits_do_not_depend_on_the_server(cuda_device):
    """On servers of one shape (128 slots: the slot count sets the decode attention's context split, so the logits'
    bits), a request's logprob bits do not depend on its neighbours, the step graph or the cache layout."""
    from metamorph_b200.engine.sampling import SamplingParams
    m, _ = _model(sparse=True)
    x = _prompts(m, 128, 70, 3)
    req = dict(inputs_embeds=x[0], logprobs=4, max_new_tokens=12)
    kw = dict(max_slots=128, max_context=128, max_new_tokens=16, start_image_token_id=1000)

    def lp_of(done):
        return [_bits(t) for t in done[0][2]]

    alone = lp_of(_serve(_server(m, **kw), [req])[0])
    crowd = lp_of(_serve(_server(m, **kw), [req] + [dict(inputs_embeds=x[i], max_new_tokens=10)
                                                    for i in range(1, 128)])[0])
    sampled = lp_of(_serve(_server(m, **kw), [req, dict(inputs_embeds=x[1], sampling=SamplingParams(
        temperature=1.0, seed=1))])[0])
    paged_srv = _server(m, kv_pool_tokens=1024, kv_block_size=16, **kw)
    paged = lp_of(_serve(paged_srv, [req])[0])
    h = paged_srv.cache_prefix(x[0][:40])
    prefixed = lp_of(_serve(paged_srv, [dict(req, inputs_embeds=x[0][40:], prefix=h)])[0])
    for other in (crowd, sampled, paged, prefixed):
        for a, b in zip(alone, other):
            assert torch.equal(a, b)


def test_scoring_a_forced_continuation_against_the_restatement(cuda_device):
    """generate(..., forced_tokens, logprobs=1) scores a continuation: each logprob agrees with the restatement's fp32
    log-softmax within 2 x the step's measured product-versus-restatement logit error (plus the kernel's bound)."""
    from oracle.weights import TINY
    m, W = _model(sparse=False)
    d = torch.load(os.path.join(G, "greedy_decode_tiny.pt"), weights_only=False)
    g = torch.Generator().manual_seed(8)
    cont = torch.randint(0, 128000, (8,), generator=g)
    cfg, x0 = dict(TINY, image_tokens=4), W["model.embed_tokens.weight"][d["prompt"]]
    cont[0] = O.trajectory_logprobs(W, cfg, x0, 0, start_id=d["start_image_token_id"])[0]["token"]   # a greedy step
    forced = cont.clone()
    ref = O.trajectory_logprobs(W, cfg, x0, 7, forced=forced.tolist(), start_id=d["start_image_token_id"])
    emb = m.get_model().embed_tokens(d["prompt"].cuda())
    # product logits of every step, from an eager server fed the same forced schedule
    srv = _server(m, use_cuda_graph=False, poll_every=1, start_image_token_id=d["start_image_token_id"])
    logits = []
    step = srv._device_step

    def snap():
        step()
        if srv.slots[0] is not None and int(srv.st["append_kind"][0]) == 0:
            logits.append(srv.logits[0, :srv.V].cpu().numpy().copy())
    srv._device_step = snap
    _serve(srv, [dict(inputs_embeds=emb[0], forced_tokens=forced, max_new_tokens=7)])
    ids, lps = m.generate(d["prompt"].cuda(), max_new_tokens=7, start_image_token_id=d["start_image_token_id"],
                          forced_tokens=forced[None], logprobs=1)
    ids, lps = ids[0].cpu(), lps[0]
    assert ids.tolist() == [s["token"] for s in ref] and len(logits) == len(ref) == ids.numel()
    for k, s in enumerate(ref):
        delta = float(np.abs(logits[k].astype(np.float64) - s["logits"]).max())
        got = float(lps.logprob[k])
        assert abs(got - s["logprob"]) <= 2 * delta + O.bound(s["logprob"]) + 1e-6, (k, got, s["logprob"], delta)
        order = np.argsort(-s["logits"].astype(np.float64), kind="stable")
        margin = float(s["logits"][order[0]] - s["logits"][order[1]])
        if margin > 2 * delta:                                           # the restatement's argmax is decided
            assert (int(lps.top_ids[k, 0]) == int(ids[k])) == s["greedy"], k


@pytest.mark.parametrize("quirk", ["q1", "q2"])
def test_quirk_goldens_decode_exactly_with_logprobs(cuda_device, quirk):
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    from tests.helpers import build_product_model
    d = torch.load(os.path.join(G, "greedy_decode_quirks.pt"), weights_only=False)[quirk]
    m = build_product_model(TINY, with_sparse_lm_head(make_weights(TINY), d["live_rows"])[0],
                            num_image_tokens=d["num_image_tokens"])
    m.eval()
    ids, img, lps = m.generate(d["prompt"].cuda(), output_image=True, max_new_tokens=d["max_new_tokens"],
                               start_image_token_id=d["start_image_token_id"],
                               end_image_token_id=d["end_image_token_id"], eos_token_id=list(d["eos_token_id"]),
                               logprobs=3)
    assert ids[0].cpu().tolist() == [int(t) for t in d["ids"]]
    assert tuple(img.shape) == tuple(d["image_embeds"].shape)
    assert len(lps) == 1 and lps[0].logprob.numel() == ids[0].numel()
    assert torch.isfinite(lps[0].logprob).all()


def test_streamed_chunks_concatenate_to_the_done_payload(cuda_device):
    m, _ = _model(sparse=True)
    x = _prompts(m, 2, 6, 4)
    srv = _server(m, poll_every=3, start_image_token_id=1000)
    done, stream = _serve(srv, [dict(inputs_embeds=x[0], logprobs=6), dict(inputs_embeds=x[1])])
    ids, img, lps = done[0]
    kinds = [k for k, _ in stream[0]]
    assert "logprobs" in kinds and kinds.count("logprobs") == kinds.count("ids")
    for f in ("logprob", "top_ids", "top_logprobs"):
        cat = torch.cat([getattr(p, f) for k, p in stream[0] if k == "logprobs"])
        assert torch.equal(_bits(cat), _bits(getattr(lps, f)))
    assert torch.equal(torch.cat([p for k, p in stream[0] if k == "ids"]), ids)
    assert all(k != "logprobs" for k, _ in stream[1]) and len(done[1]) == 2
