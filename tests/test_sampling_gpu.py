"""Seeded temperature / top-k / top-p sampling on the H100 (csrc/sampling.cu) against the fp64 restatement in
oracle/sampling.py, and through the decode engine, the model's greedy_decode / generate and the continuous batcher."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V, LD = 128258, 128264


def _params(R, T=0.0, k=0, p=1.0, seed=0, counter=0, dev="cuda"):
    f = lambda v, dt: torch.as_tensor(v, dtype=dt).expand(R).contiguous().to(dev)  # noqa: E731
    seeds = [int(s) - (1 << 64) if int(s) >= 1 << 63 else int(s) for s in np.broadcast_to(np.asarray(seed, dtype=object), (R,))]
    return (f(T, torch.float32), f(k, torch.int32), f(p, torch.float32), torch.tensor(seeds, dtype=torch.int64, device=dev),
            f(counter, torch.int32))


def _sample(buf, *prm):
    from metamorph_b200 import ops
    return ops.sample_rows(buf, V, *prm)


def _peaked_rows(R, g, dev):
    """LLM-like rows: a broad low background and ~200 tokens well above it."""
    buf = torch.randn(R, LD, generator=g) * 2.0
    for r in range(R):
        idx = torch.randperm(V, generator=g)[:200]
        buf[r, idx] += 10.0 + torch.rand(200, generator=g) * 4.0
    return buf.to(dev)


@pytest.mark.parametrize("R", [1, 8, 32])
def test_temperature_zero_is_argmax_bit_for_bit(cuda_device, R):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(R)
    buf = (torch.randn(R, LD, generator=g) * 3).to(cuda_device)
    buf[0, 77] = buf[0, 99999] = 100.0                        # exact tie: lowest index
    buf[R - 1, 16040] = float("nan")                            # NaN right at a CTA slice boundary, never chosen
    buf[R - 1, 3] = float("nan")
    if R > 1:
        buf[R // 2, V - 1] = 200.0                              # maximum in the last column
    want = ops.argmax_rows(buf, V)
    k = torch.randint(0, 50, (R,), generator=g).tolist()
    for T in (0.0, -1.0, float("nan")):                        # T <= 0 or NaN on the device: greedy
        prm = _params(R, T, k, 0.5, list(range(R)), 7, cuda_device)
        assert torch.equal(_sample(buf, *prm), want)
    assert int(want[0]) == 77
    # a row without any logit above -inf gives 0 for every parameter mix
    buf[:] = float("-inf")
    buf[0, 5] = float("nan")
    for T, kk, p in ((0.0, 0, 1.0), (1.0, 0, 1.0), (1.0, 5, 1.0), (0.7, 0, 0.5), (1.0, 3, 0.2), (1.0, 0, 0.0)):
        assert _sample(buf, *_params(R, T, kk, p, 1, 0, cuda_device)).eq(0).all(), (T, kk, p)


def test_draws_equal_the_fp64_oracle(cuda_device):
    from oracle.sampling import draw
    g = torch.Generator().manual_seed(1)
    rng = np.random.default_rng(2)
    n = 100
    buf = _peaked_rows(n, g, cuda_device)
    mixes = []
    for i in range(n):
        T = float(rng.uniform(0.4, 1.6))
        kind = i % 4
        k = int(rng.integers(1, 300)) if kind in (1, 3) else 0
        p = float(rng.uniform(0.05, 0.97)) if kind in (2, 3) else 1.0
        mixes.append((T, k, p, int(rng.integers(0, 1 << 64, dtype=np.uint64)), int(rng.integers(0, 5000))))
    T, k, p, s, c = (list(x) for x in zip(*mixes))
    prm = _params(n, T, k, p, s, c, cuda_device)
    got = _sample(buf, *prm).cpu().tolist()
    rows = buf[:, :V].cpu().numpy()
    p32 = prm[2].cpu().numpy()
    skipped = 0
    for i, (Ti, ki, _, si, ci) in enumerate(mixes):
        tok, gap, margin = draw(rows[i], np.float32(Ti), ki, float(p32[i]), si, ci)
        if gap < 1e-4 or margin < 1e-6:
            skipped += 1
            continue
        assert got[i] == tok, f"case {i} {mixes[i]}: kernel {got[i]} vs oracle {tok}"
    assert skipped < 0.02 * n, f"{skipped} of {n} cases too close to call"


@pytest.mark.parametrize("T,k,p", [(0.7, 0, 1.0), (1.0, 5, 1.0), (1.3, 0, 0.9), (1.0, 3, 0.5)])
def test_distribution_matches_the_warped_softmax(cuda_device, T, k, p):
    from scipy.stats import chisquare
    from oracle.sampling import warped_probs
    g = torch.Generator().manual_seed(3)
    row = torch.full((LD,), float("-inf"))
    live = torch.cat([torch.tensor([0, 16031, 16032, 16035, V - 1]), torch.randperm(V, generator=g)[:11]])
    row[live] = torch.randn(16, generator=g) * 1.5
    row[torch.tensor([1, 40000, 90001])] = float("nan")
    n = 4096
    buf = row.to(cuda_device).expand(n, LD).contiguous()
    tok = _sample(buf, *_params(n, T, k, p, list(range(n)), 11, cuda_device)).cpu().numpy()
    probs = warped_probs(row[:V].numpy(), np.float32(T), k, float(np.float32(p)))
    assert probs[tok].min() > 0, "a token outside the kept set was drawn"
    kept = np.flatnonzero(probs > 0)
    obs = np.array([(tok == t).sum() for t in kept], dtype=np.float64)
    exp = probs[kept] * n
    small = exp < 5                                        # pool the rare tokens into one bin
    if small.any():
        obs = np.append(obs[~small], obs[small].sum())
        exp = np.append(exp[~small], exp[small].sum())
    assert chisquare(obs, exp).pvalue > 1e-4


def test_invariance_repeats_graphs_and_switches(cuda_device):
    g = torch.Generator().manual_seed(4)
    R = 32
    buf = _peaked_rows(R, g, cuda_device)
    rng = np.random.default_rng(5)
    T = rng.uniform(0.5, 1.5, R).tolist()
    k = [int(x) for x in rng.integers(0, 100, R)]
    p = rng.uniform(0.2, 1.0, R).tolist()
    T[9] = 0.0
    prm = _params(R, T, k, p, [int(x) for x in rng.integers(0, 1 << 62, R)], list(range(R)), cuda_device)
    a = _sample(buf, *prm)
    assert torch.equal(a, _sample(buf, *prm))
    for r in (0, 9, 17, 31):                                # a row alone == the same row inside 32 others
        one = _sample(buf[r:r + 1], *(t[r:r + 1].contiguous() for t in prm))
        assert int(one[0]) == int(a[r])
    out = torch.empty(R, dtype=torch.int32, device=cuda_device)
    from metamorph_b200 import ops
    ops.sample_rows(buf, V, *prm, out=out)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        ops.sample_rows(buf, V, *prm, out=out)
    out.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a)
    # switches: k >= V is top-k off, p = 1 (and NaN on the device) is top-p off
    base = _params(R, 1.0, 0, 1.0, 123, 4, cuda_device)
    ref = _sample(buf, *base)
    for kk in (V, V + 5, -3):
        assert torch.equal(_sample(buf, base[0], torch.full_like(base[1], kk), *base[2:]), ref)
    assert torch.equal(_sample(buf, base[0], base[1], torch.full_like(base[2], float("nan")), *base[3:]), ref)


# ---------------------------------------------------------------------------------------------- decode on TINY
def _tiny_model():
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, make_weights(TINY), num_image_tokens=4)
    model.eval()
    return model


def _same(a, b):
    (ia, ea), (ib, eb) = a, b
    assert [x.cpu().tolist() for x in ia] == [x.cpu().tolist() for x in ib]
    assert len(ea) == len(eb) and all(torch.equal(x, y) for x, y in zip(ea, eb))


def test_decode_sampling(cuda_device):
    from metamorph_b200.engine.sampling import SamplingParams
    model = _tiny_model()
    g = torch.Generator().manual_seed(21)
    ids = torch.randint(0, 128000, (1, 9), generator=g).cuda()
    emb = model.get_model().embed_tokens(ids)
    run = lambda e=emb, **kw: model.greedy_decode(None, None, e, max_new_tokens=12, output_image=True, **kw)  # noqa: E731
    wrap = lambda r: ([r[0][0]], [r[1]])                                                                    # noqa: E731
    greedy = wrap(run())
    _same(wrap(run(sampling=SamplingParams(temperature=0.0, seed=3))), greedy)
    # HF-style kwargs on the custom-greedy path are ignored, as in the reference
    _same(wrap(model.generate(inputs=ids, output_image=True, do_sample=True, temperature=0.7, top_p=0.9,
                              max_new_tokens=12)), greedy)
    sp = SamplingParams(temperature=1.0, top_k=50, top_p=0.95, seed=1234)
    a = wrap(run(sampling=sp))
    _same(wrap(run(sampling=sp)), a)
    model._decode.use_cuda_graph = False
    _same(wrap(run(sampling=sp)), a)
    model._decode.use_cuda_graph = True
    b = wrap(run(sampling=SamplingParams(temperature=1.0, top_k=50, top_p=0.95, seed=1235)))
    assert a[0][0].cpu().tolist() != b[0][0].cpu().tolist()
    # a batch of 4 with one SamplingParams repeats bit for bit; a forced image block, then free-running sampled text
    B, steps = 4, 14
    e4 = model.get_model().embed_tokens(torch.randint(0, 128000, (B, 9), generator=g).cuda())
    forced = torch.full((B, steps + 2), -1, dtype=torch.int32)
    forced[:, 0] = 128256                                    # <image_start>: 4 visual embeddings, then <image_end>
    forced[:, 5] = 128257
    kw = dict(max_new_tokens=steps - 1, output_image=True, forced_tokens=forced,
              sampling=SamplingParams(temperature=1.0, top_k=20, seed=99), eos_token_id=[])
    r1 = model.greedy_decode(None, None, e4, **kw)
    _same(model.greedy_decode(None, None, e4, **kw), r1)
    for b in range(B):
        assert r1[1][b].shape[0] == 4
        t = r1[0][b].cpu().tolist()
        assert t[0] == 128256 and t[1] == 128257 and len(t) > 4
    assert len({tuple(r1[0][b].cpu().tolist()[2:]) for b in range(B)}) > 1, "sequences with seeds s+b all agree"


# ---------------------------------------------------------------------------------------------- serving
def _serve(model, reqs, max_slots=4, **kw):
    from metamorph_b200.engine.serve import ContinuousBatcher
    srv = ContinuousBatcher(model, max_slots=max_slots, max_context=64, max_new_tokens=24, poll_every=3, **kw)
    rids = [srv.submit(e, **a) for e, a in reqs]
    res = {r: p for r, kind, p in srv.run() if kind == "done"}
    return srv, [res[r] for r in rids]


def test_served_sampled_request_is_independent_of_its_neighbours(cuda_device):
    from metamorph_b200.engine.sampling import SamplingParams
    model = _tiny_model()
    g = torch.Generator().manual_seed(31)
    emb = lambda P: model.get_model().embed_tokens(torch.randint(0, 128000, (1, P), generator=g).cuda())  # noqa: E731
    target = (emb(8), dict(max_new_tokens=16, sampling=SamplingParams(temperature=0.9, top_k=40, top_p=0.9, seed=77)))
    forced = torch.randint(0, 128000, (20,), generator=g).to(torch.int32)
    forced[2] = 128256
    forced[7] = 128257
    others = [(emb(5), dict(max_new_tokens=10)),
              (emb(11), dict(max_new_tokens=12, forced_tokens=forced)),
              (emb(6), dict(max_new_tokens=20, sampling=SamplingParams(temperature=1.4, top_p=0.5, seed=5))),
              (emb(3), dict(max_new_tokens=4, sampling=SamplingParams(temperature=0.6, top_k=2, seed=6)))]
    _, (alone,) = _serve(model, [target])
    srv, mixed = _serve(model, others[:2] + [target] + others[2:])
    ids, img = mixed[2]
    assert ids.cpu().tolist() == alone[0].cpu().tolist()
    assert img.shape == alone[1].shape and torch.equal(img, alone[1])
    assert srv.sampled_graph is not None
    # greedy-only traffic never captures (or even runs) the sampled step
    srv, _ = _serve(model, others[:2])
    assert srv.sampled_graph is None and not srv._warm_sampled and srv.graph is not None


def test_quirk_golden_still_matches_next_to_a_sampled_request(cuda_device):
    import os
    from metamorph_b200.engine.sampling import SamplingParams
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    from tests.helpers import build_product_model
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "greedy_decode_quirks.pt"), weights_only=False)["q1"]
    model = build_product_model(TINY, with_sparse_lm_head(make_weights(TINY), d["live_rows"])[0],
                                num_image_tokens=d["num_image_tokens"])
    model.eval()
    g = torch.Generator().manual_seed(5)
    other = model.get_model().embed_tokens(torch.randint(0, 128000, (1, 9), generator=g).cuda())
    srv, res = _serve(model, [(other, dict(max_new_tokens=20, sampling=SamplingParams(temperature=1.0, seed=8))),
                              (model.get_model().embed_tokens(d["prompt"].cuda()), dict(max_new_tokens=d["max_new_tokens"]))],
                      max_slots=2, start_image_token_id=d["start_image_token_id"],
                      end_image_token_id=d["end_image_token_id"], eos_token_id=list(d["eos_token_id"]))
    ids, img = res[1]
    assert srv.sampled_graph is not None
    assert ids.cpu().tolist() == [int(t) for t in d["ids"]]
    torch.testing.assert_close(img.float().cpu(), d["image_embeds"], rtol=0, atol=1e-2)


def test_first_tokens_follow_the_models_warped_softmax(cuda_device):
    from scipy.stats import chisquare
    from metamorph_b200.engine.sampling import SamplingParams
    from oracle.sampling import warped_probs
    model = _tiny_model()
    g = torch.Generator().manual_seed(41)
    prompt = model.get_model().embed_tokens(torch.randint(0, 128000, (1, 7), generator=g).cuda())
    logits = model(inputs_embeds=prompt).logits[0, -1].float().cpu().numpy()
    B, reps, k = 32, 20, 8
    emb = prompt.expand(B, -1, -1).contiguous()
    first = []
    for rep in range(reps):
        sp = [SamplingParams(temperature=1.0, top_k=k, seed=rep * B + b) for b in range(B)]
        ids, _ = model.greedy_decode(None, None, emb, max_new_tokens=1, output_image=True, sampling=sp, eos_token_id=[])
        first += [int(x[0]) for x in ids]
    first = np.array(first)
    probs = warped_probs(logits, np.float32(1.0), k, 1.0)
    kept = np.flatnonzero(probs > 0)
    assert np.isin(first, kept).mean() > 0.99      # the decode logits are the bf16 KV-cache path, not bit-equal
    obs = np.array([(first == t).sum() for t in kept], dtype=np.float64)
    exp = probs[kept] * obs.sum()
    assert chisquare(obs, exp).pvalue > 1e-4
