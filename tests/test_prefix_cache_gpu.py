"""Prefix caching on the H100: `attn_fwd_paged` against the dense flash attention bit for bit, GEMM rows across BN 128
and 256, one LLaMA-3-8B-width layer prefilled whole against prefix + suffix, and a `ContinuousBatcher` serving
`submit(suffix, prefix=h)` against the same prompts submitted whole, on paged and dense servers.

Bits are compared as int16 views, so a NaN sentinel or poison compares as bits, not as a float."""
import pytest
import torch

pytestmark = pytest.mark.gpu

START, END, EOS = 128256, 128257, (128001, 128009)
NTOK = 4
NAN = float("nan")
SENT = -3.5


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ kernel
def _paged_case(q_start, n_q, bs, G, Hkv=2, seed=0):
    """Keys / values of positions 0 .. kv_len-1 scattered into a NaN pool through a random permutation (the table's
    entries past kv_len name NaN blocks too); the queries are the rows q_start.. of a fused qkv; the output sits inside a
    sentinel frame. Row r must equal row r of the dense kernel at T = kv_len."""
    from metamorph_b200 import ops
    dev = torch.device("cuda")
    kv_len, Hq, dh = q_start + n_q, G * Hkv, 128
    gen = torch.Generator(device=dev).manual_seed(seed)
    qkv = torch.randn(kv_len, (Hq + 2 * Hkv) * dh, device=dev, generator=gen).bfloat16()
    q, k, v = qkv[:, :Hq * dh], qkv[:, Hq * dh:(Hq + Hkv) * dh], qkv[:, (Hq + Hkv) * dh:]
    scale = dh ** -0.5
    dense, _ = ops.attn_fwd(q, k, v, 1, kv_len, Hq, Hkv, dh, True, scale, need_lse=False)
    max_blocks = -(-kv_len // bs) + 2
    nb = max_blocks + 5
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed + 1))
    table = perm[:max_blocks].to(torch.int32).to(dev)
    kp = torch.full((nb, Hkv, bs, dh), NAN, dtype=torch.bfloat16, device=dev)
    vp = kp.clone()
    for p0 in range(0, kv_len, bs):
        p1 = min(kv_len, p0 + bs)
        blk = int(perm[p0 // bs])
        kp[blk, :, :p1 - p0] = k[p0:p1].reshape(p1 - p0, Hkv, dh).transpose(0, 1)
        vp[blk, :, :p1 - p0] = v[p0:p1].reshape(p1 - p0, Hkv, dh).transpose(0, 1)
    kp0, vp0 = kp.clone(), vp.clone()
    frame = torch.full((n_q + 2, Hq * dh + 16), SENT, dtype=torch.bfloat16, device=dev)
    out = frame[1:1 + n_q, 8:8 + Hq * dh]
    ops.attn_fwd_paged(q[q_start:], kp, vp, table, q_start, Hq, Hkv, dh, scale, out=out)
    torch.cuda.synchronize()
    what = f"q_start={q_start} n_q={n_q} bs={bs} G={G} Hkv={Hkv}"
    assert _same_bits(out, dense[q_start:]), f"{what}: paged rows differ from the dense kernel"
    keep = torch.ones(frame.shape, dtype=torch.bool, device=dev)
    keep[1:1 + n_q, 8:8 + Hq * dh] = False
    assert bool((frame[keep] == SENT).all()), f"{what}: a guard element around the output was written"
    assert _same_bits(kp, kp0) and _same_bits(vp, vp0), f"{what}: the pool was written"


@pytest.mark.parametrize("bs", [16, 64, 128, 256])
@pytest.mark.parametrize("q_start", [0, 16, 48, 128, 144, 4096 - 128])
@pytest.mark.parametrize("n_q", [1, 127, 128, 129, 300])
def test_paged_prefill_attention_equals_dense_rows(cuda_device, q_start, n_q, bs):
    _paged_case(q_start, n_q, bs, G=4, seed=q_start * 7 + n_q + bs)


@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("q_start,n_q", [(48, 129), (256, 300)])
def test_paged_prefill_attention_for_every_gqa_group(cuda_device, G, q_start, n_q):
    _paged_case(q_start, n_q, 64, G=G, seed=G + q_start)


@pytest.mark.parametrize("q_start,n_q,bs", [(4096 - 300, 300, 64), (2048, 2048, 16), (0, 4096, 256)])
def test_paged_prefill_attention_at_llama_heads_and_4096_positions(cuda_device, q_start, n_q, bs):
    _paged_case(q_start, n_q, bs, G=4, Hkv=8, seed=n_q)


# ------------------------------------------------------------------------------------------------ GEMM rows across BN
# LLaMA-3-8B: qkv (K 4096, N 6144), o_proj + residual (K 4096, N 4096), gate|up SwiGLU (K 4096, N 28672 interleaved),
# down_proj + residual (K 14336, N 4096)
BN_SHAPES = [("qkv-store", 4096, 6144, "store"), ("o_proj-resid", 4096, 4096, "resid"),
             ("gate_up-swiglu", 4096, 28672, "swiglu"), ("down-resid", 14336, 4096, "resid")]


@pytest.mark.parametrize("name,K,N,epi", BN_SHAPES, ids=[s[0] for s in BN_SHAPES])
def test_gemm_rows_are_the_same_bits_at_bn_128_and_256(cuda_device, name, K, N, epi):
    """A prefix is prefilled at M = its length and a suffix at its own M, so the automatic BN choice can differ between
    the two (BN 128 below a wave of 256-wide tiles). Each output element runs the same k16 steps in the same order at
    either width, so the rows must be the same bits."""
    from metamorph_b200 import ops
    M = 700
    gen = torch.Generator(device=cuda_device).manual_seed(K + N)
    a = (torch.randn(M, K, device=cuda_device, generator=gen)).bfloat16()
    b = (torch.randn(N, K, device=cuda_device, generator=gen) * K ** -0.5).bfloat16()
    r = torch.randn(M, N, device=cuda_device, generator=gen).bfloat16()
    outs = {}
    for bn in (128, 256):
        if epi == "store":
            outs[bn] = (ops.gemm(a, b, force_bn=bn),)
        elif epi == "resid":
            outs[bn] = (ops.gemm(a, b, resid=r, epilogue=ops.EPI_RESID, force_bn=bn),)
        else:
            aux = torch.empty(M, N, dtype=torch.bfloat16, device=cuda_device)
            outs[bn] = (ops.gemm(a, b, aux=aux, epilogue=ops.EPI_SWIGLU, force_bn=bn), aux)
    for x, y in zip(outs[128], outs[256]):
        assert _same_bits(x, y), f"{name}: rows differ between BN 128 and BN 256"
    # and a short M (as a suffix prefill) against the long one, at the automatic choice
    short = ops.gemm(a[:24], b) if epi == "store" else None
    if short is not None:
        assert _same_bits(short, outs[256][0][:24])


# ------------------------------------------------------------------------------------------------ one real-width layer
@pytest.fixture(scope="module")
def real_layer():
    from oracle.weights import REAL_A, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(REAL_A, make_weights(REAL_A))
    model.eval()
    return model


@pytest.mark.parametrize("bs,Lp", [(64, 704), (128, 768)])
def test_one_layer_prefix_then_suffix_equals_the_whole_prompt(cuda_device, real_layer, bs, Lp):
    """LLaMA-3-8B width: a prefix of more than 640 rows (BN 256 for the qkv GEMM) then a 40-row suffix (BN 128) through
    the paged path give every position's K/V and the suffix's layer output bit for bit as one whole-prompt prefill."""
    from metamorph_b200 import ops
    from metamorph_b200.engine.llama import PagedPrefill, StackContext
    stack = real_layer.stack
    d = stack.dims
    w = real_layer.get_model().layers[0].weights()
    S = 40
    T = Lp + S
    stack.ensure_positions(T + 1)
    gen = torch.Generator(device=cuda_device).manual_seed(bs)
    x = (torch.randn(T, d.hidden, device=cuda_device, generator=gen) * 0.5).bfloat16()
    pos = torch.arange(T, dtype=torch.int32, device=cuda_device)
    ctx = StackContext(B=1, T=T, pos=pos, seqlens=None)
    want = stack.layer_forward(w, x, ctx, save=True, save_gu=False)
    qkv_full = ctx.saved.pop().qkv
    Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
    max_blocks = -(-T // bs) + 1
    nb = max_blocks + 3
    table = torch.randperm(nb, generator=torch.Generator().manual_seed(bs))[:max_blocks].to(torch.int32).to(cuda_device)
    kp = torch.full((nb, Hkv, bs, dh), NAN, dtype=torch.bfloat16, device=cuda_device)
    vp = kp.clone()
    ctx_p = StackContext(B=1, T=Lp, pos=pos[:Lp], seqlens=None)
    stack.layer_forward(w, x[:Lp].contiguous(), ctx_p, save=True, save_gu=False)
    ops.kv_prefill_paged(ctx_p.saved.pop().qkv, kp, vp, table, Lp, Hq, Hkv, dh)
    ctx_s = StackContext(B=1, T=S, pos=pos[Lp:], seqlens=None)
    got = stack.layer_forward(w, x[Lp:].contiguous(), ctx_s, save=False, save_gu=False,
                              paged=PagedPrefill(kp, vp, table, Lp))
    torch.cuda.synchronize()
    assert _same_bits(got, want[Lp:]), "suffix layer output differs from the whole-prompt prefill"
    kd = torch.empty(1, Hkv, T, dh, dtype=torch.bfloat16, device=cuda_device)
    vd = torch.empty_like(kd)
    ops.kv_prefill(qkv_full, kd, vd, 1, T, Hq, Hkv, dh)
    tl = table.long()
    for name, pool, dref in (("K", kp, kd), ("V", vp, vd)):
        logical = pool[tl].transpose(0, 1).reshape(Hkv, max_blocks * bs, dh)[:, :T]
        assert _same_bits(logical, dref[0]), f"{name} of some position differs from the whole-prompt prefill"


# ------------------------------------------------------------------------------------------------ server
def _model():
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, make_weights(TINY), num_image_tokens=NTOK)
    model.eval()
    return model


def _emb(model, g, P):
    return model.get_model().embed_tokens(torch.randint(0, 128000, (P,), generator=g).cuda())


def _server(model, **kw):
    from metamorph_b200.engine.serve import ContinuousBatcher
    args = dict(max_slots=3, max_context=160, max_new_tokens=40, poll_every=3)
    args.update(kw)
    return ContinuousBatcher(model, **args)


def _traffic(model, n, seed, s_max=20):
    """(suffix embeddings, submit kwargs): greedy, sampled and forced requests with image runs. The first suffix has one
    row, so on a block-aligned prefix it is admitted with nothing to prefill (P - 1 == Ls)."""
    from metamorph_b200.engine.sampling import SamplingParams
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        S = 1 if i == 0 else int(torch.randint(1, s_max + 1, (1,), generator=g))
        n_new = int(torch.randint(0, 40, (1,), generator=g))
        kw = dict(max_new_tokens=n_new)
        if i % 3 == 0:                                                 # forced with an image run
            f = torch.randint(0, 128000, (n_new + 1,), generator=g).to(torch.int32)
            f[min(2, n_new)] = START
            kw["forced_tokens"] = f
        elif i % 3 == 1:                                               # sampled, images forced into it
            f = torch.full((n_new + 1,), -1, dtype=torch.int32)
            f[min(1, n_new)] = START
            kw.update(forced_tokens=f, sampling=SamplingParams(temperature=0.9, top_k=40, top_p=0.9, seed=i))
        reqs.append((_emb(model, g, S), kw))
    return reqs


def _serve(srv, reqs, prefix=None):
    """reqs: (suffix, kwargs, prefix handle or None). Whole prompts when `prefix` maps handles to embeddings."""
    rids = []
    for e, kw, h in reqs:
        if prefix is not None:
            rids.append(srv.submit(torch.cat([prefix[h], e]) if h is not None else e, **kw))
        else:
            rids.append(srv.submit(e, prefix=h, **kw))
    res = srv.run_until_idle()
    return [res[r] for r in rids]


def _assert_same(got, want, what):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a[0].cpu().tolist() == b[0].cpu().tolist(), f"{what}: request {i} ids differ"
        assert _same_bits(a[1], b[1]), f"{what}: request {i} visual embeddings differ"


def _assert_whole_pool(srv):
    a = srv.alloc
    assert sorted(a.free) == list(range(a.num_blocks)) and not a.owned and not a.shared and not a.prefix_of
    assert (srv.table == a.scratch).all()


@pytest.mark.parametrize("bs,Lp", [(16, 32), (16, 37), (64, 64), (64, 90)])
def test_cached_server_equals_uncached_and_dense_servers(cuda_device, bs, Lp):
    model = _model()
    g = torch.Generator().manual_seed(Lp)
    pre = _emb(model, g, Lp)
    traffic = _traffic(model, 12, seed=bs + Lp)
    kw = dict(kv_pool_tokens=3 * 160, kv_block_size=bs)
    dense = _serve(_server(model), [(e, k, "p") for e, k in traffic], prefix={"p": pre})
    uncached = _serve(_server(model, **kw), [(e, k, "p") for e, k in traffic], prefix={"p": pre})
    _assert_same(uncached, dense, "uncached paged against dense")
    srv = _server(model, **kw)
    h = srv.cache_prefix(pre)
    assert h.shared_len == Lp // bs * bs and h.tail.shape[0] == Lp % bs
    cached = _serve(srv, [(e, k, h) for e, k in traffic])
    _assert_same(cached, dense, f"cached bs={bs} Lp={Lp}")
    assert any(b[1].shape[0] > 0 for b in dense), "no request produced visual embeddings"
    srv.drop_prefix(h)
    _assert_whole_pool(srv)


def test_two_prefixes_and_unprefixed_requests_share_one_server(cuda_device):
    model = _model()
    g = torch.Generator().manual_seed(2)
    pres = {"a": _emb(model, g, 48), "b": _emb(model, g, 21)}
    traffic = _traffic(model, 15, seed=5)
    names = ["a", "b", None]
    mixed = [(e, k, names[i % 3]) for i, (e, k) in enumerate(traffic)]
    dense = _serve(_server(model, max_slots=4), mixed, prefix=pres)
    srv = _server(model, max_slots=4, kv_pool_tokens=4 * 160, kv_block_size=16)
    hs = {n: srv.cache_prefix(p) for n, p in pres.items()}
    cached = _serve(srv, [(e, k, hs[n] if n else None) for e, k, n in mixed])
    _assert_same(cached, dense, "two prefixes")
    for h in hs.values():
        srv.drop_prefix(h)
    _assert_whole_pool(srv)


def test_forty_slots_share_one_prefix_and_never_write_it(cuda_device):
    """40 requests run at once on one prefix; the shared blocks' bits are unchanged after every request, frozen finished
    slots included, has been served."""
    model = _model()
    g = torch.Generator().manual_seed(40)
    pre = _emb(model, g, 80)
    traffic = _traffic(model, 60, seed=40)
    dense = _serve(_server(model, max_slots=40), [(e, k, "p") for e, k in traffic], prefix={"p": pre})
    srv = _server(model, max_slots=40, kv_pool_tokens=40 * 80, kv_block_size=16)
    h = srv.cache_prefix(pre)
    shared = torch.tensor(srv.alloc.shared[h.pid], dtype=torch.long, device=srv.kc.device)
    snap_k, snap_v = srv.kc[:, shared].clone(), srv.vc[:, shared].clone()
    occupancy = []
    step = srv._device_step

    def watched():
        occupancy.append(sum(s is not None for s in srv.slots))
        step()
    srv._device_step = watched
    cached = _serve(srv, [(e, k, h) for e, k in traffic])
    _assert_same(cached, dense, "40 slots")
    assert max(occupancy) == 40, f"at most {max(occupancy)} slots ran at once"
    assert _same_bits(srv.kc[:, shared], snap_k) and _same_bits(srv.vc[:, shared], snap_v), "a shared block was written"
    srv.drop_prefix(h)
    _assert_whole_pool(srv)


def test_drop_while_queued_and_running_and_fifo_under_pool_pressure(cuda_device):
    """A pool that holds the prefix and about two requests: requests wait for blocks in submission order, the prefix
    is dropped while some of its requests run and others are queued, and its blocks come back only after the last."""
    model = _model()
    g = torch.Generator().manual_seed(9)
    pre = _emb(model, g, 40)
    traffic = _traffic(model, 10, seed=9)
    dense = _serve(_server(model, max_slots=4), [(e, k, "p") for e, k in traffic], prefix={"p": pre})
    srv = _server(model, max_slots=4, kv_pool_tokens=12 * 16, kv_block_size=16)
    h = srv.cache_prefix(pre)
    a = srv.alloc
    shared = list(a.shared[h.pid])
    order = []
    admit = srv._admit

    def logged(req, b):
        order.append(req.rid)
        admit(req, b)
    srv._admit = logged
    waited = []
    step = srv._device_step

    def watched():                                 # after the admissions of a round: a free slot beside a queue
        waited.append(any(s is None for s in srv.slots) and bool(srv.queue))
        step()
    srv._device_step = watched
    rids = [srv.submit(e, prefix=h, **k) for e, k in traffic]
    res, dropped_at = {}, None
    for rid, kind, payload in srv.run():
        if dropped_at is None and any(s is not None for s in srv.slots) and srv.queue:
            srv.drop_prefix(h)
            dropped_at = (len(res), len(srv.queue))
            assert a.shared[h.pid] == shared, "the blocks went back while requests still use them"
        if kind == "done":
            res[rid] = payload
            if h.pid in a.shared:
                assert not set(shared) & set(a.free)
    assert dropped_at is not None and dropped_at[1] > 0, "the prefix was not dropped with requests queued"
    assert any(waited), "no request ever waited for blocks beside a free slot"
    assert order == rids
    _assert_same([res[r] for r in rids], dense, "drop under pressure")
    _assert_whole_pool(srv)
