"""The paged KV cache on the H100: `decode_attn_paged` / `kv_prefill_paged` against the dense kernels bit for bit, and
a paged `ContinuousBatcher` against a dense one with the same slots, request for request, including a pool too small
for every slot at once and the reclaim of a finished slot's blocks while that slot keeps running frozen.

Bits are compared as int16 views, so a NaN sentinel or poison compares as bits, not as a float."""
import os

import pytest
import torch

from oracle.decode_state import DecodeConfig, run_forced

pytestmark = pytest.mark.gpu

START, END, EOS = 128256, 128257, (128001, 128009)
NTOK = 4
SENTINEL = -3.5


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ kernels
def _rope_tables(n, dev):
    ang = torch.rand(n, 64, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) * 6.0
    return ang.cos().contiguous(), ang.sin().contiguous()


def _kernel_case(B, G, bs, max_blocks, splits, scratch_rows=(), Hkv=2, pos_list=None, seed=0):
    from metamorph_b200 import ops
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(seed)
    Hq, dh, Tmax = G * Hkv, 128, max_blocks * bs
    qkv = torch.randn(B, (Hq + 2 * Hkv) * dh, device=dev, generator=gen).bfloat16()
    kd = torch.randn(B, Hkv, Tmax, dh, device=dev, generator=gen).bfloat16()
    vd = torch.randn(B, Hkv, Tmax, dh, device=dev, generator=gen).bfloat16()
    edges = [0, bs - 1, bs, bs + 1, Tmax - 1] if pos_list is None else pos_list
    rnd = torch.randint(0, Tmax, (B,), generator=torch.Generator().manual_seed(seed)).tolist()
    pos_h = [edges[b] if b < len(edges) else rnd[b] for b in range(B)]
    for b in scratch_rows:
        pos_h[b] = 0                              # an idle slot: position 0 of the scratch block, nothing else
    pos = torch.tensor(pos_h, dtype=torch.int32, device=dev)
    cos, sin = _rope_tables(Tmax + 1, dev)
    # pool: every slot's blocks through a random permutation, a few spare blocks, the scratch block last
    live = [b for b in range(B) if b not in scratch_rows]
    nb = len(live) * max_blocks + 3
    scratch = nb
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed + 1))
    table_h = torch.full((B, max_blocks), scratch, dtype=torch.int32)
    for i, b in enumerate(live):
        table_h[b] = perm[i * max_blocks:(i + 1) * max_blocks].to(torch.int32)
    table = table_h.to(dev)
    kp = torch.full((nb + 1, Hkv, bs, dh), SENTINEL, dtype=torch.bfloat16, device=dev)
    vp = kp.clone()
    for b in live:                                # scatter the logical cache into its blocks
        blocks = table_h[b].long().to(dev)
        kp[blocks] = kd[b].reshape(Hkv, max_blocks, bs, dh).transpose(0, 1)
        vp[blocks] = vd[b].reshape(Hkv, max_blocks, bs, dh).transpose(0, 1)
    kp0, vp0 = kp.clone(), vp.clone()
    scale = dh ** -0.5
    out_d = ops.decode_attn(qkv, kd, vd, pos, cos, sin, Hq, Hkv, dh, scale, splits=splits)
    out_p = ops.decode_attn_paged(qkv, kp, vp, table, pos, cos, sin, Hq, Hkv, dh, scale, splits=splits)
    torch.cuda.synchronize()
    assert _same_bits(out_d, out_p), f"attention output differs (B={B} G={G} bs={bs} splits={splits})"
    # the appended K/V at its pool row, every other byte as it was
    want_k, want_v = kp0.clone(), vp0.clone()
    for b in live:
        p = pos_h[b]
        blk = int(table_h[b, p // bs])
        want_k[blk, :, p % bs] = kd[b, :, p]
        want_v[blk, :, p % bs] = vd[b, :, p]
    if scratch_rows:                              # idle rows race on scratch row 0: each element is one of their appends
        got_k, got_v = kp[scratch, :, 0], vp[scratch, :, 0]
        rows = list(scratch_rows)
        assert (_bits(kd[rows, :, 0]) == _bits(got_k)[None]).any(0).all()
        assert (_bits(vd[rows, :, 0]) == _bits(got_v)[None]).any(0).all()
        want_k[scratch, :, 0], want_v[scratch, :, 0] = got_k, got_v
    assert _same_bits(kp, want_k), "K pool: wrong append or a stray write"
    assert _same_bits(vp, want_v), "V pool: wrong append or a stray write"


@pytest.mark.parametrize("bs,max_blocks", [(16, 20), (64, 6), (256, 3)])
@pytest.mark.parametrize("splits", [1, 3, 16])
def test_paged_attention_equals_dense_at_block_and_chunk_edges(cuda_device, bs, max_blocks, splits):
    _kernel_case(B=33, G=4, bs=bs, max_blocks=max_blocks, splits=splits, scratch_rows=(7, 20, 31), seed=bs + splits)


@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_paged_attention_equals_dense_for_every_gqa_group(cuda_device, G):
    _kernel_case(B=9, G=G, bs=64, max_blocks=5, splits=3, scratch_rows=(8,), seed=G)


@pytest.mark.parametrize("B", [1, 33, 128])
def test_paged_attention_equals_dense_across_batch_sizes(cuda_device, B):
    scratch = () if B == 1 else tuple(range(5, B, max(1, B // 6)))
    _kernel_case(B=B, G=4, bs=16, max_blocks=9, splits=None if B == 128 else 16, scratch_rows=scratch, seed=100 + B)


def test_paged_attention_at_4096_positions_in_one_split(cuda_device):
    """The largest shared-memory case: a 4096-position logical context in one CTA per (sequence, kv head)."""
    _kernel_case(B=3, G=8, bs=64, max_blocks=64, splits=1, Hkv=8, pos_list=[4095, 4032, 63], seed=9)


@pytest.mark.parametrize("bs", [16, 64])
@pytest.mark.parametrize("T_kind", ["one", "ragged", "full"])
def test_paged_prefill_copies_the_dense_bits(cuda_device, bs, T_kind):
    from metamorph_b200 import ops
    dev = torch.device("cuda")
    Hq, Hkv, dh, max_blocks = 8, 2, 128, 5
    Tmax = max_blocks * bs
    T = {"one": 1, "ragged": 2 * bs + 5, "full": Tmax}[T_kind]
    gen = torch.Generator(device=dev).manual_seed(bs)
    qkv = torch.randn(T, (Hq + 2 * Hkv) * dh, device=dev, generator=gen).bfloat16()
    kd = torch.full((1, Hkv, Tmax, dh), SENTINEL, dtype=torch.bfloat16, device=dev)
    vd = kd.clone()
    ops.kv_prefill(qkv, kd, vd, 1, T, Hq, Hkv, dh)
    nb = 2 * max_blocks + 1
    table = torch.randperm(nb, generator=torch.Generator().manual_seed(bs))[:max_blocks].to(torch.int32).to(dev)
    kp = torch.full((nb, Hkv, bs, dh), SENTINEL, dtype=torch.bfloat16, device=dev)
    vp = kp.clone()
    ops.kv_prefill_paged(qkv, kp, vp, table, T, Hq, Hkv, dh)
    torch.cuda.synchronize()
    want_k = torch.full_like(kp, SENTINEL)
    want_v = want_k.clone()
    blocks = table.long()
    want_k[blocks] = kd[0].reshape(Hkv, max_blocks, bs, dh).transpose(0, 1)
    want_v[blocks] = vd[0].reshape(Hkv, max_blocks, bs, dh).transpose(0, 1)
    assert _same_bits(kp, want_k) and _same_bits(vp, want_v)
    assert not _same_bits(kd[0, :, :T], torch.full_like(kd[0, :, :T], SENTINEL))


# ------------------------------------------------------------------------------------------------ server
def _model(weights=None, ntok=NTOK):
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, weights if weights is not None else make_weights(TINY), num_image_tokens=ntok)
    model.eval()
    return model


def _emb(model, g, P):
    return model.get_model().embed_tokens(torch.randint(0, 128000, (1, P), generator=g).cuda())


def _schedule(g, n, **at):
    f = torch.randint(0, 128000, (n,), generator=g).to(torch.int32)
    for i, t in at.items():
        f[int(i)] = t
    return f


def _server(model, **kw):
    from metamorph_b200.engine.serve import ContinuousBatcher
    args = dict(max_slots=2, max_context=96, max_new_tokens=40, poll_every=3)
    args.update(kw)
    return ContinuousBatcher(model, **args)


def _traffic(model, n, seed):
    """Greedy, sampled and forced requests with image runs, prompts and lengths of every size the server takes."""
    from metamorph_b200.engine.sampling import SamplingParams
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        P = int(torch.randint(1, 40, (1,), generator=g))
        n_new = int(torch.randint(0, 40, (1,), generator=g))
        kind = i % 3
        kw = dict(max_new_tokens=n_new)
        if kind == 0:                                            # forced with an image run
            kw["forced_tokens"] = _schedule(g, n_new + 1, **{str(min(2, n_new)): START})
        elif kind == 1:                                          # sampled, images forced into it
            f = torch.full((n_new + 1,), -1, dtype=torch.int32)
            f[min(1, n_new)] = START
            kw.update(forced_tokens=f, sampling=SamplingParams(temperature=0.9, top_k=40, top_p=0.9, seed=i))
        else:                                                    # free-running greedy
            pass
        reqs.append((_emb(model, g, P), kw))
    return reqs


def _serve(srv, reqs):
    rids = [srv.submit(e, **kw) for e, kw in reqs]
    res = srv.run_until_idle()
    return [res[r] for r in rids]


def _assert_same(got, want, what):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a[0].cpu().tolist() == b[0].cpu().tolist(), f"{what}: request {i} ids differ"
        assert _same_bits(a[1], b[1]), f"{what}: request {i} visual embeddings differ"


@pytest.mark.parametrize("slots", [2, 40])
@pytest.mark.parametrize("bs", [16, 64])
def test_paged_server_equals_dense_server(cuda_device, slots, bs):
    model = _model()
    reqs = _traffic(model, 12 if slots == 2 else 50, seed=slots + bs)
    dense = _serve(_server(model, max_slots=slots), reqs)
    srv = _server(model, max_slots=slots, kv_pool_tokens=slots * 96, kv_block_size=bs)
    paged = _serve(srv, reqs)
    _assert_same(paged, dense, f"slots={slots} bs={bs}")
    assert sorted(srv.alloc.free) == list(range(srv.alloc.num_blocks)) and not srv.alloc.owned
    assert (srv.table == srv.alloc.scratch).all()
    assert any(b[1].shape[0] > 0 for b in dense), "no request produced visual embeddings"


@pytest.mark.parametrize("quirk", ["q1", "q2"])
def test_paged_server_serves_the_reference_free_run(cuda_device, quirk):
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "greedy_decode_quirks.pt"), weights_only=False)[quirk]
    model = _model(with_sparse_lm_head(make_weights(TINY), d["live_rows"])[0], d["num_image_tokens"])
    kw = dict(start_image_token_id=d["start_image_token_id"], end_image_token_id=d["end_image_token_id"],
              eos_token_id=list(d["eos_token_id"]))
    emb = model.get_model().embed_tokens(d["prompt"].cuda())
    P, n = emb.reshape(-1, emb.shape[-1]).shape[0], d["max_new_tokens"]
    srv = _server(model, max_context=P + n + 2, max_new_tokens=n, kv_pool_tokens=P + n + 1, kv_block_size=16, **kw)
    rid = srv.submit(emb, max_new_tokens=n)
    ids, img = srv.run_until_idle()[rid]
    assert ids.cpu().tolist() == [int(t) for t in d["ids"]]
    torch.testing.assert_close(img.float().cpu(), d["image_embeds"], rtol=0, atol=1e-2)


def test_oversubscribed_pool_waits_for_blocks_in_fifo_order(cuda_device):
    model = _model()
    slots, ctx = 6, 96
    reqs = _traffic(model, 24, seed=3)
    dense = _serve(_server(model, max_slots=slots, max_context=ctx), reqs)
    srv = _server(model, max_slots=slots, max_context=ctx, kv_pool_tokens=2 * ctx, kv_block_size=16)
    assert srv.alloc.num_blocks * 16 < slots * ctx
    order, waited = [], []
    admit = srv._admit

    def logged(req, b):
        order.append(req.rid)
        admit(req, b)
    srv._admit = logged
    step = srv._device_step

    def watched():
        free_slot = any(s is None for s in srv.slots)
        waited.append(free_slot and bool(srv.queue))
        step()
    srv._device_step = watched
    paged = _serve(srv, reqs)
    _assert_same(paged, dense, "oversubscribed")
    assert order == sorted(order) == list(range(len(reqs)))
    assert any(waited), "no request ever waited for blocks beside a free slot"
    assert sorted(srv.alloc.free) == list(range(srv.alloc.num_blocks))


def test_reclaimed_blocks_are_never_written_by_their_frozen_slot(cuda_device):
    """slot 0 finishes first; the queue head needs the whole free pool, so slot 0 stays idle; slot 2 finishes at a
    later poll and the head is admitted into slot 0 with slot 2's blocks, its last one included, then runs long
    enough to read every block it holds. Meanwhile the finished slot 2 keeps appending at its frozen position."""
    model = _model()
    g = torch.Generator().manual_seed(21)
    bs = 16
    reqs = [  # (P, max_new, forced schedule): all fully forced
        (5, 10, _schedule(g, 11, **{"1": EOS[0]})),                       # slot 0: 1 block, done after 2 steps
        (5, 40, _schedule(g, 41, **{"3": START})),                         # slot 1: 3 blocks, runs throughout
        (20, 30, _schedule(g, 31, **{"2": START, "13": EOS[1]})),          # slot 2: 4 blocks, done after 14 steps
        (30, 45, _schedule(g, 46, **{"5": START, "20": START})),           # head: 5 blocks = the pool less slot 1's
    ]
    embs = [_emb(model, g, P) for P, _, _ in reqs]
    kws = [dict(max_new_tokens=n, forced_tokens=f) for _, n, f in reqs]
    cfg = lambda n: DecodeConfig(NTOK, n, START, END, EOS)                 # noqa: E731
    srv = _server(model, max_slots=3, max_context=80, max_new_tokens=48, poll_every=2, kv_pool_tokens=8 * bs,
                  kv_block_size=bs)
    a = srv.alloc
    assert [a.reservation(P, n) for P, n, _ in reqs] == [1, 3, 4, 5] and a.num_blocks == 8
    admitted = {}
    admit = srv._admit

    def poisoned(req, b):                          # stale blocks hold NaN when a request receives them
        free = torch.tensor(a.free, dtype=torch.long, device=srv.kc.device)
        srv.kc[:, free] = float("nan")
        srv.vc[:, free] = float("nan")
        idle = [i for i, s in enumerate(srv.slots) if s is None]
        admit(req, b)
        admitted[req.rid] = (b, list(a.owned[req.rid]), idle, srv.steps_run)
    srv._admit = poisoned
    step = srv._device_step

    def checked():                                 # before every step: idle rows are all scratch
        t = srv.table.cpu()
        for i, s in enumerate(srv.slots):
            if s is None:
                assert (t[i] == a.scratch).all(), f"idle slot {i} still points at pool blocks"
            else:
                assert sorted(t[i][t[i] != a.scratch].tolist()) == sorted(a.owned[s.rid])
        step()
    srv._device_step = checked
    rids = [srv.submit(e, **kw) for e, kw in zip(embs, kws)]
    res = srv.run_until_idle()
    slot2_blocks = admitted[rids[2]][1]
    b3, blocks3, idle_then, at_step = admitted[rids[3]]
    want2 = run_forced(reqs[2][2].tolist(), cfg(30))
    assert run_forced(reqs[0][2].tolist(), cfg(10)).total_output == 2 and want2.total_output == 14
    # slot 0 finished at the poll after step 2 and stayed idle; slot 2 finished at the poll after step 14
    assert at_step == 14 and b3 == 0 and 0 in idle_then and 2 in idle_then
    frozen = slot2_blocks[(20 + want2.total_output - 1) // bs]       # where the finished slot 2 keeps appending
    assert slot2_blocks[-1] in blocks3 and frozen in blocks3
    assert set(blocks3) == set(range(8)) - set(admitted[rids[1]][1])
    for rid, (P, n, f) in zip(rids, reqs):
        want = run_forced(f.tolist(), cfg(n))
        assert res[rid][0].cpu().tolist() == want.ids and res[rid][1].shape[0] == len(want.kept_steps)
        assert not torch.isnan(res[rid][1].float()).any()
    assert run_forced(reqs[3][2].tolist(), cfg(45)).total_output == 46     # the head read all its 5 blocks
    dense = _server(model, max_slots=3, max_context=80, max_new_tokens=48, poll_every=2)
    want = _serve(dense, list(zip(embs, kws)))
    _assert_same([res[r] for r in rids], want, "reclaim")


def test_graph_replay_and_block_placement_do_not_change_a_request(cuda_device):
    model = _model()
    reqs = _traffic(model, 9, seed=77)
    kw = dict(max_slots=3, kv_pool_tokens=3 * 96, kv_block_size=16)
    base = _serve(_server(model, **kw), reqs)
    eager = _serve(_server(model, use_cuda_graph=False, **kw), reqs)
    _assert_same(eager, base, "stream launches against graph replay")
    srv = _server(model, **kw)
    srv.alloc.free.reverse()
    _assert_same(_serve(srv, reqs), base, "free list reversed")
    srv = _server(model, **kw)
    srv.alloc.free = srv.alloc.free[1::2] + srv.alloc.free[0::2]
    _assert_same(_serve(srv, reqs), base, "free list interleaved")
    assert srv.sampled_graph is not None
