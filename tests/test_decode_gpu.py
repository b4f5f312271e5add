"""Decode kernels on H100 against torch fp32 restatements: skinny GEMM epilogues, split-context attention
with RoPE + cache append, two-stage argmax, batched state machine vs the oracle loop."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _close(a, b, rel, what):
    a, b = a.float(), b.float()
    err = (a - b).abs().max().item()
    scale = b.abs().max().item() + 1e-6
    assert err <= rel * scale, f"{what}: max_err={err:.5f} scale={scale:.4f}"


@pytest.mark.parametrize("m", [1, 5, 8, 12, 16, 27, 32])
def test_skinny_gemm(cuda_device, m):
    from metamorph_b200 import ops
    from metamorph_b200.engine.packing import interleave_gate_up
    torch.manual_seed(0)
    K, N = 4096, 1184
    x = torch.randn(m, K, device=cuda_device).bfloat16()
    w = (torch.randn(N, K, device=cuda_device) * 0.03).bfloat16()
    bias = torch.randn(N, device=cuda_device).bfloat16()
    res = torch.randn(m, N, device=cuda_device).bfloat16()
    base = x.float() @ w.float().t()
    _close(ops.skinny_gemm(x, w), base, 1e-2, "store")
    _close(ops.skinny_gemm(x, w, bias=bias, epilogue=ops.SK_BIAS), base + bias.float(), 1e-2, "bias")
    _close(ops.skinny_gemm(x, w, bias=bias, epilogue=ops.SK_BIAS_GELU), F.gelu(base + bias.float()), 1e-2, "gelu")
    _close(ops.skinny_gemm(x, w, resid=res, epilogue=ops.SK_RESID), base + res.float(), 1e-2, "resid")
    out32 = torch.empty(m, N, device=cuda_device, dtype=torch.float32)
    ops.skinny_gemm(x, w, out=out32)
    _close(out32, base, 2e-3, "fp32 out")
    wg = (torch.randn(512, K, device=cuda_device) * 0.03).bfloat16()
    wu = (torch.randn(512, K, device=cuda_device) * 0.03).bfloat16()
    act = ops.skinny_gemm(x, interleave_gate_up(wg, wu), epilogue=ops.SK_SWIGLU)
    _close(act, F.silu(x.float() @ wg.float().t()) * (x.float() @ wu.float().t()), 1e-2, "swiglu")
    if m > 8:
        # more sequences = more n8 tiles of the same MMA: a sequence's result does not depend on who shares the step
        assert torch.equal(ops.skinny_gemm(x, w)[3:7], ops.skinny_gemm(x[3:7].contiguous(), w))
        assert torch.equal(act[m - 2:], ops.skinny_gemm(x[m - 2:].contiguous(), interleave_gate_up(wg, wu), epilogue=ops.SK_SWIGLU))


def test_skinny_gemm_batch32_wide_outputs(cuda_device):
    """32 sequences x wide outputs (gate/up, lm_head shapes) take the 64-row weight slabs: ragged N (out-of-bounds rows of
    the last slab) and the SwiGLU pairing of two [16 gate | 16 up] groups per slab."""
    from metamorph_b200 import ops
    from metamorph_b200.engine.packing import interleave_gate_up
    torch.manual_seed(1)
    K = 1024
    x = torch.randn(32, K, device=cuda_device).bfloat16()
    for N in (19001, 19072):
        w = (torch.randn(N, K, device=cuda_device) * 0.03).bfloat16()
        out32 = torch.empty(32, N, device=cuda_device, dtype=torch.float32)
        ops.skinny_gemm(x, w, out=out32)
        _close(out32, x.float() @ w.float().t(), 2e-3, f"fp32 out N={N}")
        assert torch.equal(ops.skinny_gemm(x, w)[9:14], ops.skinny_gemm(x[9:14].contiguous(), w))
    wg = (torch.randn(9536, K, device=cuda_device) * 0.03).bfloat16()
    wu = (torch.randn(9536, K, device=cuda_device) * 0.03).bfloat16()
    act = ops.skinny_gemm(x, interleave_gate_up(wg, wu), epilogue=ops.SK_SWIGLU)
    _close(act, F.silu(x.float() @ wg.float().t()) * (x.float() @ wu.float().t()), 1e-2, "swiglu 64-row slabs")
    assert torch.equal(act[:8], ops.skinny_gemm(x[:8].contiguous(), interleave_gate_up(wg, wu), epilogue=ops.SK_SWIGLU))


@pytest.mark.parametrize("splits", [1, 3, 5])
def test_decode_attention_split_context(cuda_device, splits):
    from metamorph_b200 import ops
    torch.manual_seed(1)
    B, Hq, Hkv, d, Tmax = 3, 8, 2, 128, 300
    pos = torch.tensor([0, 57, 299], device=cuda_device, dtype=torch.int32)
    kc = torch.randn(B, Hkv, Tmax, d, device=cuda_device).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, d, device=cuda_device).bfloat16()
    qkv = torch.randn(B, (Hq + 2 * Hkv) * d, device=cuda_device).bfloat16()
    inv = 1.0 / (500000.0 ** (torch.arange(0, d, 2, device=cuda_device).float() / d))
    ang = torch.arange(Tmax + 1, device=cuda_device).float()[:, None] * inv[None]
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    kc0, vc0 = kc.clone(), vc.clone()
    out = ops.decode_attn(qkv, kc, vc, pos, cos, sin, Hq, Hkv, d, 1 / math.sqrt(d), splits=splits)

    def rope(x, p):
        c, s = cos[p], sin[p]
        x1, x2 = x[..., :d // 2], x[..., d // 2:]
        return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)

    for b in range(B):
        p = int(pos[b])
        q = rope(qkv[b, :Hq * d].float().view(Hq, d), p).bfloat16().float()
        kn = rope(qkv[b, Hq * d:(Hq + Hkv) * d].float().view(Hkv, d), p).bfloat16()
        vn = qkv[b, (Hq + Hkv) * d:].view(Hkv, d)
        assert torch.equal(kc[b, :, p], kn) and torch.equal(vc[b, :, p], vn), "new k/v must be appended"
        assert torch.equal(kc[b, :, :p], kc0[b, :, :p]) and torch.equal(vc[b, :, p + 1:], vc0[b, :, p + 1:])
        K = kc[b, :, :p + 1].float().repeat_interleave(Hq // Hkv, 0)
        V = vc[b, :, :p + 1].float().repeat_interleave(Hq // Hkv, 0)
        s = torch.einsum("hd,hpd->hp", q, K) / math.sqrt(d)
        ref = torch.einsum("hp,hpd->hd", s.softmax(-1), V).reshape(-1)
        _close(out[b], ref, 2e-2, f"decode attn b={b}")


def test_argmax_two_stage(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(2)
    V, ld = 128258, 128264
    buf = torch.randn(8, ld, device=cuda_device)
    buf[3, 77] = 100.0
    buf[3, 99999] = 100.0   # tie -> smallest index
    assert ops.argmax_rows(buf, V).long().equal(buf[:, :V].argmax(-1)) or int(ops.argmax_rows(buf, V)[3]) == 77
    assert int(ops.argmax_rows(buf, V)[3]) == 77


@pytest.mark.parametrize("B", [4, 20])
def test_batched_decode_matches_single_sequence_runs(cuda_device, B):
    """Batched decode (per-sequence device state machines, ragged prompts; 20 sequences = three n8 batch tiles of the
    weight-streaming GEMM) must reproduce each sequence decoded alone (teacher-forced schedule so that bf16 argmax ties
    cannot make the runs diverge)."""
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, make_weights(TINY), num_image_tokens=4)
    model.eval()
    g = torch.Generator().manual_seed(5)
    P, steps = 10, 14
    lens = torch.cat([torch.tensor([10, 7, 9, 4]), torch.randint(3, P + 1, (B - 4,), generator=g)]).to(torch.int32)
    prompts = torch.randint(0, 128000, (B, P), generator=g)
    forced = torch.randint(0, 128000, (B, steps + 2), generator=g).to(torch.int32)
    forced[0, 2] = 128256; forced[0, 9] = 128257          # image in sequence 0
    forced[2, 0] = 128256                                    # image right away in sequence 2
    forced[3, 6] = 128009                                    # EOS stops sequence 3 early
    emb = model.get_model().embed_tokens(prompts.cuda())
    for b in range(B):
        emb[b, int(lens[b]):] = 0
    ids, imgs = model.greedy_decode(None, None, emb, max_new_tokens=steps - 1, output_image=True,
                                    prompt_lens=lens, forced_tokens=forced)
    for b in range(B):
        eb = emb[b:b + 1, :int(lens[b])].contiguous()
        i1, im1 = model.greedy_decode(None, None, eb, max_new_tokens=steps - 1, output_image=True,
                                      forced_tokens=forced[b:b + 1])
        assert ids[b].cpu().tolist() == i1[0].cpu().tolist(), f"ids differ for sequence {b}"
        assert imgs[b].shape[0] == (im1.shape[0] if im1.dim() == 2 else 0)
        if imgs[b].shape[0]:
            _close(imgs[b], im1, 3e-2, f"image embeds seq {b}")
    assert ids[3].cpu().tolist()[-1] == 128009 and len(ids[3]) == 7
    assert imgs[0].shape[0] == 4 and imgs[2].shape[0] == 4 and imgs[1].shape[0] == 0


def test_engine_cuda_graph_replay_matches_stream_launches(cuda_device):
    """The decode step is captured once and replayed (all per-step state lives on the device): graph replay must emit
    exactly what plain stream launches emit — same ids (teacher-forced schedule with image blocks), same embeddings."""
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, make_weights(TINY), num_image_tokens=4)
    model.eval()
    g = torch.Generator().manual_seed(11)
    B, P, steps = 3, 9, 16
    prompts = torch.randint(0, 128000, (B, P), generator=g)
    forced = torch.randint(0, 128000, (B, steps + 2), generator=g).to(torch.int32)
    forced[0, 1] = 128256; forced[0, 8] = 128257
    forced[1, 5] = 128256
    emb = model.get_model().embed_tokens(prompts.cuda())
    outs = {}
    for use_graph in (False, True):
        model._decode.use_cuda_graph = use_graph
        outs[use_graph] = model.greedy_decode(None, None, emb, max_new_tokens=steps - 1, output_image=True,
                                              forced_tokens=forced)
        assert model._decode.last_timing["cuda_graph"] == use_graph
    model._decode.use_cuda_graph = True
    for b in range(B):
        assert outs[True][0][b].cpu().tolist() == outs[False][0][b].cpu().tolist()
        assert outs[True][1][b].shape == outs[False][1][b].shape
        if outs[True][1][b].shape[0]:
            assert torch.equal(outs[True][1][b], outs[False][1][b])


def test_continuous_batching_matches_single_request_decodes(cuda_device):
    """SURVEY §8f N4: requests streamed through 2 slots (queueing, slot reuse, admission between steps, per-slot output
    limits, mixed teacher-forced / free-running sequences) must each reproduce their own stand-alone greedy_decode."""
    from metamorph_b200.engine.serve import ContinuousBatcher
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, make_weights(TINY), num_image_tokens=4)
    model.eval()
    g = torch.Generator().manual_seed(17)
    specs = [(10, 14), (7, 9), (3, 20), (9, 6), (4, 12), (12, 5)]          # (prompt positions, max_new_tokens)
    reqs = []
    for i, (P, n_new) in enumerate(specs):
        prompt = torch.randint(0, 128000, (1, P), generator=g)
        forced = torch.randint(0, 128000, (n_new + 2,), generator=g).to(torch.int32)
        if i == 0:
            forced[2] = 128256; forced[9] = 128257
        if i == 2:
            forced[0] = 128256; forced[7] = 128256
        if i == 3:
            forced[3] = 128009                                              # EOS ends request 3 early
        reqs.append((model.get_model().embed_tokens(prompt.cuda()), n_new, forced))
    srv = ContinuousBatcher(model, max_slots=2, max_context=64, max_new_tokens=24, poll_every=3)
    rids = [srv.submit(e, max_new_tokens=n, forced_tokens=f) for e, n, f in reqs]
    free_rid = srv.submit(reqs[1][0], max_new_tokens=5)                     # a free-running request in the mix
    results, streamed = {}, {}
    for rid, kind, payload in srv.run():
        if kind == "done":
            results[rid] = payload
        else:
            streamed.setdefault((rid, kind), []).append(payload)
    assert set(results) == set(rids) | {free_rid}
    for rid, (emb, n_new, forced) in zip(rids, reqs):
        ids1, img1 = model.greedy_decode(None, None, emb, max_new_tokens=n_new, output_image=True,
                                         forced_tokens=forced.reshape(1, -1))
        ids, img = results[rid]
        assert ids.cpu().tolist() == ids1[0].cpu().tolist(), f"request {rid}: ids differ"
        n1 = img1.shape[0] if img1.dim() == 2 else 0
        assert img.shape[0] == n1, f"request {rid}: {img.shape[0]} vs {n1} visual embeddings"
        if n1:
            _close(img, img1, 3e-2, f"request {rid} image embeds")
        # the streamed chunks are the same data, in order
        cat = torch.cat(streamed.get((rid, "ids"), [torch.empty(0, dtype=torch.int32, device="cuda")]))
        assert cat.cpu().tolist() == ids.cpu().tolist()
    ids_f, img_f = results[free_rid]
    assert 1 <= ids_f.numel() + img_f.shape[0] <= 6
    assert results[rids[3]][0].cpu().tolist()[-1] == 128009 and results[rids[3]][0].numel() == 4


@pytest.mark.parametrize("quirk", ["q1", "q2"])
def test_served_request_matches_reference_golden(cuda_device, quirk):
    """SURVEY section 8f N4 pinned to the REFERENCE (not to the product's own greedy_decode): a request served by the
    continuous batcher next to an unrelated one must reproduce, free-running, the token ids and visual embeddings of the
    reference's generate() stored by oracle/make_golden_decode_quirks.py."""
    import os
    from metamorph_b200.engine.serve import ContinuousBatcher
    from oracle.weights import TINY, make_weights, with_sparse_lm_head
    from tests.helpers import build_product_model
    d = torch.load(os.path.join(os.path.dirname(__file__), "golden", "greedy_decode_quirks.pt"), weights_only=False)[quirk]
    model = build_product_model(TINY, with_sparse_lm_head(make_weights(TINY), d["live_rows"])[0],
                                num_image_tokens=d["num_image_tokens"])
    model.eval()
    srv = ContinuousBatcher(model, max_slots=2, max_context=64, max_new_tokens=24, poll_every=3,
                            start_image_token_id=d["start_image_token_id"], end_image_token_id=d["end_image_token_id"],
                            eos_token_id=list(d["eos_token_id"]))
    g = torch.Generator().manual_seed(5)
    other = model.get_model().embed_tokens(torch.randint(0, 128000, (1, 9), generator=g).cuda())
    rid_other = srv.submit(other, max_new_tokens=20)
    rid = srv.submit(model.get_model().embed_tokens(d["prompt"].cuda()), max_new_tokens=d["max_new_tokens"])
    results = {r: payload for r, kind, payload in srv.run() if kind == "done"}
    assert set(results) == {rid, rid_other}
    ids, img = results[rid]
    assert ids.cpu().tolist() == [int(t) for t in d["ids"]]
    assert tuple(img.shape) == tuple(d["image_embeds"].shape)
    torch.testing.assert_close(img.float().cpu(), d["image_embeds"], rtol=0, atol=1e-2)
