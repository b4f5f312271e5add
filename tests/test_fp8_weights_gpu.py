"""FP8 (E4M3) weights on the H100 (DESIGN.md §1): the quantise / dequantise kernels against oracle/kv_fp8.py's rule on
the [N, K / 128, 128] group view, the FP8 weight-streaming GEMMs against the bf16 kernels on W-hat bit for bit, then
decode and the continuous batcher with weight_dtype="fp8_e4m3" against the bf16 path on a model whose five quantised
matrices hold W-hat."""
import numpy as np
import pytest
import torch

from oracle.kv_fp8 import quantise_rows
from tests.test_fp8_weights import edge_matrix

pytestmark = pytest.mark.gpu


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def _same(a, b):
    """The same bits, or NaN in both."""
    if a.shape != b.shape:
        return False
    if not a.is_floating_point():
        return torch.equal(a, b)
    return bool(((_bits(a) == _bits(b)) | (torch.isnan(a) & torch.isnan(b))).all())


# ------------------------------------------------------------------------------------------------ quantise / dequantise
def _check_against_oracle(w):
    from metamorph_b200 import ops
    N, K = w.shape
    fw = ops.weight_quant_fp8(w)
    wh = ops.weight_dequant_fp8(fw)
    torch.cuda.synchronize()
    oq, osc, owh = quantise_rows(w.double().cpu().numpy().reshape(N, K // 128, 128))
    assert np.array_equal(fw.q.cpu().numpy(), oq.reshape(N, K)), "bytes differ from the oracle"
    assert np.array_equal(fw.scale.cpu().numpy(), osc), "scales differ from the oracle"
    assert np.array_equal(wh.double().cpu().numpy(), owh.reshape(N, K), equal_nan=True), "W-hat differs from the oracle"
    return fw, wh


def test_quant_dequant_edge_groups_equal_the_oracle(cuda_device):
    _check_against_oracle(torch.tensor(edge_matrix()).bfloat16().to(cuda_device))


@pytest.mark.parametrize("N,K", [(64, 128), (37, 384), (200, 4096), (48, 14336)])
def test_quant_dequant_random_weights_equal_the_oracle(cuda_device, N, K):
    g = torch.Generator().manual_seed(N + K)
    w = torch.randn(N, K, generator=g) * torch.pow(2.0, torch.randint(-30, 30, (N, K // 128, 1), generator=g).float()
                                                   ).repeat_interleave(128, 1).reshape(N, K)
    w = w.bfloat16().to(cuda_device)
    w[0, :128] = 0
    w[1, 5] = float("nan")
    _check_against_oracle(w)


def test_quant_of_a_strided_view_and_dequant_into_a_strided_view(cuda_device):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(4)
    big = torch.randn(40, 512 + 64, generator=g).bfloat16().to(cuda_device)
    fw = ops.weight_quant_fp8(big[:, :512])
    ref = ops.weight_quant_fp8(big[:, :512].contiguous())
    assert torch.equal(fw.q, ref.q) and torch.equal(fw.scale, ref.scale)
    frame = torch.full((40, 512 + 64), 7.0, dtype=torch.bfloat16, device=cuda_device)
    ops.weight_dequant_fp8(fw, out=frame[:, 32:544])
    torch.cuda.synchronize()
    assert _same(frame[:, 32:544], ops.weight_dequant_fp8(ref))
    assert bool((frame[:, :32] == 7).all()) and bool((frame[:, 544:] == 7).all()), "dequant wrote outside its view"


# ------------------------------------------------------------------------------------------------ GEMMs
def _gemm_case(m, N, K, epi, seed, wide, out_f32=False, nan_group=False):
    """skinny_gemm on the FP8 weight against the bf16 kernel on W-hat: the same bits (NaN where NaN)."""
    from metamorph_b200 import ops
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(N, K, device=dev, generator=g) * 0.05).bfloat16()
    if nan_group:
        w[N // 3, 128:256][17] = float("nan")
    fw = ops.weight_quant_fp8(w)
    wh = ops.weight_dequant_fp8(fw)
    x = torch.randn(m, K, device=dev, generator=g).bfloat16()
    n_out = N // 2 if epi == ops.SK_SWIGLU else N
    bias = (torch.randn(N, device=dev, generator=g) * 0.1).bfloat16()
    resid = torch.randn(m, N, device=dev, generator=g).bfloat16()
    kw = dict(epilogue=epi, wide=wide)
    if epi in (ops.SK_BIAS, ops.SK_BIAS_GELU):
        kw["bias"] = bias
    if epi == ops.SK_RESID:
        kw["resid"] = resid
    outs = []
    for wt in (fw, wh):
        if out_f32:                                              # a padded fp32 ldy, as lm_head's logits
            buf = torch.full((m, (n_out + 7) // 8 * 8 + 8), -3.0, dtype=torch.float32, device=dev)
            ops.skinny_gemm(x, wt, out=buf[:, :n_out], **kw)
            outs.append(buf)
        else:
            outs.append(ops.skinny_gemm(x, wt, **kw))
    torch.cuda.synchronize()
    what = f"m={m} N={N} K={K} epi={epi} wide={wide} f32={out_f32}"
    assert _same(outs[0], outs[1]), f"{what}: FP8 output differs from the bf16 kernel on W-hat"
    if nan_group:
        assert bool(torch.isnan(outs[0].float()).any()), f"{what}: the NaN group did not reach the output"
    else:
        assert bool(torch.isfinite(outs[0].float()).all())
    if out_f32:
        assert bool((outs[0][:, n_out:] == -3.0).all()), f"{what}: wrote past N in the padded rows"


EPIS = ("SK_STORE", "SK_BIAS", "SK_RESID", "SK_BIAS_GELU", "SK_SWIGLU")


@pytest.mark.parametrize("K", [128, 384, 4096, 14336])
@pytest.mark.parametrize("m", [1, 7, 8, 9, 16, 17, 31, 32])
def test_skinny_gemm_fp8_equals_bf16_on_w_hat(cuda_device, m, K):
    from metamorph_b200 import ops
    for i, e in enumerate(EPIS):
        _gemm_case(m, 1024 if e == "SK_SWIGLU" else 1184, K, getattr(ops, e), seed=m * 7 + K + i, wide=False)
    # ragged N into a padded fp32 ldy (lm_head); at this N the 32-row (m <= 16) and 64-row (m > 16) slabs run
    _gemm_case(m, 19001, min(K, 4096), ops.SK_STORE, seed=m + K, wide=False, out_f32=True)
    _gemm_case(m, 18432, min(K, 4096), ops.SK_SWIGLU, seed=m + K + 1, wide=False)
    _gemm_case(m, 1184, K, ops.SK_STORE, seed=m + K + 2, wide=False, nan_group=K > 128)


@pytest.mark.parametrize("N,K", [(1184, 128), (1184, 384), (1184, 4096), (4096, 14336), (19001, 4096), (1024, 256)])
@pytest.mark.parametrize("m", [33, 64, 100, 128])
def test_skinny_gemm_wide_fp8_equals_bf16_on_w_hat(cuda_device, m, N, K):
    """One split (K = 128, N = 19001) and several (N = 1184 at K = 384 / 4096, N = 4096 at K = 14336)."""
    from metamorph_b200 import ops
    for i, e in enumerate(EPIS):
        if e == "SK_SWIGLU" and N % 32:
            continue
        _gemm_case(m, N, K, getattr(ops, e), seed=m * 5 + N + K + i, wide=True)
    _gemm_case(m, N, K, ops.SK_STORE, seed=m + N, wide=True, out_f32=True)
    if K > 128:
        _gemm_case(m, N, K, ops.SK_STORE, seed=m + N + 1, wide=True, nan_group=True)


def test_wide_fp8_at_narrow_batches_equals_wide_bf16(cuda_device):
    from metamorph_b200 import ops
    for m in (1, 32):
        _gemm_case(m, 1184, 4096, ops.SK_RESID, seed=m, wide=True)


# ------------------------------------------------------------------------------------------------ decode and serving
from tests.test_prefix_cache_gpu import START, _emb, _model, _serve, _server, _traffic  # noqa: E402

FP8W = dict(weight_dtype="fp8_e4m3")


@pytest.fixture(scope="module")
def models():
    """(model, its twin whose wqkv / wo / wgu / wd and lm_head hold W-hat)."""
    from metamorph_b200 import ops
    a, b = _model(), _model()
    with torch.no_grad():
        for la, lb in zip(a.get_model().layers, b.get_model().layers):
            for pa, pb in ((la.self_attn.qkv_proj, lb.self_attn.qkv_proj), (la.self_attn.o_proj, lb.self_attn.o_proj),
                           (la.mlp.gate_up_proj, lb.mlp.gate_up_proj), (la.mlp.down_proj, lb.mlp.down_proj)):
                pb.weight.data.copy_(ops.weight_dequant_fp8(ops.weight_quant_fp8(pa.weight.data)))
        b.lm_head.weight.data.copy_(ops.weight_dequant_fp8(ops.weight_quant_fp8(a.lm_head.weight.data)))
    torch.cuda.synchronize()
    return a, b


def _params(model):
    return {k: v.detach().clone() for k, v in model.state_dict().items()}


def _same_results(got, want, what):
    assert len(got) == len(want)
    for i, (x, y) in enumerate(zip(got, want)):
        assert x[0].cpu().tolist() == y[0].cpu().tolist(), f"{what}: sequence {i} ids differ"
        assert _same(x[1], y[1]), f"{what}: sequence {i} visual embeddings differ"
        if len(x) > 2 or len(y) > 2:
            for u, v in zip(x[2], y[2]):
                assert _same(u, v), f"{what}: sequence {i} log-probabilities differ"


def _per_seq(res):
    return [tuple(r[b] for r in res) for b in range(len(res[0]))]


@pytest.mark.parametrize("kv", ["bf16", "fp8_e4m3"])
@pytest.mark.parametrize("B", [3, 40])
def test_decode_engine_fp8_weights_equal_bf16_on_w_hat(cuda_device, models, B, kv):
    from metamorph_b200.engine.sampling import SamplingParams
    a, b = models
    before = _params(a)
    g = torch.Generator().manual_seed(B)
    emb = torch.stack([_emb(a, g, 20) for _ in range(B)])
    forced = torch.full((B, 31), -1, dtype=torch.int32)
    forced[::2, 2] = START
    greedy = dict(max_new_tokens=30, forced_tokens=forced, logprobs=5, kv_cache_dtype=kv)
    sampled = dict(greedy, sampling=SamplingParams(temperature=0.8, top_k=50, top_p=0.9, seed=3))
    for kw, what in ((greedy, "greedy"), (sampled, "sampled")):
        got = a._decode.generate(emb, **kw, **FP8W)
        assert a._decode.last_timing["quant_ms"] >= 0.0
        want = b._decode.generate(emb, **kw)
        _same_results(_per_seq(got), _per_seq(want), f"B={B} kv={kv} {what}")
        assert any(r[1].shape[0] > 0 for r in _per_seq(got)), "no sequence produced visual embeddings"
        plain = a._decode.generate(emb, **kw)
        assert any(not _same(x, y) for u, v in zip(got[2], plain[2]) for x, y in zip(u, v)), \
            "FP8 weights gave the bf16 weights' log-probabilities everywhere: are they in use?"
    ids, imgs, lps = a.greedy_decode(None, None, emb, max_new_tokens=30, forced_tokens=forced, output_image=True,
                                     logprobs=5, kv_cache_dtype=kv, **FP8W)
    want = b._decode.generate(emb, **greedy)
    _same_results(list(zip(ids, imgs, lps)), _per_seq(want), f"greedy_decode B={B} kv={kv}")
    after = _params(a)
    assert all(torch.equal(_bits(before[k]), _bits(after[k])) for k in before), "a bf16 parameter changed"


@pytest.mark.parametrize("kv", ["bf16", "fp8_e4m3"])
def test_servers_fp8_weights_equal_bf16_on_w_hat(cuda_device, models, kv):
    a, b = models
    before = _params(a)
    g = torch.Generator().manual_seed(17)
    pre = _emb(a, g, 37)
    traffic = _traffic(a, 12, seed=23)
    for i in range(0, len(traffic), 3):
        traffic[i][1]["logprobs"] = 5
    whole = [(e, k, "p") for e, k in traffic]
    kvd = dict(kv_cache_dtype=kv)
    paged = dict(kv_pool_tokens=3 * 160, kv_block_size=16, **kvd)
    want = _serve(_server(b, **kvd), whole, prefix={"p": pre})
    dense = _serve(_server(a, **kvd, **FP8W), whole, prefix={"p": pre})
    _same_results(dense, want, f"dense FP8-weight server kv={kv}")
    pg = _serve(_server(a, **paged, **FP8W), whole, prefix={"p": pre})
    _same_results(pg, want, f"paged FP8-weight server kv={kv}")
    srv = _server(a, **paged, **FP8W)
    h = srv.cache_prefix(pre)
    cached = _serve(srv, [(e, k, h) for e, k in traffic])
    _same_results(cached, want, f"prefix-cached FP8-weight server kv={kv}")
    # stand-alone: an FP8 DecodeEngine run of a request gives the bf16 run's bits on W-hat, and the served request
    # matches it as a bf16 server matches greedy_decode (tests/test_decode_gpu.py): the same ids on a forced schedule and
    # visual embeddings within bf16 noise (the server feeds the last prompt row through the decode step, not the prefill)
    for i in (0, 1, 2, 3):
        e, kw = traffic[i]
        prompt = torch.cat([pre, e])[None]
        f = kw.get("forced_tokens")
        args = dict(max_new_tokens=kw["max_new_tokens"], forced_tokens=None if f is None else f[None],
                    sampling=kw.get("sampling"), logprobs=kw.get("logprobs"), kv_cache_dtype=kv)
        alone = _per_seq(a._decode.generate(prompt, **args, **FP8W))
        _same_results(alone, _per_seq(b._decode.generate(prompt, **args)), f"request {i} alone kv={kv}")
        if i % 3 == 0:                                                   # fully forced
            assert cached[i][0].cpu().tolist() == alone[0][0].cpu().tolist(), f"request {i}: served ids differ"
            assert cached[i][1].shape == alone[0][1].shape
            if alone[0][1].numel():
                torch.testing.assert_close(cached[i][1].float(), alone[0][1].float(), rtol=0, atol=3e-2)
    after = _params(a)
    assert all(torch.equal(_bits(before[k]), _bits(after[k])) for k in before), "a bf16 parameter changed"


def test_batcher_at_128_slots_fp8_weights_equals_bf16_on_w_hat(cuda_device, models):
    a, b = models
    traffic = [(e, k, None) for e, k in _traffic(a, 128, seed=9, s_max=12)]
    kw = dict(max_slots=128, max_context=96, kv_pool_tokens=128 * 96, kv_block_size=16)
    _same_results(_serve(_server(a, **kw, **FP8W), traffic), _serve(_server(b, **kw), traffic), "128 slots")
