"""FP8 (E4M3) KV cache on the H100: the kernels against the row rule of oracle/kv_fp8.py and against the bf16 kernels on
the dequantised cache, bit for bit, then the layer, the decode engine and the continuous batcher (DESIGN.md §1).

Attention: the FP8 kernels must give the bf16 kernels' output bits on a bf16 cache holding x-hat. For the appended
position that needs the bf16 kernel's own k-hat to be an x-hat, so these cases use RoPE tables of quarter turns (cos, sin
in {(1, 0), (0, 1), (-1, 0), (0, -1)}: the rotation is exact) and new k / v rows that are already dequantised rows. The
append itself is checked with the engine's tables against the quantisation of the bf16 kernel's k-hat. Cache rows past
pos hold NaN bytes and NaN scales, so a read past the context shows."""
import numpy as np
import pytest
import torch

from oracle.kv_fp8 import E_MAX, quantise_rows
from tests.test_decode_attn_exact_gpu import check_out, decode_ref, split_edge_pos
from tests.test_kv_fp8 import edge_rows
from tests.test_rowwise_exact_gpu import _tables

pytestmark = pytest.mark.gpu

D = 128
NAN = float("nan")


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _same_x(a, b):
    """bf16 x-hats: the same bits, or NaN in both (the NaN payload of a dequantised 0x7f row is not part of the rule)."""
    return a.shape == b.shape and bool(((_bits(a) == _bits(b)) | (torch.isnan(a) & torch.isnan(b))).all())


# ------------------------------------------------------------------------------------------------ the row rule on torch
def _pow2(e):
    return ((e.to(torch.int32) + 127) << 23).view(torch.float32)


def quant(x):
    """The row rule on the device: x [..., 128] (bf16 values) -> (bytes uint8, scale fp32 [...], x-hat bf16)."""
    xf = x.float()
    a = xf.abs().amax(-1)
    bad = ~torch.isfinite(xf).all(-1)
    m, E = torch.frexp(a)
    e = torch.where(m <= 0.875, E - 9, E - 8).clamp(min=-124)
    e = torch.where((a == 0) | bad, torch.zeros_like(e), e)
    y = torch.where(bad[..., None], torch.zeros_like(xf), xf * _pow2(-e)[..., None])
    q = y.to(torch.float8_e4m3fn).view(torch.uint8)
    q = torch.where((e[..., None] == E_MAX) & ((q & 0x7F) == 0x78), (q & 0x80) | 0x77, q)
    q = torch.where(bad[..., None], torch.full_like(q, 0x7F), q)
    sc = _pow2(e)
    return q, sc, dequant(q, sc)


def dequant(q, sc):
    return (q.view(torch.float8_e4m3fn).float() * sc[..., None]).bfloat16()


def test_device_rule_equals_the_oracle(cuda_device):
    rows = np.stack(list(edge_rows().values()))
    g = np.random.default_rng(1)
    rnd = torch.tensor(g.standard_normal((64, D)) * np.ldexp(1.0, g.integers(-126, 125, (64, 1)))).bfloat16().double()
    rows = np.concatenate([rows, rnd.numpy()])
    q, sc, xh = quant(torch.tensor(rows).bfloat16().to(cuda_device))
    oq, osc, oxh = quantise_rows(torch.tensor(rows).bfloat16().double().numpy())
    assert np.array_equal(q.cpu().numpy(), oq) and np.array_equal(sc.cpu().numpy(), osc)
    assert np.array_equal(xh.double().cpu().numpy(), oxh, equal_nan=True)


# ------------------------------------------------------------------------------------------------ inputs
def quarter_tables(Tmax, dev, seed):
    r = torch.randint(0, 4, (Tmax, D // 2), generator=torch.Generator().manual_seed(seed))
    cos = torch.tensor([1.0, 0.0, -1.0, 0.0])[r]
    sin = torch.tensor([0.0, 1.0, 0.0, -1.0])[r]
    return cos.to(dev), sin.to(dev)


def fp8_case(B, G, Hkv, Tmax, pos_l, dev, seed, exp_lo=-8, exp_hi=8, edges=False):
    """qkv whose new k / v rows are x-hats, and an FP8 cache (bytes, scales) of random rows, V rows scaled by
    2^[exp_lo, exp_hi] per row, with NaN bytes and scales past pos. Returns qkv, kq, vq, ks, vs, pos, Hq."""
    Hq = G * Hkv
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(B, Hq + 2 * Hkv, D, generator=g)
    rows[:, Hq:] = quant(rows[:, Hq:].bfloat16())[2].float()
    if edges:                                                   # edge rows of the rule as new v rows
        ed = torch.tensor(np.stack([r for r in edge_rows().values()
                                    if np.isfinite(r).all() and np.abs(r).max() < 2.0 ** 64])).bfloat16()
        for b in range(B):
            rows[b, Hq + Hkv] = quant(ed[b % ed.shape[0]])[2].float()
    qkv = rows.reshape(B, -1).bfloat16().to(dev)
    caches = []
    for lo, hi in ((-8, 8), (exp_lo, exp_hi)):
        c = torch.randn(B, Hkv, Tmax, D, generator=g) * torch.pow(
            2.0, torch.randint(lo, hi + 1, (B, Hkv, Tmax, 1), generator=g).float())
        q, sc, _ = quant(c.bfloat16().to(dev))
        for b, p in enumerate(pos_l):
            q[b, :, p + 1:] = 0x7F
            sc[b, :, p + 1:] = NAN
        caches += [q, sc]
    kq, ks, vq, vs = caches
    return qkv, kq, vq, ks, vs, torch.tensor(pos_l, dtype=torch.int32, device=dev), Hq


def pool_of(c, table, nb, fill):
    """Scatter a dense logical cache [B, Hkv, Tmax, *rest] into nb blocks through table [B, max_blocks]."""
    B, Hkv, Tmax = c.shape[:3]
    mb = table.shape[1]
    bs = Tmax // mb
    pool = torch.full((nb, Hkv, bs) + tuple(c.shape[3:]), fill, dtype=c.dtype, device=c.device)
    for b in range(B):
        pool[table[b].long()] = c[b].reshape(Hkv, mb, bs, *c.shape[3:]).transpose(0, 1)
    return pool


def run_both(qkv, kq, vq, ks, vs, pos, cos, sin, Hq, Hkv, S, what, bs_list=(), fp64=True, seed=0):
    """FP8 dense (and paged at each block size) against the bf16 kernel on the dequantised cache: output bits, the
    appended bytes and scales, every other byte unchanged; the output also against fp64 (decode_ref)."""
    from metamorph_b200 import ops
    B = qkv.shape[0]
    kd, vd = dequant(kq, ks), dequant(vq, vs)
    k1, v1, ks1, vs1 = kq.clone(), vq.clone(), ks.clone(), vs.clone()
    out = ops.decode_attn_fp8(qkv, k1, v1, ks1, vs1, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=S)
    kb, vb = kd.clone(), vd.clone()
    want = ops.decode_attn(qkv, kb, vb, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=S)
    torch.cuda.synchronize()
    assert _same_bits(out, want), f"{what}: FP8 output differs from the bf16 kernel on the dequantised cache"
    b = torch.arange(B, device=qkv.device)
    pl = pos.long()
    wk, wv, wks, wvs = kq.clone(), vq.clone(), ks.clone(), vs.clone()
    qk, sk, _ = quant(kb[b, :, pl])
    qv, sv, _ = quant(vb[b, :, pl])
    wk[b, :, pl], wks[b, :, pl], wv[b, :, pl], wvs[b, :, pl] = qk, sk, qv, sv
    for name, got, exp in (("K bytes", k1, wk), ("V bytes", v1, wv), ("K scales", ks1, wks), ("V scales", vs1, wvs)):
        assert _same_bits(got, exp), f"{what}: {name}: the appended row is wrong or another row changed"
    if fp64:
        ref, err, _, _ = decode_ref(qkv, kd, vd, pos, cos, sin, Hq, Hkv, D ** -0.5, S)
        check_out(out, ref, err, what)
    Tmax = kq.shape[2]
    for bs in bs_list:
        mb = Tmax // bs
        nb = B * mb + 3
        table = torch.randperm(nb, generator=torch.Generator().manual_seed(seed + bs))[:B * mb].view(B, mb)
        table = table.to(torch.int32).to(qkv.device)
        kp, vp = pool_of(kq, table, nb, 0x7F), pool_of(vq, table, nb, 0x7F)
        ksp, vsp = pool_of(ks, table, nb, NAN), pool_of(vs, table, nb, NAN)
        outp = ops.decode_attn_paged_fp8(qkv, kp, vp, ksp, vsp, table, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=S)
        torch.cuda.synchronize()
        assert _same_bits(outp, out), f"{what} paged bs={bs}: output differs from the dense FP8 kernel"
        for name, got, exp, fill in (("K", kp, k1, 0x7F), ("V", vp, v1, 0x7F), ("K scales", ksp, ks1, NAN),
                                     ("V scales", vsp, vs1, NAN)):
            assert _same_bits(got, pool_of(exp, table, nb, fill)), f"{what} paged bs={bs}: {name} pool differs"
    return out


# ------------------------------------------------------------------------------------------------ attention bits
@pytest.mark.parametrize("S", [1, 2, 3, 7, 16])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_fp8_attention_equals_bf16_on_the_dequantised_cache(cuda_device, G, S):
    Tmax = 1024
    pos_l = split_edge_pos(S, Tmax)
    qkv, kq, vq, ks, vs, pos, Hq = fp8_case(len(pos_l), G, 2, Tmax, pos_l, cuda_device, seed=10 * G + S, edges=True)
    cos, sin = quarter_tables(Tmax, cuda_device, S)
    run_both(qkv, kq, vq, ks, vs, pos, cos, sin, Hq, 2, S, f"G={G} S={S}", bs_list=(16, 64, 256), seed=S)


@pytest.mark.parametrize("lo,hi", [(-124, -110), (100, 118), (-124, 118)])
def test_fp8_attention_at_small_and_large_scales(cuda_device, lo, hi):
    """V rows whose e sits at the clamp, near the top of the range, and both mixed."""
    Tmax = 512
    pos_l = [0, 5, 100, 511]
    qkv, kq, vq, ks, vs, pos, Hq = fp8_case(4, 4, 2, Tmax, pos_l, cuda_device, seed=lo & 0xFF, exp_lo=lo, exp_hi=hi)
    cos, sin = quarter_tables(Tmax, cuda_device, 3)
    run_both(qkv, kq, vq, ks, vs, pos, cos, sin, Hq, 2, 4, f"e in [{lo}, {hi}]", bs_list=(32,), fp64=False)


@pytest.mark.parametrize("B", [1, 33, 128])
def test_fp8_attention_llama_heads_default_split(cuda_device, B):
    from metamorph_b200.ops import _decode_attn_splits
    Tmax = 256
    g = torch.Generator().manual_seed(B)
    pos_l = torch.randint(0, Tmax, (B,), generator=g).tolist()
    qkv, kq, vq, ks, vs, pos, Hq = fp8_case(B, 4, 8, Tmax, pos_l, cuda_device, seed=B)
    cos, sin = quarter_tables(Tmax, cuda_device, B)
    S = _decode_attn_splits(B, 8, cuda_device)
    run_both(qkv, kq, vq, ks, vs, pos, cos, sin, Hq, 8, S, f"B={B}", bs_list=(64,), fp64=(B <= 33))


def test_fp8_attention_4096_positions_in_one_split(cuda_device):
    Tmax = 4096
    qkv, kq, vq, ks, vs, pos, Hq = fp8_case(2, 4, 2, Tmax, [0, Tmax - 1], cuda_device, seed=5)
    cos, sin = quarter_tables(Tmax, cuda_device, 5)
    run_both(qkv, kq, vq, ks, vs, pos, cos, sin, Hq, 2, 1, "4096 positions", bs_list=(128,))


@pytest.mark.parametrize("G", [1, 4, 8])
def test_fp8_append_quantises_the_bf16_kernels_k_hat(cuda_device, G):
    """Engine RoPE tables, random new rows with the rule's edge rows planted in them: the FP8 kernel appends the
    quantisation of exactly the k-hat and v the bf16 kernel appends, dense and paged."""
    from metamorph_b200 import ops
    Tmax, Hkv = 256, 2
    ed = [torch.tensor(r).bfloat16() for r in edge_rows().values()]
    B = len(ed)
    Hq = G * Hkv
    g = torch.Generator().manual_seed(G)
    rows = torch.randn(B, Hq + 2 * Hkv, D, generator=g).bfloat16()
    for b in range(B):
        rows[b, Hq + Hkv + (b % Hkv)] = ed[b]                              # v rows: the edge rows themselves
        rows[b, Hq + (b % Hkv), :D // 2] = ed[b][:D // 2]                  # k rows: half an edge row before RoPE
    qkv = rows.reshape(B, -1).to(cuda_device)
    pos = torch.randint(0, Tmax, (B,), generator=g).to(torch.int32).to(cuda_device)
    cos, sin = _tables(D, Tmax, cuda_device, round_bf16=True)
    kb = torch.zeros(B, Hkv, Tmax, D, dtype=torch.bfloat16, device=cuda_device)
    vb = kb.clone()
    ops.decode_attn(qkv, kb, vb, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=2)
    kq = torch.zeros(B, Hkv, Tmax, D, dtype=torch.uint8, device=cuda_device)
    vq = kq.clone()
    ks = torch.zeros(B, Hkv, Tmax, dtype=torch.float32, device=cuda_device)
    vs = ks.clone()
    ops.decode_attn_fp8(qkv, kq, vq, ks, vs, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=2)
    mb = Tmax // 16
    table = torch.randperm(B * mb, generator=g).view(B, mb).to(torch.int32).to(cuda_device)
    kp = torch.zeros(B * mb, Hkv, 16, D, dtype=torch.uint8, device=cuda_device)
    vp = kp.clone()
    ksp = torch.zeros(B * mb, Hkv, 16, dtype=torch.float32, device=cuda_device)
    vsp = ksp.clone()
    ops.decode_attn_paged_fp8(qkv, kp, vp, ksp, vsp, table, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=2)
    torch.cuda.synchronize()
    b = torch.arange(B, device=cuda_device)
    pl = pos.long()
    for name, src, byt, sc, pb, ps in (("K", kb, kq, ks, kp, ksp), ("V", vb, vq, vs, vp, vsp)):
        wq, wsc, _ = quant(src[b, :, pl])
        assert _same_bits(byt[b, :, pl], wq) and _same_bits(sc[b, :, pl], wsc), f"G={G}: appended {name} row"
        assert _same_bits(pool_of(byt, table, B * mb, 0), pb), f"G={G}: paged {name} bytes"
        assert _same_bits(pool_of(sc, table, B * mb, 0.0), ps), f"G={G}: paged {name} scales"
    assert bool((vq[b, b % Hkv, pl] == 0x7F).any()), "no NaN row reached the append"


# ------------------------------------------------------------------------------------------------ prefill and staging
@pytest.mark.parametrize("paged_bs", [None, 16, 64])
def test_quant_prefill_bytes_and_write_back(cuda_device, paged_bs):
    from metamorph_b200 import ops
    Hq, Hkv, T = 8, 2, 77                                     # T not a multiple of the block size
    B = 1 if paged_bs else 3
    g = torch.Generator().manual_seed(paged_bs or 1)
    qkv = (torch.randn(B * T, (Hq + 2 * Hkv) * D + 64, generator=g) * 3).bfloat16().to(cuda_device)[:, :-64]
    ed = [torch.tensor(r).bfloat16() for r in edge_rows().values()]
    for i, r in enumerate(ed):                                # the edge rows inside real rows, K and V
        qkv[(7 * i) % (B * T), (Hq + i % (2 * Hkv)) * D:(Hq + i % (2 * Hkv) + 1) * D] = r.to(cuda_device)
    before = qkv.clone()
    kv = before[:, Hq * D:].reshape(B, T, 2, Hkv, D)
    wq, wsc, wxh = quant(kv)                                  # [B, T, 2, Hkv, ...]
    if paged_bs is None:
        Tmax = 96
        kq = torch.full((B, Hkv, Tmax, D), 0x7F, dtype=torch.uint8, device=cuda_device)
        vq = kq.clone()
        ks = torch.full((B, Hkv, Tmax), NAN, device=cuda_device)
        vs = ks.clone()
        ops.kv_quant_prefill(qkv, kq, vq, ks, vs, B, T, Hq, Hkv, D)
        lk, lv, lks, lvs = kq[:, :, :T], vq[:, :, :T], ks[:, :, :T], vs[:, :, :T]
        assert bool((kq[:, :, T:] == 0x7F).all()) and bool(torch.isnan(vs[:, :, T:]).all()), "wrote past T"
    else:
        mb = -(-T // paged_bs) + 1
        nb = mb + 2
        table = torch.randperm(nb, generator=g)[:mb].to(torch.int32).to(cuda_device)
        kq = torch.full((nb, Hkv, paged_bs, D), 0x7F, dtype=torch.uint8, device=cuda_device)
        vq = kq.clone()
        ks = torch.full((nb, Hkv, paged_bs), NAN, device=cuda_device)
        vs = ks.clone()
        ops.kv_quant_prefill_paged(qkv, kq, vq, ks, vs, table, T, Hq, Hkv, D)
        tl = table.long()

        def logical(p):
            return p[tl].transpose(0, 1).reshape(Hkv, mb * paged_bs, *p.shape[3:])[None, :, :T]
        lk, lv, lks, lvs = logical(kq), logical(vq), logical(ks), logical(vs)
    torch.cuda.synchronize()
    for name, got, exp in (("K bytes", lk, wq[:, :, 0].transpose(1, 2)), ("V bytes", lv, wq[:, :, 1].transpose(1, 2)),
                           ("K scales", lks, wsc[:, :, 0].transpose(1, 2)),
                           ("V scales", lvs, wsc[:, :, 1].transpose(1, 2))):
        assert _same_bits(got, exp), f"{name} differ from the rule"
    assert _same_bits(qkv[:, :Hq * D], before[:, :Hq * D]), "Q columns changed"
    assert _same_x(qkv[:, Hq * D:], wxh.reshape(B * T, -1)), "K/V columns are not x-hat"


@pytest.mark.parametrize("bs", [16, 128])
def test_dequant_paged_equals_torch(cuda_device, bs):
    from metamorph_b200 import ops
    Hkv, nb, mb = 2, 9, 6
    g = torch.Generator().manual_seed(bs)
    x = (torch.randn(nb, Hkv, bs, D, generator=g) * torch.pow(2.0, torch.randint(-124, 110, (nb, Hkv, bs, 1),
                                                                                  generator=g).float()))
    q, sc, _ = quant(x.bfloat16().to(cuda_device))
    q[0, 0, 0] = 0x7F
    sc[0, 0, 0] = 1.0
    row = torch.randperm(nb, generator=g)[:mb].to(torch.int32).to(cuda_device)
    kst = torch.full((mb, Hkv, bs, D), NAN, dtype=torch.bfloat16, device=cuda_device)
    vst = kst.clone()
    n = mb - 2
    ops.kv_dequant_paged(q, q.flip(0).contiguous(), sc, sc.flip(0).contiguous(), row, n, kst, vst)
    torch.cuda.synchronize()
    rl = row.long()[:n]
    assert _same_x(kst[:n], dequant(q, sc)[rl]) and _same_x(vst[:n], dequant(q.flip(0), sc.flip(0))[rl])
    assert bool(torch.isnan(kst[n:].float()).all()), "staging blocks past n_blocks were written"


# ------------------------------------------------------------------------------------------------ one real-width layer
@pytest.fixture(scope="module")
def real_layer():
    from oracle.weights import REAL_A, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(REAL_A, make_weights(REAL_A))
    model.eval()
    return model


@pytest.mark.parametrize("bs,Lp", [(64, 704), (128, 768)])
def test_one_layer_fp8_prefix_then_suffix_equals_the_whole_prompt(cuda_device, real_layer, bs, Lp):
    from metamorph_b200.engine.llama import FP8KVStore, StackContext
    stack = real_layer.stack
    d = stack.dims
    w = real_layer.get_model().layers[0].weights()
    S = 40
    T = Lp + S
    stack.ensure_positions(T + 1)
    gen = torch.Generator(device=cuda_device).manual_seed(bs)
    x = (torch.randn(T, d.hidden, device=cuda_device, generator=gen) * 0.5).bfloat16()
    pos = torch.arange(T, dtype=torch.int32, device=cuda_device)
    Hkv, dh = d.n_kv_heads, d.head_dim
    kd = torch.zeros(1, Hkv, T, dh, dtype=torch.uint8, device=cuda_device)
    vd = kd.clone()
    ksd = torch.zeros(1, Hkv, T, device=cuda_device)
    vsd = ksd.clone()
    want = stack.layer_forward(w, x, StackContext(B=1, T=T, pos=pos, seqlens=None), save=False, save_gu=False,
                               kv=FP8KVStore(kd, vd, ksd, vsd))
    max_blocks = -(-T // bs) + 1
    nb = max_blocks + 3
    table = torch.randperm(nb, generator=torch.Generator().manual_seed(bs))[:max_blocks].to(torch.int32).to(cuda_device)
    kp = torch.full((nb, Hkv, bs, dh), 0x7F, dtype=torch.uint8, device=cuda_device)
    vp = kp.clone()
    ksp = torch.full((nb, Hkv, bs), NAN, device=cuda_device)
    vsp = ksp.clone()
    kst = torch.full((max_blocks, Hkv, bs, dh), NAN, dtype=torch.bfloat16, device=cuda_device)
    staging = (kst, kst.clone(), torch.arange(max_blocks, dtype=torch.int32, device=cuda_device))
    Ls = Lp // bs * bs
    stack.layer_forward(w, x[:Ls].contiguous(), StackContext(B=1, T=Ls, pos=pos[:Ls], seqlens=None), save=False,
                        save_gu=False, kv=FP8KVStore(kp, vp, ksp, vsp, table))
    got = stack.layer_forward(w, x[Ls:].contiguous(), StackContext(B=1, T=T - Ls, pos=pos[Ls:], seqlens=None),
                              save=False, save_gu=False, kv=FP8KVStore(kp, vp, ksp, vsp, table, Ls, staging))
    torch.cuda.synchronize()
    assert _same_bits(got, want[Ls:]), "suffix layer output differs from the whole-prompt FP8 prefill"
    tl = table.long()
    for name, pool, dref in (("K", kp, kd), ("V", vp, vd), ("K scales", ksp, ksd), ("V scales", vsp, vsd)):
        logical = pool[tl].transpose(0, 1).reshape(Hkv, max_blocks * bs, *pool.shape[3:])[:, :T]
        assert _same_bits(logical, dref[0]), f"{name} of some position differs from the whole-prompt prefill"


# ------------------------------------------------------------------------------------------------ servers
from tests.test_prefix_cache_gpu import START, _assert_same, _assert_whole_pool, _emb, _model, _server, _serve, _traffic  # noqa: E402


def _lp_same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        if len(x) > 2 or len(y) > 2:
            for u, v in zip(x[2], y[2]):
                assert _same_bits(u, v), f"{what}: request {i} log-probabilities differ"


@pytest.mark.parametrize("bs,Lp", [(16, 37), (64, 90)])
def test_fp8_servers_dense_paged_prefixed_and_graphs_agree(cuda_device, bs, Lp):
    model = _model()
    g = torch.Generator().manual_seed(Lp)
    pre = _emb(model, g, Lp)
    traffic = _traffic(model, 12, seed=bs + Lp)
    for i in range(0, len(traffic), 4):
        traffic[i][1]["logprobs"] = 5
    whole = [(e, k, "p") for e, k in traffic]
    fp8 = dict(kv_cache_dtype="fp8_e4m3")
    kw = dict(kv_pool_tokens=3 * 160, kv_block_size=bs, **fp8)
    dense = _serve(_server(model, **fp8), whole, prefix={"p": pre})
    paged = _serve(_server(model, **kw), whole, prefix={"p": pre})
    _assert_same(paged, dense, "FP8 paged against FP8 dense")
    _lp_same(paged, dense, "FP8 paged against FP8 dense")
    eager = _serve(_server(model, use_cuda_graph=False, **kw), whole, prefix={"p": pre})
    _assert_same(eager, dense, "FP8 stream launches against graph replay")
    _lp_same(eager, dense, "FP8 stream launches against graph replay")
    srv = _server(model, **kw)
    srv.alloc.free.reverse()
    h = srv.cache_prefix(pre)
    cached = _serve(srv, [(e, k, h) for e, k in traffic])
    _assert_same(cached, dense, f"FP8 prefixed bs={bs} Lp={Lp} against the whole prompt")
    _lp_same(cached, dense, "FP8 prefixed against the whole prompt")
    assert srv.sampled_graph is not None and srv.lp_graphs
    srv.drop_prefix(h)
    _assert_whole_pool(srv)
    bf16 = _serve(_server(model), whole, prefix={"p": pre})
    assert any(a[0].tolist() != b[0].tolist() or not _same_bits(a[1], b[1]) for a, b in zip(dense, bf16)), \
        "FP8 requests returned the bf16 server's bits everywhere: is the FP8 cache in use?"


def test_fp8_request_alone_equals_among_127_neighbours(cuda_device):
    model = _model()
    traffic = _traffic(model, 128, seed=9, s_max=12)
    kw = dict(max_slots=128, max_context=96, kv_pool_tokens=128 * 96, kv_block_size=16, kv_cache_dtype="fp8_e4m3")
    crowd = _serve(_server(model, **kw), [(e, k, None) for e, k in traffic])
    for i in (0, 1, 2, 77):
        alone = _serve(_server(model, **kw), [(traffic[i][0], traffic[i][1], None)])
        _assert_same(alone, [crowd[i]], f"request {i} alone against among 127 neighbours")


def test_fp8_and_bf16_servers_on_one_model_do_not_interact(cuda_device):
    model = _model()
    traffic = [(e, k, None) for e, k in _traffic(model, 8, seed=3)]
    bf16_first = _serve(_server(model), traffic)
    fp8_srv = _server(model, kv_pool_tokens=3 * 160, kv_block_size=16, kv_cache_dtype="fp8_e4m3")
    bf16_srv = _server(model)
    assert bf16_srv.scales is None and bf16_srv.kc.dtype == torch.bfloat16 and bf16_srv.staging is None
    fp8_a = _serve(fp8_srv, traffic)
    bf16_again = _serve(bf16_srv, traffic)
    fp8_b = _serve(fp8_srv, traffic)
    _assert_same(bf16_again, bf16_first, "bf16 server beside an FP8 server")
    _assert_same(fp8_b, fp8_a, "FP8 server beside a bf16 server")
    assert bf16_srv.graph is not None and bf16_srv.kc.dtype == torch.bfloat16


def test_fp8_pool_sizes_follow_the_formula(cuda_device):
    model = _model()
    d = model.stack.dims
    L = len(model.get_model().layers)
    srv = _server(model, kv_pool_tokens=1000, kv_block_size=16, kv_cache_dtype="fp8_e4m3")
    nb = -(-1000 // 16) + 1
    for t in (srv.kc, srv.vc):
        assert t.dtype == torch.uint8 and t.shape == (L, nb, d.n_kv_heads, 16, d.head_dim)
    for t in srv.scales:
        assert t.dtype == torch.float32 and t.shape == (L, nb, d.n_kv_heads, 16)
    per_pos = 2 * L * d.n_kv_heads * (d.head_dim + 4)
    got = sum(t.numel() * t.element_size() for t in (srv.kc, srv.vc, *srv.scales))
    assert got == nb * 16 * per_pos
    assert srv.staging[0].shape == (srv.max_blocks, d.n_kv_heads, 16, d.head_dim)
    dense = _server(model, kv_cache_dtype="fp8_e4m3")
    assert dense.kc.shape == (L, 3, d.n_kv_heads, 160, d.head_dim) and dense.scales[0].shape == (L, 3, d.n_kv_heads, 160)


def test_fp8_decode_engine_graph_eager_and_greedy_decode_agree(cuda_device):
    """DecodeEngine.generate(kv_cache_dtype='fp8_e4m3'): graph replay gives the stream launches' bits, greedy_decode
    passes the argument through, and the FP8 cache changes the bits."""
    from metamorph_b200.engine.decode import DecodeEngine
    model = _model()
    g = torch.Generator().manual_seed(8)
    emb = torch.stack([_emb(model, g, 20) for _ in range(3)])
    forced = torch.full((3, 31), -1, dtype=torch.int32)
    forced[:, 2] = START
    kw = dict(max_new_tokens=30, forced_tokens=forced, kv_cache_dtype="fp8_e4m3")
    graph = model._decode.generate(emb, **kw)
    eager_engine = DecodeEngine(model)
    eager_engine.use_cuda_graph = False
    eager = eager_engine.generate(emb, **kw)
    ids, imgs = model.greedy_decode(None, None, emb, max_new_tokens=30, forced_tokens=forced, output_image=True,
                                    kv_cache_dtype="fp8_e4m3")
    bf16 = model._decode.generate(emb, max_new_tokens=30, forced_tokens=forced)
    for b in range(3):
        _assert_same([(eager[0][b], eager[1][b]), (ids[b], imgs[b])], [(graph[0][b], graph[1][b])] * 2,
                     f"DecodeEngine row {b}")
    assert any(graph[1][b].shape[0] > 0 for b in range(3))
    assert any(not _same_bits(graph[1][b], bf16[1][b]) for b in range(3)), "FP8 gave the bf16 cache's bits"
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        model._decode.generate(emb, max_new_tokens=2, kv_cache_dtype="fp8")
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        model.generate(torch.zeros(1, 4, dtype=torch.long), max_new_tokens=2, kv_cache_dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        _server(model, kv_cache_dtype="e5m2")
