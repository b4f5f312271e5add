"""Decode attention (`decode_attn_kernel` + `decode_attn_combine_kernel`, csrc/decode.cu) against an fp64 restatement,
dense and paged, at its split, context, GQA and softmax edges (H100 only).

The kernel rounds q and the new k exactly as the reference below restates them, computes everything else in fp32 and
rounds the output once to bf16. Each output element must lie between the roundings of its fp64 value minus and plus a
bound derived from the kernel's own summation chains (`tests/exact.py` `assert_rounds_within`): bit equality away from a
rounding boundary, one of the two neighbours near one. Cache rows past `pos` hold NaN, so a read past the context shows
as a NaN output. The paged kernel must equal the dense one bit for bit on the same logical cache. Every case asserts the
regime it is meant to reach.

Schedule (decode.cu:197-407), per (kv head hk, sequence b, split sp) CTA of 256 threads:
  * n_ctx = pos + 1, chunk = ceil(n_ctx / S); split sp owns positions [sp * chunk, min(n_ctx, sp * chunk + chunk)),
    which is empty when sp * chunk >= n_ctx; it then reports m = -inf, l = 0 (:228-229, :381-384).
  * q-hat = bf16(rope(q)) through rope_lo / rope_hi (common.cuh: fma(a, c, -fl(b s)), fma(b, c, fl(a s))), then
    sq = fl(q-hat * scale) (:248-255). The owner of pos rotates k_new the same way, appends k-hat and v at pos and scores
    pos from its on-chip copies (:256-272, :279-284: a 128-term fp32 chain).
  * other positions: one thread per position, 16 groups of an 8-term expression added into s (:286-305);
  * per head: m = max, e_p = __expf(s_p - m), l = per-lane chain over positions lane, lane + 32, ... then a 5-level
    warp_sum (:313-326);
  * o = P V: warp w takes positions w, w + 8, ... (one fma chain per lane and dim), then the 8 warp partials are added
    in order (:328-380);
  * combine (:388-407): M = max_s m_s, w_s = __expf(m_s - M) (0 for an empty split), L = sum_s l_s w_s,
    acc = sum_s o_s w_s, out = bf16(acc / L).
Shared memory per CTA (:646-648): (9 G 128 + 256 + G cpad) floats, cpad = (ceil(Tmax / S) + 4) & ~3, at most 200 KB.
"""
import math

import pytest
import torch

from tests.exact import U, assert_rounds_within, expf_fast_rel, gamma, rounding_slack
from tests.test_rowwise_exact_gpu import _tables

pytestmark = pytest.mark.gpu

D = 128
NAN = float("nan")
SMEM_LIMIT = 200 * 1024


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def _bits(t):
    return t.contiguous().view(torch.int16)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ the restatement
def _rn32_of_sum(x, y):
    """fp32 round-to-nearest of the exact sum of two fp64 values. TwoSum gives r + e == x + y exactly; r truncated
    toward zero with its last bit set when e != 0 (round to odd) keeps 53 >= 24 + 2 bits, so one rounding to fp32 from
    it is the correct rounding of x + y."""
    r = x + y
    bp = r - x
    e = (x - (r - bp)) + (y - bp)
    away = (e != 0) & ((e > 0) != (r > 0))
    r = torch.where(away, torch.nextafter(r, torch.zeros_like(r)), r)
    bits = r.view(torch.int64)
    return torch.where(e != 0, bits | 1, bits).view(torch.float64).float()


def rope_f32(x, c, s):
    """rope_lo / rope_hi of the [..., 128] bf16 heads x with table rows c, s [..., 64], in fp32 exactly as the kernel
    has them: a c and b s of a bf16 and an fp32 value are exact in fp64; fl(b s) is one fp32 rounding; the fma is the
    single fp32 rounding of the exact a c - fl(b s) (and of b c + fl(a s))."""
    a, b = x[..., :D // 2].double(), x[..., D // 2:].double()
    c, s = c.double(), s.double()
    lo = _rn32_of_sum(a * c, -(b * s).float().double())
    hi = _rn32_of_sum(b * c, (a * s).float().double())
    return torch.cat([lo, hi], -1)


def rope_bf16(x, c, s):
    return rope_f32(x, c, s).bfloat16()


def split_ranges(n_ctx, S):
    chunk = -(-n_ctx // S)
    return chunk, [(sp * chunk, min(n_ctx, sp * chunk + chunk)) for sp in range(S)]


def decode_ref(qkv, kc, vc, pos, cos, sin, Hq, Hkv, scale, S):
    """fp64 decode attention of the rows of qkv [B, (Hq + 2 Hkv) * 128] (any row stride) over the dense logical cache
    kc / vc [B, Hkv, Tmax, 128] as it was before the call, and a bound on the kernel's fp32 error per output element.
    Returns (out64 [B, Hq, 128], err64, k-hat [B, Hkv, 128] bf16, stats per sequence).

    Scores: sq = fl(q-hat scale) is restated exactly, so a score's error is that of its dot-product chain:
      E_p = gamma_24 * sum_d |sq_d k_d| (8-term groups, 16 of them), gamma_129 at p = pos (one 128-term chain).
    Weights: the kernel's weight of p is __expf(fl(s^_p - m^_s)) __expf(fl(m^_s - M^)); exp(-M^) is common to the
    numerator and L and cancels, so relative to exp(s_p - M) the weight is off by at most
      eta_p = 1.01 (expm1(E_p) + u (|a1| + |a2|) + e_exp(a1) + e_exp(a2)),
    a1 = s_p - m_s, a2 = m_s - M, each widened by 2 max E (the rounded arguments; e_exp = `expf_fast_rel`).
    Sums (fp32 chains of the schedule): o with gamma_(ceil(chunk / 8) + 8) against sum_p e_p |v_p|, l with
    gamma_(ceil(chunk / 32) + 5), then the S-term combine of each (with the product by w_s: gamma_(S + 1)).
    With p_p = softmax(s)_p, P = sum_p p_p |v_p|, a = out64 and lambda = sum_p p_p eta_p + gamma_L:
      |acc / L - a| <= (sum_p p_p eta_p |v_p| + gamma_A P + |a| lambda) / (1 - lambda), times 1.01, plus u |a| for the
    division. __expf flushes results below 2^-126 to 0 (ex2.approx.ftz): the largest weight is __expf(0) w = 1, so L >= 1
    and a flushed term moves acc by at most 2^-126 |v| and L by 2^-126, for at most 2 n_ctx terms (weights and w_s):
    tiny = 4 n_ctx 2^-126 (max|v| + |a|). The bound is absolute and scales with P, so an output that cancels to near 0
    needs no rule of its own."""
    B = qkv.shape[0]
    G = Hq // Hkv
    scale32 = _f32(scale)
    rows = qkv.reshape(B, Hq + 2 * Hkv, D)
    dev = qkv.device
    out = torch.empty(B, Hkv, G, D, dtype=torch.float64, device=dev)
    err = torch.empty_like(out)
    khat = torch.empty(B, Hkv, D, dtype=torch.bfloat16, device=dev)
    stats = []
    for b in range(B):
        p = int(pos[b])
        n = p + 1
        c, s = cos[p], sin[p]
        qh = rope_bf16(rows[b, :Hq], c, s)
        kh = rope_bf16(rows[b, Hq:Hq + Hkv], c, s)
        khat[b] = kh
        sq = (qh.double() * scale32).float().double().view(Hkv, G, D)
        K = kc[b, :, :n].double()
        V = vc[b, :, :n].double()
        K[:, p] = kh.double()
        V[:, p] = rows[b, Hq + Hkv:].double()
        sc = sq @ K.transpose(1, 2)                                        # [Hkv, G, n]
        chain = torch.full((n,), 24.0, dtype=torch.float64, device=dev)
        chain[p] = 129.0
        Es = gamma(chain) * (sq.abs() @ K.abs().transpose(1, 2))
        M = sc.amax(-1, keepdim=True)
        e = torch.exp(sc - M)
        pr = e / e.sum(-1, keepdim=True)
        a = pr @ V
        Va = V.abs()
        chunk, ranges = split_ranges(n, S)
        split = (torch.arange(n, device=dev) // chunk).expand(Hkv, G, n)
        ms = torch.full((Hkv, G, S), -math.inf, dtype=torch.float64, device=dev)
        ms.scatter_reduce_(-1, split, sc, "amax")
        m_p = ms.gather(-1, split)
        wide = 2 * Es.amax(-1, keepdim=True)
        a1 = (sc - m_p).abs() + wide
        a2 = (m_p - M).abs() + wide
        eta = 1.01 * (torch.expm1(Es) + U * (a1 + a2) + expf_fast_rel(a1) + expf_fast_rel(a2))
        lam = (pr * eta).sum(-1, keepdim=True) + gamma(-(-chunk // 32) + 5 + S + 1)
        aerr = (pr * eta) @ Va + gamma(-(-chunk // 8) + 8 + S + 1) * (pr @ Va)
        tiny = 4 * n * 2.0 ** -126 * (Va.amax() + a.abs())
        out[b] = a
        err[b] = 1.01 * (aerr + a.abs() * lam) / (1 - lam) + 1.01 * U * a.abs() + tiny
        live = torch.tensor([p1 > p0 for p0, p1 in ranges], device=dev)
        stats.append({"n_ctx": n, "chunk": chunk, "n_empty": int((~live).sum()), "m_split": ms, "M": M[..., 0],
                      "live": live, "argmax": sc.argmax(-1)})
    return out.view(B, Hq, D), err.view(B, Hq, D), khat, stats


def smem_bytes(G, Tmax, S):
    cpad = (-(-Tmax // S) + 4) & ~3
    return (G * D + 2 * D + 8 * G * D + G * cpad) * 4


def tmax_limit(G, S=1):
    """The largest Tmax the launch check (decode.cu:646-648) admits."""
    t = 1
    while smem_bytes(G, t + 1, S) <= SMEM_LIMIT:
        t += 1
    return t


def check_out(out, ref, err, what):
    """The bf16 output [B, Hq * 128] against the fp64 reference; prints how many elements needed the fp32 slack."""
    got = out.view(ref.shape)
    n = assert_rounds_within(got, ref, err, what)
    n2, worst = rounding_slack(got, ref, err)
    assert n2 == n
    print(f"{what}: {n} of {got.numel()} elements needed the slack (worst at {worst:.3g} of the bound)")
    return n, worst


# ------------------------------------------------------------------------------------------------ inputs
def make_inputs(B, G, Hkv, Tmax, pos_l, dev, seed, tables="engine", v_scale=None):
    """randn qkv rows and caches; the cache row at pos holds stale values (not k-hat), rows past pos hold NaN."""
    Hq = G * Hkv
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, (Hq + 2 * Hkv) * D, generator=g).bfloat16().to(dev)
    kc = torch.randn(B, Hkv, Tmax, D, generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, D, generator=g)
    if v_scale is not None:
        vc *= torch.pow(2.0, torch.randint(-6, v_scale + 1, vc.shape, generator=g).float())
    vc = vc.bfloat16()
    for b, p in enumerate(pos_l):
        kc[b, :, p + 1:] = NAN
        vc[b, :, p + 1:] = NAN
    pos = torch.tensor(pos_l, dtype=torch.int32, device=dev)
    cos, sin = _tables(D, Tmax, dev, round_bf16=(tables == "engine"))
    return qkv, kc.to(dev), vc.to(dev), pos, cos, sin, Hq


def share_prefix(kc, vc, pos_l, L):
    """Make two sequences' logical caches equal on positions [0, L) (what prefix caching shares): (b0, b1, L), or None."""
    both = [b for b, p in enumerate(pos_l) if p >= L]
    if len(both) < 2:
        return None
    b0, b1 = both[:2]
    kc[b1, :, :L] = kc[b0, :, :L]
    vc[b1, :, :L] = vc[b0, :, :L]
    return b0, b1, L


def split_edge_pos(S, Tmax):
    """0, S - 2 (n_ctx < S: empty splits), 7 S - 1 (the chunk, 7, divides n_ctx), 7 S + 2 (it does not, S > 3), 63,
    64, 127, 128, 700 and Tmax - 1."""
    pos = [0, 63, 64, 127, 128, 7 * S - 1, 7 * S + 2, 700, Tmax - 1]
    if S >= 2:
        pos.append(S - 2)
    return pos


def split_inputs(G, S, dev, seed, tables="engine", Hkv=2, Tmax=1024):
    pos_l = split_edge_pos(S, Tmax)
    qkv, kc, vc, pos, cos, sin, Hq = make_inputs(len(pos_l), G, Hkv, Tmax, pos_l, dev, seed, tables)
    share = share_prefix(kc, vc, pos_l, 256)
    return qkv, kc, vc, pos, cos, sin, Hq, Hkv, share


def peaked_inputs(S, dev, seed, G=4, Hkv=2, Tmax=1024):
    """One sequence at pos = Tmax - 1 whose scores are planted per split (head h of a group sees them times 1 + h / 4):
    about +12 at position 0, -20 over a middle split, +16 at one position of the second-to-last split, +20 on the
    appended token and below -85 over split S - 3, whose w_s underflows; N(0, 1 / 4) elsewhere. The cache rows carry the
    plants along the rotated, scaled q of the group's first head; the appended token's k_new is the plant rotated back
    through the table row, so that the kernel's own k-hat carries it. v: random signs, magnitudes 2^-6 .. 2^10."""
    pos_l = [Tmax - 1]
    qkv, kc, vc, pos, cos, sin, Hq = make_inputs(1, G, Hkv, Tmax, pos_l, dev, seed, "engine", v_scale=10)
    g = torch.Generator().manual_seed(seed + 1)
    p = Tmax - 1
    chunk, ranges = split_ranges(Tmax, S)
    rows = qkv.view(1, Hq + 2 * Hkv, D)
    c, s = cos[p].double(), sin[p].double()
    for hk in range(Hkv):
        q0 = rows[0, hk * G].float()
        for h in range(1, G):
            rows[0, hk * G + h] = (q0 * (1 + h / 4)).bfloat16()
        u = rope_bf16(rows[0, hk * G], cos[p], sin[p]).double() * _f32(D ** -0.5)
        dirn = (u / u.dot(u)).cpu()
        t = torch.randn(Tmax, generator=g, dtype=torch.float64) * 0.5
        t[0] = 12.0
        a0, a1 = ranges[S // 2]
        t[a0:a1] = -20.0 + 0.5 * torch.rand(a1 - a0, generator=g, dtype=torch.float64)
        b0, b1 = ranges[S - 2]
        t[(b0 + b1) // 2] = 16.0
        f0, f1 = ranges[S - 3]
        t[f0:f1] = -90.0 + 4 * torch.rand(f1 - f0, generator=g, dtype=torch.float64)
        kc[0, hk, :p] = (t[:p, None] * dirn[None]).to(dev).bfloat16()
        kc[0, hk, p] = 0.0                                            # stale, not k-hat
        tgt = 20.0 * dirn.to(dev)
        lo, hi = tgt[:D // 2], tgt[D // 2:]
        rows[0, Hq + hk] = torch.cat([lo * c + hi * s, hi * c - lo * s]).bfloat16()
    return qkv, kc, vc, pos, cos, sin, Hq, Hkv


# ------------------------------------------------------------------------------------------------ running
def run_dense(qkv, kc, vc, pos, cos, sin, Hq, Hkv, S, what):
    """decode_attn on copies of the caches; checks the output against fp64, the appended row against k-hat and v, and
    every other cache byte unchanged. Returns (out, kc after, vc after, stats, (slack count, worst ratio))."""
    from metamorph_b200 import ops
    B = qkv.shape[0]
    k1, v1 = kc.clone(), vc.clone()
    out = ops.decode_attn(qkv, k1, v1, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=S)
    torch.cuda.synchronize()
    ref, err, khat, stats = decode_ref(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, S)
    slack = check_out(out, ref, err, what)
    want_k, want_v = kc.clone(), vc.clone()
    b = torch.arange(B, device=qkv.device)
    pl = pos.long()
    want_k[b, :, pl] = khat
    want_v[b, :, pl] = qkv.reshape(B, Hq + 2 * Hkv, D)[:, Hq + Hkv:]
    assert _same_bits(k1, want_k), f"{what}: K cache: the appended row is not k-hat, or another row changed"
    assert _same_bits(v1, want_v), f"{what}: V cache: the appended row is not v, or another row changed"
    return out, k1, v1, stats, slack


def to_pool(kc, table, nb):
    """Scatter the dense logical cache [B, Hkv, Tmax, 128] into a pool of nb blocks through table [B, max_blocks];
    blocks no table names hold NaN."""
    B, Hkv, Tmax, _ = kc.shape
    mb = table.shape[1]
    bs = Tmax // mb
    pool = torch.full((nb, Hkv, bs, D), NAN, dtype=kc.dtype, device=kc.device)
    for b in range(B):
        pool[table[b].long()] = kc[b].reshape(Hkv, mb, bs, D).transpose(0, 1)
    return pool


def run_paged(qkv, kc, vc, pos, cos, sin, Hq, Hkv, S, out_dense, k_after, v_after, bs, seed, share, what):
    """decode_attn_paged on a pool holding the same logical cache: every sequence's blocks through one random
    permutation (tables not monotone), three NaN blocks no table names, and with `share` = (b0, b1, L) sequence b1's
    first L / bs entries naming b0's blocks (its own become unnamed NaN blocks). The output must equal the dense
    output bit for bit and the pool must equal the dense cache after the call, scattered the same way."""
    from metamorph_b200 import ops
    B, _, Tmax, _ = kc.shape
    mb = Tmax // bs
    assert mb * bs == Tmax
    nb = B * mb + 3
    perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed))
    table = perm[:B * mb].view(B, mb).clone().to(torch.int32)
    for b in range(B):                                                  # a short table can come out sorted
        if bool((table[b, 1:] > table[b, :-1]).all()):
            table[b] = table[b].flip(0)
    if share is not None and share[2] >= bs:
        b0, b1, L = share
        table[b1, :L // bs] = table[b0, :L // bs]
    assert any(bool((table[b, 1:] < table[b, :-1]).any()) for b in range(B)), "the block tables are monotone"
    table = table.to(qkv.device)
    unnamed = torch.ones(nb, dtype=torch.bool)
    unnamed[table.long().flatten().cpu()] = False
    assert int(unnamed.sum()) >= 3
    kp, vp = to_pool(kc, table, nb), to_pool(vc, table, nb)
    out = ops.decode_attn_paged(qkv, kp, vp, table, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=S)
    torch.cuda.synchronize()
    assert _same_bits(out, out_dense), f"{what} paged bs={bs}: output differs from the dense kernel"
    assert _same_bits(kp, to_pool(k_after, table, nb)), f"{what} paged bs={bs}: K pool: wrong append or a stray write"
    assert _same_bits(vp, to_pool(v_after, table, nb)), f"{what} paged bs={bs}: V pool: wrong append or a stray write"
    assert bool(torch.isnan(kp[unnamed.to(kp.device)]).all()), f"{what} paged bs={bs}: an unnamed block was written"


# ------------------------------------------------------------------------------------------------ 1. split edges
@pytest.mark.parametrize("tables", ["engine", "fp32"])
@pytest.mark.parametrize("S", [1, 2, 3, 7, 16, 17, 63, 64])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_decode_attn_split_edges(cuda_device, G, S, tables):
    qkv, kc, vc, pos, cos, sin, Hq, Hkv, share = split_inputs(G, S, cuda_device, seed=100 * G + S, tables=tables)
    what = f"decode G={G} S={S} {tables} tables"
    out, k1, v1, stats, _ = run_dense(qkv, kc, vc, pos, cos, sin, Hq, Hkv, S, what)
    assert any(st["n_empty"] > 0 for st in stats) == (S > 1), "empty splits"
    assert any(st["n_ctx"] % st["chunk"] == 0 and st["n_ctx"] >= 2 * S for st in stats), "a chunk dividing n_ctx"
    if S > 3:
        assert any(st["n_ctx"] % st["chunk"] != 0 for st in stats), "a chunk not dividing n_ctx"
    for st in stats:
        if st["n_ctx"] >= 2 * S and S > 1:                          # split maxima differ: some w_s != 1
            m = st["m_split"][..., st["live"]]
            assert bool((m.amin(-1) < st["M"]).all())
    for bs in (16, 64, 256):
        run_paged(qkv, kc, vc, pos, cos, sin, Hq, Hkv, S, out, k1, v1, bs, seed=G * S + bs, share=share, what=what)


# ------------------------------------------------------------------------------------------------ 2. peaked softmax
@pytest.mark.parametrize("S", [8, 17, 64])
def test_decode_attn_peaked_softmax_across_splits(cuda_device, S):
    qkv, kc, vc, pos, cos, sin, Hq, Hkv = peaked_inputs(S, cuda_device, seed=S)
    what = f"decode peaked S={S}"
    out, k1, v1, stats, _ = run_dense(qkv, kc, vc, pos, cos, sin, Hq, Hkv, S, what)
    st = stats[0]
    assert st["n_empty"] == 0
    assert bool((st["argmax"] == st["n_ctx"] - 1).all()), "the appended token must carry the maximum"
    m, M = st["m_split"], st["M"][..., None]
    assert bool((m[..., 0] - M[..., 0] < -3).all()), "position 0's split must sit below the maximum"
    assert bool(((m - M) < -88).any(-1).all()), "no split's w_s underflows to 0 (__expf below 2^-126)"
    assert bool(((m - M > -80) & (m - M < -10)).any(-1).all()), "the middle split must have a small, nonzero w_s"
    assert bool((torch.unique(m[0, 0]).numel() == S)), "split maxima must all differ"
    vv = vc[0, :, :st["n_ctx"]]
    assert bool((vv < 0).any()) and bool((vv > 0).any()) and float(vv.abs().max()) >= 2.0 ** 9
    for bs in (16, 64, 256):
        run_paged(qkv, kc, vc, pos, cos, sin, Hq, Hkv, S, out, k1, v1, bs, seed=S + bs, share=None, what=what)


# ------------------------------------------------------------------------------------------------ 3. long contexts
# (G, Tmax, S, paged block size): the engine's max_pos at S = 1 (~150 KB of shared memory, the path of every batch of 33
# or more sequences at 8 KV heads on 132 SMs), the largest Tmax the check admits for G = 8 and 4, 8192 at S = 16 and 64.
LONG = [(4, 8192, 1, 256), (8, "limit", 1, 16), (4, "limit", 1, 16), (4, 8192, 16, 256), (4, 8192, 64, 256)]


@pytest.mark.parametrize("case", LONG, ids=[f"G{g}-T{t}-S{s}" for g, t, s, _ in LONG])
def test_decode_attn_long_context(cuda_device, case):
    G, Tmax, S, bs = case
    Tmax = tmax_limit(G, S) if Tmax == "limit" else Tmax
    assert tmax_limit(4) == 11583 and tmax_limit(8) == 5215 and tmax_limit(1) == 49791 and tmax_limit(2) == 24319
    smem = smem_bytes(G, Tmax, S)
    assert smem <= SMEM_LIMIT and (smem > 48 * 1024) == (S == 1)     # S = 1 needs the opt-in above 48 KB
    if (Tmax, S) == (8192, 1):
        assert 145 * 1024 < smem < 150 * 1024 + 1024
    pos_l = [Tmax - 1, 4097, 5]
    qkv, kc, vc, pos, cos, sin, Hq = make_inputs(3, G, 2, Tmax, pos_l, cuda_device, seed=Tmax + S)
    share = share_prefix(kc, vc, pos_l, 256)
    what = f"decode G={G} Tmax={Tmax} S={S} ({smem} B of shared memory)"
    out, k1, v1, stats, _ = run_dense(qkv, kc, vc, pos, cos, sin, Hq, 2, S, what)
    assert stats[0]["n_ctx"] == Tmax
    # paged: Tmax rounded down to whole blocks, which the check admits as well
    Tp = Tmax // bs * bs
    if Tp != Tmax:
        pos_p = torch.tensor([Tp - 1, 4097, 5], dtype=torch.int32, device=cuda_device)
        kp, vp = kc[:, :, :Tp].clone(), vc[:, :, :Tp].clone()
        outp, kp1, vp1, _, _ = run_dense(qkv, kp, vp, pos_p, cos, sin, Hq, 2, S, what + f" (Tmax {Tp})")
        run_paged(qkv, kp, vp, pos_p, cos, sin, Hq, 2, S, outp, kp1, vp1, bs, seed=Tp, share=share, what=what)
    else:
        run_paged(qkv, kc, vc, pos, cos, sin, Hq, 2, S, out, k1, v1, bs, seed=Tmax + S, share=share, what=what)


@pytest.mark.parametrize("G", [4, 8])
def test_decode_attn_refuses_one_position_past_the_shared_memory_limit(cuda_device, G):
    from metamorph_b200 import ops
    from metamorph_b200._lib import MetaMorphB200Error
    Tmax = tmax_limit(G) + 1
    assert smem_bytes(G, Tmax, 1) > SMEM_LIMIT >= smem_bytes(G, Tmax - 1, 1)
    qkv, kc, vc, pos, cos, sin, Hq = make_inputs(1, G, 1, Tmax, [Tmax - 1], cuda_device, seed=G)
    k0, v0 = kc.clone(), vc.clone()
    out = torch.full((1, Hq * D), NAN, dtype=torch.bfloat16, device=cuda_device)
    with pytest.raises(MetaMorphB200Error, match="too large"):
        ops.decode_attn(qkv, kc, vc, pos, cos, sin, Hq, 1, D, D ** -0.5, out=out, splits=1)
    # paged: the smallest whole number of 16-row blocks past the limit
    mb = -(-Tmax // 16)
    table = torch.arange(mb, dtype=torch.int32, device=cuda_device)[None]
    kp = torch.zeros(mb, 1, 16, D, dtype=torch.bfloat16, device=cuda_device)
    vp = kp.clone()
    with pytest.raises(MetaMorphB200Error, match="too large"):
        ops.decode_attn_paged(qkv, kp, vp, table, pos, cos, sin, Hq, 1, D, D ** -0.5, out=out, splits=1)
    torch.cuda.synchronize()
    assert _same_bits(kc, k0) and _same_bits(vc, v0), "a refused call changed the cache"
    assert bool((kp == 0).all()) and bool((vp == 0).all()), "a refused paged call changed the pool"
    assert bool(torch.isnan(out).all()), "a refused call wrote the output"


# ------------------------------------------------------------------------------------------------ 4. LLaMA dims
@pytest.mark.parametrize("B", [1, 17, 32, 33, 128])
def test_decode_attn_llama_dims_default_split(cuda_device, B):
    from metamorph_b200 import ops
    Hkv, G, Tmax = 8, 4, 1024
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    S = ops._decode_attn_splits(B, Hkv, cuda_device)
    assert S == max(1, min(16, -(-2 * sms // (B * Hkv))))
    if sms == 132:                                                   # H100 SXM
        assert S == {1: 16, 17: 2, 32: 2, 33: 1, 128: 1}[B]
    g = torch.Generator().manual_seed(B)
    pos_l = torch.randint(0, Tmax, (B,), generator=g).tolist()
    pos_l[0], pos_l[-1] = Tmax - 1, 0 if B > 1 else Tmax - 1
    qkv, kc, vc, pos, cos, sin, Hq = make_inputs(B, G, Hkv, Tmax, pos_l, cuda_device, seed=B)
    assert Hq == 32
    k1, v1 = kc.clone(), vc.clone()
    out = ops.decode_attn(qkv, k1, v1, pos, cos, sin, Hq, Hkv, D, D ** -0.5)
    ref, err, _, _ = decode_ref(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, S)
    check_out(out, ref, err, f"decode LLaMA B={B} S={S}")
    again = ops.decode_attn(qkv, k1, v1, pos, cos, sin, Hq, Hkv, D, D ** -0.5)
    assert _same_bits(again, out), "two calls gave different bits"
    for b in sorted({0, B // 2, B - 1}):
        alone = ops.decode_attn(qkv[b:b + 1], k1[b:b + 1], v1[b:b + 1], pos[b:b + 1], cos, sin, Hq, Hkv, D, D ** -0.5,
                                splits=S)
        assert _same_bits(alone, out[b:b + 1]), f"sequence {b} alone differs from its row in the batch of {B}"


# ------------------------------------------------------------------------------------------------ 5. strided operands
def test_decode_attn_strided_qkv_and_out(cuda_device):
    from metamorph_b200 import ops
    G, Hkv, Tmax, S = 4, 2, 512, 3
    pos_l = [0, 1, 300, 511]
    qkv0, kc, vc, pos, cos, sin, Hq = make_inputs(4, G, Hkv, Tmax, pos_l, cuda_device, seed=7)
    W = (Hq + 2 * Hkv) * D
    wide = torch.full((4, W + 192), NAN, dtype=torch.bfloat16, device=cuda_device)
    wide[:, 64:64 + W] = qkv0
    qkv = wide[:, 64:64 + W]
    obuf = torch.full((4, Hq * D + 256), NAN, dtype=torch.bfloat16, device=cuda_device)
    out = obuf[:, 128:128 + Hq * D]
    assert qkv.stride(0) > W and out.stride(0) > Hq * D
    k1, v1 = kc.clone(), vc.clone()
    ops.decode_attn(qkv, k1, v1, pos, cos, sin, Hq, Hkv, D, D ** -0.5, out=out, splits=S)
    ref, err, _, _ = decode_ref(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, S)
    check_out(out, ref, err, "decode strided qkv / out")
    assert bool(torch.isnan(obuf[:, :128]).all()) and bool(torch.isnan(obuf[:, 128 + Hq * D:]).all()), \
        "guard columns around out were written"
    dense = ops.decode_attn(qkv0, kc.clone(), vc.clone(), pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=S)
    assert _same_bits(out, dense), "strided operands changed the bits"
