"""Flash attention (padded and packed layouts, forward and backward) and decode attention at their mask, tile and
online-softmax edges.

Two tools:
  * uniform-softmax mask probes. With q = 0 every score is 0, so the softmax is exactly uniform over the keys the mask
    allows: each allowed key gets P = 1/n and every other key exactly 0. Make one feature column of v (forward) or of dO
    (backward) one-hot at one key (query row) and the output reads the mask directly: an off-by-one causal mask, a wrong
    key-tile bound or a padded key that leaks turns an exact 0 into a non-zero value, whatever the sequence length.
  * peaked softmax: scores spanning about +-20 with dominant keys planted in the first key tile, a middle tile and the
    last key tile a row sees, so the running max both jumps late and stays put. Each result (out, lse, dQ, dK, dV) is
    held to at most twice the error of the same formula computed by torch in bf16 (bf16 operands, fp32 accumulation and
    softmax, P cast to bf16) against fp64, plus a floor stated where it is used.
"""
import pytest
import torch

from tests.exact import U, assert_equal, assert_no_worse_than, assert_within, ulp_bf16

pytestmark = pytest.mark.gpu

D = 128
BIG = 1.0e4             # finite garbage for rows outside a sequence (the kernels require those rows to be finite)
GQA = [(2, 2), (4, 2), (8, 2), (8, 1)]          # (Hq, Hkv): groups 1, 2, 4, 8


def _gid(hq_hkv):
    return f"G{hq_hkv[0] // hq_hkv[1]}"


def _split(qkv, Hq, Hkv):
    return qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]


def _bhtd(x, B, T, H):
    """[B*T, H*D] -> [B, H, T, D]"""
    return x.reshape(B, T, H, -1).transpose(1, 2)


def _allowed(lens, T, causal, device):
    """[B, 1, T, T]: key j is visible from query row i."""
    j = torch.arange(T, device=device)
    m = j[None, None, None, :] < torch.as_tensor(lens, device=device).view(-1, 1, 1, 1)
    if causal:
        m = m & (j[None, None, None, :] <= j[None, None, :, None])
    return m


def _valid_rows(lens, T, device):
    return torch.arange(T, device=device)[None, :] < torch.as_tensor(lens, device=device)[:, None]     # [B, T]


def _edges(T, L):
    e = {0, 1, 62, 63, 64, 65, 126, 127, 128, 129, 254, 255, 256, 257, T - 1, L - 1, L, L + 1}
    return sorted(x for x in e if 0 <= x < T)


# ------------------------------------------------------------------------------------------------ padded layout probes
SHAPES = {"lens=1..257-T259": (259, [1, 63, 64, 65, 127, 128, 129, 255, 257]),
          "padded-tiles-T512-L100": (512, [100, 512])}


def probe_inputs(T, lens, Hq, Hkv, device, seed):
    """Padded-layout probe data: q = 0, random k, and v column c of kv head hk (of sequence b) one-hot at key
    jkey[b, hk, c], spread over the tile edges and the sequence end. Returns (qkv [B*T, (Hq + 2 Hkv) D] bf16, jkey)."""
    B = len(lens)
    gen = torch.Generator(device=device).manual_seed(seed)
    qkv = torch.zeros(B * T, (Hq + 2 * Hkv) * D, device=device, dtype=torch.bfloat16)
    qkv[:, Hq * D:(Hq + Hkv) * D] = torch.randn(B * T, Hkv * D, device=device, generator=gen).bfloat16()
    jkey = torch.zeros(B, Hkv, D, dtype=torch.long)
    for b, L in enumerate(lens):
        e = _edges(T, L)
        for hk in range(Hkv):
            for c in range(D):
                jkey[b, hk, c] = e[(c + 5 * hk) % len(e)]
    vb = _bhtd(qkv[:, (Hq + Hkv) * D:], B, T, Hkv)          # a view: writes land in qkv
    bi, hi, ci = torch.meshgrid(torch.arange(B), torch.arange(Hkv), torch.arange(D), indexing="ij")
    vb[bi.reshape(-1), hi.reshape(-1), jkey.reshape(-1), ci.reshape(-1)] = 1.0
    return qkv, jkey.to(device)


def check_probe_fwd(o, lse, jkey, lens, T, G, causal, what):
    """o [B, Hq, T, D], lse [B, Hq, T] of the probe: on every valid row i, out[i, c] is exactly 0 where key j_c is masked
    and within one bf16 ulp of 1/n_i where it is allowed; lse = ln n_i."""
    B, Hq = o.shape[:2]
    dev = o.device
    o = o.double()
    L_b = torch.as_tensor(lens, device=dev).view(B, 1, 1, 1)
    rows = torch.arange(T, device=dev)[None, None, :, None]
    jk = jkey.repeat_interleave(G, 1)[:, :, None, :]                                           # [B, Hq, 1, D]
    n = torch.minimum(rows + 1, L_b) if causal else L_b.expand(B, 1, T, 1)
    ok = ((jk < L_b) & ((jk <= rows) if causal else True)).expand_as(o)
    want = (ok.double() / n.double()).expand_as(o)
    valid = _valid_rows(lens, T, dev)
    sel = valid[:, None, :, None].expand_as(o)
    assert_equal(o[sel & ~ok], torch.zeros_like(o[sel & ~ok]), f"{what}: masked keys")
    assert_within(o[sel & ok], want[sel & ok], ulp_bf16(want[sel & ok]), f"{what}: allowed keys")
    # lse = ln n: the running max is 0 and the sum n is exact; ln through log2 and a product by ln 2 costs a few fp32
    # roundings (u each) and an approximate log2 (<= 2 ulp): 16u relative to max(1, ln n) covers them
    ln_n = torch.log(n[..., 0].double()).expand(B, Hq, T)
    vl = valid[:, None, :].expand(B, Hq, T)
    assert_within(lse[vl], ln_n[vl], 16 * U * ln_n[vl].clamp(min=1.0), f"{what}: lse")


@pytest.mark.parametrize("hq_hkv", GQA, ids=_gid)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_padded_attention_mask_probe(cuda_device, shape, hq_hkv):
    from metamorph_b200 import ops
    T, lens = SHAPES[shape]
    Hq, Hkv = hq_hkv
    G, B = Hq // Hkv, len(lens)
    qkv, jkey = probe_inputs(T, lens, Hq, Hkv, cuda_device, seed=T * 10 + G)
    q, k, v = _split(qkv, Hq, Hkv)
    seqlens = torch.tensor(lens, device=cuda_device, dtype=torch.int32)
    valid = _valid_rows(lens, T, cuda_device)
    rows = torch.arange(T, device=cuda_device)[None, None, :, None]
    scale = D ** -0.5
    for causal in (True, False):
        out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, D, causal, scale, seqlens=seqlens)
        check_probe_fwd(_bhtd(out, B, T, Hq), lse, jkey, lens, T, G, causal, f"{shape} G={G} causal={causal}")

    # backward (causal): q = 0, dO one-hot per column at one valid row i_c, in one query head of the group only.
    # dV[j, c] = P[i_c, j] = 1/(i_c + 1) for j <= i_c and exactly 0 past i_c or L; dK = dS^T Q scale = 0 exactly.
    out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, D, True, scale, seqlens=seqlens)
    dout = torch.zeros(B * T, Hq * D, device=cuda_device, dtype=torch.bfloat16)
    db = _bhtd(dout, B, T, Hq)
    icol = torch.zeros(B, Hkv, D, dtype=torch.long)
    for b, L in enumerate(lens):
        e = [x for x in _edges(T, L) if x < L]
        for hk in range(Hkv):
            for c in range(D):
                i = e[(3 * c + hk) % len(e)]
                icol[b, hk, c] = i
                db[b, hk * G + c % G, i, c] = 1.0
    g = torch.full_like(qkv, float("nan"))
    dq, dk, dv = _split(g, Hq, Hkv)
    ops.attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, B, T, Hq, Hkv, D, scale, seqlens=seqlens)
    vrow = valid.reshape(-1)
    assert_equal(g[~vrow], torch.zeros_like(g[~vrow]), f"{shape}: gradients of padded rows")
    assert_equal(dk[vrow], torch.zeros_like(dk[vrow]), f"{shape}: dK with q = 0")
    dvb = _bhtd(dv, B, T, Hkv).double()
    ic = icol.to(cuda_device)[:, :, None, :]
    ok = rows <= ic
    want = ok.double() / (ic + 1).double()
    sel = valid[:, None, :, None].expand_as(dvb)
    wantx = want.expand_as(dvb)
    assert_equal(dvb[sel & ~ok], torch.zeros_like(dvb[sel & ~ok]), f"{shape} {_gid(hq_hkv)}: dV past the one-hot row")
    assert_within(dvb[sel & ok], wantx[sel & ok], ulp_bf16(wantx[sel & ok]), f"{shape} {_gid(hq_hkv)}: dV")


# ------------------------------------------------------------------------------------------------ packed layout probe
def test_packed_attention_mask_probe(cuda_device):
    """Segments of 129, 1, 64, 65, 128 and 300 rows at arbitrary offsets, the last ending on the buffer's last row (the
    TMA out-of-bounds path). Each segment's columns of v hold one-hot keys inside it, so a key leaking across segments
    shows as a wrong count."""
    from metamorph_b200 import ops
    Hq, Hkv = 8, 2
    G = Hq // Hkv
    segs = [(0, 129), (129, 1), (133, 64), (197, 65), (262, 128), (390, 300)]
    R = 690
    gen = torch.Generator(device=cuda_device).manual_seed(3)
    qkv = torch.zeros(R, (Hq + 2 * Hkv) * D, device=cuda_device, dtype=torch.bfloat16)
    qkv[:, Hq * D:(Hq + Hkv) * D] = torch.randn(R, Hkv * D, device=cuda_device, generator=gen).bfloat16()
    q, k, v = _split(qkv, Hq, Hkv)
    dout = torch.zeros(R, Hq * D, device=cuda_device, dtype=torch.bfloat16)
    jk, ic = {}, {}
    for s, (a, n) in enumerate(segs):
        e = [x for x in _edges(n, n) if x < n]
        for hk in range(Hkv):
            for c in range(D):
                j = e[(c + 5 * hk) % len(e)]
                jk[s, hk, c] = j
                v[a + j, hk * D + c] = 1.0
                i = e[(3 * c + hk) % len(e)]
                ic[s, hk, c] = i
                dout[a + i, (hk * G + c % G) * D + c] = 1.0
    tab = ops.SegmentTables(segs, cuda_device)
    scale = D ** -0.5
    out = torch.full((R, Hq * D), 7.0, device=cuda_device, dtype=torch.bfloat16)
    _, lse = ops.attn_fwd_varlen(q, k, v, tab, Hq, Hkv, D, scale, out=out)
    g = torch.full_like(qkv, float("nan"))
    dq, dk, dv = _split(g, Hq, Hkv)
    ops.attn_bwd_varlen(q, k, v, out, dout, lse, dq, dk, dv, tab, Hq, Hkv, D, scale)
    for s, (a, n) in enumerate(segs):
        rows = torch.arange(n, device=cuda_device)[:, None]
        o = out[a:a + n].double().view(n, Hq, D)
        j = torch.tensor([[jk[s, h // G, c] for c in range(D)] for h in range(Hq)], device=cuda_device)[None]
        ok = j <= rows[:, :, None]
        want = ok.double() / (rows[:, :, None] + 1).double()
        assert_equal(o[~ok], torch.zeros_like(o[~ok]), f"packed segment {s}: masked keys")
        assert_within(o[ok], want.expand_as(o)[ok], ulp_bf16(want.expand_as(o)[ok]), f"packed segment {s}: out")
        ln_n = torch.log((rows + 1).double()).view(1, n).expand(Hq, n)
        assert_within(lse[s, :, :n], ln_n, 16 * U * ln_n.clamp(min=1.0), f"packed segment {s}: lse")
        assert_equal(dk[a:a + n], torch.zeros_like(dk[a:a + n]), f"packed segment {s}: dK with q = 0")
        i = torch.tensor([[ic[s, hk, c] for c in range(D)] for hk in range(Hkv)], device=cuda_device)[None]
        dvs = dv[a:a + n].double().view(n, Hkv, D)
        ok = rows[:, :, None] <= i
        want = ok.double() / (i + 1).double()
        assert_equal(dvs[~ok], torch.zeros_like(dvs[~ok]), f"packed segment {s}: dV past the one-hot row")
        assert_within(dvs[ok], want.expand_as(dvs)[ok], ulp_bf16(want.expand_as(dvs)[ok]), f"packed segment {s}: dV")
    gap = torch.ones(R, dtype=torch.bool, device=cuda_device)
    for a, n in segs:
        gap[a:a + n] = False
    assert bool((out[gap] == 7.0).all()) and bool(torch.isnan(g[gap]).all()), "rows between segments were written"


# ------------------------------------------------------------------------------------------------ decode probe
@pytest.mark.parametrize("splits", [1, 3, 7, 16])
@pytest.mark.parametrize("hq_hkv", GQA, ids=_gid)
def test_decode_attention_mask_probe(cuda_device, hq_hkv, splits):
    """q = 0 survives RoPE, so out[b, h, c] = (#one-hots of column c at positions <= pos) / (pos + 1). A cache column is
    one-hot at j_c; positions past pos hold BIG and must not be read; the new v, appended at pos, is one-hot in every
    fifth column. pos covers 0, the tile edges, the last position of a split chunk (pos + 1 a multiple of the chunk) and
    Tmax - 1; splits 7 and 16 do not divide Tmax."""
    from metamorph_b200 import ops
    Hq, Hkv = hq_hkv
    G = Hq // Hkv
    Tmax = 300
    pos_l = [0, 1, 63, 64, 69, 127, 128, 200, 209, 299]
    B = len(pos_l)
    gen = torch.Generator(device=cuda_device).manual_seed(G * 100 + splits)
    kc = torch.randn(B, Hkv, Tmax, D, device=cuda_device, generator=gen).bfloat16()
    vc = torch.zeros(B, Hkv, Tmax, D, device=cuda_device, dtype=torch.bfloat16)
    e = [0, 1, 63, 64, 65, 69, 70, 127, 128, 129, 199, 200, 201, 209, 210, 298, 299]
    jc = torch.zeros(B, Hkv, D, dtype=torch.long)
    for b, p in enumerate(pos_l):
        for hk in range(Hkv):
            for c in range(D):
                jc[b, hk, c] = e[(c + 3 * hk + b) % len(e)]
                vc[b, hk, jc[b, hk, c], c] = 1.0
        vc[b, :, p + 1:] = BIG
    qkv = torch.zeros(B, (Hq + 2 * Hkv) * D, device=cuda_device, dtype=torch.bfloat16)
    qkv[:, Hq * D:(Hq + Hkv) * D] = torch.randn(B, Hkv * D, device=cuda_device, generator=gen).bfloat16()
    new_v = (torch.arange(D, device=cuda_device) % 5 == 0).bfloat16()
    qkv[:, (Hq + Hkv) * D:] = new_v.repeat(Hkv)
    pos = torch.tensor(pos_l, device=cuda_device, dtype=torch.int32)
    inv = 1.0 / (500000.0 ** (torch.arange(0, D, 2, device=cuda_device).float() / D))
    ang = torch.arange(Tmax + 1, device=cuda_device).float()[:, None] * inv[None]
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    out = ops.decode_attn(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D, D ** -0.5, splits=splits)
    p = pos.long().view(B, 1, 1)
    cnt = (jc.to(cuda_device) < p).double() + new_v.double().view(1, 1, D)      # [B, Hkv, D]
    want = (cnt / (p + 1).double()).repeat_interleave(G, 1)                     # [B, Hq, D]
    o = out.double().view(B, Hq, D)
    zero = want == 0
    assert_equal(o[zero], torch.zeros_like(o[zero]), f"decode G={G} splits={splits}: positions past pos or masked")
    assert_within(o[~zero], want[~zero], ulp_bf16(want[~zero]), f"decode G={G} splits={splits}")
    for b, pp in enumerate(pos_l):
        assert torch.equal(vc[b, :, pp], new_v.expand(Hkv, D)), "the new v must be appended at pos"


# ------------------------------------------------------------------------------------------------ peaked softmax
def _ref64(q, k, v, do, allowed, scale, G):
    """fp64 attention and its gradients. q, do [B, Hq, T, d]; k, v [B, Hkv, T, d]."""
    q, k, v = (x.double().clone().requires_grad_(True) for x in (q, k, v))
    kk, vv = k.repeat_interleave(G, 1), v.repeat_interleave(G, 1)
    s = (q @ kk.transpose(-1, -2) * scale).masked_fill(~allowed, float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = torch.exp(s - lse[..., None]) @ vv
    if do is None:
        return o.detach(), lse.detach(), None
    o.backward(do.double())
    return o.detach(), lse.detach(), (q.grad, k.grad, v.grad)


def _torch_bf16(q, k, v, do, allowed, scale, G):
    """The same formulas as torch would run them in bf16: bf16 operands, fp32 accumulation, fp32 softmax, P and dS cast
    to bf16 before their products, outputs rounded to bf16."""
    B, Hkv = k.shape[:2]
    f = lambda x: x.float()
    kk, vv = f(k).repeat_interleave(G, 1), f(v).repeat_interleave(G, 1)
    s = (f(q) @ kk.transpose(-1, -2) * scale).masked_fill(~allowed, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    pb = p.bfloat16().float()
    o = (pb @ vv).bfloat16()
    if do is None:
        return o, lse, None
    dp = f(do) @ vv.transpose(-1, -2)
    delta = (f(do) * o.float()).sum(-1, keepdim=True)
    dsb = (p * (dp - delta)).bfloat16().float()
    grp = lambda x: x.reshape(B, Hkv, G, *x.shape[2:]).sum(2)
    dq = (dsb @ kk * scale).bfloat16()
    dk = grp(dsb.transpose(-1, -2) @ f(q) * scale).bfloat16()
    dv = grp(pb.transpose(-1, -2) @ f(do)).bfloat16()
    return o, lse, (dq, dk, dv)


PEAK_T, PEAK_LENS = 523, [523, 389]


def peaked_inputs(Hq, Hkv, device, seed):
    """(qkv [B*T, (Hq + 2 Hkv) D], dO [B*T, Hq D]) in bf16, zero on rows outside the sequences: every query is 4 e + noise
    for one unit vector e, and planted keys c e score about +12 (key 5, first tile), -20 (key 140), +16 (key 263, third
    tile) and +20 (key L - 3, the last tile of the sequence)."""
    T, lens = PEAK_T, PEAK_LENS
    B, scale = len(lens), D ** -0.5
    gen = torch.Generator(device=device).manual_seed(seed)
    e = torch.randn(D, device=device, generator=gen)
    e = e / e.norm()
    qkv = 1.5 * torch.randn(B * T, (Hq + 2 * Hkv) * D, device=device, generator=gen)
    qkv[:, :Hq * D].view(B * T, Hq, D).add_(4 * e)
    kv = qkv[:, Hq * D:(Hq + Hkv) * D].view(B, T, Hkv, D)
    for b, L in enumerate(lens):
        for j, score in ((5, 12.0), (140, -20.0), (263, 16.0), (L - 3, 20.0)):
            kv[b, j] = score / (4 * scale) * e + 0.1 * kv[b, j]
    qkv = qkv.bfloat16()
    dout = torch.randn(B * T, Hq * D, device=device, generator=gen).bfloat16()
    valid = _valid_rows(lens, T, device).reshape(-1)
    qkv[~valid], dout[~valid] = 0, 0
    return qkv, dout


@pytest.mark.parametrize("hq_hkv", GQA, ids=_gid)
def test_padded_attention_peaked_softmax_and_padded_rows(cuda_device, hq_hkv):
    """Scores spanning about +-20 (peaked_inputs): rows past key 263 keep their max through the middle tiles and jump in
    the last one. T = 523 is not a multiple of 8. Rows outside a sequence then get BIG in q, k, v and dO: nothing valid
    may change, and their gradients are exactly 0."""
    from metamorph_b200 import ops
    Hq, Hkv = hq_hkv
    G = Hq // Hkv
    B, T, lens = 2, PEAK_T, PEAK_LENS
    scale = D ** -0.5
    qkv, dout = peaked_inputs(Hq, Hkv, cuda_device, seed=G)
    valid = _valid_rows(lens, T, cuda_device).reshape(-1)
    seqlens = torch.tensor(lens, device=cuda_device, dtype=torch.int32)

    def run(qkv, dout):
        q, k, v = _split(qkv, Hq, Hkv)
        out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, D, True, scale, seqlens=seqlens)
        g = torch.full_like(qkv, float("nan"))
        dq, dk, dv = _split(g, Hq, Hkv)
        ops.attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, B, T, Hq, Hkv, D, scale, seqlens=seqlens)
        return out, lse, g

    out, lse, g = run(qkv, dout)
    qkv2, dout2 = qkv.clone(), dout.clone()
    qkv2[~valid], dout2[~valid] = BIG, BIG
    out2, lse2, g2 = run(qkv2, dout2)
    vl = _valid_rows(lens, T, cuda_device)[:, None, :].expand(B, Hq, T)
    assert torch.equal(out[valid], out2[valid]) and torch.equal(lse[vl], lse2[vl]), "padded rows changed the forward"
    assert torch.equal(g[valid], g2[valid]), "padded rows changed the gradients"
    for x in (g, g2):
        assert_equal(x[~valid], torch.zeros_like(x[~valid]), "gradients of padded rows")

    q, k, v = (_bhtd(x, B, T, h) for x, h in zip(_split(qkv, Hq, Hkv), (Hq, Hkv, Hkv)))
    do = _bhtd(dout, B, T, Hq)
    allowed = _allowed(lens, T, True, cuda_device)
    o64, lse64, gr64 = _ref64(q, k, v, do, allowed, scale, G)
    ot, lset, grt = _torch_bf16(q, k, v, do, allowed, scale, G)
    vr = _valid_rows(lens, T, cuda_device)
    sel = lambda x: x.transpose(1, 2)[vr]          # [B, H, T, d] -> valid rows [n, H, d]
    kern = [_bhtd(x, B, T, h) for x, h in zip(_split(g, Hq, Hkv), (Hq, Hkv, Hkv))]
    # floors: 2^-12 of the largest reference entry (an eighth of a bf16 ulp there) for the bf16 tensors; for lse,
    # 2^-14 of its largest value (fp32 scores of norm-~60 keys carry ~gamma_128 relative error in both paths)
    for name, got, ref, tp in (("out", _bhtd(out, B, T, Hq), o64, ot), ("dQ", kern[0], gr64[0], grt[0]),
                               ("dK", kern[1], gr64[1], grt[1]), ("dV", kern[2], gr64[2], grt[2])):
        r = sel(ref)
        assert_no_worse_than(sel(got), r, sel(tp), f"G={G} {name}", floor=2.0 ** -12 * float(r.abs().max()))
    assert_no_worse_than(lse[vl], lse64[vl], lset[vl], f"G={G} lse", floor=2.0 ** -14 * float(lse64[vl].abs().max()))


# ------------------------------------------------------------------------------------------------ SigLIP head slots
def test_siglip_head_slots_match_unpadded_fp64(cuda_device):
    """SigLIP's 16 heads of 72 sit zero-padded in 128-wide slots: non-causal, T = 729, 3 images, scale 72^-1/2, no lse.
    The result must match the unpadded fp64 attention at d = 72 as well as torch's bf16 path does, and the pad columns
    of the output must be exactly 0."""
    from metamorph_b200 import ops
    n, T, H, dh = 3, 729, 16, 72
    scale = dh ** -0.5
    gen = torch.Generator(device=cuda_device).manual_seed(72)
    x = torch.randn(3, n * T, H, dh, device=cuda_device, generator=gen).bfloat16()
    qkv = torch.zeros(n * T, 3, H, D, device=cuda_device, dtype=torch.bfloat16)
    qkv[:, :, :, :dh] = x.permute(1, 0, 2, 3)
    qkv = qkv.view(n * T, 3 * H * D)
    W = H * D
    out, lse = ops.attn_fwd(qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:], n, T, H, H, D, False, scale, need_lse=False)
    assert lse is None
    o = out.view(n * T, H, D)
    assert_equal(o[:, :, dh:], torch.zeros_like(o[:, :, dh:]), "SigLIP pad columns")
    q, k, v = (_bhtd(x[i].reshape(n * T, H * dh), n, T, H) for i in range(3))
    allowed = _allowed([T] * n, T, False, cuda_device)
    o64, _, _ = _ref64(q, k, v, None, allowed, scale, 1)
    ot, _, _ = _torch_bf16(q, k, v, None, allowed, scale, 1)
    got = _bhtd(o[:, :, :dh].reshape(n * T, H * dh), n, T, H)
    assert_no_worse_than(got, o64, ot, "SigLIP slots", floor=2.0 ** -12 * float(o64.abs().max()))
