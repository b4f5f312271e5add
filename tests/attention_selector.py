"""Selector inputs for flash attention: q, k, v and dO on which every rounding the kernels perform is exact (tests only).

Every score is exactly 0 ("selected") or exactly -C:
  * D = 128 columns split into N_GROUPS selector columns plus one null column, q-payload columns and k-payload
    columns. The payloads are disjoint, so they add exactly 0 to q . k.
  * Key j is one-hot (1) in the selector column of its group h_j; inactive keys use the null column, which no query
    selects. Keys carry small-integer payload.
  * Query i holds 0 in the columns of its chosen groups A_i and -C in every other selector column (the null one too),
    plus small-integer payload. C * scale * log2(e) >= 160, so exp2 of an unselected score is exactly 0 in the kernels
    (`fast_exp2` is ex2.approx.ftz, attention_tc.cuh:11-15).
  * Group sizes are powers of two cycling 1, 2, 4, 8, 16, and the groups fill the active keys in sequence order. A row
    chooses only among groups complete at it (causal), as one group of size n or as n/2 + n/4 + ... + n/2^k with the
    last size twice, so n_i = #{selected keys} is a power of two in 1..16. Some rows choose only groups whose keys all lie
    past the first 128-key tile: the forward's running max then jumps from -C scale to 0 and its rescale factor is
    exactly 0 (attention_tc.cu:194-197).
  * Active keys sit in every 64-key tile and at positions 0, 63, 64, 127, 128 and L - 1 (as many as whole groups
    allow), and the first 128 keys hold whole groups.
  * V holds integers in [-2, 2]; dO two entries of +-1 per row, so a_j = dO_i . V_j lies in [-4, 4] and
    n a_j - sum_sel a fits 8 significant bits.
Then the forward has P = 1 or 0, l = n, O = sum_sel V / n (a bf16 value) and lse = ln n to within a few fp32 ulps; the
backward has bf16(P) = 1/n, dS = scale (n a_j - sum_sel a) / n^2 (a bf16 value for a power-of-two scale), and dQ, dK, dV
are sums of exact products.

`reference` computes O, lse, dQ, dK and dV in fp64 as sparse gathers and scatters (at most 16 keys per row) and
certifies the premise: every quantity the kernels round to bf16 (O, P, dS) is representable, and for every accumulated
element (S, dP, delta, O, dQ, dK, dV) the sum of |terms| is below 2^24 times the power-of-two grid its terms share, taken
per output column. Every partial sum of such terms is an fp32 value, so any summation order gives the exact sum. The
unselected weights exp(-C scale - ln n) < 2^-160 are 0 in the kernels and are left out of the reference.
"""
import math

import torch

from tests.exact import round_bf16_from_fp64

D = 128
C = 2048.0                     # -C: the score of an unselected key
N_GROUPS = 79
NULL = N_GROUPS                # selector column of inactive keys
QPAY = (80, 104)               # q-payload columns
KPAY = (104, 128)              # k-payload columns
SIZES = (1, 2, 4, 8, 16)
NSEL = 16
LATE = 128                     # rows at or past this may select only groups whose keys all lie at or past it
GARBAGE = 1.0e4                # finite values in rows outside a sequence
LOG2E = math.log2(math.e)


def _capacity(g):
    return sum(SIZES[i % 5] for i in range(g))


# groups a row may select: n = 2^k as one group of size n, or n/2 + n/4 + ... + n/2^r + n/2^r (size indices below)
PATTERNS = []
for _k in range(5):
    PATTERNS.append([_k])
    for _r in range(1, min(_k, 3) + 1):
        PATTERNS.append(list(range(_k - 1, _k - _r - 1, -1)) + [_k - _r])
NEED = torch.tensor([[p.count(s) for s in range(5)] for p in PATTERNS])                       # [n_pat, 5]
SLOT = torch.tensor([p + [-1] * (4 - len(p)) for p in PATTERNS])                               # [n_pat, 4]
DUP = torch.tensor([[0 < i < len(p) and p[i] == p[i - 1] for i in range(4)] for p in PATTERNS])
NPAT = torch.tensor([2 ** p[0] if len(p) == 1 else 2 ** (p[0] + 1) for p in PATTERNS])


def key_layout(L, gen):
    """Active key positions of one sequence of L keys, filled into groups in order. Returns (group of each position,
    -1 when inactive [L]; keys [n_groups, 16] positions of each group's keys, -1 padded)."""
    fixed = [p for p in (0, 63, 64, 127, 128, L - 1) if 0 <= p < L]
    tiles = [64 * t + int(torch.randint(min(64, L - 64 * t), (1,), generator=gen)) for t in range((L + 63) // 64)]
    req = list(dict.fromkeys(fixed + tiles))

    def pick(lo, hi, count):
        """count positions in [lo, hi): the required ones first, then random others."""
        mine = [p for p in req if lo <= p < hi]
        if len(mine) >= count:
            return mine[:count]
        free = torch.ones(hi - lo, dtype=torch.bool)
        free[[p - lo for p in mine]] = False
        rest = free.nonzero().view(-1) + lo
        return mine + rest[torch.randperm(len(rest), generator=gen)[:count - len(mine)]].tolist()

    # whole groups inside the first 128 keys, so that later groups lie entirely past the first key tile
    h0 = min(L, LATE)
    g0 = 0
    while g0 < N_GROUPS and _capacity(g0) < max(len([p for p in req if p < h0]), round(0.12 * h0)) and \
            _capacity(g0 + 1) <= h0:
        g0 += 1
    g = g0
    while g < N_GROUPS and _capacity(g) < max(len(req), round(0.12 * L)) and \
            _capacity(g + 1) - _capacity(g0) <= L - h0:
        g += 1
    pos = pick(0, h0, _capacity(g0)) + (pick(h0, L, _capacity(g) - _capacity(g0)) if L > h0 else [])
    pos = torch.tensor(sorted(pos), dtype=torch.long)
    sizes = torch.tensor([SIZES[i % 5] for i in range(g)], dtype=torch.long)
    grp = torch.full((L,), -1, dtype=torch.long)
    grp[pos] = torch.repeat_interleave(torch.arange(g), sizes)
    keys = torch.full((g, NSEL), -1, dtype=torch.long)
    start = torch.cumsum(sizes, 0) - sizes
    for i in range(g):
        keys[i, :sizes[i]] = pos[start[i]:start[i] + sizes[i]]
    return grp, keys


def select_rows(keys, T, causal, n_heads, gen):
    """Groups chosen by rows 0..T-1 of n_heads query heads over one key layout. Returns (groups [n_heads, T, 4] (-1
    unused), selected key positions [n_heads, T, 16] (-1 unused), n [n_heads, T], late [n_heads, T])."""
    ng = keys.shape[0]
    ends = keys.max(1).values
    rows = torch.arange(T)
    E = (ends[None, :] <= rows[:, None]).sum(1) if causal else torch.full((T,), ng)             # complete groups
    s_idx = torch.arange(5)
    count = ((E[:, None] - s_idx[None, :] + 4) // 5).clamp(min=0)                                # [T, 5]
    tot = ((ng - s_idx + 4) // 5).clamp(min=0)
    lo_late = torch.tensor([next((t for t in range(int(tot[s])) if int(keys[5 * t + s, 0]) >= LATE), int(tot[s]))
                            for s in range(5)])
    R = n_heads * T
    count = count.repeat(n_heads, 1)
    r = rows.repeat(n_heads)
    late = (r >= LATE) & (torch.rand(R, generator=gen) < 0.125)
    feas = None
    for _ in range(2):
        lo = torch.where(late[:, None], lo_late[None, :], torch.zeros_like(count))
        avail = (count - lo).clamp(min=0)
        feas = (avail[:, None, :] >= NEED[None]).all(-1)                                         # [R, n_pat]
        late = late & feas.any(1)
    assert bool(feas.any(1).all()), "a row with no complete group"
    choice = torch.where(feas, torch.rand(feas.shape, generator=gen), torch.full(feas.shape, -1.0)).argmax(1)
    slot_s, dup = SLOT[choice], DUP[choice]                                                      # [R, 4]
    groups = torch.full((R, 4), -1, dtype=torch.long)
    t_prev = torch.zeros(R, dtype=torch.long)
    for i in range(4):
        s = slot_s[:, i].clamp(min=0)
        a = avail.gather(1, s[:, None])[:, 0]
        l0 = lo.gather(1, s[:, None])[:, 0]
        u = torch.rand(R, generator=gen)
        t = l0 + (u * a).long().clamp(max=(a - 1).clamp(min=0))
        recent = torch.rand(R, generator=gen) < 0.25                                             # the newest group
        t = torch.where(recent, l0 + (a - 1).clamp(min=0), t)
        t2 = l0 + (t_prev - l0 + 1 + (u * (a - 1).clamp(min=0)).long()) % a.clamp(min=1)
        t = torch.where(dup[:, i], t2, t)
        ok = slot_s[:, i] >= 0
        groups[:, i] = torch.where(ok, 5 * t + s, torch.full_like(t, -1))
        t_prev = t
    kk = torch.where(groups[:, :, None] >= 0, keys[groups.clamp(min=0)], torch.full((R, 4, NSEL), -1)).view(R, -1)
    order = torch.sort((kk < 0).to(torch.int8), dim=1, stable=True).indices[:, :NSEL]
    sel = kk.gather(1, order)
    n = (sel >= 0).sum(1)
    assert torch.equal(n, NPAT[choice]), "a selection is not the power of two its pattern names"
    return groups.view(n_heads, T, 4), sel.view(n_heads, T, NSEL), n.view(n_heads, T), late.view(n_heads, T)


class Selector:
    """Selector inputs of B sequences in a padded [B, T] layout (q, do [B, T, Hq, D]; k, v [B, T, Hkv, D], bf16 on the
    CPU). Rows at or past lens[b] hold GARBAGE in k, v and dO and selector rows in q (so the forward of a padded row has
    an exact value too). sel [B, Hq, T, 16], n [B, Hq, T], late [B, Hq, T]."""

    def __init__(self, lens, T, Hq, Hkv, seed, causal=True):
        assert Hq % Hkv == 0 and all(1 <= L <= T for L in lens)
        self.lens, self.T, self.Hq, self.Hkv, self.causal = list(lens), T, Hq, Hkv, causal
        B, G = len(lens), Hq // Hkv
        gen = torch.Generator().manual_seed(seed)
        q = torch.empty(B, T, Hq, D)
        k = torch.empty(B, T, Hkv, D)
        v = torch.empty(B, T, Hkv, D)
        do = torch.empty(B, T, Hq, D)
        self.sel = torch.empty(B, Hq, T, NSEL, dtype=torch.long)
        self.n = torch.empty(B, Hq, T, dtype=torch.long)
        self.late = torch.empty(B, Hq, T, dtype=torch.bool)
        ints = lambda *shape: torch.randint(-2, 3, shape, generator=gen).float()
        garbage = lambda *shape: GARBAGE * (2 * torch.randint(0, 2, shape, generator=gen).float() - 1)
        for b, L in enumerate(lens):
            for hk in range(Hkv):
                hs = slice(hk * G, hk * G + G)
                grp, keys = key_layout(L, gen)
                groups, sel, n, late = select_rows(keys, T, causal, G, gen)
                self.sel[b, hs], self.n[b, hs], self.late[b, hs] = sel, n, late
                qq = torch.zeros(G, T, D + 1)
                qq[:, :, :NULL + 1] = -C
                qq[:, :, QPAY[0]:QPAY[1]] = ints(G, T, QPAY[1] - QPAY[0])
                qq.scatter_(2, torch.where(groups >= 0, groups, torch.full_like(groups, D)), 0.0)
                kk = torch.zeros(T, D)
                kk[torch.arange(L), torch.where(grp >= 0, grp, torch.full_like(grp, NULL))] = 1.0
                kk[:L, KPAY[0]:KPAY[1]] = ints(L, KPAY[1] - KPAY[0])
                kk[L:] = garbage(T - L, D)
                perm = torch.randperm(D, generator=gen)                      # q . k is unchanged by a joint permutation
                q[b, :, hs] = qq[:, :, :D][:, :, perm].transpose(0, 1)
                k[b, :, hk] = kk[:, perm]
                v[b, :L, hk] = ints(L, D)
                v[b, L:, hk] = garbage(T - L, D)
                dd = torch.zeros(G * L, D)
                c1 = torch.randint(D, (G * L,), generator=gen)
                c2 = (c1 + 1 + torch.randint(D - 1, (G * L,), generator=gen)) % D
                dd.scatter_(1, torch.stack([c1, c2], 1), 2 * torch.randint(0, 2, (G * L, 2), generator=gen).float() - 1)
                do[b, :L, hs] = dd.view(G, L, D).transpose(0, 1)
                do[b, L:, hs] = garbage(T - L, G, D)
        self.q, self.k, self.v, self.do = (x.bfloat16() for x in (q, k, v, do))


# ------------------------------------------------------------------------------------------------ reference + certificate
def lowbit(x):
    """The value of the lowest set bit of every element of an fp64 tensor (inf where x is 0 or not finite): x is an
    integer multiple of lowbit(x)."""
    x = x.double().abs()
    m, e = torch.frexp(x)
    M = torch.ldexp(m, torch.full_like(m, 53.0)).long()
    tz = torch.log2((M & -M).double())
    r = torch.ldexp(torch.ones_like(x), e.double() - 53.0 + tz)
    return torch.where((x == 0) | ~torch.isfinite(x), torch.full_like(x, math.inf), r)


def _col_lowbit(x):
    """[..., D] -> [D]: the grid every element of a column shares."""
    return lowbit(x.reshape(-1, x.shape[-1])).amin(0) if x.numel() else torch.full((x.shape[-1],), math.inf,
                                                                                    dtype=torch.float64,
                                                                                    device=x.device)


def _ratio(abs_sum, grid):
    """max over elements of sum|terms| / (2^24 grid) (0 where there are no terms)."""
    r = abs_sum / (2.0 ** 24 * grid)
    return float(torch.nan_to_num(torch.where(abs_sum == 0, torch.zeros_like(r), r), nan=math.inf).max()) \
        if abs_sum.numel() else 0.0


def _representable(x):
    return bool((round_bf16_from_fp64(x).double() == x).all())


class CertificateError(AssertionError):
    pass


def reference(s, scale, device, chunk=1024):
    """fp64 O [B, T, Hq, D], lse [B, Hq, T], and for rows < lens[b] dQ [B, T, Hq, D], dK, dV [B, T, Hkv, D] (0 on rows
    past the sequence) of the selector inputs `s` at `scale`, with the certificate's largest ratios (each < 1). Raises
    CertificateError when a case fails the premise."""
    if C * scale * LOG2E < 160:
        raise CertificateError(f"C scale log2(e) = {C * scale * LOG2E:.1f} < 160: exp2 of -C would not flush to 0")
    pw = torch.log2(torch.tensor(scale, dtype=torch.float64))
    bwd_exact = bool(pw == torch.round(pw))
    B, T, Hq, Hkv = len(s.lens), s.T, s.Hq, s.Hkv
    G = Hq // Hkv
    f64 = dict(dtype=torch.float64, device=device)
    o = torch.zeros(B, T, Hq, D, **f64)
    dq = torch.zeros(B, T, Hq, D, **f64)
    dk = torch.zeros(B, T, Hkv, D, **f64)
    dv = torch.zeros(B, T, Hkv, D, **f64)
    n_all = s.n.to(device)
    if not bool(((n_all & (n_all - 1)) == 0).all() & (n_all >= 1).all() & (n_all <= NSEL).all()):
        raise CertificateError("a row count that is not a power of two in 1..16")
    lse = torch.log(n_all.double())
    cert = dict.fromkeys(("S", "dP", "delta", "O", "dQ", "dK", "dV"), 0.0)
    bad = []
    for b, L in enumerate(s.lens):
        for hk in range(Hkv):
            hs = slice(hk * G, hk * G + G)
            K = s.k[b, :, hk].to(device).double()
            V = s.v[b, :, hk].to(device).double()
            Q = s.q[b, :, hs].to(device).double().transpose(0, 1)            # [G, T, D]
            dO = s.do[b, :, hs].to(device).double().transpose(0, 1)
            sel, n = s.sel[b, hs].to(device), n_all[b, hs].double()
            lbK, lbV = _col_lowbit(K[:L]), _col_lowbit(V[:L])
            lbQ, lbdO = _col_lowbit(Q[:, :L]), _col_lowbit(dO[:, :L])
            # S over every (row, key < L) pair the kernels compute, dP over rows < L: bounds from column maxima
            cert["S"] = max(cert["S"], float((Q.abs().amax((0, 1)) * K[:L].abs().amax(0)).sum()) /
                            (2.0 ** 24 * float(lowbit(Q).min()) * float(lowbit(K[:L]).min())))
            cert["dP"] = max(cert["dP"], float(dO[:, :L].abs().sum(-1).max() * V[:L].abs().max()) /
                             (2.0 ** 24 * float(lowbit(dO[:, :L]).min()) * float(lowbit(V[:L]).min())))
            dk_acc, dv_acc = torch.zeros(T, D, **f64), torch.zeros(T, D, **f64)
            dk_abs, dv_abs = torch.zeros(T, D, **f64), torch.zeros(T, D, **f64)
            dq_abs_max = torch.zeros(D, **f64)
            lb_ds, lb_p = math.inf, math.inf
            for r0 in range(0, T, chunk):
                rs = slice(r0, min(T, r0 + chunk))
                m = sel[:, rs] >= 0
                idx = sel[:, rs].clamp(min=0)
                nn = n[:, rs, None]
                Vs = V[idx] * m[..., None]                                    # [G, r, 16, D]
                oc = Vs.sum(2) / nn
                o[b, rs, hs] = oc.transpose(0, 1)
                if not _representable(oc):
                    bad.append(f"O of sequence {b} kv head {hk} is not a bf16 value")
                cert["O"] = max(cert["O"], _ratio(Vs.abs().sum(2), lbV))
                live = (torch.arange(r0, rs.stop, device=device) < L)[None, :, None]     # rows of the sequence
                a = (dO[:, rs, None, :] * Vs).sum(-1)                         # dP of the selected pairs [G, r, 16]
                ds = scale * (nn * a - (a * m).sum(-1, keepdim=True)) / nn ** 2 * (m & live)
                p = m.double() / nn * live
                if bwd_exact and not _representable(ds):
                    bad.append(f"dS of sequence {b} kv head {hk} is not a bf16 value")
                lb_ds = min(lb_ds, float(lowbit(ds).min()))
                lb_p = min(lb_p, float(lowbit(p).min()))
                Ks = K[idx]
                dq[b, rs, hs] = (ds[..., None] * Ks).sum(2).transpose(0, 1)
                dq_abs_max = torch.maximum(dq_abs_max, (ds.abs()[..., None] * Ks.abs()).sum(2).amax((0, 1)))
                flat = idx.reshape(-1)
                dk_acc.index_add_(0, flat, (ds[..., None] * Q[:, rs, None, :]).reshape(-1, D))
                dk_abs.index_add_(0, flat, (ds.abs()[..., None] * Q[:, rs, None, :].abs()).reshape(-1, D))
                dv_acc.index_add_(0, flat, (p[..., None] * dO[:, rs, None, :]).reshape(-1, D))
                dv_abs.index_add_(0, flat, (p[..., None] * dO[:, rs, None, :].abs()).reshape(-1, D))
                # delta = sum_c dO o over the rows of the sequence: one chain per row, grid per row
                dl = (dO[:, rs] * oc).abs() * live
                grid = lowbit(dO[:, rs]).amin(-1) * lowbit(oc).amin(-1)
                cert["delta"] = max(cert["delta"], _ratio(dl.sum(-1), grid))
            dk[b, :, hk], dv[b, :, hk] = dk_acc, dv_acc
            cert["dQ"] = max(cert["dQ"], _ratio(dq_abs_max, lb_ds * lbK))
            cert["dK"] = max(cert["dK"], _ratio(dk_abs, lb_ds * lbQ))
            cert["dV"] = max(cert["dV"], _ratio(dv_abs, lb_p * lbdO))
    if not bwd_exact:
        for x in ("dP", "delta", "dQ", "dK", "dV"):
            cert.pop(x)
    over = {x: r for x, r in cert.items() if not r < 1.0}
    if bad or over:
        raise CertificateError("; ".join(bad[:4] + [f"{x}: sum|terms| = {r:.3g} x 2^24 grid" for x, r in over.items()]))
    return dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv, cert=cert)
