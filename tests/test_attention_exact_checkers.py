"""The exact flash-attention checks have teeth, and their premise holds (CPU only).

* The selector generator certifies every case tests/test_attention_exact_gpu.py runs, and the cases together reach
  every regime of the schedule that file restates.
* `emulate` restates the kernels' rounding points in fp32: S and dP exact, the online softmax with exp2 flushed to 0
  below 2^-126, P and dS rounded to bf16 before their products, and every accumulation in fp32 tile by tile in a
  random order (terms shuffled, cut into random chunks, the chunk sums added in sequence). On selector inputs it
  reproduces the reference bits under any order, so the exact check does not depend on the kernels' summation order.
* With one kernel bug emulated, the same check rejects the result with at least one differing bit.
Nothing here builds or runs a kernel.
"""
import math

import pytest
import torch

from tests.attention_selector import C, LOG2E, reference
from tests.test_attention_exact_gpu import (CASES, NONCAUSAL, PADDED, PAGED, SCALE_BWD, SCALE_ENGINE, check_bwd,
                                            check_fwd, regimes)

D = 128
BUGS = ["dq_drops_last_key_tile", "dkv_sums_G_minus_1_heads", "odd_key_tile_starts_late", "ring_reuses_it_minus_2",
        "delta_without_scale", "stats_of_neighbour_row", "causal_lt", "padded_tile_leaves_dq", "fwd_skips_o_rescale"]
EMU_CASE = next(c for c in PADDED if c.name == "T192")       # padded q tile, odd 64-key tile, n_it = 8, G = 4


def _ex2(x):
    """ex2.approx.ftz: results below 2^-126 flush to 0."""
    y = torch.exp2(x)
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _bf(x):
    return x.bfloat16().float()


def acc32(terms, dim, gen):
    """fp32 sum of `terms` along `dim` in a random order: shuffled, cut into chunks of 1..32, chunk sums (torch's own
    order) added one after another."""
    n = terms.shape[dim]
    terms = terms.index_select(dim, torch.randperm(n, generator=gen))
    out = None
    i = 0
    while i < n:
        w = int(torch.randint(1, 33, (1,), generator=gen))
        part = terms.narrow(dim, i, min(w, n - i)).sum(dim, dtype=torch.float32)
        out = part if out is None else out + part
        i += w
    return out if out is not None else terms.sum(dim)


def emulate_fwd(Q, K, V, L, causal, scale, gen, bug=None):
    """One (sequence, kv head): Q [G, T, D], K / V [T, D] fp32. Returns out [G, T, D] bf16, lse [G, T] fp32."""
    G, T, _ = Q.shape
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)
    rows = torch.arange(T)
    kv_end = torch.clamp((rows // 128) * 128 + 128, max=L) if causal else torch.full((T,), L)
    n_tiles = (kv_end + 127) // 128
    m = torch.full((G, T), -math.inf)
    l = torch.zeros(G, T)
    o = torch.zeros(G, T, D)
    for j in range((L + 127) // 128):
        cols = torch.arange(j * 128, j * 128 + 128)
        Kt = torch.where((cols < T)[:, None], K[cols.clamp(max=T - 1)], torch.zeros(1))   # TMA zero fill past T
        Vt = torch.where((cols < T)[:, None], V[cols.clamp(max=T - 1)], torch.zeros(1))
        S = Q @ Kt.T
        allowed = (cols[None, :] < L) & ((cols[None, :] <= rows[:, None]) if causal else True)
        S = torch.where(allowed[None], S, torch.full_like(S, -math.inf))
        m_new = torch.maximum(m, S.amax(-1) * sl2)
        f = torch.where(m_new == -math.inf, torch.ones_like(m), _ex2(m - m_new))
        m_eff = torch.where(m_new == -math.inf, torch.zeros_like(m), m_new)
        e = _ex2(_fma(S, sl2, -m_eff[..., None]))
        l_new = l * f + acc32(e, 2, gen)
        o_new = o * f[..., None] if (j > 0 and bug != "fwd_skips_o_rescale") else o
        o_new = o_new + acc32(_bf(e)[..., None] * Vt[None, None], 2, gen)
        visit = (j < n_tiles)[None]
        m, l = torch.where(visit, m_new, m), torch.where(visit, l_new, l)
        o = torch.where(visit[..., None], o_new, o)
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    lse = torch.where(l > 0, (m + torch.log2(l)) / LOG2E, torch.full_like(l, -math.inf))
    return (o * inv[..., None]).bfloat16(), lse


def emulate_dq(Q, K, V, O, dO, lse, L, scale, gen, bug=None):
    """flash_bwd_dq_kernel for one (sequence, kv head): returns dq [G, T, D] bf16 (NaN where a kernel would not write)
    and the workspace rows lse2, delta [G, Tp]."""
    G, T, _ = Q.shape
    Tp = (T + 127) // 128 * 128
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)
    rows = torch.arange(T)
    qt = rows // 128
    ok_row = rows < L
    d = acc32(dO * O.float(), 2, gen)
    delta = torch.where(ok_row, d if bug == "delta_without_scale" else d * scale, torch.zeros_like(d))
    lse2 = torch.where(ok_row, lse * torch.tensor(LOG2E, dtype=torch.float32), torch.zeros_like(lse))
    dq = torch.zeros(G, T, D)
    for j in range((L + 127) // 128):
        for hf in range(2):
            cols = torch.arange(j * 128 + hf * 64, j * 128 + hf * 64 + 64)
            Kt = torch.where((cols < T)[:, None], K[cols.clamp(max=T - 1)], torch.zeros(1))
            Vt = torch.where((cols < T)[:, None], V[cols.clamp(max=T - 1)], torch.zeros(1))
            S, dP = Q @ Kt.T, dO @ Vt.T
            causal = (cols[None, :] < rows[:, None]) if bug == "causal_lt" else (cols[None, :] <= rows[:, None])
            ok = ok_row[:, None] & causal & (cols[None, :] < L) & (j <= qt)[:, None]
            if bug == "dq_drops_last_key_tile":
                ok = ok & (j != qt)[:, None]
            pv = torch.where(ok[None], _ex2(_fma(S, sl2, -lse2[..., None])), torch.zeros_like(S))
            ds = _bf(pv * _fma(dP, torch.tensor(scale), -delta[..., None]))
            dq = dq + acc32(ds[..., None] * Kt[None, None], 2, gen)
    padded_tile = (qt * 128 >= L)
    dq = torch.where(ok_row[None, :, None], dq, torch.zeros_like(dq))
    if bug == "padded_tile_leaves_dq":
        dq = torch.where(padded_tile[None, :, None], torch.full_like(dq, math.nan), dq)
    pad = lambda x: torch.cat([x, torch.zeros(G, Tp - T)], 1)
    return dq.bfloat16(), pad(lse2), pad(delta)


def emulate_dkv(Q, K, V, dO, lse2, delta, L, scale, gen, bug=None):
    """flash_bwd_dkv_kernel for one (sequence, kv head): returns dk, dv [T, D] bf16."""
    G, T, _ = Q.shape
    Tp = lse2.shape[1]
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)
    Qp = torch.cat([Q, torch.zeros(G, Tp - T, D)], 1)                      # TMA zero fill past T
    dOp = torch.cat([dO, torch.zeros(G, Tp - T, D)], 1)
    dk, dv = torch.zeros(T, D), torch.zeros(T, D)
    for jt in range(2 * ((T + 127) // 128)):
        kv0 = jt * 64
        if kv0 >= L:
            continue
        keys = torch.arange(kv0, kv0 + 64)
        Kt = torch.where((keys < T)[:, None], K[keys.clamp(max=T - 1)], torch.zeros(1))
        Vt = torch.where((keys < T)[:, None], V[keys.clamp(max=T - 1)], torch.zeros(1))
        qt_begin = kv0 // 128 + (1 if bug == "odd_key_tile_starts_late" and jt % 2 else 0)
        n_qt = (L + 127) // 128 - qt_begin
        ak, av = torch.zeros(64, D), torch.zeros(64, D)
        for it in range(n_qt * G):
            if bug == "dkv_sums_G_minus_1_heads" and it // n_qt == G - 1:
                continue
            src = it - 2 if bug == "ring_reuses_it_minus_2" and it >= 2 and (it >> 1) & 1 else it
            q0 = (qt_begin + it % n_qt) * 128
            hq, s0 = src // n_qt, (qt_begin + src % n_qt) * 128
            Qt, dOt = Qp[hq, s0:s0 + 128], dOp[hq, s0:s0 + 128]
            ql = torch.arange(128) ^ (1 if bug == "stats_of_neighbour_row" else 0)
            l2, dl = lse2[hq, s0 + ql], delta[hq, s0 + ql]
            qrow = q0 + torch.arange(128)
            St, dPt = Kt @ Qt.T, Vt @ dOt.T                                 # [64 keys, 128 queries]
            causal = (keys[:, None] < qrow[None, :]) if bug == "causal_lt" else (keys[:, None] <= qrow[None, :])
            ok = (keys[:, None] < L) & (qrow[None, :] < L) & causal
            pv = torch.where(ok, _ex2(_fma(St, sl2, -l2[None, :])), torch.zeros_like(St))
            av = av + acc32(_bf(pv)[..., None] * dOt[None], 1, gen)
            ak = ak + acc32(_bf(pv * _fma(dPt, torch.tensor(scale), -dl[None, :]))[..., None] * Qt[None], 1, gen)
        n = min(64, T - kv0)
        live = (keys[:n] < L)[:, None]
        dk[kv0:kv0 + n] = torch.where(live, ak[:n], torch.zeros(1))
        dv[kv0:kv0 + n] = torch.where(live, av[:n], torch.zeros(1))
    return dk.bfloat16(), dv.bfloat16()


def emulate(s, gen, bug=None, scale_fwd=SCALE_BWD):
    """Every kernel of the padded layout on selector inputs `s`: out, lse (forward at scale_fwd), dq, dk, dv (backward
    at SCALE_BWD on the forward at SCALE_BWD), as [B, T, H, D] / [B, Hq, T]."""
    B, T, Hq, Hkv = len(s.lens), s.T, s.Hq, s.Hkv
    G = Hq // Hkv
    out = torch.full((B, T, Hq, D), math.nan, dtype=torch.bfloat16)
    lse = torch.full((B, Hq, T), math.nan)
    dq = torch.full_like(out, math.nan)
    dk = torch.full((B, T, Hkv, D), math.nan, dtype=torch.bfloat16)
    dv = torch.full_like(dk, math.nan)
    for b, L in enumerate(s.lens):
        for hk in range(Hkv):
            hs = slice(hk * G, hk * G + G)
            Q, dO = s.q[b, :, hs].float().transpose(0, 1), s.do[b, :, hs].float().transpose(0, 1)
            K, V = s.k[b, :, hk].float(), s.v[b, :, hk].float()
            o, l = emulate_fwd(Q, K, V, L, s.causal, scale_fwd, gen, bug)
            out[b, :, hs], lse[b, hs] = o.transpose(0, 1), l
            if scale_fwd != SCALE_BWD:
                o, l = emulate_fwd(Q, K, V, L, s.causal, SCALE_BWD, gen, bug)
            g, lse2, delta = emulate_dq(Q, K, V, o, dO, l, L, SCALE_BWD, gen, bug)
            dq[b, :, hs] = g.transpose(0, 1)
            dk[b, :, hk], dv[b, :, hk] = emulate_dkv(Q, K, V, dO, lse2, delta, L, SCALE_BWD, gen, bug)
    return out, lse, dq, dk, dv


def _check_all(s, ref, res, what):
    out, lse, dq, dk, dv = res
    rows = torch.ones(len(s.lens), s.T, dtype=torch.bool)
    check_fwd(out[rows], lse.transpose(1, 2)[rows], ref, rows, what)
    check_bwd(dq[rows], dk[rows], dv[rows], ref, rows, what)


# ------------------------------------------------------------------------------------------------ the premise
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_selector_certificate_holds(case):
    s = case.selector()
    scale = SCALE_ENGINE if case in (PAGED,) else 72 ** -0.5 if case is NONCAUSAL else SCALE_BWD
    ref = reference(s, scale, "cpu")
    assert C * SCALE_ENGINE * LOG2E >= 160                     # the padded cases also run the forward at 128^-1/2
    assert all(r < 1 for r in ref["cert"].values())
    n = s.n[:, :, :max(s.lens)]
    assert set(torch.unique(n).tolist()) <= {1, 2, 4, 8, 16}
    assert case.reaches <= regimes(case, s.late), f"{case}: misses {case.reaches - regimes(case, s.late)}"
    print(f"{case}: worst sum|terms| / (2^24 grid): " + ", ".join(f"{k} {v:.3g}" for k, v in ref["cert"].items()))


def test_cases_cover_the_schedule():
    need = {"G1", "G2", "G4", "G8", "n_it=1", "n_it=2", "n_it=3", "n_it>=4", "padded_q_tile", "padded_k_tile",
            "odd_last_k_tile", "kv_len=64mod128", "max_jump"}
    need |= {f"{k}_grid{r}SMs" for k in ("dq", "dkv") for r in "<=>"}
    got = set().union(*(c.reaches for c in PADDED + [c for c in CASES if c.name.startswith(("bench", "config"))]))
    assert need <= got, f"no case reaches {need - got}"


# ------------------------------------------------------------------------------------------------ the check's teeth
@pytest.fixture(scope="module")
def emu_case():
    s = EMU_CASE.selector()
    return s, reference(s, SCALE_BWD, "cpu")


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_emulation_reproduces_reference_bits_in_any_order(emu_case, seed):
    s, ref = emu_case
    gen = torch.Generator().manual_seed(seed)
    _check_all(s, ref, emulate(s, gen, scale_fwd=SCALE_ENGINE if seed == 3 else SCALE_BWD), f"order seed {seed}")


@pytest.mark.parametrize("bug", BUGS)
def test_exact_check_rejects(emu_case, bug):
    s, ref = emu_case
    with pytest.raises(AssertionError) as e:
        _check_all(s, ref, emulate(s, torch.Generator().manual_seed(7), bug=bug), bug)
    print(f"rejected: {e.value}")
