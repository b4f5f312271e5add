"""Flash attention forward and backward (attention_tc.cu, attention_bwd_tc.cu) held to exact fp64 results on selector
inputs (tests/attention_selector.py), at the training shapes and the schedule's tile, ring and grid edges (H100 only).

On selector inputs every rounding inside the kernels is exact (the generator certifies it per case), so O, dQ, dK and
dV must equal round_bf16_from_fp64 of the fp64 reference bit for bit, whatever order the kernels sum in; lse must be
within 16u max(1, ln n) of ln n. Outputs start as NaN: rows past a sequence must come back exactly 0 (gradients), gap
rows of the packed layout keep their sentinels. A random-data case extends the peaked-softmax check of
test_attention_edges_gpu.py to the benchmark's shape, where P is not a power of two.

Schedule (what the cases are derived from):
  forward, flash_fwd_wgmma_kernel (attention_tc.cu): one CTA = 128 query rows of one (sequence, q head); padded grid
    (ceil(T / 128), Hq, B) walked last tile first (:67), packed grid (work items, Hq) (:338). Key tiles of 128 up to
    min(kv_len, q0 + 128) (:72-75) through a two-stage K/V ring (:104-152). Masking only on tiles that reach kv_len or
    the diagonal (:177-185); the running max m_new, the rescale f = exp2(m_run - m_new) applied to l and, from the second
    tile on, to O (:186-211). Rows past kv_len of a padded sequence are computed and stored (row < T, :246); packed rows
    past the segment are not (:77). The paged variant fills a tile with one TMA box per block and zeroes V rows at or
    past kv_len in shared memory (:107-142, :216-230).
  dQ, flash_bwd_dq_kernel (attention_bwd_tc.cu): grid as the forward (:439). A query tile at or past kv_len writes zero
    dQ and neutral statistics (:72-84); otherwise delta = rowsum(dO o O) scale and lse2 = lse log2(e) are written to the
    workspace (:145-173), and each key tile 0..qt is processed in two 64-key halves: P = exp2(S sl2 - lse2),
    dS = P (dP scale - delta) to bf16, dQ += dS K (:189-227).
  dK/dV, flash_bwd_dkv_kernel: one CTA = 64 keys of one (sequence, kv head); padded grid (Hkv B, 2 ceil(T / 128))
    (:440). A key tile at or past kv_len writes zeros (:255-264). qt_begin = kv0 / 128 (:265): the odd 64-key tile
    shares its first query tile with the even one. n_it = n_qt G iterations walk head hq = hk G + it / n_qt and query
    tile qt_begin + it % n_qt (:303-306) through a two-buffer Q/dO/statistics ring: buffer it & 1, phase (it >> 1) & 1
    (:304-308, :336-338); n_it >= 3 reuses buffer 0, n_it >= 4 both buffers. Causal mask key <= query (:360).
H100 SXM has 132 SMs: grids below, at and above that count are different dispatch regimes.
"""
import pytest
import torch

from tests.attention_selector import D, Selector, reference
from tests.exact import U, assert_equal, assert_no_worse_than, assert_within, round_bf16_from_fp64

pytestmark = pytest.mark.gpu

SMS = 132
SCALE_BWD = 2.0 ** -3           # dS exact needs a power of two
SCALE_ENGINE = D ** -0.5        # the forward is exact at any scale


class Case:
    def __init__(self, name, T, lens, Hq, Hkv, reaches, seed=None, causal=True):
        self.name, self.T, self.lens, self.Hq, self.Hkv = name, T, list(lens), Hq, Hkv
        self.reaches, self.causal = set(reaches), causal
        self.seed = seed if seed is not None else sum(map(ord, name))

    def __repr__(self):
        return self.name

    def selector(self):
        return Selector(self.lens, self.T, self.Hq, self.Hkv, self.seed, causal=self.causal)


def regimes(case, late=None):
    """The schedule regimes the padded-layout case reaches (module docstring)."""
    G, T = case.Hq // case.Hkv, case.T
    nt = (T + 127) // 128
    out = {f"G{G}"}
    grid_q, grid_k = nt * case.Hq * len(case.lens), case.Hkv * len(case.lens) * 2 * nt
    for name, g in (("dq", grid_q), ("dkv", grid_k)):
        out.add(f"{name}_grid" + ("<" if g < SMS else "=" if g == SMS else ">") + "SMs")
    for L in case.lens:
        if any(qt * 128 >= L for qt in range(nt)):
            out.add("padded_q_tile")
        if any(jt * 64 >= L for jt in range(2 * nt)):
            out.add("padded_k_tile")
        if ((L - 1) // 64) % 2 == 1:
            out.add("odd_last_k_tile")
        if L % 128 == 64:
            out.add("kv_len=64mod128")
        for jt in range((L + 63) // 64):
            n_it = ((L + 127) // 128 - jt // 2) * G
            out.add(f"n_it={n_it}" if n_it < 4 else "n_it>=4")
    if late is not None and bool(late.any()):
        out.add("max_jump")
    return out


PADDED = [
    Case("T1", 1, [1], 2, 2, {"G1", "n_it=1", "dq_grid<SMs", "dkv_grid<SMs", "padded_k_tile"}),
    Case("T63", 63, [63, 17], 4, 2, {"G2", "n_it=2", "padded_k_tile"}),
    Case("T64", 64, [64, 1], 8, 2, {"G4", "n_it>=4", "padded_k_tile"}),
    Case("T65", 65, [65, 64], 8, 1, {"G8", "padded_k_tile", "kv_len=64mod128", "odd_last_k_tile"}),
    Case("T127", 127, [127, 100], 2, 2, {"G1", "n_it=1", "odd_last_k_tile"}),
    Case("T128", 128, [128, 128], 4, 2, {"G2", "n_it=2", "odd_last_k_tile"}),
    Case("T129", 129, [129, 64], 2, 2, {"G1", "n_it=2", "n_it=1", "padded_q_tile", "padded_k_tile"}),
    Case("T191", 191, [191, 65], 8, 1, {"G8", "padded_q_tile", "max_jump"}),
    Case("T192", 192, [192, 100], 8, 2, {"G4", "kv_len=64mod128", "padded_q_tile", "max_jump"}),
    Case("T255", 255, [255, 250], 2, 2, {"G1", "n_it=2", "odd_last_k_tile"}),
    Case("T257-at-SMs", 257, [257] * 11, 4, 2, {"G2", "dq_grid=SMs", "dkv_grid=SMs", "max_jump"}),
    Case("T257-G1", 257, [257, 129], 2, 2, {"G1", "n_it=3", "padded_q_tile"}),
    Case("T523", 523, [523, 320, 64, 389], 16, 4, {"G4", "dq_grid>SMs", "dkv_grid>SMs", "kv_len=64mod128",
                                                   "padded_q_tile", "padded_k_tile", "max_jump"}),
    Case("T523-G8", 523, [523, 192], 16, 2, {"G8", "dq_grid>SMs", "dkv_grid<SMs", "max_jump"}),
]
TRAINING = [
    Case("bench-B4-T4096", 4096, [4096] * 4, 32, 8, {"G4", "dq_grid>SMs", "dkv_grid>SMs", "max_jump"}),
    Case("config5-B1-T8192", 8192, [8192], 32, 8, {"G4", "dq_grid>SMs", "dkv_grid>SMs", "max_jump"}),
    Case("ragged-T4096", 4096, [4096, 2112, 1, 3001], 32, 8, {"padded_q_tile", "padded_k_tile", "kv_len=64mod128",
                                                             "odd_last_k_tile", "max_jump"}),
]
# packed: segments of 1, 64, 65, 128, 129 and 300 rows, 16 times over (144 query work items), unaligned offsets, the
# last segment ending on the buffer's last row
PACKED_LENS = [1, 64, 65, 128, 129, 300] * 16
PACKED = Case("packed", 300, PACKED_LENS, 8, 2, {"G4"})
PAGED = Case("paged-T4096", 4096, [4096], 8, 2, {"G4", "max_jump"})
PAGED_Q = [(0, 300), (48, 300), (4096 - 300, 300)]
NONCAUSAL = Case("siglip-T729", 729, [729] * 3, 16, 16, {"G1", "max_jump"}, causal=False)
CASES = PADDED + TRAINING + [PACKED, PAGED, NONCAUSAL]


def packed_offsets(lens, seed):
    """Segment starts with gaps of 0..5 rows; the buffer ends with the last segment."""
    gen = torch.Generator().manual_seed(seed)
    starts, row = [], 3
    for L in lens:
        starts.append(row)
        row += L + int(torch.randint(0, 6, (1,), generator=gen))
    R = starts[-1] + lens[-1]
    return starts, R


# ------------------------------------------------------------------------------------------------ checks
def check_fwd(out, lse, ref, rows, what):
    """out [..., D] bf16 and lse of the rows selected by `rows` (a bool mask over [B, T]) against the reference."""
    o64 = ref["o"][rows]
    assert_equal(out, round_bf16_from_fp64(o64).view(out.shape), f"{what}: out")
    if lse is not None:
        ln_n = ref["lse"].transpose(1, 2)[rows]
        assert_within(lse, ln_n, 16 * U * ln_n.clamp(min=1.0), f"{what}: lse")


def check_bwd(dq, dk, dv, ref, rows, what):
    for name, got, want in (("dQ", dq, ref["dq"]), ("dK", dk, ref["dk"]), ("dV", dv, ref["dv"])):
        assert_equal(got, round_bf16_from_fp64(want[rows]).view(got.shape), f"{what}: {name}")


def _fused(s, device):
    """q, k, v as column slices of one [B T, (Hq + 2 Hkv) D] buffer."""
    B, T = len(s.lens), s.T
    qkv = torch.cat([s.q.reshape(B * T, -1), s.k.reshape(B * T, -1), s.v.reshape(B * T, -1)], 1).to(device)
    Wq, Wk = s.Hq * D, s.Hkv * D
    return qkv, qkv[:, :Wq], qkv[:, Wq:Wq + Wk], qkv[:, Wq + Wk:]


def run_padded(case, device):
    """Forward at the engine scale and at 2^-3, backward at 2^-3, every operand strided; checks everything."""
    from metamorph_b200 import ops
    s = case.selector()
    assert case.reaches <= regimes(case, s.late), f"{case}: misses {case.reaches - regimes(case, s.late)}"
    B, T, Hq, Hkv = len(s.lens), s.T, s.Hq, s.Hkv
    qkv, q, k, v = _fused(s, device)
    seqlens = torch.tensor(s.lens, device=device, dtype=torch.int32)
    allrows = torch.ones(B, T, dtype=torch.bool, device=device)
    valid = torch.arange(T, device=device)[None, :] < seqlens[:, None]
    ref = reference(s, SCALE_BWD, device)
    for scale in (SCALE_ENGINE, SCALE_BWD):
        obuf = torch.full((B * T, Hq * D + 128), float("nan"), device=device, dtype=torch.bfloat16)
        out = obuf[:, :Hq * D]                                       # a pitch wider than Hq 128
        out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, D, True, scale, seqlens=seqlens, out=out)
        assert bool(torch.isnan(obuf[:, Hq * D:].float()).all()), f"{case}: out written past its width"
        check_fwd(out.view(B, T, Hq, D)[allrows], lse.transpose(1, 2)[allrows], ref, allrows,
                  f"{case} scale={scale:.4g}")
    g = torch.full((B * T, (Hq + 2 * Hkv) * D), float("nan"), device=device, dtype=torch.bfloat16)
    dq, dk, dv = g[:, :Hq * D], g[:, Hq * D:(Hq + Hkv) * D], g[:, (Hq + Hkv) * D:]
    dout = s.do.reshape(B * T, -1).to(device)
    ops.attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, B, T, Hq, Hkv, D, SCALE_BWD, seqlens=seqlens)
    check_bwd(dq.view(B, T, Hq, D)[allrows], dk.view(B, T, Hkv, D)[allrows], dv.view(B, T, Hkv, D)[allrows], ref,
              allrows, f"{case}")
    pad = ~valid.reshape(-1)
    assert_equal(g[pad], torch.zeros_like(g[pad]), f"{case}: gradients of rows past the sequence")
    return ref


# ------------------------------------------------------------------------------------------------ selector cases
@pytest.mark.parametrize("case", PADDED, ids=repr)
def test_attention_exact_padded(cuda_device, case):
    run_padded(case, cuda_device)


@pytest.mark.parametrize("case", TRAINING, ids=repr)
def test_attention_exact_training_shapes(cuda_device, case):
    ref = run_padded(case, cuda_device)
    print(f"{case}: certificate {ref['cert']}")


def test_attention_exact_noncausal_siglip(cuda_device):
    """Non-causal, 3 images of T = 729 in one launch, as the SigLIP tower runs it (no seqlens)."""
    from metamorph_b200 import ops
    case = NONCAUSAL
    s = case.selector()
    assert case.reaches <= regimes(case, s.late)
    B, T, H = len(s.lens), s.T, s.Hq
    _, q, k, v = _fused(s, cuda_device)
    ref = reference(s, 72 ** -0.5, cuda_device)
    out, lse = ops.attn_fwd(q, k, v, B, T, H, H, D, False, 72 ** -0.5)
    rows = torch.ones(B, T, dtype=torch.bool, device=cuda_device)
    check_fwd(out.view(B, T, H, D)[rows], lse.transpose(1, 2)[rows], ref, rows, "non-causal")


def test_attention_exact_packed(cuda_device):
    """attn_fwd_varlen / attn_bwd_varlen over 96 segments; gap rows keep 7.0 in out and NaN in dq / dk / dv."""
    from metamorph_b200 import ops
    case = PACKED
    s = case.selector()
    Hq, Hkv = s.Hq, s.Hkv
    starts, R = packed_offsets(s.lens, case.seed)
    segs = list(zip(starts, s.lens))
    tab = ops.SegmentTables(segs, cuda_device)
    assert tab.n_work_q > SMS
    W = (Hq + 2 * Hkv) * D
    qkv = torch.full((R, W), 3.0, dtype=torch.bfloat16)
    dout = torch.full((R, Hq * D), 3.0, dtype=torch.bfloat16)
    for b, (a, L) in enumerate(segs):
        qkv[a:a + L] = torch.cat([s.q[b, :L].reshape(L, -1), s.k[b, :L].reshape(L, -1), s.v[b, :L].reshape(L, -1)], 1)
        dout[a:a + L] = s.do[b, :L].reshape(L, -1)
    qkv, dout = qkv.to(cuda_device), dout.to(cuda_device)
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    ref = reference(s, SCALE_BWD, cuda_device)
    out = torch.full((R, Hq * D), 7.0, device=cuda_device, dtype=torch.bfloat16)
    _, lse = ops.attn_fwd_varlen(q, k, v, tab, Hq, Hkv, D, SCALE_BWD, out=out)
    g = torch.full((R, W), float("nan"), device=cuda_device, dtype=torch.bfloat16)
    dq, dk, dv = g[:, :Hq * D], g[:, Hq * D:(Hq + Hkv) * D], g[:, (Hq + Hkv) * D:]
    ops.attn_bwd_varlen(q, k, v, out, dout, lse, dq, dk, dv, tab, Hq, Hkv, D, SCALE_BWD)
    rows = torch.arange(s.T, device=cuda_device)[None, :] < torch.tensor(s.lens, device=cuda_device)[:, None]
    gather = torch.cat([torch.arange(a, a + L) for a, L in segs]).to(cuda_device)
    check_fwd(out[gather].view(-1, Hq, D), lse.transpose(1, 2)[rows], ref, rows, "packed")
    check_bwd(dq[gather].view(-1, Hq, D), dk[gather].view(-1, Hkv, D), dv[gather].view(-1, Hkv, D), ref, rows,
              "packed")
    gap = torch.ones(R, dtype=torch.bool, device=cuda_device)
    gap[gather] = False
    assert int(gap.sum()) > 0
    assert bool((out[gap] == 7.0).all()), "packed: out rows between segments were written"
    assert bool(torch.isnan(g[gap].float()).all()), "packed: gradient rows between segments were written"


@pytest.mark.parametrize("block_size", [16, 64, 256])
def test_attention_exact_paged_prefill(cuda_device, block_size):
    """attn_fwd_paged through a shuffled block table; pool rows past kv_len hold NaN."""
    from metamorph_b200 import ops
    case = PAGED
    s = case.selector()
    assert case.reaches <= regimes(case, s.late)
    Hq, Hkv, T = s.Hq, s.Hkv, s.T
    ref = reference(s, SCALE_ENGINE, cuda_device)
    gen = torch.Generator().manual_seed(block_size)
    max_blocks = T // block_size
    num_blocks = max_blocks + 5
    table = torch.randperm(num_blocks, generator=gen)[:max_blocks].to(torch.int32).to(cuda_device)
    q = s.q[0].reshape(T, -1).to(cuda_device)
    kk, vv = s.k[0].to(cuda_device), s.v[0].to(cuda_device)
    for q_start, n_q in PAGED_Q:
        kv = q_start + n_q
        kpool = torch.full((num_blocks, Hkv, block_size, D), float("nan"), device=cuda_device, dtype=torch.bfloat16)
        vpool = torch.full_like(kpool, float("nan"))
        pos = torch.arange(kv, device=cuda_device)
        blk, off = table[pos // block_size].long(), pos % block_size
        kpool[blk, :, off] = kk[:kv]
        vpool[blk, :, off] = vv[:kv]
        out = ops.attn_fwd_paged(q[q_start:kv], kpool, vpool, table, q_start, Hq, Hkv, D, SCALE_ENGINE)
        rows = torch.zeros(1, T, dtype=torch.bool, device=cuda_device)
        rows[0, q_start:kv] = True
        check_fwd(out.view(n_q, Hq, D), None, ref, rows, f"paged bs={block_size} q_start={q_start}")


# ------------------------------------------------------------------------------------------------ random data
def _peaked_long(T, Hq, Hkv, device, seed):
    """peaked_inputs of test_attention_edges_gpu.py at one sequence of T: queries 4 e + noise, planted keys scoring
    about +12 (key 5), -20 (key 140), +16 (key 263), +18 (key T / 2) and +20 (key T - 3)."""
    scale = D ** -0.5
    gen = torch.Generator(device=device).manual_seed(seed)
    e = torch.randn(D, device=device, generator=gen)
    e = e / e.norm()
    qkv = 1.5 * torch.randn(T, (Hq + 2 * Hkv) * D, device=device, generator=gen)
    qkv[:, :Hq * D].view(T, Hq, D).add_(4 * e)
    kv = qkv[:, Hq * D:(Hq + Hkv) * D].view(T, Hkv, D)
    for j, score in ((5, 12.0), (140, -20.0), (263, 16.0), (T // 2, 18.0), (T - 3, 20.0)):
        kv[j] = score / (4 * scale) * e + 0.1 * kv[j]
    return qkv.bfloat16(), torch.randn(T, Hq * D, device=device, generator=gen).bfloat16()


def test_attention_random_peaked_bench_shape(cuda_device):
    """Random peaked data at T = 4096, 32 / 8 heads: each of out, lse, dQ, dK, dV no worse than twice torch's bf16
    path against fp64 (computed one kv head at a time), with the floors of the T = 523 check."""
    from metamorph_b200 import ops
    from tests.test_attention_edges_gpu import _allowed, _ref64, _torch_bf16
    T, Hq, Hkv = 4096, 32, 8
    G, scale = Hq // Hkv, D ** -0.5
    qkv, dout = _peaked_long(T, Hq, Hkv, cuda_device, seed=4096)
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    out, lse = ops.attn_fwd(q, k, v, 1, T, Hq, Hkv, D, True, scale)
    g = torch.full_like(qkv, float("nan"))
    dq, dk, dv = g[:, :Hq * D], g[:, Hq * D:(Hq + Hkv) * D], g[:, (Hq + Hkv) * D:]
    ops.attn_bwd(q, k, v, out, dout, lse, dq, dk, dv, 1, T, Hq, Hkv, D, scale)
    allowed = _allowed([T], T, True, cuda_device)
    heads = lambda x, H: x.view(T, H, D).transpose(0, 1)                       # [H, T, D]
    got = {"out": heads(out, Hq), "dQ": heads(dq, Hq), "dK": heads(dk, Hkv), "dV": heads(dv, Hkv)}
    ref = {n: [] for n in ("out", "lse", "dQ", "dK", "dV")}
    tor = {n: [] for n in ref}
    for hk in range(Hkv):
        hs = slice(hk * G, hk * G + G)
        qh, doh = heads(q, Hq)[hs][None], heads(dout, Hq)[hs][None]
        kh, vh = heads(k, Hkv)[hk:hk + 1][None], heads(v, Hkv)[hk:hk + 1][None]
        for store, fn in ((ref, _ref64), (tor, _torch_bf16)):
            o, l, (gq, gk, gv) = fn(qh, kh, vh, doh, allowed, scale, G)
            for n, x in zip(("out", "lse", "dQ", "dK", "dV"), (o, l, gq, gk, gv)):
                store[n].append(x[0].to(torch.float64 if fn is _ref64 else x.dtype))
            del o, l, gq, gk, gv
    ratios = {}
    for n in ("out", "dQ", "dK", "dV"):
        r, t = torch.cat(ref[n]), torch.cat(tor[n])
        g_max, t_max = assert_no_worse_than(got[n], r, t, f"T=4096 {n}", floor=2.0 ** -12 * float(r.abs().max()))
        ratios[n] = g_max / t_max
    r, t = torch.cat(ref["lse"]), torch.cat(tor["lse"])
    g_max, t_max = assert_no_worse_than(lse[0], r, t, "T=4096 lse", floor=2.0 ** -14 * float(r.abs().max()))
    ratios["lse"] = g_max / t_max
    print("max error / torch bf16 max error: " + ", ".join(f"{n} {x:.3f}" for n, x in ratios.items()))
