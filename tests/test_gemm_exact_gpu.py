"""`mm_gemm_bf16` and the decode weight-streaming GEMMs against fp64, at the edges of their schedules.

Main tool: integer-exact cases. Operands are bf16 integers in {-1, 0, 1} (with at most 8192 non-zero terms per dot
product), so every product is exact and every partial sum is an integer below 2^13 in magnitude by construction: the
result does not depend on how the tensor core orders, aligns or rounds its fp32 accumulator. The fp64 product of the same
values is then the exact answer; fp32 outputs must equal it and bf16 outputs must equal it rounded once to bf16 (round to
nearest even, as pack_bf16x2 does). alpha is a power of two and bias / residual are integers, so the linear epilogues stay
exact too. A dropped, doubled or misplaced k-slice, row group, tile or column chunk changes some element.

Every case derives from its shape and the device's SM count the part of the schedule it is meant to reach (tiles per CTA,
k blocks against the ring depth, tile width, a partial rasterisation group, the wide kernel's K split) and asserts it.
The schedule is not exported, so it is restated below from the kernel sources with line references.

Poisoning: outputs start as NaN (unless accumulating), so every element must be written; operands are views into larger
buffers with NaN past K (columns of K-major operands, rows of MN-major ones) and past M / N, so a read of the padding
shows; outputs sit inside buffers whose surrounding rows and columns hold a sentinel that must survive.
"""
import math

import pytest
import torch

from tests.exact import assert_equal, assert_within, gamma, ints, ulp_bf16

pytestmark = pytest.mark.gpu

NAN = float("nan")
SENT = 12288.0            # sentinel around output views: exact in bf16 and fp32, larger than any result here

# ------------------------------------------------------------------------------------------------ the schedule, restated
# metamorph_b200/csrc/gemm_tcgen05.cu
BM, BK = 128, 64                                  # l.25-26: tile rows, k per ring stage
K_STAGES = {128: 5, 256: 3}                       # l.58: Cfg<BN>::kStages


def cdiv(a, b):
    return -(-a // b)


def group_m(K):
    """Row blocks per rasterisation group: clamp(16 MB / (BM * K * 2 bytes), 11, 64) (l.425-427)."""
    return min(64, max(11, (16 << 20) // (BM * K * 2)))


class Sched:
    """What one launch does: grid = min(#tiles, #SMs) persistent CTAs (l.418-419), CTA b runs tiles b, b + grid, ..."""

    def __init__(self, M, N, K, bn, sms):
        self.bn, self.stages = bn, K_STAGES[bn]
        self.num_m, self.num_n = cdiv(M, BM), cdiv(N, bn)
        self.tiles = self.num_m * self.num_n
        self.grid = min(self.tiles, sms)
        self.max_per_cta, self.min_per_cta = cdiv(self.tiles, self.grid), self.tiles // self.grid
        self.kb = cdiv(K, BK)
        self.gm = group_m(K)
        self.partial_group = self.num_m > self.gm and self.num_m % self.gm != 0


# metamorph_b200/csrc/decode_wide.cu l.187-192
def wide_splits(N, K, sms):
    slabs, nk, s = cdiv(N, 128), cdiv(K, 64), 1
    while s < 8 and 10 * slabs * s < 9 * sms and 2 * (s + 1) <= nk:
        s += 1
    return s


def _sms(device):
    return torch.cuda.get_device_properties(device).multi_processor_count


# ------------------------------------------------------------------------------------------------ poisoned buffers
def operand(data):
    """`data` [rows, cols] copied into a buffer with >= 1 NaN column past cols (pitch a multiple of 8) and one NaN row
    past rows; returns the view."""
    rows, cols = data.shape
    buf = torch.full((rows + 1, cdiv(cols + 1, 8) * 8), NAN, dtype=torch.bfloat16, device=data.device)
    buf[:rows, :cols] = data
    return buf[:rows, :cols]


class Out:
    """An [M, N] output view at (1, 8) inside a buffer with one sentinel row above and below and >= 8 sentinel columns on
    each side."""

    def __init__(self, M, N, dtype, device, init=NAN):
        self.M, self.N = M, N
        self.buf = torch.full((M + 2, cdiv(N + 16, 8) * 8), SENT, dtype=dtype, device=device)
        self.view = self.buf[1:1 + M, 8:8 + N]
        if isinstance(init, torch.Tensor):
            self.view.copy_(init)
        else:
            self.view.fill_(init)

    def check_sentinels(self, what):
        keep = torch.ones(self.buf.shape, dtype=torch.bool, device=self.buf.device)
        keep[1:1 + self.M, 8:8 + self.N] = False
        bad = self.buf[keep] != SENT
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the output view were written"


def int_operands(M, N, K, a_mn, b_mn, device, seed):
    """{-1, 0, 1} operands in the storage each layout uses, as poisoned views, and their fp64 product [M, N].
    Above K = 8192 the A rows are thinned (row i keeps k with (k + i) % s == 0) to at most 8192 non-zero terms, so the
    partial sums stay below 2^13 whatever the depth; every k position is still used by some rows."""
    gen = torch.Generator(device=device).manual_seed(seed)
    a = ints((M, K), -1, 1, device, gen=gen)
    b = ints((N, K), -1, 1, device, gen=gen)
    if K > 8192:
        s = cdiv(K, 8192)
        keep = (torch.arange(K, device=device)[None, :] + torch.arange(M, device=device)[:, None]) % s == 0
        a = a * keep
    c64 = a.double() @ b.double().t()
    a_v = operand(a.t().contiguous() if a_mn else a)
    b_v = operand(b.t().contiguous() if b_mn else b)
    return a_v, b_v, c64


LAYOUTS = {"KK": (False, False), "KM": (False, True), "MM": (True, True)}   # (A MN-major, B MN-major)


# ------------------------------------------------------------------------------------------------ the case list
def _cases():
    """(id, layout, bn, shape(sms) -> (M, N, K), regime(sched, sms) -> bool). The id names the regime; the test asserts it."""
    cs = []
    for bn, lay in ((128, "KK"), (256, "KM"), (128, "MM"), (256, "MM")):
        # tiles per CTA: one M-tail tile column (N < BN) with #tiles = #SMs - 1, #SMs, #SMs + 1
        cs.append((f"bn{bn}-{lay}-tiles=sms-1", lay, bn, lambda s, bn=bn: (128 * (s - 1) - 61, bn - 24, 200),
                   lambda S, s: S.tiles == s - 1 and S.max_per_cta == 1))
        cs.append((f"bn{bn}-{lay}-tiles=sms", lay, bn, lambda s, bn=bn: (128 * s, bn, 65),
                   lambda S, s: S.tiles == s and S.max_per_cta == 1 == S.min_per_cta))
        cs.append((f"bn{bn}-{lay}-tiles=sms+1", lay, bn, lambda s, bn=bn: (128 * (s + 1) - 1, bn - 100, 56),
                   lambda S, s: S.tiles == s + 1 and S.max_per_cta == 2 and S.min_per_cta == 1))
        # between one and two tiles per CTA, and three or more
        cs.append((f"bn{bn}-{lay}-tiles/cta=1..2", lay, bn, lambda s, bn=bn: (128 * (s // 2), 3 * bn - 5, 64),
                   lambda S, s: S.min_per_cta == 1 and S.max_per_cta == 2))
        cs.append((f"bn{bn}-{lay}-tiles/cta>=3-N%32", lay, bn, lambda s, bn=bn: (128 * (3 * s // 4 + 1) - 63, 4 * bn - 31, 16),
                   lambda S, s: S.max_per_cta >= 3))
    # k blocks per tile against the ring depth, with >= 3 tiles per CTA so the ring phase carries across tiles; the last
    # row tile has 63 rows, so its second consumer warpgroup owns none
    for bn in (128, 256):
        st = K_STAGES[bn]
        for kb_name, K in (("1", 8), ("stages-1", 64 * (st - 1)), ("stages", 64 * st - 1), ("stages+1", 64 * st + 1)):
            for lay in ("KK", "MM") if kb_name in ("1", "stages+1") else ("KM",):
                kb = cdiv(K, BK)
                cs.append((f"bn{bn}-{lay}-kb={kb_name}-K{K}", lay, bn, lambda s, bn=bn, K=K: (128 * s - 65, 3 * bn - 7, K),
                           lambda S, s, kb=kb: S.kb == kb and S.max_per_cta >= 3))
    # K edges, in all three layouts
    for K in (1, 8, 16, 56, 64, 65, 200):
        for lay in LAYOUTS:
            bn = 256 if K % 2 else 128
            cs.append((f"bn{bn}-{lay}-K{K}", lay, bn, lambda s, K=K: (300, 520, K), lambda S, s: True))
    # M tails (M < 64: one consumer warpgroup owns no rows) at N % 256 = 128, where the second half of the last 256-wide
    # tile is skipped
    for M in (1, 63, 64, 65, 127, 129):
        lay = ("KK", "KM", "MM")[M % 3]
        cs.append((f"bn256-{lay}-M{M}-N%256=128", lay, 256, lambda s, M=M: (M, 384, 136), lambda S, s: S.num_n == 2))
    # N tails
    for N, lay in ((1, "KK"), (17, "KM"), (100, "MM"), (257, "KK"), (2 * 256 + 96, "KM")):
        for bn in (128, 256):
            cs.append((f"bn{bn}-{lay}-N{N}", lay, bn, lambda s, N=N: (129, N, 72), lambda S, s: True))
    # a partial last rasterisation group: K = 4096 gives groups of 16 row blocks; 33 row blocks = 16 + 16 + 1
    for bn, lay in ((128, "KK"), (256, "MM")):
        cs.append((f"bn{bn}-{lay}-raster-33=16+16+1", lay, bn, lambda s: (33 * 128 - 5, 3 * 256 - 40, 4096),
                   lambda S, s: S.gm == 16 and S.num_m == 33 and S.partial_group))
    # lm_head depth at reduced width: the dgrad dX = dlogits . W has K = 128258 (K % 64 = 2) and dlogits' pitch 128264
    for bn in (128, 256):
        cs.append((f"bn{bn}-KM-lm_head-dgrad-K128258", "KM", bn, lambda s: (200, 96, 128258),
                   lambda S, s: S.kb * BK - 128258 == 62))
    return cs


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gemm_integer_exact_at_schedule_edges(cuda_device, case):
    from metamorph_b200 import ops
    name, lay, bn, shape, regime = case
    sms = _sms(cuda_device)
    M, N, K = shape(sms)
    S = Sched(M, N, K, bn, sms)
    assert regime(S, sms), f"{name}: M={M} N={N} K={K} does not reach its regime: {vars(S)}"
    a_mn, b_mn = LAYOUTS[lay]
    a, b, c64 = int_operands(M, N, K, a_mn, b_mn, cuda_device, seed=M * 31 + N * 7 + K)
    if K == 128258:
        assert a.stride(0) == 128264
    for dtype in (torch.float32, torch.bfloat16):
        o = Out(M, N, dtype, cuda_device)
        ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=o.view, out_dtype=dtype, force_bn=bn)
        assert_equal(o.view, c64.to(dtype), f"{name} {dtype}")
        o.check_sentinels(f"{name} {dtype}")


def test_gemm_lm_head_wgrad_accumulates_fp32_across_chunks(cuda_device):
    """dW[V, H] += dlogits[chunk]^T X[chunk] per row chunk in fp32, as the lm_head weight gradient is formed: M = V = 128258
    (pitch 128264), (MN, MN) layout, K = the chunk's (arbitrary) row count. The first call overwrites NaN."""
    from metamorph_b200 import ops
    sms = _sms(cuda_device)
    V, H = 128258, 96
    o = Out(V, H, torch.float32, cuda_device)
    want = torch.zeros(V, H, dtype=torch.float64, device=cuda_device)
    for i, (rows, bn) in enumerate(((77, 128), (50, 256), (131, 128))):
        S = Sched(V, H, rows, bn, sms)
        assert S.max_per_cta >= 3, vars(S)
        a, b, c64 = int_operands(V, H, rows, True, True, cuda_device, seed=100 + i)
        assert a.stride(0) == 128264
        ops.gemm(a, b, a_mn=True, b_mn=True, out=o.view, out_dtype=torch.float32, accumulate=i > 0, force_bn=bn)
        want += c64
        assert_equal(o.view, want.float(), f"lm_head wgrad after chunk {i}")
    o.check_sentinels("lm_head wgrad")


# ------------------------------------------------------------------------------------------------ every epilogue, multi-tile
def _epi_shape(sms):
    # N = 1160: the last 32-column chunk is partial (N % 32 = 8) and N % 256 = 136; K = 320 = 5 k blocks. The SwiGLU
    # epilogues need N % 32 == 0 and take the first N_SWIGLU = 1152 columns (N_SWIGLU % 256 = 128).
    return 128 * (sms // 3) - 37, 1160, 320


N_SWIGLU = 1152


def _nonlinear_bound(ref, slack):
    """Two bf16 ulps of the fp64 value (the fp32 evaluation is off by a few ulps of fp32, the store rounds once) plus
    `slack`, an absolute term for the cancellation near zero, derived per epilogue below."""
    return 2 * ulp_bf16(ref) + slack


def _swiglu_ref(c, alpha):
    """C columns interleaved [16 gate | 16 up] per 32: out[m, 16 j + i] = silu(g) * u of chunk j."""
    M, N = c.shape
    v = (c * alpha).view(M, N // 32, 2, 16)
    g, u = v[:, :, 0], v[:, :, 1]
    return (g * torch.sigmoid(g) * u).reshape(M, N // 2), g.reshape(M, -1), u.reshape(M, -1)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("lay", list(LAYOUTS))
def test_gemm_every_epilogue_on_multi_tile_shapes(cuda_device, lay, bn):
    from metamorph_b200 import ops
    sms = _sms(cuda_device)
    M, N, K = _epi_shape(sms)
    S = Sched(M, N, K, bn, sms)
    assert S.max_per_cta >= 2 and S.kb == 5 and N % 32 != 0, vars(S)
    a_mn, b_mn = LAYOUTS[lay]
    a, b, c = int_operands(M, N, K, a_mn, b_mn, cuda_device, seed=7 + bn)
    gen = torch.Generator(device=cuda_device).manual_seed(11)
    bias_buf = torch.full((N + 64,), NAN, dtype=torch.bfloat16, device=cuda_device)
    bias_buf[:N] = ints((N,), -8, 8, cuda_device, gen=gen)
    bias = bias_buf[:N]                     # NaN past N: the bias of columns past N must not be read
    bias64 = bias.double()
    r = ints((M, N), -64, 64, cuda_device, gen=gen)
    kw = dict(a_mn=a_mn, b_mn=b_mn, force_bn=bn)

    def run(what, dtype=torch.bfloat16, init=NAN, **k):
        o = Out(M, N, dtype, cuda_device, init=init)
        ops.gemm(a, b, out=o.view, out_dtype=dtype, **kw, **k)
        o.check_sentinels(f"{lay} bn={bn} {what}")
        return o.view

    def exact(what, got, want):
        assert_equal(got, want.to(got.dtype), f"{lay} bn={bn} {what}")

    exact("store", run("store"), c)
    exact("alpha", run("alpha", alpha=0.25), c * 0.25)
    exact("bias", run("bias", alpha=0.5, bias=bias, epilogue=ops.EPI_BIAS), c * 0.5 + bias64)
    r_v = operand(r)
    exact("resid", run("resid", alpha=0.5, resid=r_v, epilogue=ops.EPI_RESID), c * 0.5 + r.double())
    exact("bias+resid", run("bias+resid", alpha=0.5, bias=bias, resid=r_v, epilogue=ops.EPI_BIAS_RESID),
          c * 0.5 + bias64 + r.double())
    # residual in place: C aliases R
    o = Out(M, N, torch.bfloat16, cuda_device, init=r)
    ops.gemm(a, b, out=o.view, resid=o.view, alpha=0.5, epilogue=ops.EPI_RESID, **kw)
    exact("resid in place", o.view, c * 0.5 + r.double())
    o.check_sentinels("resid in place")
    # accumulate: C += result in C's own dtype; twice in fp32 (accumulation across calls)
    exact("bf16 accumulate", run("bf16 accumulate", init=r, accumulate=True), c + r.double())
    r32 = r.float() * 4
    o = Out(M, N, torch.float32, cuda_device, init=r32)
    for _ in range(2):
        ops.gemm(a, b, out=o.view, out_dtype=torch.float32, accumulate=True, **kw)
    exact("fp32 accumulate x2", o.view, r32.double() + 2 * c)
    o.check_sentinels("fp32 accumulate")

    # GELUs: alpha = 2^-3 keeps the pre-activation x = C/8 + bias exact in fp32. 0.5 x (1 + erff(x / sqrt 2)) (and the
    # tanhf form) is within a few fp32 ulps of the value except where 1 + erf(.) cancels (x << 0): there erff's error of
    # <= 2 ulp at 1 (2^-22) times 0.5 |x| is absolute, so slack = |x| 2^-21 (twice that).
    x = c * 0.125 + bias64
    g_erf = 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    got = run("gelu_erf", alpha=0.125, bias=bias, epilogue=ops.EPI_BIAS_GELU_ERF)
    assert_within(got, g_erf, _nonlinear_bound(g_erf, x.abs() * 2 ** -21), f"{lay} bn={bn} gelu_erf")
    kk = math.sqrt(2 / math.pi)
    g_tanh = 0.5 * x * (1 + torch.tanh(kk * (x + 0.044715 * x ** 3)))
    got = run("gelu_tanh", alpha=0.125, bias=bias, epilogue=ops.EPI_BIAS_GELU_TANH)
    assert_within(got, g_tanh, _nonlinear_bound(g_tanh, x.abs() * 2 ** -21), f"{lay} bn={bn} gelu_tanh")

    N = N_SWIGLU
    b, c = (b[:, :N] if b_mn else b[:N]), c[:, :N]
    if lay == "KK":     # SwiGLU fuses gate/up projections, which are K-major (nn.Linear)
        act, _, _ = _swiglu_ref(c, 0.125)
        for with_aux in (False, True):
            aux = Out(M, N, torch.bfloat16, cuda_device) if with_aux else None
            o = Out(M, N // 2, torch.bfloat16, cuda_device)
            ops.gemm(a, b, out=o.view, aux=aux.view if aux else None, alpha=0.125, epilogue=ops.EPI_SWIGLU, **kw)
            # silu(g) = g / (1 + __expf(-g)): __expf is within (2 + 1.2 |g|) fp32 ulps, far below a bf16 ulp of the result
            assert_within(o.view, act, _nonlinear_bound(act, 2.0 ** -40), f"bn={bn} swiglu aux={with_aux}")
            o.check_sentinels("swiglu")
            if aux:
                exact("swiglu aux", aux.view, c * 0.125)
                aux.check_sentinels("swiglu aux")
    if lay == "KM":     # SwiGLU backward fused into the down_proj dgrad (B = W_down stored [H, I], MN-major)
        d = c * 0.125
        gu = ints((M, 2 * N), -16, 16, cuda_device, gen=gen) * 0.125     # gate|up in [-2, 2], exact in bf16
        gu_v = Out(M, 2 * N, torch.bfloat16, cuda_device, init=gu)
        o = Out(M, N, torch.bfloat16, cuda_device)
        ops.gemm(a, b, out=o.view, aux=gu_v.view, alpha=0.125, epilogue=ops.EPI_SWIGLU_BWD, **kw)
        blocks = gu.double().view(M, N // 16, 2, 16)
        g, u = blocks[:, :, 0].reshape(M, N), blocks[:, :, 1].reshape(M, N)
        s = torch.sigmoid(g)
        av = g * s
        dg = d * u * (s + av * (1 - s))
        du = d * av
        # s + a (1 - s) cancels near g = -1.28; the fp32 terms carry (2 + 1.2 |g|) ulps from __expf and a few roundings:
        # slack = 2^-16 |d u| (s + |a| (1 - s)), still 2^-7 of a bf16 ulp of the terms
        slack = 2.0 ** -16 * (d * u).abs() * (s + av.abs() * (1 - s))
        assert_within(o.view, av * u, _nonlinear_bound(av * u, 2.0 ** -40), f"bn={bn} swiglu_bwd act")
        got = gu_v.view.double().view(M, N // 16, 2, 16)
        assert_within(got[:, :, 0].reshape(M, N), dg, _nonlinear_bound(dg, slack), f"bn={bn} swiglu_bwd dgate")
        assert_within(got[:, :, 1].reshape(M, N), du, _nonlinear_bound(du, 2.0 ** -40), f"bn={bn} swiglu_bwd dup")
        o.check_sentinels("swiglu_bwd act")
        gu_v.check_sentinels("swiglu_bwd aux")


# ------------------------------------------------------------------------------------------------ random data: derived bound
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("lay,M,N,K", [("KK", 4000, 1160, 4096), ("KM", 1541, 2100, 1000), ("MM", 2900, 4104, 333)])
def test_gemm_random_within_derived_bound(cuda_device, lay, M, N, K, bn):
    """|C - C64| <= gamma_K sum_k |a_ik b_kj| (+ half a bf16 ulp of C for the bf16 store), per element.
    bf16 x bf16 products are exact in fp32, so only the additions err; each output is a chain of at most K of them.
    The unit roundoff is taken as u = 2^-23, twice fp32's, to allow an accumulator that truncates instead of rounding."""
    from metamorph_b200 import ops
    S = Sched(M, N, K, bn, _sms(cuda_device))
    assert S.tiles > 1, vars(S)
    a_mn, b_mn = LAYOUTS[lay]
    gen = torch.Generator(device=cuda_device).manual_seed(M + N + K)
    a = torch.randn(M, K, device=cuda_device, generator=gen).bfloat16()
    b = torch.randn(N, K, device=cuda_device, generator=gen).bfloat16()
    c64 = a.double() @ b.double().t()
    bound = gamma(K, u=2.0 ** -23) * (a.double().abs() @ b.double().abs().t())
    av, bv = operand(a.t().contiguous() if a_mn else a), operand(b.t().contiguous() if b_mn else b)
    o = Out(M, N, torch.float32, cuda_device)
    ops.gemm(av, bv, a_mn=a_mn, b_mn=b_mn, out=o.view, out_dtype=torch.float32, force_bn=bn)
    worst = assert_within(o.view, c64, bound, f"{lay} bn={bn} fp32")
    print(f"{lay} bn={bn} M={M} N={N} K={K}: worst fp32 err / bound = {worst:.3g}")
    o16 = Out(M, N, torch.bfloat16, cuda_device)
    ops.gemm(av, bv, a_mn=a_mn, b_mn=b_mn, out=o16.view, force_bn=bn)
    assert_within(o16.view, c64, bound + 0.5 * ulp_bf16(torch.maximum(o16.view.double().abs(), c64.abs())),
                  f"{lay} bn={bn} bf16")
    o.check_sentinels("random fp32")
    o16.check_sentinels("random bf16")


# ------------------------------------------------------------------------------------------------ schedule invariance
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("lay", list(LAYOUTS))
def test_gemm_rows_do_not_depend_on_their_tile(cuda_device, lay, bn):
    """With the same BN and K, a row's bits do not depend on which tile or CTA computes it (rows r0.. of a sliced A land
    in another tile position: r0 = 200 is not a multiple of 128), and repeated calls give the same bits. Random data,
    so the check is not an artefact of exact arithmetic. Equality across BN = 128 and 256 is not promised."""
    from metamorph_b200 import ops
    M, N, K = 3000, 1160, 1000
    r0, r1 = 200, 2963
    a_mn, b_mn = LAYOUTS[lay]
    gen = torch.Generator(device=cuda_device).manual_seed(5)
    a = torch.randn((K, M) if a_mn else (M, K), device=cuda_device, generator=gen).bfloat16()
    b = torch.randn((K, N) if b_mn else (N, K), device=cuda_device, generator=gen).bfloat16()
    full = [ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn) for _ in range(3)]
    assert torch.equal(full[0], full[1]) and torch.equal(full[0], full[2]), "repeated calls differ"
    part = ops.gemm(a[:, r0:r1] if a_mn else a[r0:r1], b, a_mn=a_mn, b_mn=b_mn, force_bn=bn)
    assert_equal(part, full[0][r0:r1], f"{lay} bn={bn}: rows {r0}:{r1} computed alone")


# ------------------------------------------------------------------------------------------------ weight-streaming GEMMs
# (m, N, K, split of the wide kernel); the splits hold for any card with >= 100 SMs
SKINNY = [(1, 200, 1024, None), (7, 1000, 416, None), (32, 520, 512, None),
          (33, 300, 96, 1), (77, 1000, 416, 3), (100, 520, 512, 4), (128, 200, 1024, 8)]


@pytest.mark.parametrize("m,N,K,split", SKINNY, ids=[f"m{m}-N{N}-K{K}" + (f"-split{s}" if s else "")
                                                     for m, N, K, s in SKINNY])
def test_skinny_gemms_integer_exact(cuda_device, m, N, K, split):
    """mm_skinny_gemm (m <= 32) and mm_skinny_gemm_wide (m >= 33) on {-1, 0, 1} activations and {-1/8, 0, 1/8} weights:
    every partial sum is a multiple of 1/8 below 2^10, exact in fp32 in any order, so a dropped or doubled split partial
    or k stage shows. Every SK_* epilogue; ragged N."""
    from metamorph_b200 import ops
    sms = _sms(cuda_device)
    if split is not None:
        assert wide_splits(N, K, sms) == split, f"K split {wide_splits(N, K, sms)} on {sms} SMs"
    gen = torch.Generator(device=cuda_device).manual_seed(m * 1000 + N)
    x = operand(ints((m, K), -1, 1, cuda_device, gen=gen))
    w = operand(ints((N, K), -1, 1, cuda_device, gen=gen) * 0.125)
    c = x.double() @ w.double().t()
    bias = ints((N,), -8, 8, cuda_device, gen=gen)
    r = ints((m, N), -64, 64, cuda_device, gen=gen)
    for epi, want, k in ((ops.SK_STORE, c, {}), (ops.SK_BIAS, c + bias.double(), dict(bias=bias)),
                         (ops.SK_RESID, c + r.double(), dict(resid=operand(r)))):
        for dtype in (torch.float32, torch.bfloat16):
            o = Out(m, N, dtype, cuda_device)
            ops.skinny_gemm(x, w, epilogue=epi, out=o.view, **k)
            assert_equal(o.view, want.to(dtype), f"skinny m={m} epi={epi} {dtype}")
            o.check_sentinels(f"skinny m={m} epi={epi}")
    xg = c + bias.double()
    ref = 0.5 * xg * (1 + torch.erf(xg / math.sqrt(2)))
    o = Out(m, N, torch.bfloat16, cuda_device)
    ops.skinny_gemm(x, w, bias=bias, epilogue=ops.SK_BIAS_GELU, out=o.view)
    assert_within(o.view, ref, 2 * ulp_bf16(ref) + xg.abs() * 2 ** -21, f"skinny m={m} gelu")
    o.check_sentinels("skinny gelu")
    N2 = cdiv(N, 32) * 32
    w2 = operand(ints((N2, K), -1, 1, cuda_device, gen=gen) * 0.125)
    act, _, _ = _swiglu_ref(x.double() @ w2.double().t(), 1.0)
    o = Out(m, N2 // 2, torch.bfloat16, cuda_device)
    ops.skinny_gemm(x, w2, epilogue=ops.SK_SWIGLU, out=o.view)
    assert_within(o.view, act, 2 * ulp_bf16(act) + 2.0 ** -40, f"skinny m={m} swiglu")
    o.check_sentinels("skinny swiglu")
