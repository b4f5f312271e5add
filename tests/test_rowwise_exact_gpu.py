"""The norm, RoPE, activation, copy and vision-reduction kernels against fp64 restatements, at their row, vector and
grid-stride edges (H100 only).

Each kernel computes in fp32 and rounds once (or twice, where the reference it mirrors does) to bf16. The checks bound
the fp32 error before each rounding and require the bf16 result to lie between the roundings of the fp64 value minus
and plus that bound (`tests/exact.py` `assert_rounds_within` / `assert_between`): bit equality away from a rounding
boundary, one of the two neighbours near it. The schedules the cases are derived from are restated next to each test,
with the source lines they come from; every case asserts the regime it is meant to reach.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.exact import U, assert_between, assert_equal, assert_rounds_within, gamma, round_bf16_from_fp64

pytestmark = pytest.mark.gpu

F32_TINY = 2.0 ** -148           # absolute slack for fp32 results in the subnormal range


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def _rnd(x):
    return round_bf16_from_fp64(x).double()


# ------------------------------------------------------------------------------------------------ RMSNorm forward
# norm_rope.cu:306-322: VPT = ceil(H / 8 / 256) 8-wide vectors per thread, instantiated as 1, 2 or 4 (3 runs as 4);
# grid = min(M, cap) blocks of 256 threads, cap = #SMs * 8 (VPT <= 2) or #SMs * 2 (VPT = 4). Block b owns rows b,
# b + grid, ...; norm_rope.cu:39-62 prefetches row r + grid before reducing row r, and alternates red[0] / red[1].
# Per row: each thread adds its 8 * VPT squares (f.x^2 + f.y^2 pairs), warp_sum (5 levels), then 8 warp partials in
# order: a chain of at most 8 * VPT + 13 fp32 additions of exact products.
def rms_vpt(H):
    v = -(-(H // 8) // 256)
    return 4 if v > 2 else v


def rms_cap(H, sms):
    return sms * (8 if rms_vpt(H) <= 2 else 2)


def rmsnorm_interval(x, w, eps):
    """Bounds on the kernel's y = bf16(w * bf16(x * rstd)) (HF LlamaRMSNorm), per element.

    rstd: S = sum x^2 is computed with relative error gamma_n (n = 8 VPT + 13, positive terms); S / H and + eps add a
    rounding each (2u); rsqrtf is within 2 ulp <= 4u of its argument's exact rsqrt, and rsqrt halves a relative error:
    |rstd - rstd64| <= rstd64 * d_r, d_r = 1.01 * (0.5 (gamma_n + 2u) + 4u) (1.01 covers the products of small terms).
    n = fl(x * rstd): |n - x rstd64| <= |x rstd64| (d_r + u) * 1.01, then rounded to bf16: n is one of the values
    between round(n64 - e) and round(n64 + e). w * n is exact in fp32 (8 x 8 bits), so y is the single rounding of
    w * n for one of those n: y lies between round(w n_lo) and round(w n_hi)."""
    x64, w64 = x.double(), w.double()
    H = x.shape[1]
    n = 8 * rms_vpt(H) + 13
    eps32 = _f32(eps)
    rstd = 1.0 / torch.sqrt(x64.pow(2).mean(1, keepdim=True) + eps32)
    d_r = 1.01 * (0.5 * (gamma(n) + 2 * U) + 4 * U)
    n64 = x64 * rstd
    e = n64.abs() * (d_r + U) * 1.01
    n_lo, n_hi = _rnd(n64 - e), _rnd(n64 + e)
    ya, yb = _rnd(w64 * n_lo), _rnd(w64 * n_hi)
    return torch.minimum(ya, yb), torch.maximum(ya, yb)


def rms_inputs(M, H, dev, seed):
    """randn rows scaled by 2^(r mod 16 - 8) (a neighbour's rstd is off by a power of two), and one-hot rows: mass in
    column 0 (vector 0) and in the last column (vector nvec - 1, which sits in the last VPT slot)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, H, generator=g, dtype=torch.float64)
    x *= torch.pow(2.0, (torch.arange(M) % 16 - 8).double())[:, None]
    for r, col in ([(M // 2, 0)] if M > 2 else []) + [(M - 1, H - 1)]:
        x[r] = 0
        x[r, col] = 3.0 * 2.0 ** (r % 16 - 8)
    w = (1 + 0.1 * torch.randn(H, generator=g)).bfloat16()
    return x.bfloat16().to(dev), w.to(dev)


@pytest.mark.parametrize("H", [8, 2048, 2056, 4096, 4104, 8192])
@pytest.mark.parametrize("Mk", ["1", "cap-1", "cap", "cap+1", "3cap+5"])
def test_rmsnorm_fwd_rounds_like_hf(cuda_device, H, Mk):
    from metamorph_b200 import ops
    cap = rms_cap(H, _sms(cuda_device))
    M = {"1": 1, "cap-1": cap - 1, "cap": cap, "cap+1": cap + 1, "3cap+5": 3 * cap + 5}[Mk]
    grid = min(M, cap)
    rows_per_block = -(-M // grid)
    assert rows_per_block == {"1": 1, "cap-1": 1, "cap": 1, "cap+1": 2, "3cap+5": 4}[Mk]
    assert rms_vpt(H) == {8: 1, 2048: 1, 2056: 2, 4096: 2, 4104: 4, 8192: 4}[H]
    x, w = rms_inputs(M, H, cuda_device, seed=H + M)
    buf = torch.full((M + 3, H), float("nan"), device=cuda_device, dtype=torch.bfloat16)
    ops.rmsnorm(x, w, 1e-5, out=buf[:M])
    lo, hi = rmsnorm_interval(x, w, 1e-5)
    assert_between(buf[:M], lo, hi, f"rmsnorm H={H} M={M} (VPT {rms_vpt(H)}, {rows_per_block} rows per block)")
    assert bool(torch.isnan(buf[M:]).all()), "rows past M were written"


# ------------------------------------------------------------------------------------------------ LayerNorm
# norm_rope.cu:206-260, 299-302: grid = min(M, #SMs * 8) blocks of 256 threads, grid-stride over rows; each thread
# holds up to kMaxVec = 4 vectors. Two block_sum reductions per row (mean, then sum of (x - mean)^2): per-thread
# chains of at most 2 * 8 * VPT additions, then 5 + 5 shuffle levels.
def layernorm_ref(x, w, b, eps):
    """fp64 LayerNorm and a bound on the kernel's fp32 error before its one bf16 rounding, per element.

    mean: sum x with |error| <= gamma_n1 sum|x| (n1 = 16 VPT + 10), / H one more rounding:
      dmu = 1.01 (gamma_n1 sum|x| / H + u (|mu| + gamma_n1 sum|x| / H)).
    d = fl(x - mu_hat): e_i = dmu + u (|d_i| + dmu).
    var: sum d_hat^2 (products rounded: n2 = n1 + 1) differs from sum d^2 by at most E1 = sum(2 |d| e + e^2) plus
      gamma_n2 (sum d^2 + E1); / H and + eps add 2u: rho = that / (H var_eps) + 2u; rsqrtf 2 ulp (4u) and the square
      root halve rho: d_r = 1.01 (0.5 rho + 4u).
    y = d_hat * rstd * w + b, three roundings: err = 1.01 (|w| r (e_i + |d_i| (d_r + 2u)) + u |y64|)."""
    x64, w64, b64 = x.double(), w.double(), b.double()
    H = x.shape[1]
    vpt = -(-(H // 8) // 256)
    n1 = 16 * vpt + 10
    eps32 = _f32(eps)
    mu = x64.mean(1, keepdim=True)
    sabs = x64.abs().sum(1, keepdim=True) / H
    dmu = 1.01 * (gamma(n1) * sabs + U * (mu.abs() + gamma(n1) * sabs))
    d = x64 - mu
    e = dmu + U * (d.abs() + dmu)
    ss = d.pow(2).sum(1, keepdim=True)
    E1 = (2 * d.abs() * e + e * e).sum(1, keepdim=True)
    var_eps = ss / H + eps32
    rho = (E1 + gamma(n1 + 1) * (ss + E1)) / (H * var_eps) + 2 * U
    r = 1.0 / torch.sqrt(var_eps)
    d_r = 1.01 * (0.5 * rho + 4 * U)
    y = d * r * w64 + b64
    err = 1.01 * (w64.abs() * r * (e + d.abs() * (d_r + 2 * U)) + U * y.abs())
    return y, err


def ln_inputs(M, H, dev, seed):
    """Rows of three kinds, by r mod 3: 64 + N(0, 1) (a large common offset), constant, and N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, H, generator=g)
    kind = torch.arange(M) % 3
    x[kind == 0] += 64
    x[kind == 1] = torch.randn(int((kind == 1).sum()), 1, generator=g) * 4
    w = torch.randn(H, generator=g).bfloat16()
    b = torch.randn(H, generator=g).bfloat16()
    return x.bfloat16().to(dev), w.to(dev), b.to(dev), kind.to(dev)


@pytest.mark.parametrize("H", [8, 1152, 2056, 8192])
@pytest.mark.parametrize("Mk", ["1", "cap-1", "cap+1", "3*729"])
def test_layernorm_within_fp64_bound(cuda_device, H, Mk):
    from metamorph_b200 import ops
    cap = _sms(cuda_device) * 8
    M = {"1": 1, "cap-1": cap - 1, "cap+1": cap + 1, "3*729": 3 * 729}[Mk]
    assert (-(-M // min(M, cap)) > 1) == (Mk in ("cap+1", "3*729"))     # grid-stride rows only past the cap
    x, w, b, kind = ln_inputs(M, H, cuda_device, seed=H * 7 + M)
    y = ops.layernorm(x, w, b, 1e-6)
    ref, err = layernorm_ref(x, w, b, 1e-6)
    n = assert_rounds_within(y, ref, err, f"layernorm H={H} M={M}")
    const = kind == 1
    if bool(const.any()):
        assert_equal(y[const], b.expand(int(const.sum()), H), "layernorm of a constant row must be b exactly")
    print(f"layernorm H={H} M={M}: {n} of {y.numel()} elements needed the fp32 slack")


# ------------------------------------------------------------------------------------------------ l2norm_rows
# vision_reduce.cu:85-117, 131-138: one warp per row, 8 warps per block, grid = min(ceil(R / 8), #SMs * 8); warp w of
# block b takes rows b * 8 + w, + grid * 8, ... Lane l adds the squares of vectors l, l + 32, ... (8 * ceil(C / 256)
# additions), then warp_sum (5). F.normalize's bf16 semantics: norm = bf16(sqrt), clamp at eps, bf16 divide.
def bf16_norm_interval(x, eps, n_chain):
    """Bounds on bf16(x / max(bf16(sqrtf(sum x^2)), eps)) per element, rows of x along the last dim.

    sum x^2 of exact products within gamma_n relative; sqrtf is correctly rounded: |sqrt_hat - sqrt64| <=
    sqrt64 (0.5 gamma_n + u) * 1.01, so the bf16 norm is between round(nrm64 -+ that). The quotient is rounded to fp32
    and then to bf16 (u relative before the last rounding), for whichever norm the kernel got: y lies between the
    roundings of the extreme quotients widened by u."""
    x64 = x.double()
    eps32 = _f32(eps)
    nrm = x64.pow(2).sum(-1, keepdim=True).sqrt()
    e = nrm * (0.5 * gamma(n_chain) + U) * 1.01
    n_lo, n_hi = _rnd(nrm - e).clamp(min=eps32), _rnd(nrm + e).clamp(min=eps32)
    q1, q2 = x64 / n_lo, x64 / n_hi
    qa, qb = torch.minimum(q1, q2), torch.maximum(q1, q2)
    return _rnd(qa - U * qa.abs()), _rnd(qb + U * qb.abs())


@pytest.mark.parametrize("C", [8, 256, 1152, 4096])
@pytest.mark.parametrize("Rk", ["1", "7", "8", "9", "sms*64+3"])
def test_l2norm_rows_rounds_like_f_normalize(cuda_device, C, Rk):
    from metamorph_b200 import ops
    sms = _sms(cuda_device)
    R = sms * 64 + 3 if Rk == "sms*64+3" else int(Rk)
    grid = min(-(-R // 8), sms * 8)
    assert (R > grid * 8) == (Rk == "sms*64+3")                 # some warp takes a second row
    g = torch.Generator().manual_seed(C + R)
    x = (torch.randn(R, C, generator=g) * torch.pow(2.0, (torch.arange(R) % 9 - 4).float())[:, None])
    x[R // 2] = 0
    x = x.bfloat16().to(cuda_device)
    y = ops.l2norm_rows(x)
    lo, hi = bf16_norm_interval(x, 1e-12, 8 * -(-C // 256) + 5)
    assert_between(y, lo, hi, f"l2norm_rows C={C} R={R}")
    assert bool((y[R // 2] == 0).all()), "an all-zero row must give exact zeros"


# ------------------------------------------------------------------------------------------------ RoPE
# norm_rope.cu:262-297, 362-376: one thread per (row, rotated head, 8-wide vector of the first half), 256 threads per
# block, grid = min(ceil(total / 256), #SMs * 16): every thread strides by grid * 256. It reads a = x[j], b = x[j + d/2]
# and writes a c - b s and b c + a s (backward: s -> -s).
LLAMA_SCALING = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                 "original_max_position_embeddings": 8192}


def rope_ref(x, c, s, d):
    """fp64 rotate-half of the [M, n, d] heads x with per-row tables c, s [M, 1, d/2]; the kernel's fp32 evaluation, in
    any contraction order, is within u (|a c| + |b s| + |y|) of it (two rounded products at most, one rounded sum)."""
    x64 = x.double()
    a, b = x64[..., :d // 2], x64[..., d // 2:]
    c, s = c.double(), s.double()
    lo, hi = a * c - b * s, b * c + a * s
    elo = 1.01 * U * ((a * c).abs() + (b * s).abs() + lo.abs())
    ehi = 1.01 * U * ((b * c).abs() + (a * s).abs() + hi.abs())
    return torch.cat([lo, hi], -1), torch.cat([elo, ehi], -1)


def _tables(d, n_pos, dev, round_bf16=True):
    from metamorph_b200.engine.llama import LlamaDims, rope_tables
    dims = LlamaDims(hidden=4096, n_layers=1, n_heads=32, n_kv_heads=8, head_dim=d, intermediate=14336, vocab=128258,
                     rope_scaling=LLAMA_SCALING, max_pos=n_pos)
    return rope_tables(dims, n_pos, dev, round_bf16=round_bf16)


@pytest.mark.parametrize("d", [64, 128])
def test_rope_forward_and_backward_round_like_fp64(cuda_device, d):
    from metamorph_b200 import ops
    M, ld, n_rot, n_pos = 16384, 6144, 40, 8192
    total = M * n_rot * (d // 16)
    cap_threads = _sms(cuda_device) * 16 * 256
    assert total > 4 * cap_threads                              # several grid-stride trips per thread
    cos, sin = _tables(d, n_pos, cuda_device)
    g = torch.Generator().manual_seed(d)
    pos = torch.randint(0, n_pos, (M,), generator=g, dtype=torch.int32)
    pos[:3] = 0
    pos[3:6] = n_pos - 1
    pos[100:200] = 4242                                        # repeated positions
    pos = pos.to(cuda_device)
    qkv = torch.randn(M, ld, generator=g).bfloat16().to(cuda_device)
    c, s = cos[pos.long()][:, None], sin[pos.long()][:, None]
    for backward in (False, True):
        t = qkv.clone()
        ops.rope_(t, pos, cos, sin, n_rot, d, backward=backward)
        x = qkv[:, :n_rot * d].view(M, n_rot, d)
        ref, err = rope_ref(x, c, -s if backward else s, d)
        n = assert_rounds_within(t[:, :n_rot * d].view(M, n_rot, d), ref, err, f"rope d={d} backward={backward}")
        assert_equal(t[:, n_rot * d:], qkv[:, n_rot * d:], "columns past the rotated heads must be untouched")
        print(f"rope d={d} backward={backward}: {n} elements needed the fp32 slack")


# decode.cu:242-257: the CTA that owns position p rotates the new K head (rope_lo / rope_hi of common.cuh) and appends K
# and V at p; decode.cu:395-410 copies rows [0, T) of a prefilled (rope_'d) qkv into the cache. A context that was
# prefilled and one that was decoded must hold the same bits. With the engine's tables (bf16 values) every product is
# exact and any evaluation order agrees; with full fp32 tables only the same order does, and a differing order shows in
# about one element in 10^5, hence ~10^6 rotated K elements per case.
@pytest.mark.parametrize("round_tables", [True, False], ids=["engine_tables", "fp32_tables"])
def test_decode_rope_append_equals_rope_then_prefill(cuda_device, round_tables):
    from metamorph_b200 import ops
    B, Hq, Hkv, d, Tmax, reps = 32, 32, 8, 128, 8192, 32
    W = (Hq + 2 * Hkv) * d
    cos, sin = _tables(d, Tmax, cuda_device, round_bf16=round_tables)
    g = torch.Generator().manual_seed(int(round_tables))
    kc = torch.full((B, Hkv, Tmax, d), 5.0, device=cuda_device, dtype=torch.bfloat16)
    vc = kc.clone()
    for rep in range(reps):
        rows = torch.randn(B, W, generator=g).bfloat16().to(cuda_device)
        pos = torch.randint(0, Tmax, (B,), generator=g, dtype=torch.int32)
        pos[0], pos[1], pos[3] = 0, Tmax - 1, pos[2]            # the table's first and last rows, a repeated position
        pos = pos.to(cuda_device)
        ops.decode_attn(rows, kc, vc, pos, cos, sin, Hq, Hkv, d, d ** -0.5)
        pre = rows.clone()
        ops.rope_(pre, pos, cos, sin, Hq + Hkv, d)
        b = torch.arange(B, device=cuda_device)
        want = pre.view(B, Hq + 2 * Hkv, d)
        assert_equal(kc[b, :, pos.long()], want[:, Hq:Hq + Hkv], f"decoded K vs rope_ (rep {rep})")
        assert_equal(vc[b, :, pos.long()], want[:, Hq + Hkv:], f"decoded V vs the qkv row (rep {rep})")
        if rep == 0:                                            # and the prefill copy of those rows, at T = 1
            kp = torch.full((B, Hkv, 4, d), 5.0, device=cuda_device, dtype=torch.bfloat16)
            vp = kp.clone()
            ops.kv_prefill(pre, kp, vp, B, 1, Hq, Hkv, d)
            assert_equal(kp[:, :, 0], kc[b, :, pos.long()], "rope_ + kv_prefill vs decoded K")
            assert_equal(vp[:, :, 0], vc[b, :, pos.long()], "kv_prefill vs decoded V")


@pytest.mark.parametrize("B,T,Tmax,Hkv", [(1, 1, 4, 1), (3, 37, 40, 8), (1, 129, 1000, 1), (3, 1500, 1501, 8)])
def test_kv_prefill_copies_bit_exact_and_keeps_sentinels(cuda_device, B, T, Tmax, Hkv):
    from metamorph_b200 import ops
    Hq, d = 4 * Hkv, 128
    total = B * T * Hkv * (d // 8)
    trips = -(-total // (min(-(-total // 256), _sms(cuda_device) * 16) * 256))
    assert (trips > 1) == (T == 1500)
    g = torch.Generator().manual_seed(T)
    qkv = torch.randn(B * T, (Hq + 2 * Hkv) * d, generator=g).bfloat16().to(cuda_device)
    kc = torch.full((B, Hkv, Tmax, d), -3.0, device=cuda_device, dtype=torch.bfloat16)
    vc = torch.full_like(kc, -7.0)
    ops.kv_prefill(qkv, kc, vc, B, T, Hq, Hkv, d)
    q = qkv.view(B, T, Hq + 2 * Hkv, d)
    assert_equal(kc[:, :, :T], q[:, :, Hq:Hq + Hkv].transpose(1, 2), "K cache rows < T")
    assert_equal(vc[:, :, :T], q[:, :, Hq + Hkv:].transpose(1, 2), "V cache rows < T")
    assert bool((kc[:, :, T:] == -3.0).all()) and bool((vc[:, :, T:] == -7.0).all()), "rows >= T overwritten"


# ------------------------------------------------------------------------------------------------ GELU
# elementwise.cu:51-83, 189-195: one thread per 8-element vector, 256 threads per block, grid = min(ceil(n / 8 / 256),
# #SMs * 16), grid-stride. gelu = 0.5 x (1 + erff(x * c)), gelu' = 0.5 (1 + erff(x c)) + x * k * __expf(-0.5 x^2).
def all_bf16(dev):
    """Every bf16 bit pattern that is not NaN (±0, subnormals, normals, ±inf), one NaN, zero-padded to a multiple of 8."""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    v = torch.cat([v[~torch.isnan(v)], torch.tensor([float("nan")], dtype=torch.bfloat16)])
    v = torch.cat([v, torch.zeros((-v.numel()) % 8, dtype=torch.bfloat16)])
    return v.to(dev)


def expf_fast_rel(arg):
    """__expf: 2 + floor(1.173 |x|) ulp (CUDA C Programming Guide, intrinsic functions), 1 ulp <= 2u relative."""
    return (2 + torch.floor(1.173 * arg.abs())) * 2 * U


def gelu_ref(x):
    """fp64 erf GELU and the kernel's error. t = fl(x * c32): 2u relative (c32 is 1/sqrt 2 rounded); erf moves by
    erf'(t) |t| 2u; erff is within 2 ulp (<= 4u |erf|); 1 + erf rounds (u |1 + erf|); 0.5 x (...) rounds once more.
    err = 1.01 (0.5 |x| ((2/sqrt(pi)) e^-t^2 |t| 2u + 4u |erf t| + u (1 + erf t)) + u |y|) + 2^-148."""
    x64 = x.double()
    t = x64 / math.sqrt(2)
    one_p = torch.special.erfc(-t)
    y = 0.5 * x64 * one_p
    derf = 2 / math.sqrt(math.pi) * torch.exp(-t * t) * t.abs() * 2 * U
    e_cdf = derf + 4 * U * torch.erf(t).abs() + U * one_p
    err = 1.01 * (0.5 * x64.abs() * e_cdf + U * y.abs()) + F32_TINY
    return y, torch.nan_to_num(err, nan=0.0), one_p, e_cdf


def gelu_bwd_ref(x, da):
    """fp64 da * gelu'(x) and the kernel's error: cdf = 0.5 (1 + erf) within 0.5 e_cdf (as in gelu_ref); the pdf term
    x * k32 * __expf(fl(-0.5 x x)): the argument is u-relative (exp moves by u |arg|), __expf as `expf_fast_rel`, k32
    and the two products u each; the sum and the final da * product one rounding each.
    err = 1.01 (|da| (0.5 e_cdf + |x| pdf (u |arg| + e_exp + 3u) + u |g|) + u |y|) + 2^-148."""
    x64, d64 = x.double(), da.double()
    _, _, one_p, e_cdf = gelu_ref(x)
    arg = -0.5 * x64 * x64
    pdf = torch.exp(arg) / math.sqrt(2 * math.pi)
    gr = 0.5 * one_p + x64 * pdf
    y = d64 * gr
    e_g = 0.5 * e_cdf + (x64 * pdf).abs() * (U * arg.abs() + expf_fast_rel(arg) + 3 * U) + U * gr.abs()
    err = 1.01 * (d64.abs() * e_g + U * y.abs()) + F32_TINY
    return y, torch.nan_to_num(err, nan=0.0)


@pytest.mark.parametrize("reps", [1, "past_cap"])
def test_gelu_fwd_bwd_every_bf16_value(cuda_device, reps):
    from metamorph_b200 import ops
    v = all_bf16(cuda_device)
    cap_vec = _sms(cuda_device) * 16 * 256
    if reps == "past_cap":
        v = v.repeat(-(-(2 * cap_vec * 8 + 64) // v.numel()))
        assert v.numel() // 8 > 2 * cap_vec                      # every thread makes at least two trips
    g = torch.Generator().manual_seed(5)
    da = torch.randn(v.numel(), generator=g).bfloat16().to(cuda_device)
    y = ops.gelu(v)
    ref, err, _, _ = gelu_ref(v)
    n = assert_rounds_within(y, ref, err, "gelu")
    ref, err = gelu_bwd_ref(v, da)
    m = assert_rounds_within(ops.gelu_bwd(v, da), ref, err, "gelu_bwd")
    print(f"gelu n={v.numel()}: {n} (fwd), {m} (bwd) elements needed the fp32 slack")


# ------------------------------------------------------------------------------------------------ swiglu_bwd
# elementwise.cu:13-49, 199-207: gu rows are [16 gate | 16 up] chunks; one thread per (row, chunk, 8-column half),
# total M * I / 16 * 2 threads, grid-stride. s = 1 / (1 + __expf(-g)), a = g s: act = bf16(a u),
# dgate = bf16(d u (s + a (1 - s))), dup = bf16(d a).
def swiglu_ref(g, u, d):
    """fp64 SwiGLU backward and the kernel's errors. sigma: __expf(-g) within e_e = expf_fast_rel(g); 1 + e moves by
    e_e (1 - sigma) relative, plus the add and the divide (2u); where e overflows the kernel has s = 0 and sigma <
    2^-126: err_s = 1.01 sigma (e_e (1 - sigma) + 2u) + 2^-126. a = g s: err_a = |g| err_s + u |a|.
    t = s + a (1 - s): err_t = err_s + |1 - sigma| err_a + |a| (err_s + u |1 - sigma|) + u |a (1 - sigma)| + u |t|.
    act = fl(a u): |u| err_a + u |act|; dgate = fl(fl(d u) t), d u exact: |d u| err_t + u |dg|; dup: |d| err_a + u |du|.
    Each times 1.01, plus 2^-148."""
    g64, u64, d64 = g.double(), u.double(), d.double()
    sg = torch.sigmoid(g64)
    e_e = expf_fast_rel(g64)
    err_s = 1.01 * sg * (e_e * (1 - sg) + 2 * U) + 2.0 ** -126
    a = g64 * sg
    err_a = g64.abs() * err_s + U * a.abs()
    t = sg + a * (1 - sg)
    err_t = err_s + (1 - sg).abs() * err_a + a.abs() * (err_s + U * (1 - sg).abs()) + U * (a * (1 - sg)).abs() + U * t.abs()
    act, dg, du = a * u64, d64 * u64 * t, d64 * a
    fix = lambda e: torch.nan_to_num(1.01 * e + F32_TINY, nan=0.0, posinf=0.0)  # noqa: E731
    return ((act, fix(u64.abs() * err_a + U * act.abs())), (dg, fix((d64 * u64).abs() * err_t + U * dg.abs())),
            (du, fix(d64.abs() * err_a + U * du.abs())))


def _interleave(gate, up):
    M, I = gate.shape
    return torch.stack([gate.view(M, I // 16, 16), up.view(M, I // 16, 16)], 2).reshape(M, 2 * I)


@pytest.mark.parametrize("I", [16, 32, 528])
def test_swiglu_bwd_every_bf16_gate(cuda_device, I):
    from metamorph_b200 import ops
    gv = all_bf16(cuda_device)
    pairs = [(1.0, 1.0), (-0.375, 3.0), (2.5, -0.0078125)]
    n = gv.numel() * len(pairs)
    M = -(-n // I)
    gate = torch.zeros(M * I, device=cuda_device, dtype=torch.bfloat16)
    up, d = gate.clone(), gate.clone()
    for k, (uu, dd) in enumerate(pairs):
        sl = slice(k * gv.numel(), (k + 1) * gv.numel())
        gate[sl], up[sl], d[sl] = gv, uu, dd
    gate, up, d = gate.view(M, I), up.view(M, I), d.view(M, I)
    gu = _interleave(gate, up).contiguous()
    act = torch.empty(M, I, device=cuda_device, dtype=torch.bfloat16)
    dgu = ops.swiglu_bwd(gu, d, act=act)
    (ra, ea), (rg, eg), (ru, eu) = swiglu_ref(gate, up, d)
    dgu = dgu.view(M, I // 16, 2, 16)
    na = assert_rounds_within(act, ra, ea, f"swiglu act I={I}")
    ng = assert_rounds_within(dgu[:, :, 0].reshape(M, I), rg, eg, f"swiglu dgate I={I}")
    nu = assert_rounds_within(dgu[:, :, 1].reshape(M, I), ru, eu, f"swiglu dup I={I}")
    nan = torch.isnan(gate)
    assert bool(torch.isnan(act[nan]).all()) and bool(torch.isnan(dgu[:, :, 0].reshape(M, I)[nan]).all())
    print(f"swiglu I={I}: {na}, {ng}, {nu} elements needed the fp32 slack")


@pytest.mark.parametrize("I", [16, 32, 528])
def test_swiglu_bwd_one_hot_dact_lands_in_its_chunk(cuda_device, I):
    from metamorph_b200 import ops
    cols = sorted({0, 7, 8, 15, min(16, I - 1), I // 2, I - 9, I - 8, I - 1})
    M = len(cols)
    g = torch.Generator().manual_seed(I)
    gate = (torch.randn(M, I, generator=g) + 0.5).bfloat16().to(cuda_device)
    up = (torch.randn(M, I, generator=g) + 0.5).bfloat16().to(cuda_device)
    d = torch.zeros(M, I, device=cuda_device, dtype=torch.bfloat16)
    for r, j in enumerate(cols):
        d[r, j] = 1.0
    dgu = ops.swiglu_bwd(_interleave(gate, up).contiguous(), d)
    want = torch.zeros(M, 2 * I, dtype=torch.bool, device=cuda_device)
    for r, j in enumerate(cols):
        want[r, (j // 16) * 32 + j % 16] = want[r, (j // 16) * 32 + 16 + j % 16] = True
    assert bool((dgu[~want] == 0).all()), "a one-hot dact wrote outside its [16 gate | 16 up] pair"
    assert bool((dgu[want] != 0).all()), "a one-hot dact gave no gradient at its column"


# ------------------------------------------------------------------------------------------------ im2col, pos emb
# elementwise.cu:111-153: one thread per output element (im2col) or 8-wide vector (add_pos_emb), grid-stride.
@pytest.mark.parametrize("S", [14, 27, 384, 392])
@pytest.mark.parametrize("ldp", [592, 640])
def test_im2col_patch14_equals_unfold(cuda_device, S, ldp):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(S + ldp)
    img = torch.randn(2, 3, S, S, generator=g).bfloat16().to(cuda_device)
    out = ops.im2col_patch14(img, ldp)
    G = S // 14
    ref = F.unfold(img.float(), 14, stride=14).bfloat16().transpose(1, 2).reshape(2 * G * G, 588)
    assert_equal(out[:, :588], ref, f"im2col S={S}")
    assert bool((out[:, 588:] == 0).all()), "pad columns must be exactly 0"


@pytest.mark.parametrize("R", [729, 729 + 5, 3 * 729])
def test_add_pos_emb_single_rounding(cuda_device, R):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(R)
    x = (torch.randn(R, 1152, generator=g) * 4).bfloat16().to(cuda_device)
    pos = torch.randn(729, 1152, generator=g).bfloat16().to(cuda_device)
    want = (x.float() + pos.float()[torch.arange(R, device=cuda_device) % 729]).bfloat16()
    assert_equal(ops.add_pos_emb_(x.clone(), pos), want, f"add_pos_emb R={R}")


# ------------------------------------------------------------------------------------------------ bilinear + l2norm
# vision_reduce.cu:24-82, 121-129: one block per output token, thread i holds channels [8 i, 8 i + 8) (C <= 2048);
# taps follow ATen's area_pixel_compute_source_index; the norm is a block_sum of 8 squares per thread (chain 8 + 10).
@pytest.mark.parametrize("S", [8, 24, 27])
@pytest.mark.parametrize("C", [8, 1152, 2048])
@pytest.mark.parametrize("n_img", [1, 3])
def test_bilinear_l2norm_every_side(cuda_device, S, C, n_img):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(S * C + n_img)
    x = torch.randn(n_img, S * S, C, generator=g).bfloat16().to(cuda_device)
    xi = x.view(n_img, S, S, C).permute(0, 3, 1, 2).contiguous().float()   # NCHW, as siglip_encoder.py:159-160
    for T in (1, 2, 8, 12, 16, 24, 26, 32):
        raw = ops.bilinear_l2norm(x, T, normalize=False)
        ref = F.interpolate(xi, size=(T, T), mode="bilinear", align_corners=False).to(torch.bfloat16)
        assert_equal(raw, ref.permute(0, 2, 3, 1).reshape(n_img, T * T, C), f"bilinear S={S} T={T} C={C}")
        y = ops.bilinear_l2norm(x, T)
        lo, hi = bf16_norm_interval(raw, 1e-12, 8 + 10)
        assert_between(y, lo, hi, f"bilinear_l2norm S={S} T={T} C={C}")
    z = ops.bilinear_l2norm(torch.zeros_like(x), 8)
    assert bool((z == 0).all()), "an all-zero feature map must normalise to zeros"
