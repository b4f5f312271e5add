"""The gradient reductions of the train step against fp64 restatements, at their edges, and bit-for-bit repeats.

The train step promises the same bits on every run with the same inputs. The reductions that make that promise (bias
column sums, the RMSNorm weight gradient, the embedding-table gradient, the squared gradient norm) are checked here two
ways:
  * parity with an fp64 torch restatement. Integer-valued bf16 inputs sum exactly in fp32 while every partial sum stays
    below 2^24, so for them the kernel must equal the fp64 result exactly (after one rounding to the output dtype): a
    dropped, doubled or misplaced row fails. Random inputs are held to a bound derived from the summation length,
    written next to each assert (gamma_n = n u / (1 - n u), u = 2^-24 the fp32 unit roundoff);
  * three runs of the same call on fresh, equal outputs with random non-integer data must be torch.equal (integer data
    sums exactly in any order and would hide an order dependence).
"""
import math

import pytest
import torch

from tests.exact import U, gamma as _gamma, ints as _ints, ulp_bf16 as _ulp_bf16

pytestmark = pytest.mark.gpu


def _sms(device):
    return torch.cuda.get_device_properties(device).multi_processor_count


# ------------------------------------------------------------------------------------------------ colsum (bias gradients)
@pytest.mark.parametrize("N", [2, 62, 64, 66, 1154, 4096])
@pytest.mark.parametrize("R", [1, 7, 8, 9, 4097, 32768])
def test_colsum_exact_bounded_and_repeatable(cuda_device, R, N):
    from metamorph_b200 import ops
    gen = torch.Generator(device=cuda_device).manual_seed(R * 7919 + N)
    pad = 4                                          # x is a column slice of a wider buffer: ld = N + 10, even offset

    def run(x, out0):
        buf = torch.full((N + 2 * pad,), 1234.5, device=cuda_device)
        buf[pad:pad + N] = out0
        ops.colsum_accum(x, buf[pad:pad + N])
        assert (buf[:pad] == 1234.5).all() and (buf[pad + N:] == 1234.5).all(), "colsum wrote outside out"
        return buf[pad:pad + N].clone()

    # exact: |partial sums| <= 4 * 32768 + 100 < 2^24, so every fp32 addition is exact
    wide = _ints((R, N + 10), -4, 4, cuda_device, gen=gen)
    x = wide[:, 4:4 + N]
    out0 = _ints((N,), -100, 100, cuda_device, torch.float32, gen=gen)
    got = run(x, out0)
    want = (out0.double() + x.double().sum(0)).float()
    assert torch.equal(got, want), f"colsum R={R} N={N}: integer sums differ"

    # random: each thread adds ceil(R/8) rows in order, then the 8 row phases are added in order and the result is added
    # to out: every term reaches the result through at most n = ceil(R/8) + 8 fp32 additions
    wide = torch.randn((R, N + 10), device=cuda_device, generator=gen).bfloat16()
    x = wide[:, 4:4 + N]
    out0 = torch.randn((N,), device=cuda_device, generator=gen)
    exact = out0.double() + x.double().sum(0)
    bound = _gamma(math.ceil(R / 8) + 8) * (out0.double().abs() + x.double().abs().sum(0))
    runs = [run(x, out0.clone()) for _ in range(3)]
    err = (runs[0].double() - exact).abs()
    assert (err <= bound).all(), f"colsum R={R} N={N}: max err {float(err.max()):.3e} over the gamma_n bound"
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2]), "colsum is not bit-reproducible"


# ------------------------------------------------------------------------------------------------ RMSNorm weight gradient
def _rms_shapes():
    # M relative to the backward's grid G = 4 * #SMs (blocks own rows r, r + G, ...): one row, fewer / exactly / more
    # rows than blocks, several rows per block, and a full-size batch; the H cover VPT = 1, 2 and 4 and the H <= 8192 limit
    return [("1", 0, 1), ("G-1", 1, -1), ("G", 1, 0), ("G+1", 1, 1), ("3G+7", 3, 7), ("8192", 0, 8192)]


@pytest.mark.parametrize("with_dres", [False, True])
@pytest.mark.parametrize("H", [8, 1152, 2048, 2056, 4096, 8192])
@pytest.mark.parametrize("m_case", _rms_shapes(), ids=lambda c: c[0])
def test_rmsnorm_bwd_dw_and_dx_match_fp64(cuda_device, m_case, H, with_dres):
    from metamorph_b200 import ops
    G = 4 * _sms(cuda_device)
    _, g_mult, add = m_case
    M = g_mult * G + add
    eps = 1e-5
    gen = torch.Generator(device=cuda_device).manual_seed(M * 31 + H)
    x = torch.randn(M, H, device=cuda_device, generator=gen).bfloat16()
    w = (1 + 0.1 * torch.randn(H, device=cuda_device, generator=gen)).bfloat16()
    dy = torch.randn(M, H, device=cuda_device, generator=gen).bfloat16()
    dres = torch.randn(M, H, device=cuda_device, generator=gen).bfloat16() if with_dres else None
    dw0 = torch.randn(H, device=cuda_device, generator=gen)

    xd, wd, dyd = x.double(), w.double(), dy.double()
    xr = xd.clone().requires_grad_(True)
    (wd * (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + eps))).backward(dyd)
    dx_ref = xr.grad + (dres.double() if with_dres else 0.0)
    rstd = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    terms = dyd * xd * rstd
    dw_ref = dw0.double() + terms.sum(0)

    runs = []
    for _ in range(3):
        dw = dw0.clone()
        dx = ops.rmsnorm_bwd(dy, x, w, eps, dres_in=dres, dw_accum=dw)
        runs.append((dx, dw))
    torch.cuda.synchronize()
    dx, dw = runs[0]

    # rstd: sum x^2 is a sum of exact fp32 squares, <= 8*VPT per thread, then a 5-level warp tree and 8 warp sums:
    # relative error <= gamma_{8 VPT + 13}; /H, +eps (2 roundings), rsqrtf (<= 2 ulp = 4u), the square root halving the first
    # part: e_rstd <= gamma_{8 VPT + 15} / 2 + 4u.
    vpt = {1: 1, 2: 2}.get(-(-H // 2048), 4)
    e_rstd = _gamma(8 * vpt + 15) / 2 + 4 * U
    # dw: a block adds its rows (at most ceil(M/G)) in order, the second launch adds the G' = min(M, G) partials in order
    # and adds to dw0: depth n = ceil(M/G) + G' + 1; each term dy*x*rstd is within (e_rstd + u) of its exact value.
    n = math.ceil(M / G) + min(M, G) + 1
    bound = (_gamma(n) + e_rstd + U) * (dw0.double().abs() + terms.abs().sum(0))
    err = (dw.double() - dw_ref).abs()
    assert (err <= bound).all(), f"rmsnorm dw M={M} H={H}: max err {float(err.max()):.3e}"

    # dx = dres + rstd*dy*w - x * rstd^3 * sum(dy*w*x)/H in fp32, rounded once to bf16. The signed sum sum(dy*w*x) has
    # absolute error <= gamma_{8 VPT + 15} * sum|dy*w*x| (2 product roundings + the summation depth above); rstd^3 carries
    # 3 e_rstd + 2u; the final combination adds 4u of |A| + |B| + |dres|. e32 bounds the fp32 value, and the bf16
    # rounding adds half an ulp: |dx - ref| <= e32 + ulp_bf16(max(|dx|, |ref|)) / 2 + ... <= e32 + ulp.
    A = (rstd * dyd * wd).abs()
    s_abs = (dyd * wd * xd).abs().sum(-1, keepdim=True)
    B = xd.abs() * rstd.pow(3) * s_abs / H
    C = dres.double().abs() if with_dres else 0.0
    e32 = (3 * e_rstd + _gamma(8 * vpt + 15) + 6 * U) * (A + B) + 4 * U * (A + B + C)
    dxd = dx.double()
    tol = e32 + _ulp_bf16(torch.maximum(dxd.abs(), dx_ref.abs()))
    err = (dxd - dx_ref).abs()
    assert (err <= tol).all(), f"rmsnorm dx M={M} H={H}: max err {float(err.max()):.3e}"

    for dx_i, dw_i in runs[1:]:
        assert torch.equal(dw_i, dw) and torch.equal(dx_i, dx), "rmsnorm_bwd is not bit-reproducible"


# ------------------------------------------------------------------------------------------------ embedding scatter
R_SCATTER, V_SCATTER, NI_SCATTER = 4096, 512, 300


def _row_map(case, device):
    """int32 row map of R rows: >= 0 token id, -1 padding, <= -2 image row."""
    R = R_SCATTER
    if case == "one_token_everywhere":
        return torch.full((R,), 5, dtype=torch.int32, device=device)
    g = torch.Generator().manual_seed(17)
    rm = torch.randint(2, 40, (R,), generator=g, dtype=torch.int32)   # tokens 2..39: each on ~100 rows in many windows
    rm[0] = rm[R - 1] = 0                                              # token 0: the first and the last row only
    rm[100:230] = 1                                                    # token 1: one run over five 32-row windows
    rest = torch.tensor([r for r in range(1, R - 1) if not 100 <= r < 230])
    pick = rest[torch.randperm(rest.numel(), generator=g)]
    rm[pick[:50]] = -1
    rm[pick[50:50 + NI_SCATTER]] = -(torch.arange(NI_SCATTER, dtype=torch.int32)) - 2
    return rm.to(device)                                               # tokens 40..511 are absent


def _scatter_ref(dout, rm, dembed0):
    """fp64 sums (exact for these data up to fp64 rounding) and sum|terms| per embedding row."""
    tok = rm >= 0
    idx = rm[tok].long()
    ref = dembed0.double().index_add(0, idx, dout[tok].double())
    abs_sum = dembed0.double().abs().index_add(0, idx, dout[tok].double().abs())
    count = torch.bincount(idx, minlength=dembed0.shape[0])
    return ref, abs_sum, count


@pytest.mark.parametrize("H", [8, 1032, 2056, 4096])
@pytest.mark.parametrize("case", ["mixed", "one_token_everywhere"])
def test_interleave_scatter_exact_bounded_and_repeatable(cuda_device, case, H):
    from metamorph_b200 import ops
    R, V, NI = R_SCATTER, V_SCATTER, NI_SCATTER
    rm = _row_map(case, cuda_device)
    gen = torch.Generator(device=cuda_device).manual_seed(H)
    present = torch.bincount(rm[rm >= 0].long(), minlength=V) > 0
    im = rm <= -2
    img_idx = (-(rm[im]) - 2).long()

    # exact: integer terms, |sums| <= 4 * 4096 + 8 < 2^24, so the fp32 row sums are exact and one rounding to bf16 is
    # all that separates kernel and reference
    dout = _ints((R, H), -4, 4, cuda_device, gen=gen)
    dembed0 = _ints((V, H), -8, 8, cuda_device, gen=gen)
    demb, dimg = dembed0.clone(), torch.zeros(NI, H, device=cuda_device, dtype=torch.bfloat16)
    ops.interleave_scatter(dout, rm, demb, dimg)
    ref, _, _ = _scatter_ref(dout, rm, dembed0)
    assert torch.equal(demb, ref.bfloat16()), "embedding gradient of integer data is not exact"
    assert torch.equal(demb[~present], dembed0[~present]), "rows of absent tokens changed"
    assert torch.equal(dimg[img_idx], dout[im]), "image rows must be copied exactly"

    # random data: the warp of a token's first row adds dembed0 and the token's k rows in row order in fp32 (k additions),
    # then rounds to bf16. |s32 - s64| <= gamma_k sum|terms|, and the two bf16 roundings add at most half an ulp each.
    dout = torch.randn(R, H, device=cuda_device, generator=gen).bfloat16()
    dembed0 = torch.randn(V, H, device=cuda_device, generator=gen).bfloat16()
    ref, abs_sum, count = _scatter_ref(dout, rm, dembed0)
    runs = []
    for _ in range(3):
        demb, dimg = dembed0.clone(), torch.zeros(NI, H, device=cuda_device, dtype=torch.bfloat16)
        ops.interleave_scatter(dout, rm, demb, dimg)
        runs.append((demb, dimg))
    demb, dimg = runs[0]
    gam = torch.tensor([_gamma(int(k)) for k in count.tolist()], device=cuda_device, dtype=torch.float64)[:, None]
    got = demb.double()
    tol = _ulp_bf16(torch.maximum(got.abs(), ref.abs())) + gam * abs_sum
    err = (got - ref).abs()
    assert (err <= tol).all(), f"embedding gradient: max err {float(err.max()):.3e}"
    assert torch.equal(demb[~present], dembed0[~present]), "rows of absent tokens changed"
    assert torch.equal(dimg[img_idx], dout[im])
    for d_e, d_i in runs[1:]:
        assert torch.equal(d_e, demb) and torch.equal(d_i, dimg), "interleave_scatter is not bit-reproducible"

    # dembed=None: only the image rows are written; dimg=None: only the embedding gradient
    dimg2 = torch.zeros(NI, H, device=cuda_device, dtype=torch.bfloat16)
    ops.interleave_scatter(dout, rm, None, dimg2)
    assert torch.equal(dimg2, dimg)
    demb2 = dembed0.clone()
    ops.interleave_scatter(dout, rm, demb2, None)
    assert torch.equal(demb2, demb)


# ------------------------------------------------------------------------------------------------ squared gradient norm
def _sumsq_chain(n, sms):
    """Longest chain of fp32 additions from one x^2 term to a block partial: each thread adds its 8-element vectors
    (8 * per-thread vector count), then block_sum's two 5-level warp trees; +2 for the fp64 finish and the one fp32 rounding."""
    n8 = n // 8
    grid = max(1, min(-(-n8 // 256), 16 * sms))
    return 8 * -(-n8 // (grid * 256)) + 10 + 2


@pytest.mark.parametrize("n", [8, 8 * 255, 2 ** 20 + 8, 2 ** 26])
def test_sumsq_exact_bounded_and_repeatable(cuda_device, n):
    from metamorph_b200 import ops
    gen = torch.Generator(device=cuda_device).manual_seed(n % 100003)

    # exact: squares of {-1, 0, 1} are 0 or 1; a block owns at most n / 16 elements (grid >= 16 for n = 2^26), so every
    # block partial is an integer below 2^24 and exact in fp32; the fp64 finish adds the partials exactly and rounds once
    x = _ints((n,), -1, 1, cuda_device, gen=gen)
    acc = torch.full((1,), 3.0, device=cuda_device)
    ops.sumsq_accum(x, acc)
    want = torch.tensor([3.0 + float((x != 0).sum())], dtype=torch.float64).float()
    assert torch.equal(acc.cpu(), want), (float(acc), float(want))

    # random: all terms are non-negative, so the error is <= gamma_chain * (exact sum)
    x = torch.randn(n, device=cuda_device, generator=gen).bfloat16()
    acc0 = torch.full((1,), 0.75, device=cuda_device)
    exact = 0.75 + float(x.double().pow(2).sum())
    runs = []
    for _ in range(3):
        acc = acc0.clone()
        ops.sumsq_accum(x, acc)
        runs.append(acc)
    got = float(runs[0])
    assert abs(got - exact) <= _gamma(_sumsq_chain(n, _sms(cuda_device))) * exact, (got, exact)
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2]), \
        f"sumsq_accum n={n} is not bit-reproducible: {[float(r) for r in runs]}"


# ------------------------------------------------------------------------------------------------ clip coefficient
def _clip_pair(grads, max_norm):
    """(coef, norm) from the library (sumsq_accum over the bf16 gradients, then clip_coef) and from
    torch.nn.utils.clip_grad_norm_ on fp32 copies (coef rebuilt with torch's formula; the clipped grads returned too)."""
    from metamorph_b200 import ops
    acc = torch.zeros(1, device=grads[0].device)
    for g in grads:
        ops.sumsq_accum(g.reshape(-1), acc)
    out = ops.clip_coef(acc, max_norm)
    params = [torch.zeros(g.shape, device=g.device, requires_grad=True) for g in grads]
    for p, g in zip(params, grads):
        p.grad = g.float()
    t_norm = torch.nn.utils.clip_grad_norm_(params, max_norm)
    t_coef = torch.clamp(max_norm / (t_norm + 1e-6), max=1.0)
    return float(out[0]), float(out[1]), float(t_coef), float(t_norm), [p.grad for p in params]


@pytest.mark.parametrize("where", ["below", "at", "above"])
def test_clip_coef_matches_torch(cuda_device, where):
    gen = torch.Generator(device=cuda_device).manual_seed(5)
    shapes = [(64, 130), (3000,), (8,), (256, 256)]
    grads = [torch.randn(s, device=cuda_device, generator=gen).bfloat16() for s in shapes]
    exact = math.sqrt(sum(float(g.double().pow(2).sum()) for g in grads))
    max_norm = {"below": 4.0 * exact, "at": exact, "above": 0.25 * exact}[where]
    c, norm, t_c, t_norm, _ = _clip_pair(grads, max_norm)
    sms = _sms(cuda_device)
    # library norm: the squared norm is within gamma_(chain + #calls) of exact (non-negative terms; each call adds its
    # result to the accumulator with one more rounding); sqrtf halves that and rounds once more
    e_lib = _gamma(max(_sumsq_chain(g.numel(), sms) for g in grads) + len(grads)) / 2 + U
    assert abs(norm - exact) <= e_lib * exact, (norm, exact)
    # torch's norm: whatever its summation order, n non-negative terms sum within gamma_n; a norm of the per-tensor
    # norms adds #tensors + 2 roundings, and the two square roots one each
    e_torch = _gamma(max(g.numel() for g in grads) + len(grads) + 4) / 2 + 2 * U
    assert abs(t_norm - exact) <= e_torch * exact, (t_norm, exact)
    # the coefficient max_norm / (norm + 1e-6) adds two roundings; the clamp at 1 does not increase a difference
    assert abs(c - t_c) <= (e_lib + e_torch + 4 * U) * max(c, t_c), (c, t_c)
    if where == "below":
        assert c == 1.0 and t_c == 1.0
    if where == "above":
        assert c < 0.3


@pytest.mark.parametrize("special", ["zero", "inf", "nan"])
def test_clip_coef_non_finite_and_zero_norms_match_torch(cuda_device, special):
    grads = [torch.zeros(64, 16, device=cuda_device, dtype=torch.bfloat16),
             torch.zeros(1024, device=cuda_device, dtype=torch.bfloat16)]
    if special != "zero":
        grads[0].normal_()
        grads[1].normal_()
        grads[1][77] = float(special)
    c, norm, t_c, t_norm, clipped = _clip_pair(grads, 1.0)
    if special == "zero":                      # 1 / (0 + 1e-6) clamps to 1: nothing to clip
        assert norm == 0.0 and t_norm == 0.0 and c == 1.0 and t_c == 1.0
    elif special == "inf":                     # max_norm / inf = 0, as in torch
        assert norm == math.inf and t_norm == math.inf and c == 0.0 and t_c == 0.0
    else:                                      # torch's clamp(max=1) keeps NaN: every gradient becomes NaN
        assert math.isnan(t_norm) and math.isnan(t_c) and all(torch.isnan(g).all() for g in clipped)
        assert math.isnan(norm), norm
        assert math.isnan(c), f"a NaN gradient norm must give a NaN clip coefficient, got {c}"


# ------------------------------------------------------------------------------------------------ AdamW with a device scale
@pytest.mark.parametrize("grad_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
def test_adamw_grad_scale_tensor_matches_fp64_adamw(cuda_device, grad_scale, grad_dtype):
    """The clip coefficient reaches the update through grad_scale_tensor: g * grad_scale * tensor must be what
    torch.optim.AdamW (fp64, same fp32 hyper-parameters) sees, over 3 steps with weight decay."""
    import numpy as np
    from metamorph_b200 import ops
    f32 = lambda v: float(np.float32(v))     # the kernel receives fp32 hyper-parameters; hand torch the same values
    lr, b1, b2, eps, wd = f32(1e-3), f32(0.9), f32(0.999), f32(1e-8), f32(0.1)
    gen = torch.Generator(device=cuda_device).manual_seed(9)
    n = 4 * 3075                                             # not a multiple of the 1024 elements a block step covers
    tensor_scale = torch.tensor([0.375], device=cuda_device)
    scale = grad_scale * 0.375                               # 3/16 or 3/8: exact in fp32, and g * scale is exact for bf16 g
    p = torch.randn(n, device=cuda_device, generator=gen)
    ref = p.double().clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    p32, m, v, p16 = p.clone(), torch.zeros_like(p), torch.zeros_like(p), p.bfloat16()
    m_env = torch.zeros(n, device=cuda_device, dtype=torch.float64)      # b1-weighted sum of |g|: m's terms, unsigned
    bound = torch.zeros(n, device=cuda_device, dtype=torch.float64)
    for t in range(1, 4):
        g = torch.randn(n, device=cuda_device, generator=gen).to(grad_dtype)
        gs = g.double() * scale
        p_prev = ref.detach().clone()
        ref.grad = gs
        opt.step()
        ops.adamw_step_(p16, p32, m, v, g, lr=lr, beta1=b1, beta2=b2, eps=eps, wd=wd, step=t, grad_scale=grad_scale,
                        grad_scale_tensor=tensor_scale)
        st = opt.state[ref]
        m_env = b1 * m_env + (1 - b1) * gs.abs()
        c1, c2 = 1 - b1 ** t, 1 - b2 ** t
        den = st["exp_avg_sq"].sqrt() / math.sqrt(c2) + eps
        # Error budget of the fp32 kernel against this fp64 run, per element and step:
        #  * decay p *= 1 - lr*wd and the final subtraction: <= 4u |p|;
        #  * m: <= 4 roundings per step (g*scale, two products, one add), relative to m's unsigned envelope: 4t u m_env;
        #  * v: non-negative terms, <= 6 roundings per step (g*scale counts twice in g^2): 6t u relative; sqrt halves it;
        #  * c1 = 1 - powf(b1, t), c2 likewise: powf is within 4 ulp (8u), and 1 - b^t (exact, b^t >= 1/2) amplifies that
        #    by b^t / (1 - b^t); sqrt(c2) halves c2's error; + lr / c1, / sqrt_c2, + eps, the divide, the product:
        e_c1 = 8 * U * b1 ** t / c1 + U
        e_c2 = 8 * U * b2 ** t / c2 + U
        e_rel = e_c1 + (6 * t * U + e_c2) / 2 + 6 * U
        upd_err = lr / c1 * (4 * t * U * m_env + st["exp_avg"].abs() * e_rel) / den
        bound += 4 * U * p_prev.abs() + upd_err
    err = (p32.double() - ref.detach()).abs()
    assert (err <= bound).all(), f"adamw: max err {float(err.max()):.3e}, worst err/bound {float((err / bound).max()):.2f}"
    assert torch.equal(p16, p32.bfloat16())


# ------------------------------------------------------------------------------------------------ per-stream scratch
def test_scratch_is_private_to_each_stream(cuda_device):
    """ce_fwd_bwd (loss sum), rmsnorm_bwd (weight gradient) and sumsq_accum keep their partial sums in library scratch
    private to (device, stream). Enqueued back to back on two side streams with no synchronisation between them, each
    stream's results must equal a serial run on one stream bit for bit."""
    from metamorph_b200 import ops
    gen = torch.Generator(device=cuda_device).manual_seed(21)
    R, V, M, H = 256, 32000, 2048, 4096

    def inputs():
        return dict(logits=torch.randn(R, V, device=cuda_device, generator=gen) * 3,
                    labels=torch.randint(0, V, (R,), device=cuda_device, generator=gen, dtype=torch.int32),
                    x=torch.randn(M, H, device=cuda_device, generator=gen).bfloat16(),
                    dy=torch.randn(M, H, device=cuda_device, generator=gen).bfloat16(),
                    w=(1 + 0.1 * torch.randn(H, device=cuda_device, generator=gen)).bfloat16())

    def work(d):
        loss = torch.zeros(1, device=cuda_device)
        dl = torch.empty(R, V, device=cuda_device, dtype=torch.bfloat16)
        dw = torch.zeros(H, device=cuda_device)
        sq = torch.zeros(1, device=cuda_device)
        for _ in range(2):                       # several launches per stream, so the two streams overlap
            ops.ce_fwd_bwd(d["logits"], d["labels"], V, loss, dlogits=dl, grad_scale=1.0 / R)
            ops.rmsnorm_bwd(d["dy"], d["x"], d["w"], 1e-5, dw_accum=dw)
            ops.sumsq_accum(d["dy"].reshape(-1), sq)
        return loss, dl, dw, sq

    ins = [inputs(), inputs()]
    torch.cuda.synchronize()
    serial = [work(d) for d in ins]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    main = torch.cuda.current_stream()
    outs = [None, None]
    for i, s in enumerate(streams):
        s.wait_stream(main)
    for i, s in enumerate(streams):
        with torch.cuda.stream(s):
            outs[i] = work(ins[i])
    for s in streams:
        main.wait_stream(s)
    torch.cuda.synchronize()
    for i in range(2):
        for name, a, b in zip(("loss", "dlogits", "dw", "sumsq"), outs[i], serial[i]):
            assert torch.equal(a, b), f"stream {i}: {name} differs from the single-stream run"
