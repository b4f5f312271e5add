"""Cross-entropy, the cosine loss and the vocabulary argmax against fp64 restatements, at their vector tails, split
edges and grid-stride rows (H100 only). Schedules are restated next to each test with their source lines, and each
case asserts the regime it reaches; the loss sums are rebuilt exactly from the fixed-point rule of loss.cu:16-55."""
import math

import numpy as np
import pytest
import torch

from tests.exact import U, assert_between, assert_equal, assert_rounds_within, assert_within, gamma, round_bf16_from_fp64

pytestmark = pytest.mark.gpu

CE_THREADS = 512


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _rnd(x):
    return round_bf16_from_fp64(x).double()


def _expf_rel(arg):
    """__expf: 2 + floor(1.173 |x|) ulp (CUDA C Programming Guide, intrinsic functions); 1 ulp <= 2u relative."""
    return (2 + torch.floor(1.173 * arg.abs())) * 2 * U


# ------------------------------------------------------------------------------------------------ cross-entropy
# loss.cu:57-124, 256-269: one 512-thread block per row. Pass 1 (online max / sum): thread t takes float4 vectors at
# 4t, 4t + 2048, ... below V4 = V & ~3 (loss.cu:78-86), then the scalar tail V4 + t < V (loss.cu:87-94); block_max,
# rescale, block_sum; lse = gm + logf(gs). Pass 2 (gradient): 8-wide vectors below V8 = V & ~7 (loss.cu:110-118), then
# the scalar tail [V8, ld_d), zero past V (loss.cu:119-123). A row whose label is ignore_index and that wants no lse
# only zeroes its gradient row (loss.cu:67-74).
def ce_lse_bound(x, V):
    """fp64 logsumexp of the [R, V] rows and a bound on the kernel's lse error.

    A thread's running sum rescales at most n_it + 1 times (n_it = its vector and tail iterations) and the arguments of
    all its rescales add up to at most W = max - min of the row, so every exp term reaches gs with a relative error of at
    most 2u (2 (n_it + 2) + 1.7 (W + |x_j - max|)) (__expf as `_expf_rel`, plus u |arg| for each rounded argument);
    the terms within 40 of the max carry all but e^-40 of the sum, the rest are bounded by their share. The sum adds
    at most gamma_(4 n_it + 10). ln(1 + rho) <= rho; logf is within 1 ulp and gm + log one more rounding."""
    x64 = x.double()
    m = x64.amax(1, keepdim=True)
    lse = m[:, 0] + torch.log(torch.exp(x64 - m).sum(1))
    W = (m - x64.amin(1, keepdim=True))[:, 0]
    n_it = -(-(V // 4) // CE_THREADS) + 1
    rho = 2 * U * (2 * (n_it + 2) + 1.7 * (W + 40)) + gamma(4 * n_it + 10) + math.exp(-40)
    log_gs = lse - m[:, 0]
    err = 1.01 * (rho + 2 * U * log_gs.abs() + U * lse.abs())
    return lse, err


def ce_dlogits_ref(x, lse, lse64, labels, gs):
    """fp64 (softmax - onehot) * gs (0 on ignored rows) and the kernel's error before its bf16 rounding. The kernel
    uses its own lse (returned in lse_out), so that error is measured, not bounded: exp(fl(x - lse)) is off by
    |lse - lse64| + u |arg| + `_expf_rel`(arg) relative; - onehot and * gs round once each.
    err = 1.01 gs (p (dlse + u |arg| + e_exp) + u |p - onehot|) + u |ref| + 2^-148."""
    x64 = x.double()
    valid = (labels != -100)[:, None]
    p = torch.exp(x64 - lse64[:, None])
    oh = torch.zeros_like(p)
    rows = torch.nonzero(valid[:, 0])[:, 0]
    oh[rows, labels.long()[rows]] = 1.0
    ref = (p - oh) * gs * valid
    dlse = (lse.double() - lse64).abs()[:, None]
    arg = x64 - lse.double()[:, None]
    err = 1.01 * gs * (p * (dlse + U * arg.abs() + _expf_rel(arg)) + U * (p - oh).abs()) + U * ref.abs() + 2.0 ** -148
    return ref, err * valid


def ce_rows(R, V, gen):
    """Rows by kind r mod 4: flat N(0, 1); peaked (one logit 80 above the rest, at the last column on odd rows: the
    maximum sits in both scalar tails when V mod 8 != 0); N(0, 1) + 1e4; N(0, 1) - 1e4."""
    x = torch.randn(R, V, generator=gen, dtype=torch.float64)
    for r in range(R):
        k = r % 4
        if k == 1:
            x[r, V - 1 if r % 2 else int(torch.randint(0, V, (1,), generator=gen))] += 80
        elif k == 2:
            x[r] += 1e4
        elif k == 3:
            x[r] -= 1e4
    return x.float()


def ce_labels(R, V):
    """0, V - 1, V - 2 and one label in each scalar tail, cycled; two rows ignored."""
    tail = [V & ~3, V & ~7, (V & ~7) + 3]
    cyc = [0, V - 1, max(V - 2, 0)] + [t for t in tail if t < V]
    lab = [cyc[r % len(cyc)] for r in range(R)]
    lab[3] = lab[R - 2] = -100
    return torch.tensor(lab, dtype=torch.int32)


@pytest.mark.parametrize("V", [1, 3, 4, 7, 8, 9, 2047, 128258])
@pytest.mark.parametrize("pad_d", [0, 8])
def test_cross_entropy_tails_lse_dlogits_and_exact_sum(cuda_device, V, pad_d):
    from metamorph_b200 import ops
    R = 12
    ld, ld_d = -(-V // 4) * 4, -(-V // 8) * 8 + pad_d
    V4, V8 = V & ~3, V & ~7
    assert (V4 < V) == (V % 4 != 0) and (V8 < V) == (V % 8 != 0)
    gen = torch.Generator().manual_seed(V + pad_d)
    xv = ce_rows(R, V, gen)
    labels = ce_labels(R, V)
    big_row = 5                                              # one term above the fixed-point limit: the fp64 side sum
    limit = float(np.float32(2.0 ** 62 / (2.0 ** 32 * R)))
    labels[big_row] = 0
    xv[big_row] = 0.0
    if V > 1:
        xv[big_row, 0] = -3e8
    buf = torch.full((R, ld), 1e30, dtype=torch.float32)      # pitch padding the kernel must not read
    buf[:, :V] = xv
    buf, labels = buf.to(cuda_device), labels.to(cuda_device)
    x = buf[:, :V]
    valid = labels != -100
    n_valid = int(valid.sum())
    gs = float(np.float32(1.0 / n_valid))                     # the kernel's fp32 grad_scale
    loss = torch.zeros(1, device=cuda_device)
    lse = torch.full((R,), float("nan"), device=cuda_device)
    dl = torch.full((R, ld_d), float("nan"), device=cuda_device, dtype=torch.bfloat16)
    ops.ce_fwd_bwd(buf, labels, V, loss, dlogits=dl, grad_scale=gs, lse_out=lse)

    lse64, lerr = ce_lse_bound(x, V)
    worst = assert_within(lse, lse64, lerr, f"CE lse V={V}")
    ref, err = ce_dlogits_ref(x, lse, lse64, labels, gs)
    n = assert_rounds_within(dl[:, :V], ref, err, f"CE dlogits V={V} ld_d={ld_d}")
    lab = labels.long()
    assert bool((dl[:, V:] == 0).all()), "columns [V, ld_d) must be exactly 0"
    assert bool((dl[~valid] == 0).all()), "ignored rows must have exactly 0 gradient"

    # the loss sum, exactly: terms fp32(lse_r - x[r, label_r]); |t| < limit as llrint(t * 2^32), the rest in fp64
    terms = (lse[valid] - x[valid, lab[valid]]).cpu().numpy().astype(np.float32)
    fixed, big = 0, 0.0
    for t in terms:
        if abs(t) < limit:
            fixed += round(float(t) * 2.0 ** 32)
        else:
            big += float(t)
    assert (V == 1) or big > 0, "no term took the fp64 side sum"
    want = np.float32(float(fixed) / 2.0 ** 32 + big)
    assert loss.item() == float(want), f"CE loss sum {loss.item()!r} != {float(want)!r}"

    # the same rows without lse_out: ignored rows take the early exit; the sum and gradient do not change
    loss2 = torch.zeros(1, device=cuda_device)
    dl2 = torch.full_like(dl, float("nan"))
    ops.ce_fwd_bwd(buf, labels, V, loss2, dlogits=dl2, grad_scale=gs)
    assert loss2.item() == loss.item()
    assert_equal(dl2, dl, "dlogits without lse_out")
    print(f"CE V={V} ld_d={ld_d}: lse at {worst:.3g} of its bound; {n} dlogits needed the fp32 slack")


# ------------------------------------------------------------------------------------------------ cosine loss
# loss.cu:127-204, 271-285: one warp per row, 4 warps per block, grid = min(ceil(R / 4), #SMs * 8); lane l takes the
# 8-wide vectors l, l + 32, ... (C / 8 of them). pn = max(bf16(sqrtf(sum p^2)), 1e-12); h = bf16(p / pn) is pred_norm;
# tp, tt, hh sums; cos = tp / (max(sqrtf(tt), 1e-8) max(sqrtf(hh), 1e-8)); loss term -cos / R;
# dpred = bf16(g (t / tn - cos p / pn)), g = -grad_scale / (R pn).
def _pn_candidates(p64, n_chain):
    nrm = p64.pow(2).sum(1, keepdim=True).sqrt()
    e = nrm * (0.5 * gamma(n_chain) + U) * 1.01
    e12 = float(np.float32(1e-12))
    return _rnd(nrm - e).clamp(min=e12), _rnd(nrm + e).clamp(min=e12)


def cosine_ref(pred, tgt, h, R, gscale):
    """fp64 cosine loss from the kernel's own (checked) pred_norm h, for each possible bf16 norm pn.

    Sums of exact products within gamma_n of sum |terms| (n = 8 ceil(C / 256) + 5); sqrtf adds u, the divide 2u:
      err_cos = gamma_n sum|t h| / (tn hn) + |cos| (gamma_n + 4u).
    inner = t / tn - cos p / pn: err_in = |t / tn| (0.5 gamma_n + 2u) + |p / pn| (err_cos + 2u |cos|) + u |inner|.
    dpred = fl(g inner), g within 3u: err = 1.01 (|g| err_in + 4u |dpred|).
    Returns ((lo, hi) of dpred over both norms, loss64, loss bound)."""
    p64, t64, h64 = pred.double(), tgt.double(), h.double()
    C = p64.shape[1]
    n = 8 * -(-C // 256) + 5
    tn = t64.pow(2).sum(1, keepdim=True).sqrt().clamp(min=1e-8)
    hn = h64.pow(2).sum(1, keepdim=True).sqrt().clamp(min=float(np.float32(1e-8)))
    tp = (t64 * h64).sum(1, keepdim=True)
    cos = tp / (tn * hn)
    err_cos = gamma(n) * (t64 * h64).abs().sum(1, keepdim=True) / (tn * hn) + cos.abs() * (gamma(n) + 4 * U)
    lo = hi = None
    for pn in _pn_candidates(p64, n):
        g = -gscale / (R * pn)
        inner = t64 / tn - cos * p64 / pn
        err_in = (t64 / tn).abs() * (0.5 * gamma(n) + 2 * U) + (p64 / pn).abs() * (err_cos + 2 * U * cos.abs()) \
            + U * inner.abs()
        ref = g * inner
        err = 1.01 * (g.abs() * err_in + 4 * U * ref.abs())
        a, b = _rnd(ref - err), _rnd(ref + err)
        lo = a if lo is None else torch.minimum(lo, a)
        hi = b if hi is None else torch.maximum(hi, b)
    loss = float((-cos / R).sum())
    lerr = float((err_cos + 2 * U * cos.abs()).sum() / R) + R * 2.0 ** -40 + U * abs(loss)
    return (lo, hi), loss, lerr


@pytest.mark.parametrize("C", [8, 248, 256, 264, 1152, 4096])
@pytest.mark.parametrize("Rk", ["1", "3", "4", "5", "sms*32+1"])
def test_cosine_loss_against_bf16_semantics_in_fp64(cuda_device, C, Rk):
    from metamorph_b200 import ops
    from tests.test_rowwise_exact_gpu import bf16_norm_interval
    sms = _sms(cuda_device)
    R = sms * 32 + 1 if Rk == "sms*32+1" else int(Rk)
    grid = min(-(-R // 4), sms * 8)
    assert (R > grid * 4) == (Rk == "sms*32+1")                 # a warp takes a second row
    gen = torch.Generator().manual_seed(C * 31 + R)
    pred = torch.randn(R, C, generator=gen) * torch.pow(2.0, (torch.arange(R) % 5 - 2).float())[:, None]
    tgt = torch.randn(R, C, generator=gen)
    pred[R // 2] = 0                                             # a zero prediction: pred_norm 0, a finite loss
    pred, tgt = pred.bfloat16().to(cuda_device), tgt.bfloat16().to(cuda_device)
    gscale = 0.75
    ls = torch.zeros(1, device=cuda_device)
    pn = torch.full_like(pred, float("nan"))
    dp = torch.full_like(pred, float("nan"))
    ops.cosine_loss(pred, tgt, loss_sum=ls, pred_norm=pn, dpred=dp, grad_scale=gscale)
    n_chain = 8 * -(-C // 256) + 5
    lo, hi = bf16_norm_interval(pred, 1e-12, n_chain)
    assert_between(pn, lo, hi, f"cosine pred_norm C={C} R={R}")
    assert bool((pn[R // 2] == 0).all())
    (dlo, dhi), loss64, lerr = cosine_ref(pred, tgt, pn, R, gscale)
    assert_between(dp, dlo, dhi, f"cosine dpred C={C} R={R}")
    assert math.isfinite(ls.item())
    worst = abs(ls.item() - loss64) / lerr
    assert worst <= 1.0, f"cosine loss {ls.item()!r} vs fp64 {loss64!r}: {worst:.3g} x the bound {lerr:.3e}"
    # without a target only pred_norm is written
    ls2 = torch.full((1,), 5.0, device=cuda_device)
    pn2 = torch.full_like(pred, float("nan"))
    dp2 = torch.full_like(pred, float("nan"))
    ops.cosine_loss(pred, None, loss_sum=ls2, pred_norm=pn2, dpred=dp2)
    assert_equal(pn2, pn, "pred_norm without a target")
    assert bool(torch.isnan(dp2).all()) and ls2.item() == 5.0, "target=None must write only pred_norm"
    print(f"cosine C={C} R={R}: loss at {worst:.3g} of its bound")


# ------------------------------------------------------------------------------------------------ argmax
# loss.cu:206-252, 287-302: stage 1 is a (R, 64) grid; split s scans [s per, min(V, (s + 1) per)), per = ceil(V / 64),
# so splits from ceil(V / per) on are empty; a thread keeps the first index of its strict maximum, then warp and block
# combines take the larger value or, on a tie, the lower index. Stage 2 combines the 64 partials the same way. NaN never
# compares greater, so it is never chosen; a row with no value above -inf returns 0 (DESIGN.md section 1), where
# torch.argmax would return the first NaN or 0.
def argmax_ref(x):
    """Lowest index of the maximum over the non-NaN values; 0 when no value is above -inf."""
    y = torch.nan_to_num(x.double(), nan=-math.inf, posinf=math.inf, neginf=-math.inf)
    m = y.amax(1, keepdim=True)
    idx = (y == m).int().argmax(1)
    return torch.where(m[:, 0] > -math.inf, idx, torch.zeros_like(idx)).int()


ARGMAX_KINDS = ["first_col", "last_col", "split_edge", "tie_across_splits", "pos_inf", "neg_inf_but_one", "nan_mixed",
                "all_neg_inf", "all_nan", "nan_and_neg_inf", "random"]
NO_FINITE = ["all_neg_inf", "all_nan", "nan_and_neg_inf"]


def argmax_row(kind, V, r, gen):
    per = -(-V // 64)
    x = torch.randn(V, generator=gen)

    def top(j, v=50.0):
        x[min(j, V - 1)] = v

    if kind == "first_col":
        top(0)
    elif kind == "last_col":
        top(V - 1)
    elif kind == "split_edge":
        top(((r % 63) + 1) * per)
    elif kind == "tie_across_splits":
        top(V - 1, 60.0)
        top(V // 2, 60.0)
        top(per, 60.0)
    elif kind == "pos_inf":
        top(V - 1, math.inf)
        top((V * 2) // 3, math.inf)
    elif kind == "neg_inf_but_one":
        x[:] = -math.inf
        top(int(torch.randint(0, V, (1,), generator=gen)), -1e30)
    elif kind == "nan_mixed":
        x[torch.randint(0, V, (max(1, V // 10),), generator=gen)] = math.nan
        top(V // 3, 7.0)
        if V > 2:                                              # NaN first and right after the maximum
            x[0] = x[V // 3 + 1] = math.nan
    elif kind == "all_neg_inf":
        x[:] = -math.inf
    elif kind == "all_nan":
        x[:] = math.nan
    elif kind == "nan_and_neg_inf":
        x[:] = -math.inf
        x[torch.randint(0, V, (max(1, V // 3),), generator=gen)] = math.nan
    return x


def _argmax_case(dev, R, V, kinds, seed):
    from metamorph_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    ld = V + 3
    buf = torch.full((R, ld), 1e38)                            # pitch padding above every row's maximum: never read
    for r in range(R):
        buf[r, :V] = argmax_row(kinds[r % len(kinds)], V, r, gen)
    buf = buf.to(dev)
    got = ops.argmax_rows(buf, V)
    want = argmax_ref(buf[:, :V])
    assert_equal(got, want, f"argmax V={V} R={R}")
    prm = (torch.zeros(R, device=dev), torch.zeros(R, dtype=torch.int32, device=dev), torch.ones(R, device=dev),
           torch.zeros(R, dtype=torch.int64, device=dev), torch.zeros(R, dtype=torch.int32, device=dev))
    sampled = ops.sample_rows(buf, V, *prm)
    assert_equal(sampled, got, f"sample_rows at T = 0 vs argmax V={V} R={R}")


@pytest.mark.parametrize("V", [1, 63, 64, 65, 128258])
@pytest.mark.parametrize("R", [1, 37, 128])
def test_argmax_rows_splits_ties_inf_nan(cuda_device, V, R):
    per = -(-V // 64)
    used = -(-V // per)
    assert (used < 64) == (V in (1, 63, 65))                    # empty splits below V = 64 and at 65 (per = 2)
    kinds = [k for k in ARGMAX_KINDS if k not in NO_FINITE]
    if R == 1:
        for i, k in enumerate(kinds):
            _argmax_case(cuda_device, 1, V, [k], seed=V + i)
    else:
        _argmax_case(cuda_device, R, V, kinds, seed=V + R)


@pytest.mark.parametrize("V", [1, 63, 64, 65, 128258])
def test_argmax_rows_without_a_value_above_minus_inf_give_0(cuda_device, V):
    """All -inf, all NaN, and NaN mixed with -inf: 0, the sampler's answer for such rows, never 0x7fffffff."""
    for R in (1, 37):
        _argmax_case(cuda_device, R, V, NO_FINITE + ["random"], seed=V * 3 + R)
