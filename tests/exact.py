"""Exactness and error-bound checkers shared by the fp64 parity tests (tests only).

The parity tests hold a kernel to an fp64 restatement of the same operation in one of three ways:
  * integer-valued inputs whose every partial sum is exactly representable: the kernel must equal the reference after
    one rounding to its output dtype (`assert_equal`);
  * a bound derived per element from the summation length (`gamma`, `ulp_bf16`, `assert_within`);
  * for attention, where the kernel's error has no closed form: no worse than k times the error of the same formula
    computed by torch in bf16 (`assert_no_worse_than`);
  * for kernels that compute in fp32 and round once to bf16: between the correct roundings of the fp64 value minus and
    plus a derived fp32 error bound (`round_bf16_from_fp64`, `assert_rounds_within`, `assert_between`).
Each check names the worst element, so a failure points at a tile, a row group and a column chunk.
"""
import torch

U = 2.0 ** -24          # fp32 unit roundoff


def gamma(n, u=U):
    """Higham's gamma_n: a sum evaluated along a chain of n fp32 additions is within gamma_n * sum|terms| of the exact sum."""
    return n * u / (1 - n * u)


def expf_fast_rel(arg):
    """__expf: 2 + floor(1.173 |x|) ulp (CUDA C Programming Guide, intrinsic functions), 1 ulp <= 2u relative."""
    return (2 + torch.floor(1.173 * arg.abs())) * 2 * U


def ints(shape, lo, hi, device, dtype=torch.bfloat16, gen=None):
    return torch.randint(lo, hi + 1, shape, device=device, generator=gen).to(dtype)


def ulp_bf16(y):
    """Spacing of bf16 numbers at |y| (8 significant bits): 2^(e - 8) for y = f * 2^e, 0.5 <= |f| < 1."""
    _, e = torch.frexp(y.abs().float())
    return torch.ldexp(torch.ones_like(y, dtype=torch.float64), e.to(torch.float64) - 8)


def _where(t, flat):
    return tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), t.shape))


def assert_equal(got, want, what):
    """Bit equality (NaN never equals anything), reporting the first differing element and the number of them."""
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    g, w = got.double(), want.double()
    bad = ~(g == w)
    if bool(bad.any()):
        flat = int(bad.reshape(-1).nonzero()[0])
        idx = _where(g, flat)
        raise AssertionError(f"{what}: {int(bad.sum())} of {g.numel()} elements differ; first at {idx}: "
                             f"got {float(g[idx])!r}, want {float(w[idx])!r}")


def assert_within(got, ref, bound, what):
    """|got - ref| <= bound element by element (a NaN fails). Reports the worst element's index and err / bound there.
    Returns the largest ratio err / bound, for the caller to report."""
    err = (got.double() - ref.double()).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=err.device).expand_as(err)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    flat = int(ratio.reshape(-1).argmax())
    idx = _where(err, flat)
    worst = float(ratio[idx])
    assert worst <= 1.0, (f"{what}: worst element {idx}: got {float(got[idx])!r}, ref {float(ref[idx])!r}, "
                          f"err {float(err[idx]):.3e} = {worst:.3g} x the bound {float(bound[idx]):.3e}; "
                          f"{int((ratio > 1).sum())} elements over")
    return worst


def round_bf16_from_fp64(x):
    """fp64 -> bf16 rounded once, to nearest even. torch's float64 -> bfloat16 cast goes through fp32 and so rounds
    twice (1 + 2^-8 + 2^-30 becomes 1.0, not 1 + 2^-7). Here the fp32 step rounds to odd instead: truncate towards zero,
    then set the last bit if anything was dropped. 24 bits is more than 8 + 2, so the final round-to-nearest-even from
    that fp32 value is the correctly rounded bf16 value; overflow past fp32 truncates to FLT_MAX (odd), which rounds to
    inf as it should, and NaN and inf pass through."""
    x = x.double()
    f = x.float()
    over = f.double().abs() > x.abs()                                     # rounded away from zero: step back
    f = torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)
    inexact = (f.double() != x) & torch.isfinite(x)
    bits = f.view(torch.int32)
    f = torch.where(inexact, bits | 1, bits).view(torch.float32)
    return f.to(torch.bfloat16)


def assert_between(got, lo, hi, what):
    """lo <= got <= hi element by element; a NaN bound demands a NaN result, and a NaN result needs a NaN bound.
    Reports the worst element in units of the bf16 spacing there. Returns the number of elements that are not lo
    (with lo == hi that is 0)."""
    g, lo, hi = got.double(), lo.double(), hi.double()
    assert g.shape == lo.shape == hi.shape, f"{what}: shapes {tuple(g.shape)} {tuple(lo.shape)} {tuple(hi.shape)}"
    want_nan = torch.isnan(lo) | torch.isnan(hi)
    bad_nan = want_nan != torch.isnan(g)
    inside = want_nan | ((g >= lo) & (g <= hi))
    out = torch.where(inside, torch.zeros_like(g), torch.maximum(lo - g, g - hi))
    out = torch.nan_to_num(out, nan=float("inf"), posinf=float("inf"))
    score = torch.where(bad_nan, torch.full_like(g, float("inf")),
                        out / ulp_bf16(torch.where(torch.isfinite(lo), lo, g)).clamp(min=2.0 ** -133))
    score = torch.nan_to_num(score, nan=float("inf"))
    flat = int(score.reshape(-1).argmax())
    idx = _where(g, flat)
    if float(score[idx]) > 0:
        raise AssertionError(f"{what}: {int((score > 0).sum())} of {g.numel()} elements outside their rounding "
                             f"interval; worst {idx}: got {float(g[idx])!r}, allowed [{float(lo[idx])!r}, "
                             f"{float(hi[idx])!r}] ({float(score[idx]):.3g} bf16 ulps out)")
    return int(((g != lo) & ~want_nan).sum())


def assert_rounds_within(got_bf16, ref64, err64, what):
    """A kernel that computes ref64 in fp32 with an error of at most err64 and rounds once to bf16 must return a value in
    [round(ref64 - err64), round(ref64 + err64)] (`round_bf16_from_fp64`). Away from a rounding boundary that is bit
    equality with round(ref64); within err64 of one it admits exactly the two neighbours. ±inf and NaN references
    demand the same result. Returns the number of elements that differ from round(ref64) (they needed err64)."""
    ref64 = ref64.double()
    err64 = torch.as_tensor(err64, dtype=torch.float64, device=ref64.device).expand_as(ref64)
    assert bool((err64 >= 0).all()), f"{what}: negative error bound"
    fin = torch.isfinite(ref64)
    lo = torch.where(fin, ref64 - err64, ref64)
    hi = torch.where(fin, ref64 + err64, ref64)
    assert_between(got_bf16, round_bf16_from_fp64(lo).double(), round_bf16_from_fp64(hi).double(), what)
    r = round_bf16_from_fp64(ref64).double()
    return int(((got_bf16.double() != r) & ~torch.isnan(r)).sum())


def rounding_slack(got_bf16, ref64, err64):
    """How far into its bound a result that passed `assert_rounds_within` went: (the number of elements that differ from
    round(ref64), the largest |midpoint - ref64| / err64 over them). Such an element's fp32 value lay beyond the midpoint
    between round(ref64) and the value returned, so the ratio is a lower bound on that element's err / bound."""
    g, ref64 = got_bf16.double(), ref64.double()
    err64 = torch.as_tensor(err64, dtype=torch.float64, device=ref64.device).expand_as(ref64)
    r = round_bf16_from_fp64(ref64).double()
    off = (g != r) & torch.isfinite(r) & torch.isfinite(g)
    if not bool(off.any()):
        return 0, 0.0
    mid = (g[off] + r[off]) / 2
    return int(off.sum()), float(((mid - ref64[off]).abs() / err64[off]).max())


def err_stats(x, ref):
    """(max, rms) of |x - ref| in fp64."""
    e = (x.double() - ref.double()).abs()
    return float(e.max()), float(e.pow(2).mean().sqrt())


def assert_no_worse_than(got, ref64, torch_path, what, k=2.0, floor=0.0):
    """The kernel's max and rms error against fp64 must not exceed k times the error of `torch_path` (the same formula
    evaluated in bf16 / fp32 by torch) against fp64, plus `floor`. Non-finite results fail."""
    assert bool(torch.isfinite(got.double()).all()), f"{what}: non-finite output"
    g_max, g_rms = err_stats(got, ref64)
    t_max, t_rms = err_stats(torch_path, ref64)
    assert g_max <= k * t_max + floor, f"{what}: max err {g_max:.3e} > {k} x torch bf16 {t_max:.3e} + {floor:.1e}"
    assert g_rms <= k * t_rms + floor, f"{what}: rms err {g_rms:.3e} > {k} x torch bf16 {t_rms:.3e} + {floor:.1e}"
    return g_max, t_max
