"""Exactness and error-bound checkers shared by the fp64 parity tests (tests only).

The parity tests hold a kernel to an fp64 restatement of the same operation in one of three ways:
  * integer-valued inputs whose every partial sum is exactly representable: the kernel must equal the reference after
    one rounding to its output dtype (`assert_equal`);
  * a bound derived per element from the summation length (`gamma`, `ulp_bf16`, `assert_within`);
  * for attention, where the kernel's error has no closed form: no worse than k times the error of the same formula
    computed by torch in bf16 (`assert_no_worse_than`).
Each check names the worst element, so a failure points at a tile, a row group and a column chunk.
"""
import torch

U = 2.0 ** -24          # fp32 unit roundoff


def gamma(n, u=U):
    """Higham's gamma_n: a sum evaluated along a chain of n fp32 additions is within gamma_n * sum|terms| of the exact sum."""
    return n * u / (1 - n * u)


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
