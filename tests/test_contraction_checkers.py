"""The checkers of the GEMM and attention parity tests have teeth (CPU only).

Each test emulates in torch one kernel bug those tests exist to catch, on the shapes and data generators the GPU tests
use, and requires the GPU tests' own checker to reject it; the clean emulation must pass the same checker. Nothing here
builds or runs a kernel.
"""
import math

import pytest
import torch

from tests.exact import assert_equal, assert_no_worse_than
from tests.test_attention_edges_gpu import (D, PEAK_LENS, PEAK_T, SHAPES, _allowed, _bhtd, _ref64, _split, _torch_bf16,
                                            check_probe_fwd, peaked_inputs, probe_inputs)
from tests.test_gemm_exact_gpu import BM, _epi_shape, int_operands

CPU = torch.device("cpu")
SMS = 132                  # the H100 SXM's SM count, for the GPU tests' shapes


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.fixture(scope="module")
def gemm_case():
    """The epilogue test's (K, K) operands and fp64 product, with its integer bias and residual."""
    M, N, K = _epi_shape(SMS)
    a, b, c = int_operands(M, N, K, False, False, CPU, seed=7 + 128)
    gen = torch.Generator().manual_seed(11)
    bias = torch.randint(-8, 9, (N,), generator=gen).double()
    r = torch.randint(-64, 65, (M, N), generator=gen).double()
    return a.double(), b.double(), c, bias, r


def _bug_dropped_k_slice(a, b, c, bias, r):
    """k-slice 3 (k 48..63) dropped for the second 64-row half of tile (1, 2) at BN = 128."""
    rows, cols, ks = slice(BM + 64, 2 * BM), slice(256, 384), slice(48, 64)
    got = c.clone()
    got[rows, cols] -= a[rows, ks] @ b[cols, ks].t()
    return got, c


def _bug_swapped_row_groups(a, b, c, bias, r):
    """Row groups 136..143 and 144..151 (two 8-row groups of one warp's fragment) swapped."""
    got = c.clone()
    got[136:144], got[144:152] = c[144:152], c[136:144]
    return got, c


def _bug_partial_chunk_without_bias(a, b, c, bias, r):
    """EPI_BIAS at alpha 1/2: the last, partial 32-column chunk (columns 1152..1159) misses its bias."""
    want = c * 0.5 + bias
    got = want.clone()
    got[:, 1152:] -= bias[1152:]
    return got, want


def _bug_alpha_after_residual(a, b, c, bias, r):
    """EPI_RESID at alpha 1/2 computing alpha (C + R) instead of alpha C + R."""
    return 0.5 * (c + r), 0.5 * c + r


def _bug_previous_n_block(a, b, c, bias, r):
    """Tile (2, 3) at BN = 128 computed with tile (2, 2)'s n-block."""
    got = c.clone()
    got[2 * BM:3 * BM, 384:512] = c[2 * BM:3 * BM, 256:384]
    return got, c


GEMM_BUGS = [_bug_dropped_k_slice, _bug_swapped_row_groups, _bug_partial_chunk_without_bias, _bug_alpha_after_residual,
             _bug_previous_n_block]


@pytest.mark.parametrize("bug", GEMM_BUGS, ids=lambda f: f.__name__[5:])
def test_gemm_exact_check_rejects(gemm_case, bug):
    got, want = bug(*gemm_case)
    assert_equal(want.to(torch.bfloat16), want.to(torch.bfloat16), "clean")
    with pytest.raises(AssertionError) as e:
        assert_equal(got.to(torch.bfloat16), want.to(torch.bfloat16), bug.__name__[5:])
    print(f"rejected: {e.value}")


# ------------------------------------------------------------------------------------------------ attention
def _flash_fwd(q, k, v, allowed, scale, G, skip_rescale_tile=None):
    """The forward kernel's online softmax over 128-key tiles in fp32 (P cast to bf16 before P V), optionally without
    the O rescale on one tile."""
    kk, vv = k.float().repeat_interleave(G, 1), v.float().repeat_interleave(G, 1)
    q = q.float()
    B, H, T, _ = q.shape
    m = torch.full((B, H, T, 1), float("-inf"))
    l = torch.zeros(B, H, T, 1)
    o = torch.zeros(B, H, T, D)
    for t in range(math.ceil(T / 128)):
        ks = slice(128 * t, 128 * (t + 1))
        s = (q @ kk[:, :, ks].transpose(-1, -2) * scale).masked_fill(~allowed[..., ks], float("-inf"))
        m_new = torch.maximum(m, s.amax(-1, keepdim=True))
        live = m_new > float("-inf")
        corr = torch.where(live, torch.exp(m - m_new), torch.ones_like(m))
        p = torch.where(live, torch.exp(s - m_new), torch.zeros_like(s))
        l = l * corr + p.sum(-1, keepdim=True)
        if t != skip_rescale_tile:
            o = o * corr
        o = o + p.bfloat16().float() @ vv[:, :, ks]
        m = m_new
    return (o / l).bfloat16(), (m + torch.log(l))[..., 0]


@pytest.fixture(scope="module")
def peaked_case():
    Hq, Hkv = 8, 2
    qkv, dout = peaked_inputs(Hq, Hkv, CPU, seed=4)
    B, T = len(PEAK_LENS), PEAK_T
    q, k, v = (_bhtd(x, B, T, h) for x, h in zip(_split(qkv, Hq, Hkv), (Hq, Hkv, Hkv)))
    allowed = _allowed(PEAK_LENS, T, True, CPU)
    o64, _, _ = _ref64(q, k, v, None, allowed, D ** -0.5, Hq // Hkv)
    ot, _, _ = _torch_bf16(q, k, v, None, allowed, D ** -0.5, Hq // Hkv)
    return q, k, v, allowed, o64, ot, Hq // Hkv


def test_peaked_check_rejects_a_missing_rescale_on_a_late_tile(peaked_case):
    """Tile 4 is the last key tile of the 523-row sequence; its key 520 lifts the running max by about 4."""
    q, k, v, allowed, o64, ot, G = peaked_case
    vr = torch.arange(PEAK_T)[None, :] < torch.tensor(PEAK_LENS)[:, None]
    sel = lambda x: x.transpose(1, 2)[vr]
    clean, _ = _flash_fwd(q, k, v, allowed, D ** -0.5, G)
    floor = 2.0 ** -12 * float(sel(o64).abs().max())
    assert_no_worse_than(sel(clean), sel(o64), sel(ot), "clean online softmax", floor=floor)
    bad, _ = _flash_fwd(q, k, v, allowed, D ** -0.5, G, skip_rescale_tile=4)
    with pytest.raises(AssertionError) as e:
        assert_no_worse_than(sel(bad), sel(o64), sel(ot), "no O rescale on tile 4", floor=floor)
    print(f"rejected: {e.value}")


@pytest.fixture(scope="module")
def probe_case():
    T, lens = SHAPES["lens=1..257-T259"]
    Hq, Hkv = 8, 2
    qkv, jkey = probe_inputs(T, lens, Hq, Hkv, CPU, seed=1)
    B = len(lens)
    q, k, v = (_bhtd(x, B, T, h) for x, h in zip(_split(qkv, Hq, Hkv), (Hq, Hkv, Hkv)))
    return q, k, v, jkey, T, lens, Hq // Hkv


def _probe_run(probe_case, allowed, lse_bug=False):
    q, k, v, jkey, T, lens, G = probe_case
    o, lse, _ = _torch_bf16(q, k, v, None, allowed, D ** -0.5, G)
    if lse_bug:
        lse = lse.clone()
        lse[8, 1, 70] += math.log(2)
    return o, lse


def _mask_causal_strict(T, lens):
    j = torch.arange(T)
    return _allowed(lens, T, True, CPU) & (j[None, None, None, :] < j[None, None, :, None])


def _mask_last_partial_key_tile_dropped(T, lens):
    full_tiles = torch.tensor(lens) // 128 * 128
    keep = torch.arange(T)[None, :] < torch.where(torch.tensor(lens) % 128 == 0, torch.tensor(lens), full_tiles)[:, None]
    return _allowed(lens, T, True, CPU) & keep[:, None, None, :]


PROBE_BUGS = {"causal mask col < row": (_mask_causal_strict, False),
              "last partial key tile dropped": (_mask_last_partial_key_tile_dropped, False),
              "lse off by ln 2 on one row": (lambda T, lens: _allowed(lens, T, True, CPU), True)}


@pytest.mark.parametrize("bug", list(PROBE_BUGS))
def test_mask_probe_rejects(probe_case, bug):
    q, k, v, jkey, T, lens, G = probe_case
    o, lse = _probe_run(probe_case, _allowed(lens, T, True, CPU))
    check_probe_fwd(o, lse, jkey, lens, T, G, True, "clean")
    mask, lse_bug = PROBE_BUGS[bug]
    o, lse = _probe_run(probe_case, mask(T, lens), lse_bug)
    with pytest.raises(AssertionError) as e:
        check_probe_fwd(o, lse, jkey, lens, T, G, True, bug)
    print(f"rejected: {e.value}")
