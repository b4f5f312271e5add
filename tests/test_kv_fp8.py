"""CPU tests of the FP8 KV-cache row rule (oracle/kv_fp8.py) and of the kv_cache_dtype argument checks.

The oracle's bytes must equal torch's float8_e4m3fn conversion of x 2^-e (round to nearest even) on random rows and at
the rule's edges, and its x-hat must be a bf16 value."""
import numpy as np
import pytest
import torch

from oracle.kv_fp8 import E_MAX, E_MIN, NAN_BYTE, dequantise, e4m3_decode, quantise_rows, row_exponent

D = 128


def _bf16(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float64)).bfloat16().double().numpy()


def _torch_bytes(row, e):
    """RNE_e4m3(x 2^-e) by torch, with the rule's one exception: at e = 120 a 256 (0x78) stores 240 (0x77)."""
    q = torch.tensor(np.ldexp(row, -e), dtype=torch.float64).float().to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    return np.where((q & 0x7F) == 0x78, (q & 0x80) | 0x77, q).astype(np.uint8) if e == E_MAX else q


def edge_rows():
    """Rows of bf16 values at the edges of the rule, each with a name."""
    g = np.random.default_rng(7)
    base = _bf16(g.standard_normal(D))
    rows = {"zero": np.zeros(D), "neg_zero": -np.zeros(D)}
    for k in (-3, 0, 5):                                  # a = 448 2^k exactly and one bf16 ulp either side
        r = _bf16(base / np.abs(base).max() * 400 * 2.0 ** k)
        for name, a in (("at", 448.0 * 2.0 ** k), ("above", 448.0 * 2.0 ** k * (1 + 2.0 ** -7))):
            rr = r.copy()
            rr[3] = a
            rows[f"a_{name}_448x2^{k}"] = _bf16(rr)
        rr = r.copy()
        rr[3] = 448.0 * 2.0 ** k * (1 - 2.0 ** -8)               # the bf16 value below 448 2^k
        rows[f"a_below_448x2^{k}"] = _bf16(rr)
    sub = base.copy()                                     # entries that land on E4M3 subnormals (below 2^-6 after scaling)
    sub[:32] = base[:32] * 2.0 ** -9
    sub[5] = 448.0
    rows["subnormal_e4m3"] = _bf16(sub)
    rows["half_way_ties"] = _bf16(np.concatenate([[448.0], (np.arange(1, D) % 16 + 16.5) / 16 * 2.0 ** -3]))
    rows["e_min_clamp"] = _bf16(base * 2.0 ** -128)       # a far below 448 2^-124: e clamps at -124
    rows["at_e_min"] = _bf16(base / np.abs(base).max() * 448 * 2.0 ** -124)
    rows["bf16_min_subnormal"] = _bf16(np.where(np.arange(D) % 2, 2.0 ** -133, -(2.0 ** -133)))
    big = float(torch.finfo(torch.bfloat16).max)
    rows["largest_bf16"] = _bf16(np.where(np.arange(D) % 3, big, -big / 3))
    for name, bad in (("inf", np.inf), ("neg_inf", -np.inf), ("nan", np.nan)):
        rr = base.copy()
        rr[17] = bad
        rows[name] = rr
    return rows


def test_oracle_bytes_equal_torch_e4m3_on_random_rows():
    g = np.random.default_rng(0)
    x = _bf16(g.standard_normal((256, D)) * np.ldexp(1.0, g.integers(-126, 125, (256, 1))))
    q, sc, xh = quantise_rows(x)
    for r in range(x.shape[0]):
        e = row_exponent(x[r])
        assert float(sc[r]) == 2.0 ** e
        assert np.array_equal(q[r], _torch_bytes(x[r], e)), r
        assert np.abs(x[r]).max() <= 448 * 2.0 ** e and (e == E_MIN or np.abs(x[r]).max() > 448 * 2.0 ** (e - 1))
    assert np.array_equal(_bf16(xh), xh), "x-hat is not a bf16 value"


@pytest.mark.parametrize("name", list(edge_rows()))
def test_oracle_edge_rows(name):
    row = edge_rows()[name]
    q, sc, xh = quantise_rows(row[None])
    q, sc, xh = q[0], float(sc[0]), xh[0]
    if not np.all(np.isfinite(row)):
        assert (q == NAN_BYTE).all() and sc == 1.0 and np.isnan(xh).all()
        return
    e = row_exponent(row)
    assert sc == 2.0 ** e and np.float32(sc) == sc and (sc >= 2.0 ** -126)
    if not np.any(row):
        assert e == 0 and np.array_equal(q, np.where(np.signbit(row), 0x80, 0).astype(np.uint8))
    assert np.array_equal(q, _torch_bytes(row, e)), name
    assert np.array_equal(_bf16(xh), xh), f"{name}: x-hat is not a bf16 value"
    assert np.array_equal(xh, e4m3_decode(q) * sc)
    # one rounding: within half an E4M3 quantum of x (relative 2^-4 for normals)
    y = np.ldexp(row, -e)
    quantum = np.where(np.abs(y) < 2.0 ** -6, 2.0 ** -9, np.ldexp(1.0, np.floor(np.log2(np.maximum(np.abs(y), 2.0 ** -6))).astype(int) - 3))
    capped = (e == E_MAX) & (np.abs(row) >= 1.9375 * 2.0 ** 127)
    assert np.all((np.abs(np.ldexp(xh, -e) - y) <= quantum / 2) | capped)
    assert np.all(np.abs(xh[capped]) == 240 * 2.0 ** 120)
    if name.startswith("e_min"):
        assert e == E_MIN
    if name == "largest_bf16":
        assert e == E_MAX and capped.any() and np.isfinite(xh).all()
    if name.startswith("a_at_448"):
        k = int(name.split("^")[1])
        assert e == k and (q[3] & 0x7F) == 0x7E                       # 448 = 0x7e
    if name.startswith("a_above_448"):
        assert e == int(name.split("^")[1]) + 1
    if name.startswith("a_below_448"):
        assert e == int(name.split("^")[1])


def test_dequantise_round_trips_through_bf16():
    g = np.random.default_rng(3)
    q = g.integers(0, 256, (64, D)).astype(np.uint8)
    q[(q & 0x7F) == 0x7F] = 0
    sc = np.ldexp(1.0, g.integers(E_MIN, 121, 64)).astype(np.float32)
    xh = dequantise(q, sc)
    assert np.array_equal(_bf16(xh), xh)
    assert np.array_equal(torch.tensor(xh).bfloat16().double().numpy(), xh)
    want = torch.tensor(q).view(torch.float8_e4m3fn).double().numpy() * sc[:, None].astype(np.float64)
    assert np.array_equal(xh, want)


def test_check_kv_cache_dtype_refusals():
    from metamorph_b200.engine.decode import check_kv_cache_dtype
    check_kv_cache_dtype("bf16")
    check_kv_cache_dtype("fp8_e4m3")
    for bad in ("fp8", "FP8_E4M3", "e5m2", None, torch.float8_e4m3fn, torch.bfloat16, 8, ""):
        with pytest.raises(ValueError, match="kv_cache_dtype"):
            check_kv_cache_dtype(bad)


def test_fp8_entry_points_refuse_bad_arguments_without_gpu():
    from ctypes import c_float, c_int, c_void_p
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    n = c_void_p(0)
    a = c_void_p(256)
    with pytest.raises(MetaMorphB200Error, match="scale arrays missing"):
        call("mm_decode_attn_fp8", a, ll(768), a, a, n, n, a, a, a, a, ll(512), c_int(1), c_int(4), c_int(1),
             c_int(128), c_int(64), c_float(0.1), a, ll(1 << 20), c_int(1), n)
    with pytest.raises(MetaMorphB200Error, match="block_size"):
        call("mm_decode_attn_paged_fp8", a, ll(768), a, a, a, a, a, c_int(4), c_int(24), a, a, a, a, ll(512), c_int(1),
             c_int(4), c_int(1), c_int(128), c_float(0.1), a, ll(1 << 20), c_int(1), n)
    with pytest.raises(MetaMorphB200Error, match="head_dim 128"):
        call("mm_decode_attn_paged_fp8", a, ll(768), a, a, a, a, a, c_int(4), c_int(16), a, a, a, a, ll(512), c_int(1),
             c_int(4), c_int(1), c_int(64), c_float(0.1), a, ll(1 << 20), c_int(1), n)
    with pytest.raises(MetaMorphB200Error, match="scale arrays missing"):
        call("mm_kv_quant_prefill", a, ll(768), a, a, a, n, c_int(1), c_int(4), c_int(4), c_int(1), c_int(128),
             c_int(8), n)
    with pytest.raises(MetaMorphB200Error, match="T <= Tmax"):
        call("mm_kv_quant_prefill", a, ll(768), a, a, a, a, c_int(1), c_int(9), c_int(4), c_int(1), c_int(128),
             c_int(8), n)
    with pytest.raises(MetaMorphB200Error, match="8-byte aligned"):
        call("mm_kv_quant_prefill", a, ll(766), a, a, a, a, c_int(1), c_int(4), c_int(4), c_int(1), c_int(128),
             c_int(8), n)
    with pytest.raises(MetaMorphB200Error, match="block table missing"):
        call("mm_kv_quant_prefill_paged", a, ll(768), a, a, a, a, n, c_int(4), c_int(16), c_int(4), c_int(4), c_int(1),
             c_int(128), n)
    with pytest.raises(MetaMorphB200Error, match="T <= max_blocks"):
        call("mm_kv_quant_prefill_paged", a, ll(768), a, a, a, a, a, c_int(1), c_int(16), c_int(17), c_int(4),
             c_int(1), c_int(128), n)
    with pytest.raises(MetaMorphB200Error, match="block_size"):
        call("mm_kv_dequant_paged", a, a, a, a, a, c_int(4), c_int(512), c_int(1), c_int(1), c_int(128), a, a, n)
    with pytest.raises(MetaMorphB200Error, match="scale arrays missing"):
        call("mm_kv_dequant_paged", a, a, n, a, a, c_int(4), c_int(16), c_int(1), c_int(1), c_int(128), a, a, n)
    with pytest.raises(MetaMorphB200Error, match="n_blocks"):
        call("mm_kv_dequant_paged", a, a, a, a, a, c_int(4), c_int(16), c_int(5), c_int(1), c_int(128), a, a, n)
