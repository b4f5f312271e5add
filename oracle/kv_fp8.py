"""fp64 restatement of the FP8 (E4M3) KV-cache row rule (DESIGN.md §1, include/metamorph_b200.h).

One (position, kv head) row x[0..128) of bf16 values is stored as E4M3 bytes q_i = RNE_e4m3(x_i 2^-e) and one fp32
scale 2^e, with a = max |x_i| and e the least integer such that a <= 448 2^e, clamped below at E_MIN = -124. A zero row
stores zeros (signed as x) with e = 0; a row holding any Inf or NaN stores 0x7f (the E4M3 NaN) in every entry with
e = 0. One exception to round-to-nearest: at e = 120, the largest e a bf16 row reaches, an entry that rounds to 256
(|x| >= 1.9375 2^127) would dequantise to 2^128, past the bf16 range; it stores 240 (0x77), the largest magnitude whose
x-hat is finite. The dequantised row x-hat_i = float(q_i) 2^e is exact and a bf16 value. Everything here is exact in
fp64."""
from __future__ import annotations

import numpy as np

E_MIN = -124
E_MAX = 120            # e of a row whose max is the largest bf16 value, (2 - 2^-7) 2^127
E4M3_MAX = 448.0
NAN_BYTE = 0x7F


def row_exponent(x) -> int:
    """e of one finite row (fp64 array of its values): the least integer with max |x| <= 448 2^e, at least E_MIN;
    0 for a zero row."""
    a = float(np.max(np.abs(np.asarray(x, dtype=np.float64))))
    if a == 0.0:
        return 0
    f, E = np.frexp(a)                   # a = f 2^E, f in [0.5, 1); 448 = 0.875 2^9
    return max(int(E) - 9 if f <= 0.875 else int(E) - 8, E_MIN)


def e4m3_encode(y):
    """Bytes of RNE_e4m3(y) for finite fp64 y with |y| <= 448 (round half to even; -0 keeps its sign)."""
    y = np.asarray(y, dtype=np.float64)
    assert np.all(np.isfinite(y)) and np.all(np.abs(y) <= E4M3_MAX)
    sign = np.signbit(y).astype(np.uint8) << 7
    m = np.abs(y)
    _, E = np.frexp(np.where(m > 0, m, 1.0))
    E = E.astype(np.int64) - 1                                 # floor(log2 m) for m > 0
    quantum = np.where(m < 2.0 ** -6, 2.0 ** -9, np.ldexp(1.0, np.maximum(E, -6) - 3))
    q = np.rint(m / quantum) * quantum                         # exact: m / quantum is a division by a power of two
    _, Eq = np.frexp(np.where(q > 0, q, 1.0))
    Eq = Eq.astype(np.int64) - 1
    normal = q >= 2.0 ** -6
    exp_field = np.where(normal, Eq + 7, 0)
    mant = np.where(normal, q / np.ldexp(1.0, Eq - 3) - 8, q / 2.0 ** -9)
    return (sign | (exp_field.astype(np.uint8) << 3) | mant.astype(np.uint8)).astype(np.uint8)


def e4m3_decode(b):
    """fp64 values of E4M3 bytes (0x7f / 0xff are NaN)."""
    b = np.asarray(b, dtype=np.uint8).astype(np.int64)
    s = np.where(b & 0x80, -1.0, 1.0)
    ef, mf = (b >> 3) & 0xF, b & 0x7
    v = np.where(ef == 0, mf * 2.0 ** -9, (8 + mf) * np.ldexp(1.0, ef - 7 - 3))
    return np.where((b & 0x7F) == 0x7F, np.nan, s * v)


def quantise_rows(x):
    """x [..., 128] (bf16 values, any float dtype) -> (bytes uint8 [..., 128], scale float32 [...], x-hat fp64
    [..., 128])."""
    x = np.asarray(x, dtype=np.float64)
    rows = x.reshape(-1, x.shape[-1])
    q = np.empty(rows.shape, dtype=np.uint8)
    sc = np.empty(rows.shape[0], dtype=np.float32)
    for r, row in enumerate(rows):
        if not np.all(np.isfinite(row)):
            q[r], sc[r] = NAN_BYTE, 1.0
            continue
        e = row_exponent(row)
        q[r] = e4m3_encode(np.ldexp(row, -e))
        if e == E_MAX:
            q[r] = np.where((q[r] & 0x7F) == 0x78, (q[r] & 0x80) | 0x77, q[r])
        sc[r] = np.float32(np.ldexp(1.0, e))
    q = q.reshape(x.shape)
    sc = sc.reshape(x.shape[:-1])
    return q, sc, dequantise(q, sc)


def dequantise(q, scale):
    """x-hat = float(q) 2^e, fp64 [..., 128]."""
    return e4m3_decode(q) * np.asarray(scale, dtype=np.float64)[..., None]
