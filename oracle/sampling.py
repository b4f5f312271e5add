"""numpy restatement of the decode sampler (metamorph_b200/csrc/sampling.cu, contract in DESIGN.md §1 row A9).

Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), the kept set of HF's
Temperature -> TopK -> TopP warpers decided by value in fp64 (every token tied at a boundary is kept), and the
Gumbel-max draw over it. Test infrastructure only: the product never imports it."""
from __future__ import annotations

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: [..., 4] uint32-valued, key: (k0, k1). Returns [..., 4] uint32 words."""
    c = np.asarray(ctr, dtype=np.uint64) & _MASK
    c0, c1, c2, c3 = c[..., 0], c[..., 1], c[..., 2], c[..., 3]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _MASK, p1 >> np.uint64(32), p1 & _MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def uniform_words(V: int, seed: int, counter: int) -> np.ndarray:
    """Word (i & 3) of Philox4x32-10(counter (i >> 2, c, 0, 0), key (s & 0xffffffff, s >> 32)) for i in [0, V)."""
    n = (V + 3) // 4
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(n, dtype=np.uint64)
    ctr[:, 1] = counter & 0xFFFFFFFF
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).reshape(-1)[:V]


def gumbel_noise(V: int, seed: int, counter: int) -> np.ndarray:
    """-log(-log u) in fp64 with u = (w + 0.5) * 2^-32."""
    u = (uniform_words(V, seed, counter).astype(np.float64) + 0.5) * 2.0 ** -32
    return -np.log(-np.log(u))


def scaled(logits, temperature: float) -> np.ndarray:
    """z = l / T in fp32 (IEEE divide), NaN -> -inf, returned as fp64."""
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        z = (np.asarray(logits, dtype=np.float32) / np.float32(temperature)).astype(np.float64)
    z[np.isnan(z)] = -np.inf
    return z


def kept_set(z: np.ndarray, top_k: int, top_p: float):
    """fp64 kept set of one row of scaled logits. Returns (mask, top-p margin): the margin is
    min_i |mass(z_j > z_i) - p * M| / M over the top-k set (inf when top-p is off), the distance of the row from a
    top-p decision flip."""
    V = z.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        thr = np.sort(z)[::-1][top_k - 1]
        keep = z >= thr
    margin = np.inf
    if top_p <= 0:
        keep &= z == z.max()
    elif top_p < 1:
        zmax = z.max()
        mass = np.where(keep, np.exp(z - zmax), 0.0)
        M = mass.sum()
        vals, inv = np.unique(z, return_inverse=True)          # ascending unique values
        per_val = np.bincount(inv, weights=mass, minlength=vals.size)
        above = np.concatenate([np.cumsum(per_val[::-1])[::-1][1:], [0.0]])   # mass strictly above each value
        G = above[inv]
        margin = float(np.min(np.abs(G[keep] - top_p * M)) / M)
        keep &= G < top_p * M
    return keep, margin


def draw(logits, temperature: float, top_k: int, top_p: float, seed: int, counter: int):
    """The sampled token of one row and the relative gap between its perturbed value and the runner-up
    (inf when only one token is kept). T <= 0 is greedy: the lowest index of the maximum, NaN never chosen. A row with
    no logit above -inf gives 0; a row whose max l / T is not finite in fp32 gives the argmax as well."""
    logits = np.asarray(logits, dtype=np.float32)
    if not temperature > 0:
        return int(np.argmax(np.where(np.isnan(logits), -np.inf, logits))), np.inf, np.inf
    clean = np.where(np.isnan(logits), np.float32(-np.inf), logits)
    if not (clean > -np.inf).any():
        return 0, np.inf, np.inf
    with np.errstate(over="ignore", divide="ignore"):
        zmax = clean.max() / np.float32(temperature)
    if np.isinf(zmax):          # a +inf logit, or |max l| / T beyond fp32: the limit T -> 0, the argmax, lowest index
        return int(np.argmax(clean)), np.inf, np.inf
    z = scaled(logits, temperature)
    keep, margin = kept_set(z, top_k, top_p)
    score = np.where(keep, z + gumbel_noise(z.shape[0], seed, counter), -np.inf)
    tok = int(np.argmax(score))
    rest = np.delete(score, tok)
    second = rest.max() if rest.size else -np.inf
    gap = (score[tok] - second) / max(1.0, abs(score[tok])) if np.isfinite(second) else np.inf
    return tok, gap, margin


def warped_probs(logits, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    """The distribution the draw follows: softmax of z over the kept set, fp64."""
    z = scaled(logits, temperature)
    keep, _ = kept_set(z, top_k, top_p)
    w = np.where(keep, np.exp(z - z[keep].max()), 0.0)
    return w / w.sum()
