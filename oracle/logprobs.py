"""fp64 restatement of the decode log-probability contract (DESIGN.md, "Log-probability contract"; kernel:
csrc/sampling.cu decode_logprobs_kernel), and a helper that scores a trajectory with oracle/restatement.py's fp32 model.

For one fp32 logits row l (NaN read as -inf), m = max l, S = sum_j exp(l_j - m):
  logprob(i) = l_i - m - ln S (a +inf max: -ln c on its c +inf entries, -inf elsewhere; no logit above -inf: NaN);
  top-n = (l, index) by value descending, lowest index first among ties; entries past V get id -1 and -inf;
  a token outside [0, V) reports NaN; only steps with append_kind == 0 report, at index n_ids - 1 when < max_ids.
The kernel's fp32 value lies within bound(x) = 0.5 ulp_fp32(x) + EPS_ABS + EPS_REL |x| of the exact value x."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np

TOP_MAX = 20
EPS_ABS = 2.0 ** -21      # expf's 2 ulp per term (2^-22 relative in S, so in ln S) plus fp64 rounding, with headroom
EPS_REL = 2.0 ** -51      # the two fp64 roundings of (l - m) - ln S


def clean(row) -> np.ndarray:
    r = np.asarray(row, dtype=np.float32).astype(np.float64)
    return np.where(np.isnan(r), -np.inf, r)


def row_stats(row) -> Tuple[int, float, float]:
    """(mode, m, lnS): mode 0 a distribution (lnS = ln S), 1 a +inf max (lnS = ln c), 2 no logit above -inf."""
    r = clean(row)
    m = r.max() if r.size else -np.inf
    if m == -np.inf:
        return 2, m, float("nan")
    if m == np.inf:
        return 1, m, math.log(int((r == np.inf).sum()))
    return 0, m, math.log(float(np.exp(r - m).sum()))


def logprob64(v: float, stats) -> float:
    mode, m, lnS = stats
    if mode == 2:
        return float("nan")
    if mode == 1:
        return -lnS if v == np.inf else -np.inf
    return (float(v) - m) - lnS


def order(row) -> np.ndarray:
    """Indices in top-n order: value descending, lowest index first among ties (NaN = -inf)."""
    r = clean(row)
    return np.lexsort((np.arange(r.size), -r))


def report(row, token: int, n: int):
    """-> (logprob of token (fp64), top ids [n] int, top logprobs [n] fp64) for one step."""
    r = clean(row)
    V = r.size
    st = row_stats(row)
    lp = logprob64(r[token], st) if 0 <= token < V else float("nan")
    idx = order(row)[:n]
    ids = np.full(n, -1, dtype=np.int64)
    lps = np.full(n, -np.inf)
    ids[:idx.size] = idx
    lps[:idx.size] = [logprob64(r[i], st) for i in idx]
    return lp, ids, lps


def ulp32(x: float) -> float:
    x = abs(float(x))
    if not math.isfinite(x):
        return 0.0
    f = np.float32(min(x, 3.4028234663852886e38))
    return float(np.spacing(f))


def bound(x: float) -> float:
    return 0.5 * ulp32(x) + EPS_ABS + EPS_REL * abs(x)


def excess(got: float, exact: float) -> float:
    """|got - exact| beyond 0.5 ulp_fp32, as a fraction of the contract's eps (<= 1 passes; inf = a wrong special value).
    Non-finite exact values (after rounding to fp32) must be matched bit for bit."""
    got = float(got)
    e32 = float(np.float32(exact)) if not math.isnan(exact) else float("nan")
    if math.isnan(e32) or math.isinf(e32) or math.isnan(got) or math.isinf(got):
        same = (math.isnan(got) and math.isnan(e32)) or got == e32
        return 0.0 if same else float("inf")
    err = abs(got - exact) - 0.5 * max(ulp32(exact), ulp32(got))
    return max(0.0, err) / (EPS_ABS + EPS_REL * abs(exact))


def check_report(lp, ids, lps, row, token: int, n: int, what: str = "") -> float:
    """Assert one reported step against the restatement: ids exact, every value within the bound. Returns the largest
    fraction of eps reached."""
    want_lp, want_ids, want_lps = report(row, token, n)
    ids = np.asarray(ids).reshape(-1)[:n]
    assert np.array_equal(ids, want_ids), f"{what}: top ids {ids.tolist()} != {want_ids.tolist()}"
    worst = excess(lp, want_lp)
    assert worst <= 1.0, f"{what}: logprob {lp!r} vs exact {want_lp!r}"
    for k in range(n):
        e = excess(np.asarray(lps).reshape(-1)[k], want_lps[k])
        assert e <= 1.0, f"{what}: top entry {k} {lps[k]!r} vs exact {want_lps[k]!r}"
        worst = max(worst, e)
    return worst


def store(trace: Sequence[Tuple[np.ndarray, int, int, int]], max_ids: int, n: int):
    """The store rule over one sequence's steps [(logits row, chosen token, append_kind, n_ids after the step)]:
    -> (lp [max_ids], top ids [max_ids, n], top lps [max_ids, n]) as the kernel leaves them, NaN / -2 where untouched."""
    lp = np.full(max_ids, np.nan)
    ids = np.full((max_ids, n), -2, dtype=np.int64)
    lps = np.full((max_ids, n), np.nan)
    for row, tok, kind, n_ids in trace:
        slot = n_ids - 1
        if kind != 0 or slot < 0 or slot >= max_ids:
            continue
        lp[slot], ids[slot], lps[slot] = report(row, tok, n)
    return lp, ids, lps


def check_stored(lp, ids, lps, trace, max_ids: int, n: int, poison_id: int, what: str = "") -> float:
    """Assert one sequence's output row (lp [max_ids], ids / lps [max_ids, >= n]) against the store rule over its trace:
    a slot the rule writes holds that step's report, every other slot keeps its poison (NaN logprob, poison_id ids).
    Returns the largest fraction of eps reached."""
    rows = {}
    for row, tok, kind, n_ids in trace:
        if kind == 0 and 0 <= n_ids - 1 < max_ids:
            rows[n_ids - 1] = (row, tok)
    worst = 0.0
    for s in range(max_ids):
        if s in rows:
            worst = max(worst, check_report(lp[s], ids[s][:n], lps[s][:n], rows[s][0], rows[s][1], n, f"{what} slot {s}"))
        else:
            assert math.isnan(float(lp[s])) and all(int(i) == poison_id for i in ids[s][:n]), \
                f"{what}: slot {s} was written but no step reports there"
    return worst


def close_calls(row, n: int, tol: float) -> List[int]:
    """Positions k < n of the top-n list whose value is within tol of the next one: an oracle fed logits that differ
    from the product's by up to tol cannot call their order."""
    r = clean(row)
    idx = order(row)[:n + 1]
    return [k for k in range(min(n, idx.size - 1)) if r[idx[k]] - r[idx[k + 1]] <= tol]


def trajectory_logprobs(p, cfg, inputs_embeds, max_new_tokens: int, forced: Optional[Sequence[int]] = None,
                        start_id=128256, end_id=128257, eos=(128001, 128009)):
    """Run oracle/restatement.py's fp32 model along the decode loop of metamorph_llama.py:502-597 (no cache), the
    token of step s being forced[s] when that entry exists and is >= 0, else the argmax. Returns one dict per emitted
    id: token, the fp32 log-softmax of the step's logits at it, the logits row (fp32 numpy) and whether the token is
    the argmax."""
    import torch
    import torch.nn.functional as F
    from . import restatement as R

    x = inputs_embeds.float()
    out = []
    in_image, n_img_tok, n_out = False, 0, 0
    ntok = cfg["image_tokens"]
    emb_w = p["model.embed_tokens.weight"].float()
    while True:
        T = x.shape[1]
        hidden = R.llama_forward(p, x, torch.arange(T)[None], torch.ones(1, T, dtype=torch.bool), cfg["layers"],
                                 cfg["heads"], cfg["kv_heads"], cfg["rms_eps"], cfg["rope_theta"])
        if in_image:
            pred_z = F.normalize(R.mlp_gelu(p, "vision_head.", hidden[:, -1]), p=2, dim=-1)
            hidden = hidden.clone()
            hidden[:, -1] = R.mlp_gelu(p, "model.mm_projector.", pred_z)
        logits = F.linear(hidden[:, -1], p["lm_head.weight"].float())[0]
        am = int(logits.argmax())
        f = forced[n_out] if forced is not None and n_out < len(forced) else -1
        tok = int(f) if f >= 0 else am
        emitted = True
        if not in_image and tok == start_id:
            in_image = True
            x = torch.cat([x, emb_w[tok][None, None]], 1)
        elif in_image and n_img_tok < ntok:
            n_img_tok += 1
            emitted = False
            x = torch.cat([x, hidden[:, -1:, :]], 1)
            if n_img_tok == ntok:
                in_image = False
        elif tok == end_id:
            in_image, n_img_tok = False, 0
            x = torch.cat([x, emb_w[tok][None, None]], 1)
        else:
            x = torch.cat([x, emb_w[tok][None, None]], 1)
        if emitted:
            ls = torch.log_softmax(logits, -1)
            out.append(dict(token=tok, logprob=float(ls[tok]), logits=logits.numpy().astype(np.float32),
                            greedy=tok == am))
        n_out += 1
        if tok in eos or n_out > max_new_tokens:
            break
    return out
