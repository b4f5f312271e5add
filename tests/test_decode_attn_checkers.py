"""The decode-attention checker has teeth (CPU only).

`emulate` restates the schedule of decode_attn_kernel + decode_attn_combine_kernel (csrc/decode.cu:197-407) in fp32
torch: per split a max, exponentials, l and the unnormalised P V, then the combine. Each test runs it on the data of a
GPU case in tests/test_decode_attn_exact_gpu.py with one kernel bug emulated and requires that test's reference and
checker to reject the result; the clean emulation must pass the same checker. Nothing here builds or runs a kernel.
"""
import pytest
import torch

from tests.exact import assert_rounds_within, ulp_bf16
from tests.test_decode_attn_exact_gpu import D, decode_ref, rope_f32, split_inputs, split_ranges

CPU = torch.device("cpu")
BUGS = ["no_rescale", "rescale_l_not_o", "split_drops_last", "stale_new_row", "q_not_rounded", "new_not_attended",
        "kv_head_modulo", "empty_split_keeps_old_partial"]


def emulate(qkv, kc, vc, pos, cos, sin, Hq, Hkv, scale, S, bug=None, old_parts=None):
    """The kernel's arithmetic in fp32 (chain orders aside). Returns (out [B, Hq * 128] bf16, partials): partials[b] is
    the [Hq, S] m and l and the [Hq, S, 128] o the split CTAs would leave in the workspace."""
    B = qkv.shape[0]
    G = Hq // Hkv
    rows = qkv.reshape(B, Hq + 2 * Hkv, D)
    scale32 = torch.tensor(scale, dtype=torch.float32)
    out = torch.empty(B, Hq, D, dtype=torch.bfloat16)
    parts = []
    for b in range(B):
        p = int(pos[b])
        c, s = cos[p], sin[p]
        qf = rope_f32(rows[b, :Hq], c, s)
        if bug != "q_not_rounded":
            qf = qf.bfloat16().float()
        sq = qf * scale32
        kh = rope_f32(rows[b, Hq:Hq + Hkv], c, s).bfloat16()
        K = kc[b].float().clone()
        V = vc[b].float().clone()
        if bug != "stale_new_row":
            K[:, p] = kh.float()
        V[:, p] = rows[b, Hq + Hkv:].float()
        n = p if bug == "new_not_attended" else p + 1
        chunk, ranges = split_ranges(max(n, 1), S)
        m = torch.full((Hq, S), -torch.inf)
        l = torch.zeros(Hq, S)
        o = torch.zeros(Hq, S, D)
        for h in range(Hq):
            hk = h % Hkv if bug == "kv_head_modulo" else h // G
            for sp, (p0, p1) in enumerate(ranges):
                if bug == "split_drops_last" and n % chunk and p1 - p0 == chunk:
                    p1 -= 1
                if p1 <= p0:
                    if bug == "empty_split_keeps_old_partial":
                        om, ol, oo = old_parts[b]
                        m[h, sp], l[h, sp], o[h, sp] = om[h, sp], ol[h, sp], oo[h, sp]
                    continue
                sc = K[hk, p0:p1] @ sq[h]
                m[h, sp] = sc.max()
                e = torch.exp(sc - m[h, sp])
                l[h, sp] = e.sum()
                o[h, sp] = e @ V[hk, p0:p1]
        M = m.amax(1, keepdim=True)
        w = torch.where(m == -torch.inf, torch.zeros_like(m), torch.exp(m - M))
        if bug == "no_rescale":
            w = (m > -torch.inf).float()
        L = (l * w).sum(1)
        acc = (o * (torch.ones_like(w) if bug == "rescale_l_not_o" else w)[..., None]).sum(1)
        out[b] = (acc / L[:, None]).bfloat16()
        parts.append((m, l, o))
    return out.view(B, Hq * D), parts


def _case():
    """test_decode_attn_split_edges at G = 4, S = 7 (empty splits, chunks that do and do not divide n_ctx), with the
    full fp32 tables."""
    qkv, kc, vc, pos, cos, sin, Hq, Hkv, _ = split_inputs(4, 7, CPU, seed=407, tables="fp32")
    return qkv, kc, vc, pos, cos, sin, Hq, Hkv


def test_clean_emulation_passes_and_the_bound_is_tight_enough():
    qkv, kc, vc, pos, cos, sin, Hq, Hkv = _case()
    ref, err, _, stats = decode_ref(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, 7)
    assert any(st["n_empty"] > 0 for st in stats)
    out, _ = emulate(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, 7)
    assert_rounds_within(out.view(ref.shape), ref, err, "clean emulation")
    # the bound sits far below the output's spacing: for the median element under 1 / 16 of a bf16 ulp (it exceeds an
    # ulp only where the output cancels to far below P = sum_p p_p |v_p|)
    r = err / ulp_bf16(ref)
    assert float(r.median()) < 1 / 16 and float((r > 1 / 4).double().mean()) < 0.1


@pytest.mark.parametrize("bug", BUGS)
def test_decode_attn_check_rejects(bug):
    qkv, kc, vc, pos, cos, sin, Hq, Hkv = _case()
    S = 7
    ref, err, _, _ = decode_ref(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, S)
    old = None
    if bug == "empty_split_keeps_old_partial":
        # the previous call: other rows, every sequence at its last position, so no split of it was empty
        q2, k2, v2, _, _, _, _, _, _ = split_inputs(4, S, CPU, seed=999, tables="fp32")
        full = torch.full_like(pos, kc.shape[2] - 1)
        k2[:, :, -1] = 1.0
        v2[:, :, -1] = 1.0
        _, old = emulate(q2, k2.nan_to_num(0.5), v2.nan_to_num(0.5), full, cos, sin, Hq, Hkv, D ** -0.5, S)
        assert all(bool((m > -torch.inf).all()) for m, _, _ in old)
    good, _ = emulate(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, S)
    assert_rounds_within(good.view(ref.shape), ref, err, "clean")
    bad, _ = emulate(qkv, kc, vc, pos, cos, sin, Hq, Hkv, D ** -0.5, S, bug=bug, old_parts=old)
    with pytest.raises(AssertionError) as e:
        assert_rounds_within(bad.view(ref.shape), ref, err, bug)
    print(f"rejected: {e.value}")
