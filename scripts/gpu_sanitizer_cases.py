"""A handful of small launches of every hand-written tcgen05 / TMA kernel, for `compute-sanitizer` (SURVEY.md section 5:
memcheck / racecheck per kernel; VERDICT r1 item 7). Shapes are tiny so that the instrumented run finishes in minutes:
    compute-sanitizer --tool memcheck  python scripts/gpu_sanitizer_cases.py
    compute-sanitizer --tool racecheck python scripts/gpu_sanitizer_cases.py
Each case also checks its result against torch so that a "clean" report is about a kernel that computed the right thing."""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from metamorph_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)
only = set(sys.argv[1:])


def close(a, b, rel, what):
    err = (a.float() - b.float()).abs().max().item()
    scale = b.float().abs().max().item() + 1e-6
    assert err <= rel * scale, (what, err, scale)
    print(f"ok {what}: max err {err:.4g} of {scale:.4g}", flush=True)


def case(name):
    return not only or name in only


def attn_ref(q, k, v, scale, seqlens):
    # causal GQA attention in fp32; q [B,T,Hq,d], k/v [B,T,Hkv,d]; keys >= seqlens[b] are masked
    B, T, Hq, d = q.shape
    k = k.repeat_interleave(Hq // k.shape[2], dim=2)
    v = v.repeat_interleave(Hq // v.shape[2], dim=2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    mask = torch.tril(torch.ones(T, T, dtype=torch.bool, device=q.device))[None, None]
    mask = mask & (torch.arange(T, device=q.device)[None, None, None, :] < seqlens.view(B, 1, 1, 1))
    return torch.einsum("bhqk,bkhd->bqhd", s.masked_fill(~mask, float("-inf")).softmax(-1), v)


if case("gemm"):
    for force, (M, N, K) in ((128, (304, 200, 136)), (256, (264, 520, 200)), (512, (512, 512, 256)), (512, (304, 264, 72))):
        a = torch.randn(M, K, device=dev).bfloat16()
        b = torch.randn(N, K, device=dev).bfloat16()
        close(ops.gemm(a, b, force_bn=force), a.float() @ b.float().t(), 1e-2, f"gemm force_bn={force} {M}x{N}x{K}")
        bt = b.t().contiguous()
        close(ops.gemm(a, bt, b_mn=True, force_bn=force), a.float() @ b.float().t(), 1e-2, f"gemm b_mn force_bn={force}")
        at = a.t().contiguous()
        close(ops.gemm(at, bt, a_mn=True, b_mn=True, force_bn=force), a.float() @ b.float().t(), 1e-2, f"gemm mn/mn force_bn={force}")

if case("attn"):
    for B, T, Hq, Hkv in ((2, 200, 4, 2), (1, 300, 2, 1)):
        d = 128
        qkv = (torch.randn(B * T, (Hq + 2 * Hkv) * d, device=dev) * 0.5).bfloat16()
        q, k, v = qkv[:, :Hq * d], qkv[:, Hq * d:(Hq + Hkv) * d], qkv[:, (Hq + Hkv) * d:]
        sl = torch.tensor([T, T - 33][:B], device=dev, dtype=torch.int32)
        out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, d, True, 1 / math.sqrt(d), seqlens=sl)
        dout = torch.randn(B * T, Hq * d, device=dev).bfloat16()
        for b in range(B):
            dout.view(B, T, -1)[b, int(sl[b]):] = 0
        g = torch.zeros_like(qkv)
        ops.attn_bwd(q, k, v, out, dout, lse, g[:, :Hq * d], g[:, Hq * d:(Hq + Hkv) * d], g[:, (Hq + Hkv) * d:], B, T, Hq,
                     Hkv, d, 1 / math.sqrt(d), seqlens=sl)
        qf, kf, vf = (t.float().view(B, T, -1, d).clone().requires_grad_(True) for t in (q, k, v))
        ref = attn_ref(qf, kf, vf, 1 / math.sqrt(d), sl)
        ref.backward(dout.float().view(B, T, Hq, d))
        gref = torch.cat([t.grad.reshape(B * T, -1) for t in (qf, kf, vf)], 1)
        for b in range(B):
            L = int(sl[b])
            close(out.view(B, T, -1)[b, :L], ref.detach().reshape(B, T, -1)[b, :L], 2e-2, f"attn fwd T={T} b={b}")
            close(g.view(B, T, -1)[b, :L], gref.view(B, T, -1)[b, :L], 4e-2, f"attn bwd T={T} b={b}")
    segs = [(0, 150), (150, 40), (200, 130)]
    tab = ops.SegmentTables(segs, dev)
    qkv = (torch.randn(330, 4 * 128, device=dev) * 0.5).bfloat16()
    q, k, v = qkv[:, :256], qkv[:, 256:384], qkv[:, 384:]
    o = torch.zeros(330, 256, device=dev).bfloat16()
    _, lse = ops.attn_fwd_varlen(q, k, v, tab, 2, 1, 128, 0.088, out=o)
    g = torch.zeros_like(qkv)
    ops.attn_bwd_varlen(q, k, v, o, torch.randn_like(o), lse, g[:, :256], g[:, 256:384], g[:, 384:], tab, 2, 1, 128, 0.088)
    torch.cuda.synchronize()
    assert torch.isfinite(g).all()
    print("ok attn varlen", flush=True)

if case("decode"):
    K, N = 4096, 1184
    for m in (1, 8):
        x = torch.randn(m, K, device=dev).bfloat16()
        w = (torch.randn(N, K, device=dev) * 0.03).bfloat16()
        close(ops.skinny_gemm(x, w), x.float() @ w.float().t(), 1e-2, f"skinny gemm m={m}")
    B, Hq, Hkv, d, Tmax = 2, 4, 2, 128, 96
    pos = torch.tensor([0, 57], device=dev, dtype=torch.int32)
    kc = torch.randn(B, Hkv, Tmax, d, device=dev).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, d, device=dev).bfloat16()
    qkv = torch.randn(B, (Hq + 2 * Hkv) * d, device=dev).bfloat16()
    inv = 1.0 / (500000.0 ** (torch.arange(0, d, 2, device=dev).float() / d))
    ang = torch.arange(Tmax + 1, device=dev).float()[:, None] * inv[None]
    o = ops.decode_attn(qkv, kc, vc, pos, ang.cos().contiguous(), ang.sin().contiguous(), Hq, Hkv, d, 1 / math.sqrt(d), splits=2)
    torch.cuda.synchronize()
    assert torch.isfinite(o).all()
    print("ok decode attn", flush=True)

if case("misc"):
    x = torch.randn(37, 4096, device=dev).bfloat16()
    w = torch.randn(4096, device=dev).bfloat16()
    y = ops.rmsnorm(x, w, 1e-5)
    ref = x.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + 1e-5) * w.float()
    close(y, ref, 1e-2, "rmsnorm")
    lg = torch.randn(5, 1000, device=dev)
    lab = torch.tensor([1, 999, -100, 5, 7], device=dev, dtype=torch.int32)
    ls = torch.zeros(1, device=dev)
    dl = torch.empty(5, 1000, device=dev, dtype=torch.bfloat16)
    ops.ce_fwd_bwd(lg, lab, 1000, ls, dlogits=dl)
    refl = torch.nn.functional.cross_entropy(lg, lab.long(), ignore_index=-100, reduction="sum")
    close(ls, refl.reshape(1), 1e-4, "cross entropy")
torch.cuda.synchronize()
print("ALL CASES DONE", flush=True)
