"""Per-kernel parity tests (H100 only): each CUDA kernel, called through the C-ABI, against a plain
torch fp32 restatement of the same op. Tolerances are bf16-level and written next to each check."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _close(a, b, rel, what, rms_rel=None):
    """max |a-b| <= rel * max|b|, AND (VERDICT r1 weak 5: a bound relative to the largest entry lets a systematic error in
    the small entries through) rms(a-b) <= rms_rel * rms(b); rms_rel defaults to rel / 2."""
    a, b = a.float(), b.float()
    err = (a - b).abs().max().item()
    scale = b.abs().max().item() + 1e-6
    floor = 1e-6                       # a reference that is exactly zero (e.g. dQ of a one-token sequence) vs fp32 dust
    assert err <= rel * scale + floor, f"{what}: max_err={err:.5f} scale={scale:.4f} rel={err/scale:.5f} > {rel}"
    rms_rel = rel / 2 if rms_rel is None else rms_rel
    rms_e = (a - b).pow(2).mean().sqrt().item()
    rms_b = b.pow(2).mean().sqrt().item()
    assert rms_e <= rms_rel * rms_b + floor, f"{what}: rms_err={rms_e:.6f} rms_ref={rms_b:.5f} rel={rms_e/(rms_b + 1e-12):.5f} > {rms_rel}"


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("shape", [(128, 256, 64), (304, 520, 200), (1024, 1152, 4096), (729 * 2, 4304, 1152)])
def test_gemm_layouts(cuda_device, a_mn, b_mn, shape):
    from metamorph_b200 import ops
    M, N, K = shape
    if (a_mn or b_mn) and (M % 8 or N % 8):
        pytest.skip("MN-major operands need 16-byte aligned pitches")
    torch.manual_seed(0)
    a = torch.randn((K, M) if a_mn else (M, K), device=cuda_device).bfloat16()
    b = torch.randn((K, N) if b_mn else (N, K), device=cuda_device).bfloat16()
    ref = (a.float().t() if a_mn else a.float()) @ (b.float() if b_mn else b.float().t())
    for bn in (128, 256):   # both tile widths of the wgmma kernel
        out = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, force_bn=bn)
        _close(out, ref, 1e-2, f"gemm bn={bn}")


@pytest.mark.parametrize("force_bn", [0, 256])      # 0 picks the 128-wide tile at this size; 256 forces the wide one
def test_gemm_epilogues(cuda_device, force_bn):
    from metamorph_b200 import ops
    torch.manual_seed(1)
    M, N, K = 520, 1160, 320
    a = torch.randn(M, K, device=cuda_device).bfloat16()
    w = (torch.randn(N, K, device=cuda_device) * 0.05).bfloat16()
    bias = torch.randn(N, device=cuda_device).bfloat16()
    res = torch.randn(M, N, device=cuda_device).bfloat16()
    base = a.float() @ w.float().t()
    kw = dict(force_bn=force_bn)
    _close(ops.gemm(a, w, **kw), base, 1e-2, "store")
    _close(ops.gemm(a, w, alpha=0.5, **kw), 0.5 * base, 1e-2, "alpha")
    _close(ops.gemm(a, w, bias=bias, epilogue=ops.EPI_BIAS, **kw), base + bias.float(), 1e-2, "bias")
    _close(ops.gemm(a, w, bias=bias, epilogue=ops.EPI_BIAS_GELU_ERF, **kw), F.gelu(base + bias.float()), 1e-2, "gelu_erf")
    _close(ops.gemm(a, w, bias=bias, epilogue=ops.EPI_BIAS_GELU_TANH, **kw),
           F.gelu(base + bias.float(), approximate="tanh"), 1e-2, "gelu_tanh")
    _close(ops.gemm(a, w, resid=res, epilogue=ops.EPI_RESID, **kw), base + res.float(), 1e-2, "resid")
    _close(ops.gemm(a, w, bias=bias, resid=res, epilogue=ops.EPI_BIAS_RESID, **kw), base + bias.float() + res.float(), 1e-2, "bias_resid")
    # in-place residual (C aliases R)
    r2 = res.clone()
    ops.gemm(a, w, resid=r2, out=r2, epilogue=ops.EPI_RESID, **kw)
    _close(r2, base + res.float(), 1e-2, "resid in place")
    # a column slice of a wider buffer as the output (pitch != N): the store must respect ldc and leave the rest alone
    wide = torch.full((M, N + 72), 5.0, device=cuda_device, dtype=torch.bfloat16)
    ops.gemm(a, w, out=wide[:, 8:8 + N], **kw)
    _close(wide[:, 8:8 + N], base, 1e-2, "strided out")
    assert torch.all(wide[:, :8].float() == 5.0) and torch.all(wide[:, 8 + N:].float() == 5.0)
    # fp32 output + accumulate
    c32 = torch.ones(M, N, device=cuda_device, dtype=torch.float32)
    ops.gemm(a, w, out=c32, out_dtype=torch.float32, accumulate=True, **kw)
    _close(c32, base + 1.0, 1e-3, "f32 accumulate")
    c16 = res.clone()
    ops.gemm(a, w, out=c16, accumulate=True, **kw)
    _close(c16, base + res.float(), 1e-2, "bf16 accumulate")
    # swiglu: columns interleaved in chunks of [16 gate | 16 up]
    N2 = 1152
    wg = (torch.randn(N2 // 2, K, device=cuda_device) * 0.05).bfloat16()
    wu = (torch.randn(N2 // 2, K, device=cuda_device) * 0.05).bfloat16()
    from metamorph_b200.engine.packing import interleave_gate_up
    wgu = interleave_gate_up(wg, wu)
    aux = torch.empty(M, N2, device=cuda_device, dtype=torch.bfloat16)
    act = ops.gemm(a, wgu, aux=aux, epilogue=ops.EPI_SWIGLU)
    g, u = a.float() @ wg.float().t(), a.float() @ wu.float().t()
    _close(act, F.silu(g) * u, 1e-2, "swiglu")
    _close(aux, (a.float() @ wgu.float().t()), 1e-2, "swiglu aux")
    # SwiGLU backward fused into the down_proj dgrad epilogue: acc = d(act), aux = gate|up -> d(gate|up), C = act
    from metamorph_b200.engine.packing import deinterleave_gate_up
    I = 512
    dy = torch.randn(M, 320, device=cuda_device).bfloat16()
    wd = (torch.randn(320, I, device=cuda_device) * 0.05).bfloat16()            # down_proj weight [H, I]
    g_ = torch.randn(M, I, device=cuda_device).bfloat16()
    u_ = torch.randn(M, I, device=cuda_device).bfloat16()
    gu = interleave_gate_up(g_.t().contiguous(), u_.t().contiguous()).t().contiguous()   # [M, 2I]
    gf, uf = g_.float().requires_grad_(True), u_.float().requires_grad_(True)
    dact_ref = dy.float() @ wd.float()
    (F.silu(gf) * uf).backward(dact_ref)
    act2 = torch.empty(M, I, device=cuda_device, dtype=torch.bfloat16)
    ops.gemm(dy, wd, b_mn=True, out=act2, aux=gu, epilogue=ops.EPI_SWIGLU_BWD)
    dg, du = deinterleave_gate_up(gu.t().contiguous())
    _close(act2, F.silu(g_.float()) * u_.float(), 1e-2, "fused swiglu_bwd act")
    _close(dg.t(), gf.grad, 2e-2, "fused swiglu_bwd dgate")
    _close(du.t(), uf.grad, 2e-2, "fused swiglu_bwd dup")


def test_rmsnorm_fwd_bwd(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(2)
    M, H, eps = 300, 4096, 1e-5
    x = torch.randn(M, H, device=cuda_device).bfloat16()
    w = (1 + 0.1 * torch.randn(H, device=cuda_device)).bfloat16()
    dy = torch.randn(M, H, device=cuda_device).bfloat16()
    dres = torch.randn(M, H, device=cuda_device).bfloat16()
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    ref = wf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))
    ref.backward(dy.float())
    _close(ops.rmsnorm(x, w, eps), ref, 1e-2, "rmsnorm fwd")
    dw = torch.zeros(H, device=cuda_device, dtype=torch.float32)
    dx = ops.rmsnorm_bwd(dy, x, w, eps, dres_in=dres, dw_accum=dw)
    _close(dx, xf.grad + dres.float(), 1e-2, "rmsnorm dx")
    _close(dw, wf.grad, 1e-2, "rmsnorm dw")


def test_layernorm(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(3)
    x = torch.randn(729, 1152, device=cuda_device).bfloat16()
    w = torch.randn(1152, device=cuda_device).bfloat16()
    b = torch.randn(1152, device=cuda_device).bfloat16()
    ref = F.layer_norm(x.float(), (1152,), w.float(), b.float(), 1e-6)
    _close(ops.layernorm(x, w, b, 1e-6), ref, 1e-2, "layernorm")


def test_rope_roundtrip(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(4)
    M, Hq, Hkv, d = 200, 4, 2, 128
    qkv = torch.randn(M, (Hq + 2 * Hkv) * d, device=cuda_device).bfloat16()
    pos = torch.randint(0, 500, (M,), device=cuda_device, dtype=torch.int32)
    inv = 1.0 / (500000.0 ** (torch.arange(0, d, 2, device=cuda_device).float() / d))
    ang = torch.arange(512, device=cuda_device).float()[:, None] * inv[None]
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    x = qkv.float().view(M, Hq + 2 * Hkv, d)[:, :Hq + Hkv]
    c, s = cos[pos.long()][:, None], sin[pos.long()][:, None]
    x1, x2 = x[..., :d // 2], x[..., d // 2:]
    ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)
    orig = qkv.clone()
    ops.rope_(qkv, pos, cos, sin, Hq + Hkv, d)
    _close(qkv.view(M, -1, d)[:, :Hq + Hkv], ref, 1e-2, "rope fwd")
    assert torch.equal(qkv.view(M, -1, d)[:, Hq + Hkv:], orig.view(M, -1, d)[:, Hq + Hkv:]), "v must be untouched"
    ops.rope_(qkv, pos, cos, sin, Hq + Hkv, d, backward=True)
    _close(qkv, orig, 2e-2, "rope bwd inverts fwd")


def test_swiglu_bwd_and_gelu(cuda_device):
    from metamorph_b200 import ops
    from metamorph_b200.engine.packing import interleave_gate_up, deinterleave_gate_up
    torch.manual_seed(5)
    M, I = 100, 512
    g = torch.randn(M, I, device=cuda_device).bfloat16()
    u = torch.randn(M, I, device=cuda_device).bfloat16()
    gu = interleave_gate_up(g.t().contiguous(), u.t().contiguous()).t().contiguous()  # [M, 2I]
    dact = torch.randn(M, I, device=cuda_device).bfloat16()
    gf, uf = g.float().requires_grad_(True), u.float().requires_grad_(True)
    (F.silu(gf) * uf).backward(dact.float())
    act = torch.empty(M, I, device=cuda_device, dtype=torch.bfloat16)
    dgu = ops.swiglu_bwd(gu, dact, act=act)
    dg, du = deinterleave_gate_up(dgu.t().contiguous())
    _close(dg.t(), gf.grad, 1e-2, "swiglu dgate")
    _close(du.t(), uf.grad, 1e-2, "swiglu dup")
    _close(act, F.silu(g.float()) * u.float(), 1e-2, "swiglu act recompute")
    z = torch.randn(64, 256, device=cuda_device).bfloat16()
    da = torch.randn(64, 256, device=cuda_device).bfloat16()
    zf = z.float().requires_grad_(True)
    F.gelu(zf).backward(da.float())
    _close(ops.gelu(z), F.gelu(z.float()), 1e-2, "gelu")
    _close(ops.gelu_bwd(z, da), zf.grad, 1e-2, "gelu bwd")
    cs = torch.zeros(256, device=cuda_device)
    ops.colsum_accum(z, cs)
    _close(cs, z.float().sum(0), 1e-3, "colsum")


def test_interleave_gather_scatter_bitexact(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(6)
    V, H, NI = 1000, 4096, 130
    emb = torch.randn(V, H, device=cuda_device).bfloat16()
    img = torch.randn(NI, H, device=cuda_device).bfloat16()
    R = 777
    rm = torch.randint(0, V, (R,), device=cuda_device, dtype=torch.int32)
    img_rows = torch.randperm(R, device=cuda_device)[:NI]
    rm[img_rows] = -(torch.arange(NI, device=cuda_device, dtype=torch.int32)) - 2
    pad_rows = torch.tensor([5, 99, 776], device=cuda_device)
    rm[pad_rows] = -1
    out = ops.interleave_gather(emb, img, rm)
    ref = torch.zeros(R, H, device=cuda_device, dtype=torch.bfloat16)
    tok = rm >= 0
    ref[tok] = emb[rm[tok].long()]
    im = rm <= -2
    ref[im] = img[(-(rm[im]) - 2).long()]
    assert torch.equal(out, ref), "gather-interleave must be bit-exact"
    dout = torch.randn(R, H, device=cuda_device).bfloat16()
    demb = torch.zeros(V, H, device=cuda_device, dtype=torch.bfloat16)
    dimg = torch.zeros(NI, H, device=cuda_device, dtype=torch.bfloat16)
    ops.interleave_scatter(dout, rm, demb, dimg)
    assert torch.equal(dimg[(-(rm[im]) - 2).long()], dout[im])
    ref_e = torch.zeros(V, H, device=cuda_device, dtype=torch.float32)
    ref_e.index_add_(0, rm[tok].long(), dout[tok].float())
    _close(demb, ref_e, 2e-2, "embedding grad scatter")
    idx = torch.randperm(R, device=cuda_device)[:50].int()
    assert torch.equal(ops.gather_rows(dout, idx), dout[idx.long()])


def test_bilinear_l2norm_matches_torch(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(7)
    x = torch.randn(3, 729, 1152, device=cuda_device).bfloat16()
    y = ops.bilinear_l2norm(x, 8)
    xi = x.view(3, 27, 27, 1152).permute(0, 3, 1, 2).contiguous()
    r = F.interpolate(xi.float(), size=(8, 8), mode="bilinear", align_corners=False).to(x.dtype)
    r = r.permute(0, 2, 3, 1).contiguous().flatten(1, 2)
    r = F.normalize(r, p=2, dim=-1)
    _close(y, r, 1e-2, "bilinear+l2norm")
    y16 = ops.bilinear_l2norm(x, 16, normalize=False)
    r16 = F.interpolate(xi.float(), size=(16, 16), mode="bilinear", align_corners=False).to(x.dtype)
    assert torch.equal(y16, r16.permute(0, 2, 3, 1).contiguous().flatten(1, 2)), "bilinear taps must match ATen"


def test_ce_and_cosine(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(8)
    R, V = 37, 128258
    ld = 128264
    buf = torch.zeros(R, ld, device=cuda_device, dtype=torch.float32)
    buf[:, :V] = torch.randn(R, V, device=cuda_device) * 3
    labels = torch.randint(0, V, (R,), device=cuda_device, dtype=torch.int32)
    labels[::5] = -100
    lf = buf[:, :V].clone().requires_grad_(True)
    n_valid = int((labels != -100).sum())
    ref = F.cross_entropy(lf, labels.long(), ignore_index=-100, reduction="sum") / n_valid
    ref.backward()
    loss = torch.zeros(1, device=cuda_device)
    dl = torch.empty(R, ld, device=cuda_device, dtype=torch.bfloat16)
    ops.ce_fwd_bwd(buf, labels, V, loss, dlogits=dl, grad_scale=1.0 / n_valid)
    assert abs(loss.item() / n_valid - ref.item()) < 1e-4 * abs(ref.item()) + 1e-5
    _close(dl[:, :V], lf.grad, 1e-2, "dlogits")
    assert (dl[:, V:] == 0).all()
    assert ops.argmax_rows(buf, V).long().equal(buf[:, :V].argmax(-1))
    # cosine
    Rr, C = 50, 1152
    pred = torch.randn(Rr, C, device=cuda_device).bfloat16()
    tgt = F.normalize(torch.randn(Rr, C, device=cuda_device), dim=-1).bfloat16()
    pf = pred.float().requires_grad_(True)
    lref = -F.cosine_similarity(tgt.float(), F.normalize(pf, dim=-1), dim=-1).mean()
    lref.backward()
    ls = torch.zeros(1, device=cuda_device)
    dp = torch.empty_like(pred)
    pn = torch.empty_like(pred)
    ops.cosine_loss(pred, tgt, loss_sum=ls, pred_norm=pn, dpred=dp)
    assert abs(ls.item() - lref.item()) < 5e-3
    _close(dp, pf.grad, 2e-2, "cosine dpred")
    _close(pn, F.normalize(pred.float(), dim=-1), 1e-2, "pred_norm")


def test_adamw_matches_torch(cuda_device):
    from metamorph_b200 import ops
    torch.manual_seed(9)
    n = 4096 * 3
    p = torch.randn(n, device=cuda_device)
    ref_p = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref_p], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1)
    p32, m, v = p.clone(), torch.zeros(n, device=cuda_device), torch.zeros(n, device=cuda_device)
    p16 = p.bfloat16()
    for step in range(1, 4):
        g = torch.randn(n, device=cuda_device).bfloat16()
        ref_p.grad = g.float()
        opt.step()
        ops.adamw_step_(p16, p32, m, v, g, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.1, step=step)
    _close(p32, ref_p.detach(), 1e-5, "adamw master")
    assert torch.equal(p16, p32.bfloat16())


def _attn_ref(q, k, v, causal, scale, seqlens=None):
    # q [B,T,Hq,d], k/v [B,T,Hkv,d] fp32
    B, T, Hq, d = q.shape
    Hkv = k.shape[2]
    k = k.repeat_interleave(Hq // Hkv, dim=2)
    v = v.repeat_interleave(Hq // Hkv, dim=2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    mask = torch.ones(B, 1, T, T, dtype=torch.bool, device=q.device)
    if causal:
        mask &= torch.tril(torch.ones(T, T, dtype=torch.bool, device=q.device))
    if seqlens is not None:
        mask = mask & (torch.arange(T, device=q.device)[None, None, None, :] < seqlens.view(B, 1, 1, 1))
    s = s.masked_fill(~mask, float("-inf"))
    p = s.softmax(-1)
    return torch.einsum("bhqk,bkhd->bqhd", p, v)


@pytest.mark.parametrize("B,T,Hq,Hkv,d,causal", [(2, 300, 8, 2, 128, True), (1, 1024, 4, 4, 128, True),
                                                 (2, 640, 4, 2, 128, False)])
def test_attention_fwd(cuda_device, B, T, Hq, Hkv, d, causal):
    from metamorph_b200 import ops
    torch.manual_seed(10)
    qkv = torch.randn(B * T, (Hq + 2 * Hkv) * d, device=cuda_device).bfloat16()
    q, k, v = qkv[:, :Hq * d], qkv[:, Hq * d:(Hq + Hkv) * d], qkv[:, (Hq + Hkv) * d:]
    scale = 1.0 / math.sqrt(d)
    seqlens = None
    if causal:
        seqlens = torch.tensor([T, max(1, T - 77)][:B], device=cuda_device, dtype=torch.int32)
    out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, d, causal, scale, seqlens=seqlens)
    ref = _attn_ref(q.float().view(B, T, Hq, d), k.float().view(B, T, Hkv, d), v.float().view(B, T, Hkv, d),
                    causal, scale, seqlens)
    o = out.view(B, T, Hq, d).float()
    if seqlens is not None:
        for b in range(B):
            L = int(seqlens[b])
            _close(o[b, :L], ref[b, :L], 2e-2, f"attn fwd b={b}")
    else:
        _close(o, ref, 2e-2, "attn fwd")


@pytest.mark.parametrize("B,T,Hq,Hkv", [(2, 200, 8, 2), (1, 512, 4, 1), (1, 384, 2, 2), (2, 1501, 8, 2), (1, 2050, 4, 1)])
def test_attention_bwd(cuda_device, B, T, Hq, Hkv):
    from metamorph_b200 import ops
    torch.manual_seed(11)
    d = 128
    W = (Hq + 2 * Hkv) * d
    qkv = (torch.randn(B * T, W, device=cuda_device) * 0.5).bfloat16()
    q, k, v = qkv[:, :Hq * d], qkv[:, Hq * d:(Hq + Hkv) * d], qkv[:, (Hq + Hkv) * d:]
    scale = 1.0 / math.sqrt(d)
    seqlens = torch.tensor([T, T - 33][:B], device=cuda_device, dtype=torch.int32)
    out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, d, True, scale, seqlens=seqlens)
    dout = torch.randn(B * T, Hq * d, device=cuda_device).bfloat16()
    for b in range(B):  # reference semantics: no gradient flows into padded positions
        dout.view(B, T, -1)[b, int(seqlens[b]):] = 0
    dqkv = torch.zeros_like(qkv)
    ops.attn_bwd(q, k, v, out, dout, lse, dqkv[:, :Hq * d], dqkv[:, Hq * d:(Hq + Hkv) * d],
                 dqkv[:, (Hq + Hkv) * d:], B, T, Hq, Hkv, d, scale, seqlens=seqlens)
    qf = q.float().view(B, T, Hq, d).clone().requires_grad_(True)
    kf = k.float().view(B, T, Hkv, d).clone().requires_grad_(True)
    vf = v.float().view(B, T, Hkv, d).clone().requires_grad_(True)
    ref = _attn_ref(qf, kf, vf, True, scale, seqlens)
    ref = torch.nan_to_num(ref)
    ref.backward(dout.float().view(B, T, Hq, d))
    for b in range(B):
        L = int(seqlens[b])
        _close(dqkv[:, :Hq * d].view(B, T, Hq, d)[b, :L], qf.grad[b, :L], 3e-2, "dq")
        _close(dqkv[:, Hq * d:(Hq + Hkv) * d].view(B, T, Hkv, d)[b, :L], kf.grad[b, :L], 3e-2, "dk")
        _close(dqkv[:, (Hq + Hkv) * d:].view(B, T, Hkv, d)[b, :L], vf.grad[b, :L], 3e-2, "dv")
        # padded positions are outside the sequence: exactly zero gradients
        assert float(dqkv.view(B, T, -1)[b, L:].abs().max() if L < T else 0.0) == 0.0


def test_attention_bwd_ignores_padded_dout_and_is_deterministic(cuda_device):
    """The wgmma backward treats rows >= seqlens[b] as outside the sequence (the reference's masked positions carry no
    gradient): a non-zero dO there must not change any result; and with no atomics two runs agree bit for bit."""
    from metamorph_b200 import ops
    torch.manual_seed(12)
    B, T, Hq, Hkv, d = 2, 777, 8, 2, 128
    W = (Hq + 2 * Hkv) * d
    qkv = (torch.randn(B * T, W, device=cuda_device) * 0.5).bfloat16()
    q, k, v = qkv[:, :Hq * d], qkv[:, Hq * d:(Hq + Hkv) * d], qkv[:, (Hq + Hkv) * d:]
    scale = 1.0 / math.sqrt(d)
    seqlens = torch.tensor([T, 300], device=cuda_device, dtype=torch.int32)
    out, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, d, True, scale, seqlens=seqlens)
    dout = torch.randn(B * T, Hq * d, device=cuda_device).bfloat16()
    res = []
    for variant in range(3):
        do = dout.clone()
        if variant < 2:
            do.view(B, T, -1)[1, 300:] = 0
        g = torch.full_like(qkv, float("nan"))
        ops.attn_bwd(q, k, v, out, do, lse, g[:, :Hq * d], g[:, Hq * d:(Hq + Hkv) * d], g[:, (Hq + Hkv) * d:], B, T, Hq,
                     Hkv, d, scale, seqlens=seqlens)
        res.append(g)
    assert torch.equal(res[0], res[1])                        # bit-reproducible
    assert torch.equal(res[0], res[2])                        # dO of the padded rows is ignored
    assert torch.isfinite(res[0]).all() and float(res[0].view(B, T, -1)[1, 300:].abs().max()) == 0.0


def test_attention_varlen_packed_segments(cuda_device):
    """SURVEY section 8f N2: block-diagonal causal attention over packed sequences in ONE launch per direction
    (mm_attn_fwd_tc_varlen / mm_attn_bwd_tc_varlen) against a per-segment fp32 torch reference; segment starts are
    arbitrary (not tile aligned), rows between segments must stay untouched."""
    from metamorph_b200 import ops
    torch.manual_seed(13)
    Hq, Hkv, d = 8, 2, 128
    segs = [(0, 300), (300, 77), (400, 1029), (1429, 128), (1557, 1)]
    R = 1600
    W = (Hq + 2 * Hkv) * d
    qkv = (torch.randn(R, W, device=cuda_device) * 0.5).bfloat16()
    q, k, v = qkv[:, :Hq * d], qkv[:, Hq * d:(Hq + Hkv) * d], qkv[:, (Hq + Hkv) * d:]
    scale = 1.0 / math.sqrt(d)
    tab = ops.SegmentTables(segs, cuda_device)
    assert tab.n_work_q == sum((n + 127) // 128 for _, n in segs) == tab.n_work_k
    out = torch.full((R, Hq * d), 7.0, device=cuda_device).bfloat16()
    _, lse = ops.attn_fwd_varlen(q, k, v, tab, Hq, Hkv, d, scale, out=out)
    dout = torch.randn(R, Hq * d, device=cuda_device).bfloat16()
    g = torch.full_like(qkv, 3.0)
    ops.attn_bwd_varlen(q, k, v, out, dout, lse, g[:, :Hq * d], g[:, Hq * d:(Hq + Hkv) * d], g[:, (Hq + Hkv) * d:], tab,
                        Hq, Hkv, d, scale)
    covered = torch.zeros(R, dtype=torch.bool, device=cuda_device)
    for r0, n in segs:
        covered[r0:r0 + n] = True
        qf = q[r0:r0 + n].float().view(1, n, Hq, d).clone().requires_grad_(True)
        kf = k[r0:r0 + n].float().view(1, n, Hkv, d).clone().requires_grad_(True)
        vf = v[r0:r0 + n].float().view(1, n, Hkv, d).clone().requires_grad_(True)
        ref = _attn_ref(qf, kf, vf, True, scale)
        ref.backward(dout[r0:r0 + n].float().view(1, n, Hq, d))
        _close(out[r0:r0 + n].view(1, n, Hq, d), ref.detach(), 2e-2, f"varlen fwd seg {r0}")
        _close(g[r0:r0 + n, :Hq * d].view(1, n, Hq, d), qf.grad, 3e-2, f"varlen dq seg {r0}")
        _close(g[r0:r0 + n, Hq * d:(Hq + Hkv) * d].view(1, n, Hkv, d), kf.grad, 3e-2, f"varlen dk seg {r0}")
        _close(g[r0:r0 + n, (Hq + Hkv) * d:].view(1, n, Hkv, d), vf.grad, 3e-2, f"varlen dv seg {r0}")
    assert torch.all(out[~covered].float() == 7.0) and torch.all(g[~covered].float() == 3.0)   # gap rows untouched


def test_loss_sums_carry_non_finite_terms_and_are_reproducible(cuda_device):
    """The loss sums are order-independent (fixed point), yet a NaN term still makes the sum NaN and an Inf term makes
    it Inf, as torch's cross-entropy / cosine losses report them; finite sums match torch and repeat bit for bit."""
    from metamorph_b200 import ops
    torch.manual_seed(3)
    R, V = 64, 1000
    logits = torch.randn(R, V, device=cuda_device) * 3
    labels = torch.randint(0, V, (R,), device=cuda_device, dtype=torch.int32)
    labels[5] = -100
    ref = F.cross_entropy(logits, labels.long(), ignore_index=-100, reduction="sum").item()

    def ce(lg):
        s = torch.zeros(1, device=cuda_device)
        ops.ce_fwd_bwd(lg, labels, V, s)
        return s.item()

    sums = [ce(logits) for _ in range(3)]
    assert sums[0] == sums[1] == sums[2]
    assert abs(sums[0] - ref) <= 1e-4 * abs(ref)
    bad = logits.clone()
    bad[7, 3] = float("nan")
    assert math.isnan(ce(bad))
    inf = logits.clone()
    inf[9, int(labels[9])] = float("-inf")        # that row's term lse - x[label] is +Inf
    assert ce(inf) == float("inf")
    assert ce(logits) == sums[0]                  # a non-finite launch leaves the accumulator clean

    pred = torch.randn(48, 1152, device=cuda_device).bfloat16()
    tgt = torch.randn(48, 1152, device=cuda_device).bfloat16()

    def cos(p):
        s = torch.zeros(1, device=cuda_device)
        ops.cosine_loss(p, tgt, loss_sum=s)
        return s.item()

    want = -F.cosine_similarity(pred.float(), tgt.float()).mean().item()
    got = cos(pred)
    assert got == cos(pred)
    assert abs(got - want) <= 2e-3
    pbad = pred.clone()
    pbad[4, 10] = float("nan")
    assert math.isnan(cos(pbad))
