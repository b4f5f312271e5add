"""Python wrappers over the C-ABI kernels. Each wrapper validates shapes, allocates outputs with
torch (caller-owned memory, SURVEY.md §8b) and enqueues the kernel on torch's current stream."""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib
from ._lib import c_float, c_int, c_void_p, call, ll, ptr, require_cuda, stream_ptr

EPI_STORE, EPI_BIAS, EPI_BIAS_GELU_ERF, EPI_BIAS_GELU_TANH, EPI_RESID, EPI_BIAS_RESID, EPI_SWIGLU, EPI_SWIGLU_BWD = range(8)


ATTN_BWD_TC = True  # wgmma backward (csrc/attention_bwd_tc.cu); the mma.sync kernel stays selectable with tc=False

# bench.py instrumentation: when a list, every GEMM launch appends (start_event, end_event, flops)
GEMM_PROFILE = None


def _ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, "expected a row-major 2-D view"
    return t.stride(0)


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
         resid: Optional[torch.Tensor] = None, aux: Optional[torch.Tensor] = None,
         epilogue: int = EPI_STORE, out_dtype: torch.dtype = torch.bfloat16,
         accumulate: bool = False, alpha: float = 1.0, force_bn: int = 0) -> torch.Tensor:
    """bf16 tensor-core GEMM (wgmma). Operand storage:
         a_mn=False: a is [M, K] row-major;  a_mn=True: a is stored [K, M] row-major (A = a^T)
         b_mn=False: b is [N, K] row-major (C = A b^T, nn.Linear);  b_mn=True: b is [K, N] (C = A b)
    """
    require_cuda(a, b, out, bias, resid, aux)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    n_out = N // 2 if epilogue == EPI_SWIGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=out_dtype, device=a.device)
    assert out.shape == (M, n_out) and out.dtype == out_dtype
    prof = GEMM_PROFILE
    if prof is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
    call("mm_gemm_bf16", ptr(a), ptr(b), ptr(out), ptr(bias), ptr(resid), ptr(aux),
         ll(M), ll(N), ll(K), ll(_ld(a)), ll(_ld(b)), ll(_ld(out)),
         ll(_ld(resid) if resid is not None else 0), ll(_ld(aux) if aux is not None else 0),
         c_int(int(a_mn)), c_int(int(b_mn)), c_int(epilogue),
         c_int(1 if out_dtype == torch.float32 else 0), c_int(int(accumulate)), c_float(alpha),
         c_int(force_bn), stream_ptr())
    if prof is not None:
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        prof.append((e0, e1, 2.0 * M * N * K))
    return out


# ------------------------------------------------------------------------------------------------
# norms / rope
# ------------------------------------------------------------------------------------------------
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None):
    require_cuda(x, w)
    assert x.dim() == 2 and x.is_contiguous() and x.dtype == torch.bfloat16
    out = torch.empty_like(x) if out is None else out
    call("mm_rmsnorm_fwd", ptr(x), ptr(w), ptr(out), ll(x.shape[0]), ll(x.shape[1]), c_float(eps),
         stream_ptr())
    return out


def rmsnorm_bwd(dy, x, w, eps, dres_in=None, dw_accum=None, out=None):
    """dx = dres_in + d(rmsnorm)/dx ; dw_accum (fp32 [H]) += sum_rows dy * xhat."""
    require_cuda(dy, x, w)
    assert dy.is_contiguous() and x.is_contiguous()
    out = torch.empty_like(x) if out is None else out
    call("mm_rmsnorm_bwd", ptr(dy), ptr(x), ptr(w), ptr(dres_in), ptr(out), ptr(dw_accum),
         ll(x.shape[0]), ll(x.shape[1]), c_float(eps), stream_ptr())
    if dw_accum is not None:
        _lib.launch_count += 1     # the in-order reduction of the weight-gradient partials
    return out


def layernorm(x, w, b, eps, out=None):
    require_cuda(x, w, b)
    assert x.dim() == 2 and x.is_contiguous()
    out = torch.empty_like(x) if out is None else out
    call("mm_layernorm_fwd", ptr(x), ptr(w), ptr(b), ptr(out), ll(x.shape[0]), ll(x.shape[1]),
         c_float(eps), stream_ptr())
    return out


def rope_(qkv: torch.Tensor, pos: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor,
          n_rot_heads: int, head_dim: int, backward: bool = False):
    """In-place rotary embedding on the first n_rot_heads heads of each row of qkv [M, ld]."""
    require_cuda(qkv, pos, cos, sin)
    assert pos.dtype == torch.int32 and cos.dtype == torch.float32 and cos.is_contiguous()
    assert qkv.dim() == 2 and qkv.stride(1) == 1
    call("mm_rope_inplace", ptr(qkv), ptr(pos), ptr(cos), ptr(sin), ll(qkv.shape[0]),
         ll(qkv.stride(0)), c_int(n_rot_heads), c_int(head_dim), c_int(int(backward)), stream_ptr())
    return qkv


# ------------------------------------------------------------------------------------------------
# elementwise
# ------------------------------------------------------------------------------------------------
def swiglu_bwd(gu, dact, dgu=None, act=None):
    require_cuda(gu, dact)
    M, I2 = gu.shape
    I = I2 // 2
    assert gu.is_contiguous() and dact.is_contiguous() and dact.shape == (M, I)
    dgu = torch.empty_like(gu) if dgu is None else dgu
    call("mm_swiglu_bwd", ptr(gu), ptr(dact), ptr(dgu), ptr(act), ll(M), ll(I), stream_ptr())
    return dgu


def gelu(z, out=None):
    require_cuda(z)
    assert z.is_contiguous()
    out = torch.empty_like(z) if out is None else out
    call("mm_gelu_fwd", ptr(z), ptr(out), ll(z.numel()), stream_ptr())
    return out


def gelu_bwd(z, da, out=None):
    require_cuda(z, da)
    assert z.is_contiguous() and da.is_contiguous()
    out = torch.empty_like(z) if out is None else out
    call("mm_gelu_bwd", ptr(z), ptr(da), ptr(out), ll(z.numel()), stream_ptr())
    return out


def colsum_accum(x, out_f32):
    require_cuda(x, out_f32)
    assert x.dim() == 2 and x.stride(1) == 1 and out_f32.dtype == torch.float32
    call("mm_colsum_accum", ptr(x), ptr(out_f32), ll(x.shape[0]), ll(x.shape[1]), ll(x.stride(0)),
         stream_ptr())
    return out_f32


def im2col_patch14(images: torch.Tensor, ldp: int = 640):
    require_cuda(images)
    n, c, s, s2 = images.shape
    assert c == 3 and s == s2 and images.is_contiguous() and images.dtype == torch.bfloat16
    g = s // 14
    out = torch.empty((n * g * g, ldp), dtype=torch.bfloat16, device=images.device)
    call("mm_im2col_patch14", ptr(images), ptr(out), c_int(n), c_int(s), c_int(ldp), stream_ptr())
    return out


def add_pos_emb_(x, pos):
    require_cuda(x, pos)
    assert x.is_contiguous() and pos.is_contiguous()
    call("mm_add_pos_emb", ptr(x), ptr(pos), ll(x.shape[0]), c_int(pos.shape[0]), c_int(x.shape[1]),
         stream_ptr())
    return x


def sumsq_accum(x, out_f32):
    require_cuda(x, out_f32)
    assert x.is_contiguous()
    call("mm_sumsq_bf16_accum", ptr(x), ptr(out_f32), ll(x.numel()), stream_ptr())
    return out_f32


# ------------------------------------------------------------------------------------------------
# interleave (K9) and row gathers
# ------------------------------------------------------------------------------------------------
def interleave_gather(embed_w, img_feats, row_map, out=None):
    require_cuda(embed_w, img_feats, row_map)
    assert row_map.dtype == torch.int32 and embed_w.is_contiguous()
    H = embed_w.shape[1]
    R = row_map.numel()
    out = torch.empty((R, H), dtype=torch.bfloat16, device=embed_w.device) if out is None else out
    call("mm_interleave_gather", ptr(embed_w), ptr(img_feats), ptr(row_map), ptr(out), ll(R), c_int(H),
         stream_ptr())
    return out


def interleave_scatter(dout, row_map, dembed, dimg):
    require_cuda(dout, row_map, dembed, dimg)
    assert dout.is_contiguous()
    call("mm_interleave_scatter", ptr(dout), ptr(row_map), ptr(dembed), ptr(dimg), ll(dout.shape[0]),
         c_int(dout.shape[1]), stream_ptr())


def gather_rows(x, idx, out=None):
    require_cuda(x, idx)
    assert idx.dtype == torch.int32 and x.is_contiguous()
    out = torch.empty((idx.numel(), x.shape[1]), dtype=x.dtype, device=x.device) if out is None else out
    if idx.numel() > 0:
        call("mm_gather_rows", ptr(x), ptr(idx), ptr(out), ll(idx.numel()), c_int(x.shape[1]), stream_ptr())
    return out


def scatter_add_rows_(x, idx, g):
    require_cuda(x, idx, g)
    if idx.numel() > 0:
        call("mm_scatter_add_rows", ptr(x), ptr(idx), ptr(g), ll(idx.numel()), c_int(x.shape[1]), stream_ptr())
    return x


# ------------------------------------------------------------------------------------------------
# vision feature reduction (K7)
# ------------------------------------------------------------------------------------------------
def bilinear_l2norm(x, out_side: int, normalize: bool = True, eps: float = 1e-12):
    """x [N, S*S, C] bf16 -> [N, out_side^2, C]: bilinear (align_corners=False) + L2 normalise."""
    require_cuda(x)
    n, ss, c = x.shape
    s = int(round(ss ** 0.5))
    assert s * s == ss and x.is_contiguous()
    out = torch.empty((n, out_side * out_side, c), dtype=x.dtype, device=x.device)
    call("mm_bilinear_l2norm", ptr(x), ptr(out), c_int(n), c_int(s), c_int(out_side), c_int(c),
         c_int(int(normalize)), c_float(eps), stream_ptr())
    return out


def l2norm_rows(x, eps: float = 1e-12, out=None):
    require_cuda(x)
    assert x.dim() == 2 and x.is_contiguous()
    out = torch.empty_like(x) if out is None else out
    call("mm_l2norm_rows", ptr(x), ptr(out), ll(x.shape[0]), c_int(x.shape[1]), c_float(eps), stream_ptr())
    return out


# ------------------------------------------------------------------------------------------------
# losses
# ------------------------------------------------------------------------------------------------
def ce_fwd_bwd(logits_f32, labels_i32, V, loss_sum, dlogits=None, grad_scale=1.0, lse_out=None,
               ignore_index=-100):
    require_cuda(logits_f32, labels_i32, loss_sum)
    assert logits_f32.dtype == torch.float32 and logits_f32.stride(1) == 1
    assert labels_i32.dtype == torch.int32
    R = logits_f32.shape[0]
    call("mm_ce_fwd_bwd", ptr(logits_f32), ll(logits_f32.stride(0)), ptr(labels_i32), ptr(dlogits),
         ll(dlogits.stride(0) if dlogits is not None else 0), ptr(loss_sum), ptr(lse_out), ll(R),
         c_int(V), c_float(grad_scale), c_int(ignore_index), stream_ptr())


def cosine_loss(pred, target, loss_sum=None, pred_norm=None, dpred=None, grad_scale=1.0):
    require_cuda(pred, target)
    assert pred.is_contiguous() and pred.dim() == 2
    call("mm_cosine_loss", ptr(pred), ptr(target), ptr(pred_norm), ptr(dpred), ptr(loss_sum),
         ll(pred.shape[0]), c_int(pred.shape[1]), c_float(grad_scale), stream_ptr())


_ws_cache = {}


def _workspace(key, nbytes, device):
    buf = _ws_cache.get((key, str(device)))
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _ws_cache[(key, str(device))] = buf
    return buf


def argmax_rows(logits_f32, V, out=None):
    require_cuda(logits_f32)
    R = logits_f32.shape[0]
    out = torch.empty((R,), dtype=torch.int32, device=logits_f32.device) if out is None else out
    ws = _workspace("argmax", R * 64 * 8, logits_f32.device)
    call("mm_argmax_rows", ptr(logits_f32), ll(logits_f32.stride(0)), ll(R), c_int(V), ptr(out), ptr(ws),
         ll(ws.numel()), stream_ptr())
    return out


def sample_rows(logits_f32, V, temperature, top_k, top_p, seed, counter, out=None):
    """One seeded draw per row from the temperature / top-k / top-p warped distribution (csrc/sampling.cu).
    Per-row device arrays: temperature fp32, top_k int32, top_p fp32, seed int64 (the bits of a uint64), counter int32
    (the number of steps the sequence has taken). Rows with temperature 0 get exactly argmax_rows' token."""
    require_cuda(logits_f32, temperature, top_k, top_p, seed, counter, out)
    R = logits_f32.shape[0]
    assert logits_f32.dtype == torch.float32 and logits_f32.stride(1) == 1
    for t, dt in ((temperature, torch.float32), (top_k, torch.int32), (top_p, torch.float32), (seed, torch.int64),
                  (counter, torch.int32)):
        assert t.dtype == dt and t.is_contiguous() and t.numel() >= R, "sample_rows: bad per-row array"
    out = torch.empty((R,), dtype=torch.int32, device=logits_f32.device) if out is None else out
    call("mm_sample_rows", ptr(logits_f32), ll(logits_f32.stride(0)), ll(R), c_int(V), ptr(temperature), ptr(top_k),
         ptr(top_p), ptr(seed), ptr(counter), ptr(out), stream_ptr())
    return out


LOGPROB_TOP_MAX = 20


def decode_logprobs(logits_f32, V, append_kind, token, n_ids, n_top, lp_out, top_ids, top_lp):
    """Log-probabilities of the tokens a decode step appended (csrc/sampling.cu, DESIGN.md's log-probability
    contract). Row r with append_kind[r] == 0 and n_top[r] >= 0 writes lp_out[r, n_ids[r] - 1] = the raw
    log-softmax of token[r] and the first min(n_top[r], 20) entries of top_ids / top_lp [r, n_ids[r] - 1, :]; a slot
    past lp_out's max_ids columns and every other row are left untouched. Per-row int32 device arrays; lp_out fp32
    [R, max_ids], top_ids int32 / top_lp fp32 [R, max_ids, 20], contiguous."""
    require_cuda(logits_f32, append_kind, token, n_ids, n_top, lp_out, top_ids, top_lp)
    R = logits_f32.shape[0]
    assert logits_f32.dtype == torch.float32 and logits_f32.stride(1) == 1
    for t in (append_kind, token, n_ids, n_top):
        assert t.dtype == torch.int32 and t.is_contiguous() and t.numel() >= R, "decode_logprobs: bad per-row array"
    max_ids = lp_out.shape[1]
    assert lp_out.dtype == torch.float32 and lp_out.is_contiguous() and lp_out.shape[0] >= R
    for t, dt in ((top_ids, torch.int32), (top_lp, torch.float32)):
        assert t.dtype == dt and t.is_contiguous() and tuple(t.shape[1:]) == (max_ids, LOGPROB_TOP_MAX) \
            and t.shape[0] >= R, "decode_logprobs: bad top-n buffer"
    call("mm_decode_logprobs", ptr(logits_f32), ll(logits_f32.stride(0)), ll(R), c_int(V), ptr(append_kind),
         ptr(token), ptr(n_ids), ptr(n_top), c_int(max_ids), ptr(lp_out), ptr(top_ids), ptr(top_lp), stream_ptr())


# ------------------------------------------------------------------------------------------------
# optimizer
# ------------------------------------------------------------------------------------------------
def adamw_step_(p16, p32, m, v, grad, *, lr, beta1, beta2, eps, wd, step, grad_scale=1.0,
                grad_scale_tensor=None):
    require_cuda(p16, p32, m, v, grad)
    n = p32.numel()
    assert p16.numel() == n and m.numel() == n and v.numel() == n and grad.numel() == n
    assert p16.is_contiguous() and p32.is_contiguous() and grad.is_contiguous()
    call("mm_adamw_step", ptr(p16), ptr(p32), ptr(m), ptr(v), ptr(grad),
         c_int(1 if grad.dtype == torch.float32 else 0), ll(n), c_float(lr), c_float(beta1),
         c_float(beta2), c_float(eps), c_float(wd), c_int(step), ptr(grad_scale_tensor),
         c_float(grad_scale), stream_ptr())


def adamw_step_bcast_(multicast_ptr, peers_dev_ptr, n_peers, slice_offset, p32, m, v, grad, *, lr, beta1, beta2, eps, wd, step,
                      grad_scale=1.0, grad_scale_tensor=None, grad_multicast_ptr=0, grad_f32=None):
    """AdamW on this rank's slice with the all-gather fused in (csrc/optimizer.cu): the updated bf16 values go straight
    into every rank's parameter buffer (multicast address of the slice, or per-peer stores).
    grad_multicast_ptr != 0: the gradient is read through that multicast address (multimem.ld_reduce = the sum over all
    ranks' symmetric gradient buffers, formed inside the NVSwitch): reduce-scatter fused in as well (`grad` is ignored)."""
    require_cuda(p32, m, v)
    n = p32.numel()
    assert m.numel() == n and v.numel() == n
    if grad_multicast_ptr:
        g_ptr, g_f32 = c_void_p(grad_multicast_ptr), bool(grad_f32)
    else:
        require_cuda(grad)
        assert grad.numel() == n and grad.is_contiguous()
        g_ptr, g_f32 = ptr(grad), grad.dtype == torch.float32
    call("mm_adamw_step_bcast", c_void_p(multicast_ptr or 0), c_void_p(peers_dev_ptr or 0), c_int(n_peers), ll(slice_offset),
         ptr(p32), ptr(m), ptr(v), g_ptr, c_int(int(g_f32)), c_int(1 if grad_multicast_ptr else 0), ll(n), c_float(lr),
         c_float(beta1), c_float(beta2), c_float(eps), c_float(wd), c_int(step), ptr(grad_scale_tensor),
         c_float(grad_scale), stream_ptr())


def clip_coef(sumsq, max_norm):
    out = torch.empty(2, dtype=torch.float32, device=sumsq.device)
    call("mm_clip_coef", ptr(sumsq), ptr(out), c_float(max_norm), stream_ptr())
    return out


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def attn_fwd(q, k, v, B, T, Hq, Hkv, head_dim, causal, scale, seqlens=None, out=None, need_lse=True,
             tc=None):
    """q/k/v: 2-D row-major views [B*T, *] (may be column slices of one fused QKV buffer)."""
    require_cuda(q, k, v, seqlens)
    assert q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    if out is None:
        out = torch.empty((B * T, Hq * head_dim), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((B, Hq, T), dtype=torch.float32, device=q.device) if need_lse else None
    # One kernel on the product path: wgmma, 128-wide head slots (narrower heads are zero-padded into such slots by their
    # caller, as SiglipVisionTower does). tc=False selects the mma.sync comparison kernels (tests / microbenchmarks only).
    use_tc = True if tc is None else tc
    if use_tc and head_dim != 128:
        raise ValueError(f"attn_fwd: the wgmma attention takes head_dim 128 (got {head_dim}); pad the heads into 128-wide "
                         "slots or pass tc=False for the mma.sync comparison kernel")
    call("mm_attn_fwd_tc" if use_tc else "mm_attn_fwd", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(seqlens), ll(q.stride(0)),
         ll(k.stride(0)), ll(v.stride(0)), ll(out.stride(0)), c_int(B), c_int(T), c_int(Hq),
         c_int(Hkv), c_int(head_dim), c_int(int(causal)), c_float(scale), stream_ptr())
    return out, lse


def attn_bwd(q, k, v, o, dout, lse, dq, dk, dv, B, T, Hq, Hkv, head_dim, scale, seqlens=None,
             workspace=None, tc=None):
    require_cuda(q, k, v, o, dout, lse, dq, dk, dv)
    from ._lib import lib
    use_tc = ATTN_BWD_TC if tc is None else tc   # tc=False: the mma.sync kernel, kept as a test-only comparison
    fn = lib().mm_attn_bwd_tc_workspace_bytes if use_tc else lib().mm_attn_bwd_workspace_bytes
    fn.restype = ctypes_ll
    need = fn(c_int(B), c_int(T), c_int(Hq))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=q.device)
    call("mm_attn_bwd_tc" if use_tc else "mm_attn_bwd", ptr(q), ptr(k), ptr(v), ptr(o), ptr(dout), ptr(lse), ptr(dq), ptr(dk), ptr(dv),
         ptr(seqlens), ll(q.stride(0)), ll(k.stride(0)), ll(v.stride(0)), ll(o.stride(0)),
         ll(dout.stride(0)), ll(dq.stride(0)), ll(dk.stride(0)), ll(dv.stride(0)), c_int(B), c_int(T),
         c_int(Hq), c_int(Hkv), c_int(head_dim), c_float(scale), ptr(workspace), ll(workspace.numel()),
         stream_ptr())
    return workspace


class SegmentTables:
    """Device tables of a packed batch (SURVEY section 8f N2) for the one-launch block-diagonal attention kernels:
    sequence s occupies rows [start[s], start[s] + length[s]) of the token dimension. The work lists name every
    128-row tile that exists — (sequence, query tile) for the forward / dQ kernels, (sequence, key tile) for the dK/dV
    kernel — heaviest first (a query tile attends to tile+1 key tiles, a key tile is visited by n_tiles-tile query tiles)."""

    def __init__(self, segments, device):
        self.segments = [(int(a), int(n)) for a, n in segments]
        self.n_seg = len(self.segments)
        self.max_len = max(n for _, n in self.segments)
        self.total = sum(n for _, n in self.segments)
        wq, wk = [], []
        for s, (_, n) in enumerate(self.segments):
            nt = (n + 127) // 128
            wq += [(t + 1, s, t) for t in range(nt)]
            wk += [(nt - t, s, t) for t in range(nt)]
        wq.sort(key=lambda x: -x[0])
        wk.sort(key=lambda x: -x[0])
        host = torch.tensor([a for a, _ in self.segments] + [n for _, n in self.segments] +
                            [v for _, s_, t in wq for v in (s_, t)] + [v for _, s_, t in wk for v in (s_, t)],
                            dtype=torch.int32)
        dev = host.to(device, non_blocking=True)
        S = self.n_seg
        self.start, self.length = dev[:S], dev[S:2 * S]
        self.n_work_q, self.n_work_k = len(wq), len(wk)
        self.work_q = dev[2 * S:2 * S + 2 * len(wq)]
        self.work_k = dev[2 * S + 2 * len(wq):]


def attn_fwd_varlen(q, k, v, seg: SegmentTables, Hq, Hkv, head_dim, scale, out, need_lse=True):
    """Block-diagonal causal attention over the packed sequences of `seg` in ONE launch (wgmma kernel).
    Rows outside every sequence are not written. Returns (out, lse [n_seg, Hq, max_len])."""
    require_cuda(q, k, v, out)
    assert q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1 and head_dim == 128
    lse = torch.empty((seg.n_seg, Hq, seg.max_len), dtype=torch.float32, device=q.device) if need_lse else None
    call("mm_attn_fwd_tc_varlen", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(seg.start), ptr(seg.length),
         c_int(seg.n_seg), c_int(seg.max_len), ptr(seg.work_q), c_int(seg.n_work_q), ll(q.shape[0]), ll(q.stride(0)),
         ll(k.stride(0)), ll(v.stride(0)), ll(out.stride(0)), c_int(Hq), c_int(Hkv), c_int(head_dim), c_float(scale),
         stream_ptr())
    return out, lse


def attn_bwd_varlen(q, k, v, o, dout, lse, dq, dk, dv, seg: SegmentTables, Hq, Hkv, head_dim, scale, workspace=None):
    require_cuda(q, k, v, o, dout, lse, dq, dk, dv)
    from ._lib import lib
    fn = lib().mm_attn_bwd_tc_workspace_bytes
    fn.restype = ctypes_ll
    need = fn(c_int(seg.n_seg), c_int(seg.max_len), c_int(Hq))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=q.device)
    call("mm_attn_bwd_tc_varlen", ptr(q), ptr(k), ptr(v), ptr(o), ptr(dout), ptr(lse), ptr(dq), ptr(dk), ptr(dv),
         ptr(seg.start), ptr(seg.length), c_int(seg.n_seg), c_int(seg.max_len), ptr(seg.work_q), c_int(seg.n_work_q),
         ptr(seg.work_k), c_int(seg.n_work_k), ll(q.shape[0]), ll(q.stride(0)), ll(k.stride(0)), ll(v.stride(0)),
         ll(o.stride(0)), ll(dout.stride(0)), ll(dq.stride(0)), ll(dk.stride(0)), ll(dv.stride(0)), c_int(Hq),
         c_int(Hkv), c_int(head_dim), c_float(scale), ptr(workspace), ll(workspace.numel()), stream_ptr())
    return workspace


import ctypes as _ctypes  # noqa: E402

ctypes_ll = _ctypes.c_longlong


# ------------------------------------------------------------------------------------------------
# decode (KV-cached step)
# ------------------------------------------------------------------------------------------------
SK_STORE, SK_BIAS, SK_RESID, SK_BIAS_GELU, SK_SWIGLU = range(5)


def skinny_gemm(x, w, *, bias=None, resid=None, epilogue=SK_STORE, out=None, out_dtype=torch.bfloat16, wide=None):
    """y[m<=128, N] = x[m, K] w[N, K]^T — HBM-bound weight streaming for the decode step.
    m <= 32 runs `mm_skinny_gemm` (mma.sync, the batch is 1, 2 or 4 n8 tiles); 33 <= m <= 128 runs `mm_skinny_gemm_wide`
    (wgmma over a 128-wide batch operand, split-K reduced in a fixed order). The two agree within bf16 rounding; within one
    kernel a row's bits do not depend on the other rows. `wide=True` forces the wide kernel for any m (comparisons)."""
    require_cuda(x, w, bias, resid, out)
    m, K = x.shape
    N = w.shape[0]
    n_out = N // 2 if epilogue == SK_SWIGLU else N
    if wide is None:
        wide = m > 32
    if out is None:
        out = torch.empty((m, n_out), dtype=out_dtype, device=x.device)
    call("mm_skinny_gemm_wide" if wide else "mm_skinny_gemm", ptr(x), ptr(w), ptr(out), ptr(bias), ptr(resid), ll(x.stride(0)),
         ll(w.stride(0)), ll(out.stride(0)), ll(resid.stride(0) if resid is not None else 0), c_int(m),
         c_int(N), c_int(K), c_int(epilogue), c_int(1 if out.dtype == torch.float32 else 0), stream_ptr())
    return out


def _decode_attn_splits(B, Hkv, device):
    """Default context split of decode_attn / decode_attn_paged: enough CTAs to cover the SMs, B*Hkv*splits >= ~2 x
    #SMs."""
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    return max(1, min(16, -(-2 * sms // (B * Hkv))))


def decode_attn(qkv, kcache, vcache, pos, cos, sin, Hq, Hkv, head_dim, scale, out=None, splits=None):
    require_cuda(qkv, kcache, vcache, pos, cos, sin)
    B = qkv.shape[0]
    Tmax = kcache.shape[2]
    if splits is None:
        splits = _decode_attn_splits(B, Hkv, qkv.device)
    if out is None:
        out = torch.empty((B, Hq * head_dim), dtype=torch.bfloat16, device=qkv.device)
    ws = _workspace("decode_attn", B * Hkv * splits * (Hq // Hkv) * (2 + head_dim) * 4, qkv.device)
    call("mm_decode_attn", ptr(qkv), ll(qkv.stride(0)), ptr(kcache), ptr(vcache), ptr(pos), ptr(cos),
         ptr(sin), ptr(out), ll(out.stride(0)), c_int(B), c_int(Hq), c_int(Hkv), c_int(head_dim),
         c_int(Tmax), c_float(scale), ptr(ws), ll(ws.numel()), c_int(splits), stream_ptr())
    return out


def kv_prefill(qkv, kcache, vcache, B, T, Hq, Hkv, head_dim):
    require_cuda(qkv, kcache, vcache)
    call("mm_kv_prefill", ptr(qkv), ll(qkv.stride(0)), ptr(kcache), ptr(vcache), c_int(B), c_int(T),
         c_int(Hq), c_int(Hkv), c_int(head_dim), c_int(kcache.shape[2]), stream_ptr())


def decode_attn_paged(qkv, kpool, vpool, table, pos, cos, sin, Hq, Hkv, head_dim, scale, out=None, splits=None):
    """decode_attn over a paged cache: kpool / vpool [num_blocks, Hkv, block_size, head_dim], table [B, max_blocks]
    int32 (device) mapping block p // block_size of sequence b to a pool block. With equal `splits` the output and the
    appended K/V are bit-identical to decode_attn on the same logical cache of max_blocks * block_size positions."""
    require_cuda(qkv, kpool, vpool, table, pos, cos, sin)
    assert table.dtype == torch.int32 and table.dim() == 2 and table.is_contiguous(), "table: [B, max_blocks] int32"
    B = qkv.shape[0]
    assert table.shape[0] >= B
    if splits is None:
        splits = _decode_attn_splits(B, Hkv, qkv.device)
    if out is None:
        out = torch.empty((B, Hq * head_dim), dtype=torch.bfloat16, device=qkv.device)
    ws = _workspace("decode_attn", B * Hkv * splits * (Hq // Hkv) * (2 + head_dim) * 4, qkv.device)
    call("mm_decode_attn_paged", ptr(qkv), ll(qkv.stride(0)), ptr(kpool), ptr(vpool), ptr(table),
         c_int(table.shape[1]), c_int(kpool.shape[2]), ptr(pos), ptr(cos), ptr(sin), ptr(out), ll(out.stride(0)),
         c_int(B), c_int(Hq), c_int(Hkv), c_int(head_dim), c_float(scale), ptr(ws), ll(ws.numel()), c_int(splits),
         stream_ptr())
    return out


def kv_prefill_paged(qkv, kpool, vpool, table_row, T, Hq, Hkv, head_dim):
    """kv_prefill for one sequence into the blocks of its table row (table_row [max_blocks] int32, device)."""
    require_cuda(qkv, kpool, vpool, table_row)
    assert table_row.dtype == torch.int32 and table_row.dim() == 1 and table_row.stride(0) == 1
    call("mm_kv_prefill_paged", ptr(qkv), ll(qkv.stride(0)), ptr(kpool), ptr(vpool), ptr(table_row),
         c_int(table_row.shape[0]), c_int(kpool.shape[2]), c_int(T), c_int(Hq), c_int(Hkv), c_int(head_dim),
         stream_ptr())


def attn_fwd_paged(q, kpool, vpool, table_row, q_start, Hq, Hkv, head_dim, scale, out=None):
    """Causal attention of the query rows of positions q_start .. q_start + n_q - 1 (q: [n_q, *] row-major view, e.g. the
    Q columns of a fused qkv) over keys / values 0 .. q_start + n_q - 1 of a paged pool (kpool / vpool [num_blocks, Hkv,
    block_size, head_dim], table_row [max_blocks] int32 on the device). Row r of the output is bit-identical to row r of
    attn_fwd(B=1, T=q_start + n_q, causal) on the same K/V. Returns out [n_q, Hq * head_dim]."""
    require_cuda(q, kpool, vpool, table_row, out)
    assert q.dim() == 2 and q.stride(1) == 1
    assert kpool.dim() == 4 and kpool.is_contiguous() and vpool.shape == kpool.shape and vpool.is_contiguous()
    assert table_row.dtype == torch.int32 and table_row.dim() == 1 and table_row.stride(0) == 1
    n_q = q.shape[0]
    if out is None:
        out = torch.empty((n_q, Hq * head_dim), dtype=torch.bfloat16, device=q.device)
    call("mm_attn_fwd_tc_paged", ptr(q), ll(q.stride(0)), ptr(kpool), ptr(vpool), c_int(kpool.shape[0]), ptr(table_row),
         c_int(table_row.shape[0]), c_int(kpool.shape[2]), ptr(out), ll(out.stride(0)), c_int(q_start), c_int(n_q),
         c_int(Hq), c_int(Hkv), c_int(head_dim), c_float(scale), stream_ptr())
    return out


def decode_state_step(st: dict, argmax_tok, forced, step, B, num_image_tokens, max_new_tokens,
                      start_id, end_id, eos0, eos1, pred_z, img_out):
    call("mm_decode_state_step", ptr(st["in_image_mode"]), ptr(st["total_image_tokens"]),
         ptr(st["total_output"]), ptr(st["finished"]), ptr(st["pos"]), ptr(st["n_ids"]), ptr(st["n_img"]),
         ptr(st["ids_out"]), ptr(st["append_kind"]), ptr(st["next_token"]), ptr(argmax_tok), ptr(forced),
         c_int(forced.stride(0) if forced is not None else 0), c_int(step), c_int(B),
         c_int(num_image_tokens), c_int(max_new_tokens), c_int(st["ids_out"].shape[1]), c_int(start_id),
         c_int(end_id), c_int(eos0), c_int(eos1), ptr(pred_z), ptr(img_out), c_int(img_out.shape[1]),
         c_int(img_out.shape[2]), stream_ptr())


def decode_state_step_slots(st: dict, argmax_tok, forced, max_new_slot, B, num_image_tokens, start_id, end_id, eos0,
                            eos1, pred_z, img_out):
    """The greedy_decode state machine with one output limit per batch slot (continuous batching)."""
    call("mm_decode_state_step_slots", ptr(st["in_image_mode"]), ptr(st["total_image_tokens"]),
         ptr(st["total_output"]), ptr(st["finished"]), ptr(st["pos"]), ptr(st["n_ids"]), ptr(st["n_img"]),
         ptr(st["ids_out"]), ptr(st["append_kind"]), ptr(st["next_token"]), ptr(argmax_tok), ptr(forced),
         c_int(forced.stride(0) if forced is not None else 0), ptr(max_new_slot), c_int(B), c_int(num_image_tokens),
         c_int(st["ids_out"].shape[1]), c_int(start_id), c_int(end_id), c_int(eos0), c_int(eos1), ptr(pred_z),
         ptr(img_out), c_int(img_out.shape[1]), c_int(img_out.shape[2]), stream_ptr())


def decode_next_input(kind, tok, embed_w, pred, x):
    call("mm_decode_next_input", ptr(kind), ptr(tok), ptr(embed_w), ptr(pred), ptr(x), c_int(x.shape[0]),
         c_int(x.shape[1]), stream_ptr())


def decode_select_hidden(mode, hidden, pred, out):
    call("mm_decode_select_hidden", ptr(mode), ptr(hidden), ptr(pred), ptr(out), c_int(out.shape[0]),
         c_int(out.shape[1]), stream_ptr())
