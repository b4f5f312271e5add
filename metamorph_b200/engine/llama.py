"""LLaMA decoder stack on the sm_90a kernels: explicit forward + hand-written backward.

Arithmetic spec: HF `LlamaModel` (transformers modeling_llama.py: LlamaRMSNorm:53, rotary:73-168,
LlamaMLP:171, LlamaAttention:225, LlamaDecoderLayer:292), called by the reference at
metamorph_llama.py:349-359.  No autograd graph is built for the stack: the backward below issues the
dgrad / wgrad GEMMs, flash-attention backward, RMSNorm/RoPE/SwiGLU backward kernels directly, with
selective recomputation (norms and, optionally, the gate/up GEMM) instead of per-layer checkpointing.

Fused device layout (see engine/packing.py for the HF <-> fused mapping):
    wqkv  [(Hq+2Hkv)*dh, H]   rows = q heads | k heads | v heads
    wo    [H, Hq*dh]
    wgu   [2I, H]             gate/up interleaved in blocks of 16 rows
    wd    [H, I]
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch

from .. import ops


@dataclass
class LlamaDims:
    hidden: int
    n_layers: int
    n_heads: int
    n_kv_heads: int
    head_dim: int
    intermediate: int
    vocab: int
    rms_eps: float = 1e-5
    rope_theta: float = 500000.0
    rope_scaling: Optional[dict] = None
    max_pos: int = 8192

    @property
    def qkv_width(self) -> int:
        return (self.n_heads + 2 * self.n_kv_heads) * self.head_dim


def rope_tables(dims: LlamaDims, n_pos: int, device, round_bf16: bool = True):
    """cos/sin [n_pos, dh/2] fp32 following HF LlamaRotaryEmbedding (default and 'llama3' scaling).
    HF casts cos/sin to the activation dtype (bf16) before use; `round_bf16` reproduces that."""
    dh = dims.head_dim
    inv = 1.0 / (dims.rope_theta ** (torch.arange(0, dh, 2, dtype=torch.int64).float() / dh))
    rs = dims.rope_scaling
    if rs and rs.get("rope_type", rs.get("type")) == "llama3":
        factor, lo, hi = rs["factor"], rs["low_freq_factor"], rs["high_freq_factor"]
        old = rs["original_max_position_embeddings"]
        wavelen = 2 * math.pi / inv
        inv_l = torch.where(wavelen > old / lo, inv / factor, inv)
        smooth = (old / wavelen - lo) / (hi - lo)
        smoothed = (1 - smooth) * inv_l / factor + smooth * inv_l
        is_med = ~(wavelen < old / hi) * ~(wavelen > old / lo)
        inv = torch.where(is_med, smoothed, inv_l)
    ang = torch.arange(n_pos, dtype=torch.float32)[:, None] * inv[None, :].float()
    cos, sin = ang.cos(), ang.sin()
    if round_bf16:
        cos, sin = cos.bfloat16().float(), sin.bfloat16().float()
    return cos.contiguous().to(device), sin.contiguous().to(device)


@dataclass
class LayerWeights:
    ln1: torch.Tensor
    wqkv: torch.Tensor
    wo: torch.Tensor
    ln2: torch.Tensor
    wgu: torch.Tensor
    wd: torch.Tensor


@dataclass
class LayerGrads:
    """Destination buffers for one layer's parameter gradients (bf16 matrices, fp32 norm vectors)."""
    wqkv: torch.Tensor
    wo: torch.Tensor
    wgu: torch.Tensor
    wd: torch.Tensor
    ln1: torch.Tensor  # fp32 [H]
    ln2: torch.Tensor  # fp32 [H]


@dataclass
class LayerSaved:
    x_in: torch.Tensor
    qkv: torch.Tensor
    attn: torch.Tensor
    lse: torch.Tensor
    h_mid: torch.Tensor
    gu: Optional[torch.Tensor] = None


@dataclass
class StackContext:
    B: int
    T: int
    pos: torch.Tensor            # int32 [B*T]
    seqlens: Optional[torch.Tensor]
    saved: List[LayerSaved] = field(default_factory=list)
    # sequence packing: flat (first row, length) of every sample in the [B*T] token dimension; attention is
    # block-diagonal causal over these segments (ONE launch per layer through the segment tables), every other kernel is
    # per token and does not care
    segments: Optional[List[tuple]] = None
    seg_tables: Optional["ops.SegmentTables"] = None
    x_final_in: Optional[torch.Tensor] = None  # input of the final norm


@dataclass
class PagedPrefill:
    """One layer's view of a paged KV cache for a prefill that continues a cached prefix: the rows of `layer_forward`
    are positions q_start .. q_start + T - 1 of ONE sequence, whose keys / values 0 .. q_start - 1 already sit in the
    pool blocks named by `table_row`. q_start is a multiple of the block size."""
    kpool: torch.Tensor          # [num_blocks, Hkv, block_size, dh] of this layer
    vpool: torch.Tensor
    table_row: torch.Tensor      # int32 [max_blocks] (device)
    q_start: int


@dataclass
class FP8KVStore:
    """One layer's FP8 KV cache (E4M3 bytes + one fp32 scale per (position, kv head) row, ops.kv_quant_prefill) for the
    rows of a prefill. `layer_forward` quantises their post-RoPE K/V into it right after RoPE and attends over what it
    holds: the K/V columns of qkv are overwritten with the dequantised rows.
      dense (table_row None): kc / vc [B, Hkv, Tmax, dh] uint8, ks / vs [B, Hkv, Tmax] fp32, rows = B sequences of T;
      paged: pools [num_blocks, Hkv, block_size, dh] and scales [num_blocks, Hkv, block_size]; the rows are positions
        q_start .. q_start + T - 1 of ONE sequence, written through its table row. With q_start > 0 (a cached prefix of
        q_start positions, a block multiple) `staging` = (kst, vst, identity row) holds bf16 pools [max_blocks, Hkv,
        block_size, dh]: the prefix blocks are dequantised into them, the new rows follow, and attention reads keys
        0 .. q_start + T - 1 from there (ops.attn_fwd_paged), so it sees exactly the values the cache holds."""
    kc: torch.Tensor
    vc: torch.Tensor
    ks: torch.Tensor
    vs: torch.Tensor
    table_row: Optional[torch.Tensor] = None
    q_start: int = 0
    staging: Optional[tuple] = None

    def write(self, qkv: torch.Tensor, B: int, T: int, Hq: int, Hkv: int, dh: int) -> None:
        if self.table_row is None:
            ops.kv_quant_prefill(qkv, self.kc, self.vc, self.ks, self.vs, B, T, Hq, Hkv, dh)
            return
        bs = self.kc.shape[2]
        assert B == 1 and self.q_start % bs == 0 and (self.q_start == 0 or self.staging is not None), \
            "a paged FP8 prefill continues one sequence at a block boundary, through staging after a prefix"
        first = self.q_start // bs
        if self.staging is not None:
            kst, vst, ident = self.staging
            ops.kv_dequant_paged(self.kc, self.vc, self.ks, self.vs, self.table_row, first, kst, vst)
        ops.kv_quant_prefill_paged(qkv, self.kc, self.vc, self.ks, self.vs, self.table_row[first:], T, Hq, Hkv, dh)
        if self.staging is not None:
            ops.kv_prefill_paged(qkv, kst, vst, ident[first:], T, Hq, Hkv, dh)


class LlamaStack:
    """Forward/backward over a list of LayerWeights. Stateless apart from the RoPE tables."""

    def __init__(self, dims: LlamaDims, device):
        self.dims = dims
        self.device = device
        self.cos, self.sin = rope_tables(dims, dims.max_pos, device)
        self.scale = 1.0 / math.sqrt(dims.head_dim)
        self._attn_ws = None

    def ensure_positions(self, n_pos: int):
        if n_pos > self.cos.shape[0]:
            self.cos, self.sin = rope_tables(self.dims, n_pos, self.device)

    # ------------------------------------------------------------------ forward
    def layer_forward(self, w: LayerWeights, x: torch.Tensor, ctx: StackContext, save: bool,
                      save_gu: bool, paged: Optional[PagedPrefill] = None,
                      kv: Optional[FP8KVStore] = None) -> torch.Tensor:
        """paged: the rows continue a sequence cached in a paged pool (prefix caching). Their post-RoPE K/V are written
        into the pool blocks from position q_start on, and attention reads keys 0 .. q_start + T - 1 from the pool.
        kv: an FP8 cache the rows' post-RoPE K/V are quantised into before attention, which then reads the dequantised
        values (FP8KVStore); None keeps the bf16 path."""
        d = self.dims
        B, T = ctx.B, ctx.T
        Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
        n1 = ops.rmsnorm(x, w.ln1, d.rms_eps)
        qkv = ops.gemm(n1, w.wqkv)
        del n1
        ops.rope_(qkv, ctx.pos, self.cos, self.sin, Hq + Hkv, dh)
        q, k, v = qkv[:, :Hq * dh], qkv[:, Hq * dh:(Hq + Hkv) * dh], qkv[:, (Hq + Hkv) * dh:]
        if kv is not None:
            kv.write(qkv, B, T, Hq, Hkv, dh)
        if kv is not None and kv.staging is not None:
            kst, vst, ident = kv.staging
            attn, lse = ops.attn_fwd_paged(q, kst, vst, ident, kv.q_start, Hq, Hkv, dh, self.scale), None
        elif paged is not None:
            bs = paged.kpool.shape[2]
            assert B == 1 and paged.q_start % bs == 0, "a paged prefill continues one sequence at a block boundary"
            ops.kv_prefill_paged(qkv, paged.kpool, paged.vpool, paged.table_row[paged.q_start // bs:], x.shape[0], Hq,
                                 Hkv, dh)
            attn, lse = ops.attn_fwd_paged(q, paged.kpool, paged.vpool, paged.table_row, paged.q_start, Hq, Hkv, dh,
                                           self.scale), None
        elif ctx.segments is None:
            attn, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, dh, True, self.scale, seqlens=ctx.seqlens,
                                     need_lse=save)
        else:
            if ctx.seg_tables is None:
                ctx.seg_tables = ops.SegmentTables(ctx.segments, x.device)
            attn = torch.zeros((x.shape[0], Hq * dh), dtype=torch.bfloat16, device=x.device)   # pad rows stay finite
            _, lse = ops.attn_fwd_varlen(q, k, v, ctx.seg_tables, Hq, Hkv, dh, self.scale, out=attn, need_lse=save)
        h_mid = ops.gemm(attn, w.wo, resid=x, epilogue=ops.EPI_RESID)
        n2 = ops.rmsnorm(h_mid, w.ln2, d.rms_eps)
        gu = torch.empty((x.shape[0], 2 * d.intermediate), dtype=torch.bfloat16, device=x.device) \
            if (save and save_gu) else None
        act = ops.gemm(n2, w.wgu, aux=gu, epilogue=ops.EPI_SWIGLU)
        del n2
        out = ops.gemm(act, w.wd, resid=h_mid, epilogue=ops.EPI_RESID)
        del act
        if save:
            ctx.saved.append(LayerSaved(x, qkv, attn, lse, h_mid, gu))
        return out

    def forward(self, layers: List[LayerWeights], final_norm: torch.Tensor, x: torch.Tensor,
                ctx: StackContext, save: bool = True, n_save_gu: int = 0) -> torch.Tensor:
        """x: inputs_embeds [B*T, H] bf16.  Returns the final-norm output [B*T, H]."""
        self.ensure_positions(int(ctx.T) + 1)
        L = len(layers)
        for i, w in enumerate(layers):
            x = self.layer_forward(w, x, ctx, save, save_gu=(i >= L - n_save_gu))
        if save:
            ctx.x_final_in = x
        return ops.rmsnorm(x, final_norm, self.dims.rms_eps)

    # ------------------------------------------------------------------ backward
    def final_norm_backward(self, final_norm, dh_final, ctx: StackContext, dw_accum):
        return ops.rmsnorm_bwd(dh_final, ctx.x_final_in, final_norm, self.dims.rms_eps, dw_accum=dw_accum)

    def layer_backward(self, w: LayerWeights, g: Optional[LayerGrads], s: LayerSaved, dx_out: torch.Tensor,
                       ctx: StackContext, accumulate: bool = False, need_wgrad: bool = True) -> torch.Tensor:
        d = self.dims
        B, T = ctx.B, ctx.T
        Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
        M = dx_out.shape[0]
        # ---- MLP: out = h_mid + down(swiglu(gate_up(norm2(h_mid))))
        n2 = ops.rmsnorm(s.h_mid, w.ln2, d.rms_eps)
        if s.gu is not None:
            gu = s.gu
        else:  # selective recompute of the gate/up projection
            gu = torch.empty((M, 2 * d.intermediate), dtype=torch.bfloat16, device=dx_out.device)
            tmp = ops.gemm(n2, w.wgu, aux=gu, epilogue=ops.EPI_SWIGLU)
            del tmp
        # d(act) = dout * Wd with the SwiGLU backward fused into the epilogue: d(act) is never written,
        # gu <- d(gate|up) in place, act = silu(g)*u recomputed for the down_proj wgrad
        act = torch.empty((M, d.intermediate), dtype=torch.bfloat16, device=dx_out.device)
        ops.gemm(dx_out, w.wd, b_mn=True, out=act, aux=gu, epilogue=ops.EPI_SWIGLU_BWD)
        if need_wgrad:
            ops.gemm(dx_out, act, a_mn=True, b_mn=True, out=g.wd, accumulate=accumulate)   # dWd = dout^T act
        del act
        if need_wgrad:
            ops.gemm(gu, n2, a_mn=True, b_mn=True, out=g.wgu, accumulate=accumulate)       # dWgu = dgu^T n2
        dn2 = ops.gemm(gu, w.wgu, b_mn=True)                                            # [M, H]
        del gu, n2
        s.gu = None
        dh_mid = ops.rmsnorm_bwd(dn2, s.h_mid, w.ln2, d.rms_eps, dres_in=dx_out, dw_accum=g.ln2 if need_wgrad else None)
        del dn2
        # ---- attention: h_mid = x + o_proj(attn(rope(qkv(norm1(x)))))
        if need_wgrad:
            ops.gemm(dh_mid, s.attn, a_mn=True, b_mn=True, out=g.wo, accumulate=accumulate)  # dWo
        dattn = ops.gemm(dh_mid, w.wo, b_mn=True)                                         # [M, Hq*dh]
        q, k, v = s.qkv[:, :Hq * dh], s.qkv[:, Hq * dh:(Hq + Hkv) * dh], s.qkv[:, (Hq + Hkv) * dh:]
        if ctx.segments is None:
            dqkv = torch.empty_like(s.qkv)
            self._attn_ws = ops.attn_bwd(q, k, v, s.attn, dattn, s.lse, dqkv[:, :Hq * dh],
                                         dqkv[:, Hq * dh:(Hq + Hkv) * dh], dqkv[:, (Hq + Hkv) * dh:],
                                         B, T, Hq, Hkv, dh, self.scale, seqlens=ctx.seqlens,
                                         workspace=self._attn_ws)
        else:
            dqkv = torch.zeros_like(s.qkv)                    # rows between / after the segments get no gradient
            self._attn_ws = ops.attn_bwd_varlen(q, k, v, s.attn, dattn, s.lse, dqkv[:, :Hq * dh],
                                                dqkv[:, Hq * dh:(Hq + Hkv) * dh], dqkv[:, (Hq + Hkv) * dh:],
                                                ctx.seg_tables, Hq, Hkv, dh, self.scale, workspace=self._attn_ws)
        del dattn
        ops.rope_(dqkv, ctx.pos, self.cos, self.sin, Hq + Hkv, dh, backward=True)
        if need_wgrad:
            n1 = ops.rmsnorm(s.x_in, w.ln1, d.rms_eps)
            ops.gemm(dqkv, n1, a_mn=True, b_mn=True, out=g.wqkv, accumulate=accumulate)      # dWqkv
            del n1
        dn1 = ops.gemm(dqkv, w.wqkv, b_mn=True)
        del dqkv
        dx = ops.rmsnorm_bwd(dn1, s.x_in, w.ln1, d.rms_eps, dres_in=dh_mid, dw_accum=g.ln1 if need_wgrad else None)
        return dx

    def backward(self, layers: List[LayerWeights], grads_for: Optional[Callable[[int], LayerGrads]],
                 dx: torch.Tensor, ctx: StackContext,
                 on_layer_done: Optional[Callable[[int, LayerGrads], None]] = None,
                 accumulate: bool = False, need_wgrad: bool = True) -> torch.Tensor:
        """dx: gradient w.r.t. the last layer's output (i.e. after final_norm_backward).
        need_wgrad=False (frozen stack, e.g. stage-1 projector training): only the dgrad chain runs."""
        for i in reversed(range(len(layers))):
            s = ctx.saved[i]
            g = grads_for(i) if need_wgrad else None
            dx = self.layer_backward(layers[i], g, s, dx, ctx, accumulate=accumulate, need_wgrad=need_wgrad)
            ctx.saved[i] = None
            if need_wgrad and on_layer_done is not None:
                on_layer_done(i, g)
        return dx
