"""The kernels of one KV-cached decode step, shared by DecodeEngine (one batch to completion) and
ContinuousBatcher (a stream of requests): decoder stack on the weight-streaming GEMMs, then the heads
(final norm, vision head -> projector feedback branch, lm_head, argmax or seeded draw). Reference arithmetic:
metamorph_llama.py:363-377, 482-490 (decoding branch of llm_forward) and 526-582 (greedy_decode loop body)."""
from __future__ import annotations

import torch

from .. import ops


def decoder_stack_step(layers, x, kc, vc, cur_pos, stack, table=None):
    """x [B, H] -> [B, H] through all layers; K/V of the fed position are appended to kc/vc [L, B, Hkv, Tmax, dh].
    With a block table [B, max_blocks] (int32, device) kc/vc are paged pools [L, num_blocks, Hkv, block_size, dh] and
    the attention addresses them through it (ops.decode_attn_paged: the same bits as the dense cache)."""
    d = stack.dims
    Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
    for i, w in enumerate(layers):
        n1 = ops.rmsnorm(x, w.ln1, d.rms_eps)
        qkv = ops.skinny_gemm(n1, w.wqkv)
        if table is None:
            attn = ops.decode_attn(qkv, kc[i], vc[i], cur_pos, stack.cos, stack.sin, Hq, Hkv, dh, stack.scale)
        else:
            attn = ops.decode_attn_paged(qkv, kc[i], vc[i], table, cur_pos, stack.cos, stack.sin, Hq, Hkv, dh,
                                         stack.scale)
        hmid = ops.skinny_gemm(attn, w.wo, resid=x, epilogue=ops.SK_RESID)
        n2 = ops.rmsnorm(hmid, w.ln2, d.rms_eps)
        act = ops.skinny_gemm(n2, w.wgu, epilogue=ops.SK_SWIGLU)
        x = ops.skinny_gemm(act, w.wd, resid=hmid, epilogue=ops.SK_RESID)
    return x


def decode_heads(m, h_pre_norm, in_image_mode, logits, V, sampling=None, counter=None):
    """-> (token [B] int32, pred_z [B, C] (normalised visual embedding), prediction [B, H] (its projection)).
    The image-mode branch is computed for every sequence and selected per sequence (graph friendly).
    sampling: None = argmax (metamorph_llama.py:542); else a SamplingArrays of per-row device parameters, and the token
    is the seeded draw of ops.sample_rows with `counter` [B] int32 (steps each sequence has taken) on the device."""
    inner = m.get_model()
    d = m.stack.dims
    hidden = ops.rmsnorm(h_pre_norm, inner.norm.weight.data, d.rms_eps)
    vh, pj = m.vision_head, inner.mm_projector
    z = ops.skinny_gemm(hidden, vh.fc1.weight.data, bias=vh.fc1.bias.data, epilogue=ops.SK_BIAS_GELU)
    z = ops.skinny_gemm(z, vh.fc2.weight.data, bias=vh.fc2.bias.data, epilogue=ops.SK_BIAS)
    pred_z = ops.l2norm_rows(z) if m.normalize_vision else z
    p1 = ops.skinny_gemm(pred_z, pj.fc1.weight.data, bias=pj.fc1.bias.data, epilogue=ops.SK_BIAS_GELU)
    prediction = ops.skinny_gemm(p1, pj.fc2.weight.data, bias=pj.fc2.bias.data, epilogue=ops.SK_BIAS)
    h_eff = torch.empty_like(hidden)
    ops.decode_select_hidden(in_image_mode, hidden, prediction, h_eff)
    ops.skinny_gemm(h_eff, m.lm_head.weight.data, out=logits[:, :V])
    if sampling is None:
        tok = ops.argmax_rows(logits, V)
    else:
        tok = ops.sample_rows(logits, V, sampling.temperature, sampling.top_k, sampling.top_p, sampling.seed, counter)
    return tok, pred_z, prediction
