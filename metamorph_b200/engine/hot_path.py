"""The MetaMorph training/eval hot path on H100: vision tower -> projector -> gather-interleave ->
LLaMA stack -> {lm_head + cross-entropy, vision_head + cosine regression} and the matching
hand-written backward. Mirrors the data flow of the reference's
`MetaMorphLlamaForCausalLM.forward` (metamorph_llama.py:603-660) = `prepare_inputs_labels_for_multimodal`
(metamorph_arch.py:177-425) + `llm_forward` (metamorph_llama.py:285-498); each step cites its lines.

Gradients are delivered to a `GradProvider` (plain buffers owned by the caller) — never through an
autograd graph — so the optimizer can be fused into the backward sweep (engine/trainer.py).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import TYPE_CHECKING, Dict, List, Optional

import torch

from .. import ops
from ..constants import IGNORE_INDEX
from .llama import LayerGrads, StackContext

if TYPE_CHECKING:  # avoid a model <-> engine import cycle
    from ..model.interleave_plan import InterleavePlan


class GradProvider:
    """Where parameter gradients go. Default implementation: lazily allocated standalone buffers."""

    def __init__(self, model):
        self.model = model
        self.buffers: Dict[str, torch.Tensor] = {}
        # True while a later micro-batch of a gradient-accumulation window runs: destinations are added to, not overwritten
        self.accumulate = False

    def get(self, name: str, like: torch.Tensor, fp32: bool = False, zero: bool = False) -> torch.Tensor:
        buf = self.buffers.get(name)
        if buf is None:
            buf = torch.zeros(like.shape, dtype=torch.float32 if fp32 else like.dtype, device=like.device)
            self.buffers[name] = buf
        elif zero and not self.accumulate:
            buf.zero_()
        return buf

    def layer(self, i: int) -> LayerGrads:
        l = self.model.model.layers[i]
        p = f"model.layers.{i}."
        return LayerGrads(
            wqkv=self.get(p + "self_attn.qkv_proj.weight", l.self_attn.qkv_proj.weight),
            wo=self.get(p + "self_attn.o_proj.weight", l.self_attn.o_proj.weight),
            wgu=self.get(p + "mlp.gate_up_proj.weight", l.mlp.gate_up_proj.weight),
            wd=self.get(p + "mlp.down_proj.weight", l.mlp.down_proj.weight),
            ln1=self.get(p + "input_layernorm.weight", l.input_layernorm.weight, fp32=True, zero=True),
            ln2=self.get(p + "post_attention_layernorm.weight", l.post_attention_layernorm.weight, fp32=True, zero=True))

    def layer_done(self, i: int, g: LayerGrads):  # hook for fused optimizers / gradient collectives
        pass

    def group_done(self, group: str, written=None):
        pass


def _param(mod, dotted: str) -> torch.Tensor:
    sub, leaf = dotted.split(".")
    return getattr(getattr(mod, sub), leaf)


@dataclass
class HeadResult:
    loss: torch.Tensor            # fp32 scalar tensor (device)
    loss_language: torch.Tensor   # fp32 [1] device
    loss_image_ar: torch.Tensor   # fp32 [1] device
    d_hidden: Optional[torch.Tensor]
    logits: Optional[torch.Tensor]


class HotPath:
    def __init__(self, model):
        self.m = model  # MetaMorphLlamaForCausalLM
        self.ce_chunk_rows = 2048
        self.skip_unlabelled_rows = True

    # ------------------------------------------------------------------ vision side (A1, A2)
    def encode_images_train(self, images):
        """-> (ar_feats [N*n, H], target feats [N, n, C], projector saved-for-backward)."""
        tower = self.m.get_vision_tower()
        feats = tower(images)                                   # [N, n, C] bf16, no grad (frozen)
        n_img, n_tok, C = feats.shape
        y, saved = self.m.get_model().mm_projector.forward_train(feats.reshape(n_img * n_tok, C))
        return y, feats, saved

    # ------------------------------------------------------------------ heads + losses (A6, A7)
    def heads(self, hidden: torch.Tensor, plan: InterleavePlan, labels: Optional[torch.Tensor],
              targets: Optional[torch.Tensor], want_grad: bool, want_logits: bool,
              grads: Optional[GradProvider], use_vision_ar: bool, vision_coef: float,
              train_lm_head: bool = True, train_vision_head: bool = True) -> HeadResult:
        """hidden: final-norm output [B*T, H]. Reproduces metamorph_llama.py:398-474."""
        m = self.m
        B, T = plan.batch, plan.seq_len
        M, H = hidden.shape
        V = m.lm_head.weight.shape[0]
        dev = hidden.device
        ldv = (V + 7) // 8 * 8
        logits_full = None
        if want_logits:
            buf = torch.empty((M, ldv), dtype=torch.float32, device=dev)
            logits_full = buf[:, :V]
            ops.gemm(hidden, m.lm_head.weight.data, out=logits_full, out_dtype=torch.float32)
        if labels is None:
            z = torch.zeros(1, dtype=torch.float32, device=dev)
            return HeadResult(None, z, z, None, logits_full.view(B, T, V) if want_logits else None)

        # shifted labels: position t predicts label t+1 (metamorph_llama.py:404-405)
        shift = torch.full((B, T), IGNORE_INDEX, dtype=torch.int64)
        shift[:, :-1] = labels[:, 1:]
        n_valid = int((shift != IGNORE_INDEX).sum())
        shift_dev = shift.to(torch.int32).reshape(-1).to(dev, non_blocking=True)

        # image-AR rows: hidden[:, :-1][image_positions[:, 1:] == 1]  (metamorph_llama.py:384-390, 425-432)
        ip = plan.image_positions
        sel = torch.zeros((B, T), dtype=torch.bool)
        sel[:, :-1] = ip[:, 1:] != 0
        sel_rows = torch.nonzero(sel.reshape(-1)).reshape(-1).to(torch.int32)
        n_pred = int(sel_rows.numel())
        have_targets = targets is not None
        n_tgt = int(targets.shape[0] * targets.shape[1]) if have_targets else 0
        # reference: shape mismatch inside F.cosine_similarity is swallowed -> loss_image_ar = loss (:451-455);
        # image_features None -> loss_image_ar = loss (:461-462)
        img_loss_is_lang = (not have_targets) or (n_pred != n_tgt and not (n_pred == 1 or n_tgt == 1))

        loss_lang = torch.zeros(1, dtype=torch.float32, device=dev)
        loss_img = torch.zeros(1, dtype=torch.float32, device=dev)
        ce_scale = 1.0 / max(n_valid, 1)
        ce_grad_mult = 1.0
        if use_vision_ar and img_loss_is_lang:
            ce_grad_mult = 1.0 + vision_coef   # loss = loss + coef * loss

        # Rows whose shifted label is IGNORE_INDEX contribute neither to the loss nor to any gradient, and
        # in training mode the logits are not returned: run lm_head / CE / dgrad / wgrad only on the rows that
        # carry a label (identical loss and gradients; the reference computes all [B,T,V] logits because it
        # returns them, metamorph_llama.py:398-413).
        compact = self.skip_unlabelled_rows and not want_logits and 0 < n_valid < M
        self.last_head_rows = (n_valid if compact else M, M)
        if compact:
            vrows = torch.nonzero(shift.reshape(-1) != IGNORE_INDEX).reshape(-1).to(torch.int32).to(dev, non_blocking=True)
            h_src = ops.gather_rows(hidden, vrows)
            lab_src = shift.reshape(-1)[shift.reshape(-1) != IGNORE_INDEX].to(torch.int32).to(dev, non_blocking=True)
        else:
            h_src, lab_src = hidden, shift_dev
        Ms = h_src.shape[0]
        d_hidden = None
        d_src = None
        acc = bool(want_grad and grads.accumulate)
        written = []
        if want_grad:
            d_src = torch.empty_like(h_src)
            if train_lm_head:
                g_lm = grads.get("lm_head.weight", m.lm_head.weight, fp32=True)
                written.append("lm_head.weight")
        R = self.ce_chunk_rows
        for r0 in range(0, Ms, R):
            r1 = min(Ms, r0 + R)
            hs = h_src[r0:r1]
            if want_logits:
                lg = buf[r0:r1]
            else:
                cbuf = torch.empty((r1 - r0, ldv), dtype=torch.float32, device=dev)
                lg = cbuf
                ops.gemm(hs, m.lm_head.weight.data, out=cbuf[:, :V], out_dtype=torch.float32)
            if want_grad:
                dl = torch.empty((r1 - r0, ldv), dtype=torch.bfloat16, device=dev)
                ops.ce_fwd_bwd(lg, lab_src[r0:r1], V, loss_lang, dlogits=dl, grad_scale=ce_scale * ce_grad_mult)
                ops.gemm(dl[:, :V], m.lm_head.weight.data, b_mn=True, out=d_src[r0:r1])
                if train_lm_head:
                    ops.gemm(dl[:, :V], hs, a_mn=True, b_mn=True, out=g_lm, out_dtype=torch.float32,
                             accumulate=(r0 > 0 or acc))
                del dl
            else:
                ops.ce_fwd_bwd(lg, lab_src[r0:r1], V, loss_lang)
        if want_grad:
            if compact:
                d_hidden = torch.zeros_like(hidden)
                ops.scatter_add_rows_(d_hidden, vrows, d_src)
            else:
                d_hidden = d_src
        if n_valid > 0:
            loss_lang = loss_lang * ce_scale
        else:  # CrossEntropyLoss(mean) over zero valid targets is NaN in the reference
            loss_lang = loss_lang + float("nan")

        if img_loss_is_lang:
            loss_img = loss_lang.clone()
        else:
            vh = m.vision_head
            if n_pred > 0:
                rows = sel_rows.to(dev, non_blocking=True)
                hsel = ops.gather_rows(hidden, rows)
                pred, vh_saved = vh.forward_train(hsel)
                tgt = targets.reshape(-1, targets.shape[-1]).contiguous()
                if n_pred != n_tgt:  # broadcast case (one side has a single row)
                    tgt = tgt.expand(n_pred, -1).contiguous() if n_tgt == 1 else tgt
                dpred = torch.empty_like(pred) if want_grad else None
                if m.normalize_vision:
                    ops.cosine_loss(pred, tgt, loss_sum=loss_img, dpred=dpred,
                                    grad_scale=vision_coef if use_vision_ar else 0.0)
                else:
                    raise NotImplementedError("only normalize_vision=True (cosine loss) is in scope")
                if want_grad and use_vision_ar:
                    vg = None
                    if train_vision_head:
                        vg = {k: grads.get("vision_head." + k, _param(vh, k), fp32=k.endswith("bias"),
                                           zero=k.endswith("bias"))
                              for k in ("0.weight", "0.bias", "2.weight", "2.bias")}
                        written += ["vision_head." + k for k in vg]
                    dh_sel = vh.backward_train(vh_saved, dpred, vg, need_dx=True, accumulate=acc)
                    ops.scatter_add_rows_(d_hidden, rows, dh_sel)
            else:
                # reference: mean over zero rows -> NaN, and NaN != 0 so it is added to the loss
                loss_img = loss_img + float("nan")

        loss = loss_lang.clone()
        if use_vision_ar:
            # reference adds the image loss unless it is exactly 0 (metamorph_llama.py:470-474)
            loss = loss + vision_coef * loss_img
        if want_grad:
            # only the buffers written in THIS pass: a step without answer images gives the vision head no gradient (as
            # in the reference), so a stale buffer of an earlier step must not reach the optimizer
            grads.group_done("heads", written=written)
        return HeadResult(loss.reshape(()), loss_lang, loss_img, d_hidden,
                          logits_full.view(B, T, V) if want_logits else None)

    # ------------------------------------------------------------------ full step pieces
    def forward_backward(self, plan: InterleavePlan, images, grads: Optional[GradProvider],
                         want_grad: bool, want_logits: bool = False, n_save_gu: int = 0,
                         train_embed: bool = True, train_projector: bool = True, train_llm: bool = True,
                         train_lm_head: bool = True, train_vision_head: bool = True):
        """One pass of the hot path over one batch. Returns HeadResult (+ last hidden)."""
        m = self.m
        model = m.get_model()
        dev = model.embed_tokens.weight.device
        B, T = plan.batch, plan.seq_len
        ar_feats, feats, proj_saved = self.encode_images_train(images)
        n_img = feats.shape[0]
        if len(plan.target_image_idx) == n_img:
            targets = feats
        else:
            tidx = torch.tensor(plan.target_image_idx, dtype=torch.int32).to(feats.device, non_blocking=True)
            targets = ops.gather_rows(feats.reshape(n_img, -1).contiguous(), tidx).view(-1, *feats.shape[1:])
        row_map = plan.row_map.reshape(-1).to(dev, non_blocking=True)
        x = ops.interleave_gather(model.embed_tokens.weight.data, ar_feats, row_map)
        pos = plan.position_ids.reshape(-1).to(torch.int32).to(dev, non_blocking=True)
        seqlens = plan.seqlens.to(dev, non_blocking=True)
        flat_segments = None
        if plan.segments is not None:
            flat_segments = [(r * T + off, n) for r, segs in enumerate(plan.segments) for off, n in segs]
        elif plan.padding_side != "right" and bool((plan.seqlens != T).any()):
            # left padding (tokenizer_padding_side == "left", metamorph_arch.py:373-386): sample b occupies the LAST
            # seqlens[b] rows of its batch row -> one segment per sample for the segment-aware attention kernels
            flat_segments = [(b * T + T - int(n), int(n)) for b, n in enumerate(plan.seqlens.tolist()) if int(n) > 0]
            # the reference forwards position_ids=None (metamorph_arch.py:405-406), so HF LlamaModel numbers the rows of
            # the padded batch 0..T-1 (cache_position), pads included; RoPE only sees differences, but the bf16-rounded
            # cos/sin entries are those of the absolute row index
            pos = torch.arange(T, dtype=torch.int32).repeat(B).to(dev, non_blocking=True)
        ctx = StackContext(B=B, T=T, pos=pos, seqlens=seqlens, segments=flat_segments)
        stack = m.stack
        layers = [l.weights() for l in model.layers]
        hidden = stack.forward(layers, model.norm.weight.data, x, ctx, save=want_grad, n_save_gu=n_save_gu)
        del x
        res = self.heads(hidden, plan, plan.labels, targets, want_grad, want_logits, grads,
                         m.use_vision_ar, m.vision_coef, train_lm_head=train_lm_head,
                         train_vision_head=train_vision_head)
        if not want_grad:
            return res, hidden
        acc = grads.accumulate
        g_norm = grads.get("model.norm.weight", model.norm.weight, fp32=True, zero=True) if train_llm else None
        dx = stack.final_norm_backward(model.norm.weight.data, res.d_hidden, ctx, g_norm)
        res.d_hidden = None
        if train_llm:
            grads.group_done("final_norm")
            dx = stack.backward(layers, grads.layer, dx, ctx, on_layer_done=grads.layer_done, accumulate=acc)
        else:   # frozen language model (stage 1): only the dgrad chain runs, no wgrad GEMM / norm-weight reduction
            dx = stack.backward(layers, None, dx, ctx, need_wgrad=False)
        # d(inputs_embeds) -> embedding table + projector output
        d_embed = grads.get("model.embed_tokens.weight", model.embed_tokens.weight, zero=True) if train_embed else None
        d_img = torch.empty_like(ar_feats) if train_projector else None
        if d_img is not None:
            d_img.zero_()  # image rows dropped by truncation / overflow receive no gradient
        ops.interleave_scatter(dx, row_map, d_embed, d_img)
        del dx
        if train_embed:
            grads.group_done("embed")
        if train_projector:
            pj = model.mm_projector
            pg = {k: grads.get("model.mm_projector." + k, _param(pj, k), fp32=k.endswith("bias"),
                               zero=k.endswith("bias"))
                  for k in ("0.weight", "0.bias", "2.weight", "2.bias")}
            pj.backward_train(proj_saved, d_img, pg, need_dx=False, accumulate=acc)
            grads.group_done("projector")
        return res, hidden
