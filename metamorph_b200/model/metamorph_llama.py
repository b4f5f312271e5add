"""Drop-in `MetaMorphLlamaForCausalLM` for the H100 hot path.

Mirrors `metamorph/model/language_model/metamorph_llama.py`: `MetaMorphConfig` (:129),
`MetaMorphLlamaModel` (:133), `MetaMorphLlamaForCausalLM` (:223) with `forward` (:603),
`llm_forward` (:285), `greedy_decode` (:502), `generate` (:666) and the side-effect attributes
`loss_language` / `loss_image_ar` (:464-466). Same constructor arguments, same return types
(`CausalLMOutputWithPast`, with `hidden_states` = last hidden state, not a tuple (:492-498)).

Differences a caller can observe, all by design (DESIGN.md):
  * compute runs only on CUDA sm_90a through the C-ABI kernels; CPU tensors raise (no fallback);
  * in training mode `logits` is None unless `config.output_logits_in_training` (the reference
    materialises an 8.4 GB fp32 [B,T,V] tensor each step; the fused head never does);
  * `loss.backward()` triggers the hand-written backward (no autograd graph through the stack);
  * `greedy_decode` keeps a KV cache (the reference forces use_cache=False and re-runs the prefix).
Checkpoints use the reference's HF parameter names (state_dict()/load_state_dict() translate to and
from the fused device layout).
"""
from __future__ import annotations

import json
import os
from typing import List, Optional

import torch
import torch.nn as nn

from .. import ops
from ..constants import EOS_TOKEN_IDS, IGNORE_INDEX, IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID, VISION_FEATURE_DIM
from ..engine.decode import DecodeEngine
from ..engine.logprobs import check_logprobs
from ..engine.hot_path import GradProvider, HotPath
from ..engine.llama import LlamaDims, LlamaStack, StackContext
from ..engine.packing import deinterleave_gate_up, interleave_gate_up
from .layers import FusedDecoderLayer, KernelLinear, MlpGelu, NormWeight, TokenEmbedding
from .metamorph_arch import MetaMorphMetaForCausalLM, MetaMorphMetaModel

try:
    from transformers import AutoConfig, LlamaConfig
    from transformers.modeling_outputs import CausalLMOutputWithPast
except Exception as e:  # pragma: no cover
    raise ImportError("transformers is required for LlamaConfig / CausalLMOutputWithPast") from e


class MetaMorphConfig(LlamaConfig):
    model_type = "metamorph_llama"


def _rope_params(config):
    theta = getattr(config, "rope_theta", None)
    scaling = getattr(config, "rope_scaling", None)
    rp = getattr(config, "rope_parameters", None)
    if isinstance(rp, dict):
        theta = theta or rp.get("rope_theta")
        if rp.get("rope_type", "default") not in (None, "default"):
            scaling = rp
    return float(theta or 10000.0), scaling


def dims_from_config(config) -> LlamaDims:
    theta, scaling = _rope_params(config)
    head_dim = getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads
    return LlamaDims(hidden=config.hidden_size, n_layers=config.num_hidden_layers,
                     n_heads=config.num_attention_heads,
                     n_kv_heads=getattr(config, "num_key_value_heads", None) or config.num_attention_heads,
                     head_dim=head_dim, intermediate=config.intermediate_size, vocab=config.vocab_size,
                     rms_eps=config.rms_norm_eps, rope_theta=theta, rope_scaling=scaling,
                     max_pos=max(8192, int(getattr(config, "tokenizer_model_max_length", 0) or 0) + 1))


class MetaMorphLlamaModel(nn.Module, MetaMorphMetaModel):
    config_class = MetaMorphConfig

    def __init__(self, config, vision_delay_load=True, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.config = config
        d = dims_from_config(config)
        self.embed_tokens = TokenEmbedding(config.vocab_size, d.hidden, dtype, device)
        self.layers = nn.ModuleList([
            FusedDecoderLayer(d.hidden, d.n_heads, d.n_kv_heads, d.head_dim, d.intermediate, dtype, device)
            for _ in range(d.n_layers)])
        self.norm = NormWeight(d.hidden, False, dtype, device)
        self._init_vision(config, vision_delay_load=vision_delay_load, dtype=dtype, device=device)


class _EngineLoss(torch.autograd.Function):
    """Gives the scalar loss a grad_fn so `loss.backward()` (HF-Trainer style loops) works: the
    hand-written backward already ran inside forward(); here the stashed gradients are published to
    `param.grad`, scaled by the upstream gradient."""

    @staticmethod
    def forward(ctx, anchor, loss_value, model):
        ctx.model = model
        return loss_value.clone()

    @staticmethod
    def backward(ctx, g):
        ctx.model._publish_grads(float(g))
        return None, None, None


class MetaMorphLlamaForCausalLM(nn.Module, MetaMorphMetaForCausalLM):
    config_class = MetaMorphConfig

    def __init__(self, config, use_vision_ar=True, vision_head="None", vision_coef=1.0,
                 normalize_vision=False, apply_softmax=False, vision_delay_load=True, full_ar=False,
                 dtype=torch.bfloat16, device=None):
        super().__init__()
        self.config = config
        self.model = MetaMorphLlamaModel(config, vision_delay_load=vision_delay_load, dtype=dtype, device=device)
        self.pretraining_tp = getattr(config, "pretraining_tp", 1)
        self.vocab_size = config.vocab_size
        self.lm_head = KernelLinear(config.hidden_size, config.vocab_size, False, dtype, device)
        self.normalize_vision = normalize_vision
        self.apply_softmax = apply_softmax
        if getattr(config, "normalize_vision", False):
            self.normalize_vision = True
        vision_head = getattr(config, "vision_head_type", vision_head)
        H = config.hidden_size
        if vision_head == "linear":
            self.vision_head = KernelLinear(H, H, True, dtype, device)
        elif vision_head == "mlp":
            self.vision_head = MlpGelu(H, H, VISION_FEATURE_DIM, dtype, device)
        elif vision_head == "mlp2x_gelu":
            raise NotImplementedError("vision_head='mlp2x_gelu' is unused by the reference scripts (out of scope)")
        else:
            self.vision_head = KernelLinear(H, VISION_FEATURE_DIM, True, dtype, device)
        self.use_vision_ar = use_vision_ar
        self.vision_coef = vision_coef
        self.loss_language = 0.0
        self.loss_image_ar = 0.0
        self._stack = None
        self._hot = HotPath(self)
        self._decode = DecodeEngine(self)
        self._grads: Optional[GradProvider] = None
        self.n_save_gu_layers = 0  # how many (last) layers keep gate/up activations instead of recomputing

    # ------------------------------------------------------------------ plumbing
    @property
    def stack(self) -> LlamaStack:
        dev = self.lm_head.weight.device
        if self._stack is None or self._stack.device != dev:
            self._stack = LlamaStack(dims_from_config(self.config), dev)
        return self._stack

    @property
    def device(self):
        return self.lm_head.weight.device

    @property
    def dtype(self):
        return self.lm_head.weight.dtype

    def get_model(self):
        return self.model

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    def resize_token_embeddings(self, new_num_tokens: int):
        old = self.model.embed_tokens.weight.data
        if new_num_tokens == old.shape[0]:
            return self.model.embed_tokens
        for mod in (self.model.embed_tokens, self.lm_head):
            w = mod.weight.data
            nw = torch.empty((new_num_tokens, w.shape[1]), dtype=w.dtype, device=w.device).normal_(0.0, 0.02)
            n = min(new_num_tokens, w.shape[0])
            nw[:n] = w[:n]
            mod.weight = nn.Parameter(nw, requires_grad=mod.weight.requires_grad)
        self.model.embed_tokens.num_embeddings = new_num_tokens
        self.lm_head.out_features = new_num_tokens
        self.config.vocab_size = self.vocab_size = new_num_tokens
        return self.model.embed_tokens

    # ------------------------------------------------------------------ reference-format checkpoints
    def state_dict(self, *args, **kwargs):
        sd = super().state_dict(*args, **kwargs)
        out = {}
        d = dims_from_config(self.config)
        qw, kw = d.n_heads * d.head_dim, d.n_kv_heads * d.head_dim
        for k, v in sd.items():
            if k.endswith("self_attn.qkv_proj.weight"):
                base = k[:-len("qkv_proj.weight")]
                out[base + "q_proj.weight"] = v[:qw]
                out[base + "k_proj.weight"] = v[qw:qw + kw]
                out[base + "v_proj.weight"] = v[qw + kw:]
            elif k.endswith("mlp.gate_up_proj.weight"):
                base = k[:-len("gate_up_proj.weight")]
                g, u = deinterleave_gate_up(v)
                out[base + "gate_proj.weight"] = g
                out[base + "up_proj.weight"] = u
            else:
                out[k] = v
        tower = self.get_vision_tower()
        if tower is not None and tower.is_loaded:
            for k, v in tower.vision_tower._extra_state_tensors.items():
                out["model.vision_tower.vision_tower." + k] = v
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        sd = dict(state_dict)
        fused = {}
        L = len(self.model.layers)
        for i in range(L):
            p = f"model.layers.{i}."
            qk = [p + f"self_attn.{n}_proj.weight" for n in ("q", "k", "v")]
            if all(k in sd for k in qk):
                fused[p + "self_attn.qkv_proj.weight"] = torch.cat([sd.pop(k) for k in qk], 0)
            gk, uk = p + "mlp.gate_proj.weight", p + "mlp.up_proj.weight"
            if gk in sd and uk in sd:
                fused[p + "mlp.gate_up_proj.weight"] = interleave_gate_up(sd.pop(gk), sd.pop(uk))
        sd.update(fused)
        tower = self.get_vision_tower()
        pre = "model.vision_tower.vision_tower."
        if tower is not None and tower.is_loaded:
            for k in [k for k in sd if k.startswith(pre + "head.")]:
                tower.vision_tower._extra_state_tensors[k[len(pre):]] = sd.pop(k)
            tower.vision_tower.invalidate_packed()
        elif tower is not None:
            # delay-loaded tower: keep the checkpoint's tower tensors for the coming load_model() instead of dropping
            # them (a silently random frozen tower would poison every later step)
            stash = {}
            for k in [k for k in sd if k.startswith("model.vision_tower.")]:
                v = sd.pop(k)
                if k.startswith(pre):
                    name = k[len(pre):]
                    stash[name[len("vision_model."):] if name.startswith("vision_model.") else name] = v
            if stash:
                tower.stash_checkpoint_state(stash)
        else:
            for k in [k for k in sd if k.startswith("model.vision_tower.")]:
                sd.pop(k)
        return super().load_state_dict(sd, strict=strict)

    # names whose absence from a checkpoint is legitimate: the dead vision_proj layer, the tower's unused pooling head /
    # post_layernorm, rotary buffers; projector / vision head / tower are absent from a plain LLaMA base checkpoint
    # (stage 1 starts them from their initialisation, as HF `from_pretrained` does with a "newly initialized" warning)
    _OPTIONAL_PREFIXES = ("model.vision_proj.", "model.vision_tower.", "model.mm_projector.", "vision_head.")

    def check_loaded_keys(self, result, what: str):
        """Inspect the IncompatibleKeys of a non-strict load: a LLaMA-core tensor (embeddings, decoder layers, final
        norm, lm_head) that the checkpoint lacks means a naming mismatch that would leave random weights -> raise;
        optional groups and unexpected keys are reported with a warning."""
        import warnings
        missing = list(result.missing_keys)
        core = [k for k in missing if not k.startswith(self._OPTIONAL_PREFIXES)]
        if core:
            raise RuntimeError(f"{what}: {len(core)} core tensors are missing from the checkpoint (would stay randomly "
                               f"initialised), e.g. {core[:4]}")
        opt = sorted({k.split(".")[0] + "." + k.split(".")[1] for k in missing})
        if opt:
            warnings.warn(f"{what}: not in the checkpoint, left at their initialisation: {opt}", stacklevel=2)
        unexpected = [k for k in result.unexpected_keys if "rotary_emb.inv_freq" not in k]
        if unexpected:
            warnings.warn(f"{what}: {len(unexpected)} unexpected tensors ignored, e.g. {unexpected[:4]}", stacklevel=2)
        return result

    def save_pretrained(self, save_directory: str, state_dict=None, max_shard_size="5GB", safe_serialization=True,
                        **kwargs):
        """HF layout, as the reference's `trainer._save` leaves it (train.py:213-222): config.json + (sharded)
        safetensors under the reference's parameter names, streamed tensor by tensor from the fused device layout."""
        from .. import checkpoint
        if state_dict is None and safe_serialization:
            checkpoint.save_model(self, save_directory, max_shard_size=max_shard_size)
            return
        os.makedirs(save_directory, exist_ok=True)
        self.config.save_pretrained(save_directory)
        sd = state_dict if state_dict is not None else self.state_dict()
        torch.save({k: v.detach().cpu() for k, v in sd.items()}, os.path.join(save_directory, "pytorch_model.bin"))

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=torch.bfloat16, device=None, config=None, **kwargs):
        """Loads config + HF-named weights (pytorch_model*.bin / *.safetensors) from a local dir."""
        if config is None:
            with open(os.path.join(path, "config.json")) as f:
                raw = json.load(f)
            raw.pop("model_type", None)
            raw.pop("architectures", None)
            config = MetaMorphConfig(**raw)
        ctor = {k: kwargs.pop(k) for k in ("use_vision_ar", "vision_coef", "vision_head", "normalize_vision",
                                           "apply_softmax", "vision_delay_load", "full_ar") if k in kwargs}
        # the tower is built AFTER the checkpoint has been read, so that its tensors (model.vision_tower.vision_tower.*)
        # are the first source of its weights; only then the pretrained SigLIP (siglip_tower.SiglipVisionTower.load_model)
        load_tower_now = not ctor.get("vision_delay_load", True)
        ctor["vision_delay_load"] = True
        model = cls(config, dtype=torch_dtype, device=device, **ctor)
        from .. import checkpoint
        sd = checkpoint.load_model_state(path)     # index-aware; never reads optimizer-*.safetensors of a checkpoint-N dir
        if not sd:
            raise FileNotFoundError(f"no model weights (*.safetensors / pytorch_model*.bin) under {path}")
        model.check_loaded_keys(model.load_state_dict(sd, strict=False), f"from_pretrained({path})")
        tower = model.get_vision_tower()
        if load_tower_now and tower is not None and not tower.is_loaded:
            tower.load_model(device=device, dtype=torch_dtype)
        return model

    # ------------------------------------------------------------------ gradients for loss.backward()
    def _publish_grads(self, scale: float):
        if self._grads is None:
            return
        named = dict(self.named_parameters())
        for name, buf in self._grads.buffers.items():
            p = named.get(name)
            if p is None or not p.requires_grad:
                continue
            g = buf.to(p.dtype) if buf.dtype != p.dtype else buf.clone()
            if scale != 1.0:
                g.mul_(scale)
            if p.grad is None:
                p.grad = g
            else:
                p.grad.add_(g)

    # ------------------------------------------------------------------ forward
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, images=None, image_sizes=None, return_dict=None,
                cache_position=None, image_embeds=None):
        tower = self.get_vision_tower()
        fused = (inputs_embeds is None and tower is not None and (images is not None or image_embeds is not None)
                 and input_ids is not None and input_ids.shape[1] != 1)
        if not fused:
            image_positions = None
            target = None
            if inputs_embeds is None:
                (input_ids, position_ids, attention_mask, past_key_values, inputs_embeds, labels,
                 image_positions, target) = self.prepare_inputs_labels_for_multimodal(
                    input_ids, position_ids, attention_mask, past_key_values, labels, images, image_sizes,
                    image_embeds)
            return self.llm_forward(input_ids=input_ids, attention_mask=attention_mask,
                                    position_ids=position_ids, past_key_values=past_key_values,
                                    inputs_embeds=inputs_embeds, labels=labels, use_cache=use_cache,
                                    return_dict=return_dict, image_positions=image_positions,
                                    image_features=target)
        if image_embeds is not None:
            raise NotImplementedError("image_embeds on the fused train path: pass images (tower runs on device)")
        if type(images) is list or images.ndim == 5:
            raise NotImplementedError("list / 5-D (anyres) image inputs are unused by the reference scripts")
        plan = self.plan_inputs(input_ids, attention_mask, labels, images.shape[0])
        if labels is None:
            plan.labels = None
        want_grad = (torch.is_grad_enabled() and labels is not None and
                     any(p.requires_grad for p in self.parameters()))
        want_logits = (not want_grad) or bool(getattr(self.config, "output_logits_in_training", False))
        if want_grad and self._grads is None:
            self._grads = GradProvider(self)
        train_embed = self.model.embed_tokens.weight.requires_grad
        res, hidden = self._hot.forward_backward(plan, images.to(self.device), self._grads, want_grad,
                                                 want_logits=want_logits, n_save_gu=self.n_save_gu_layers,
                                                 train_embed=train_embed)
        self._last_plan = plan
        loss = res.loss
        if labels is not None:
            both = torch.cat([res.loss_language.reshape(1), res.loss_image_ar.reshape(1)]).cpu()  # one sync
            self.loss_language, self.loss_image_ar = float(both[0]), float(both[1])
            if want_grad:
                loss = _EngineLoss.apply(self.lm_head.weight, loss, self)
        B, T = plan.batch, plan.seq_len
        return CausalLMOutputWithPast(loss=loss, logits=res.logits, past_key_values=None,
                                      hidden_states=hidden.view(B, T, -1), attentions=None)

    def llm_forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                    inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                    output_hidden_states=None, return_dict=None, cache_position=None,
                    image_positions=None, decoding=False, image_features=None):
        """metamorph_llama.py:285-498 on precomputed `inputs_embeds` (inference / evaluation path:
        no gradients; training goes through forward()). With decoding=True the last position's hidden
        state is replaced by mm_projector(normalize(vision_head(h))) and `loss` carries pred_z."""
        if inputs_embeds is None:
            inputs_embeds = self.model.embed_tokens(input_ids)
        if torch.is_grad_enabled() and labels is not None and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("training from precomputed inputs_embeds is not supported: call "
                                      "forward(input_ids=..., images=...) or metamorph_b200.train")
        B, T, H = inputs_embeds.shape
        dev = inputs_embeds.device
        if attention_mask is not None and attention_mask.shape[-1] == T and attention_mask.dim() == 2:
            am = attention_mask.bool()
            seqlens = am.sum(-1).to(torch.int32)
            if not bool((am == (torch.arange(T, device=am.device)[None] < seqlens[:, None].to(am.device))).all()):
                raise NotImplementedError("only right-padded attention masks are supported")
        else:
            seqlens = torch.full((B,), T, dtype=torch.int32)
        if position_ids is None:
            pos = torch.arange(T, dtype=torch.int32).repeat(B)
        else:
            pos = position_ids.to(torch.int32).expand(B, T).reshape(-1)
        ctx = StackContext(B=B, T=T, pos=pos.to(dev), seqlens=seqlens.to(dev))
        layers = [l.weights() for l in self.model.layers]
        with torch.no_grad():
            hidden = self.stack.forward(layers, self.model.norm.weight.data,
                                        inputs_embeds.reshape(B * T, H).contiguous(), ctx, save=False)
            pred_z = None
            if decoding:
                last = (torch.arange(B, dtype=torch.int32) * T + (T - 1)).to(dev)
                h_last = ops.gather_rows(hidden, last)
                pred_z = self.vision_head(h_last)
                if self.normalize_vision:
                    pred_z = ops.l2norm_rows(pred_z)
                prediction = self.model.mm_projector(pred_z)
                hidden.view(B, T, H)[:, -1, :] = prediction
            V = self.lm_head.weight.shape[0]
            buf = torch.empty((B * T, (V + 7) // 8 * 8), dtype=torch.float32, device=dev)
            ops.gemm(hidden, self.lm_head.weight.data, out=buf[:, :V], out_dtype=torch.float32)
            logits = buf[:, :V].view(B, T, V)
            loss = None
            if labels is not None:
                from ..model.interleave_plan import InterleavePlan
                ip = image_positions if image_positions is not None else torch.zeros((B, T), dtype=torch.int64)
                plan = InterleavePlan(None, labels.cpu(), ip.cpu(), None, None, seqlens.cpu(), [], [], "right")
                plan.row_map = torch.zeros((B, T), dtype=torch.int32)
                res = self._hot.heads(hidden, plan, labels.cpu(),
                                      image_features if image_positions is not None else None,
                                      False, False, None, self.use_vision_ar, self.vision_coef)
                loss = res.loss
                if image_positions is not None:
                    self.loss_language = float(res.loss_language)
                    self.loss_image_ar = float(res.loss_image_ar)
                else:
                    loss = res.loss_language.reshape(())
        return CausalLMOutputWithPast(loss=pred_z if decoding else loss, logits=logits, past_key_values=None,
                                      hidden_states=hidden.view(B, T, H), attentions=None)

    # ------------------------------------------------------------------ decode
    @torch.no_grad()
    def greedy_decode(self, position_ids, attention_mask, inputs_embeds,
                      start_image_token_id=IMAGE_START_TOKEN_ID, end_image_token_id=IMAGE_END_TOKEN_ID,
                      eos_token_id=list(EOS_TOKEN_IDS), do_sample=None, temperature=None, top_p=None,
                      num_beams=None, max_new_tokens=1024, use_cache=None, output_image=False,
                      prompt_lens=None, forced_tokens=None, sampling=None, logprobs=None):
        """metamorph_llama.py:502-597 with a KV cache; accepts a batch (<= 8) of right-padded prompts.
        sampling: None (greedy, as the reference), a SamplingParams (sequence b draws with seed + b) or one per
        sequence (metamorph_b200.engine.sampling). The seeded draw replaces the argmax of metamorph_llama.py:542 and
        nothing else. `do_sample`, `temperature` and `top_p` are accepted and ignored, as the reference's
        greedy_decode ignores them: sampling is asked for with `sampling=` only.
        logprobs: None, or an int n in [0, 20]: the list of TokenLogprobs per sequence (engine/logprobs.py) is appended
        as the last return element; without it the return convention is the reference's."""
        res = self._decode.generate(inputs_embeds, prompt_lens=prompt_lens, max_new_tokens=max_new_tokens,
                                    start_image_token_id=start_image_token_id,
                                    end_image_token_id=end_image_token_id, eos_token_id=eos_token_id,
                                    forced_tokens=forced_tokens, sampling=sampling, logprobs=logprobs)
        ids, imgs = res[0], res[1]
        B = inputs_embeds.shape[0]
        if B == 1:  # reference return convention: [ids] and a [n, 1152] tensor
            img = imgs[0] if imgs[0].shape[0] > 0 else torch.tensor([], dtype=torch.float32, device=inputs_embeds.device)
            out = (ids[:1], img) if output_image else (ids[:1],)
            lps = res[2][:1] if logprobs is not None else None
        else:
            out = (ids, imgs) if output_image else (ids,)
            lps = res[2] if logprobs is not None else None
        if lps is not None:
            return out + (lps,)
        return out if output_image else out[0]

    @torch.no_grad()
    def generate(self, inputs=None, images=None, image_sizes=None, output_image=False,
                 use_customize_greedy=True, image_embeds=None, **kwargs):
        """metamorph_llama.py:666-717. Pass `sampling=SamplingParams(...)` (forwarded to greedy_decode) to sample;
        `do_sample` / `temperature` / `top_p` are dropped on this custom-greedy path, as in the reference."""
        check_logprobs(kwargs.get("logprobs"))
        position_ids = kwargs.pop("position_ids", None)
        attention_mask = kwargs.pop("attention_mask", None)
        prompt_lens = None
        if images is not None or image_embeds is not None:
            (inputs, position_ids, attention_mask, _, inputs_embeds, _, _, _) = \
                self.prepare_inputs_labels_for_multimodal(inputs, position_ids, attention_mask, None, None,
                                                          images, image_sizes=image_sizes, image_embeds=image_embeds)
            prompt_lens = self._last_plan.seqlens
        else:
            inputs_embeds = self.get_model().embed_tokens(inputs.to(self.device))
            if attention_mask is not None:
                prompt_lens = attention_mask.bool().sum(-1).to(torch.int32).cpu()
        if not use_customize_greedy:
            raise NotImplementedError("HF sampling generate() is outside the hot path; use_customize_greedy=True")
        for k in ("do_sample", "temperature", "top_p", "num_beams", "use_cache", "pad_token_id", "bos_token_id"):
            kwargs.pop(k, None)
        return self.greedy_decode(position_ids=position_ids, attention_mask=attention_mask,
                                  inputs_embeds=inputs_embeds, output_image=output_image,
                                  prompt_lens=prompt_lens, **kwargs)


try:
    AutoConfig.register("metamorph_llama", MetaMorphConfig)
except Exception:  # already registered (e.g. the reference package imported in the same process)
    pass
