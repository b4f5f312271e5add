"""`load_pretrained_model` (metamorph/model/builder.py:13-144): the full-model branch (:86-92, :120-142) and the
projector-only branch (:73-84: base LLaMA weights + the stage-1 `mm_projector.bin` of `model_path`).
LoRA / 4-bit / 8-bit branches are unused by the reference scripts: out of scope."""
from __future__ import annotations

import torch

from ..constants import DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IMAGE_PATCH_TOKEN
from .metamorph_llama import MetaMorphLlamaForCausalLM


def load_pretrained_model(model_path, model_base, model_name, load_8bit=False, load_4bit=False,
                          device_map="auto", device="cuda", use_flash_attn=False, torch_dtype=torch.float16,
                          **kwargs):
    if load_8bit or load_4bit:
        raise NotImplementedError("quantised loading is out of scope for the H100 hot path")
    if "lora" in model_name.lower():
        raise NotImplementedError("LoRA checkpoints are out of scope (unused by the scripts)")
    if torch_dtype != torch.bfloat16:
        # the kernels compute in bf16 (fp32 accumulate); fp16 checkpoints are converted on load
        torch_dtype = torch.bfloat16
    from transformers import AutoTokenizer
    if model_base is not None:
        # "this may be mm projector only" (builder.py:73-84): language model from model_base, config and the stage-1
        # projector weights from model_path
        import json
        import os
        from .. import checkpoint
        from .metamorph_llama import MetaMorphConfig
        tokenizer = AutoTokenizer.from_pretrained(model_base, use_fast=False)
        with open(os.path.join(model_path, "config.json")) as fh:
            raw = json.load(fh)
        raw.pop("model_type", None)
        raw.pop("architectures", None)
        model = MetaMorphLlamaForCausalLM.from_pretrained(model_base, torch_dtype=torch_dtype, device=device,
                                                          config=MetaMorphConfig(**raw), vision_delay_load=False,
                                                          **kwargs)
        checkpoint.load_mm_projector(model, model_path)
    else:
        tokenizer = AutoTokenizer.from_pretrained(model_path, use_fast=False)
        model = MetaMorphLlamaForCausalLM.from_pretrained(model_path, torch_dtype=torch_dtype, device=device,
                                                          vision_delay_load=False, **kwargs)
    mm_use_im_start_end = getattr(model.config, "mm_use_im_start_end", False)
    mm_use_im_patch_token = getattr(model.config, "mm_use_im_patch_token", True)
    if mm_use_im_patch_token:
        tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN], special_tokens=True)
    if mm_use_im_start_end:
        tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)
    model.resize_token_embeddings(len(tokenizer))
    vision_tower = model.get_vision_tower()
    if not vision_tower.is_loaded:
        vision_tower.load_model(device=device, dtype=torch_dtype)
    image_processor = vision_tower.image_processor
    context_len = getattr(model.config, "max_sequence_length", 2048)
    return tokenizer, model, image_processor, context_len
