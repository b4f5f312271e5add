"""The weights a decode step streams, bf16 or FP8 (E4M3 groups, DESIGN.md §1).

With weight_dtype="fp8_e4m3" the four matrices of every decoder layer (wqkv, wo, wgu, wd) and lm_head are quantised
into `ops.FP8Weight`s: 128 consecutive k of a row share one power-of-two scale, under the FP8 KV cache's row rule. The
decode step streams them through the FP8 weight-streaming GEMMs, which give the bf16 kernels' bits on W-hat =
float(q) * scale. The norms, embed_tokens, the vision head and the projector stay bf16. The prefill (full-sequence
wgmma GEMMs) dequantises one layer at a time into a bf16 scratch layer and runs unchanged, so every pass of a request
sees exactly W-hat: an FP8 run returns the bits of the bf16 path on a model whose quantised matrices hold W-hat.

Memory: the FP8 copy (1 byte per parameter plus 4 bytes per 128) and one layer of bf16 scratch sit beside the model's
bf16 parameters, which stay: the module is also the training and checkpoint model. The bf16 parameters are only read.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Union

import torch

from .. import ops
from .llama import LayerWeights

_MATRICES = ("wqkv", "wo", "wgu", "wd")


@dataclass
class DecodeWeights:
    """layers: one LayerWeights per decoder layer (FP8: its four matrices are FP8Weights, the norms the model's bf16
    vectors); lm_head: the bf16 parameter or its FP8Weight; scratch: FP8 only, one bf16 layer that `prefill_layer`
    dequantises into."""
    layers: List[LayerWeights]
    lm_head: Union[torch.Tensor, ops.FP8Weight]
    scratch: Optional[LayerWeights] = None

    def prefill_layer(self, i: int) -> LayerWeights:
        """bf16 weights of layer i for the prefill: the model's own (bf16), or W-hat written into the scratch layer
        (FP8; stream ordered, so the previous layer's GEMMs have read the scratch before it is overwritten)."""
        w = self.layers[i]
        if self.scratch is None:
            return w
        for name in _MATRICES:
            ops.weight_dequant_fp8(getattr(w, name), out=getattr(self.scratch, name))
        self.scratch.ln1, self.scratch.ln2 = w.ln1, w.ln2
        return self.scratch


def decode_weights(model, weight_dtype: str = "bf16") -> DecodeWeights:
    """The decode weights of `model` (a MetaMorphLlamaForCausalLM) for weight_dtype 'bf16' (its parameters, nothing
    copied) or 'fp8_e4m3' (quantised now, on the model's device, plus one layer of bf16 scratch)."""
    layers = [l.weights() for l in model.get_model().layers]
    lm_head = model.lm_head.weight.data
    if weight_dtype == "bf16":
        return DecodeWeights(layers, lm_head)
    q = [LayerWeights(w.ln1, *(ops.weight_quant_fp8(getattr(w, n)) for n in ("wqkv", "wo")), w.ln2,
                      *(ops.weight_quant_fp8(getattr(w, n)) for n in ("wgu", "wd"))) for w in layers]
    w0 = layers[0]
    scratch = LayerWeights(w0.ln1, *(torch.empty_like(getattr(w0, n)) for n in ("wqkv", "wo")), w0.ln2,
                           *(torch.empty_like(getattr(w0, n)) for n in ("wgu", "wd")))
    return DecodeWeights(q, ops.weight_quant_fp8(lm_head), scratch)
