"""Parameter-holding modules of the drop-in model. They carry the reference's parameter names
(SURVEY.md §8b state-dict contract) but compute ONLY through the sm_90a kernels — there is no
eager/CPU fallback: calling them with CPU tensors raises (see _lib.require_cuda)."""
from __future__ import annotations

import math
import re

import torch
import torch.nn as nn

from .. import ops


class KernelLinear(nn.Module):
    """nn.Linear-shaped parameter holder; forward = wgmma GEMM with a fused bias epilogue."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, dtype=torch.bfloat16,
                 device=None, std: float = 0.02):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.empty(out_features, dtype=dtype, device=device)) if bias else None
        self._std = std
        self.reset_parameters()

    def reset_parameters(self):
        with torch.no_grad():
            self.weight.normal_(0.0, self._std)
            if self.bias is not None:
                self.bias.zero_()

    def forward(self, x: torch.Tensor, epilogue: int = None) -> torch.Tensor:
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        if self.bias is not None:
            y = ops.gemm(x2, self.weight, bias=self.bias, epilogue=ops.EPI_BIAS if epilogue is None else epilogue)
        else:
            y = ops.gemm(x2, self.weight)
        return y.view(*shp[:-1], self.out_features)


class NormWeight(nn.Module):
    def __init__(self, dim: int, bias: bool = False, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(dim, dtype=dtype, device=device)) if bias else None


class TokenEmbedding(nn.Module):
    def __init__(self, vocab: int, dim: int, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.num_embeddings, self.embedding_dim = vocab, dim
        self.weight = nn.Parameter(torch.empty(vocab, dim, dtype=dtype, device=device))
        with torch.no_grad():
            self.weight.normal_(0.0, 0.02)

    def forward(self, ids: torch.Tensor) -> torch.Tensor:
        """embed_tokens(ids) through the gather kernel (metamorph_arch.py:298, metamorph_llama.py:544)."""
        flat = ids.reshape(-1).to(torch.int32)
        out = ops.interleave_gather(self.weight, None, flat.contiguous())
        return out.view(*ids.shape, self.embedding_dim)


class MlpGelu(nn.Module):
    """`mlp2x_gelu` projector / `mlp` vision head: Linear -> GELU(erf) -> Linear, parameter names
    '0.*' and '2.*' as in nn.Sequential (multimodal_projector/builder.py:52-59,
    metamorph_llama.py:252-256)."""

    def __init__(self, d_in: int, d_hidden: int, d_out: int, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.add_module("0", KernelLinear(d_in, d_hidden, True, dtype, device))
        self.add_module("2", KernelLinear(d_hidden, d_out, True, dtype, device))

    @property
    def fc1(self) -> KernelLinear:
        return getattr(self, "0")

    @property
    def fc2(self) -> KernelLinear:
        return getattr(self, "2")

    def __getitem__(self, i: int):
        return getattr(self, str(i))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = self.fc1(x, epilogue=ops.EPI_BIAS_GELU_ERF)
        return self.fc2(h)

    # training path: keeps the pre-activation for the GELU backward
    def forward_train(self, x2: torch.Tensor):
        z = ops.gemm(x2, self.fc1.weight, bias=self.fc1.bias, epilogue=ops.EPI_BIAS)
        a = ops.gelu(z)
        y = ops.gemm(a, self.fc2.weight, bias=self.fc2.bias, epilogue=ops.EPI_BIAS)
        return y, (x2, z, a)

    def backward_train(self, saved, dy: torch.Tensor, grads, need_dx: bool, accumulate: bool = False):
        """grads: dict name -> tensor for '0.weight','0.bias','2.weight','2.bias' (bias fp32, zeroed by the caller unless
        accumulating), or None when these parameters are frozen (only dx is produced)."""
        x2, z, a = saved
        if grads is not None:
            ops.gemm(dy, a, a_mn=True, b_mn=True, out=grads["2.weight"], accumulate=accumulate)
            ops.colsum_accum(dy, grads["2.bias"])
        da = ops.gemm(dy, self.fc2.weight, b_mn=True)
        dz = ops.gelu_bwd(z, da)
        if grads is not None:
            ops.gemm(dz, x2, a_mn=True, b_mn=True, out=grads["0.weight"], accumulate=accumulate)
            ops.colsum_accum(dz, grads["0.bias"])
        if need_dx:
            return ops.gemm(dz, self.fc1.weight, b_mn=True)
        return None


class FusedAttentionParams(nn.Module):
    def __init__(self, hidden, n_heads, n_kv_heads, head_dim, dtype, device):
        super().__init__()
        self.qkv_proj = KernelLinear(hidden, (n_heads + 2 * n_kv_heads) * head_dim, False, dtype, device)
        self.o_proj = KernelLinear(n_heads * head_dim, hidden, False, dtype, device)


class FusedMlpParams(nn.Module):
    def __init__(self, hidden, intermediate, dtype, device):
        super().__init__()
        self.gate_up_proj = KernelLinear(hidden, 2 * intermediate, False, dtype, device)
        self.down_proj = KernelLinear(intermediate, hidden, False, dtype, device)


class FusedDecoderLayer(nn.Module):
    """Parameters of one LLaMA decoder layer in the fused layout (engine/llama.py)."""

    def __init__(self, hidden, n_heads, n_kv_heads, head_dim, intermediate, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.input_layernorm = NormWeight(hidden, False, dtype, device)
        self.self_attn = FusedAttentionParams(hidden, n_heads, n_kv_heads, head_dim, dtype, device)
        self.post_attention_layernorm = NormWeight(hidden, False, dtype, device)
        self.mlp = FusedMlpParams(hidden, intermediate, dtype, device)

    def weights(self):
        from ..engine.llama import LayerWeights
        return LayerWeights(self.input_layernorm.weight.data, self.self_attn.qkv_proj.weight.data,
                            self.self_attn.o_proj.weight.data, self.post_attention_layernorm.weight.data,
                            self.mlp.gate_up_proj.weight.data, self.mlp.down_proj.weight.data)
