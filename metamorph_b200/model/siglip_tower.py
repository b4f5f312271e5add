"""SigLIP vision tower on the sm_90a kernels (SURVEY.md rows A1, K1-K7).

Mirrors `metamorph.model.multimodal_encoder.siglip_encoder.SiglipVisionTower` (siglip_encoder.py:62-213)
for the configuration every reference script uses: SigLIP-SO400M/14@384 (hard-coded at :113),
`hidden_states[select_layer]` (pre-post_layernorm), `image_token_reduction="interpolation"`
(27x27 -> sqrt(n) x sqrt(n) bilinear in fp32), optional L2 normalisation, tower frozen.
Other reductions (mlpmixer / concat_interpolation / softmax) are unused by the scripts: out of scope,
they raise NotImplementedError.

The arithmetic spec is HF `SiglipVisionModel` (transformers modeling_siglip.py: embeddings:116,
attention:252, MLP:315, encoder layer:330). Parameter names follow HF's `vision_model.*` keys so
checkpoints load/save unchanged (`model.vision_tower.vision_tower.*`).
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from .. import ops
from ..constants import VISION_FEATURE_DIM
from .layers import KernelLinear, NormWeight

_VALID_PREFIXES = {
    "siglip/CLIP-ViT-SO400M-14-384": "hf-hub:timm/ViT-SO400M-14-SigLIP-384",
    "timm/ViT-SO400M-14-SigLIP-384": "hf-hub:timm/ViT-SO400M-14-SigLIP-384",
    "siglip/CLIP-ViT-SO400M-14": "hf-hub:timm/ViT-SO400M-14-SigLIP",
    "timm/ViT-SO400M-14-SigLIP": "hf-hub:timm/ViT-SO400M-14-SigLIP",
}


def extract_res_interp(model_name: str):
    """Same parsing rules as siglip_encoder.py:34-59 (unknown names raise ValueError)."""
    res = 384 if "384" in model_name else 224
    interp = None
    for prefix, base in _VALID_PREFIXES.items():
        if model_name.startswith(prefix):
            base_model_name = base
            break
    else:
        raise ValueError(f"Unknown vision tower: {model_name}")
    for part in model_name.split("-"):
        if part.startswith("res"):
            res = int(part[3:])
        elif part.startswith("interp"):
            interp = int(part[6:])
    return base_model_name, res, interp


class _PatchEmbedding(nn.Module):
    def __init__(self, width, patch, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(width, 3, patch, patch, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(width, dtype=dtype, device=device))
        with torch.no_grad():
            self.weight.normal_(0.0, 1.0 / math.sqrt(3 * patch * patch))


class _PosEmbedding(nn.Module):
    def __init__(self, n, width, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(n, width, dtype=dtype, device=device))
        with torch.no_grad():
            self.weight.normal_(0.0, 1.0 / math.sqrt(width))


class _Embeddings(nn.Module):
    def __init__(self, width, patch, n_pos, dtype, device):
        super().__init__()
        self.patch_embedding = _PatchEmbedding(width, patch, dtype, device)
        self.position_embedding = _PosEmbedding(n_pos, width, dtype, device)


class _Attn(nn.Module):
    def __init__(self, width, dtype, device):
        super().__init__()
        std = 1.0 / math.sqrt(width)
        self.k_proj = KernelLinear(width, width, True, dtype, device, std)
        self.v_proj = KernelLinear(width, width, True, dtype, device, std)
        self.q_proj = KernelLinear(width, width, True, dtype, device, std)
        self.out_proj = KernelLinear(width, width, True, dtype, device, std)


class _Mlp(nn.Module):
    def __init__(self, width, inter, dtype, device):
        super().__init__()
        self.fc1 = KernelLinear(width, inter, True, dtype, device, 1.0 / math.sqrt(width))
        self.fc2 = KernelLinear(inter, width, True, dtype, device, 1.0 / math.sqrt(inter))


class _EncoderLayer(nn.Module):
    def __init__(self, width, inter, dtype, device):
        super().__init__()
        self.layer_norm1 = NormWeight(width, True, dtype, device)
        self.self_attn = _Attn(width, dtype, device)
        self.layer_norm2 = NormWeight(width, True, dtype, device)
        self.mlp = _Mlp(width, inter, dtype, device)


class _Encoder(nn.Module):
    def __init__(self, n_layers, width, inter, dtype, device):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(width, inter, dtype, device) for _ in range(n_layers)])


class SiglipVisionTransformerParams(nn.Module):
    """HF `SiglipVisionTransformer` parameter tree (embeddings / encoder / post_layernorm)."""

    def __init__(self, width=1152, inter=4304, n_layers=27, n_heads=16, image_size=384, patch=14,
                 eps=1e-6, dtype=torch.bfloat16, device=None):
        super().__init__()
        self.cfg = SimpleNamespace(hidden_size=width, intermediate_size=inter, num_hidden_layers=n_layers,
                                   num_attention_heads=n_heads, image_size=image_size, patch_size=patch,
                                   layer_norm_eps=eps)
        n_pos = (image_size // patch) ** 2
        self.embeddings = _Embeddings(width, patch, n_pos, dtype, device)
        self.encoder = _Encoder(n_layers, width, inter, dtype, device)
        self.post_layernorm = NormWeight(width, True, dtype, device)  # unused by the reference path
        self._extra_state_tensors = {}  # e.g. pooling `head.*` tensors of a loaded checkpoint
        self._packed = None

    @property
    def config(self):
        return self.cfg

    @property
    def dtype(self):
        return self.embeddings.patch_embedding.weight.dtype

    @property
    def device(self):
        return self.embeddings.patch_embedding.weight.device

    def invalidate_packed(self):
        self._packed = None

    def _pack(self):
        c = self.cfg
        pe = self.embeddings.patch_embedding
        kpad = 640
        wpe = torch.zeros(c.hidden_size, kpad, dtype=pe.weight.dtype, device=pe.weight.device)
        wpe[:, :3 * c.patch_size * c.patch_size] = pe.weight.data.reshape(c.hidden_size, -1)
        # Attention runs on the wgmma flash kernel (head_dim 128, csrc/attention_tc.cu): every head of width dh (72 for
        # SO400M) is laid out in a 128-wide slot whose tail is exactly zero — zero rows in the fused QKV weight/bias, zero
        # columns in out_proj — so QK^T, softmax and the visible part of PV are those of the dh-wide heads
        # (HF modeling_siglip.py:229-249), with no pad/unpad pass over the activations.
        heads, W = c.num_attention_heads, c.hidden_size
        dh, dp = W // heads, 128
        assert dh <= dp, "SigLIP head_dim above 128 is not supported by the attention kernel"
        layers = []
        for l in self.encoder.layers:
            a = l.self_attn
            wqkv = torch.zeros(3 * heads * dp, W, dtype=wpe.dtype, device=wpe.device)
            bqkv = torch.zeros(3 * heads * dp, dtype=wpe.dtype, device=wpe.device)
            for j, proj in enumerate((a.q_proj, a.k_proj, a.v_proj)):
                wqkv.view(3, heads, dp, W)[j, :, :dh] = proj.weight.data.view(heads, dh, W)
                bqkv.view(3, heads, dp)[j, :, :dh] = proj.bias.data.view(heads, dh)
            wo = torch.zeros(W, heads * dp, dtype=wpe.dtype, device=wpe.device)
            wo.view(W, heads, dp)[:, :, :dh] = a.out_proj.weight.data.view(W, heads, dh)
            layers.append(dict(wqkv=wqkv, bqkv=bqkv, wo=wo))
        self._packed = dict(wpe=wpe, kpad=kpad, layers=layers, head_slot=dp)

    def forward_features(self, images: torch.Tensor, n_layers_to_run: int) -> torch.Tensor:
        """images [N,3,S,S] -> hidden state after `n_layers_to_run` encoder layers, [N*P, width]."""
        c = self.cfg
        assert c.patch_size == 14, "patch-embed im2col kernel is specialised for 14x14 patches"
        if self._packed is None:
            self._pack()
        pk = self._packed
        n = images.shape[0]
        heads, dh = c.num_attention_heads, c.hidden_size // c.num_attention_heads
        P = (c.image_size // c.patch_size) ** 2
        x = ops.gemm(ops.im2col_patch14(images.contiguous(), pk["kpad"]), pk["wpe"],
                     bias=self.embeddings.patch_embedding.bias.data, epilogue=ops.EPI_BIAS)
        ops.add_pos_emb_(x, self.embeddings.position_embedding.weight.data)
        scale = dh ** -0.5
        Wp = heads * pk["head_slot"]                         # width of the padded q / k / v blocks
        for li in range(n_layers_to_run):
            l, pl = self.encoder.layers[li], pk["layers"][li]
            h = ops.layernorm(x, l.layer_norm1.weight.data, l.layer_norm1.bias.data, c.layer_norm_eps)
            qkv = ops.gemm(h, pl["wqkv"], bias=pl["bqkv"], epilogue=ops.EPI_BIAS)
            attn, _ = ops.attn_fwd(qkv[:, :Wp], qkv[:, Wp:2 * Wp], qkv[:, 2 * Wp:], n, P, heads, heads, pk["head_slot"],
                                   False, scale, need_lse=False)
            x = ops.gemm(attn, pl["wo"], bias=l.self_attn.out_proj.bias.data, resid=x, epilogue=ops.EPI_BIAS_RESID)
            h = ops.layernorm(x, l.layer_norm2.weight.data, l.layer_norm2.bias.data, c.layer_norm_eps)
            h = ops.gemm(h, l.mlp.fc1.weight.data, bias=l.mlp.fc1.bias.data, epilogue=ops.EPI_BIAS_GELU_TANH)
            x = ops.gemm(h, l.mlp.fc2.weight.data, bias=l.mlp.fc2.bias.data, resid=x, epilogue=ops.EPI_BIAS_RESID)
        return x


class SiglipVisionTower(nn.Module):
    def __init__(self, vision_tower_name, args, delay_load=False, tower_dims: dict = None):
        super().__init__()
        base_model_name, res, interp = extract_res_interp(vision_tower_name)
        self.is_loaded = False
        self.select_layer = getattr(args, "mm_vision_select_layer", -2)
        self.select_feature = getattr(args, "mm_vision_select_feature", "patch")
        self.image_token_reduction = getattr(args, "image_token_reduction", "none")
        self.image_token_len = getattr(args, "num_image_tokens", 256)
        self.freeze_vision = getattr(args, "freeze_vision", False)
        self.vision_coef = getattr(args, "vision_coef", 1.0)
        self.normalize_vision = getattr(args, "normalize_vision", False)
        self.apply_softmax = getattr(args, "apply_softmax", False)
        self.vision_tower_name = base_model_name
        self._image_size = res if res is not None else 512
        self._interp_size = interp
        self._tower_dims = dict(tower_dims or getattr(args, "mm_vision_tower_dims", None) or {})
        self.hidden_size = VISION_FEATURE_DIM
        self.image_processor = None
        self._pending_state = None
        self._tower_path = getattr(args, "mm_vision_tower_path", None)
        self._allow_random_init = bool(getattr(args, "mm_vision_tower_random_init", False))
        if not delay_load:
            self.load_model()

    HF_TOWER_NAME = "google/siglip-so400m-patch14-384"   # what the reference downloads (siglip_encoder.py:113)

    def stash_checkpoint_state(self, state_dict):
        """Tower tensors found in a model checkpoint while the tower is still delay-loaded: kept (host side) and applied
        by the next load_model() instead of being dropped."""
        self._pending_state = dict(state_dict)

    def _pretrained_state(self):
        """SigLIP weights as the reference gets them: `AutoModel.from_pretrained("google/siglip-so400m-patch14-384")
        .vision_model` (siglip_encoder.py:113,122). A local directory can be named with MM_SIGLIP_PATH or
        config.mm_vision_tower_path; offline, the hub cache is the only other source. None if nothing is available."""
        import os
        src = os.environ.get("MM_SIGLIP_PATH") or self._tower_path or self.HF_TOWER_NAME
        try:
            from transformers import SiglipVisionModel
            hf = SiglipVisionModel.from_pretrained(src)
        except Exception as e:  # noqa: BLE001 - no network / no cache / not a SigLIP directory
            self._pretrained_error = f"{type(e).__name__}: {str(e).splitlines()[0][:200]}"
            return None
        return {k[len("vision_model."):]: v for k, v in hf.state_dict().items() if k.startswith("vision_model.")}

    def load_model(self, device_map=None, state_dict=None, device=None, dtype=torch.bfloat16, allow_random_init=None):
        """Builds the tower and loads its weights. Sources, in order: the `state_dict` argument; tower tensors of the
        model checkpoint that was loaded while the tower was delay-loaded (`model.vision_tower.vision_tower.*`); the
        pretrained SigLIP the reference downloads (siglip_encoder.py:113). With none of them the call RAISES — a
        silently random frozen tower would make every training run regress against noise — unless random init was
        asked for explicitly (`allow_random_init=True` / `config.mm_vision_tower_random_init`: synthetic benchmarks
        and tests, which then load their own tower tensors through `model.load_state_dict`)."""
        self.vision_model = "siglip"
        dims = dict(width=1152, inter=4304, n_layers=27, n_heads=16, image_size=self._image_size, patch=14)
        dims.update(self._tower_dims)
        self.vision_tower = SiglipVisionTransformerParams(dtype=dtype, device=device, **dims)
        sd, source = state_dict, "state_dict argument"
        if sd is None and self._pending_state is not None:
            sd, source = self._pending_state, "model checkpoint"
        if sd is None:
            sd, source = self._pretrained_state(), "pretrained SigLIP"
        if allow_random_init is None:
            allow_random_init = self._allow_random_init
        if sd is not None:
            own = set(self.vision_tower.state_dict().keys())
            res = self.vision_tower.load_state_dict({k: v for k, v in sd.items() if k in own}, strict=False)
            missing = [k for k in res.missing_keys if not k.startswith(("post_layernorm.", "head."))]
            if missing:
                raise RuntimeError(f"SigLIP tower weights from the {source} lack {len(missing)} tensors, e.g. {missing[:4]}")
            for k, v in sd.items():
                if k.startswith("head."):
                    self.vision_tower._extra_state_tensors[k] = v
            self.vision_tower.invalidate_packed()
            self.weights_source = source
        elif allow_random_init:
            import warnings
            warnings.warn("SiglipVisionTower: RANDOMLY INITIALISED tower (allow_random_init) - valid for synthetic "
                          "benchmarks/tests only", stacklevel=2)
            self.weights_source = "random init"
        else:
            raise RuntimeError(
                "SiglipVisionTower.load_model: no SigLIP weights available - the checkpoint holds no "
                "model.vision_tower.vision_tower.* tensors and the pretrained tower could not be loaded "
                f"({getattr(self, '_pretrained_error', 'unknown')}). Point MM_SIGLIP_PATH / config.mm_vision_tower_path at a "
                f"local copy of {self.HF_TOWER_NAME}, or pass allow_random_init=True for synthetic runs.")
        self._pending_state = None
        self.image_processor = self._make_image_processor(device)
        self.hidden_size = self.vision_tower.cfg.hidden_size
        self.is_loaded = True

    def _make_image_processor(self, device):
        """SURVEY section 8f N1: on a CUDA device the drop-in caller gets the on-GPU pre-processing (bit-exact with the
        HF PIL processor, tests/test_preprocess_gpu.py) behind the same `.preprocess(images, return_tensors)` call; the
        HF CPU processor only when the tower lives on the host (CPU-side plumbing tests)."""
        dev = torch.device(device) if device is not None else self.vision_tower.device
        if dev.type == "cuda":
            from ..preprocess import SiglipGpuImageProcessor
            return SiglipGpuImageProcessor(device=dev)
        try:
            from transformers import SiglipImageProcessor
            proc = SiglipImageProcessor(size={"height": 384, "width": 384})
            proc.crop_size = {"height": 384, "width": 384}
            return proc
        except Exception:  # noqa: BLE001
            return None

    def _n_layers_to_run(self) -> int:
        L = self.vision_tower.cfg.num_hidden_layers
        idx = self.select_layer if self.select_layer >= 0 else (L + 1) + self.select_layer
        if not 0 <= idx <= L:
            raise IndexError(f"mm_vision_select_layer {self.select_layer} out of range for {L} layers")
        return idx

    def feature_select(self, hidden):
        if self.select_feature not in ("patch", "cls_patch"):
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        return hidden

    @torch.no_grad()
    def forward(self, images: torch.Tensor) -> torch.Tensor:
        if not self.freeze_vision and torch.is_grad_enabled() and self.training:
            raise NotImplementedError(
                "metamorph_b200: the SigLIP tower is forward-only (every reference script sets "
                "freeze_vision=True); training the tower is out of scope.")
        in_dtype = images.dtype
        x = images.to(device=self.device, dtype=self.dtype)
        n = x.shape[0]
        hid = self.feature_select(self.vision_tower.forward_features(x, self._n_layers_to_run()))
        P = hid.shape[0] // n
        feats = hid.view(n, P, -1)
        if self.apply_softmax:
            raise NotImplementedError("apply_softmax branch is unused by the reference scripts")
        if P != self.image_token_len:
            if self.image_token_len == -1:
                return torch.zeros_like(feats).to(in_dtype)
            if self.image_token_reduction != "interpolation":
                raise NotImplementedError(
                    f"image_token_reduction={self.image_token_reduction!r}: only 'interpolation' is in scope")
            side = int(math.sqrt(self.image_token_len))
            feats = ops.bilinear_l2norm(feats, side, normalize=self.normalize_vision)
        elif self.normalize_vision:
            feats = ops.l2norm_rows(feats.reshape(n * P, -1)).view(n, P, -1)
        return feats.to(in_dtype) if in_dtype in (torch.bfloat16,) else feats

    @property
    def dtype(self):
        return self.vision_tower.dtype

    @property
    def device(self):
        return self.vision_tower.device

    @property
    def config(self):
        return self.vision_tower.config if self.is_loaded else SimpleNamespace(hidden_size=VISION_FEATURE_DIM)

    @property
    def num_patches_per_side(self):
        return self._image_size // 14

    @property
    def num_patches(self):
        return (self._image_size // 14) ** 2


def build_vision_tower(vision_tower_cfg, **kwargs):
    """multimodal_encoder/builder.py:11-14: always a SiglipVisionTower."""
    name = getattr(vision_tower_cfg, "mm_vision_tower", getattr(vision_tower_cfg, "vision_tower", None))
    return SiglipVisionTower(name, args=vision_tower_cfg, **kwargs)
