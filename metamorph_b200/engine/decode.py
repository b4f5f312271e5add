"""KV-cached greedy (or seeded sampled) decode emitting text tokens and continuous visual-token embeddings.

Semantics = the reference's `greedy_decode` (metamorph_llama.py:502-597) including its quirks (EOS
test on the logits of the overwritten hidden state while in image mode; the image-token counter is
only reset by <image_end>), but (a) with a KV cache instead of re-running the growing prefix
(F6 in SURVEY.md), (b) batched: every sequence carries its own mode state machine on the device,
(c) without per-step host syncs: the loop polls `finished` once every `poll_every` steps.
"""
from __future__ import annotations

from typing import Optional, Sequence, Union

import torch

from .. import ops
from ..constants import EOS_TOKEN_IDS, IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
from .decode_step import decode_heads, decoder_stack_step
from .fp8_weights import decode_weights
from .llama import FP8KVStore, StackContext
from .logprobs import LogprobBuffers, check_logprobs
from .sampling import SamplingArrays, SamplingParams, per_sequence


def check_forced_tokens(forced_tokens: Optional[torch.Tensor], embed_rows: int) -> None:
    """A forced id becomes a row index into the embedding table (the next-input gather reads row `id` unchecked), so
    every entry must lie in [-1, embed_rows); -1 is free-running. Raises ValueError on the host, before any device
    work."""
    if forced_tokens is None or forced_tokens.numel() == 0:
        return
    if forced_tokens.dtype.is_floating_point or forced_tokens.dtype == torch.bool:
        raise ValueError(f"forced_tokens must hold integer token ids (got {forced_tokens.dtype})")
    lo, hi = int(forced_tokens.min()), int(forced_tokens.max())
    if lo < -1 or hi >= embed_rows:
        raise ValueError(f"forced_tokens must lie in [-1, {embed_rows}): -1 is free-running and an id indexes the "
                         f"embedding table's {embed_rows} rows (got min {lo}, max {hi})")


KV_CACHE_DTYPES = ("bf16", "fp8_e4m3")


def check_kv_cache_dtype(kv_cache_dtype) -> None:
    """'bf16' (the default cache) or 'fp8_e4m3' (E4M3 rows with one power-of-two scale each, DESIGN.md §1). Raises
    ValueError on the host, before any device work."""
    if not isinstance(kv_cache_dtype, str) or kv_cache_dtype not in KV_CACHE_DTYPES:
        raise ValueError(f"kv_cache_dtype must be one of {KV_CACHE_DTYPES} (got {kv_cache_dtype!r})")


WEIGHT_DTYPES = ("bf16", "fp8_e4m3")


def check_weight_dtype(weight_dtype) -> None:
    """'bf16' (the model's parameters) or 'fp8_e4m3' (the decode step streams E4M3 weight groups with one power-of-two
    scale per 128 k, DESIGN.md §1). Raises ValueError on the host, before any device work."""
    if not isinstance(weight_dtype, str) or weight_dtype not in WEIGHT_DTYPES:
        raise ValueError(f"weight_dtype must be one of {WEIGHT_DTYPES} (got {weight_dtype!r})")


def alloc_kv_cache(kv_cache_dtype: str, shape, dev):
    """(kc, vc, scales) for a cache of `shape` [..., dh]: bf16 and scales None, or uint8 E4M3 bytes and (ks, vs) fp32
    [...] (one scale per row). Zero-filled."""
    if kv_cache_dtype == "bf16":
        kc = torch.zeros(shape, dtype=torch.bfloat16, device=dev)
        return kc, torch.zeros_like(kc), None
    kc = torch.zeros(shape, dtype=torch.uint8, device=dev)
    ks = torch.zeros(shape[:-1], dtype=torch.float32, device=dev)
    return kc, torch.zeros_like(kc), (ks, torch.zeros_like(ks))


class DecodeEngine:
    def __init__(self, model):
        self.m = model
        self.use_cuda_graph = True

    @torch.no_grad()
    def generate(self, inputs_embeds: torch.Tensor, prompt_lens: Optional[torch.Tensor] = None,
                 max_new_tokens: int = 1024, start_image_token_id: int = IMAGE_START_TOKEN_ID,
                 end_image_token_id: int = IMAGE_END_TOKEN_ID, eos_token_id=EOS_TOKEN_IDS,
                 forced_tokens: Optional[torch.Tensor] = None, poll_every: int = 16,
                 max_steps: Optional[int] = None,
                 sampling: Union[None, SamplingParams, Sequence[SamplingParams]] = None,
                 logprobs: Optional[int] = None, kv_cache_dtype: str = "bf16", weight_dtype: str = "bf16"):
        """inputs_embeds [B, P, H] (right-padded to P; prompt_lens[b] valid rows). B <= 128.
        sampling: None (greedy), one SamplingParams (sequence b draws with seed + b) or one per sequence. The draw
        replaces the argmax only: image mode, the EOS test on the drawn token and forced tokens are unchanged. When
        every temperature is 0 this is the greedy path, kernel for kernel.
        forced_tokens: None or [B, n] integer ids indexed by each sequence's own step count. An entry >= 0 replaces the
        step's token, -1 is free-running, and so is every step past column n - 1: a schedule shorter than the run ends
        and the sequence free-runs from there, exactly as a request served by `ContinuousBatcher` does. Ids outside
        [-1, embedding rows) raise ValueError before any device work.
        logprobs: None, or an int n in [0, 20]: every sequence also reports, for each id it emits, that id's
        log-probability under the step's raw distribution and the n most likely ids with theirs (engine/logprobs.py).
        Anything else raises ValueError before any device work. Ids and embeddings do not change.
        kv_cache_dtype: 'bf16' (default) or 'fp8_e4m3': the KV cache holds E4M3 rows with one power-of-two scale each
        (half the bytes), and every attention, prefill and decode, reads the values the cache holds. Right-padded
        prompts quantise their pad rows like any other row; nothing reads them. Anything else raises ValueError before
        any device work.
        weight_dtype: 'bf16' (default) or 'fp8_e4m3': the call first quantises the decoder-layer matrices and lm_head
        into E4M3 groups (engine/fp8_weights.py; about 1.03 bytes per parameter, beside the bf16 parameters, plus one
        layer of bf16 scratch) and the decode steps stream those, about half the bytes. The prefill dequantises them
        layer by layer, so the run returns the bits of the bf16 path on a model holding W-hat. The quantisation time is
        `last_timing['quant_ms']`, outside 'decode_ms'. Anything else raises ValueError before any device work.
        Returns (ids list per sequence (int32 tensors), image_embeds list per sequence [n, C]), and with logprobs a
        third element: one TokenLogprobs per sequence, entry k belonging to ids[k]."""
        check_logprobs(logprobs)
        check_kv_cache_dtype(kv_cache_dtype)
        check_weight_dtype(weight_dtype)
        B, P, H = inputs_embeds.shape
        assert B <= 128, f"decode batch is limited to 128 sequences per step (got {B}): the weight-streaming GEMM " \
                         "serves at most 128 batch rows"
        m = self.m
        model = m.get_model()
        if forced_tokens is not None and (forced_tokens.dim() != 2 or forced_tokens.shape[0] != B):
            raise ValueError(f"forced_tokens must be [B={B}, n] (got {tuple(forced_tokens.shape)})")
        check_forced_tokens(forced_tokens, model.embed_tokens.weight.shape[0])
        stack = m.stack
        d = stack.dims
        dev = inputs_embeds.device
        params = per_sequence(sampling, B)
        Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
        L = len(model.layers)
        ntok = m.get_vision_tower().image_token_len if m.get_vision_tower() is not None else 0
        C = m.vision_head.fc2.out_features
        steps_cap = max_new_tokens + 1 if max_steps is None else max_steps
        Tmax = P + steps_cap + 1
        stack.ensure_positions(Tmax + 1)
        if prompt_lens is None:
            prompt_lens = torch.full((B,), P, dtype=torch.int32)
        prompt_lens_dev = prompt_lens.to(dev, dtype=torch.int32)
        eos = list(eos_token_id) if isinstance(eos_token_id, (list, tuple)) else [eos_token_id]
        if len(eos) > 2:
            raise NotImplementedError("at most two EOS ids (the reference's default is [128001, 128009])")
        # an empty list never matches (token ids are >= 0), like `next_token.item() in []` (metamorph_llama.py:583)
        eos0 = eos[0] if eos else -1
        eos1 = eos[1] if len(eos) > 1 else eos0

        qev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        qev[0].record()
        dw = decode_weights(m, weight_dtype)
        qev[1].record()
        kc, vc, scales = alloc_kv_cache(kv_cache_dtype, (L, B, Hkv, Tmax, dh), dev)

        # ---- prefill: full-sequence kernels, K/V captured into the cache
        pos = torch.arange(P, dtype=torch.int32).repeat(B).to(dev)
        ctx = StackContext(B=B, T=P, pos=pos, seqlens=prompt_lens_dev)
        layers = dw.layers
        x = inputs_embeds.reshape(B * P, H).contiguous()
        for i in range(L):
            w = dw.prefill_layer(i)
            if scales is not None:
                x = stack.layer_forward(w, x, ctx, save=True, save_gu=False,
                                        kv=FP8KVStore(kc[i], vc[i], scales[0][i], scales[1][i]))
                ctx.saved.pop()
                continue
            x = stack.layer_forward(w, x, ctx, save=True, save_gu=False)
            s = ctx.saved.pop()
            ops.kv_prefill(s.qkv, kc[i], vc[i], B, P, Hq, Hkv, dh)
            del s
        last_rows = (torch.arange(B, dtype=torch.int32) * P + (prompt_lens.to(torch.int32) - 1)).to(dev)
        h_last = ops.gather_rows(x, last_rows)                      # [B, H] pre-final-norm
        del x

        st = {k: torch.zeros(B, dtype=torch.int32, device=dev) for k in
              ("in_image_mode", "total_image_tokens", "total_output", "finished", "n_ids", "n_img",
               "append_kind", "next_token")}
        st["pos"] = prompt_lens_dev.clone()
        max_img = max(1, (steps_cap // max(ntok, 1) + 1) * max(ntok, 1))
        st["ids_out"] = torch.full((B, steps_cap + 1), -1, dtype=torch.int32, device=dev)
        img_out = torch.zeros((B, max_img, C), dtype=torch.bfloat16, device=dev)
        forced = forced_tokens.to(dev, dtype=torch.int32).contiguous() if forced_tokens is not None else None
        samp = SamplingArrays.of(params, dev) if params is not None else None
        xin = torch.empty((B, H), dtype=torch.bfloat16, device=dev)
        V = m.lm_head.weight.shape[0]
        logits = torch.empty((B, (V + 7) // 8 * 8), dtype=torch.float32, device=dev)
        lpb = None
        if logprobs is not None:
            lpb = LogprobBuffers(B, st["ids_out"].shape[1], dev)
            lpb.n_top.fill_(int(logprobs))

        def heads_and_state(h_pre_norm, step):
            tok, pred_z, prediction = decode_heads(m, h_pre_norm, st["in_image_mode"], logits, V, samp,
                                                   st["total_output"], dw.lm_head)
            ops.decode_state_step(st, tok, forced, step, B, ntok, max_new_tokens, start_image_token_id,
                                  end_image_token_id, eos0, eos1, pred_z, img_out)
            if lpb is not None:
                lpb.launch(logits, V, st)
            ops.decode_next_input(st["append_kind"], st["next_token"], model.embed_tokens.weight.data,
                                  prediction, xin)

        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()                                   # prefill done (enqueued) -> decode steps start
        heads_and_state(h_last, 0)

        def one_step_body():
            # position of the token being fed = pos - 1 (the state step already advanced pos)
            return decoder_stack_step(layers, xin, kc, vc, st["pos"] - 1, stack, scales=scales)

        # One captured CUDA graph is replayed for every step (launch-bound inner loop): all per-step state,
        # including the index into the forced-token schedule, lives in device memory.
        step = 1
        graph = None
        if self.use_cuda_graph and steps_cap > 2:
            heads_and_state(one_step_body(), 1)              # eager warm-up step (sets kernel attributes)
            step = 2
            ev[1].record()
            try:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    heads_and_state(one_step_body(), 0)
                graph = g
            except Exception:  # noqa: BLE001 - capture unsupported: stay on stream launches
                graph = None
                torch.cuda.synchronize()
            ev[2].record()
        else:
            ev[1].record()
            ev[2].record()
        while step < steps_cap:
            if step % poll_every == 0 and bool(st["finished"].all()):
                break
            if graph is not None:
                graph.replay()
            else:
                heads_and_state(one_step_body(), step)
            step += 1

        ev[3].record()
        n_ids = st["n_ids"].cpu().tolist()
        n_img = st["n_img"].cpu().tolist()
        ids_cpu = st["ids_out"]
        out_ids = [ids_cpu[b, :n_ids[b]].clone() for b in range(B)]
        out_img = [img_out[b, :n_img[b]].clone() for b in range(B)]
        self.last_steps = step
        # device time of the decode steps (graph capture is a one-off host-side cost, reported separately)
        self.last_timing = {"steps": step, "decode_ms": ev[0].elapsed_time(ev[1]) + ev[2].elapsed_time(ev[3]),
                            "capture_ms": ev[1].elapsed_time(ev[2]), "cuda_graph": graph is not None,
                            "quant_ms": qev[0].elapsed_time(qev[1])}
        if lpb is not None:
            return out_ids, out_img, [lpb.take(b, 0, n_ids[b], int(logprobs)) for b in range(B)]
        return out_ids, out_img
