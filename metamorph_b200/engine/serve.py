"""Continuous-batching decode server (SURVEY.md §8f row N4): the per-sequence text / image state machine of
`greedy_decode` (metamorph_llama.py:502-597) for a stream of requests instead of one batch.

The reference serves one request at a time (inference/demo.py:117-179: `generate` -> visualise the returned image
embeddings). Here up to `max_slots` (<= 128) requests share every weight-streaming decode step:
  * each batch slot owns a KV-cache region, its mode / counters / position on the device and its own output limit;
  * a queued request is admitted into a free slot BETWEEN steps: its first P-1 prompt positions are prefilled with the
    full-sequence kernels (wgmma GEMMs + flash attention) straight into the slot's cache region, and the last prompt
    position is fed through the ordinary decode step — no special first-token path;
  * the step itself (decoder stack + heads + argmax + state machine + next-input gather) is ONE captured CUDA graph
    replayed for all slots, exactly the kernels of DecodeEngine; idle / finished slots are frozen by the device state;
  * a request may sample (`submit(..., sampling=SamplingParams(...))`): its slot's parameters and seed are written on
    admission and the step counter is the slot's `total_output`. While a sampled request is in flight the step runs a
    second graph, captured the first time it is needed, whose seeded draw replaces the argmax; a temperature-0 slot
    gets the argmax token from it, so the graph choice never changes a greedy request's output;
  * the host polls the tiny state arrays every `poll_every` steps, hands out finished requests, streams the new text
    ids / visual embeddings of running ones (`run()` yields them), and refills the freed slots.
With `kv_pool_tokens` set, the slots share a paged KV cache instead of each reserving `max_context` positions: one pool
of fixed-size blocks per layer and a device block table [max_slots, ceil(max_context / kv_block_size)] (see
KVBlockAllocator for the reservation and reclaim rules). The paged attention kernel gives the dense one's bits, so a
request's output does not depend on the cache layout or on which blocks it received.
A paged server also caches prompt prefixes: `h = cache_prefix(prefix)` prefills the prefix's whole blocks once,
`submit(suffix, prefix=h)` shares them and prefills only the prefix tail and the suffix (attention reads the shared
keys through the block table, `ops.attn_fwd_paged`), and `drop_prefix(h)` lets the blocks go once no request uses them.
The request returns the bits of the whole prompt submitted without a prefix.
A request may ask for token log-probabilities (`submit(..., logprobs=n)`): while one is in flight the step runs a graph
that adds the logprob kernel after the state step (captured the first time it is needed, for the greedy and the sampled
step alike); its slot's `n_top` is written on admission, -1 for every request that did not ask. The kernel only reads
the logits and the state, so ids and embeddings keep their bits, and the reported bits do not depend on the neighbours.
Every request's output equals what `greedy_decode` produces for it alone (tests/test_decode_gpu.py), a forced schedule
shorter than the run included: in both, the request free-runs once its schedule ends (tests/test_serve_lifecycle_gpu.py).
"""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass, field
from typing import Deque, Dict, List, Optional, Tuple

import torch

from .. import ops
from ..constants import EOS_TOKEN_IDS, IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
from .decode import check_forced_tokens
from .decode_step import decode_heads, decoder_stack_step
from .llama import PagedPrefill, StackContext
from .logprobs import LogprobBuffers, TokenLogprobs, cat as cat_logprobs, check_logprobs
from .sampling import SamplingArrays, SamplingParams


class PrefixHandle:
    """A prompt prefix cached by one paged `ContinuousBatcher` (`cache_prefix`). Its first `shared_len` positions (whole
    KV blocks) are prefilled once and shared by every request submitted with `prefix=` this handle; the `length -
    shared_len` tail rows are kept as embeddings and prefilled with each request's suffix."""

    def __init__(self, server, pid: int, length: int, shared_len: int, tail: torch.Tensor):
        self.server, self.pid, self.length, self.shared_len, self.tail = server, pid, length, shared_len, tail

    def __repr__(self):
        return f"PrefixHandle(pid={self.pid}, length={self.length}, shared_len={self.shared_len})"


@dataclass
class _Request:
    rid: int
    embeds: torch.Tensor                 # [P - start, H] bf16 (device): the prompt rows from position `start` on
    max_new_tokens: int
    forced: Optional[torch.Tensor]       # [n] int32 (host) or None
    sampling: Optional[SamplingParams] = None
    prefix: Optional[PrefixHandle] = None   # positions 0 .. start-1 are this prefix's shared blocks (start = shared_len)
    logprobs: Optional[int] = None       # alternatives reported per emitted id, None = no log-probabilities
    slot: int = -1
    sent_ids: int = 0
    sent_img: int = 0
    ids: List[torch.Tensor] = field(default_factory=list)
    img: List[torch.Tensor] = field(default_factory=list)
    lps: List[TokenLogprobs] = field(default_factory=list)


class KVBlockAllocator:
    """Host-side bookkeeping of the paged KV cache: which pool blocks are free and which request owns which.

    Blocks 0 .. num_blocks-1 are handed out; block `scratch` (= num_blocks) never is. Every table entry of an idle
    slot, and every entry past a request's reservation, points at the scratch block: idle and finished slots still
    run every step and append K/V at their frozen position, and those writes must land where no request reads.

    Reservation, not growth: a request gets on admission every block it can write. With P prompt positions and
    max_new_tokens n, the prefill writes positions 0 .. P-2 and the decode state machine (decode_state_kernel) feeds
    the token at pos-1, starting at pos = P and advancing pos once per step for at most n+1 steps; a finished slot
    keeps rewriting its frozen position pos-1 = P+n until the host reclaims it. So positions 0 .. P+n are written and
    read: ceil((P + n + 1) / block_size) blocks, never more (an early EOS only freezes the slot sooner).

    Shared prefix blocks: `pin` takes the blocks of a cached prefix, held by the prefix handle and by every queued and
    running request that names it (`ref`); they return to the free list when the last of these lets go. A request on a
    prefix of Ls positions (a multiple of block_size) reserves only its private blocks, reservation(P - Ls, n): positions
    Ls .. P+n, the only ones it writes."""

    def __init__(self, num_blocks: int, block_size: int):
        check_kv_block_size(block_size)
        if num_blocks < 1:
            raise ValueError(f"a paged KV cache needs at least one block (num_blocks={num_blocks})")
        self.num_blocks, self.block_size = num_blocks, block_size
        self.scratch = num_blocks
        self.free: List[int] = list(range(num_blocks))   # handed out from the front, returned to the back
        self.owned: Dict[int, List[int]] = {}
        self.shared: Dict[int, List[int]] = {}           # prefix id -> its pinned blocks
        self.refs: Dict[int, int] = {}                   # prefix id -> holders (the handle, queued and running requests)
        self.prefix_of: Dict[int, int] = {}              # request id -> the prefix it names

    def reservation(self, prompt_len: int, max_new_tokens: int) -> int:
        """Blocks a request of `prompt_len` positions and `max_new_tokens` new tokens holds while it runs."""
        return -(-(prompt_len + max_new_tokens + 1) // self.block_size)

    def can_reserve(self, n_blocks: int) -> bool:
        return n_blocks <= len(self.free)

    def reserve(self, rid: int, n_blocks: int) -> List[int]:
        assert rid not in self.owned, f"request {rid} already holds blocks"
        assert self.can_reserve(n_blocks), f"{n_blocks} blocks requested, {len(self.free)} free"
        blocks, self.free = self.free[:n_blocks], self.free[n_blocks:]
        self.owned[rid] = blocks
        return blocks

    def release(self, rid: int) -> None:
        """A request is handed out: its private blocks go back, and its hold on a shared prefix ends."""
        self.free.extend(self.owned.pop(rid))
        if rid in self.prefix_of:
            self.unref(self.prefix_of.pop(rid))

    def pinned(self) -> int:
        """Blocks held by cached prefixes (dropped ones included until their last user is handed out)."""
        return sum(len(b) for b in self.shared.values())

    def pin(self, pid: int, n_blocks: int) -> List[int]:
        """Take n_blocks for prefix `pid`, held by its handle."""
        assert pid not in self.shared, f"prefix {pid} already holds blocks"
        assert self.can_reserve(n_blocks), f"{n_blocks} blocks requested, {len(self.free)} free"
        blocks, self.free = self.free[:n_blocks], self.free[n_blocks:]
        self.shared[pid], self.refs[pid] = blocks, 1
        return blocks

    def ref(self, pid: int, rid: int) -> None:
        """Request `rid` names prefix `pid` from submission until it is handed out (release)."""
        assert pid in self.shared and rid not in self.prefix_of
        self.refs[pid] += 1
        self.prefix_of[rid] = pid

    def unref(self, pid: int) -> None:
        self.refs[pid] -= 1
        if self.refs[pid] == 0:
            del self.refs[pid]
            self.free.extend(self.shared.pop(pid))


def check_kv_block_size(block_size) -> None:
    if not isinstance(block_size, int) or not 16 <= block_size <= 256 or block_size & (block_size - 1):
        raise ValueError(f"kv_block_size must be a power of two in [16, 256] (got {block_size!r})")


class ContinuousBatcher:
    def __init__(self, model, max_slots: int = 8, max_context: int = 2048, max_new_tokens: int = 1024,
                 poll_every: int = 8, use_cuda_graph: bool = True, start_image_token_id: int = IMAGE_START_TOKEN_ID,
                 end_image_token_id: int = IMAGE_END_TOKEN_ID, eos_token_id=EOS_TOKEN_IDS,
                 kv_pool_tokens: Optional[int] = None, kv_block_size: int = 64):
        """kv_pool_tokens: None keeps one dense cache region of max_context positions per slot. An integer gives a
        paged cache: a pool of ceil(kv_pool_tokens / kv_block_size) blocks (plus one scratch block) shared by all
        slots; a request is admitted (strictly first come, first served) once a slot and the blocks it needs
        are free. max_context stays the longest request either way."""
        assert 1 <= max_slots <= 128, f"the weight-streaming step serves at most 128 sequences (max_slots={max_slots})"
        check_kv_block_size(kv_block_size)
        if kv_pool_tokens is not None and (not isinstance(kv_pool_tokens, int) or kv_pool_tokens < 1):
            raise ValueError(f"kv_pool_tokens must be None or a positive integer (got {kv_pool_tokens!r})")
        self.m = model
        self.inner = model.get_model()
        self.stack = model.stack
        d = self.stack.dims
        self.d = d
        self.B, self.Tmax, self.cap = max_slots, max_context, max_new_tokens
        self.poll_every = poll_every
        self.dev = self.inner.embed_tokens.weight.device
        dev, B = self.dev, max_slots
        self.L = len(self.inner.layers)
        self.layers = [l.weights() for l in self.inner.layers]
        self.ntok = model.get_vision_tower().image_token_len if model.get_vision_tower() is not None else 0
        self.C = model.vision_head.fc2.out_features
        eos = list(eos_token_id) if isinstance(eos_token_id, (list, tuple)) else [eos_token_id]
        if len(eos) > 2:
            raise NotImplementedError("at most two EOS ids (the reference's default is [128001, 128009])")
        self.eos0 = eos[0] if eos else -1                       # an empty list never matches
        self.eos1 = eos[1] if len(eos) > 1 else self.eos0
        self.start_id, self.end_id = start_image_token_id, end_image_token_id
        self.stack.ensure_positions(max_context + 1)
        if kv_pool_tokens is None:
            self.alloc, self.table = None, None
            self.kc = torch.zeros((self.L, B, d.n_kv_heads, max_context, d.head_dim), dtype=torch.bfloat16, device=dev)
        else:
            self.alloc = KVBlockAllocator(-(-kv_pool_tokens // kv_block_size), kv_block_size)
            self.max_blocks = -(-max_context // kv_block_size)
            # pools [L, num_blocks + scratch, Hkv, block_size, dh]; table rows start (and return to) all scratch
            self.kc = torch.zeros((self.L, self.alloc.num_blocks + 1, d.n_kv_heads, kv_block_size, d.head_dim),
                                  dtype=torch.bfloat16, device=dev)
            self.table = torch.full((B, self.max_blocks), self.alloc.scratch, dtype=torch.int32, device=dev)
        self.vc = torch.zeros_like(self.kc)
        self.st = {k: torch.zeros(B, dtype=torch.int32, device=dev) for k in
                   ("in_image_mode", "total_image_tokens", "total_output", "n_ids", "n_img", "append_kind",
                    "next_token")}
        self.st["finished"] = torch.ones(B, dtype=torch.int32, device=dev)          # idle slots are frozen
        self.st["pos"] = torch.ones(B, dtype=torch.int32, device=dev)
        self.max_ids = max_new_tokens + 2
        self.max_img = max(1, ((max_new_tokens + 1) // max(self.ntok, 1) + 1) * max(self.ntok, 1))
        self.st["ids_out"] = torch.full((B, self.max_ids), -1, dtype=torch.int32, device=dev)
        self.img_out = torch.zeros((B, self.max_img, self.C), dtype=torch.bfloat16, device=dev)
        self.forced = torch.full((B, max_new_tokens + 2), -1, dtype=torch.int32, device=dev)   # -1 = free running
        self.max_new_slot = torch.zeros(B, dtype=torch.int32, device=dev)
        self.xin = torch.zeros((B, d.hidden), dtype=torch.bfloat16, device=dev)
        V = model.lm_head.weight.shape[0]
        self.V = V
        self.logits = torch.empty((B, (V + 7) // 8 * 8), dtype=torch.float32, device=dev)
        self.queue: Deque[_Request] = deque()
        self.slots: List[Optional[_Request]] = [None] * B
        self.next_rid = 0
        self.prefixes: Dict[int, PrefixHandle] = {}    # cached prefixes not yet dropped
        self.next_pid = 0
        self.steps_run = 0
        self.samp = SamplingArrays(B, dev)
        self.graph = None                  # greedy step
        self.sampled_graph = None          # step with the seeded draw, captured once a sampled request is in flight
        self.use_cuda_graph = use_cuda_graph
        self._warm = False
        self._warm_sampled = False
        self.lp: Optional[LogprobBuffers] = None   # allocated when the first request asks for log-probabilities
        self.lp_graphs: Dict[bool, torch.cuda.CUDAGraph] = {}   # sampled -> step graph with the logprob kernel
        self._warm_lp = set()

    # ------------------------------------------------------------------ one device step for all slots
    def _step_body(self, sampled: bool = False, logprobs: bool = False):
        st = self.st
        x = decoder_stack_step(self.layers, self.xin, self.kc, self.vc, st["pos"] - 1, self.stack, self.table)
        tok, pred_z, prediction = decode_heads(self.m, x, st["in_image_mode"], self.logits, self.V,
                                               self.samp if sampled else None, st["total_output"])
        ops.decode_state_step_slots(st, tok, self.forced, self.max_new_slot, self.B, self.ntok, self.start_id,
                                    self.end_id, self.eos0, self.eos1, pred_z, self.img_out)
        if logprobs:
            self.lp.launch(self.logits, self.V, st)
        ops.decode_next_input(st["append_kind"], st["next_token"], self.inner.embed_tokens.weight.data, prediction,
                              self.xin)

    def _device_step(self):
        # the sampled step only while a sampled request holds a slot (finished slots are frozen: either step is fine)
        sampled = any(r is not None and r.sampling is not None for r in self.slots)
        # the logprob step only while a request that asked holds a slot (the kernel skips every other row)
        lp = any(r is not None and r.logprobs is not None for r in self.slots)
        if lp:
            graph, warm = self.lp_graphs.get(sampled), sampled in self._warm_lp
        else:
            graph = self.sampled_graph if sampled else self.graph
            warm = self._warm_sampled if sampled else self._warm
        if graph is not None:
            graph.replay()
        elif self.use_cuda_graph and warm:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(g):
                    self._step_body(sampled, lp)
                if lp:                                 # (the capture itself does not execute the step)
                    self.lp_graphs[sampled] = g
                elif sampled:
                    self.sampled_graph = g
                else:
                    self.graph = g
                g.replay()
            except Exception:  # noqa: BLE001 - capture unsupported: stay on stream launches
                self.use_cuda_graph = False
                torch.cuda.synchronize()
                self._step_body(sampled, lp)
        else:
            self._step_body(sampled, lp)               # first step of each kind eager: sets kernel attributes
            if lp:
                self._warm_lp.add(sampled)
            elif sampled:
                self._warm_sampled = True
            else:
                self._warm = True
        self.steps_run += 1

    # ------------------------------------------------------------------ requests
    @torch.no_grad()
    def submit(self, inputs_embeds: torch.Tensor, max_new_tokens: Optional[int] = None,
               forced_tokens: Optional[torch.Tensor] = None, sampling: Optional[SamplingParams] = None,
               prefix: Optional[PrefixHandle] = None, logprobs: Optional[int] = None) -> int:
        """inputs_embeds: [P, H] or [1, P, H] prompt embeddings (text + projected image rows, as `generate` builds
        them). sampling: None or temperature 0 = greedy; otherwise the request draws its tokens with these parameters
        and seed, and its output is the same whatever other requests share the server. forced_tokens: integer ids
        indexed by the request's step count; an entry >= 0 replaces the step's token, -1 and every step past the
        schedule's end are free-running (as in `DecodeEngine.generate`). Ids outside [-1, embedding rows) raise
        ValueError here, before any device work, and so does a request whose KV blocks exceed a paged server's whole
        pool. prefix: a handle from this server's `cache_prefix`; the prompt is then the prefix followed by
        inputs_embeds (the suffix, at least one row), and the request returns exactly what that whole prompt submitted
        without a prefix returns. logprobs: None, or an int n in [0, 20]: the request also reports, for every id it
        emits, its log-probability and the n most likely ids with theirs (`run()` yields them as 'logprobs' chunks and
        the 'done' payload gains a TokenLogprobs); its ids and embeddings do not change. Returns the request id."""
        check_logprobs(logprobs)
        check_forced_tokens(forced_tokens, self.inner.embed_tokens.weight.shape[0])
        if sampling is not None and not isinstance(sampling, SamplingParams):
            raise ValueError("sampling must be a SamplingParams or None")
        if prefix is not None:
            self._check_handle(prefix)
        P = inputs_embeds.reshape(-1, inputs_embeds.shape[-1]).shape[0]
        n_new = self.cap if max_new_tokens is None else int(max_new_tokens)
        if n_new > self.cap:
            raise ValueError(f"max_new_tokens {n_new} exceeds the server's limit {self.cap}")
        if prefix is not None:
            if P < 1:
                raise ValueError("a request on a cached prefix needs a suffix of at least one row")
            P += prefix.length
        if P < 1 or P + n_new + 2 > self.Tmax:
            raise ValueError(f"prompt of {P} positions + {n_new} new ones does not fit max_context {self.Tmax}")
        if self.alloc is not None:
            start = prefix.shared_len if prefix is not None else 0
            need, avail = self.alloc.reservation(P - start, n_new), self.alloc.num_blocks - self.alloc.pinned()
            if need > avail:
                where = (f"the whole pool of {avail}" if avail == self.alloc.num_blocks else
                         f"the {avail} blocks of the pool outside its cached prefixes")
                raise ValueError(f"prompt of {P} positions + {n_new} new ones needs {need} KV blocks, more than {where}")
        e = inputs_embeds.reshape(-1, inputs_embeds.shape[-1]).to(self.dev, dtype=torch.bfloat16).contiguous()
        if prefix is not None:
            e = torch.cat([prefix.tail, e])
        f = None if forced_tokens is None else forced_tokens.reshape(-1).to(torch.int32).cpu()
        if logprobs is not None and self.lp is None:
            self.lp = LogprobBuffers(self.B, self.max_ids, self.dev)
        rid = self.next_rid
        self.next_rid += 1
        if prefix is not None:
            self.alloc.ref(prefix.pid, rid)
        self.queue.append(_Request(rid, e, n_new, f, sampling if sampling is not None and not sampling.greedy else None,
                                   prefix=prefix, logprobs=None if logprobs is None else int(logprobs)))
        return rid

    # ------------------------------------------------------------------ cached prefixes
    def _check_handle(self, h) -> None:
        if self.alloc is None:
            raise ValueError("prefix caching needs a paged server (kv_pool_tokens)")
        if not isinstance(h, PrefixHandle) or h.server is not self or self.prefixes.get(h.pid) is not h:
            raise ValueError(f"{h!r} is not a live prefix of this server (unknown, dropped or another server's)")

    @torch.no_grad()
    def cache_prefix(self, prefix_embeds: torch.Tensor) -> PrefixHandle:
        """Prefill a prompt prefix ([Lp, H] or [1, Lp, H]) once and keep its KV blocks for `submit(..., prefix=h)`.
        The first Ls = floor(Lp / block_size) * block_size positions are prefilled now into Ls / block_size pinned
        blocks, which requests on the prefix share and never write; the remaining Lp - Ls rows are kept as embeddings
        and prefilled with each request's suffix. Paged servers only. Raises ValueError, before any device work, for a
        prefix shorter than one block, one that leaves no room for a request in max_context, and one whose blocks are
        not free now or would leave a queued request more private blocks than the pool holds outside the prefixes."""
        if self.alloc is None:
            raise ValueError("prefix caching needs a paged server (kv_pool_tokens)")
        bs = self.alloc.block_size
        Lp = prefix_embeds.reshape(-1, prefix_embeds.shape[-1]).shape[0]
        Ls = Lp // bs * bs
        if Ls == 0:
            raise ValueError(f"a prefix of {Lp} positions is shorter than one KV block ({bs}) and shares nothing")
        if Lp + 3 > self.Tmax:
            raise ValueError(f"a prefix of {Lp} positions leaves no room for a request in max_context {self.Tmax}")
        n_sh = Ls // bs
        if not self.alloc.can_reserve(n_sh):
            raise ValueError(f"the prefix needs {n_sh} KV blocks and only {len(self.alloc.free)} are free now")
        avail = self.alloc.num_blocks - self.alloc.pinned() - n_sh
        worst = max((self.alloc.reservation(r.embeds.shape[0], r.max_new_tokens) for r in self.queue), default=0)
        if worst > avail:
            raise ValueError(f"pinning {n_sh} blocks would leave {avail} for requests, and a queued request needs {worst}")
        d = self.d
        Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
        e = prefix_embeds.reshape(-1, prefix_embeds.shape[-1]).to(self.dev, dtype=torch.bfloat16).contiguous()
        pid = self.next_pid
        self.next_pid += 1
        blocks = self.alloc.pin(pid, n_sh)
        row = torch.tensor(blocks, dtype=torch.int32).to(self.dev)
        ctx = StackContext(B=1, T=Ls, pos=torch.arange(Ls, dtype=torch.int32, device=self.dev), seqlens=None)
        x = e[:Ls]
        for i, w in enumerate(self.layers):
            x = self.stack.layer_forward(w, x, ctx, save=True, save_gu=False)
            s = ctx.saved.pop()
            ops.kv_prefill_paged(s.qkv, self.kc[i], self.vc[i], row, Ls, Hq, Hkv, dh)
            del s
        h = PrefixHandle(self, pid, Lp, Ls, e[Ls:].clone())
        self.prefixes[pid] = h
        return h

    def drop_prefix(self, h: PrefixHandle) -> None:
        """Forget a cached prefix: no new request may name it, and its blocks return to the pool once no queued or
        running request uses it."""
        self._check_handle(h)
        del self.prefixes[h.pid]
        self.alloc.unref(h.pid)

    @torch.no_grad()
    def _admit(self, req: _Request, b: int):
        d = self.d
        Hq, Hkv, dh = d.n_heads, d.n_kv_heads, d.head_dim
        P = req.embeds.shape[0]                        # prompt rows held: P - Ls on a prefix of Ls shared positions
        if self.alloc is not None:  # the slot's table row: [its prefix's shared blocks,] its reserved blocks, then scratch
            blocks = self.alloc.reserve(req.rid, self.alloc.reservation(P, req.max_new_tokens))
            if req.prefix is not None:
                blocks = self.alloc.shared[req.prefix.pid] + blocks
            row = torch.full((self.max_blocks,), self.alloc.scratch, dtype=torch.int32)
            row[:len(blocks)] = torch.tensor(blocks, dtype=torch.int32)
            self.table[b].copy_(row.to(self.dev, non_blocking=True))
        if req.prefix is not None:
            # positions Ls .. Ls+P-2 (prefix tail + suffix but its last row) continue the shared blocks; every layer
            # writes their K/V into the private blocks and attends through the pool
            Ls = req.prefix.shared_len
            if P > 1:
                pos = torch.arange(Ls, Ls + P - 1, dtype=torch.int32, device=self.dev)
                ctx = StackContext(B=1, T=P - 1, pos=pos, seqlens=None)
                x = req.embeds[:P - 1].contiguous()
                for i, w in enumerate(self.layers):
                    x = self.stack.layer_forward(w, x, ctx, save=False, save_gu=False,
                                                 paged=PagedPrefill(self.kc[i], self.vc[i], self.table[b], Ls))
            P += Ls
        elif P > 1:   # prefill positions 0..P-2 into the slot's cache region
            pos = torch.arange(P - 1, dtype=torch.int32, device=self.dev)
            ctx = StackContext(B=1, T=P - 1, pos=pos, seqlens=None)
            x = req.embeds[:P - 1].contiguous()
            for i, w in enumerate(self.layers):
                x = self.stack.layer_forward(w, x, ctx, save=True, save_gu=False)
                s = ctx.saved.pop()
                if self.alloc is None:
                    ops.kv_prefill(s.qkv, self.kc[i, b:b + 1], self.vc[i, b:b + 1], 1, P - 1, Hq, Hkv, dh)
                else:
                    ops.kv_prefill_paged(s.qkv, self.kc[i], self.vc[i], self.table[b], P - 1, Hq, Hkv, dh)
                del s
        self.xin[b].copy_(req.embeds[-1])             # the last prompt row, fed at position P-1
        row = torch.full((self.forced.shape[1],), -1, dtype=torch.int32)
        if req.forced is not None:
            n = min(row.numel(), req.forced.numel())
            row[:n] = req.forced[:n]
        self.forced[b].copy_(row.to(self.dev, non_blocking=True))
        for k in ("in_image_mode", "total_image_tokens", "total_output", "n_ids", "n_img", "finished"):
            self.st[k][b] = 0
        self.st["append_kind"][b] = -1
        self.st["pos"][b] = P                       # the fed token sits at position P-1
        self.max_new_slot[b] = req.max_new_tokens
        self.samp.set(b, req.sampling)
        if self.lp is not None:
            self.lp.set(b, req.logprobs)
        req.slot, req.sent_ids, req.sent_img = b, 0, 0
        self.slots[b] = req

    def _next_admission(self) -> Optional[int]:
        """The lowest free slot if the queue head can be admitted now, else None. Strict FIFO: on a paged server a
        head whose blocks are not free holds back every request behind it."""
        if not self.queue:
            return None
        b = next((i for i, s in enumerate(self.slots) if s is None), None)
        if b is not None and self.alloc is not None:
            head = self.queue[0]                   # (on a prefix, the rows held give its private blocks alone)
            if not self.alloc.can_reserve(self.alloc.reservation(head.embeds.shape[0], head.max_new_tokens)):
                return None
        return b

    def _poll(self) -> Tuple[List[Tuple[int, str, torch.Tensor]], List[int]]:
        """One host sync: new ids / visual embeddings of every running request + the requests that finished."""
        snap = torch.stack([self.st["finished"], self.st["n_ids"], self.st["n_img"]]).cpu()
        events, done = [], []
        # the new log-probabilities of every request that asked, in one gather per buffer
        lp_rows = [(b, req, req.sent_ids, int(snap[1, b])) for b, req in enumerate(self.slots)
                   if req is not None and req.logprobs is not None and int(snap[1, b]) > req.sent_ids]
        lp_chunks = self.lp.gather([(b, lo, hi, req.logprobs) for b, req, lo, hi in lp_rows]) if lp_rows else []
        lp_of = {b: c for (b, _, _, _), c in zip(lp_rows, lp_chunks)}
        for b, req in enumerate(self.slots):
            if req is None:
                continue
            fin, n_ids, n_img = int(snap[0, b]), int(snap[1, b]), int(snap[2, b])
            if n_ids > req.sent_ids:
                chunk = self.st["ids_out"][b, req.sent_ids:n_ids].clone()
                req.ids.append(chunk)
                events.append((req.rid, "ids", chunk))
                if b in lp_of:
                    req.lps.append(lp_of[b])
                    events.append((req.rid, "logprobs", lp_of[b]))
                req.sent_ids = n_ids
            if n_img > req.sent_img:
                chunk = self.img_out[b, req.sent_img:n_img].clone()
                req.img.append(chunk)
                events.append((req.rid, "image_embeds", chunk))
                req.sent_img = n_img
            if fin:
                done.append(b)
        return events, done

    @torch.no_grad()
    def run(self, max_steps: Optional[int] = None):
        """Generator: serves the queue; yields (rid, 'ids' | 'image_embeds', tensor) as outputs appear and
        (rid, 'done', (ids, image_embeds)) when a request completes. A request submitted with logprobs= also gets
        (rid, 'logprobs', TokenLogprobs) after each 'ids' chunk, and its 'done' payload is (ids, image_embeds,
        TokenLogprobs). Returns when queue and slots are empty."""
        steps = 0
        while self.queue or any(s is not None for s in self.slots):
            b = self._next_admission()
            while b is not None:
                self._admit(self.queue.popleft(), b)
                b = self._next_admission()
            for _ in range(self.poll_every):
                self._device_step()
                steps += 1
            events, done = self._poll()
            for ev in events:
                yield ev
            for b in done:
                req = self.slots[b]
                self.slots[b] = None
                if self.alloc is not None:
                    # the slot stays frozen, appending K/V at its last position every step: before the next step
                    # (stream order) its row points at scratch, never at blocks another request may now receive
                    self.alloc.release(req.rid)
                    self.table[b].fill_(self.alloc.scratch)
                ids = torch.cat(req.ids) if req.ids else torch.empty(0, dtype=torch.int32, device=self.dev)
                img = torch.cat(req.img) if req.img else torch.empty((0, self.C), dtype=torch.bfloat16, device=self.dev)
                if req.logprobs is not None:
                    yield (req.rid, "done", (ids, img, cat_logprobs(req.lps, req.logprobs, self.dev)))
                else:
                    yield (req.rid, "done", (ids, img))
            if max_steps is not None and steps >= max_steps:
                return

    def run_until_idle(self) -> Dict[int, Tuple[torch.Tensor, torch.Tensor]]:
        return {rid: payload for rid, kind, payload in self.run() if kind == "done"}
