"""Token log-probabilities of decode (kernel: csrc/sampling.cu `decode_logprobs_kernel`, ops.decode_logprobs).

A sequence that asks for them (`logprobs=n`, 0 <= n <= 20) gets, for every id it emits, the log-probability of that id
under the model's raw distribution (the log-softmax of the step's logits at temperature 1, before any sampling warp)
and the n most likely ids with theirs: OpenAI-style `logprobs` / `top_logprobs`. A forced step reports the forced
token. Image-mode steps emit an embedding, not an id, and report nothing, so entry k always belongs to ids[k]. The bits
depend only on the step's logits, never on the batch, the graph or the cache layout (DESIGN.md, log-probabilities)."""
from __future__ import annotations

import numbers
from typing import List, NamedTuple, Optional

import torch

from .. import ops

TOP_MAX = ops.LOGPROB_TOP_MAX


class TokenLogprobs(NamedTuple):
    """Per emitted id k: logprob [k] fp32, top_ids [k, n] int32 and top_logprobs [k, n] fp32 (the n most likely ids of
    that step, most likely first, lowest id first among ties; id -1 / -inf past the vocabulary)."""
    logprob: torch.Tensor
    top_ids: torch.Tensor
    top_logprobs: torch.Tensor


def check_logprobs(n) -> None:
    """None (off) or an integer in [0, 20]: the number of alternatives reported per token. Raises ValueError."""
    if n is None:
        return
    if isinstance(n, bool) or not isinstance(n, numbers.Integral) or not 0 <= n <= TOP_MAX:
        raise ValueError(f"logprobs must be None or an int in [0, {TOP_MAX}] (got {n!r})")


def cat(chunks: List[TokenLogprobs], n: int, device) -> TokenLogprobs:
    if not chunks:
        return TokenLogprobs(torch.empty(0, dtype=torch.float32, device=device),
                             torch.empty((0, n), dtype=torch.int32, device=device),
                             torch.empty((0, n), dtype=torch.float32, device=device))
    return TokenLogprobs(*(torch.cat([getattr(c, f) for c in chunks]) for f in TokenLogprobs._fields))


class LogprobBuffers:
    """Per-row outputs of the logprob kernel, indexed like ids_out [B, max_ids], and the per-row n_top (-1 = off)."""

    def __init__(self, B: int, max_ids: int, device):
        self.n_top = torch.full((B,), -1, dtype=torch.int32, device=device)
        self.lp = torch.full((B, max_ids), float("nan"), dtype=torch.float32, device=device)
        self.top_ids = torch.full((B, max_ids, TOP_MAX), -1, dtype=torch.int32, device=device)
        self.top_lp = torch.full((B, max_ids, TOP_MAX), float("nan"), dtype=torch.float32, device=device)

    def set(self, b: int, n: Optional[int]) -> None:
        self.n_top[b] = -1 if n is None else int(n)

    def launch(self, logits, V: int, st: dict) -> None:
        """After the state step: report every row that appended an id this step."""
        ops.decode_logprobs(logits, V, st["append_kind"], st["next_token"], st["n_ids"], self.n_top, self.lp,
                            self.top_ids, self.top_lp)

    def gather(self, spans) -> List[TokenLogprobs]:
        """[(row b, lo, hi, n)] -> one TokenLogprobs per span (entries lo .. hi-1 of row b, n alternatives each),
        copied out with one gather per buffer, so a poll costs three launches however many requests report."""
        rows = torch.tensor([b for b, lo, hi, _ in spans for _ in range(lo, hi)], dtype=torch.long)
        cols = torch.tensor([s for _, lo, hi, _ in spans for s in range(lo, hi)], dtype=torch.long)
        rows, cols = rows.to(self.lp.device, non_blocking=True), cols.to(self.lp.device, non_blocking=True)
        lp, ids, lps = self.lp[rows, cols], self.top_ids[rows, cols], self.top_lp[rows, cols]
        out, k = [], 0
        for _, lo, hi, n in spans:
            out.append(TokenLogprobs(lp[k:k + hi - lo], ids[k:k + hi - lo, :n], lps[k:k + hi - lo, :n]))
            k += hi - lo
        return out

    def take(self, b: int, lo: int, hi: int, n: int) -> TokenLogprobs:
        """Copies of row b's entries lo .. hi-1 with n alternatives each."""
        return TokenLogprobs(self.lp[b, lo:hi].clone(), self.top_ids[b, lo:hi, :n].clone(),
                             self.top_lp[b, lo:hi, :n].clone())
