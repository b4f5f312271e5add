"""Per-sequence sampling parameters of the decode step (kernel: csrc/sampling.cu, ops.sample_rows).

A sequence samples its next token from HF's Temperature -> TopK -> TopP warped distribution with a stateless,
seeded draw: the token depends only on the logits, the parameters, the seed and the number of steps the sequence has
taken. So a run repeats bit for bit, graph replay equals stream launches, and a served request's output does not
depend on which other requests share its step. temperature == 0 is greedy decoding (the argmax path)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Sequence, Union

import torch

_U64 = 1 << 64


@dataclass
class SamplingParams:
    """temperature 0 = greedy; top_k 0 = off; top_p 1 = off; seed None = one 63-bit seed drawn from torch's default
    CPU generator (so `torch.manual_seed` makes runs reproducible)."""
    temperature: float = 0.0
    top_k: int = 0
    top_p: float = 1.0
    seed: Optional[int] = None

    def __post_init__(self):
        t, p = float(self.temperature), float(self.top_p)
        if not math.isfinite(t) or t < 0:
            raise ValueError(f"temperature must be a finite number >= 0 (got {self.temperature})")
        if int(self.top_k) != self.top_k or self.top_k < 0:
            raise ValueError(f"top_k must be an integer >= 0 (got {self.top_k})")
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"top_p must lie in [0, 1] (got {self.top_p})")
        if self.seed is None:
            self.seed = int(torch.randint(0, 2 ** 63 - 1, (), dtype=torch.int64).item())
        elif int(self.seed) != self.seed or not 0 <= self.seed < _U64:
            raise ValueError(f"seed must be an integer in [0, 2^64) (got {self.seed})")
        self.temperature, self.top_k, self.top_p, self.seed = t, int(self.top_k), p, int(self.seed)

    @property
    def greedy(self) -> bool:
        return self.temperature == 0.0


def per_sequence(sampling: Union[None, SamplingParams, Sequence[SamplingParams]], B: int) -> Optional[List[SamplingParams]]:
    """One SamplingParams per sequence, or None when every sequence is greedy. A single SamplingParams for a batch gives
    sequence b the seed `seed + b` (mod 2^64), the random stream of a lone decode with that seed."""
    if sampling is None:
        return None
    if isinstance(sampling, SamplingParams):
        sampling = [SamplingParams(sampling.temperature, sampling.top_k, sampling.top_p, (sampling.seed + b) % _U64)
                    for b in range(B)]
    else:
        sampling = list(sampling)
        if len(sampling) != B or not all(isinstance(s, SamplingParams) for s in sampling):
            raise ValueError(f"sampling must be a SamplingParams or a list of {B} of them")
    return None if all(s.greedy for s in sampling) else sampling


class SamplingArrays:
    """Per-row device arrays read by the sampling kernel (temperature 0 rows stay greedy)."""

    def __init__(self, B: int, device):
        self.temperature = torch.zeros(B, dtype=torch.float32, device=device)
        self.top_k = torch.zeros(B, dtype=torch.int32, device=device)
        self.top_p = torch.ones(B, dtype=torch.float32, device=device)
        self.seed = torch.zeros(B, dtype=torch.int64, device=device)      # the bits of a uint64

    def set(self, b: int, sp: Optional[SamplingParams]) -> None:
        sp = sp if sp is not None else SamplingParams(seed=0)
        self.temperature[b] = sp.temperature
        self.top_k[b] = sp.top_k
        self.top_p[b] = sp.top_p
        self.seed[b] = sp.seed - _U64 if sp.seed >= 1 << 63 else sp.seed

    @classmethod
    def of(cls, params: Sequence[SamplingParams], device) -> "SamplingArrays":
        a = cls(len(params), device)
        a.temperature.copy_(torch.tensor([s.temperature for s in params], dtype=torch.float32))
        a.top_k.copy_(torch.tensor([s.top_k for s in params], dtype=torch.int32))
        a.top_p.copy_(torch.tensor([s.top_p for s in params], dtype=torch.float32))
        a.seed.copy_(torch.tensor([s.seed - _U64 if s.seed >= 1 << 63 else s.seed for s in params], dtype=torch.int64))
        return a
