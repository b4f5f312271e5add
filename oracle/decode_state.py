"""Model-free restatement of the reference decode loop (metamorph_llama.py:547-582).

`oracle/restatement.py::greedy_decode_nocache` restates the whole loop with the model inside it. This file is the same
loop body with the model taken out: the token of each step is given, so what is left is the control path alone: which
id is emitted, when image mode begins and ends, which steps keep their visual embedding, what kind of row is appended
to the inputs, and when the loop breaks. Pure Python, no torch. Test infrastructure only: the product never imports it.

The quirks of the reference are kept as they are:
  * the EOS test (:578) looks at the token of every step, image-mode steps included, although those steps emit an
    embedding and not the token;
  * `total_image_tokens` is reset by <image_end> only (:567), not when a block completes (:562-563), so a second
    <image_start> after a complete block re-enters image mode (:547-549) with the counter already full and the next
    step falls through to the ordinary-token branch (:571-574) with `in_image_mode` still set;
  * with `num_image_tokens == 0` the test of :554 never holds, so only <image_end> (:565-566) leaves image mode;
  * the limit test is `total_output_tokens > max_new_tokens` (:581), so a run takes up to `max_new_tokens + 1` steps.

A forced schedule replaces the model's token where it has an entry >= 0; -1, and every step past the schedule's end,
is free-running.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

TOKEN, HIDDEN = 0, 1        # what a step appends to the inputs: the token's embedding (:551,:569,:573) or the hidden state (:560)


@dataclass(frozen=True)
class DecodeConfig:
    num_image_tokens: int
    max_new_tokens: int
    start_id: int = 128256
    end_id: int = 128257
    eos: Sequence[int] = (128001, 128009)


@dataclass
class DecodeState:
    in_image_mode: bool = False                 # :505
    total_image_tokens: int = 0                 # :507
    total_output: int = 0                       # :508
    ids: List[int] = field(default_factory=list)            # generated_ids_list (:506)
    kept_steps: List[int] = field(default_factory=list)     # the steps whose image_embed went to image_embeds_list (:558)
    appended: List[int] = field(default_factory=list)       # TOKEN / HIDDEN, one per step
    tokens: List[int] = field(default_factory=list)         # the token each step saw (forced, or the model's)
    broke: bool = False                         # :579 / :582

    def copy(self) -> "DecodeState":
        return DecodeState(self.in_image_mode, self.total_image_tokens, self.total_output, list(self.ids),
                           list(self.kept_steps), list(self.appended), list(self.tokens), self.broke)


def chosen_token(state: DecodeState, free_token: int, forced: Optional[Sequence[int]]) -> int:
    """The schedule is indexed by the sequence's own step count."""
    i = state.total_output
    if forced is not None and i < len(forced) and forced[i] >= 0:
        return int(forced[i])
    return int(free_token)


def step(state: DecodeState, free_token: int, cfg: DecodeConfig, forced: Optional[Sequence[int]] = None) -> None:
    """One pass of the loop body (:547-582). Must not be called once the loop broke."""
    assert not state.broke, "the reference loop has left (:579/:582)"
    tok = chosen_token(state, free_token, forced)
    state.tokens.append(tok)
    if (not state.in_image_mode) and tok == cfg.start_id:                                   # :547
        state.in_image_mode = True                                                          # :549
        state.ids.append(tok)                                                               # :550
        state.appended.append(TOKEN)                                                        # :551
    elif state.in_image_mode and state.total_image_tokens < cfg.num_image_tokens:           # :554
        state.total_image_tokens += 1                                                       # :556
        state.kept_steps.append(state.total_output)                                         # :558
        state.appended.append(HIDDEN)                                                       # :560
        if state.total_image_tokens == cfg.num_image_tokens:                                # :562
            state.in_image_mode = False                                                     # :563
    elif tok == cfg.end_id:                                                                 # :565
        state.in_image_mode = False                                                         # :566
        state.total_image_tokens = 0                                                        # :567
        state.ids.append(tok)                                                               # :568
        state.appended.append(TOKEN)                                                        # :569
    else:                                                                                   # :571
        state.appended.append(TOKEN)                                                        # :573
        state.ids.append(tok)                                                               # :574
    state.total_output += 1                                                                 # :576
    if tok in cfg.eos:                                                                      # :578
        state.broke = True
    elif state.total_output > cfg.max_new_tokens:                                           # :581
        state.broke = True


def run(free_tokens: Sequence[int], cfg: DecodeConfig, forced: Optional[Sequence[int]] = None) -> DecodeState:
    """Drive the loop with one given token per step until it breaks or the tokens run out."""
    state = DecodeState()
    for tok in free_tokens:
        if state.broke:
            break
        step(state, tok, cfg, forced)
    return state


def run_forced(forced: Sequence[int], cfg: DecodeConfig) -> DecodeState:
    """A fully forced request (every entry >= 0, at least max_new_tokens + 1 of them) needs no model at all."""
    assert len(forced) > cfg.max_new_tokens and all(t >= 0 for t in forced[:cfg.max_new_tokens + 1])
    return run([-1] * (cfg.max_new_tokens + 1), cfg, forced)
