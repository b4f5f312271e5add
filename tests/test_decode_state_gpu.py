"""The decode control path on the H100, kernel by kernel: `decode_state_kernel`, `decode_next_input_kernel` and
`decode_select_hidden_kernel` (csrc/decode.cu) on synthetic arrays, no model, against oracle/decode_state.py, the
model-free restatement of the reference loop body (metamorph_llama.py:547-582).

One block serves one sequence, so a launch carries every token stream over a six-letter alphabet at once and the
comparison is exhaustive, bit for bit, after every step. tests/test_decode_checkers.py shows on the CPU that the
comparisons here reject emulated kernel bugs.
"""
import numpy as np
import pytest
import torch

from oracle.decode_state import HIDDEN, TOKEN, DecodeConfig, DecodeState, step

pytestmark = pytest.mark.gpu

START, END, EOS0, EOS1 = 1000, 1001, 1002, 1003
ALPHABET = (START, END, EOS0, EOS1, 7, 0)                 # two ordinary ids, one of them 0
ARRAYS = ("in_image_mode", "total_image_tokens", "total_output", "finished", "pos", "n_ids", "n_img", "ids_out",
          "append_kind", "next_token")
NAN_BITS, GUARD_BITS = 0x7FC5, 0x7FA3                       # two NaN patterns of bf16, as int16 bit patterns


# ------------------------------------------------------------------------------------------------ expected arrays
def expected_arrays(nodes, pos0, max_ids, ids_fill=-1):
    """The ten device arrays after a launch. nodes[b] = (DecodeState after the step, whether the step ran): a sequence
    whose loop had broken before the launch is frozen, with append_kind -1."""
    B = len(nodes)
    col = lambda f: np.fromiter((f(s, live) for s, live in nodes), dtype=np.int32, count=B)   # noqa: E731
    out = {
        "in_image_mode": col(lambda s, _: int(s.in_image_mode)),
        "total_image_tokens": col(lambda s, _: s.total_image_tokens),
        "total_output": col(lambda s, _: s.total_output),
        "finished": col(lambda s, _: int(s.broke)),
        "n_ids": col(lambda s, _: len(s.ids)),
        "n_img": col(lambda s, _: len(s.kept_steps)),
        "append_kind": col(lambda s, live: s.appended[-1] if live else -1),
        "next_token": col(lambda s, _: s.tokens[-1] if s.tokens else 0),
    }
    out["pos"] = np.asarray(pos0, dtype=np.int32) + out["total_output"]
    ids = np.full((B, max_ids), ids_fill, dtype=np.int32)
    for b, (s, _) in enumerate(nodes):
        n = min(len(s.ids), max_ids)
        ids[b, :n] = s.ids[:n]
    out["ids_out"] = ids
    return out


def assert_state_equal(got, want, what):
    """Bit-for-bit equality of all ten arrays; names the first array and entry that differ."""
    for k in ARRAYS:
        g = got[k].cpu().numpy() if torch.is_tensor(got[k]) else np.asarray(got[k])
        w = np.asarray(want[k])
        assert g.shape == w.shape, f"{what}: {k} has shape {g.shape}, expected {w.shape}"
        if not np.array_equal(g, w):
            at = tuple(np.argwhere(g != w)[0])
            raise AssertionError(f"{what}: {k} differs in {int((g != w).sum())} entries, first at {at}: "
                                 f"got {g[at]}, expected {w[at]}")


def stream_tree(alphabet, L, cfg):
    """levels[l][i] = (state, live) of the i-th prefix of length l (first token most significant), and the regimes some
    prefix reached. A prefix whose loop broke keeps its parent's state object: it is frozen."""
    regimes = set()
    levels = [[(DecodeState(), False)]]
    for _ in range(L):
        nxt = []
        for s, _live in levels[-1]:
            for t in alphabet:
                if s.broke:
                    nxt.append((s, False))
                    continue
                c = s.copy()
                step(c, t, cfg)
                nxt.append((c, True))
                if s.in_image_mode and t in cfg.eos:
                    regimes.add("eos_in_image")
                if c.broke and t not in cfg.eos:
                    regimes.add("limit")
                if cfg.num_image_tokens > 0:
                    if not s.in_image_mode and t == cfg.start_id and s.total_image_tokens == cfg.num_image_tokens:
                        regimes.add("second_start")
                    if len(c.kept_steps) == 2 * cfg.num_image_tokens:
                        regimes.add("two_blocks")
                elif s.in_image_mode and c.in_image_mode and t != cfg.end_id:
                    regimes.add("only_end_leaves")
        levels.append(nxt)
    return levels, regimes


def reachable_regimes(cfg, L):
    """What `min(L, max_new_tokens + 1)` live steps can reach, counted from the loop body."""
    n, k = min(L, cfg.max_new_tokens + 1), cfg.num_image_tokens
    need = {"eos_in_image": 2, "limit": cfg.max_new_tokens + 1}
    if k > 0:
        need.update(second_start=k + 2, two_blocks=2 * k + 3)
    else:
        need.update(only_end_leaves=2)
    return {r for r, steps in need.items() if n >= steps}


# ------------------------------------------------------------------------------------------------ device side
def new_state(B, pos0, max_ids, dev, ids_fill=-1):
    st = {k: torch.zeros(B, dtype=torch.int32, device=dev) for k in ARRAYS if k not in ("pos", "ids_out")}
    st["pos"] = torch.as_tensor(np.asarray(pos0, dtype=np.int32)).to(dev)
    st["ids_out"] = torch.full((B, max_ids), ids_fill, dtype=torch.int32, device=dev)
    return st


def eos_pair(eos):
    """The engine's encoding of an EOS list of 0, 1 or 2 ids."""
    e0 = eos[0] if eos else -1
    return e0, (eos[1] if len(eos) > 1 else e0)


def launch(st, tok, cfg, pred_z, img_out, forced=None, max_new_slot=None):
    from metamorph_b200 import ops
    e0, e1 = eos_pair(list(cfg.eos))
    B = tok.shape[0]
    if max_new_slot is None:
        ops.decode_state_step(st, tok, forced, 0, B, cfg.num_image_tokens, cfg.max_new_tokens, cfg.start_id, cfg.end_id,
                              e0, e1, pred_z, img_out)
    else:
        ops.decode_state_step_slots(st, tok, forced, max_new_slot, B, cfg.num_image_tokens, cfg.start_id, cfg.end_id,
                                    e0, e1, pred_z, img_out)


def stream_tokens(n_alpha, L, l):
    """Letter index of step l of each of the n_alpha ** L streams."""
    return (np.arange(n_alpha ** L) // n_alpha ** (L - 1 - l)) % n_alpha


# ------------------------------------------------------------------------------------------------ every token stream
SETTINGS = [(k, m, 6) for k in (0, 1, 2, 4) for m in (0, 1, 3, 11)] + [(2, 100, 7)]


@pytest.mark.parametrize("ntok,max_new,L", SETTINGS)
def test_every_token_stream(cuda_device, ntok, max_new, L):
    cfg = DecodeConfig(ntok, max_new, START, END, (EOS0, EOS1))
    levels, regimes = stream_tree(ALPHABET, L, cfg)
    assert regimes == reachable_regimes(cfg, L), (regimes, reachable_regimes(cfg, L))
    A, B = len(ALPHABET), len(ALPHABET) ** L
    pos0 = 1 + np.arange(B) % 7
    st = new_state(B, pos0, L + 1, cuda_device)
    pred_z = torch.zeros((B, 8), dtype=torch.bfloat16, device=cuda_device)
    img_out = torch.zeros((B, L, 8), dtype=torch.bfloat16, device=cuda_device)
    letters = np.asarray(ALPHABET, dtype=np.int32)
    frozen_launches = 0
    for l in range(L):
        tok = torch.from_numpy(letters[stream_tokens(A, L, l)]).to(cuda_device)
        launch(st, tok, cfg, pred_z, img_out)
        nodes = levels[l + 1]
        frozen_launches += sum(1 for _, live in nodes if not live)
        want = expected_arrays(nodes, np.zeros(len(nodes), dtype=np.int32), L + 1)
        rep = B // len(nodes)
        want = {k: np.repeat(v, rep, axis=0) for k, v in want.items()}
        want["pos"] = want["pos"] + pos0.astype(np.int32)
        assert_state_equal(st, want, f"ntok={ntok} max_new={max_new} step {l}")
    # sequences that finished early stayed frozen through later launches (the comparison above covered them)
    assert frozen_launches > 0


# ------------------------------------------------------------------------------------------------ forced schedules
def _run_rows(free, forced_rows, cfgs, st, launch_fn, pos0, max_ids, what):
    """Step B oracle sequences and the device state side by side; returns the final oracle states and a per-step list
    of (live, chosen-from-schedule, past-the-schedule) counts."""
    B, L = free.shape
    states = [DecodeState() for _ in range(B)]
    seen = dict(hole=0, past_end=0, past_end_differs=0, frozen=0)
    for l in range(L):
        nodes = []
        for b in range(B):
            s, row = states[b], (forced_rows[b] if forced_rows is not None else None)
            if s.broke:
                nodes.append((s, False))
                seen["frozen"] += 1
                continue
            if row is not None:
                i = s.total_output
                if i < len(row) and row[i] < 0:
                    seen["hole"] += 1
                if i >= len(row):
                    seen["past_end"] += 1
                    seen["past_end_differs"] += int(row[-1] != free[b, l])
            step(s, int(free[b, l]), cfgs[b], row)
            nodes.append((s, True))
        launch_fn(l)
        assert_state_equal(st, expected_arrays(nodes, pos0, max_ids), f"{what} step {l}")
    return states, seen


@pytest.mark.parametrize("eos", [(EOS0,), (EOS0, EOS1), ()], ids=["one_eos", "two_eos", "no_eos"])
@pytest.mark.parametrize("width", [0, 5, 20], ids=["forced_none", "schedule_ends_early", "schedule_covers_run"])
def test_forced_schedule_with_holes(cuda_device, eos, width):
    rng = np.random.default_rng(100 + width + len(eos))
    B, L = 4096, 14
    cfg = DecodeConfig(2, 12, START, END, eos)
    letters = np.asarray(ALPHABET, dtype=np.int32)
    free = letters[rng.integers(0, len(letters), (B, L))]
    forced = None
    if width:
        forced = letters[rng.integers(0, len(letters), (B, width))]
        forced[rng.random((B, width)) < 0.3] = -1             # holes: free-running steps inside the schedule
        forced[0] = -1
    st = new_state(B, np.full(B, 3), L + 1, cuda_device)
    pred_z = torch.zeros((B, 8), dtype=torch.bfloat16, device=cuda_device)
    img_out = torch.zeros((B, L, 8), dtype=torch.bfloat16, device=cuda_device)
    fdev = torch.from_numpy(forced).to(cuda_device) if forced is not None else None
    free_dev = torch.from_numpy(free).to(cuda_device)
    rows = [forced[b].tolist() for b in range(B)] if forced is not None else None
    states, seen = _run_rows(free, rows, [cfg] * B, st,
                             lambda l: launch(st, free_dev[:, l].contiguous(), cfg, pred_z, img_out, forced=fdev),
                             np.full(B, 3), L + 1, f"eos={eos} width={width}")
    if width:
        assert seen["hole"] > 0, "no live step fell into a -1 hole"
    if width == 5:
        assert seen["past_end_differs"] > 100, "the schedule never ended before the run"
    if width == 20:
        assert seen["past_end"] == 0
    by_eos = sum(1 for s in states if s.broke and s.tokens[-1] in eos)
    if eos:
        assert by_eos > 0 and seen["frozen"] > 0
    else:                                                      # eos0 = eos1 = -1 on the device: nothing may match
        assert by_eos == 0 and all(s.total_output == 13 and s.broke for s in states)
        assert (free >= 0).all()


def test_per_slot_limits_equal_the_batch_limit_group_by_group(cuda_device):
    rng = np.random.default_rng(7)
    B, L = 1000, 9
    limits = np.asarray([0, 1, 2, 5, 50], dtype=np.int32)[np.arange(B) % 5]
    letters = np.asarray(ALPHABET, dtype=np.int32)
    free = letters[rng.choice(len(letters), (B, L), p=[0.2, 0.15, 0.03, 0.02, 0.3, 0.3])]
    cfgs = [DecodeConfig(2, int(m), START, END, (EOS0, EOS1)) for m in limits]
    st = new_state(B, np.full(B, 1), L + 1, cuda_device)
    pred_z = torch.zeros((B, 8), dtype=torch.bfloat16, device=cuda_device)
    img_out = torch.zeros((B, L, 8), dtype=torch.bfloat16, device=cuda_device)
    lim_dev = torch.from_numpy(limits).to(cuda_device)
    free_dev = torch.from_numpy(free).to(cuda_device)
    # decode_state_step_slots ignores the batch limit: run it under a config whose limit would stop everything at once
    slots_cfg = DecodeConfig(2, 0, START, END, (EOS0, EOS1))
    states, _ = _run_rows(free, None, cfgs, st,
                          lambda l: launch(st, free_dev[:, l].contiguous(), slots_cfg, pred_z, img_out,
                                           max_new_slot=lim_dev),
                          np.full(B, 1), L + 1, "per-slot limits")
    stopped_by_limit = {int(m): sum(1 for s, c in zip(states, cfgs) if c.max_new_tokens == m and s.broke
                                    and s.tokens[-1] not in (EOS0, EOS1)) for m in (0, 1, 2, 5, 50)}
    assert all(stopped_by_limit[m] > 0 for m in (0, 1, 2, 5)) and stopped_by_limit[50] == 0
    for m in (0, 1, 2, 5, 50):                                  # the same sequences through decode_state_step
        sel = np.flatnonzero(limits == m)
        g = new_state(len(sel), np.full(len(sel), 1), L + 1, cuda_device)
        pz, io = pred_z[:len(sel)], torch.zeros((len(sel), L, 8), dtype=torch.bfloat16, device=cuda_device)
        sel_dev = torch.from_numpy(sel).to(cuda_device)
        for l in range(L):
            launch(g, free_dev[sel_dev, l].contiguous(), DecodeConfig(2, m, START, END, (EOS0, EOS1)), pz, io)
        assert_state_equal(g, {k: st[k][sel_dev].cpu().numpy() for k in ARRAYS}, f"group limit {m}")


# ------------------------------------------------------------------------------------------------ stored embeddings
def _pattern(l, b, C):
    """bf16 bit pattern of pred_z[b, c] at step l: a mix of (step, sequence, column), so that a row stored from the
    wrong step, sequence or offset differs (compared as int16 bits: NaN patterns count like any other)."""
    c = np.arange(C, dtype=np.int64)
    return ((l * 40503 + b * 9973 + c * 257 + (c >> 3) * 31 + 12345) & 0xFFFF).astype(np.uint16).view(np.int16)


def expected_img_bits(states, max_img, C, pad):
    """img_out as int16 bits, `pad` guard elements after it: row j of sequence b is the j-th kept step's pred_z, rows
    past max_img are dropped, everything else keeps the guard. Returns (bits, dropped rows)."""
    B = len(states)
    bits = np.full(B * max_img * C + pad, GUARD_BITS, dtype=np.int16)
    view = bits[:B * max_img * C].reshape(B, max_img, C)
    dropped = 0
    for b, s in enumerate(states):
        for j, l in enumerate(s.kept_steps):
            if j < max_img:
                view[b, j] = _pattern(l, b, C)
            else:
                dropped += 1
    return bits, dropped


@pytest.mark.parametrize("C", [1, 127, 128, 129, 1152])
def test_stored_embeddings_and_their_bounds(cuda_device, C):
    B, L, ntok, max_img, max_ids, pad = 48, 12, 3, 4, 3, 37
    cfg = DecodeConfig(ntok, 100, START, END, ())
    free = np.full((B, L), 7, dtype=np.int32)
    free[:, 0] = START
    free[:, 4] = END
    free[:, 5] = START                                          # a second block: 6 kept steps, max_img holds 4
    free[B // 2:, 5] = 7                                        # ... in the first half only
    free[1::2, 0] = 0                                           # odd sequences start their first block a step later
    free[1::2, 1] = START
    free[1::2, 4], free[1::2, 5] = 7, END
    free[1::2, 6] = free[0::2, 5]
    img_flat = torch.full((B * max_img * C + pad,), GUARD_BITS, dtype=torch.int16, device=cuda_device)
    img_out = img_flat[:B * max_img * C].view(torch.bfloat16).view(B, max_img, C)
    ids_flat = torch.full((B * max_ids + pad,), -7, dtype=torch.int32, device=cuda_device)
    st = new_state(B, np.full(B, 2), max_ids, cuda_device)
    st["ids_out"] = ids_flat[:B * max_ids].view(B, max_ids)
    free_dev = torch.from_numpy(free).to(cuda_device)
    states = [DecodeState() for _ in range(B)]
    for l in range(L):
        bits = np.stack([_pattern(l, b, C) for b in range(B)])
        pred_z = torch.from_numpy(bits).to(cuda_device).view(torch.bfloat16)
        launch(st, free_dev[:, l].contiguous(), cfg, pred_z, img_out)
        for b in range(B):
            step(states[b], int(free[b, l]), cfg)
    want_img, dropped = expected_img_bits(states, max_img, C, pad)
    assert dropped > 0 and any(len(s.kept_steps) <= max_img for s in states), "max_img never dropped a row"
    assert np.array_equal(img_flat.cpu().numpy(), want_img), "img_out (rows, order, untouched rest, guard) differs"
    want = expected_arrays([(s, True) for s in states], np.full(B, 2), max_ids, ids_fill=-7)
    assert min(len(s.ids) for s in states) > max_ids, "max_ids never dropped an id"
    assert_state_equal(st, want, f"C={C}")
    assert (ids_flat[B * max_ids:] == -7).all(), "ids_out written past its end"


# ------------------------------------------------------------------------------------------------ the gathers
def _guarded(rows, H, dev, fill):
    """[rows, H] bf16 view in the middle of an int16 buffer with one guard row on each side."""
    flat = torch.full(((rows + 2) * H,), GUARD_BITS, dtype=torch.int16, device=dev)
    flat[H:(rows + 1) * H] = fill
    return flat, flat[H:(rows + 1) * H].view(torch.bfloat16).view(rows, H)


@pytest.mark.parametrize("H", [8, 256, 1016, 1024, 4096])
def test_next_input_gather(cuda_device, H):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(H)
    B, rows = 33, 50
    embed = torch.randint(-32768, 32767, (rows, H), generator=g, dtype=torch.int16).to(cuda_device)
    pred = torch.randint(-32768, 32767, (B, H), generator=g, dtype=torch.int16).to(cuda_device)
    kind = torch.tensor([(0, 1, -1)[b % 3] for b in range(B)], dtype=torch.int32)
    tok = torch.randint(0, rows, (B,), generator=g, dtype=torch.int32)
    tok[0], tok[3] = 0, rows - 1                                # the table's first and last row, on kind-0 sequences
    flat, x = _guarded(B, H, cuda_device, NAN_BITS)
    ops.decode_next_input(kind.to(cuda_device), tok.to(cuda_device), embed.view(torch.bfloat16),
                          pred.view(torch.bfloat16), x)
    got = flat.cpu().view(B + 2, H)
    e, p = embed.cpu(), pred.cpu()
    assert (got[0] == GUARD_BITS).all() and (got[-1] == GUARD_BITS).all()
    counts = {0: 0, 1: 0, -1: 0}
    for b in range(B):
        k = int(kind[b])
        want = e[int(tok[b])] if k == TOKEN else p[b] if k == HIDDEN else torch.full((H,), NAN_BITS, dtype=torch.int16)
        assert torch.equal(got[b + 1], want), f"H={H} row {b} kind {k}"
        counts[k] += 1
    assert min(counts.values()) >= 10


@pytest.mark.parametrize("H", [8, 256, 1016, 1024, 4096])
def test_select_hidden(cuda_device, H):
    from metamorph_b200 import ops
    g = torch.Generator().manual_seed(H + 1)
    B = 35
    mode = torch.tensor([(0, 1, -3, 7, 2 ** 31 - 1)[b % 5] for b in range(B)], dtype=torch.int32)
    hidden = torch.randint(-32768, 32767, (B, H), generator=g, dtype=torch.int16)
    pred = torch.randint(-32768, 32767, (B, H), generator=g, dtype=torch.int16)
    want = torch.where((mode != 0)[:, None], pred, hidden)
    hidden[mode != 0] = NAN_BITS                                # the side that must not be read holds NaN
    pred[mode == 0] = NAN_BITS
    flat, out = _guarded(B, H, cuda_device, 0)
    ops.decode_select_hidden(mode.to(cuda_device), hidden.to(cuda_device).view(torch.bfloat16),
                             pred.to(cuda_device).view(torch.bfloat16), out)
    got = flat.cpu().view(B + 2, H)
    assert (got[0] == GUARD_BITS).all() and (got[-1] == GUARD_BITS).all()
    assert torch.equal(got[1:-1], want)
    assert not (got[1:-1] == NAN_BITS).all(1).any()


def test_gathers_reject_a_row_length_off_the_vector_width(cuda_device):
    from metamorph_b200 import ops
    from metamorph_b200._lib import MetaMorphB200Error
    B, H = 4, 12
    z = torch.zeros((B, H), dtype=torch.bfloat16, device=cuda_device)
    i = torch.zeros(B, dtype=torch.int32, device=cuda_device)
    flat, out = _guarded(B, H, cuda_device, NAN_BITS)
    with pytest.raises(MetaMorphB200Error, match="H%8"):
        ops.decode_next_input(i, i, z, z, out)
    with pytest.raises(MetaMorphB200Error, match="H%8"):
        ops.decode_select_hidden(i, z, z, out)
    torch.cuda.synchronize()
    got = flat.cpu()
    assert (got[H:-H] == NAN_BITS).all() and (got[:H] == GUARD_BITS).all() and (got[-H:] == GUARD_BITS).all()


# ------------------------------------------------------------------------------------------------ graph replay
def test_graph_replay_equals_stream_launches(cuda_device):
    """The step is captured once: the schedule index is the device's `total_output`, not a launch argument."""
    from metamorph_b200 import ops
    rng = np.random.default_rng(3)
    B, L, H, width = 512, 12, 64, 7
    cfg = DecodeConfig(2, 9, START, END, (EOS0,))
    letters = np.asarray(ALPHABET, dtype=np.int32)
    free = torch.from_numpy(letters[rng.integers(0, len(letters), (B, L))]).to(cuda_device)
    forced = letters[rng.integers(0, len(letters), (B, width))]
    forced[rng.random((B, width)) < 0.4] = -1
    forced = torch.from_numpy(forced).to(cuda_device)
    g = torch.Generator().manual_seed(9)
    embed = torch.randn((1004, H), generator=g).bfloat16().to(cuda_device)
    preds = torch.randn((L, B, H), generator=g).bfloat16().to(cuda_device)

    def fresh():
        st = new_state(B, np.full(B, 4), L + 1, cuda_device)
        return st, torch.zeros((B, L, H), dtype=torch.bfloat16, device=cuda_device), \
            torch.zeros((B, H), dtype=torch.bfloat16, device=cuda_device)

    def body(st, tok, pred, img_out, xin):
        launch(st, tok, cfg, pred, img_out, forced=forced)
        ops.decode_next_input(st["append_kind"], st["next_token"], embed, pred, xin)

    st, img_out, xin = fresh()
    trace = []
    for l in range(L):
        body(st, free[:, l].contiguous(), preds[l], img_out, xin)
        trace.append(({k: st[k].clone() for k in ARRAYS}, img_out.clone(), xin.clone()))
    assert int(st["finished"].sum()) > 0 and int((st["total_output"] > width).sum()) > 0
    st, img_out, xin = fresh()
    tok_buf, pred_buf = torch.zeros(B, dtype=torch.int32, device=cuda_device), torch.zeros_like(preds[0])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body(st, tok_buf, pred_buf, img_out, xin)
    for l in range(L):
        tok_buf.copy_(free[:, l])
        pred_buf.copy_(preds[l])
        graph.replay()
        want, want_img, want_x = trace[l]
        assert_state_equal(st, {k: v.cpu().numpy() for k, v in want.items()}, f"replay {l}")
        assert torch.equal(img_out, want_img) and torch.equal(xin, want_x), f"replay {l}: embeddings differ"
