"""CPU tests of the paged KV cache: the block allocator of the continuous batcher (reservation counts, FIFO admission,
ownership, the scratch block), the server's argument checks, and the paged C-ABI functions rejecting bad arguments,
all without a GPU."""
import random
from ctypes import c_float, c_int, c_void_p

import pytest

from metamorph_b200.engine.serve import ContinuousBatcher, KVBlockAllocator


@pytest.fixture(scope="module")
def _built():
    from metamorph_b200 import _build
    _build.build(verbose=False)


# ------------------------------------------------------------------------------------------------ reservation
@pytest.mark.parametrize("bs", [16, 64, 256])
def test_reservation_covers_every_position_the_state_machine_writes(bs):
    """A request writes positions 0 .. P+n (prefill 0..P-2, steps at P-1 .. P-1+n, then its frozen position P+n)."""
    a = KVBlockAllocator(1000, bs)
    for total in (bs - 1, bs, bs + 1, 2 * bs - 1, 2 * bs, 2 * bs + 1):   # total = P + n
        for P in (1, 2, total // 2 + 1):
            n = total - P
            if n < 0:
                continue
            last_written = P + n
            want = last_written // bs + 1
            assert a.reservation(P, n) == want, (bs, P, n)
    assert a.reservation(bs - 1, 0) == 1 and a.reservation(bs, 0) == 2 and a.reservation(bs - 2, 0) == 1


def test_scratch_block_is_never_handed_out_and_the_pool_comes_back_whole():
    rng = random.Random(3)
    a = KVBlockAllocator(37, 16)
    assert a.scratch == 37 and sorted(a.free) == list(range(37))
    live = {}
    for rid in range(400):
        if live and (rng.random() < 0.45 or not a.can_reserve(1)):
            a.release(live.pop(rng.choice(sorted(live))))
            continue
        n = rng.randint(1, 9)
        if not a.can_reserve(n):
            continue
        blocks = a.reserve(rid, n)
        assert len(blocks) == n and a.scratch not in blocks
        live[rid] = rid
        held = [b for bl in a.owned.values() for b in bl]
        assert len(held) == len(set(held)), "a block is owned twice"
        assert not set(held) & set(a.free), "an owned block is on the free list"
        assert len(held) + len(a.free) == 37
    for rid in list(live):
        a.release(rid)
    assert sorted(a.free) == list(range(37)) and not a.owned


def test_double_reserve_and_overdraw_are_refused():
    a = KVBlockAllocator(4, 32)
    a.reserve(0, 3)
    with pytest.raises(AssertionError):
        a.reserve(0, 1)
    with pytest.raises(AssertionError):
        a.reserve(1, 2)
    assert not a.can_reserve(2) and a.can_reserve(1)


# ------------------------------------------------------------------------------------------------ FIFO admission
class _Req:
    def __init__(self, rid, P, n):
        import torch
        self.rid, self.embeds, self.max_new_tokens = rid, torch.empty(P, 0), n
        self.P, self.n = P, n


def _admission_trace(alloc, n_slots, reqs, durations):
    """The batcher's own admission rule (`_next_admission`) on a host-only stub: each round admits what it allows,
    reserving blocks as `_admit` does; then every running request ages one round and a finished one gives its blocks
    back, as `run` does. Returns [(round, rid, slot)] in admission order."""
    from collections import deque
    srv = ContinuousBatcher.__new__(ContinuousBatcher)
    srv.alloc, srv.slots, srv.queue = alloc, [None] * n_slots, deque(reqs)
    left, trace, rnd = {}, [], 0
    while srv.queue or any(s is not None for s in srv.slots):
        b = srv._next_admission()
        while b is not None:
            head = srv.queue.popleft()
            alloc.reserve(head.rid, alloc.reservation(head.P, head.n))
            srv.slots[b], left[head.rid] = head, durations[head.rid]
            trace.append((rnd, head.rid, b))
            b = srv._next_admission()
        for b, r in enumerate(srv.slots):
            if r is None:
                continue
            left[r.rid] -= 1
            if left[r.rid] == 0:
                alloc.release(r.rid)
                srv.slots[b] = None
        rnd += 1
        assert rnd < 1000
    return trace


def test_a_head_that_does_not_fit_holds_back_a_smaller_request_behind_it():
    bs = 16
    alloc = KVBlockAllocator(6, bs)
    reqs = [_Req(0, 30, 33), _Req(1, 60, 35), _Req(2, 3, 4)]       # 4, 6 and 1 blocks
    assert [alloc.reservation(r.P, r.n) for r in reqs] == [4, 6, 1]
    trace = _admission_trace(alloc, 3, reqs, {0: 2, 1: 1, 2: 1})
    # request 2 fits beside request 0 (5 of 6 blocks) but waits until the head, request 1, has run
    assert trace == [(0, 0, 0), (2, 1, 0), (3, 2, 0)]
    assert sorted(alloc.free) == list(range(6))


def test_admission_order_is_submission_order_under_pressure():
    rng = random.Random(11)
    alloc = KVBlockAllocator(20, 16)
    reqs = [_Req(i, rng.randint(1, 100), rng.randint(0, 150)) for i in range(60)]
    reqs = [r for r in reqs if alloc.reservation(r.P, r.n) <= 20]
    trace = _admission_trace(alloc, 5, reqs, {r.rid: rng.randint(1, 6) for r in reqs})
    assert [rid for _, rid, _ in trace] == [r.rid for r in reqs]
    assert sorted(alloc.free) == list(range(20)) and not alloc.owned


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("bs", [0, 8, 15, 24, 48, 100, 512, -64, 64.0, "64"])
def test_bad_block_sizes_are_refused_before_device_work(bs):
    with pytest.raises(ValueError, match="kv_block_size"):
        ContinuousBatcher(None, kv_pool_tokens=1024, kv_block_size=bs)
    with pytest.raises(ValueError, match="kv_block_size"):
        KVBlockAllocator(8, bs)


@pytest.mark.parametrize("tokens", [0, -1, 2.5])
def test_an_empty_pool_is_refused_before_device_work(tokens):
    with pytest.raises(ValueError, match="kv_pool_tokens"):
        ContinuousBatcher(None, kv_pool_tokens=tokens)


def test_a_request_larger_than_the_whole_pool_is_refused_by_submit():
    """submit's checks run on shapes alone: a server stub with a 2-block pool of 16 positions."""
    import torch
    srv = ContinuousBatcher.__new__(ContinuousBatcher)

    class _Emb:
        weight = torch.empty(10, 8)
    srv.inner = type("Inner", (), {"embed_tokens": _Emb})()
    srv.cap, srv.Tmax, srv.alloc = 40, 64, KVBlockAllocator(2, 16)
    srv.dev = torch.device("meta")                   # any device work on the prompt would fail differently
    with pytest.raises(ValueError, match="more than the whole pool of 2"):
        srv.submit(torch.zeros(20, 8), max_new_tokens=12)          # positions 0..32: 3 blocks
    with pytest.raises(ValueError, match="max_context"):
        srv.submit(torch.zeros(30, 8), max_new_tokens=33)


def test_paged_abi_rejects_bad_arguments_without_gpu(_built):
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    a = c_void_p(256)                                   # aligned, never dereferenced: every call fails its checks first

    def attn(block_size=64, max_blocks=4, table=a, Hq=32, Hkv=8, head_dim=128, splits=1):
        call("mm_decode_attn_paged", a, ll(Hq * 128 * 3), a, a, table, c_int(max_blocks), c_int(block_size), a, a, a,
             a, ll(Hq * 128), c_int(2), c_int(Hq), c_int(Hkv), c_int(head_dim), c_float(0.088), a, ll(1 << 30),
             c_int(splits), c_void_p(0))

    def prefill(block_size=64, max_blocks=4, table=a, T=10, head_dim=128):
        call("mm_kv_prefill_paged", a, ll(3 * 128), a, a, table, c_int(max_blocks), c_int(block_size), c_int(T),
             c_int(1), c_int(1), c_int(head_dim), c_void_p(0))

    for fn in (attn, prefill):
        for bs in (0, 8, 48, 512, -16):
            with pytest.raises(MetaMorphB200Error, match="power of two"):
                fn(block_size=bs)
        for mb in (0, -1):
            with pytest.raises(MetaMorphB200Error, match="max_blocks"):
                fn(max_blocks=mb)
        with pytest.raises(MetaMorphB200Error, match="block table missing"):
            fn(table=c_void_p(0))
        with pytest.raises(MetaMorphB200Error, match="head_dim 128"):
            fn(head_dim=64)
    for Hq in (24, 96):                                  # G = 3, 12
        with pytest.raises(MetaMorphB200Error, match="GQA group"):
            attn(Hq=Hq)
    with pytest.raises(MetaMorphB200Error, match="splits"):
        attn(splits=0)
    # the logical context max_blocks * block_size sizes the shared-memory bound as the dense call's Tmax does
    with pytest.raises(MetaMorphB200Error, match="too large"):
        attn(block_size=256, max_blocks=64, splits=1)
    with pytest.raises(MetaMorphB200Error, match="T<=max_blocks"):
        prefill(T=4 * 64 + 1)
