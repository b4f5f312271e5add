"""CPU tests of prefix caching: the shared-block reference counts of the KV block allocator, the server's refusals of
bad prefixes and prefixed requests (raised before any device work), and `mm_attn_fwd_tc_paged` rejecting bad arguments,
all without a GPU."""
import random
from collections import deque
from ctypes import c_float, c_int, c_void_p

import pytest
import torch

from metamorph_b200.engine.serve import ContinuousBatcher, KVBlockAllocator, PrefixHandle


@pytest.fixture(scope="module")
def _built():
    from metamorph_b200 import _build
    _build.build(verbose=False)


# ------------------------------------------------------------------------------------------------ allocator
def test_shared_blocks_return_only_after_the_drop_and_the_last_user():
    a = KVBlockAllocator(12, 16)
    shared = a.pin(0, 3)
    assert a.scratch not in shared and a.pinned() == 3 and len(a.free) == 9
    a.ref(0, rid=10)                         # queued
    a.ref(0, rid=11)
    a.reserve(10, 2)                         # admitted: private blocks only
    a.release(10)                            # handed out; the handle and request 11 still hold the prefix
    assert a.pinned() == 3 and 0 in a.shared and len(a.free) == 9
    a.unref(0)                               # the handle is dropped; request 11 (still queued) holds it
    assert a.shared[0] == shared and len(a.free) == 9
    a.reserve(11, 4)
    assert not set(a.owned[11]) & set(shared)
    a.release(11)                            # the last user: the shared blocks come back whole
    assert sorted(a.free) == list(range(12)) and not a.shared and not a.refs and not a.prefix_of


def test_dropping_an_unused_prefix_frees_it_at_once():
    a = KVBlockAllocator(5, 32)
    a.pin(3, 5)
    assert not a.can_reserve(1)
    a.unref(3)
    assert sorted(a.free) == list(range(5))


def test_scratch_is_never_handed_out_and_nothing_is_held_twice_with_prefixes():
    rng = random.Random(7)
    a = KVBlockAllocator(40, 16)
    live, prefixes, rid, pid = set(), {}, 0, 0
    for _ in range(600):
        op = rng.random()
        if op < 0.1 and a.can_reserve(3):
            a.pin(pid, rng.randint(1, 3))
            prefixes[pid] = True
            pid += 1
        elif op < 0.2 and any(prefixes.values()):
            p = rng.choice([k for k, v in prefixes.items() if v])
            prefixes[p] = False
            a.unref(p)
        elif op < 0.6:
            n = rng.randint(1, 6)
            if a.can_reserve(n):
                live_p = [k for k, v in prefixes.items() if v]
                if live_p and rng.random() < 0.6:
                    a.ref(rng.choice(live_p), rid)
                a.reserve(rid, n)
                live.add(rid)
                rid += 1
        elif live:
            r = rng.choice(sorted(live))
            live.discard(r)
            a.release(r)
        held = [b for bl in a.owned.values() for b in bl] + [b for bl in a.shared.values() for b in bl]
        assert a.scratch not in held and a.scratch not in a.free
        assert len(held) == len(set(held)) and not set(held) & set(a.free)
        assert len(held) + len(a.free) == 40
    for r in sorted(live):
        a.release(r)
    for p, alive in prefixes.items():
        if alive:
            a.unref(p)
    assert sorted(a.free) == list(range(40)) and not a.owned and not a.shared and not a.prefix_of


@pytest.mark.parametrize("bs", [16, 64, 256])
def test_private_reservation_plus_shared_blocks_is_the_whole_prompt_reservation(bs):
    """A request on a prefix of Ls = k * bs positions reserves reservation(P - Ls, n) private blocks: with the k shared
    ones that is exactly reservation(P, n), so its table row covers positions 0 .. P+n as an unshared request's does."""
    a = KVBlockAllocator(10000, bs)
    for k in (1, 2, 5):
        Ls = k * bs
        for P in (Ls + 1, Ls + 2, Ls + bs - 1, Ls + bs, Ls + 3 * bs + 5):
            for n in (0, 1, bs - 2, bs - 1, bs, 2 * bs + 3):
                assert a.reservation(P - Ls, n) + k == a.reservation(P, n), (bs, Ls, P, n)
                assert a.reservation(P - Ls, n) >= 1


# ------------------------------------------------------------------------------------------------ server refusals
def _stub(num_blocks=10, bs=16, Tmax=200, cap=40, paged=True):
    """A server stub with a meta device: any device work on a prompt would fail with something other than ValueError."""
    srv = ContinuousBatcher.__new__(ContinuousBatcher)

    class _Emb:
        weight = torch.empty(10, 8)
    srv.inner = type("Inner", (), {"embed_tokens": _Emb})()
    srv.cap, srv.Tmax = cap, Tmax
    srv.alloc = KVBlockAllocator(num_blocks, bs) if paged else None
    srv.dev = torch.device("meta")
    srv.prefixes, srv.next_pid, srv.next_rid, srv.queue = {}, 0, 0, deque()
    return srv


def _handle(srv, Lp, pid=None):
    """Register a prefix on the stub as cache_prefix would, without the prefill."""
    bs = srv.alloc.block_size
    pid = srv.next_pid if pid is None else pid
    srv.next_pid = pid + 1
    h = PrefixHandle(srv, pid, Lp, Lp // bs * bs, torch.empty(Lp % bs, 8))
    srv.alloc.pin(pid, Lp // bs)
    srv.prefixes[pid] = h
    return h


def test_a_dense_server_refuses_prefix_caching():
    srv = _stub(paged=False)
    with pytest.raises(ValueError, match="paged server"):
        srv.cache_prefix(torch.zeros(40, 8))
    other = _stub()
    h = _handle(other, 40)
    with pytest.raises(ValueError, match="paged server"):
        srv.submit(torch.zeros(3, 8), max_new_tokens=2, prefix=h)


def test_cache_prefix_refuses_before_device_work():
    srv = _stub(num_blocks=10, bs=16, Tmax=100)
    with pytest.raises(ValueError, match="shorter than one KV block"):
        srv.cache_prefix(torch.zeros(15, 8))
    with pytest.raises(ValueError, match="no room"):
        srv.cache_prefix(torch.zeros(98, 8))
    srv.alloc.reserve(99, 7)                                     # a running request holds 7 of the 10 blocks
    with pytest.raises(ValueError, match="free now"):
        srv.cache_prefix(torch.zeros(64, 8))                     # 4 blocks
    srv.alloc.release(99)
    # a queued request needing 8 private blocks: pinning 3 would leave 7
    srv.queue.append(type("R", (), {"embeds": torch.empty(100, 0), "max_new_tokens": 27})())
    assert srv.alloc.reservation(100, 27) == 8
    with pytest.raises(ValueError, match="a queued request needs 8"):
        srv.cache_prefix(torch.zeros(48, 8))
    assert sorted(srv.alloc.free) == list(range(10)) and not srv.alloc.shared and not srv.prefixes


def test_submit_on_a_prefix_refuses_before_device_work():
    srv = _stub(num_blocks=10, bs=16, Tmax=200)
    h = _handle(srv, 40)                                         # Ls = 32: 2 shared blocks, 8 left
    with pytest.raises(ValueError, match="at least one row"):
        srv.submit(torch.zeros(0, 8), max_new_tokens=2, prefix=h)
    with pytest.raises(ValueError, match="max_context"):
        srv.submit(torch.zeros(140, 8), max_new_tokens=40, prefix=h)    # P = 180: 180 + 40 + 2 > 200
    with pytest.raises(ValueError, match="exceeds the server's limit"):
        srv.submit(torch.zeros(3, 8), max_new_tokens=41, prefix=h)
    # private blocks: reservation(P - 32, n) = ceil((48 + 40 + 1) / 16) = 6 fit the 8 outside the prefix; make the pool
    # smaller instead: pin 3 more blocks, leaving 5
    _handle(srv, 48)
    assert srv.alloc.pinned() == 5
    with pytest.raises(ValueError, match="needs 6 KV blocks, more than the 5 blocks of the pool outside"):
        srv.submit(torch.zeros(40, 8), max_new_tokens=40, prefix=h)     # P = 80, positions 32 .. 120
    # an unprefixed request is held to the same bound
    with pytest.raises(ValueError, match="needs 6 KV blocks, more than the 5 blocks"):
        srv.submit(torch.zeros(50, 8), max_new_tokens=40)
    assert not srv.queue and srv.alloc.refs == {0: 1, 1: 1} and not srv.alloc.prefix_of


def test_unknown_dropped_and_foreign_handles_are_refused():
    srv, other = _stub(), _stub()
    h, g = _handle(srv, 32), _handle(other, 32)
    with pytest.raises(ValueError, match="not a live prefix"):
        srv.submit(torch.zeros(3, 8), max_new_tokens=2, prefix=g)
    with pytest.raises(ValueError, match="not a live prefix"):
        srv.submit(torch.zeros(3, 8), max_new_tokens=2, prefix="h")
    fake = PrefixHandle(srv, h.pid, 32, 32, torch.empty(0, 8))    # same id, not the server's handle
    with pytest.raises(ValueError, match="not a live prefix"):
        srv.submit(torch.zeros(3, 8), max_new_tokens=2, prefix=fake)
    with pytest.raises(ValueError, match="not a live prefix"):
        srv.drop_prefix(g)
    srv.drop_prefix(h)
    assert sorted(srv.alloc.free) == list(range(10))
    with pytest.raises(ValueError, match="not a live prefix"):
        srv.submit(torch.zeros(3, 8), max_new_tokens=2, prefix=h)
    with pytest.raises(ValueError, match="not a live prefix"):
        srv.drop_prefix(h)


# ------------------------------------------------------------------------------------------------ C ABI
def test_paged_prefill_attention_abi_rejects_bad_arguments_without_gpu(_built):
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    a = c_void_p(256)                                   # aligned, never dereferenced: every call fails its checks first

    def attn(block_size=64, max_blocks=4, table=a, Hq=32, Hkv=8, head_dim=128, q_start=0, n_q=10, num_blocks=8,
             ldq=32 * 128 * 3 // 2, q=a, ldo=32 * 128):
        call("mm_attn_fwd_tc_paged", q, ll(ldq), a, a, c_int(num_blocks), table, c_int(max_blocks),
             c_int(block_size), a, ll(ldo), c_int(q_start), c_int(n_q), c_int(Hq), c_int(Hkv), c_int(head_dim),
             c_float(0.088), c_void_p(0))

    for bs in (0, 8, 48, 512, -16):
        with pytest.raises(MetaMorphB200Error, match="power of two"):
            attn(block_size=bs)
    for mb in (0, -1):
        with pytest.raises(MetaMorphB200Error, match="max_blocks"):
            attn(max_blocks=mb)
    with pytest.raises(MetaMorphB200Error, match="block table missing"):
        attn(table=c_void_p(0))
    with pytest.raises(MetaMorphB200Error, match="head_dim"):
        attn(head_dim=64)
    for Hq, Hkv in ((30, 8), (8, 0), (0, 8)):
        with pytest.raises(MetaMorphB200Error, match="head counts"):
            attn(Hq=Hq, Hkv=Hkv)
    for nb in (0, -3, 1 << 24):
        with pytest.raises(MetaMorphB200Error, match="num_blocks"):
            attn(num_blocks=nb)
    with pytest.raises(MetaMorphB200Error, match="q_start >= 0"):
        attn(q_start=-1)
    with pytest.raises(MetaMorphB200Error, match="n_q >= 1"):
        attn(n_q=0)
    with pytest.raises(MetaMorphB200Error, match="exceeds max_blocks"):
        attn(q_start=250, n_q=7)                        # 257 > 4 * 64
    attn_ok_edge = dict(q_start=250, n_q=6)             # 256 = 4 * 64 passes the bound, then fails on alignment below
    with pytest.raises(MetaMorphB200Error, match="alignment"):
        attn(ldq=33, **attn_ok_edge)
    with pytest.raises(MetaMorphB200Error, match="alignment"):
        attn(q=c_void_p(258))
    with pytest.raises(MetaMorphB200Error, match="alignment"):
        attn(ldo=4100)
