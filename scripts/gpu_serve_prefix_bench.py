"""Prefix caching in the continuous batcher on one GPU. Prints one JSON object (and writes it with --out, after every
section):
  * kernel: attn_fwd_paged against attn_fwd (LLaMA-3-8B heads: 32 q / 8 kv) for context + suffix pairs 1024 + 128 and
    4096 + 512 at block sizes 16, 64 and 256; CUDA-event us per call, the kernels alternated, min of 3 rounds. Two paged
    calls: the suffix rows only (what a prefixed admission runs), and every row (q_start 0: the dense call's work, so
    paged_full_over_dense is the cost of the paged addressing). Output rows asserted bit-equal to the dense ones;
  * serving: the 32-layer model at max_context 4096 with 128 slots; 256 forced requests sharing a 2048-position prefix
    (text with a 64-row image), suffixes of 16-256 rows, 64-512 new positions; the same paged server with the prefix
    cached (submit(suffix, prefix=h)) and without (the whole prompt submitted), same pool; positions/s, total admission
    time (CUDA events around every admission), mean and p90 time to first ids (host clock from the start of run() to the
    request's first streamed ids), torch.cuda.max_memory_allocated, mean occupied slots per step. Outputs asserted
    bit-equal between the two;
  * the GPU's name, power limit and max SM clock, read in the same run.

    python scripts/gpu_serve_prefix_bench.py --out build/serve_prefix_bench.json
"""
import argparse
import gc
import json
import sys
import time

import torch

sys.path.insert(0, ".")

from scripts.gpu_decode_wide_bench import gpu_info  # noqa: E402

KV_BYTES_PER_POSITION_PER_LAYER = 2 * 8 * 128 * 2          # K and V, 8 kv heads x 128 dims, bf16


def _time_us(fn, iters=30, warm=3):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def kernel_times(dev):
    from metamorph_b200 import ops
    Hq, Hkv, dh = 32, 8, 128
    scale = dh ** -0.5
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for ctx, sfx in ((1024, 128), (4096, 512)):
        T = ctx + sfx
        qkv = torch.randn(T, (Hq + 2 * Hkv) * dh, device=dev, generator=g).bfloat16()
        q, k, v = qkv[:, :Hq * dh], qkv[:, Hq * dh:(Hq + Hkv) * dh], qkv[:, (Hq + Hkv) * dh:]
        dense = lambda: ops.attn_fwd(q, k, v, 1, T, Hq, Hkv, dh, True, scale, need_lse=False)[0]   # noqa: E731
        want = dense()
        row = {}
        for bs in (16, 64, 256):
            mb = -(-T // bs)
            table = torch.randperm(mb, device=dev, generator=g).to(torch.int32)
            kp = torch.zeros(mb, Hkv, bs, dh, dtype=torch.bfloat16, device=dev)
            vp = torch.zeros_like(kp)
            ops.kv_prefill_paged(qkv, kp, vp, table, T, Hq, Hkv, dh)
            suffix = lambda: ops.attn_fwd_paged(q[ctx:], kp, vp, table, ctx, Hq, Hkv, dh, scale)   # noqa: E731
            full = lambda: ops.attn_fwd_paged(q, kp, vp, table, 0, Hq, Hkv, dh, scale)             # noqa: E731
            assert torch.equal(suffix().view(torch.int16), want[ctx:].view(torch.int16))
            assert torch.equal(full().view(torch.int16), want.view(torch.int16))
            t = {"dense": [], "suffix": [], "full": []}
            for _ in range(3):
                for name, fn in (("dense", dense), ("suffix", suffix), ("full", full)):
                    t[name].append(_time_us(fn))
            d, s, f = min(t["dense"]), min(t["suffix"]), min(t["full"])
            row[f"bs={bs}"] = {"dense_all_rows_us": round(d, 2), "paged_suffix_rows_us": round(s, 2),
                               "paged_all_rows_us": round(f, 2), "paged_full_over_dense": round(f / d, 4)}
            del kp, vp
        out[f"{ctx}+{sfx}"] = row
    return out


def _workload(model, dev, n_req, g):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    H = model.get_model().embed_tokens.weight.shape[1]
    emb = model.get_model().embed_tokens
    prefix = emb(torch.randint(0, 128000, (2048,), generator=g).to(dev))
    prefix[1000:1064] = (torch.randn(64, H, generator=g) * 0.02).to(dev, torch.bfloat16)          # a 64-row image
    reqs = []
    for _ in range(n_req):
        S = int(torch.randint(16, 257, (1,), generator=g))
        n = int(torch.randint(64, 513, (1,), generator=g))
        suffix = emb(torch.randint(0, 128000, (S,), generator=g).to(dev))
        sched = torch.randint(0, 128000, (n + 1,), generator=g).to(torch.int32)
        for s in range(20, n - 70, 200):
            sched[s] = IMAGE_START_TOKEN_ID
            sched[s + 65] = IMAGE_END_TOKEN_ID
        reqs.append((suffix, n, sched))
    return prefix, reqs


def _serve(srv, reqs, prefix, cached):
    """Runs reqs through srv (a warm-up pass of 2 short requests first); returns (outputs, stats)."""
    h = srv.cache_prefix(prefix) if cached else None

    def submit(e, n, f):
        return srv.submit(e, max_new_tokens=n, forced_tokens=f, prefix=h) if cached else \
            srv.submit(torch.cat([prefix, e]), max_new_tokens=n, forced_tokens=f)
    for e, n, f in reqs[:2]:
        submit(e, 8, f)
    srv.run_until_idle()
    torch.cuda.synchronize()
    occ, admits, used = [], [], []
    step, admit = srv._device_step, srv._admit

    def counted():
        occ.append(sum(s is not None for s in srv.slots))
        used.append(srv.alloc.num_blocks - len(srv.alloc.free))
        step()

    def timed(req, b):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        admit(req, b)
        e1.record()
        admits.append((e0, e1))
    srv._device_step, srv._admit = counted, timed
    torch.cuda.reset_peak_memory_stats()
    rids = [submit(e, n, f) for e, n, f in reqs]
    first, res = {}, {}
    t0 = time.perf_counter()
    for rid, kind, payload in srv.run():
        if kind == "ids" and rid not in first:
            first[rid] = time.perf_counter() - t0
        elif kind == "done":
            res[rid] = payload
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    del srv._device_step, srv._admit
    if h is not None:
        srv.drop_prefix(h)
    outs = [res[r] for r in rids]
    got = sum(int(i.numel() + im.shape[0]) for i, im in outs)
    ttf = sorted(first.get(r, dt) for r in rids)
    return outs, {"wall_s": round(dt, 3), "device_steps": len(occ), "positions_out": got,
                  "positions_per_s": round(got / dt, 1),
                  "admission_total_s": round(sum(a.elapsed_time(b) for a, b in admits) / 1e3, 3),
                  "admissions": len(admits),
                  "time_to_first_ids_mean_s": round(sum(ttf) / len(ttf), 3),
                  "time_to_first_ids_p90_s": round(ttf[int(0.9 * (len(ttf) - 1))], 3),
                  "mean_occupied_slots": round(sum(occ) / max(len(occ), 1), 2),
                  "peak_kv_blocks_in_use": max(used),
                  "peak_kv_in_use_GB": round(max(used) * srv.alloc.block_size * KV_BYTES_PER_POSITION_PER_LAYER *
                                             len(srv.layers) / 1e9, 2),
                  "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2)}


def serving(dev, n_req, ctx=4096, slots=128):
    from metamorph_b200 import synthetic
    from metamorph_b200.engine.serve import ContinuousBatcher
    L = 32
    model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=L)), device=dev)
    model.eval()
    for p in model.parameters():
        p.requires_grad_(False)
    torch.cuda.synchronize()
    res = {"layers": L, "max_context": ctx, "slots": slots, "requests": n_req, "prefix_positions": 2048,
           "model_GB": round(torch.cuda.memory_allocated() / 1e9, 2)}
    prefix, reqs = _workload(model, dev, n_req, torch.Generator().manual_seed(11))
    res["mean_prompt_positions"] = round(2048 + sum(e.shape[0] for e, _, _ in reqs) / n_req, 1)
    res["mean_new_positions"] = round(sum(n for _, n, _ in reqs) / n_req, 1)
    # the whole prompts the uncached arm queues (2048 + S rows each) stay on the device while queued
    whole_bytes = sum((2048 + e.shape[0]) * e.shape[1] * 2 for e, _, _ in reqs)
    free, _ = torch.cuda.mem_get_info()
    headroom = 4 * 2 ** 30 + whole_bytes                           # prefill activations, fragmentation, queued prompts
    pool_tokens = (free - headroom) // (KV_BYTES_PER_POSITION_PER_LAYER * L)
    res.update(free_after_model_GB=round(free / 1e9, 2), pool_tokens=int(pool_tokens),
               pool_GB=round(pool_tokens * KV_BYTES_PER_POSITION_PER_LAYER * L / 1e9, 2))
    outs = {}
    for kind, cached in (("uncached", False), ("cached_prefix", True)):
        srv = ContinuousBatcher(model, max_slots=slots, max_context=ctx, max_new_tokens=512, poll_every=8,
                                kv_pool_tokens=int(pool_tokens), kv_block_size=64)
        o, st = _serve(srv, reqs, prefix, cached)
        outs[kind], res[kind] = o, st
        del srv
        gc.collect()
        torch.cuda.empty_cache()
    a, b = outs["uncached"], outs["cached_prefix"]
    assert len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1].view(torch.int16), y[1].view(torch.int16))
                                    for x, y in zip(a, b)), "cached-prefix outputs differ from the uncached ones"
    res["outputs_bit_equal"] = True
    res["cached_over_uncached_positions_per_s"] = round(res["cached_prefix"]["positions_per_s"] /
                                                        res["uncached"]["positions_per_s"], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: kernel,serving")
    ap.add_argument("--requests", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_serve_prefix_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    skip = set(filter(None, args.skip.split(",")))
    res = {"gpu": gpu_info(),
           "timed": "kernel: CUDA events over 30 back-to-back calls, min of 3 alternating rounds; serving: host clock "
                    "around run() ending in a device synchronise, after a warm-up pass"}

    def dump():
        if args.out:
            with open(args.out, "w") as f:
                f.write(json.dumps(res) + "\n")
    with torch.no_grad():
        if "kernel" not in skip:
            res["kernel_us"] = kernel_times(dev)
            dump()
        if "serving" not in skip:
            res["serving_32_layers"] = serving(dev, args.requests)
            dump()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
