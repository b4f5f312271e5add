"""The paged KV cache of the continuous batcher on one GPU. Prints one JSON object (and writes it with --out, after
every section):
  * kernel: decode_attn_paged against decode_attn at batch 128 (LLaMA-3-8B heads: 32 q / 8 kv), every sequence at the
    last position of a 512 / 2048 / 4096-position context, block sizes 16 and 64; CUDA-event us per call, the two
    kernels alternated, min of 3 rounds;
  * overhead: the serving workload of scripts/gpu_decode_wide_bench.py (8 layers, 160 requests, 32 and 128 slots,
    max_context 1024) on a dense server and on a paged one of equal capacity (slots x max_context positions), outputs
    asserted bit-equal;
  * capacity: the 32-layer model at max_context 4096; a paged 128-slot server whose pool takes the memory left, against
    the largest dense server that fits (slots computed from 131,072 B per position per slot at 32 layers, not found by
    running out of memory); a ragged forced mix (prompts of 128-1024 positions, each with a 64-row image, 96-2048 new
    positions); positions/s, torch.cuda.max_memory_allocated and the mean number of occupied slots per step;
  * the GPU's name, power limit and max SM clock, read in the same run.

    python scripts/gpu_serve_paged_bench.py --out build/serve_paged_bench.json
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


def kernel_times(dev):
    from metamorph_b200 import ops
    B, Hq, Hkv, dh = 128, 32, 8, 128
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(B, (Hq + 2 * Hkv) * dh, device=dev, generator=g).bfloat16()
    out = {}
    for ctx in (512, 2048, 4096):
        kd = torch.randn(B, Hkv, ctx, dh, device=dev, generator=g).bfloat16()
        vd = torch.randn_like(kd)
        pos = torch.full((B,), ctx - 1, dtype=torch.int32, device=dev)
        ang = torch.rand(ctx + 1, 64, device=dev, generator=g)
        cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
        scale = dh ** -0.5
        row = {}
        for bs in (16, 64):
            mb = ctx // bs
            perm = torch.randperm(B * mb, device=dev, generator=g).to(torch.int32)
            table = perm.reshape(B, mb).contiguous()
            kp = torch.empty(B * mb, Hkv, bs, dh, dtype=torch.bfloat16, device=dev)
            vp = torch.empty_like(kp)
            kp[table.long()] = kd.reshape(B, Hkv, mb, bs, dh).transpose(1, 2)
            vp[table.long()] = vd.reshape(B, Hkv, mb, bs, dh).transpose(1, 2)
            dense = lambda: ops.decode_attn(qkv, kd, vd, pos, cos, sin, Hq, Hkv, dh, scale)          # noqa: E731
            paged = lambda: ops.decode_attn_paged(qkv, kp, vp, table, pos, cos, sin, Hq, Hkv, dh, scale)  # noqa: E731
            assert torch.equal(dense().view(torch.int16), paged().view(torch.int16))
            t = {"dense": [], "paged": []}
            for _ in range(3):
                for name, fn in (("dense", dense), ("paged", paged)):
                    t[name].append(_time_us(fn))
            d, p = min(t["dense"]), min(t["paged"])
            row[f"bs={bs}"] = {"dense_us": round(d, 2), "paged_us": round(p, 2), "paged_over_dense": round(p / d, 4)}
            del kp, vp
        out[f"ctx={ctx}"] = row
        del kd, vd
        torch.cuda.empty_cache()
    return out


def _time_us(fn, iters=50, warm=5):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def _serve(srv, reqs, warm=None):
    """Runs `reqs` [(embeds, max_new, forced)] through srv after a warm-up pass; returns (outputs, stats)."""
    if warm:
        for e, n, f in warm:
            srv.submit(e, max_new_tokens=min(n, 8), forced_tokens=f)
        srv.run_until_idle()
    torch.cuda.synchronize()
    occ = []
    step = srv._device_step

    def counted():
        occ.append(sum(s is not None for s in srv.slots))
        step()
    srv._device_step = counted
    torch.cuda.reset_peak_memory_stats()
    rids = [srv.submit(e, max_new_tokens=n, forced_tokens=f) for e, n, f in reqs]
    t0 = time.perf_counter()
    res = srv.run_until_idle()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    del srv._device_step                               # no reference cycle: the server's memory goes with `del srv`
    outs = [res[r] for r in rids]
    got = sum(int(i.numel() + im.shape[0]) for i, im in outs)
    return outs, {"wall_s": round(dt, 3), "device_steps": len(occ), "positions_out": got,
                  "positions_per_s": round(got / dt, 1), "mean_occupied_slots": round(sum(occ) / max(len(occ), 1), 2),
                  "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2)}


def _same(a, b):
    return all(torch.equal(x[0], y[0]) and torch.equal(x[1].view(torch.int16), y[1].view(torch.int16))
               for x, y in zip(a, b)) and len(a) == len(b)


def overhead(model, dev):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.serve import ContinuousBatcher
    out = {}
    for n_req, slots in ((160, 32), (160, 128)):
        g = torch.Generator().manual_seed(7)                   # the requests of gpu_decode_wide_bench.serve_times
        P = 128
        lens = torch.randint(96, 513, (n_req,), generator=g).tolist()
        reqs = []
        for n in lens:
            prompt = torch.randint(0, 128000, (1, P), generator=g)
            sched = torch.randint(0, 128000, (n + 2,), generator=g).to(torch.int32)
            for s in range(20, n - 70, 150):
                sched[s] = IMAGE_START_TOKEN_ID
                sched[s + 65] = IMAGE_END_TOKEN_ID
            reqs.append((model.get_model().embed_tokens(prompt.to(dev)), n, sched))
        row = {}
        results = {}
        for rep in range(2):                                   # alternate dense and paged; keep the faster round
            for kind, kw in (("dense", {}), ("paged_bs64", dict(kv_pool_tokens=slots * 1024, kv_block_size=64))):
                srv = ContinuousBatcher(model, max_slots=slots, max_context=1024, max_new_tokens=512, poll_every=8, **kw)
                outs, st = _serve(srv, reqs, warm=reqs[:slots])
                results.setdefault(kind, outs)
                if kind not in row or st["positions_per_s"] > row[kind]["positions_per_s"]:
                    row[kind] = st
                del srv
                torch.cuda.empty_cache()
        assert _same(results["dense"], results["paged_bs64"]), "paged server output differs from the dense one"
        row["outputs_bit_equal"] = True
        row["paged_over_dense_positions_per_s"] = round(row["paged_bs64"]["positions_per_s"] /
                                                        row["dense"]["positions_per_s"], 4)
        out[f"{n_req} requests / {slots} slots"] = row
    return out


def capacity(dev, n_req, ctx=4096):
    from metamorph_b200 import synthetic
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.serve import ContinuousBatcher
    L = 32
    model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=L)), device=dev)
    model.eval()
    for p in model.parameters():
        p.requires_grad_(False)
    torch.cuda.synchronize()
    res = {"layers": L, "max_context": ctx, "model_GB": round(torch.cuda.memory_allocated() / 1e9, 2)}
    H = model.get_model().embed_tokens.weight.shape[1]
    g = torch.Generator().manual_seed(11)
    reqs = []
    for _ in range(n_req):
        P = int(torch.randint(128, 1025, (1,), generator=g))
        n = int(torch.randint(96, 2049, (1,), generator=g))
        prompt = model.get_model().embed_tokens(torch.randint(0, 128000, (1, P), generator=g).to(dev))
        at = int(torch.randint(1, P - 64, (1,), generator=g))
        prompt[0, at:at + 64] = torch.randn(64, H, generator=g).to(dev, torch.bfloat16) * 0.02   # a 64-row image
        sched = torch.randint(0, 128000, (n + 1,), generator=g).to(torch.int32)
        for s in range(30, n - 70, 400):
            sched[s] = IMAGE_START_TOKEN_ID
            sched[s + 65] = IMAGE_END_TOKEN_ID
        reqs.append((prompt, n, sched))
    res["requests"] = n_req
    res["mean_positions_needed"] = round(sum(e.shape[1] + n + 1 for e, n, _ in reqs) / n_req, 1)
    # everything but the cache: a probe server with a 1-block pool, warmed (graphs, workspaces, prefill activations)
    probe = ContinuousBatcher(model, max_slots=128, max_context=ctx, max_new_tokens=2048, poll_every=8,
                              kv_pool_tokens=ctx, kv_block_size=64)
    for e, n, f in reqs[:2]:
        probe.submit(e[:, :ctx // 2], max_new_tokens=4, forced_tokens=f)
    probe.run_until_idle()
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    del probe
    gc.collect()
    torch.cuda.empty_cache()
    headroom = 3 * 2 ** 30                                      # allocator fragmentation, prefill activations
    per_slot = KV_BYTES_PER_POSITION_PER_LAYER * L * ctx        # 131,072 B per position at 32 layers
    budget = free - headroom
    dense_slots = max(0, min(128, budget // per_slot))
    pool_tokens = budget // (KV_BYTES_PER_POSITION_PER_LAYER * L)
    res.update(free_after_model_GB=round(free / 1e9, 2), headroom_GB=round(headroom / 1e9, 2),
               bytes_per_position_per_slot=KV_BYTES_PER_POSITION_PER_LAYER * L,
               largest_dense_slots=int(dense_slots), paged_pool_tokens=int(pool_tokens),
               dense_128_slots_cache_GB=round(128 * per_slot / 1e9, 2))
    outs = {}
    for kind, kw in (("paged_128_slots", dict(max_slots=128, kv_pool_tokens=int(pool_tokens), kv_block_size=64)),
                     (f"dense_{dense_slots}_slots", dict(max_slots=int(dense_slots)))):
        if kw["max_slots"] < 1:
            res[kind] = "does not fit"
            continue
        srv = ContinuousBatcher(model, max_context=ctx, max_new_tokens=2048, poll_every=8, **kw)
        o, st = _serve(srv, reqs, warm=reqs[:2])
        outs[kind] = o
        res[kind] = st
        del srv
        gc.collect()
        torch.cuda.empty_cache()
    if len(outs) == 2:
        a, b = outs.values()
        res["outputs_bit_equal"] = _same(a, b)
        k = list(outs)
        res["paged_over_dense_positions_per_s"] = round(res[k[0]]["positions_per_s"] / res[k[1]]["positions_per_s"], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: kernel,overhead,capacity")
    ap.add_argument("--capacity-requests", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_serve_paged_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    skip = set(filter(None, args.skip.split(",")))
    res = {"gpu": gpu_info(),
           "timed": "kernel: CUDA events over 50 back-to-back calls, min of 3 alternating rounds; serving: host clock "
                    "around run_until_idle ending in a device synchronise, after a warm-up pass"}

    def dump():
        if args.out:
            with open(args.out, "w") as f:
                f.write(json.dumps(res) + "\n")
    with torch.no_grad():
        if "kernel" not in skip:
            res["kernel_us_batch128"] = kernel_times(dev)
            dump()
        if "overhead" not in skip:
            from metamorph_b200 import synthetic
            model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=8)), device=dev)
            model.eval()
            res["overhead_8_layers"] = overhead(model, dev)
            del model
            torch.cuda.empty_cache()
            dump()
        if "capacity" not in skip:
            res["capacity_32_layers"] = capacity(dev, args.capacity_requests)
            dump()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
