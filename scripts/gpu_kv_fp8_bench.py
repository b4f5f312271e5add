"""The FP8 (E4M3) KV cache against bf16 on one GPU, alternating the two in one process. Prints one JSON object (and
writes it with --out after every section):
  * attention: decode_attn / decode_attn_fp8 (dense) and the paged pair at block sizes 16 and 64, LLaMA-3-8B heads
    (32 q / 8 kv), batch 8, 32 and 128, every sequence at the last position of a 512 / 2048 / 4096-position context;
    CUDA-event us per call (100 launches, min of 3 alternating rounds), the K/V bytes a call reads and the rate;
  * decode step: greedy_decode of the synthetic model (--layers, default 8) at batch 8, 32 and 128, 128-position prompts
    and 512 forced new positions (two 64-row images), bf16 against FP8, ms per step (min of 2 alternating rounds);
  * serving: paged servers of equal pool bytes (bf16 at --pool-tokens positions, FP8 at 2 * 128 / (128 + 4) times as
    many), 128 slots, max_context 4096, a ragged forced mix (prompts of 128-1024 positions, 96-2048 new ones);
    positions/s, mean occupied slots per step, peak allocated memory and the time to the first ids of the first wave;
  * divergence: the same forced schedule through a bf16 and an FP8 server: max / mean |d logit| of the last step's
    logits, top-1 agreement over every step, cosine of the visual embeddings. The weights are synthetic: a sanity
    figure, not a statement about LLaMA-3's quality;
  * the GPU's name, power limit and max SM clock, read in the same run.

    python scripts/gpu_kv_fp8_bench.py --out build/kv_fp8_bench.json
"""
import argparse
import gc
import json
import sys
import time

import torch

sys.path.insert(0, ".")

from scripts.gpu_decode_wide_bench import gpu_info, time_us  # noqa: E402

HQ, HKV, DH = 32, 8, 128


def _save(res, path):
    line = json.dumps(res)
    if path:
        with open(path, "w") as f:
            f.write(line + "\n")
    return line


def attention_times(dev):
    from metamorph_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for B in (8, 32, 128):
        qkv = torch.randn(B, (HQ + 2 * HKV) * DH, device=dev, generator=g).bfloat16()
        for ctx in (512, 2048, 4096):
            kd = torch.randn(B, HKV, ctx, DH, device=dev, generator=g).bfloat16()
            vd = torch.randn_like(kd)
            kq = torch.randint(0, 0x7E, kd.shape, device=dev, generator=g, dtype=torch.uint8)
            vq = torch.randint(0, 0x7E, kd.shape, device=dev, generator=g, dtype=torch.uint8)
            ks = torch.ones(B, HKV, ctx, device=dev)
            vs = torch.ones_like(ks)
            pos = torch.full((B,), ctx - 1, dtype=torch.int32, device=dev)
            ang = torch.rand(ctx + 1, 64, device=dev, generator=g)
            cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
            sc = DH ** -0.5
            fns = {"dense_bf16": lambda: ops.decode_attn(qkv, kd, vd, pos, cos, sin, HQ, HKV, DH, sc),
                   "dense_fp8": lambda: ops.decode_attn_fp8(qkv, kq, vq, ks, vs, pos, cos, sin, HQ, HKV, DH, sc)}
            pools = []
            for bs in (16, 64):
                mb = ctx // bs
                table = torch.randperm(B * mb, device=dev, generator=g).to(torch.int32).reshape(B, mb).contiguous()
                kp = torch.empty(B * mb, HKV, bs, DH, dtype=torch.bfloat16, device=dev)
                vp = torch.empty_like(kp)
                kp[table.long()] = kd.reshape(B, HKV, mb, bs, DH).transpose(1, 2)
                vp[table.long()] = vd.reshape(B, HKV, mb, bs, DH).transpose(1, 2)
                kpq = torch.empty(B * mb, HKV, bs, DH, dtype=torch.uint8, device=dev)
                vpq = torch.empty_like(kpq)
                kpq[table.long()] = kq.reshape(B, HKV, mb, bs, DH).transpose(1, 2)
                vpq[table.long()] = vq.reshape(B, HKV, mb, bs, DH).transpose(1, 2)
                ksp = torch.ones(B * mb, HKV, bs, device=dev)
                pools.append((kp, vp, kpq, vpq, ksp, table))
                fns[f"paged{bs}_bf16"] = (lambda kp=kp, vp=vp, t=table: ops.decode_attn_paged(
                    qkv, kp, vp, t, pos, cos, sin, HQ, HKV, DH, sc))
                fns[f"paged{bs}_fp8"] = (lambda kp=kpq, vp=vpq, s=ksp, t=table: ops.decode_attn_paged_fp8(
                    qkv, kp, vp, s, s, t, pos, cos, sin, HQ, HKV, DH, sc))
            t = {k: [] for k in fns}
            for _ in range(3):
                for k, fn in fns.items():
                    t[k].append(time_us(fn))
            row = {}
            for k, v in t.items():
                us = min(v)
                elem = 1 if k.endswith("fp8") else 2
                nbytes = 2 * B * HKV * ctx * (DH * elem + (4 if elem == 1 else 0))
                row[k] = {"us": round(us, 2), "spread_us": round(max(v) - us, 2), "kv_bytes": nbytes,
                          "GBps": round(nbytes / (us * 1e-6) / 1e9, 1)}
            for lay in ("dense", "paged16", "paged64"):
                row[f"{lay}_fp8_over_bf16"] = round(row[f"{lay}_fp8"]["us"] / row[f"{lay}_bf16"]["us"], 4)
            out[f"B={B} ctx={ctx}"] = row
            del kd, vd, kq, vq, pools, fns
            torch.cuda.empty_cache()
    return out


def _forced(g, new_positions):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    sched = []
    for _ in range(2):
        sched += torch.randint(0, 128000, (30,), generator=g).tolist() + [IMAGE_START_TOKEN_ID] + [7] * 64 + \
            [IMAGE_END_TOKEN_ID]
    sched += torch.randint(0, 128000, (new_positions - len(sched),), generator=g).tolist()
    return sched[:new_positions]


def decode_times(model, dev, prompt_len=128, new_positions=512):
    model.eval()
    out = {}
    for batch in (8, 32, 128):
        g = torch.Generator().manual_seed(batch)
        prompts = torch.randint(0, 128000, (batch, prompt_len), generator=g)
        forced = torch.tensor([_forced(g, new_positions)] * batch, dtype=torch.int32)
        emb = model.get_model().embed_tokens(prompts.to(dev))
        ms = {"bf16": [], "fp8_e4m3": []}
        for _ in range(2):
            for kvd in ms:
                model.greedy_decode(None, None, emb, max_new_tokens=new_positions - 1, output_image=True,
                                    forced_tokens=forced, kv_cache_dtype=kvd)
                torch.cuda.synchronize()
                t = model._decode.last_timing
                ms[kvd].append(t["decode_ms"] / t["steps"])
        out[f"batch={batch}"] = {"bf16_ms_per_step": round(min(ms["bf16"]), 4),
                                 "fp8_ms_per_step": round(min(ms["fp8_e4m3"]), 4),
                                 "fp8_over_bf16": round(min(ms["fp8_e4m3"]) / min(ms["bf16"]), 4)}
    return out


def _requests(model, dev, n_req, seed=11):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for _ in range(n_req):
        P = int(torch.randint(128, 1025, (1,), generator=g))
        n = int(torch.randint(96, 2049, (1,), generator=g))
        prompt = torch.randint(0, 128000, (1, P), generator=g)
        sched = torch.randint(0, 128000, (n + 2,), generator=g).to(torch.int32)
        sched[10] = IMAGE_START_TOKEN_ID
        sched[75] = IMAGE_END_TOKEN_ID
        reqs.append((model.get_model().embed_tokens(prompt.to(dev)), n, sched))
    return reqs


def serve_times(model, dev, n_req, pool_tokens):
    from metamorph_b200.engine.serve import ContinuousBatcher
    model.eval()
    reqs = _requests(model, dev, n_req)
    out = {}
    fp8_tokens = pool_tokens * 2 * DH // (DH + 4)
    for kvd, tokens in (("bf16", pool_tokens), ("fp8_e4m3", fp8_tokens)):
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        srv = ContinuousBatcher(model, max_slots=128, max_context=4096, max_new_tokens=2048, poll_every=8,
                                kv_pool_tokens=tokens, kv_block_size=64, kv_cache_dtype=kvd)
        pool_bytes = sum(t.numel() * t.element_size() for t in (srv.kc, srv.vc, *(srv.scales or ())))
        for e, n, f in reqs[:4]:                                   # warm-up (kernel attributes, graph capture)
            srv.submit(e, max_new_tokens=4, forced_tokens=f)
        srv.run_until_idle()
        torch.cuda.synchronize()
        for e, n, f in reqs:
            srv.submit(e, max_new_tokens=n, forced_tokens=f)
        occ, first = [], None
        step = srv._device_step

        def counted():
            occ.append(sum(s is not None for s in srv.slots))
            step()
        srv._device_step = counted
        steps0 = srv.steps_run
        t0 = time.perf_counter()
        got = 0
        for rid, kind, payload in srv.run():
            if kind == "ids" and first is None:
                torch.cuda.synchronize()
                first = time.perf_counter() - t0
            if kind == "done":
                got += int(payload[0].numel() + payload[1].shape[0])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        out[kvd] = {"pool_tokens": tokens, "pool_bytes": pool_bytes, "wall_s": round(dt, 2),
                    "device_steps": srv.steps_run - steps0, "positions_out": got,
                    "positions_per_s": round(got / dt, 1), "mean_occupied_slots": round(sum(occ) / max(len(occ), 1), 2),
                    "peak_allocated_GB": round(torch.cuda.max_memory_allocated() / 1e9, 2),
                    "first_ids_s": round(first, 3) if first is not None else None}
        del srv
    out["fp8_over_bf16_positions_per_s"] = round(out["fp8_e4m3"]["positions_per_s"] / out["bf16"]["positions_per_s"], 4)
    return out


def divergence(model, dev, n_req=16, new_positions=256):
    """Teacher-forced: the same schedule through a bf16 and an FP8 server; compares the per-step top-1 (logprobs=1) and
    the last step's logits row of slot 0."""
    from metamorph_b200.engine.serve import ContinuousBatcher
    model.eval()
    g = torch.Generator().manual_seed(5)
    reqs = []
    for _ in range(n_req):
        prompt = torch.randint(0, 128000, (1, 512), generator=g)
        reqs.append((model.get_model().embed_tokens(prompt.to(dev)), torch.tensor(_forced(g, new_positions) + [0, 0],
                                                                                    dtype=torch.int32)))
    res, logits = {}, {}
    for kvd in ("bf16", "fp8_e4m3"):
        srv = ContinuousBatcher(model, max_slots=n_req, max_context=1024, max_new_tokens=new_positions, poll_every=8,
                                kv_cache_dtype=kvd)
        rids = [srv.submit(e, max_new_tokens=new_positions, forced_tokens=f, logprobs=1) for e, f in reqs]
        r = srv.run_until_idle()
        res[kvd] = [r[i] for i in rids]
        logits[kvd] = srv.logits[:, :srv.V].clone()
        del srv
    d = (logits["bf16"] - logits["fp8_e4m3"]).abs()
    agree = total = 0
    cos = []
    for a, b in zip(res["bf16"], res["fp8_e4m3"]):
        ta, tb = a[2].top_ids[:, 0], b[2].top_ids[:, 0]
        agree += int((ta == tb).sum())
        total += ta.numel()
        if a[1].shape[0]:
            cos.append(float(torch.nn.functional.cosine_similarity(a[1].float(), b[1].float(), dim=-1).mean()))
    return {"note": "synthetic weights: a sanity figure, not a quality claim", "requests": n_req,
            "last_step_max_abs_dlogit": round(float(d.max()), 5), "last_step_mean_abs_dlogit": round(float(d.mean()), 6),
            "top1_agreement": round(agree / max(total, 1), 5), "steps_compared": total,
            "visual_embedding_cosine_mean": round(sum(cos) / len(cos), 6) if cos else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--serve-layers", type=int, default=32)
    ap.add_argument("--requests", type=int, default=192)
    ap.add_argument("--pool-tokens", type=int, default=131072)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: attention,decode,serve,divergence")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_kv_fp8_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    skip = set(filter(None, args.skip.split(",")))
    res = {"gpu": gpu_info(), "timed": "kernels: CUDA events; decode: DecodeEngine's device-event step time; serving: "
                                       "host clock around run() ending in a device synchronise"}
    from metamorph_b200 import synthetic
    if "attention" not in skip:
        res["attention"] = attention_times(dev)
        print(_save(res, args.out), flush=True)
    if "decode" not in skip or "divergence" not in skip:
        model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=args.layers)), device=dev)
        if "decode" not in skip:
            res["decode_step"] = {"layers": args.layers, **decode_times(model, dev)}
            print(_save(res, args.out), flush=True)
        if "divergence" not in skip:
            res["divergence"] = {"layers": args.layers, **divergence(model, dev)}
            print(_save(res, args.out), flush=True)
        del model
        gc.collect()
        torch.cuda.empty_cache()
    if "serve" not in skip:
        model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=args.serve_layers)), device=dev)
        res["serve"] = {"layers": args.serve_layers, "requests": args.requests,
                        **serve_times(model, dev, args.requests, args.pool_tokens)}
    print(_save(res, args.out), flush=True)


if __name__ == "__main__":
    main()
