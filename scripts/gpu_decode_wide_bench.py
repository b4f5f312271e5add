"""Decode and serving above 32 sequences per step on one GPU. Prints one JSON object (and writes it with --out):
  * bench.decode_bench's workload (8 layers, 128-token prompts, 512 positions with 4 x 64 visual embeddings) at batches
    8, 32, 64, 96 and 128: ms per step, tokens/s and HBM bytes/s against 3.35 TB/s; one sampled (T + top-k + top-p) run
    at 128;
  * CUDA-event time of the wide GEMM at the five LLaMA-3-8B decode shapes for m = 64 and 128, beside the skinny kernel at
    m = 32 and the training GEMM (mm_gemm_bf16) at m = 128;
  * continuous batching as scripts/gpu_serve_bench.py: 24 requests through 8 slots, 160 through 32 and through 128;
  * the GPU's name and power limit, read in the same run.

    python scripts/gpu_decode_wide_bench.py --out build/decode_wide_bench.json
"""
import argparse
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")

SHAPES = {"qkv 6144x4096": (6144, 4096, "store"), "o_proj 4096x4096 +resid": (4096, 4096, "resid"),
          "gate/up 28672x4096 swiglu": (28672, 4096, "swiglu"), "down 4096x14336 +resid": (4096, 14336, "resid"),
          "lm_head 128258x4096 fp32": (128258, 4096, "f32")}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None,
            "torch_name": torch.cuda.get_device_name(0)}


def time_us(fn, iters=100, warm=10):
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
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for name, (N, K, epi) in SHAPES.items():
        w = (torch.randn(N, K, device=dev, generator=g) * 0.02).bfloat16()
        x = torch.randn(128, K, device=dev, generator=g).bfloat16()
        res = torch.randn(128, N, device=dev, generator=g).bfloat16()
        logits = torch.empty(128, (N + 7) // 8 * 8, device=dev)

        def skinny(m, wide):
            kw = {}
            if epi == "resid":
                kw = dict(resid=res[:m], epilogue=ops.SK_RESID)
            elif epi == "swiglu":
                kw = dict(epilogue=ops.SK_SWIGLU)
            elif epi == "f32":
                kw = dict(out=logits[:m, :N])
            return lambda: ops.skinny_gemm(x[:m], w, wide=wide, **kw)

        row = {}
        for rep in range(2):                                 # alternate the kernels; keep the faster round
            for key, fn in (("skinny_m32", skinny(32, False)), ("wide_m64", skinny(64, True)),
                            ("wide_m128", skinny(128, True)),
                            ("gemm_bf16_m128", lambda: ops.gemm(x, w, out=logits[:, :N], out_dtype=torch.float32) if epi == "f32"
                             else ops.gemm(x, w))):
                row.setdefault(key, []).append(time_us(fn))
        row = {k: round(min(v), 2) for k, v in row.items()}
        wbytes = N * K * 2
        row["weight_GBps_wide_m128"] = round(wbytes / (row["wide_m128"] * 1e-6) / 1e9, 1)
        row["weight_GBps_skinny_m32"] = round(wbytes / (row["skinny_m32"] * 1e-6) / 1e9, 1)
        out[name] = row
        del w, x, res, logits
        torch.cuda.empty_cache()
    return out


def decode_times(model, dev, layers):
    import bench
    res = {}
    for batch in (8, 32, 64, 96, 128):
        r = bench.decode_bench(model, dev, {}, layers, batch=batch)
        res[f"batch={batch}"] = {"ms_per_step": round(r["ms_per_step"], 4), "tokens_per_s": round(r["value"], 1),
                                 "hbm_GBps": round(r["roofline"]["achieved"], 1),
                                 "hbm_frac_of_3350": round(r["roofline"]["frac"], 4)}
    return res


def sampled_decode(model, dev, batch=128, prompt_len=128, new_positions=512):
    """decode_bench's workload at batch 128 with every sequence sampling (T = 1, top-k 50, top-p 0.9)."""
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.sampling import SamplingParams
    g = torch.Generator().manual_seed(4321)
    prompts = torch.randint(0, 128000, (batch, prompt_len), generator=g)
    sched = []
    for _ in range(4):
        sched += torch.randint(0, 128000, (30,), generator=g).tolist() + [IMAGE_START_TOKEN_ID] + [7] * 64 + \
            [IMAGE_END_TOKEN_ID]
    sched += torch.randint(0, 128000, (new_positions - len(sched),), generator=g).tolist()
    forced = torch.tensor([sched[:new_positions]] * batch, dtype=torch.int32)
    emb = model.get_model().embed_tokens(prompts.to(dev))
    model.eval()
    ms = []
    for rep in range(2):
        model.greedy_decode(None, None, emb, max_new_tokens=new_positions - 1, output_image=True, forced_tokens=forced,
                            sampling=SamplingParams(temperature=1.0, top_k=50, top_p=0.9, seed=1))
        torch.cuda.synchronize()
        t = model._decode.last_timing
        ms.append(t["decode_ms"] / t["steps"])
    model.train()
    return {"batch": batch, "ms_per_step": round(min(ms), 4), "tokens_per_s": round(batch / (min(ms) / 1e3), 1)}


def serve_times(model, dev):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.serve import ContinuousBatcher
    model.eval()
    out = {}
    for n_req, slots in ((24, 8), (160, 32), (160, 128)):
        g = torch.Generator().manual_seed(7)
        P = 128
        lens = torch.randint(96, 513, (n_req,), generator=g).tolist()
        reqs = []
        for n in lens:
            prompt = torch.randint(0, 128000, (1, P), generator=g)
            sched = torch.randint(0, 128000, (n + 2,), generator=g).to(torch.int32)
            for s in range(20, n - 70, 150):                   # a 64-embedding image every ~150 positions
                sched[s] = IMAGE_START_TOKEN_ID
                sched[s + 65] = IMAGE_END_TOKEN_ID
            reqs.append((model.get_model().embed_tokens(prompt.to(dev)), n, sched))
        srv = ContinuousBatcher(model, max_slots=slots, max_context=1024, max_new_tokens=512, poll_every=8)
        for e, n, f in reqs[:slots]:                           # warm-up pass (kernel attributes, graph capture)
            srv.submit(e, max_new_tokens=8, forced_tokens=f)
        srv.run_until_idle()
        torch.cuda.synchronize()
        for e, n, f in reqs:
            srv.submit(e, max_new_tokens=n, forced_tokens=f)
        steps0 = srv.steps_run
        t0 = time.perf_counter()
        res = srv.run_until_idle()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        got = sum(int(i.numel() + im.shape[0]) for i, im in res.values())
        out[f"{n_req} requests / {slots} slots"] = {"wall_s": round(dt, 3), "device_steps": srv.steps_run - steps0,
                                                    "positions_out": got, "positions_per_s": round(got / dt, 1)}
        del srv
        torch.cuda.empty_cache()
    model.train()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: kernels,decode,serve")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_decode_wide_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    skip = set(filter(None, args.skip.split(",")))
    res = {"gpu": gpu_info(),
           "timed": "kernels: CUDA events over 100 back-to-back launches, min of 2 alternating rounds; decode: "
                    "bench.decode_bench (CUDA events around the 512 decode steps); serving: host clock around "
                    "run_until_idle ending in a device synchronise"}
    if "kernels" not in skip:
        res["kernel_us"] = kernel_times(dev)
    if not {"decode", "serve"} <= skip:
        from metamorph_b200 import synthetic
        model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=args.layers)), device=dev)
        if "decode" not in skip:
            res["decode"] = decode_times(model, dev, args.layers)
            res["decode_sampled_T1_k50_p0.9"] = sampled_decode(model, dev)
            d = res["decode"]
            res["batch128_over_batch32_tokens_per_s"] = round(d["batch=128"]["tokens_per_s"] /
                                                              d["batch=32"]["tokens_per_s"], 3)
        if "serve" not in skip:
            res["serve"] = serve_times(model, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
