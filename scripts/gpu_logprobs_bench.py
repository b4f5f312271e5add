"""Cost of decode log-probabilities on one GPU. Prints one JSON object (and writes it with --out):
  * CUDA-event us of mm_decode_logprobs at V = 128258 for R in {1, 8, 32, 128} x n_top in {0, 5, 20}, beside
    mm_argmax_rows and temperature-only mm_sample_rows at the same R;
  * ms per decode step with and without logprobs=5 at batch 8, 32 and 128 on bench.decode_bench's workload (8 layers,
    128-token prompts, 512 positions with 4 x 64 visual embeddings);
  * serving positions/s on scripts/gpu_decode_wide_bench.py's 160 requests through 128 slots, every request at
    logprobs=5 against none, with the outputs asserted bit-equal;
  * the GPU's name, power limit and max SM clock, read in the same run.

    python scripts/gpu_logprobs_bench.py --out build/logprobs_bench.json
"""
import argparse
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None,
            "torch_name": torch.cuda.get_device_name(0)}


def time_us(fn, iters=200, warm=10):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def kernel_times(dev, V=128258):
    from metamorph_b200 import ops
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for R in (1, 8, 32, 128):
        logits = torch.randn(R, (V + 7) // 8 * 8, device=dev, generator=g) * 4
        zeros = torch.zeros(R, dtype=torch.int32, device=dev)          # append_kind 0 (every row reports), counter 0
        tok = torch.randint(0, V, (R,), device=dev, generator=g, dtype=torch.int32)
        picked = torch.empty(R, dtype=torch.int32, device=dev)
        n_ids = torch.ones(R, dtype=torch.int32, device=dev)
        lp = torch.empty(R, 4, device=dev)
        ids = torch.empty(R, 4, 20, dtype=torch.int32, device=dev)
        lps = torch.empty(R, 4, 20, device=dev)
        T = torch.ones(R, device=dev)
        k = torch.zeros(R, dtype=torch.int32, device=dev)
        p = torch.ones(R, device=dev)
        seed = torch.arange(R, dtype=torch.int64, device=dev)
        fns = {"argmax_rows": lambda: ops.argmax_rows(logits, V, out=picked),
               "sample_rows_T1": lambda: ops.sample_rows(logits, V, T, k, p, seed, zeros, out=picked)}
        for n in (0, 5, 20):
            nt = torch.full((R,), n, dtype=torch.int32, device=dev)
            fns[f"logprobs_n{n}"] = (lambda nt=nt: ops.decode_logprobs(logits, V, zeros, tok, n_ids, nt, lp, ids, lps))
        row = {}
        for rep in range(2):                                 # alternate the kernels; keep the faster round
            for key, fn in fns.items():
                row.setdefault(key, []).append(time_us(fn))
        out[f"R={R}"] = {k: round(min(v), 2) for k, v in row.items()}
    return out


def decode_step(model, dev, batch, logprobs, prompt_len=128, new_positions=512):
    """bench.decode_bench's forced schedule; ms per step of the 512 decode steps (device time), min of 2 runs."""
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    g = torch.Generator().manual_seed(4321)
    prompts = torch.randint(0, 128000, (batch, prompt_len), generator=g)
    sched = []
    for _ in range(4):
        sched += torch.randint(0, 128000, (30,), generator=g).tolist() + [IMAGE_START_TOKEN_ID] + [7] * 64 + \
            [IMAGE_END_TOKEN_ID]
    sched += torch.randint(0, 128000, (new_positions - len(sched),), generator=g).tolist()
    forced = torch.tensor([sched[:new_positions]] * batch, dtype=torch.int32)
    emb = model.get_model().embed_tokens(prompts.to(dev))
    ms, outs = [], None
    for _ in range(2):
        res = model.greedy_decode(None, None, emb, max_new_tokens=new_positions - 1, output_image=True,
                                  forced_tokens=forced, logprobs=logprobs)
        torch.cuda.synchronize()
        t = model._decode.last_timing
        ms.append(t["decode_ms"] / t["steps"])
        outs = res
    return min(ms), outs


def decode_times(model, dev):
    model.eval()
    out = {}
    for batch in (8, 32, 128):
        row = {}
        for rep in range(2):                                 # alternate off / on; keep the faster of each
            for key, n in (("off", None), ("logprobs5", 5)):
                ms, res = decode_step(model, dev, batch, n)
                row.setdefault(key, []).append(ms)
                if n is None:
                    ref = res
                else:
                    assert all(torch.equal(a, b) for a, b in zip(ref[0], res[0]))
                    assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(ref[1], res[1]))
        off, on = min(row["off"]), min(row["logprobs5"])
        out[f"batch={batch}"] = {"ms_per_step_off": round(off, 4), "ms_per_step_logprobs5": round(on, 4),
                                 "added_pct": round(100 * (on / off - 1), 2)}
    model.train()
    return out


def serve_times(model, dev, n_req=160, slots=128):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.serve import ContinuousBatcher
    model.eval()
    g = torch.Generator().manual_seed(7)
    P = 128
    lens = torch.randint(96, 513, (n_req,), generator=g).tolist()
    reqs = []
    for n in lens:
        prompt = torch.randint(0, 128000, (1, P), generator=g)
        sched = torch.randint(0, 128000, (n + 2,), generator=g).to(torch.int32)
        for s in range(20, n - 70, 150):                       # a 64-embedding image every ~150 positions
            sched[s] = IMAGE_START_TOKEN_ID
            sched[s + 65] = IMAGE_END_TOKEN_ID
        reqs.append((model.get_model().embed_tokens(prompt.to(dev)), n, sched))
    out, results = {}, {}
    for rep in range(2):
        for key, n_lp in (("off", None), ("logprobs5", 5)):
            srv = ContinuousBatcher(model, max_slots=slots, max_context=1024, max_new_tokens=512, poll_every=8)
            for e, n, f in reqs[:slots]:                       # warm-up pass (kernel attributes, graph capture)
                srv.submit(e, max_new_tokens=8, forced_tokens=f, logprobs=n_lp)
            srv.run_until_idle()
            torch.cuda.synchronize()
            rids = [srv.submit(e, max_new_tokens=n, forced_tokens=f, logprobs=n_lp) for e, n, f in reqs]
            t0 = time.perf_counter()
            res = srv.run_until_idle()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            got = sum(int(p[0].numel() + p[1].shape[0]) for p in res.values())
            out.setdefault(key, []).append(got / dt)
            results[key] = [res[r] for r in rids]
            del srv
            torch.cuda.empty_cache()
        for a, b in zip(results["off"], results["logprobs5"]):
            assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int16), b[1].view(torch.int16))
            assert b[2].logprob.numel() == a[0].numel()
    model.train()
    off, on = max(out["off"]), max(out["logprobs5"])
    return {f"{n_req} requests / {slots} slots": {"positions_per_s_off": round(off, 1),
                                                   "positions_per_s_logprobs5": round(on, 1),
                                                   "ratio": round(on / off, 4), "outputs_bit_equal": True}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: kernels,decode,serve")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_logprobs_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    skip = set(filter(None, args.skip.split(",")))
    res = {"gpu": gpu_info(),
           "timed": "kernels: CUDA events over 200 back-to-back launches, min of 2 alternating rounds; decode: CUDA "
                    "events around the 512 decode steps, min of 2 runs per setting, settings alternated; serving: host "
                    "clock around run_until_idle ending in a device synchronise, best of 2 alternated runs"}
    if "kernels" not in skip:
        res["kernel_us"] = kernel_times(dev)
    if not {"decode", "serve"} <= skip:
        from metamorph_b200 import synthetic
        model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=args.layers)), device=dev)
        if "decode" not in skip:
            res["decode"] = decode_times(model, dev)
        if "serve" not in skip:
            res["serve"] = serve_times(model, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
