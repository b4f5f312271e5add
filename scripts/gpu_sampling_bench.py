"""Cost of seeded sampling on one GPU: CUDA-event time of mm_sample_rows against mm_argmax_rows per parameter mix, and
the decode step greedy against sampled at the decode_bench shapes (8 layers, 128-token prompts, 512 positions, the same
forced schedule, so both runs do the same work apart from the draw). Prints one JSON object; with --out also writes it.

    python scripts/gpu_sampling_bench.py --out build/sampling_bench.json
"""
import argparse
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")

V, LD = 128258, 128264
MIXES = {"T=0": (0.0, 0, 1.0), "T=1": (1.0, 0, 1.0), "T=1,k=50": (1.0, 50, 1.0), "T=1,p=0.9": (1.0, 0, 0.9),
         "T=1,k=50,p=0.9": (1.0, 50, 0.9)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None,
            "torch_name": torch.cuda.get_device_name(0)}


def time_us(fn, iters=200, warm=20):
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
    out = {}
    g = torch.Generator().manual_seed(0)
    for R in (1, 8, 32):
        buf = torch.randn(R, LD, generator=g) * 2.0
        for r in range(R):
            buf[r, torch.randperm(V, generator=g)[:200]] += 12.0
        buf = buf.to(dev)
        res = {}
        for rep in range(2):                                         # alternate argmax and the sampler
            res.setdefault("argmax", []).append(time_us(lambda: ops.argmax_rows(buf, V)))
            for name, (T, k, p) in MIXES.items():
                prm = (torch.full((R,), T, device=dev), torch.full((R,), k, dtype=torch.int32, device=dev),
                       torch.full((R,), p, device=dev), torch.arange(R, dtype=torch.int64, device=dev),
                       torch.zeros(R, dtype=torch.int32, device=dev))
                res.setdefault(name, []).append(time_us(lambda: ops.sample_rows(buf, V, *prm)))
        out[f"R={R}"] = {k: round(min(v), 2) for k, v in res.items()}
    return out


def decode_times(dev, layers=8, prompt_len=128, new_positions=512):
    from metamorph_b200 import synthetic
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.sampling import SamplingParams
    model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=layers)), device=dev)
    model.eval()
    out = {}
    for batch in (8, 32):
        g = torch.Generator().manual_seed(4321)
        prompts = torch.randint(0, 128000, (batch, prompt_len), generator=g)
        sched = []
        for _ in range(4):
            sched += torch.randint(0, 128000, (30,), generator=g).tolist() + [IMAGE_START_TOKEN_ID] + [7] * 64 + \
                [IMAGE_END_TOKEN_ID]
        sched += torch.randint(0, 128000, (new_positions - len(sched),), generator=g).tolist()
        forced = torch.tensor([sched[:new_positions]] * batch, dtype=torch.int32)
        emb = model.get_model().embed_tokens(prompts.to(dev))
        res = {"greedy": [], "sampled": []}
        for rep in range(4):                                         # alternate; the first pair is warm-up
            for name, sp in (("greedy", None), ("sampled", SamplingParams(temperature=1.0, top_k=50, top_p=0.9, seed=1))):
                model.greedy_decode(None, None, emb, max_new_tokens=new_positions - 1, output_image=True,
                                    forced_tokens=forced, sampling=sp)
                torch.cuda.synchronize()
                t = model._decode.last_timing
                if rep > 0:
                    res[name].append(t["decode_ms"] / t["steps"])
        g_ms, s_ms = min(res["greedy"]), min(res["sampled"])
        out[f"batch={batch}"] = {"greedy_ms_per_step": round(g_ms, 4), "sampled_ms_per_step": round(s_ms, 4),
                                 "sampled_over_greedy": round(s_ms / g_ms - 1, 4),
                                 "all_ms_per_step": {k: [round(x, 4) for x in v] for k, v in res.items()}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-decode", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_sampling_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "kernel_us": kernel_times(dev),
           "timed": "CUDA events: kernels over 200 back-to-back launches (min of 2 alternating rounds); decode steps "
                    "= DecodeEngine device time of 512 steps / steps (min of 3 alternating runs after one warm-up pair)"}
    if not args.no_decode:
        res["decode_step"] = decode_times(dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
