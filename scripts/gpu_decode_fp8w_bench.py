"""FP8 (E4M3) weights against bf16 weights on one GPU, alternating the two in one process on the same seeded inputs.
Prints one JSON object (and writes it with --out):
  * decode: greedy_decode of the synthetic model (--layers, default 8, LLaMA-3-8B widths) at batch 1, 8, 32, 64 and 128,
    128-position prompts and 512 forced new positions (four 64-row images); ms per step from DecodeEngine's CUDA events
    around the decode steps (min of 2 alternating rounds), the weight bytes a step streams and that stream's share of
    the 3.35 TB/s HBM floor (weight bytes / 3.35 TB/s over the step time; KV and activations not counted);
  * quantisation: DecodeEngine's quant_ms (every decoder-layer matrix and lm_head);
  * prefill: the added cost per admission, CUDA events around the per-layer dequantise into the bf16 scratch layer for
    every layer (what an FP8 server adds to each prefill);
  * serving: ContinuousBatcher on the README's mix (160 requests, 128-position prompts, 96-512 new positions with an
    image every ~150) through 32 and 128 slots, positions/s (host clock around run_until_idle ending in a synchronise);
  * the GPU's name, power limit and max SM clock, read in the same run.

    python scripts/gpu_decode_fp8w_bench.py --out build/decode_fp8w_bench.json
"""
import argparse
import json
import sys
import time

import torch

sys.path.insert(0, ".")

from scripts.gpu_decode_wide_bench import gpu_info  # noqa: E402

HBM = 3.35e12
WD = ("bf16", "fp8_e4m3")


def weight_bytes(model):
    """Bytes of the matrices one decode step streams, bf16 and FP8 (1 byte per weight + 4 per 128); the norms, the
    vision head and the projector (bf16 either way) are left out."""
    n = sum(p.numel() for l in model.get_model().layers
            for p in (l.self_attn.qkv_proj.weight, l.self_attn.o_proj.weight, l.mlp.gate_up_proj.weight,
                      l.mlp.down_proj.weight)) + model.lm_head.weight.numel()
    return {"params": n, "bf16": 2 * n, "fp8_e4m3": n + 4 * n // 128}


def _forced(g, new_positions):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    sched = []
    for _ in range(4):
        sched += torch.randint(0, 128000, (30,), generator=g).tolist() + [IMAGE_START_TOKEN_ID] + [7] * 64 + \
            [IMAGE_END_TOKEN_ID]
    sched += torch.randint(0, 128000, (new_positions - len(sched),), generator=g).tolist()
    return sched[:new_positions]


def decode_times(model, dev, prompt_len=128, new_positions=512):
    wb = weight_bytes(model)
    out, quant = {}, []
    for batch in (1, 8, 32, 64, 128):
        g = torch.Generator().manual_seed(batch)
        prompts = torch.randint(0, 128000, (batch, prompt_len), generator=g)
        forced = torch.tensor([_forced(g, new_positions)] * batch, dtype=torch.int32)
        emb = model.get_model().embed_tokens(prompts.to(dev))
        ms = {w: [] for w in WD}
        for _ in range(2):
            for w in WD:
                model.greedy_decode(None, None, emb, max_new_tokens=new_positions - 1, output_image=True,
                                    forced_tokens=forced, weight_dtype=w)
                torch.cuda.synchronize()
                t = model._decode.last_timing
                ms[w].append(t["decode_ms"] / t["steps"])
                if w == "fp8_e4m3":
                    quant.append(t["quant_ms"])
        r = {}
        for w in WD:
            best = min(ms[w])
            r[w] = {"ms_per_step": round(best, 4), "weight_GB_per_step": round(wb[w] / 1e9, 3),
                    "weight_floor_ms": round(wb[w] / HBM * 1e3, 4), "share_of_floor": round(wb[w] / HBM * 1e3 / best, 4)}
        r["fp8_over_bf16"] = round(r["fp8_e4m3"]["ms_per_step"] / r["bf16"]["ms_per_step"], 4)
        out[f"batch={batch}"] = r
    return out, {"quant_ms_min": round(min(quant), 3), "quant_ms_max": round(max(quant), 3), "params": wb["params"]}


def prefill_dequant_ms(model):
    from metamorph_b200.engine.fp8_weights import decode_weights
    dw = decode_weights(model, "fp8_e4m3")
    L = len(dw.layers)
    for i in range(L):                                           # warm-up
        dw.prefill_layer(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        for i in range(L):
            dw.prefill_layer(i)
    e1.record()
    torch.cuda.synchronize()
    return {"layers": L, "ms_per_admission": round(e0.elapsed_time(e1) / reps, 4)}


def serve_times(model, dev):
    from metamorph_b200.constants import IMAGE_END_TOKEN_ID, IMAGE_START_TOKEN_ID
    from metamorph_b200.engine.serve import ContinuousBatcher
    out = {}
    for n_req, slots in ((160, 32), (160, 128)):
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
        r = {w: [] for w in WD}
        for _ in range(2):
            for w in WD:
                srv = ContinuousBatcher(model, max_slots=slots, max_context=1024, max_new_tokens=512, poll_every=8,
                                        weight_dtype=w)
                for e, n, f in reqs[:slots]:                   # warm-up pass (kernel attributes, graph capture)
                    srv.submit(e, max_new_tokens=8, forced_tokens=f)
                srv.run_until_idle()
                torch.cuda.synchronize()
                for e, n, f in reqs:
                    srv.submit(e, max_new_tokens=n, forced_tokens=f)
                t0 = time.perf_counter()
                res = srv.run_until_idle()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                got = sum(int(i.numel() + im.shape[0]) for i, im in res.values())
                r[w].append(got / dt)
                del srv
                torch.cuda.empty_cache()
        out[f"{n_req} requests / {slots} slots"] = {**{w: {"positions_per_s": round(max(r[w]), 1)} for w in WD},
                                                    "fp8_over_bf16": round(max(r["fp8_e4m3"]) / max(r["bf16"]), 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: decode,prefill,serve")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_decode_fp8w_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    skip = set(filter(None, args.skip.split(",")))
    res = {"gpu": gpu_info(), "layers": args.layers,
           "timed": "decode: DecodeEngine's CUDA events around the decode steps; prefill: CUDA events; serving: host "
                    "clock around run_until_idle ending in a device synchronise"}
    from metamorph_b200 import synthetic
    model = synthetic.build_model(synthetic.make_config(llama=dict(num_hidden_layers=args.layers)), device=dev)
    model.eval()
    if "decode" not in skip:
        res["decode"], res["quantise"] = decode_times(model, dev)
    if "prefill" not in skip:
        res["prefill_dequant"] = prefill_dequant_ms(model)
    if "serve" not in skip:
        res["serve"] = serve_times(model, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
