"""Attention microbench at the train-step shape (B=4, T=4096, 32q/8kv heads, d=128)."""
import math
import sys

import torch

sys.path.insert(0, ".")
from metamorph_b200 import ops  # noqa: E402


def timeit(fn, iters=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    B, T, Hq, Hkv, d = 4, 4096, 32, 8, 128
    torch.manual_seed(0)
    qkv = (torch.randn(B * T, (Hq + 2 * Hkv) * d, device="cuda") * 0.5).bfloat16()
    q, k, v = qkv[:, :Hq * d], qkv[:, Hq * d:(Hq + Hkv) * d], qkv[:, (Hq + Hkv) * d:]
    scale = 1 / math.sqrt(d)
    fl_fwd = 4 * B * Hq * T * T * d / 2
    ms = timeit(lambda: ops.attn_fwd(q, k, v, B, T, Hq, Hkv, d, True, scale))
    print(f"fwd: {ms:.3f} ms  {fl_fwd/ms/1e9:.1f} TFLOP/s", flush=True)
    o, lse = ops.attn_fwd(q, k, v, B, T, Hq, Hkv, d, True, scale)
    dout = torch.randn_like(o)
    dqkv = torch.zeros_like(qkv)
    ms = timeit(lambda: ops.attn_bwd(q, k, v, o, dout, lse, dqkv[:, :Hq * d], dqkv[:, Hq * d:(Hq + Hkv) * d],
                                     dqkv[:, (Hq + Hkv) * d:], B, T, Hq, Hkv, d, scale), iters=3)
    print(f"bwd: {ms:.3f} ms  {2.5*fl_fwd/ms/1e9:.1f} TFLOP/s", flush=True)


if __name__ == "__main__":
    main()
