"""Time the step's dominant GEMM shapes (CUDA events, L2-cold: operands > 126 MB)."""
import sys

import torch

sys.path.insert(0, ".")
from metamorph_b200 import ops  # noqa: E402

torch.manual_seed(0)
M = 16384
shapes = [("fwd gate/up  [M,4096]x[28672,4096]^T", (M, 28672, 4096), False, False),
          ("fwd down     [M,14336]x[4096,14336]^T", (M, 4096, 14336), False, False),
          ("dgrad gate/up [M,28672]x[28672,4096]", (M, 4096, 28672), False, True),
          ("wgrad gate/up [M,28672]^T x [M,4096]", (28672, 4096, M), True, True),
          ("fwd qkv      [M,4096]x[6144,4096]^T", (M, 6144, 4096), False, False)]
for name, (m, n, k), a_mn, b_mn in shapes:
    a = (torch.randn((k, m) if a_mn else (m, k), device="cuda") * 0.1).bfloat16()
    b = (torch.randn((k, n) if b_mn else (n, k), device="cuda") * 0.1).bfloat16()
    out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    it = 10
    e0.record()
    for _ in range(it):
        ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / it
    ref = (a.float().t() if a_mn else a.float())[:256] @ (b.float() if b_mn else b.float().t())
    err = (out[:256].float() - ref).abs().max().item() / (ref.abs().max().item() + 1e-9)
    print(f"{name}: {ms:.3f} ms  {2.0 * m * n * k / ms / 1e9:.0f} TFLOP/s  rel err {err:.2e}", flush=True)
    del a, b, out
