#!/bin/bash
# Two-GPU evidence run: 1-vs-2-rank NCCL equality test, the DP bench line (ZeRO-1 sharded optimizer), A/B against the
# replicated optimizer, and the extra-config code path of the 8-GPU line on a shallow model.
mkdir -p gpurun_out
o=gpurun_out
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1"
timeout 400 python -m pytest tests/test_dp_nccl_gpu.py -m gpu -q -rs > $o/r02_nccl_test.log 2>&1
timeout 400 $TR --master-port 29511 bench.py --gpus 2 --steps 6 --warmup 3 > $o/r02_bench_n2.json 2> $o/r02_bench_n2.err
timeout 400 $TR --master-port 29513 bench.py --gpus 2 --steps 6 --warmup 3 --no-shard > $o/r02_bench_n2_noshard.json 2> $o/r02_bench_n2_noshard.err
timeout 300 $TR --master-port 29514 bench.py --gpus 2 --steps 3 --warmup 2 --layers 8 --extra-configs on > $o/r02_bench_n2_extra_l8.json 2> $o/r02_bench_n2_extra_l8.err
tail -5 $o/r02_nccl_test.log
for f in r02_bench_n2 r02_bench_n2_noshard r02_bench_n2_extra_l8; do python - "$o/$f.json" <<'PY'
import json, sys
try:
    d = json.load(open(sys.argv[1]))
    print(sys.argv[1], "ms/step", round(d["ms_per_step"], 1), "tok/s", round(d["value"]), "gemm TF/s", round(d["roofline"]["achieved"]),
          "state GB", d["config"].get("optimizer_state_gb_per_gpu"), "peak GB", d["config"].get("peak_hbm_gb"),
          {k: (v.get("value") and round(v["value"]), v.get("error")) for k, v in d.items() if k.startswith("config") and isinstance(v, dict) and k != "config"})
except Exception as e:
    print(sys.argv[1], "unreadable:", e)
PY
done
