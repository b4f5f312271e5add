"""1-vs-N-rank equality ON HARDWARE (SURVEY.md section 4 "multi-GPU"; VERDICT r1 weak 4): the 2-rank NCCL step
(reduce-scatter -> sharded AdamW -> all-gather, engine/trainer.py) on a global batch of two halves must leave the
parameters that a single rank computes from the same two halves as micro-batches (mean of the two gradients — the
data-parallel semantics of the reference under DDP / ZeRO: each rank averages over its own micro-batch, ranks are
averaged). Needs 2 GPUs: `python -m pytest tests/test_dp_nccl_gpu.py -m gpu` on a 2-GPU machine; skipped on 1 GPU."""
import os
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu


def _halves():
    from oracle.weights import TINY, make_batch
    out = []
    for seed in (1, 7):
        ids, mask, labs, images = make_batch(TINY, seed=seed)
        out.append(dict(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16()))
    return out


def _rank_main(rank, world, init_file, out_dir, shard, fused):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method=f"file://{init_file}", rank=rank, world_size=world,
                            device_id=torch.device("cuda", rank))
    from metamorph_b200.engine.trainer import TrainEngine
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    model = build_product_model(TINY, make_weights(TINY), device=f"cuda:{rank}")
    eng = TrainEngine(model, lr=1e-3, constant_lr=True, shard_optimizer=shard, fused_allgather=fused)
    assert eng.world == 2 and eng.shard_world == (2 if shard else 1)
    if fused:
        assert eng.fused_allgather, "symmetric memory / fused all-gather could not be set up on this box"
        assert all(b.symm is not None for b in eng.layer_buckets)
    halves = _halves()
    for _ in range(2):
        out = eng.step(halves[rank])
    torch.cuda.synchronize()
    sd = {n: p.detach().float().cpu() for n, p in model.named_parameters() if p.requires_grad}
    mc = bool(eng.fused_allgather and int(eng.layer_buckets[0].symm.multicast_ptr or 0))
    torch.save(dict(params=sd, loss=float(out["loss"]), state_bytes=eng.optimizer_state_bytes(), multicast=mc,
                    fused_reduce=bool(eng.fused_reduce)),
               os.path.join(out_dir, f"rank{rank}_{int(shard)}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("shard,fused", [(True, True), (True, False), (False, False)])
def test_two_rank_step_equals_one_rank_accumulated_step(cuda_device, shard, fused):
    """shard + fused: reduce-scatter -> ONE kernel doing AdamW on the slice and the all-gather (multimem.st through the
    NVSwitch multicast address of the symmetric parameter buffer, or P2P stores); shard only: NCCL all-gather;
    neither: replicated optimizer with an all-reduce."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from metamorph_b200.engine.trainer import TrainEngine
    from oracle.weights import TINY, make_weights
    from tests.helpers import build_product_model
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_rank_main, args=(2, os.path.join(d, "init"), d, shard, fused), nprocs=2, join=True)
        r0 = torch.load(os.path.join(d, f"rank0_{int(shard)}.pt"))
        r1 = torch.load(os.path.join(d, f"rank1_{int(shard)}.pt"))
    for n in r0["params"]:                                     # the replicas stay bit-identical
        assert torch.equal(r0["params"][n], r1["params"][n]), n
    model = build_product_model(TINY, make_weights(TINY))
    eng = TrainEngine(model, lr=1e-3, constant_lr=True, gradient_accumulation_steps=2)
    halves = _halves()
    for _ in range(2):
        out = eng.step(halves)
    torch.cuda.synchronize()
    if shard:
        assert r0["state_bytes"] < 0.55 * eng.optimizer_state_bytes()       # the big buckets hold half of the state
    if fused:
        print(f"[nccl] fused AdamW + all-gather ran with {'NVSwitch multicast (multimem.st)' if r0['multicast'] else 'per-peer P2P stores'}"
              f"; reduce-scatter {'fused too (multimem.ld_reduce, in-switch sum)' if r0['fused_reduce'] else 'through NCCL'}")
    assert abs(out["loss"].item() - 0.5 * (r0["loss"] + r1["loss"])) < 2e-3
    for n, p in model.named_parameters():
        if not p.requires_grad or "vision_proj" in n:
            continue
        a, b = p.detach().float().cpu(), r0["params"][n]
        frac_bad = float(((a - b).abs() > 2.4e-3 + 8e-3 * b.abs()).float().mean())
        assert frac_bad < 3e-3, (n, frac_bad, float((a - b).abs().max()))
