"""Parity at the width the benchmark runs (VERDICT r1 item 1b): the CUDA hot path against digests of THE REFERENCE's own
forward / backward at LLaMA-3-8B layer dims (H=4096, 32 query / 8 kv heads, d=128, I=14336, V=128258), produced by
oracle/make_golden_realwidth.py:
  case A: 1 decoder layer, B=2: one sample of exactly T=4096 positions (32 key tiles, 2+2 images) and one ragged
          sample (2501 positions) right-padded next to it;
  case B: 2 decoder layers, batch length 1501 (T % 4 != 0: used to fall back to the mma.sync attention backward), one
          multimodal sample and one text-only sample with the dummy image.
This is the kernel combination of the benchmarked step: wgmma GEMMs at their default dispatch, GQA group 4 in
the wgmma attention forward/backward, the 16-row gate/up interleave at I=14336, lm_head row compaction at V=128258.
Tolerances as in tests/test_model_gpu.py: |ours - ref_fp32| <= 1.5 |ref_bf16 - ref_fp32| + floor for activations, losses
to 1e-3 relative, gradients by norm and by sampled entries (half of them the largest-magnitude entries)."""
import os

import pytest
import torch

from oracle.weights import REAL_A, REAL_B, make_batch_real, make_weights
from tests.helpers import build_product_model

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
CASES = {"A": (REAL_A, "realwidth_a.pt"), "B": (REAL_B, "realwidth_b.pt")}


@pytest.fixture(scope="module", params=["B", "A"])
def case(request, cuda_device):
    cfg, fname = CASES[request.param]
    fx = torch.load(os.path.join(G, fname), weights_only=False)
    W = make_weights(cfg)
    model = build_product_model(cfg, W)
    del W
    batch = make_batch_real(request.param, cfg)
    yield request.param, cfg, fx, model, batch
    del model
    torch.cuda.empty_cache()


def _budget(ours, ref32, ref16, floor, what):
    """The bf16 budget of tests/test_model_gpu.py AND a much tighter bound: the reference's eager bf16 run rounds after
    every op (its logits sit ~1.1 away from its own fp32 run at this width), the fused kernels keep fp32 accumulators:
    asserted <= 0.25 x the bf16 reference's own error."""
    err = (ours.float().cpu() - ref32).abs().max().item()
    ref_err = (ref16.float() - ref32).abs().max().item()
    bud = 1.5 * ref_err + floor
    rel_rms = ((ours.float().cpu() - ref32).pow(2).mean().sqrt() / ref32.pow(2).mean().sqrt()).item()
    print(f"[realwidth] {what}: |ours-fp32| = {err:.5f} (rms rel {rel_rms:.5f}, max |ref| {ref32.abs().max().item():.3f})  "
          f"budget {bud:.5f}  (|bf16ref-fp32| = {ref_err:.5f})")
    assert err <= bud, f"{what}: |ours-fp32|={err:.5f} > budget {bud:.5f}"
    assert err <= 0.25 * ref_err + floor, f"{what}: |ours-fp32|={err:.5f} not within a quarter of the bf16 reference's error {ref_err:.5f}"
    assert rel_rms <= 2e-2, f"{what}: rms relative error {rel_rms:.5f}"    # measured 0.4-1.2 % (bf16 operands, fp32 accumulation)


def test_realwidth_index_tensors_bit_exact(case):
    name, cfg, fx, model, (ids, mask, labs, images) = case
    plan = model.plan_inputs(ids, mask, labs, images.shape[0])
    assert plan.seq_len == fx["seq_len"]
    assert torch.equal(plan.labels.to(torch.int32), fx["new_labels"])
    assert torch.equal(plan.image_positions.to(torch.int8), fx["image_positions"])
    assert torch.equal(plan.attention_mask.bool(), fx["new_attention_mask"])


def test_realwidth_eval_forward(case):
    name, cfg, fx, model, (ids, mask, labs, images) = case
    model.eval()
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())
    pts = fx["points"].cuda()
    ours = out.logits[pts[:, 0], pts[:, 1]][:, fx["logit_cols"].cuda()]
    _budget(ours, fx["logits_sub"], fx["bf16"]["logits_sub"], 2e-3, f"case {name} logits")
    _budget(out.hidden_states[pts[:, 0], pts[:, 1], :64], fx["hidden_sub"], fx["bf16"]["hidden_sub"], 2e-3,
            f"case {name} hidden")
    for k in ("loss", "loss_language", "loss_image_ar"):
        ref = float(fx[k])
        got = float(out.loss) if k == "loss" else getattr(model, k)
        print(f"[realwidth] case {name} {k}: ours {got:.6f} ref fp32 {ref:.6f} ref bf16 {float(fx['bf16'][k]):.6f}")
        assert abs(got - ref) <= 1e-3 * abs(ref) + 2e-3, (k, got, ref)
    del out
    model.train()


def test_realwidth_train_gradients(case):
    name, cfg, fx, model, (ids, mask, labs, images) = case
    from metamorph_b200.engine.packing import deinterleave_gate_up
    model.train()
    model.zero_grad(set_to_none=True)
    out = model(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())
    assert out.logits is None
    assert abs(float(out.loss) - float(fx["loss"])) <= 1e-3 * abs(float(fx["loss"])) + 2e-3
    out.loss.backward()
    nq, nkv = cfg["heads"] * cfg["head_dim"], cfg["kv_heads"] * cfg["head_dim"]
    grads = {}
    for pname, p in model.named_parameters():
        if p.grad is None:
            continue
        g = p.grad.float().cpu()
        if pname.endswith("qkv_proj.weight"):
            base = pname[:-len("qkv_proj.weight")]
            grads[base + "q_proj.weight"], grads[base + "k_proj.weight"], grads[base + "v_proj.weight"] = \
                g[:nq], g[nq:nq + nkv], g[nq + nkv:]
        elif pname.endswith("gate_up_proj.weight"):
            base = pname[:-len("gate_up_proj.weight")]
            grads[base + "gate_proj.weight"], grads[base + "up_proj.weight"] = deinterleave_gate_up(g)
        else:
            grads[pname] = g
    checked, worst = 0, (0.0, None)
    for k, d in fx["grad_digest"].items():
        if k.startswith("model.vision_proj"):
            continue
        assert k in grads, f"missing gradient for {k}"
        g = grads[k]
        assert tuple(g.shape) == tuple(d["shape"]), (k, g.shape, d["shape"])
        ref_norm, got_norm = float(d["norm"]), float(g.norm())
        assert abs(got_norm - ref_norm) <= 3e-2 * ref_norm + 1e-6, (k, got_norm, ref_norm)
        vals = g.reshape(-1)[d["idx"]]
        scale = float(d["vals"].abs().max()) + 1e-12
        err = float((vals - d["vals"]).abs().max())
        rel = err / scale
        if rel > worst[0]:
            worst = (rel, k)
        assert err <= 4e-2 * scale + 1e-2 * ref_norm / (g.numel() ** 0.5), (k, err, scale)   # measured worst: 1.8e-2 of the max entry
        checked += 1
    print(f"[realwidth] case {name}: {checked} gradient tensors checked, worst sampled error {worst[0]:.4f} of max entry ({worst[1]})")
    assert checked >= 17
    model.zero_grad(set_to_none=True)
