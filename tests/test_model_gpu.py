"""Model-level parity on H100: the CUDA hot path (through the C-ABI) against (a) golden vectors made
by the reference itself (fp32 and bf16 runs, tests/golden/) and (b) the fp32 oracle restatement.

Tolerances. The reference runs this path in bf16 with a rounding after every op; the fused kernels
keep fp32 longer. Following SURVEY.md §7, errors are budgeted against the fp32 reference run:
    |ours - ref_fp32| <= 1.5 * |ref_bf16 - ref_fp32| + small absolute floor
and scalar losses must agree to 1e-3 relative (north_star tolerance) + 2e-3 absolute."""
import os

import pytest
import torch

from oracle import restatement as R
from oracle.weights import TINY, make_batch, make_weights
from tests.helpers import build_product_model

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def fb():
    return torch.load(os.path.join(G, "forward_backward_tiny.pt"), weights_only=False)


@pytest.fixture(scope="module")
def weights():
    return make_weights(TINY)


@pytest.fixture(scope="module")
def model(cuda_device, weights):
    return build_product_model(TINY, weights)


def _budget(ours, ref32, ref16, floor, what):
    err = (ours.float().cpu() - ref32).abs().max().item()
    bud = 1.5 * (ref16.float() - ref32).abs().max().item() + floor
    assert err <= bud, f"{what}: |ours-fp32|={err:.5f} > budget {bud:.5f}"


def test_state_dict_roundtrip_reference_names(model, weights):
    sd = model.state_dict()
    for k, v in weights.items():
        assert k in sd, k
        assert torch.equal(sd[k].float().cpu(), v.bfloat16().float()), k
    assert "model.layers.0.self_attn.q_proj.weight" in sd and "model.layers.0.mlp.gate_proj.weight" in sd


def test_prepare_inputs_matches_reference(model, fb):
    ids, mask, labs, images = make_batch(TINY)
    with torch.no_grad():
        out = model.prepare_inputs_labels_for_multimodal(ids.cuda(), None, mask.cuda(), None, labs.cuda(),
                                                         images.cuda().bfloat16())
    _, pos, am, _, emb, nl, ip, tgt = out
    assert torch.equal(nl.cpu(), fb["new_labels"])                     # bit-exact integers
    assert torch.equal(ip.cpu(), fb["image_positions"])
    assert torch.equal(am.cpu().bool(), fb["new_attention_mask"].bool())
    ref_sum = fb["inputs_embeds_sum"]
    err = (emb.float().sum(-1).cpu() - ref_sum).abs().max().item()
    assert err < 0.15, err                                             # sums of 256 bf16-rounded values
    torch.testing.assert_close(tgt.float().cpu(), fb["targets"], rtol=2e-2, atol=2e-3)


def test_eval_forward_logits_and_losses(model, fb):
    ids, mask, labs, images = make_batch(TINY)
    model.eval()
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())
    valid = fb["new_attention_mask"].bool()
    ours = out.logits[..., fb["logit_cols"].cuda()].float().cpu()
    _budget(ours[valid], fb["logits_sub"][valid], fb["bf16"]["logits_sub"][valid], 2e-3, "logits")
    _budget(out.hidden_states[..., :32].cpu()[valid], fb["hidden_sub"][valid], fb["bf16"]["hidden_sub"][valid],
            2e-3, "hidden")
    for k in ("loss", "loss_language", "loss_image_ar"):
        ref = float(fb[k])
        got = float(out.loss) if k == "loss" else getattr(model, k)
        assert abs(got - ref) <= 1e-3 * abs(ref) + 2e-3, (k, got, ref)


def test_train_forward_backward_gradients(model, fb):
    ids, mask, labs, images = make_batch(TINY)
    model.train()
    model.zero_grad(set_to_none=True)
    out = model(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())
    assert out.logits is None
    assert abs(float(out.loss) - float(fb["loss"])) <= 1e-3 * abs(float(fb["loss"])) + 2e-3
    out.loss.backward()
    sd_grads = {}
    from metamorph_b200.engine.packing import deinterleave_gate_up
    for name, p in model.named_parameters():
        if p.grad is None:
            continue
        g = p.grad.float().cpu()
        if name.endswith("qkv_proj.weight"):
            base = name[:-len("qkv_proj.weight")]
            sd_grads[base + "q_proj.weight"], sd_grads[base + "k_proj.weight"], sd_grads[base + "v_proj.weight"] = \
                g[:256], g[256:384], g[384:]
        elif name.endswith("gate_up_proj.weight"):
            base = name[:-len("gate_up_proj.weight")]
            sd_grads[base + "gate_proj.weight"], sd_grads[base + "up_proj.weight"] = deinterleave_gate_up(g)
        else:
            sd_grads[name] = g
    checked = 0
    for k, d in fb["grad_digest"].items():
        if k.startswith("model.vision_proj"):
            continue
        assert k in sd_grads, f"missing gradient for {k}"
        g = sd_grads[k]
        ref_norm = float(d["norm"])
        got_norm = float(g.norm())
        assert abs(got_norm - ref_norm) <= 5e-2 * ref_norm + 1e-6, (k, got_norm, ref_norm)
        vals = g.reshape(-1)[d["idx"]]
        scale = float(d["vals"].abs().max()) + 1e-9
        err = float((vals - d["vals"]).abs().max())
        assert err <= 8e-2 * scale + 2e-2 * ref_norm / (g.numel() ** 0.5), (k, err, scale)
        checked += 1
    assert checked >= 25


def test_decode_kv_cache_matches_reference_nocache(cuda_device, weights):
    d = torch.load(os.path.join(G, "greedy_decode_tiny.pt"), weights_only=False)
    model = build_product_model(TINY, weights, num_image_tokens=d["num_image_tokens"])
    model.eval()
    ref_ids = d["ids"]
    # Free-running decode: with random weights the top-2 logit gap at step 0 is 0.2 % (1.2413 vs 1.2388 in the
    # fp32 reference), below bf16 resolution, so token-exactness is only asserted teacher-forced (below). Here:
    # the run terminates, and its first token is one of the reference's top-3 candidates.
    ids, img = model.generate(d["prompt"].cuda(), output_image=True, max_new_tokens=d["max_new_tokens"],
                              start_image_token_id=d["start_image_token_id"])
    got = ids[0].cpu().tolist()
    x0 = weights["model.embed_tokens.weight"][d["prompt"]]
    T0 = x0.shape[1]
    hid = R.llama_forward(weights, x0.float(), torch.arange(T0)[None], torch.ones(1, T0, dtype=torch.bool),
                          TINY["layers"], TINY["heads"], TINY["kv_heads"], TINY["rms_eps"], TINY["rope_theta"])
    top3 = torch.nn.functional.linear(hid[:, -1], weights["lm_head.weight"])[0].topk(3).indices.tolist()
    assert got[0] in top3 and 1 <= len(got) <= d["max_new_tokens"] + 1
    # teacher-forced on the reference's ids: every visual embedding must match
    steps = d["max_new_tokens"] + 1
    forced = torch.zeros((1, steps + 2), dtype=torch.int32)
    seq = [int(ref_ids[0])] + [0] * d["num_image_tokens"] + [int(t) for t in ref_ids[1:]]
    forced[0, :len(seq)] = torch.tensor(seq[:steps + 2], dtype=torch.int32)
    emb = model.get_model().embed_tokens(d["prompt"].cuda())
    ids2, img2 = model.greedy_decode(None, None, emb, start_image_token_id=d["start_image_token_id"],
                                     max_new_tokens=d["max_new_tokens"], output_image=True, forced_tokens=forced)
    torch.testing.assert_close(img2.float().cpu(), d["image_embeds"], rtol=5e-2, atol=5e-3)
    assert ids2[0].cpu().tolist() == [int(t) for t in ref_ids]


@pytest.mark.parametrize("quirk", ["q1", "q2"])
def test_decode_free_running_reference_quirks(cuda_device, weights, quirk):
    """FREE-RUNNING (no teacher forcing) token-exactness against the reference's own generate() on prompts whose every
    step has a top-1/top-2 logit margin far above bf16 noise (oracle/make_golden_decode_quirks.py), covering the two
    state-machine quirks of metamorph_llama.py:502-597: q1 = EOS raised by the overwritten hidden state in the middle of
    an image (fewer than num_image_tokens embeddings come back); q2 = a second <image_start> before any <image_end>
    (tokens keep being appended as text while every step runs the decoding branch)."""
    allq = torch.load(os.path.join(G, "greedy_decode_quirks.pt"), weights_only=False)
    d = allq[quirk]
    from oracle.weights import with_sparse_lm_head
    model = build_product_model(TINY, with_sparse_lm_head(weights, d["live_rows"])[0], num_image_tokens=d["num_image_tokens"])
    model.eval()
    ids, img = model.generate(d["prompt"].cuda(), output_image=True, max_new_tokens=d["max_new_tokens"],
                              start_image_token_id=d["start_image_token_id"],
                              end_image_token_id=d["end_image_token_id"], eos_token_id=list(d["eos_token_id"]))
    assert ids[0].cpu().tolist() == [int(t) for t in d["ids"]], (quirk, ids[0].cpu().tolist(), d["ids"].tolist(), d["min_margin"])
    assert tuple(img.shape) == tuple(d["image_embeds"].shape)
    if quirk == "q1":
        assert img.shape[0] < d["num_image_tokens"]                  # generation ended inside the image
    else:
        modes = [m for _, m, _ in d["trace"]]
        assert any(modes[k] and d["trace"][k][2] == d["num_image_tokens"] for k in range(len(modes)))   # stuck-in-image state reached
    # unit-norm embeddings: 1e-2 absolute = the bf16 budget of a 2-layer path (north star: 1e-3 relative on logits)
    torch.testing.assert_close(img.float().cpu(), d["image_embeds"], rtol=0, atol=1e-2)


def test_left_padded_ragged_batch_matches_reference(cuda_device, weights):
    """tokenizer_padding_side == "left" (metamorph_arch.py:373-386) with ragged lengths: every sample sits at the END of
    its batch row; the fused attention handles it through the segment tables (round 1 raised NotImplementedError).
    Golden = the reference's own forward (oracle/make_golden_leftpad.py)."""
    lp = torch.load(os.path.join(G, "leftpad_tiny.pt"), weights_only=False)
    model = build_product_model(TINY, weights)
    model.config.tokenizer_padding_side = "left"
    ids, mask, labs, images = make_batch(TINY)
    plan = model.plan_inputs(ids, mask, labs, images.shape[0])
    assert torch.equal(plan.labels, lp["new_labels"]) and torch.equal(plan.attention_mask.bool(), lp["new_attention_mask"].bool())
    assert torch.equal(plan.image_positions, lp["image_positions"])
    for mode in ("eval", "train"):
        getattr(model, mode)()
        with torch.set_grad_enabled(mode == "train"):
            out = model(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())
        for k in ("loss", "loss_language", "loss_image_ar"):
            ref = float(lp["fp32"][k])
            got = float(out.loss) if k == "loss" else getattr(model, k)
            assert abs(got - ref) <= 1e-3 * abs(ref) + 2e-3, (mode, k, got, ref)
        if mode == "eval":
            err = (out.hidden_states[:, -1, :32].float().cpu() - lp["hidden_last"]).abs().max().item()
            assert err < 5e-2, err
        else:
            out.loss.backward()
            g = model.model.layers[0].self_attn.qkv_proj.weight.grad
            assert g is not None and torch.isfinite(g).all() and float(g.abs().sum()) > 0


def test_missing_library_or_cpu_tensor_fails_loudly(model):
    from metamorph_b200._lib import MetaMorphB200Error
    from metamorph_b200 import ops
    with pytest.raises(MetaMorphB200Error):
        ops.rmsnorm(torch.zeros(4, 256, dtype=torch.bfloat16), torch.ones(256, dtype=torch.bfloat16), 1e-5)
