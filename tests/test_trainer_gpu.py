"""TrainEngine on H100: the fused (optimizer-in-backward) step, the clipped two-phase step and a plain
`loss.backward()` + torch.optim.AdamW loop must agree on the updated parameters."""
import copy

import pytest
import torch

from oracle.weights import TINY, make_batch, make_weights
from tests.helpers import build_product_model

pytestmark = pytest.mark.gpu


def _batch():
    ids, mask, labs, images = make_batch(TINY)
    return dict(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())


def _params(model):
    return {n: p.detach().float().clone() for n, p in model.named_parameters() if p.requires_grad}


def test_fused_step_matches_autograd_style_loop(cuda_device):
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    lr = 1e-3
    # (a) fused engine
    m_a = build_product_model(TINY, W)
    eng = TrainEngine(m_a, lr=lr, weight_decay=0.0, max_grad_norm=None, constant_lr=True)
    out_a = eng.step(_batch())
    torch.cuda.synchronize()
    # (b) reference-style loop on the same model class: forward -> loss.backward() -> torch AdamW on fp32 copies
    m_b = build_product_model(TINY, W)
    m_b.train()
    out_b = m_b(**_batch())
    out_b.loss.backward()
    named = {n: p for n, p in m_b.named_parameters() if p.requires_grad and p.grad is not None}
    masters = {n: p.detach().float().clone().requires_grad_(True) for n, p in named.items()}
    opt = torch.optim.AdamW(list(masters.values()), lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    for n, p in named.items():
        masters[n].grad = p.grad.float()
    opt.step()
    assert abs(float(out_a["loss"]) - float(out_b.loss)) < 1e-3
    pa = dict(m_a.named_parameters())
    checked = 0
    for n, mref in masters.items():
        if "vision_proj" in n:
            continue
        got = pa[n].detach().float()
        exp = mref.detach().bfloat16().float()
        # AdamW's first step moves every touched weight by ~lr; bf16 grads of the two paths can differ in sign
        # only where the gradient is ~0, so compare with an absolute tolerance of 2*lr
        diff = (got - exp).abs()
        frac_bad = float((diff > 2.2 * lr + 8e-3 * exp.abs()).float().mean())
        assert frac_bad < 2e-3, (n, frac_bad, float(diff.max()))
        checked += 1
    assert checked >= 20


def test_clipped_mode_equals_fused_mode_when_not_clipping(cuda_device):
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    m_a = build_product_model(TINY, W)
    m_b = build_product_model(TINY, W)
    e_a = TrainEngine(m_a, lr=5e-4, max_grad_norm=None, constant_lr=True)
    e_b = TrainEngine(m_b, lr=5e-4, max_grad_norm=1e9, constant_lr=True)
    for _ in range(2):
        la = e_a.step(_batch())
        lb = e_b.step(_batch())
    torch.cuda.synchronize()
    assert abs(float(la["loss"]) - float(lb["loss"])) < 5e-3
    assert float(e_b.last_grad_norm) > 0
    pa, pb = _params(m_a), _params(m_b)
    for n in pa:
        if "vision_proj" in n:
            continue
        d = (pa[n] - pb[n]).abs()
        assert float((d > 1.2e-3 + 8e-3 * pb[n].abs()).float().mean()) < 2e-3, n


def _run_engine(mode, W):
    """Three steps of one engine mode on fixed batches; returns everything a step writes."""
    from metamorph_b200.engine.trainer import TrainEngine
    m = build_product_model(TINY, W)
    kw = dict(lr=1e-3, weight_decay=0.1, constant_lr=True)
    if mode == "clipped":
        kw["max_grad_norm"] = 1e-2
    elif mode == "packed":
        kw["pack_sequences"] = True
    elif mode == "accum2":
        kw["gradient_accumulation_steps"] = 2
    eng = TrainEngine(m, **kw)
    if mode == "accum2":
        batches = [[_batch(), _batch2(7)], [_batch2(7), _batch()], [_batch(), _batch2(7)]]
    else:
        batches = [_batch(), _batch2(7), _batch()]
    losses, norms = [], []
    for b in batches:
        out = eng.step(b)
        losses.append(torch.stack([out["loss"].reshape(()), out["loss_language"].reshape(()),
                                   out["loss_image_ar"].reshape(())]).clone())
        if mode == "clipped":
            norms.append(eng.last_grad_norm.clone())
    torch.cuda.synchronize()
    params = {n: p.detach().clone() for n, p in m.named_parameters()}
    state = {n: (st.p32.clone(), st.m.clone(), st.v.clone(), st.p16.clone()) for n, st in eng.opt.items()}
    return eng, losses, norms, params, state


@pytest.mark.parametrize("mode", ["fused", "clipped", "packed", "accum2"])
def test_train_step_is_bit_reproducible(cuda_device, mode, monkeypatch):
    """Two engines built from the same weights and fed the same batches compute the same bits: losses, every parameter,
    every optimizer state and the gradient norm. The fused mode runs under torch.use_deterministic_algorithms, so a torch
    op of the step without a deterministic implementation raises, and torch.empty is filled with NaN: a kernel that
    reads memory nobody wrote shows up as a NaN."""
    W = make_weights(TINY)
    was = torch.are_deterministic_algorithms_enabled()
    if mode == "fused":
        monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        torch.use_deterministic_algorithms(True)
    try:
        runs = [_run_engine(mode, W) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(was)
    (e_a, la, na, pa, sa), (_, lb, nb, pb, sb) = runs
    for i, (x, y) in enumerate(zip(la, lb)):
        assert torch.isfinite(x).all(), (mode, i, x)
        assert torch.equal(x, y), (mode, "losses of step", i + 1, x, y)
    for n in pa:
        assert torch.isfinite(pa[n].float()).all(), (mode, n)
        assert torch.equal(pa[n], pb[n]), (mode, "parameter", n)
    for n in sa:
        for what, x, y in zip(("p32", "m", "v", "p16"), sa[n], sb[n]):
            assert torch.equal(x, y), (mode, what, n)
    if mode == "clipped":
        assert float(na[0]) > e_a.max_grad_norm, "max_grad_norm must be small enough for clipping to take effect"
        for x, y in zip(na, nb):
            assert torch.equal(x, y), (mode, "last_grad_norm", na, nb)


def test_clipped_step_matches_torch_clip_grad_norm(cuda_device):
    """Clipping that takes effect: the engine's step against loss.backward() + clip_grad_norm_ + torch AdamW."""
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    # reference: autograd-style loop, gradient norm first, so that max_norm can be set to a quarter of it
    m_b = build_product_model(TINY, W)
    m_b.train()
    m_b(**_batch()).loss.backward()
    named = {n: p for n, p in m_b.named_parameters() if p.requires_grad and p.grad is not None and "vision_proj" not in n}
    grads = {n: p.grad.float() for n, p in named.items()}
    t_norm = float(torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(g) for g in grads.values()])))
    max_norm = 0.25 * t_norm

    def reference(lr, eps):
        masters = {n: p.detach().float().clone().requires_grad_(True) for n, p in named.items()}
        for n in masters:
            masters[n].grad = grads[n].clone()
        norm = float(torch.nn.utils.clip_grad_norm_(list(masters.values()), max_norm))
        opt = torch.optim.AdamW(list(masters.values()), lr=lr, betas=(0.9, 0.999), eps=eps, weight_decay=0.0)
        opt.step()
        return norm, {n: t.detach() for n, t in masters.items()}

    def engine(lr, eps):
        m_a = build_product_model(TINY, W)
        eng = TrainEngine(m_a, lr=lr, eps=eps, weight_decay=0.0, max_grad_norm=max_norm, constant_lr=True)
        eng.step(_batch())
        torch.cuda.synchronize()
        return float(eng.last_grad_norm), m_a, eng

    # (a) the usual hyper-parameters, compared as test_fused_step_matches_autograd_style_loop compares them
    lr = 1e-3
    norm_e, m_a, _ = engine(lr, 1e-8)
    norm_t, masters = reference(lr, 1e-8)
    assert norm_e > max_norm, "clipping must take effect"
    assert abs(norm_e - norm_t) <= 1e-2 * norm_t, (norm_e, norm_t)    # the two paths' bf16 gradients differ slightly
    pa = dict(m_a.named_parameters())
    for n, mref in masters.items():
        got, exp = pa[n].detach().float(), mref.bfloat16().float()
        frac_bad = float(((got - exp).abs() > 2.2 * lr + 8e-3 * exp.abs()).float().mean())
        assert frac_bad < 2e-3, (n, frac_bad)
    # (b) AdamW's first step is lr * g / (|g| + eps): with the usual eps it does not depend on the gradient's scale, so (a)
    # cannot see the clip coefficient. With eps = 1 the update is ~ lr * coef * g: compare the fp32 master updates, per
    # tensor in norm. A coefficient error of the unclipped kind would be a factor 4 off here.
    lr, eps = 1.0, 1.0
    _, _, eng = engine(lr, eps)
    _, masters = reference(lr, eps)
    checked = 0
    for n, mref in masters.items():
        st = eng.opt.get(n)
        if st is None:
            continue
        p0 = named[n].detach().float().reshape(-1)
        d_e, d_t = st.p32.reshape(-1) - p0, mref.reshape(-1) - p0
        rel = float((d_e - d_t).norm() / (d_t.norm() + 1e-30))
        assert rel < 0.1, (n, rel)
        checked += 1
    assert checked >= 20


def test_loss_decreases_over_steps(cuda_device):
    from metamorph_b200.engine.trainer import TrainEngine
    m = build_product_model(TINY, make_weights(TINY))
    eng = TrainEngine(m, lr=2e-3, constant_lr=True)
    losses = [float(eng.step(_batch())["loss"]) for _ in range(6)]
    assert losses[-1] < losses[0] - 0.5, losses


def test_training_checkpoint_resume(cuda_device, tmp_path):
    """SURVEY §8f N3: `checkpoint-N` (HF-format weights + optimizer fp32 master/m/v + trainer_state.json) restores
    the engine exactly, and the resumed run is the uninterrupted one: the train step is deterministic, so its losses
    and parameters must match bit for bit (a difference means some state is not saved or not restored)."""
    from metamorph_b200 import checkpoint as ck
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    m_a = build_product_model(TINY, W)
    e_a = TrainEngine(m_a, lr=1e-3, total_steps=10, warmup_ratio=0.2)
    for _ in range(2):
        e_a.step(_batch())
    torch.cuda.synchronize()
    ckpt = ck.save_training_checkpoint(e_a, str(tmp_path), max_shard_size="40MB")
    assert ckpt.endswith("checkpoint-2") and ck.latest_checkpoint(str(tmp_path)) == ckpt
    saved = {n: (st.p32.clone(), st.m.clone(), st.v.clone(), st.p16.clone()) for n, st in e_a.opt.items()}
    losses_a = [float(e_a.step(_batch())["loss"]) for _ in range(2)]

    m_b = build_product_model(TINY, make_weights(TINY, seed=123))       # different weights: everything must come from disk
    e_b = TrainEngine(m_b, lr=1e-3, total_steps=10, warmup_ratio=0.2)
    assert ck.load_training_checkpoint(e_b, ckpt) == 2 and e_b.step_count == 2
    for n, st in e_b.opt.items():
        p32, m, v, p16 = saved[n]
        assert torch.equal(st.p32, p32) and torch.equal(st.m, m) and torch.equal(st.v, v) and torch.equal(st.p16, p16), n
    from metamorph_b200.engine.trainer import cosine_lr
    assert e_b.current_lr == cosine_lr(1, 10, 1e-3, 0.2)                # lr of (restored) step 2 = lambda(1), as HF
    losses_b = [float(e_b.step(_batch())["loss"]) for _ in range(2)]
    assert losses_a == losses_b, (losses_a, losses_b)
    pa, pb = _params(m_a), _params(m_b)
    for n in pa:
        assert torch.equal(pa[n], pb[n]), n


def test_packed_step_equals_padded_step(cuda_device):
    """SURVEY §8f N2: packing the batch's samples end to end (block-diagonal attention, per-segment kernels) must give
    the padded batch's losses and parameter update."""
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    m_a, m_b = build_product_model(TINY, W), build_product_model(TINY, W)
    e_a = TrainEngine(m_a, lr=1e-3, constant_lr=True)
    e_b = TrainEngine(m_b, lr=1e-3, constant_lr=True, pack_sequences=True)
    out_a, out_b = e_a.step(_batch()), e_b.step(_batch())
    torch.cuda.synchronize()
    assert e_b.last_padding_saved > 0 and out_b["tokens"] < out_a["tokens"]
    # ... and, directly, the REFERENCE's losses on this batch (tests/golden/forward_backward_tiny.pt, made by the reference's
    # own forward): the packed layout is held to the reference, not only to the product's padded layout
    import os
    fb = torch.load(os.path.join(os.path.dirname(__file__), "golden", "forward_backward_tiny.pt"), weights_only=False)
    for k in ("loss", "loss_language", "loss_image_ar"):
        ref, got = float(fb[k]), float(out_b[k])
        assert abs(got - ref) <= 1e-3 * abs(ref) + 2e-3, ("packed vs reference", k, got, ref)
    for k in ("loss", "loss_language", "loss_image_ar"):
        a, b = float(out_a[k]), float(out_b[k])
        assert abs(a - b) <= 1e-3 * abs(a) + 1e-4, (k, a, b)
    pa, pb = _params(m_a), _params(m_b)
    for n in pa:
        err = (pa[n] - pb[n]).abs().max().item()
        assert err <= 2e-2 * (pa[n].abs().max().item() + 1e-3), n


def _batch2(seed):
    """A second, different batch of the same structure (other token ids / images)."""
    ids, mask, labs, images = make_batch(TINY, seed=seed)
    return dict(input_ids=ids, attention_mask=mask, labels=labs, images=images.bfloat16())


def test_gradient_accumulation(cuda_device):
    """gradient_accumulation_steps=k (TrainingArguments; scripts/*.sh pass it): k micro-batches, ONE optimizer step on the
    mean of their gradients. (a) twice the same micro-batch == one plain step on it; (b) two different micro-batches ==
    AdamW on the average of the two `loss.backward()` gradients."""
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    lr = 1e-3
    m_a, m_b = build_product_model(TINY, W), build_product_model(TINY, W)
    e_a = TrainEngine(m_a, lr=lr, constant_lr=True)
    e_b = TrainEngine(m_b, lr=lr, constant_lr=True, gradient_accumulation_steps=2)
    oa, ob = e_a.step(_batch()), e_b.step([_batch(), _batch()])
    torch.cuda.synchronize()
    assert abs(float(oa["loss"]) - float(ob["loss"])) < 1e-4
    pa, pb = _params(m_a), _params(m_b)
    for n in pa:
        if "vision_proj" in n:
            continue
        d = (pa[n] - pb[n]).abs()
        assert float((d > 1.2e-3 + 8e-3 * pb[n].abs()).float().mean()) < 2e-3, n
    with pytest.raises(ValueError):
        e_b.step(_batch())                                    # needs exactly k micro-batches
    # (b) different micro-batches against averaged autograd-style gradients
    m_c, m_d = build_product_model(TINY, W), build_product_model(TINY, W)
    e_c = TrainEngine(m_c, lr=lr, constant_lr=True, gradient_accumulation_steps=2)
    e_c.step([_batch(), _batch2(7)])
    torch.cuda.synchronize()
    m_d.train()
    for b in (_batch(), _batch2(7)):
        m_d(**b).loss.backward()                              # .grad accumulates the two micro-batch gradients
    named = {n: p for n, p in m_d.named_parameters() if p.requires_grad and p.grad is not None}
    masters = {n: p.detach().float().clone().requires_grad_(True) for n, p in named.items()}
    opt = torch.optim.AdamW(list(masters.values()), lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    for n, p in named.items():
        masters[n].grad = p.grad.float() / 2
    opt.step()
    pc = dict(m_c.named_parameters())
    for n, mref in masters.items():
        if "vision_proj" in n:
            continue
        got, exp = pc[n].detach().float(), mref.detach().bfloat16().float()
        frac_bad = float(((got - exp).abs() > 2.2 * lr + 8e-3 * exp.abs()).float().mean())
        assert frac_bad < 3e-3, (n, frac_bad)


def test_stage1_projector_only_training(cuda_device):
    """tune_mm_mlp_adapter (train.py:1516-1519): everything frozen but the projector. The frozen stack must get no
    wgrad work (no buckets, no optimizer state) and stay bit-identical, while the projector receives the very update it
    gets in full training (its gradient does not depend on which other parameters train)."""
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    m_full, m_s1 = build_product_model(TINY, W), build_product_model(TINY, W)
    for p in m_s1.parameters():
        p.requires_grad = False
    for p in m_s1.get_model().mm_projector.parameters():
        p.requires_grad = True
    before = {n: p.detach().clone() for n, p in m_s1.named_parameters()}
    e_full = TrainEngine(m_full, lr=1e-3, constant_lr=True)
    e_s1 = TrainEngine(m_s1, lr=1e-3, constant_lr=True)
    assert not e_s1.train_llm and not e_s1.layer_buckets and not e_s1.big_buckets
    assert sorted(e_s1.opt) == sorted(n for n in before if "mm_projector" in n)
    from metamorph_b200._lib import reset_launch_count
    reset_launch_count()
    o_full = e_full.step(_batch())
    torch.cuda.synchronize()
    n_full = reset_launch_count()
    o_s1 = e_s1.step(_batch())
    torch.cuda.synchronize()
    n_s1 = reset_launch_count()
    assert n_s1 < n_full                                      # the wgrad GEMMs / AdamW launches of the frozen stack are gone
    assert abs(float(o_full["loss"]) - float(o_s1["loss"])) < 1e-4
    after = dict(m_s1.named_parameters())
    full = dict(m_full.named_parameters())
    for n, p0 in before.items():
        if "mm_projector" in n:
            assert not torch.equal(after[n].detach(), p0), n
            d = (after[n].detach().float() - full[n].detach().float()).abs()
            assert float((d > 1.2e-3 + 8e-3 * full[n].detach().float().abs()).float().mean()) < 2e-3, n
        else:
            assert torch.equal(after[n].detach(), p0), f"frozen tensor {n} changed"


def test_step_without_answer_images_leaves_vision_head_untouched(cuda_device):
    """ADVICE r1: on a step whose batch has no answer-side image the reference gives vision_head no gradient (torch's
    AdamW skips it); a stale gradient buffer of the previous step must not be re-applied."""
    from metamorph_b200.engine.trainer import TrainEngine
    W = make_weights(TINY)
    m = build_product_model(TINY, W)
    eng = TrainEngine(m, lr=1e-3, constant_lr=True)
    eng.step(_batch())
    torch.cuda.synchronize()
    vh1 = {n: p.detach().clone() for n, p in m.named_parameters() if n.startswith("vision_head.")}
    ids, mask, labs, images = make_batch(TINY)
    text_only = dict(input_ids=ids[1:2], attention_mask=mask[1:2], labels=labs[1:2], images=images[2:3].bfloat16())
    out = eng.step(text_only)
    torch.cuda.synchronize()
    assert torch.isfinite(out["loss_language"]).all()
    for n, p in m.named_parameters():
        if n.startswith("vision_head."):
            assert torch.equal(p.detach(), vh1[n]), f"{n} was updated on a step that gave it no gradient"
