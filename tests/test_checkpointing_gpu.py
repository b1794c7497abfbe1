"""Activation checkpointing on the training tape (TrainEngine(checkpoint=True), HF gradient_checkpointing_enable()):
every ViT block, SVR layer, TTA layer and decoder layer keeps only its input and output and is recomputed in the backward.

  * against the fp32 oracle's autograd, with the tolerances of test_train_gpu.py, for every geometry there, a Phi-3
    sliding-window case and a LoRA case with dropout;
  * against the plain tape on the same inputs: the loss and every recomputed block output bit-identical, every gradient
    within max(2 x the spread of two plain runs, one bf16 ulp of the tensor's largest entry) - the backward's fp32
    atomics make the gradients order-dependent in their last bits, the forward is not - for one step, two accumulated
    micro-batches and a DPO step;
  * the interleaving of gradient writes and gradient-final markers (what ZeRO-1's overlapped reduce-scatter keys on)
    identical with and without checkpointing;
  * the HF surface, plain and through get_peft_model: enable / disable take effect without rebuilding the engine;
  * the activation peak at a geometry with 8 decoder layers and 4 ViT blocks: at most half of the plain tape's."""
import math

import pytest
import torch

import phi3_oracle as P3
from common import cosine, rel_err, tiny_geometry
from oracle import u2_oracle as O
from test_lora_gpu import TARGETS, _OracleLora, _lora_sd, _next_seed, _peft, _surface_model
from test_phi3 import tiny_phi3_geometry
from test_train_gpu import CASES, _labels, _oracle_loss_and_grads
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _weights(g, seed):
    sd16 = synthetic_state_dict(g, seed=seed, device="cpu", dtype=BF)
    # O(1) query tokens, so that the TTA attention is not uniform and its backward is exercised (as test_train_gpu.py)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    return sd16


def _grads(te):
    """{name: gradient} of every trainable parameter, cloned."""
    return {n: te.grad(n).clone() for n in te.lay.mat_names + te.lay.vec_names}


def _check_oracle(te, ref_g):
    """test_forward_backward_matches_oracle_autograd's criterion."""
    gmax = max(v.abs().max().item() for v in ref_g.values())
    bad = []
    for n, got in _grads(te).items():
        if n == "lm_head.weight" and te.tied:
            continue
        got, want = got.float().cpu(), ref_g[n].float().cpu()
        if want.abs().max().item() < 1e-9:
            assert got.abs().max().item() < 1e-4, f"{n}: oracle gradient is zero, got {got.abs().max().item()}"
            continue
        if rel_err(got, want) < 4e-2 and cosine(got, want) > 0.995:
            continue
        if (got - want).abs().max().item() < 2e-3 * gmax:
            continue
        bad.append((n, round(rel_err(got, want), 4), round(cosine(got, want), 5)))
    assert not bad, bad[:6]


def _capture_segments(te):
    """Wrap te._segment: every call of a block's body appends its output (a copy) to the block's list, so a
    checkpointed block holds [forward output, recomputed output] and a plain one [forward output]."""
    rec = []
    orig = te._segment

    def seg(body, x):
        outs = []
        rec.append(outs)

        def body2(x_):
            y = body(x_)
            outs.append(y.v.detach().clone())
            return y
        return orig(body2, x)
    te._segment = seg
    return rec


def _bits(t):
    """Raw bytes: a bitwise comparison that also holds for NaN / padding rows."""
    return t.detach().reshape(-1).contiguous().view(torch.uint8)


def _n_segments(g):
    return g.vit_layers + 2 * g.u2t_num_layers + g.num_hidden_layers


def _run(te, checkpoint, fn, seed=0):
    """fn(te) on a fresh gradient with te.checkpoint set; (result, gradients, segment captures)."""
    te.checkpoint = checkpoint
    rec = _capture_segments(te)
    try:
        te.zero_grad()
        torch.manual_seed(seed)   # the LoRA dropout seed of each training forward
        res = fn(te)
        torch.cuda.synchronize()
    finally:
        del te._segment
    return res, _grads(te), rec


def _ulp_bf16(m: float) -> float:
    return 2.0 ** (math.floor(math.log2(m)) - 7) if m > 0 else 0.0


def _check_against_plain(te, fn, n_seg, seed=0):
    r1, g1, rec1 = _run(te, False, fn, seed)
    r2, g2, _ = _run(te, False, fn, seed)
    rc, gc, recc = _run(te, True, fn, seed)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(r1, rc)), (r1, rc)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(r1, r2)), (r1, r2)
    assert len(rec1) == len(recc) == n_seg, (len(rec1), len(recc), n_seg)
    for i, (p, c) in enumerate(zip(rec1, recc)):
        assert len(p) == 1 and len(c) == 2, (i, len(p), len(c))
        assert torch.equal(_bits(c[0]), _bits(p[0])), f"segment {i}: checkpointed forward differs from the plain one"
        assert torch.equal(_bits(c[1]), _bits(c[0])), f"segment {i}: recomputed output differs from the forward's"
    bad = []
    n_nonzero = 0
    for n in g1:
        a, b, c = g1[n].float(), g2[n].float(), gc[n].float()
        spread = (a - b).abs().max().item()
        bound = max(2 * spread, _ulp_bf16(a.abs().max().item()))
        d = (c - a).abs().max().item()
        n_nonzero += a.abs().max().item() > 0
        if d > bound:
            bad.append((n, d, spread, a.abs().max().item()))
    assert not bad, bad[:6]
    assert n_nonzero > len(g1) // 2
    return r1


# ------------------------------------------------------------------------------------------------
# 1. against the oracle's autograd
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_checkpointed_forward_backward_matches_oracle_autograd(case):
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry(**CASES[case])
    sd16 = _weights(g, 21)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=3, n_question=7, lt=12)
    labels = _labels(ids, g.num_3d_query_token)
    ref_loss, ref_g = _oracle_loss_and_grads(sd16, g, images, ids, qids, labels)
    te = TrainEngine(g, sd16, device="cuda", checkpoint=True)
    assert te.checkpoint
    rec = _capture_segments(te)
    te.zero_grad()
    loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    torch.cuda.synchronize()
    assert [len(r) for r in rec] == [2] * _n_segments(g)   # every block ran twice: forward and recompute
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss)), (float(loss), ref_loss)
    _check_oracle(te, ref_g)


def test_checkpointed_phi3_sliding_window_matches_oracle_autograd():
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_phi3_geometry()
    sd16 = _weights(g, 31)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=30, lt=32)
    labels = _labels(ids, g.num_3d_query_token)
    assert ids.shape[1] > g.sliding_window
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    emb = O.multimodal_embeds(sd, ids.cuda(), images.cuda(), qids.cuda(), g)
    ref = O.causal_lm_loss(P3.decoder_forward(sd, emb, g)[0], labels.cuda())
    ref.backward()
    ref_g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}
    te = TrainEngine(g, sd16, device="cuda", checkpoint=True)
    te.zero_grad()
    loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) < 2e-2 * max(1.0, abs(float(ref))), (float(loss), float(ref))
    _check_oracle(te, ref_g)


def test_checkpointed_lora_dropout_matches_oracle_autograd(monkeypatch):
    from u2tokenizer_b200.train import LoraSpec, TrainEngine
    g = tiny_geometry()
    r, s, p = 8, 2.0, 0.05
    sd16 = _lora_sd(g, _weights(g, 21), r)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=3, n_question=7, lt=12)
    labels = _labels(ids, g.num_3d_query_token)
    te = TrainEngine(g, sd16, device="cuda", lora=LoraSpec(r, s, p, TARGETS), checkpoint=True)
    te.zero_grad()
    torch.manual_seed(123)
    loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    torch.cuda.synchronize()
    seed = _next_seed(123)
    assert te._lora_seed == seed
    _OracleLora(monkeypatch, None, s, p, seed)
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    ref = O.causal_lm_loss(O.forward_logits(sd, ids.cuda(), images.cuda(), qids.cuda(), g), labels.cuda())
    ref.backward()
    ref_g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}
    assert abs(float(loss) - float(ref)) < 2e-2 * max(1.0, abs(float(ref))), (float(loss), float(ref))
    _check_oracle(te, ref_g)


# ------------------------------------------------------------------------------------------------
# 2. against the plain tape on the same inputs
# ------------------------------------------------------------------------------------------------
def _engine(kind):
    from u2tokenizer_b200.train import LoraSpec, TrainEngine
    if kind == "phi3_window":
        g = tiny_phi3_geometry()
        return TrainEngine(g, _weights(g, 31), device="cuda"), g
    g = tiny_geometry()
    if kind == "lora_p005":
        return TrainEngine(g, _lora_sd(g, _weights(g, 22), 8), device="cuda", lora=LoraSpec(8, 2.0, 0.05, TARGETS)), g
    return TrainEngine(g, _weights(g, 22), device="cuda"), g


def _sft_batches(g, n):
    out = []
    for seed in range(1, n + 1):
        im, ids, q = synthetic_inputs(g, batch=2, frames=2, n_question=30, lt=32, seed=seed)
        out.append((im.cuda(), ids.cuda(), q.cuda(), _labels(ids, g.num_3d_query_token).cuda()))
    return out


@pytest.mark.parametrize("kind", ["qwen3", "lora_p005", "phi3_window"])
def test_single_step_bit_identical_forward_and_gradients_within_spread(kind):
    te, g = _engine(kind)
    (a,) = _sft_batches(g, 1)
    _check_against_plain(te, lambda te: (te.forward_backward(*a),), _n_segments(g))


@pytest.mark.parametrize("kind", ["qwen3", "lora_p005"])
def test_two_accumulated_micro_batches(kind):
    te, g = _engine(kind)
    a, b = _sft_batches(g, 2)
    _check_against_plain(te, lambda te: (te.forward_backward(*a), te.forward_backward(*b)), 2 * _n_segments(g))


@pytest.mark.parametrize("kind", ["qwen3", "lora_p005"])
def test_dpo_step(kind):
    te, g = _engine(kind)
    images, ids, qids = synthetic_inputs(g, batch=1, frames=2, n_question=6, lt=10)
    gen = torch.Generator().manual_seed(3)
    n_prompt = ids.shape[1]
    ans = torch.randint(1, g.vocab_size - 16, (2, 9), generator=gen)
    ids2 = torch.cat([ids.expand(2, -1), ans], 1).cuda()
    images2, qids2 = images.expand(2, *images.shape[1:]).contiguous().cuda(), qids.expand(2, -1).contiguous().cuda()
    mask = torch.zeros_like(ids2)
    mask[:, n_prompt:] = 1
    mask[1, -2:] = 0
    ref_logps = torch.tensor([-30.0, -28.5], device="cuda")
    _check_against_plain(te, lambda te: (te.dpo_forward_backward(images2, ids2, qids2, mask, ref_logps, 0.1),),
                         _n_segments(g))


# ------------------------------------------------------------------------------------------------
# 3. marker order
# ------------------------------------------------------------------------------------------------
def test_gradient_writes_and_markers_fire_in_the_plain_order():
    """The sequence of events 'a kernel starts writing matrix gradient X' and 'the marker of X fires' is the same with
    and without checkpointing: each block's marker still fires right after its last wgrad (ZeRO-1 starts a bucket's
    reduce-scatter there and clears stale slots there)."""
    te, g = _engine("qwen3")
    (a,) = _sft_batches(g, 1)

    def events(checkpoint):
        log = []
        begin, clear = te._gm_begin_write, te._gm_clear_stale
        te._gm_begin_write = lambda gw: (log.append(("write", te._gm_names(gw))), begin(gw))[1]
        te._gm_clear_stale = lambda names: (log.append(("final", tuple(sorted(names)))), clear(names))[1]
        try:
            te.checkpoint = checkpoint
            te.zero_grad()
            te.forward_backward(*a)
            torch.cuda.synchronize()
        finally:
            del te._gm_begin_write, te._gm_clear_stale
        return log
    plain, ck = events(False), events(True)
    finals = [e for e in plain if e[0] == "final"]
    assert len(finals) >= _n_segments(g)
    assert plain == ck


# ------------------------------------------------------------------------------------------------
# 4. the HF surface
# ------------------------------------------------------------------------------------------------
def _surface_grads(model, batch, seed=0):
    model.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    model(**batch).loss.backward()
    torch.cuda.synchronize()
    return {n: p.grad.float().clone() for n, p in model.named_parameters() if p.grad is not None}


def _surface_check(model, batch):
    p1, p2 = _surface_grads(model, batch), _surface_grads(model, batch)
    te = model.train_engine()
    assert not te.checkpoint
    model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    assert model.is_gradient_checkpointing
    rec = _capture_segments(te)
    try:
        ck = _surface_grads(model, batch)
    finally:
        del te._segment
    assert model.train_engine() is te and te.checkpoint     # no rebuild; the engine ran checkpointed
    assert rec and all(len(r) == 2 for r in rec)
    assert set(ck) == set(p1)
    bad = []
    for n in p1:
        bound = max(2 * (p1[n] - p2[n]).abs().max().item(), _ulp_bf16(p1[n].abs().max().item()))
        if (ck[n] - p1[n]).abs().max().item() > bound:
            bad.append(n)
    assert not bad, bad[:6]
    model.gradient_checkpointing_disable()
    assert not model.is_gradient_checkpointing
    rec = _capture_segments(te)
    try:
        _surface_grads(model, batch)
    finally:
        del te._segment
    assert model.train_engine() is te and not te.checkpoint
    assert rec and all(len(r) == 1 for r in rec)


def _surface_batch(g):
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10)
    return dict(images=images.cuda(), input_ids=ids.cuda(), labels=_labels(ids, g.num_3d_query_token).cuda(),
                question_ids=qids.cuda(), attention_mask=torch.ones_like(ids).cuda())


def test_gradient_checkpointing_enable_on_the_module():
    model, g = _surface_model("qwen3")
    model.get_model().vision_tower.requires_grad_(False)
    model.train()
    _surface_check(model, _surface_batch(g))


def test_gradient_checkpointing_enable_through_get_peft_model():
    model, g = _surface_model("qwen3")
    model.requires_grad_(False)
    peft = _peft(model, dropout=0.05)
    with torch.no_grad():   # non-zero B, so that A gets a gradient too
        gen = torch.Generator(device="cuda").manual_seed(4)
        for n, p in peft.named_parameters():
            if ".lora_B." in n:
                p.copy_(torch.randn(p.shape, device="cuda", generator=gen) * 0.05)
    peft.train()
    peft.enable_input_require_grads()   # what HF Trainer calls for PEFT with checkpointing
    _surface_check(peft, _surface_batch(g))


# ------------------------------------------------------------------------------------------------
# 5. memory
# ------------------------------------------------------------------------------------------------
def test_checkpointing_at_least_halves_the_activation_peak():
    """8 decoder layers (E 512, I 1536, 1024 tokens), 4 ViT blocks (ViT-width 256, 16 frames), vocabulary 512: the
    kept activations of the plain tape against one block's input per block plus one recomputed block."""
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_geometry(num_hidden_layers=8, hidden_size=512, intermediate_size=1536, num_attention_heads=8,
                      num_key_value_heads=4, head_dim=64, vit_layers=4, vit_hidden=256, vit_mlp=1024, vit_heads=4,
                      u2t_top_k=16, num_3d_query_token=16, vocab_size=512)
    te = TrainEngine(g, _weights(g, 5), device="cuda")
    images, ids, qids = synthetic_inputs(g, batch=2, frames=8, n_question=32, lt=64)
    ans = torch.randint(1, g.vocab_size - 16, (2, 512 - ids.shape[1]), generator=torch.Generator().manual_seed(1))
    ids = torch.cat([ids, ans], 1)
    args = (images.cuda(), ids.cuda(), qids.cuda(), _labels(ids, g.num_3d_query_token).cuda())

    def peak(checkpoint):
        te.checkpoint = checkpoint
        te.zero_grad()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        loss = te.forward_backward(*args)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, float(loss)
    peak(False)                     # warm-up: every lazily built workspace exists before the measured passes
    plain, lp = peak(False)
    ck, lc = peak(True)
    print(f"activation peak: plain {plain / 2 ** 20:.1f} MiB, checkpointed {ck / 2 ** 20:.1f} MiB ({ck / plain:.3f})")
    assert lp == lc
    assert torch.cuda.max_memory_allocated() < 40 * 2 ** 30
    assert ck <= 0.5 * plain, (plain, ck)


def test_score_net_gradient_is_overwritten_by_the_first_write_of_a_step():
    """The DiffTS score-net wgrad follows the matrix-slot rules of every other wgrad: after zero_grad() the step's first
    write overwrites whatever an earlier step left in the slot, so the score net's gradient does not accumulate across
    optimizer steps (the plain-versus-checkpointed comparisons above run several steps on one engine and rely on it)."""
    te, g = _engine("qwen3")
    assert g.enable_diffts
    (a,) = _sft_batches(g, 1)
    name = "model.u2tokenizer.svt_module.token_selection.score_net.weight"
    slot = te.gm(name)
    te.zero_grad()
    te.forward_backward(*a)
    slot.fill_(1.0)                 # an earlier step's gradient, far above this one's
    te.zero_grad()
    te.forward_backward(*a)
    torch.cuda.synchronize()
    assert slot.float().abs().max().item() < 0.5, slot.float().abs().max().item()
