"""Phi-3 on the CUDA training path: TrainEngine's loss and every parameter gradient, the HF-surface
`model(**batch).loss.backward()` and LoRA on the four fused targets, each against torch autograd through the fp32 Phi-3
restatement (tests/phi3_oracle.py) with the sliding window shorter than the sequence (W 24 < L 38).

Tolerances as in test_train_gpu.py: loss within 2e-2; a gradient passes with rel_err < 4e-2 and cosine > 0.995, or an
absolute error below 2e-3 of the largest gradient entry of the model (cancellation noise of bf16 arithmetic)."""
import pytest
import torch

import phi3_oracle as P3
from common import cosine, rel_err
from oracle import u2_oracle as O
from test_phi3 import tiny_phi3_config, tiny_phi3_geometry
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _labels(ids, n_vis):
    lab = ids.clone()
    lab[:, :n_vis + 1] = -100
    return lab


def _weights(g, seed):
    sd16 = synthetic_state_dict(g, seed=seed, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    return sd16


def _oracle_loss(sd, g, images, ids, qids, labels):
    emb = O.multimodal_embeds(sd, ids.cuda(), images.cuda(), qids.cuda(), g)
    return O.causal_lm_loss(P3.decoder_forward(sd, emb, g)[0], labels.cuda())


def _oracle_loss_and_grads(sd16, g, images, ids, qids, labels):
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    loss = _oracle_loss(sd, g, images, ids, qids, labels)
    loss.backward()
    return float(loss), {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}


def _compare(pairs, gmax, tol=4e-2, cos=0.995):
    bad = []
    for n, got, want in pairs:
        got, want = got.float().cpu(), want.float().cpu()
        if want.abs().max().item() < 1e-9:
            assert got.abs().max().item() < 1e-4, n
            continue
        if rel_err(got, want) < tol and cosine(got, want) > cos:
            continue
        if (got - want).abs().max().item() < 2e-3 * gmax:
            continue
        bad.append((n, round(rel_err(got, want), 4), round(cosine(got, want), 5)))
    assert not bad, bad[:6]


def _inputs(g):
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=30, lt=32)
    return images, ids, qids, _labels(ids, g.num_3d_query_token)


def test_train_engine_matches_oracle_autograd():
    from u2tokenizer_b200.train import TrainEngine
    g = tiny_phi3_geometry()
    sd16 = _weights(g, 31)
    images, ids, qids, labels = _inputs(g)
    assert ids.shape[1] > g.sliding_window
    ref_loss, ref_g = _oracle_loss_and_grads(sd16, g, images, ids, qids, labels)
    te = TrainEngine(g, sd16, device="cuda")
    te.zero_grad()
    loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    torch.cuda.synchronize()
    assert abs(float(loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss)), (float(loss), ref_loss)
    L = te.lay
    assert "model.layers.0.self_attn.qkv_proj.weight" in L.mat_off and "model.layers.0.mlp.gate_up_proj.weight" in L.mat_off
    pairs = []
    for n in L.mat_names + L.vec_names:
        pairs.append((n, te.grad(n), ref_g[n]))
    _compare(pairs, max(v.abs().max().item() for v in ref_g.values()))


def _model(cfg, sd16):
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF)
    try:
        with torch.device("cuda"):
            model = U2Phi3ForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)
    model.load_state_dict(sd16)
    return model


def test_module_loss_backward():
    """model(**batch).loss.backward() through the HF-style surface (reference train_stage1.py:244-250), full fine-tuning
    as the reference's Phi-3 stage-1 scripts run it, with the vision tower frozen."""
    from u2tokenizer_b200.geometry import Geometry
    cfg = tiny_phi3_config()
    g = Geometry.from_hf(cfg)
    sd16 = _weights(g, 32)
    model = _model(cfg, sd16)
    model.get_model().vision_tower.requires_grad_(False)
    model.train()
    images, ids, qids, labels = _inputs(g)
    ref_loss, ref_g = _oracle_loss_and_grads(sd16, g, images, ids, qids, labels)
    out = model(images=images.cuda(), input_ids=ids.cuda(), labels=labels.cuda(), question_ids=qids.cuda(),
                attention_mask=torch.ones_like(ids).cuda())
    out.loss.backward()
    assert abs(float(out.loss) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
    pairs = []
    for n, p in model.named_parameters():
        if n.startswith("model.vision_tower."):
            assert p.grad is None
            continue
        if ref_g[n].abs().max().item() >= 1e-9:
            assert p.grad is not None, n
            pairs.append((n, p.grad, ref_g[n]))
    _compare(pairs, max(v.abs().max().item() for v in ref_g.values()), tol=5e-2, cos=0.99)


def test_lora_on_the_four_phi3_targets():
    """get_peft_model with the targets the reference's find_all_linear_names returns on Phi-3 (qkv_proj, o_proj,
    gate_up_proj, down_proj), p = 0: loss and the adapters' gradients against autograd through W + s B A."""
    from u2tokenizer_b200.geometry import Geometry
    from u2tokenizer_b200.lora import LoraConfig, get_peft_model
    cfg = tiny_phi3_config()
    g = Geometry.from_hf(cfg)
    sd16 = _weights(g, 33)
    model = _model(cfg, sd16)
    targets = ["qkv_proj", "o_proj", "gate_up_proj", "down_proj"]
    peft = get_peft_model(model, LoraConfig(r=8, lora_alpha=16, target_modules=targets, lora_dropout=0.0))
    gen = torch.Generator(device="cuda").manual_seed(4)
    with torch.no_grad():   # non-zero B, so that A gets a gradient too
        for n, p in peft.named_parameters():
            if ".lora_B." in n:
                p.copy_(torch.randn(p.shape, device="cuda", generator=gen) * 0.05)
    peft.train()
    images, ids, qids, labels = _inputs(g)
    # reference: autograd through the merged weights W + s B A of every target
    s = 16 / 8
    sd = {k: v.float().cuda() for k, v in sd16.items()}
    ad = {}
    for n, p in peft.named_parameters():
        if ".lora_" in n:
            ad[n] = p.detach().float().clone().requires_grad_(True)
    for li in range(g.num_hidden_layers):
        for pre, t in (("self_attn.", "qkv_proj"), ("self_attn.", "o_proj"), ("mlp.", "gate_up_proj"), ("mlp.", "down_proj")):
            m = f"base_model.model.model.layers.{li}.{pre}{t}."
            base = f"model.layers.{li}.{pre}{t}.weight"
            sd[base] = sd[base] + s * ad[m + "lora_B.default.weight"] @ ad[m + "lora_A.default.weight"]
    for k, v in sd.items():
        if not k.startswith("model.layers.") or k.endswith("layernorm.weight"):
            v.requires_grad_(True)
    ref = _oracle_loss(sd, g, images, ids, qids, labels)
    ref.backward()
    out = peft(images=images.cuda(), input_ids=ids.cuda(), labels=labels.cuda(), question_ids=qids.cuda())
    out.loss.backward()
    assert abs(float(out.loss) - float(ref)) < 2e-2 * max(1.0, abs(float(ref)))
    pairs = [(n, p.grad, ad[n].grad) for n, p in peft.named_parameters() if ".lora_" in n]
    assert len(pairs) == 2 * 4 * g.num_hidden_layers and all(p[1] is not None for p in pairs)
    assert all(not p.requires_grad for n, p in peft.named_parameters() if ".base_layer." in n)
    _compare(pairs, max(v.grad.abs().max().item() for v in ad.values()))
