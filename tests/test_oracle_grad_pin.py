"""Groundwork for the training rows of the scope table (SURVEY.md section 8d cfg 4 / cfg 5, not implemented on the GPU yet):
the functional oracle is differentiable, so its autograd gradients can serve as the backward oracle. Here they are pinned
against the gradients of the REFERENCE modules (imported unmodified, or their recorded gradients where the reference tree
is not mounted: a fixed sample of each parameter's gradient, see tests/refshim.py) and of the HF decoder on identical
weights / inputs."""
import pytest
import torch

from common import fp32_sd, rel_err, tiny_geometry
from oracle import u2_oracle as O
import refshim


def _sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def grad_close(got, want, floor, tol=2e-4):
    """max |got - want| <= tol * max(max |want|, floor): gradients that are numerically zero (far below `floor`, the
    scale of the largest gradient in the model) are compared on that scale, not on their own rounding noise."""
    return float((got - want).abs().max()) <= tol * max(float(want.abs().max()), floor)


def _sample(t, n=256):
    """A fixed sample of a gradient's elements (all of them for a small tensor)."""
    f = t.flatten()
    if f.numel() <= n:
        return f.clone()
    return f[torch.randperm(f.numel(), generator=torch.Generator().manual_seed(f.numel()))[:n]].clone()


@pytest.mark.parametrize("attn_type", ["rma", "rope"])
def test_u2tokenizer_gradients_match_reference(attn_type):
    g = tiny_geometry(attn_type=attn_type)
    sd = fp32_sd(g, seed=5)
    pre = "model.u2tokenizer."
    gen = torch.Generator().manual_seed(0)
    v = torch.randn(2, 3, g.tokens_per_frame, g.hidden_size, generator=gen)
    t = torch.randn(2, 5, g.hidden_size, generator=gen)
    w = torch.randn(2, g.num_3d_query_token, g.hidden_size, generator=gen)   # a fixed cotangent

    def reference():
        refshim.install()
        from src.model.u2tokenizer.u2Tokenizer import u2Tokenizer
        ref = u2Tokenizer(embed_size=g.hidden_size, num_heads=g.u2t_num_heads, num_layers=g.u2t_num_layers, top_k=g.u2t_top_k,
                          use_multi_scale=True, num_3d_query_token=g.num_3d_query_token, hidden_size=g.hidden_size,
                          attn_type=attn_type, enable_diffts=True, enable_dmtp=True)
        ref.load_state_dict(_sub(sd, pre), strict=True)
        v_ref, t_ref = v.clone().requires_grad_(), t.clone().requires_grad_()
        (ref(v_token=v_ref, t_token=t_ref) * w).sum().backward()
        # parameters the reference never uses (linagg wv / dense, tta.py:47-48,62-65) have no gradient: None
        return {"v": v_ref.grad, "t": t_ref.grad, "params": {n: p.grad for n, p in ref.named_parameters()}}
    want, full = refshim.pinned(f"u2tokenizer_grads_{attn_type}", reference,
                                keep=lambda r: {"v": r["v"], "t": r["t"],
                                                "params": {n: None if x is None else _sample(x) for n, x in r["params"].items()}})
    sdg = {k: (x.clone().requires_grad_() if k.startswith(pre) else x) for k, x in sd.items()}
    v_o, t_o = v.clone().requires_grad_(), t.clone().requires_grad_()
    (O.u2tokenizer(sdg, pre, v_o, t_o, g) * w).sum().backward()
    floor = 1e-2 * float(want["v"].abs().max())
    assert grad_close(v_o.grad, want["v"], floor) and grad_close(t_o.grad, want["t"], floor)
    checked = 0
    for name, pg in want["params"].items():
        go = sdg[pre + name].grad
        if pg is None:
            assert go is None or float(go.abs().max()) == 0, name
            continue
        assert go is not None, name
        go = go if full else _sample(go)
        assert grad_close(go, pg, floor), (name, rel_err(go, pg))
        checked += 1
    assert checked > 40


@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_decoder_gradients_match_hf(family):
    from transformers import LlamaConfig, LlamaForCausalLM, Qwen3Config, Qwen3ForCausalLM
    g = tiny_geometry() if family == "qwen3" else tiny_geometry(qk_norm=False, rope_theta=500000.0, tie_word_embeddings=True)
    sd = fp32_sd(g, seed=6)
    kw = dict(hidden_size=g.hidden_size, intermediate_size=g.intermediate_size, num_hidden_layers=g.num_hidden_layers,
              num_attention_heads=g.num_attention_heads, num_key_value_heads=g.num_key_value_heads, head_dim=g.head_dim,
              vocab_size=g.vocab_size, rms_norm_eps=g.rms_norm_eps, max_position_embeddings=4096,
              tie_word_embeddings=g.tie_word_embeddings, attention_bias=False, rope_theta=g.rope_theta)
    cfg = (Qwen3Config if family == "qwen3" else LlamaConfig)(**kw)
    cfg._attn_implementation = "eager"
    hf = (Qwen3ForCausalLM if family == "qwen3" else LlamaForCausalLM)(cfg).float()
    dec = {k: v for k, v in sd.items() if k.startswith("model.layers.") or k in ("model.embed_tokens.weight", "model.norm.weight",
                                                                                  "lm_head.weight")}
    missing, unexpected = hf.load_state_dict(dec, strict=False)
    assert not unexpected
    gen = torch.Generator().manual_seed(1)
    emb = torch.randn(2, 7, g.hidden_size, generator=gen) * 0.1
    labels = torch.randint(0, g.vocab_size, (2, 7), generator=gen)
    e_hf = emb.clone().requires_grad_()
    hf(inputs_embeds=e_hf, labels=labels).loss.backward()
    sdg = {k: (x.clone().requires_grad_() if k in dec else x) for k, x in sd.items()}
    e_o = emb.clone().requires_grad_()
    O.causal_lm_loss(O.decoder_forward(sdg, e_o, g)[0], labels).backward()
    floor = 1e-2 * float(e_hf.grad.abs().max())
    assert grad_close(e_o.grad, e_hf.grad, floor)
    n = 0
    for name, p in hf.named_parameters():
        if name not in sdg or p.grad is None or sdg[name].grad is None:
            continue
        assert grad_close(sdg[name].grad, p.grad, floor), name
        n += 1
    assert n >= 10
