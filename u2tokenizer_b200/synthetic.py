"""Seeded synthetic weights and inputs with the reference's parameter names and shapes.

There is no network for checkpoints or datasets, so parity tests and the benchmark run on
random-init weights of the real architecture and synthetic volumes/prompts (SURVEY.md section 8d).
Pure data generation: no hot-path arithmetic here.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch

from .geometry import Geometry


def param_shapes(g: Geometry) -> Dict[str, Tuple[int, ...]]:
    """name -> shape for every parameter of the reference u2*ForCausalLM (state-dict contract,
    SURVEY.md section 8b; reference svr.py:11-12,48,67,97,124, tta.py:74-86,112,121-124,
    spatial_pooling_projector.py:24-28, MONAI ViT naming, HF decoder naming)."""
    s: Dict[str, Tuple[int, ...]] = {}
    E, H = g.hidden_size, g.vit_hidden
    v = "model.vision_tower.vision_tower."
    s[v + "patch_embedding.patch_embeddings.1.weight"] = (H, g.patch_dim)
    s[v + "patch_embedding.patch_embeddings.1.bias"] = (H,)
    s[v + "patch_embedding.position_embeddings"] = (1, g.n_patches, H)
    s[v + "cls_token"] = (1, 1, H)
    for i in range(g.vit_layers):
        b = f"{v}blocks.{i}."
        s[b + "norm1.weight"] = (H,); s[b + "norm1.bias"] = (H,)
        s[b + "attn.qkv.weight"] = (3 * H, H)
        s[b + "attn.out_proj.weight"] = (H, H); s[b + "attn.out_proj.bias"] = (H,)
        s[b + "norm2.weight"] = (H,); s[b + "norm2.bias"] = (H,)
        s[b + "mlp.linear1.weight"] = (g.vit_mlp, H); s[b + "mlp.linear1.bias"] = (g.vit_mlp,)
        s[b + "mlp.linear2.weight"] = (H, g.vit_mlp); s[b + "mlp.linear2.bias"] = (H,)
    s[v + "norm.weight"] = (H,); s[v + "norm.bias"] = (H,)

    p = "model.mm_projector.projector."
    s[p + "0.weight"] = (E, H); s[p + "0.bias"] = (E,)
    for i in range(1, int(g.proj_layer_num)):
        idx = 2 * i if g.proj_layer_type == "mlp" else i
        s[p + f"{idx}.weight"] = (E, E); s[p + f"{idx}.bias"] = (E,)

    if g.enable_u2tokenizer:
        u = "model.u2tokenizer."
        s[u + "query_tokens"] = (1, g.num_3d_query_token, E)

        def mha(pre, rel):
            if rel and g.attn_type not in ("rma", "rope"):
                # torch.nn.MultiheadAttention fallback (reference svr.py:17-18, tta.py:83-84)
                s[pre + "in_proj_weight"] = (3 * E, E); s[pre + "in_proj_bias"] = (3 * E,)
                s[pre + "out_proj.weight"] = (E, E); s[pre + "out_proj.bias"] = (E,)
                return
            for n in ("wq", "wk", "wv", "dense"):
                s[f"{pre}{n}.weight"] = (E, E); s[f"{pre}{n}.bias"] = (E,)
            if rel and g.attn_type == "rma":
                s[pre + "relative_bias"] = (2 * 512 - 1, g.u2t_num_heads)

        for i in range(g.u2t_num_layers):
            l = f"{u}svt_module.attention_network.layers.{i}."
            mha(l + "spatial_attention.", True)
            mha(l + "temporal_attention.", True)
        k_out = g.u2t_top_k if g.enable_diffts else 1
        s[u + "svt_module.token_selection.score_net.weight"] = (k_out, E)
        s[u + "svt_module.token_selection.score_net.bias"] = (k_out,)
        if g.enable_dmtp:
            s[u + "svt_module.dynamic_pool.gate_fc.weight"] = (1, E)
            s[u + "svt_module.dynamic_pool.gate_fc.bias"] = (1,)
        for i in range(g.u2t_num_layers):
            l = f"{u}tta_module.layers_vt.{i}."
            mha(l + "visual_cross_attention.", False)
            mha(l + "text_cross_attention.", False)
            mha(l + "self_attention.", True)
            for n in ("norm_cross_v", "norm_cross_t", "norm_self"):
                s[f"{l}{n}.weight"] = (E,); s[f"{l}{n}.bias"] = (E,)
        mha(u + "tta_module.layer_linagg.linear_aggregator.", False)

    s["model.embed_tokens.weight"] = (g.vocab_size, E)
    hq, hkv, dh, I = g.num_attention_heads, g.num_key_value_heads, g.head_dim, g.intermediate_size
    for i in range(g.num_hidden_layers):
        l = f"model.layers.{i}."
        s[l + "input_layernorm.weight"] = (E,)
        if g.decoder_family == "phi3":  # fused projections (HF modeling_phi3.py:54, Phi3Attention.qkv_proj)
            s[l + "self_attn.qkv_proj.weight"] = ((hq + 2 * hkv) * dh, E)
        else:
            s[l + "self_attn.q_proj.weight"] = (hq * dh, E)
            s[l + "self_attn.k_proj.weight"] = (hkv * dh, E)
            s[l + "self_attn.v_proj.weight"] = (hkv * dh, E)
        s[l + "self_attn.o_proj.weight"] = (E, hq * dh)
        if g.qk_norm:
            s[l + "self_attn.q_norm.weight"] = (dh,)
            s[l + "self_attn.k_norm.weight"] = (dh,)
        s[l + "post_attention_layernorm.weight"] = (E,)
        if g.decoder_family == "phi3":
            s[l + "mlp.gate_up_proj.weight"] = (2 * I, E)  # [gate; up] in halves
        else:
            s[l + "mlp.gate_proj.weight"] = (I, E)
            s[l + "mlp.up_proj.weight"] = (I, E)
        s[l + "mlp.down_proj.weight"] = (E, I)
    s["model.norm.weight"] = (E,)
    if not g.tie_word_embeddings:
        s["lm_head.weight"] = (g.vocab_size, E)
    return s


def _std_for(name: str, shape) -> Tuple[float, float]:
    """(mean, std) of the synthetic init: 'trained-like' (non-degenerate biases / norms)."""
    if name.endswith("norm.weight") or name.endswith("layernorm.weight") or ".norm1.weight" in name \
            or ".norm2.weight" in name or "norm_self.weight" in name or "norm_cross_v.weight" in name \
            or "norm_cross_t.weight" in name:
        return 1.0, 0.05
    if name.endswith("relative_bias"):
        return 0.0, 0.2
    if name.endswith(".bias"):
        return 0.0, 0.02
    if name.endswith("query_tokens") or name.endswith("position_embeddings") or name.endswith("cls_token"):
        return 0.0, 0.02
    if name.endswith("embed_tokens.weight") or name.endswith("lm_head.weight"):
        return 0.0, 0.02
    if len(shape) == 2:
        fan_in = shape[1]
        return 0.0, float(fan_in) ** -0.5
    return 0.0, 0.02


@torch.no_grad()
def synthetic_state_dict(g: Geometry, seed: int = 0, device="cpu", dtype=torch.bfloat16,
                         head_tail: float = 0.0, bigram: float = 0.0) -> Dict[str, torch.Tensor]:
    """Every parameter drawn from its own seeded generator (name-hashed), so a CPU oracle copy and a
    GPU product copy built from the same (geometry, seed) hold bit-identical bf16 values when both
    are generated on the CPU; for the big benchmark models generation happens on the device.

    head_tail > 0 gives the output head a "trained-like" peaky structure: row v of lm_head (of embed_tokens when the
    head is tied) is scaled by exp(head_tail * n_v), n_v ~ N(0, 1). An i.i.d. Gaussian head makes the top-1 / top-2
    logit gap ~ 1 / (2 ln V) of the top logit, i.e. comparable to the bf16 error, so greedy token ids could not be
    compared at all; with log-normal row norms the leading candidates are separated by a finite fraction of the top
    logit and greedy parity becomes a real check (VERDICT r1, weak #2).

    bigram > 0 (untied heads only) gives the decoder "trained-like" bigram statistics instead: embed_tokens rows are
    N(0, s^2) with s = bigram * 0.7 * sqrt(2 * layers) (so the token's own embedding is `bigram` times the random-walk
    norm of the 2 * layers residual-branch outputs) and lm_head row pi(v) is the direction of embed_tokens row v for a
    seeded permutation pi: the preferred next token of v is pi(v) with a margin that is a finite fraction of the top
    logit, the layers' contribution perturbs (and sometimes overrides) it. Greedy ids then walk through the vocabulary
    instead of repeating one id, and nearly every step has a decisive top-1 / top-2 margin."""
    out = {}
    dev = torch.device(device)
    for i, (name, shape) in enumerate(param_shapes(g).items()):
        gen = torch.Generator(device=dev).manual_seed(seed * 1000003 + i)
        mean, std = _std_for(name, shape)
        n = 1
        for d in shape:
            n *= d
        if n > (1 << 26):  # big matrices: generate directly in the target dtype to bound memory
            t = torch.empty(shape, device=dev, dtype=dtype).normal_(mean, std, generator=gen)
        else:
            t = (torch.randn(shape, device=dev, generator=gen) * std + mean).to(dtype)
        out[name] = t
    if head_tail > 0:
        name = "lm_head.weight" if "lm_head.weight" in out else "model.embed_tokens.weight"
        gen = torch.Generator(device=dev).manual_seed(seed * 1000003 + 999331)
        scale = torch.exp(head_tail * torch.randn(out[name].shape[0], 1, device=dev, generator=gen))
        out[name] = (out[name].float() * scale).to(dtype)
    if bigram > 0:
        if "lm_head.weight" not in out:
            raise ValueError("bigram structure needs an untied output head")
        V, E = out["lm_head.weight"].shape
        gen = torch.Generator(device=dev).manual_seed(seed * 1000003 + 999332)
        perm = torch.randperm(V, device=dev, generator=gen)
        s_e = bigram * 0.7 * (2 * g.num_hidden_layers) ** 0.5
        emb = torch.empty(V, E, device=dev, dtype=dtype).normal_(0.0, 1.0, generator=gen)
        head = torch.empty_like(emb)
        head[perm] = (emb.float() * 0.05).to(dtype) if V * E <= (1 << 26) else emb.mul(0.05)
        out["lm_head.weight"] = head
        out["model.embed_tokens.weight"] = emb.mul_(s_e)
    return out


@torch.no_grad()
def synthetic_inputs(g: Geometry, batch: int, frames: int, n_question: int = 32, lt: int = 512,
                     seed: int = 1234, pad_id: int = 0, im_patch_id: int = None, device="cpu"):
    """Volumes U[0,1) fp32 [B, C, D, H, W]; input_ids = n_vis x <im_patch> + n_question random ids;
    question_ids = the same ids right-padded to `lt` (SURVEY.md section 8d)."""
    gen = torch.Generator(device="cpu").manual_seed(seed)
    D, H, W = g.image_size
    images = torch.rand(batch, frames, D, H, W, generator=gen)
    n_vis = g.num_3d_query_token if g.enable_u2tokenizer else g.tokens_per_frame
    hi = max(16, g.vocab_size - 16)
    q = torch.randint(1, hi, (batch, n_question), generator=gen)
    if im_patch_id is None:
        im_patch_id = g.vocab_size - 2
    input_ids = torch.cat([torch.full((batch, n_vis), im_patch_id, dtype=torch.long), q], dim=1)
    question_ids = torch.full((batch, lt), pad_id, dtype=torch.long)
    question_ids[:, :n_question] = q
    return images.to(device), input_ids.to(device), question_ids.to(device)
