"""Size-independent properties at the FULL widths of BASELINE.json's configurations (E = 4096, 8 frames, 1024-way
selection, 1792 visual tokens, Qwen3-8B head geometry), where the fp32 oracle would take minutes: invariants the
domain offers instead of an element-wise reference."""
import math

import pytest
import torch

from common import rel_err, tiny_geometry
from u2tokenizer_b200.synthetic import synthetic_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _engine(**over):
    from u2tokenizer_b200.engine import U2Engine
    g = tiny_geometry(image_size=[32, 256, 256], patch_size=[4, 16, 16], vit_hidden=768, vit_mlp=3072, vit_layers=1,
                      vit_heads=12, u2t_num_layers=1, u2t_top_k=1024, num_3d_query_token=256, hidden_size=4096,
                      intermediate_size=12288, num_hidden_layers=2, num_attention_heads=32, num_key_value_heads=8,
                      head_dim=128, vocab_size=8192, **over)
    sd = synthetic_state_dict(g, seed=21, device="cuda", dtype=torch.bfloat16)
    return U2Engine(g, sd, device="cuda"), g


def test_diffts_constant_tokens_and_row_stochastic():
    """softmax over tokens is row-stochastic: if every token equals v, every selected token equals v (E = 4096,
    8 x 256 tokens, 1024 selection heads)."""
    eng, g = _engine()
    v = torch.randn(g.hidden_size, device=DEV).bfloat16()
    x = v.expand(2 * 8 * 256, g.hidden_size).contiguous()
    sel = eng._token_selection_diff(x, 2, 8 * 256)
    assert sel.shape == (2, 1024, g.hidden_size)
    assert rel_err(sel.float().cpu(), v.float().cpu().expand_as(sel)) < 1e-2


def test_multiscale_pool_linearity_and_mass():
    """pool(a x + b y) = a pool(x) + b pool(y) for the plain multi-scale concat; the dynamic gates sum to one."""
    from u2tokenizer_b200 import ops
    B, K, E = 2, 1024, 4096
    x, y = torch.randn(B, K, E, device=DEV).bfloat16(), torch.randn(B, K, E, device=DEV).bfloat16()
    z = (0.5 * x.float() - 0.25 * y.float()).bfloat16()
    px, py, pz = (ops.multiscale_pool(t, None, 0.0, False).float() for t in (x, y, z))
    assert px.shape == (B, 1792, E)
    assert rel_err(pz, 0.5 * px - 0.25 * py) < 2e-2
    w = torch.randn(E, device=DEV) * 0.02
    dyn = ops.multiscale_pool(x, w, 0.1, True).float()
    # K % 4 == 0: the three scales see the same global mean -> equal gates 1/3 (reference svr.py:126-151)
    assert rel_err(dyn, px / 3.0) < 2e-2


def test_cross_attention_identical_keys_gives_value_mean():
    """With identical keys the softmax is uniform: the linear aggregation returns the mean of the (raw) visual values
    for every query (dh = 512, 1792 keys)."""
    eng, g = _engine()
    B, Q, M, E = 2, 256, 1792, g.hidden_size
    q = torch.randn(B * Q, E, device=DEV).bfloat16()
    row = torch.randn(E, device=DEV).bfloat16()
    vis = row.expand(B * M, E).contiguous()
    out = eng._cross_attention(q, vis, B, Q, M, eng.linagg, residual=None).float().cpu()
    assert rel_err(out, row.float().cpu().expand_as(out)) < 1e-2


def test_decode_equals_teacher_forced_prefill_full_width():
    """Qwen3-8B widths (E 4096, 32/8 heads of 128, I 12288): KV-cached decode steps on the wgmma stream-K path
    reproduce the teacher-forced prefill logits of the same tokens (both paths share only the weights)."""
    eng, g = _engine()
    B, L = 4, 40
    emb = (torch.randn(B, L, g.hidden_size, device=DEV) * 0.5).bfloat16()
    full = eng.lm_logits(eng.prefill(emb)).float()
    cache = eng.new_cache(B, L + 4)
    eng.prefill(emb[:, :L - 6].contiguous(), cache)
    eng.reset_decode_state(B)
    bufs = eng._decode_buffers(B)
    saved = eng.embed
    try:
        for t in range(L - 6, L):
            eng.embed = emb[:, t].contiguous()           # a 4-row "table": ids 0..3 select this step's embeddings
            bufs["ids"].copy_(torch.arange(B, device=DEV).view(B, 1))
            lg = eng.decode_step(cache)
            assert rel_err(lg.cpu(), full[:, t].cpu()) < 3e-2, t
    finally:
        eng.embed = saved


def test_vit_attention_permutation_equivariance():
    """Non-causal attention without positional bias is equivariant to a permutation of the keys/values and
    the fused wgmma kernel must agree with the unfused GEMM -> softmax -> GEMM path (S = 2049)."""
    eng, g = _engine()
    F_, S, H, dh = 2, 2049, 12, 64
    Sp = (S + 7) // 8 * 8
    qkv = torch.randn(F_, Sp, 3, H, dh, device=DEV).bfloat16()
    out_f = torch.zeros(F_, Sp, H * dh, device=DEV, dtype=torch.bfloat16)
    eng.use_flash = True
    eng._attention(qkv[:, :S, 0], qkv[:, :S, 1], qkv[:, :S, 2], out_f[:, :S], dh ** -0.5)
    out_u = torch.zeros_like(out_f)
    eng.use_flash = False
    eng._attention(qkv[:, :S, 0], qkv[:, :S, 1], qkv[:, :S, 2], out_u[:, :S], dh ** -0.5)
    eng.use_flash = True
    assert rel_err(out_f.float().cpu(), out_u.float().cpu()) < 1e-2
    perm = torch.randperm(S, device=DEV)
    kv = qkv.clone()
    kv[:, :S, 1:] = qkv[:, perm][:, :, 1:]
    out_p = torch.zeros_like(out_f)
    eng._attention(qkv[:, :S, 0], kv[:, :S, 1], kv[:, :S, 2], out_p[:, :S], dh ** -0.5)
    assert rel_err(out_p.float().cpu(), out_f.float().cpu()) < 1e-2
