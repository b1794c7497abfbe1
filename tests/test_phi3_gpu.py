"""The mu2-Phi-3 family on the GPU: the head_dim-96 and sliding-window decode attention (fused single-CTA, split-KV
cluster, unfused), the windowed causal softmax, and the engine against the fp32 Phi-3 restatement (tests/phi3_oracle.py)
on a tiny Phi-3 geometry and at Phi-3-mini widths.

Tolerances as for the existing kernels: decode attention max|out - ref| <= 1e-2 * max|ref| + 1e-2 against fp32 torch
on the same bf16 cache; per stage max|out - ref| / max|ref| <= 3e-2 and cosine >= 0.999 (DESIGN.md section 4); greedy ids
exact up to the first step whose oracle top-1 / top-2 margin is below 4x the logit error."""
import math

import pytest
import torch

import phi3_oracle as P3
from common import cosine, rel_err
from oracle import u2_oracle as O
from test_phi3 import WINDOW, tiny_phi3_geometry
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL, COS = 3e-2, 0.999


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def close(out, ref, tol):
    err = (out.float() - ref.float()).abs().max().item()
    assert err <= tol * ref.float().abs().max().item() + tol, err


def _visible(T, window):
    lo = max(0, T - window) if window else 0
    return lo, T


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("splits", [1, 2, 4, 8, "unfused"])
@pytest.mark.parametrize("indirect", [False, True])
@pytest.mark.parametrize("window", [0, 37, 5000])
@pytest.mark.parametrize("dh", [96, 128])
def test_decode_attention_window(dh, G, splits, indirect, window):
    """New token at per-sequence positions (one below the window, one far past it) against fp32 torch on the same
    bf16 cache; window 37 < T, 5000 >= T, 0 = none. indirect: a beam table pointing every key t < pos at another row."""
    from u2tokenizer_b200 import ops
    B, Hkv, Tmax = 3, 2, 1400
    Hq = Hkv * G
    g = gen(dh * 31 + G * 7 + window + (3 if indirect else 0))
    pos = torch.tensor([20, 700, 1300], device=DEV, dtype=torch.int32)
    kc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    table = None
    if indirect:
        table = ((torch.arange(B, device=DEV, dtype=torch.int32)[:, None] + 1 +
                  (torch.arange(Tmax, device=DEV, dtype=torch.int32)[None] % 2)) % B).contiguous()
        # a position some sequence appends to in this launch is read from the reader's own row (no read of a row
        # another CTA writes concurrently)
        table[:, pos.long()] = torch.arange(B, device=DEV, dtype=torch.int32)[:, None]
    out = torch.empty(B, Hq * dh, device=DEV, dtype=torch.bfloat16)
    scale = 1 / math.sqrt(dh)
    if splits == "unfused":
        q = torch.randn(B, Hq * dh, device=DEV, generator=g).bfloat16()
        # the unfused kernel reads T = pos + 1 keys; the new key / value sit in the cache already
        ops.decode_attention(q, kc, vc, out, B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, T_dev=(pos + 1).contiguous(),
                             ldq=Hq * dh, ldo=Hq * dh, scale=scale, T_per_seq=True, kv_src=table, window=window)
        qf = q.float().view(B, Hq, dh)
    else:
        ld = (Hq + 2 * Hkv) * dh
        qkv = torch.randn(B, ld, device=DEV, generator=g).bfloat16()
        inv = 1.0 / (1e4 ** (torch.arange(0, dh, 2, device=DEV).float() / dh))
        ops.decode_attention_fused(qkv, kc, vc, out, B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, inv_freq=inv, scale=scale,
                                   pos_dev=pos, eps=1e-5, kv_splits=splits, pos_per_seq=True, kv_src=table,
                                   window=window)
        t = qkv.float().view(B, Hq + 2 * Hkv, dh)
        rot = lambda u: torch.cat((-u[..., dh // 2:], u[..., :dh // 2]), -1)
        qf = torch.empty(B, Hq, dh, device=DEV)
        for b in range(B):
            fr = float(pos[b]) * inv
            emb = torch.cat((fr, fr))
            q, k = t[b, :Hq], t[b, Hq:Hq + Hkv]
            qf[b] = (q * emb.cos() + rot(q) * emb.sin()).bfloat16().float()
            close(kc[b, :, int(pos[b])], (k * emb.cos() + rot(k) * emb.sin()), 1e-2)
            assert torch.equal(vc[b, :, int(pos[b])].float(), t[b, Hq + Hkv:])
    for b in range(B):
        P = int(pos[b])
        lo, hi = _visible(P + 1, window)
        rows = torch.full((P + 1,), b, device=DEV, dtype=torch.long)
        if indirect:
            rows[:P] = table[b, :P].long()
        idx = torch.arange(P + 1, device=DEV)
        K = kc[rows, :, idx].float().transpose(0, 1)[:, lo:hi]   # [Hkv, n, dh]
        V = vc[rows, :, idx].float().transpose(0, 1)[:, lo:hi]
        K, V = K.repeat_interleave(G, 0), V.repeat_interleave(G, 0)
        ref = (torch.softmax(qf[b][:, None] @ K.transpose(-1, -2) * scale, -1) @ V).reshape(Hq * dh)
        close(out[b], ref, 1e-2)


@pytest.mark.parametrize("S,Sk", [(20, 20), (300, 300), (40, 1500), (1500, 1500), (9000, 9000)])
@pytest.mark.parametrize("window", [1, 24, 2047])
def test_windowed_causal_softmax(S, Sk, window):
    """Query i of S sees keys (i + Sk - S - window, i + Sk - S] (causal + sliding window), across the row kernels
    (warp / 128 / 256-thread groups, one-CTA-per-row long rows)."""
    from u2tokenizer_b200 import ops
    g = gen(S + Sk + window)
    H = 2 if S < 5000 else 1
    Skp = (Sk + 7) // 8 * 8
    sc = torch.randn(1, H, S, Skp, device=DEV, generator=g)
    out = torch.full((1, H, S, Skp), 7.0, device=DEV, dtype=torch.bfloat16)
    off = Sk - S
    ops.softmax(sc, out, n0=1, H=H, S=S, n=Sk, in_strides=(H * S * Skp, S * Skp, Skp),
                out_strides=(H * S * Skp, S * Skp, Skp), scale=0.5, causal=True, causal_off=off, window=window,
                zero_pad_to=Skp)
    i = torch.arange(S, device=DEV)[:, None] + off
    j = torch.arange(Sk, device=DEV)[None]
    vis = (j <= i) & (j > i - window)
    ref = torch.softmax((sc[..., :Sk] * 0.5).masked_fill(~vis, float("-inf")), -1)
    close(out[..., :Sk], ref, 1e-2)
    assert out[..., :Sk].float().masked_select(~vis.expand_as(ref)).abs().max().item() == 0
    assert out[..., Sk:].float().abs().max().item() == 0 if Skp > Sk else True
    with pytest.raises(RuntimeError):
        ops.softmax(sc, out, n0=1, H=H, S=S, n=Sk, in_strides=(H * S * Skp, S * Skp, Skp),
                    out_strides=(H * S * Skp, S * Skp, Skp), window=window)   # a window needs the causal mask


def _engine(g, seed):
    from u2tokenizer_b200.engine import U2Engine
    sd16 = synthetic_state_dict(g, seed=seed, device="cpu", dtype=torch.bfloat16, bigram=1.0)
    eng = U2Engine(g, sd16, device=DEV)
    return eng, {k: v.float() for k, v in sd16.items()}


def _greedy_agrees(got, ref_ids, margins, thr, min_frac=0.9):
    compared = 0
    for b in range(got.shape[0]):
        low = (margins[b] < thr).nonzero()
        upto = int(low[0]) if len(low) else got.shape[1]
        compared += upto
        assert torch.equal(got[b, :upto].cpu(), ref_ids[b, :upto]), (b, got[b], ref_ids[b], margins[b])
    assert compared >= min_frac * got.numel(), (compared, got.numel())


def test_engine_forward_and_greedy_across_window():
    """Tiny Phi-3 (E 192, 2 heads of 96, I 384, window 24): 38 prompt positions and 16 new tokens, so both the
    prefill softmax and the decode attention cut keys off; forward logits and greedy ids against the oracle."""
    g = tiny_phi3_geometry()
    eng, sd = _engine(g, 5)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=30, lt=32)
    with torch.no_grad():
        ref_emb = O.multimodal_embeds(sd, ids, images, qids, g)
        ref_logits = P3.decoder_forward(sd, ref_emb, g)[0]
        ref_ids, margins = P3.greedy_from_embeds(sd, ref_emb, g, 16)
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    logits = eng.lm_logits(eng.prefill(emb)).float().cpu()
    assert rel_err(logits, ref_logits) < TOL and cosine(logits, ref_logits) > COS
    thr = 4.0 * (logits - ref_logits).abs().max().item()
    for impl in ("tcgen05", "gemv"):
        eng.decode_impl = impl
        for use_graph in (False, True):
            got = eng.generate_greedy(emb, max_new_tokens=16, use_graph=use_graph)
            _greedy_agrees(got, ref_ids, margins, thr)
    eng.decode_impl = "tcgen05"


@pytest.mark.parametrize("impl", ["tcgen05", "gemv"])
def test_decode_matches_prefill_across_window(impl):
    """KV-cached decode steps at positions 12..47 reproduce the windowed prefill's logits (window 24)."""
    g = tiny_phi3_geometry()
    eng, _ = _engine(g, 6)
    eng.decode_impl = impl
    emb = (torch.randn(2, 48, g.hidden_size, generator=torch.Generator().manual_seed(5)) * 0.5).bfloat16().cuda()
    full = eng.lm_logits(eng.prefill(emb))
    cache = eng.new_cache(2, 64)
    eng.prefill(emb[:, :12].contiguous(), cache)
    bufs = eng._decode_buffers(2)
    eng.reset_decode_state(2)
    saved = eng.embed
    for t in range(12, 48):
        eng.embed = emb[:, t].contiguous()   # a 2-row table: ids 0, 1 select the injected embeddings
        bufs["ids"].copy_(torch.arange(2, device=DEV).view(2, 1))
        lg = eng.decode_step(cache)
        e = rel_err(lg.cpu(), full[:, t].float().cpu())
        assert e < TOL, (t, e)
    eng.embed = saved


def test_model_surface_sampling_ragged_and_beam():
    """U2Phi3ForCausalLM.generate through the same captured step: sampling (seeded, top_k=1 == greedy), a ragged
    batch (the short row decodes as if alone) and beam search."""
    from test_phi3 import tiny_phi3_config
    from u2tokenizer_b200.geometry import Geometry
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM
    cfg = tiny_phi3_config()
    g = Geometry.from_hf(cfg)
    sd16 = synthetic_state_dict(g, seed=8, device="cpu", dtype=torch.bfloat16, bigram=1.0)
    model = U2Phi3ForCausalLM(cfg).to(torch.bfloat16)
    model.load_state_dict(sd16)
    model = model.cuda().eval()
    model.generation_config.eos_token_id = None   # fixed-length outputs: every row decodes all 12 tokens
    sd = {k: v.float() for k, v in sd16.items()}
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=24, lt=32)
    images, ids, qids = images.cuda(), ids.cuda(), qids.cuda()
    kw = dict(max_new_tokens=12, eos_token_id=None)
    greedy = model.generate(images, ids, question_ids=qids, do_sample=False, **kw)
    s1 = model.generate(images, ids, question_ids=qids, do_sample=True, top_k=1, seed=3, **kw)
    assert torch.equal(s1, greedy)
    a = model.generate(images, ids, question_ids=qids, do_sample=True, temperature=1.5, top_k=0, seed=4, **kw)
    b = model.generate(images, ids, question_ids=qids, do_sample=True, temperature=1.5, top_k=0, seed=4, **kw)
    assert torch.equal(a, b) and int(a.min()) >= 0 and int(a.max()) < g.vocab_size
    # ragged: row 1 keeps 7 fewer question tokens (right padding) and must decode like its prompt alone
    L = ids.shape[1]
    mask = torch.ones_like(ids)
    mask[1, L - 7:] = 0
    rag = model.generate(images, ids, question_ids=qids, attention_mask=mask, do_sample=False, **kw)
    with torch.no_grad():
        emb = O.multimodal_embeds(sd, ids.cpu(), images.cpu(), qids.cpu(), g)
        ref0, m0 = P3.greedy_from_embeds(sd, emb[:1], g, 12)
        ref1, m1 = P3.greedy_from_embeds(sd, emb[1:, :L - 7], g, 12)
        ref_logits = P3.decoder_forward(sd, emb, g)[0]
    logits = model(images=images, input_ids=ids, question_ids=qids).logits.float().cpu()
    thr = 4.0 * (logits - ref_logits).abs().max().item()
    _greedy_agrees(rag, torch.cat([ref0, ref1]), torch.cat([m0, m1]), thr, min_frac=0.8)
    beams = model.generate(images, ids, question_ids=qids, num_beams=3, num_return_sequences=2, do_sample=False, **kw)
    assert beams.shape == (4, 12) and int(beams.min()) >= 0 and int(beams.max()) < g.vocab_size
    sc = model.engine().last_beam_scores
    assert torch.isfinite(sc).all() and bool((sc[0::2] >= sc[1::2]).all())


def test_phi3_mini_widths():
    """E 3072, 32 heads of 96 (MHA), I 8192, V 32064, two decoder layers, mu2-tokenizer at head_dim 384, window 24
    crossed: visual tokens, prefill logits and 8 teacher-forced decode steps on the wgmma decode path, each within 3e-2
    relative error and cosine 0.999 of the oracle."""
    g = tiny_phi3_geometry(hidden_size=3072, intermediate_size=8192, num_attention_heads=32, num_key_value_heads=32,
                           vocab_size=32064)
    eng, sd = _engine(g, 9)
    assert eng._use_tc_decode(2)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=28, lt=32)
    with torch.no_grad():
        ref_vis = O.visual_tokens(sd, images, qids, g)
        ref_emb = O.multimodal_embeds(sd, ids, images, qids, g)
        ref_logits, past = P3.decoder_forward(sd, ref_emb, g)
    vis = eng.visual_tokens(images.cuda(), qids.cuda()).float().cpu()
    assert rel_err(vis, ref_vis) < TOL and cosine(vis, ref_vis) > COS
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    logits = eng.lm_logits(eng.prefill(emb)).float().cpu()
    assert rel_err(logits, ref_logits) < TOL and cosine(logits, ref_logits) > COS
    force = ref_logits[:, -1].argmax(-1, keepdim=True)
    steps = [ref_logits[:, -1]]
    nxt = force[:, 0]
    with torch.no_grad():
        for _ in range(7):
            lg, past = P3.decoder_forward(sd, torch.nn.functional.embedding(nxt[:, None], sd["model.embed_tokens.weight"]),
                                          g, past)
            steps.append(lg[:, -1])
            nxt = lg[:, -1].argmax(-1)
            force = torch.cat([force, nxt[:, None]], dim=1)
    lo = []
    eng.generate_greedy(emb, max_new_tokens=8, use_graph=False, force_ids=force, logits_out=lo)
    for s, (a, r) in enumerate(zip(lo, steps)):
        a = a.float().cpu()
        assert rel_err(a, r) < TOL and cosine(a, r) > COS, s
