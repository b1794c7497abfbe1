"""generate() over prompts of different lengths: attention_mask -> per-row prompt lengths (left padding moved to the
right before the visual-token splice), per-sequence positions in the decode kernels, one decode loop for the batch.
Each row of a ragged batch must give what a call on that row alone gives."""
import math

import pytest
import torch

from common import tiny_geometry

DEV = "cuda"


# ------------------------------------------------------------------------------------------------
# mask handling (CPU)
# ------------------------------------------------------------------------------------------------
def _rows(ids, mask, min_len=1):
    from u2tokenizer_b200.modeling import U2MetaForCausalLM
    return U2MetaForCausalLM._generate_prompt_rows(ids, mask, min_len=min_len)


def test_mask_to_lengths_and_left_to_right():
    ids = torch.tensor([[1, 2, 3, 4, 5],
                        [6, 7, 8, 0, 0],      # right-padded
                        [0, 0, 9, 10, 11],    # left-padded
                        [0, 0, 0, 0, 12]])    # left-padded, one token
    mask = torch.tensor([[1, 1, 1, 1, 1], [1, 1, 1, 0, 0], [0, 0, 1, 1, 1], [0, 0, 0, 0, 1]])
    out, lens = _rows(ids, mask)
    assert lens.tolist() == [5, 3, 3, 1]
    assert out.tolist() == [[1, 2, 3, 4, 5], [6, 7, 8, 0, 0], [9, 10, 11, 0, 0], [12, 0, 0, 0, 0]]
    # the visual tokens land at 1..n_vis of the moved row, as for the row alone
    assert out[2, 0].item() == 9


def test_all_ones_or_no_mask_keeps_the_uniform_path():
    ids = torch.arange(12).view(3, 4)
    for mask in (None, torch.ones(3, 4, dtype=torch.long), torch.ones(3, 4, dtype=torch.bool)):
        out, lens = _rows(ids, mask)
        assert out is ids and lens is None


@pytest.mark.parametrize("row", [[1, 0, 1, 1], [0, 1, 1, 0], [1, 0, 0, 1], [0, 1, 0, 1]])
def test_masks_with_holes_are_refused(row):
    ids = torch.zeros(2, 4, dtype=torch.long)
    mask = torch.tensor([[1, 1, 1, 1], row])
    with pytest.raises(NotImplementedError, match="attention_mask"):
        _rows(ids, mask)


def test_rows_too_short_for_bos_and_visual_tokens_are_refused():
    ids = torch.zeros(2, 6, dtype=torch.long)
    mask = torch.tensor([[1, 1, 1, 1, 1, 1], [0, 0, 0, 1, 1, 1]])
    assert _rows(ids, mask, min_len=3)[1].tolist() == [6, 3]
    with pytest.raises(ValueError, match="rows \\[1\\]"):
        _rows(ids, mask, min_len=4)
    with pytest.raises(ValueError):
        _rows(ids, torch.tensor([[1, 1, 1, 1, 1, 1], [0, 0, 0, 0, 0, 0]]))
    with pytest.raises(ValueError):
        _rows(ids, torch.ones(2, 5, dtype=torch.long))


def test_engine_row_lengths_and_cache_lengths():
    from u2tokenizer_b200.engine import KVCache, U2Engine
    assert U2Engine._row_lengths(None, 3, 7).tolist() == [7, 7, 7]
    assert U2Engine._row_lengths([7, 2, 5], 3, 7).tolist() == [7, 2, 5]
    for bad in ([7, 2], [8, 2, 5], [0, 2, 5]):
        with pytest.raises(ValueError):
            U2Engine._row_lengths(bad, 3, 7)
    cache = KVCache(tiny_geometry(), 3, 16, "cpu")
    cache.set_length(4)
    assert cache.length_dev.tolist() == [4, 4, 4] and cache.length_plus1_dev.tolist() == [5, 5, 5]
    cache.set_length(torch.tensor([4, 9, 1]))
    assert cache.length == 9 and cache.length_dev.tolist() == [4, 9, 1] and cache.length_plus1_dev.tolist() == [5, 10, 2]
    cache.advance_device()
    assert cache.length == 10 and cache.length_dev.tolist() == [5, 10, 2]
    with pytest.raises(ValueError):
        cache.set_length([1, 2])
    with pytest.raises(ValueError):
        cache.set_length([1, 2, 17])


# ------------------------------------------------------------------------------------------------
# ops: one position per sequence
# ------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _close(out, ref, tol=1e-2):
    err = (out.float() - ref.float()).abs().max().item()
    scale = ref.float().abs().max().item() + 1e-6
    assert err / scale < tol, f"max abs err {err:.4g} vs scale {scale:.4g}"


def _rot(u):
    h = u.shape[-1] // 2
    return torch.cat((-u[..., h:], u[..., :h]), -1)


def _fused_case(dh, Hq, Hkv, Tmax, B, seed):
    g = _gen(seed)
    ld = (Hq + 2 * Hkv) * dh
    qkv = torch.randn(B, ld, device=DEV, generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    inv = 1.0 / (1e6 ** (torch.arange(0, dh, 2, device=DEV).float() / dh))
    qw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g)
    kw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g)
    return qkv, kc, vc, inv, qw, kw


def _run_fused(qkv, kc, vc, inv, qw, kw, dh, Hq, Hkv, Tmax, splits, pos_dev, per_seq):
    from u2tokenizer_b200 import ops
    out = torch.empty(qkv.shape[0], Hq * dh, device=DEV, dtype=torch.bfloat16)
    ops.decode_attention_fused(qkv, kc, vc, out, B=qkv.shape[0], Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, inv_freq=inv,
                               scale=1 / math.sqrt(dh), pos_dev=pos_dev, q_norm_w=qw, k_norm_w=kw, eps=1e-6,
                               kv_splits=splits, pos_per_seq=per_seq)
    return out


def _check_fused_ragged(dh, Hq, Hkv, splits, positions, Tmax):
    B = len(positions)
    qkv, kc, vc, inv, qw, kw = _fused_case(dh, Hq, Hkv, Tmax, B, seed=dh * 7 + Hq + sum(positions))
    kc0, vc0 = kc.clone(), vc.clone()
    pd = torch.tensor(positions, device=DEV, dtype=torch.int32)
    out = _run_fused(qkv, kc, vc, inv, qw, kw, dh, Hq, Hkv, Tmax, splits, pd, True)
    t = qkv.float().view(B, Hq + 2 * Hkv, dh)
    for b, pos in enumerate(positions):
        q, k, v = t[b, :Hq], t[b, Hq:Hq + Hkv], t[b, Hq + Hkv:]
        q = qw * q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + 1e-6)
        k = kw * k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + 1e-6)
        emb = torch.cat((pos * inv, pos * inv))
        q = (q * emb.cos() + _rot(q) * emb.sin()).bfloat16().float()
        k = (k * emb.cos() + _rot(k) * emb.sin()).bfloat16().float()
        _close(kc[b, :, pos], k, 1e-2)
        assert torch.equal(vc[b, :, pos].float(), v)
        keep = torch.ones(Tmax, dtype=torch.bool, device=DEV)
        keep[pos] = False  # only row b's own position changed in row b's cache
        assert torch.equal(kc[b, :, keep], kc0[b, :, keep]) and torch.equal(vc[b, :, keep], vc0[b, :, keep]), b
        K = kc[b, :, :pos + 1].float().repeat_interleave(Hq // Hkv, 0)
        V = vc[b, :, :pos + 1].float().repeat_interleave(Hq // Hkv, 0)
        ref = (torch.softmax(q[:, None] @ K.transpose(-1, -2) / math.sqrt(dh), -1) @ V).reshape(Hq * dh)
        _close(out[b], ref, 1e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 2, 4, 8])
@pytest.mark.parametrize("dh,Hq,Hkv", [(128, 32, 8), (64, 8, 8), (32, 4, 2)])
def test_fused_decode_attention_per_sequence_positions(dh, Hq, Hkv, splits):
    _check_fused_ragged(dh, Hq, Hkv, splits, (0, 290, 543), Tmax=600)


@pytest.mark.gpu
@pytest.mark.parametrize("splits,positions,Tmax", [(2, (511, 512, 1100), 1200), (4, (1023, 1024, 31), 1100),
                                                   (8, (3, 2047, 2500), 2600)])
@pytest.mark.parametrize("dh,Hq,Hkv", [(128, 32, 8), (32, 4, 2)])
def test_fused_decode_attention_per_sequence_split_rounds(dh, Hq, Hkv, splits, positions, Tmax):
    """Rows whose key counts end exactly on, and one past, a cluster round (S x 256 keys), next to short rows."""
    _check_fused_ragged(dh, Hq, Hkv, splits, positions, Tmax)


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 4])
def test_fused_decode_attention_equal_positions_are_bit_identical(splits):
    dh, Hq, Hkv, Tmax = 128, 32, 8, 600
    qkv, kc, vc, inv, qw, kw = _fused_case(dh, Hq, Hkv, Tmax, 3, seed=5)
    kc2, vc2 = kc.clone(), vc.clone()
    shared = _run_fused(qkv, kc, vc, inv, qw, kw, dh, Hq, Hkv, Tmax, splits,
                        torch.tensor([290], device=DEV, dtype=torch.int32), False)
    per_row = _run_fused(qkv, kc2, vc2, inv, qw, kw, dh, Hq, Hkv, Tmax, splits,
                         torch.full((3,), 290, device=DEV, dtype=torch.int32), True)
    assert torch.equal(shared, per_row) and torch.equal(kc, kc2) and torch.equal(vc, vc2)


def _rope_run(x, inv, qw, kw, dh, Hq, Hkv, S, Tmax, pos_dev, per_batch):
    from u2tokenizer_b200 import ops
    B = x.shape[0] // S
    kc = torch.zeros(B, Hkv, Tmax, dh, device=DEV, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    ops.rope(x, rows=B * S, ld=x.shape[1], dh=dh, n_q=Hq, n_k=Hkv, n_v=Hkv, inv_freq=inv, q_norm_w=qw, k_norm_w=kw,
             eps=1e-6, pos0=0, pos_div=1, pos_mod=S, pos0_dev=pos_dev, k_cache=kc, v_cache=vc, Tmax=Tmax,
             rows_per_batch=S, pos0_per_batch=per_batch)
    return kc, vc


@pytest.mark.gpu
@pytest.mark.parametrize("dh", [32, 64, 128])
@pytest.mark.parametrize("S", [1, 4])
def test_rope_per_batch_positions(dh, S):
    Hq, Hkv, Tmax, pos0 = 4, 2, 64, (0, 37, 11)
    B = len(pos0)
    g = _gen(dh + S)
    x = torch.randn(B * S, (Hq + 2 * Hkv) * dh, device=DEV, generator=g).bfloat16()
    x0 = x.clone()
    inv = 1.0 / (10000 ** (torch.arange(0, dh, 2, device=DEV).float() / dh))
    qw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g)
    kw = 1 + 0.1 * torch.randn(dh, device=DEV, generator=g)
    pd = torch.tensor(pos0, device=DEV, dtype=torch.int32)
    kc, vc = _rope_run(x, inv, qw, kw, dh, Hq, Hkv, S, Tmax, pd, True)
    t = x0.float().view(B, S, Hq + 2 * Hkv, dh)
    got = x.float().view(B, S, Hq + 2 * Hkv, dh)
    for b, p0 in enumerate(pos0):
        q, k, v = t[b, :, :Hq], t[b, :, Hq:Hq + Hkv], t[b, :, Hq + Hkv:]
        q = qw * q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + 1e-6)
        k = kw * k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + 1e-6)
        fr = torch.outer(torch.arange(p0, p0 + S, device=DEV).float(), inv)
        emb = torch.cat((fr, fr), -1)[:, None]
        qr, kr = q * emb.cos() + _rot(q) * emb.sin(), k * emb.cos() + _rot(k) * emb.sin()
        _close(got[b, :, :Hq], qr, 1e-2)
        _close(got[b, :, Hq:Hq + Hkv], kr, 1e-2)
        assert torch.equal(got[b, :, Hq + Hkv:], v)
        _close(kc[b, :, p0:p0 + S].permute(1, 0, 2), kr, 1e-2)
        assert torch.equal(vc[b, :, p0:p0 + S].permute(1, 0, 2).float(), v)
        written = torch.zeros(Tmax, dtype=torch.bool, device=DEV)
        written[p0:p0 + S] = True
        assert kc[b, :, ~written].abs().max().item() == 0 and vc[b, :, ~written].abs().max().item() == 0
    # equal entries: the same bits as the shared position
    x1, x2 = x0.clone(), x0.clone()
    kc1, vc1 = _rope_run(x1, inv, qw, kw, dh, Hq, Hkv, S, Tmax, torch.tensor([9], device=DEV, dtype=torch.int32), False)
    kc2, vc2 = _rope_run(x2, inv, qw, kw, dh, Hq, Hkv, S, Tmax, torch.full((B,), 9, device=DEV, dtype=torch.int32), True)
    assert torch.equal(x1, x2) and torch.equal(kc1, kc2) and torch.equal(vc1, vc2)


@pytest.mark.gpu
@pytest.mark.parametrize("dh", [32, 64, 128])
def test_decode_attention_per_sequence_lengths(dh):
    from u2tokenizer_b200 import ops
    B, Hq, Hkv, Tmax, T = 3, 8, 2, 600, (1, 545, 17)
    g = _gen(dh + 1)
    q = torch.randn(B, Hq * dh, device=DEV, generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Tmax, dh, device=DEV, generator=g).bfloat16()
    kw = dict(B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, ldq=Hq * dh, ldo=Hq * dh, scale=1 / math.sqrt(dh))
    out = torch.empty(B, Hq * dh, device=DEV, dtype=torch.bfloat16)
    ops.decode_attention(q, kc, vc, out, T_dev=torch.tensor(T, device=DEV, dtype=torch.int32), T_per_seq=True, **kw)
    for b, Tb in enumerate(T):
        qq = q[b].float().view(Hq, 1, dh)
        kk = kc[b, :, :Tb].float().repeat_interleave(Hq // Hkv, 0)
        vv = vc[b, :, :Tb].float().repeat_interleave(Hq // Hkv, 0)
        ref = (torch.softmax(qq @ kk.transpose(-1, -2) / math.sqrt(dh), -1) @ vv).reshape(Hq * dh)
        _close(out[b], ref, 1e-2)
    shared = torch.empty_like(out)
    ops.decode_attention(q, kc, vc, shared, T_dev=torch.tensor([300], device=DEV, dtype=torch.int32), **kw)
    ops.decode_attention(q, kc, vc, out, T_dev=torch.full((B,), 300, device=DEV, dtype=torch.int32), T_per_seq=True,
                         **kw)
    assert torch.equal(shared, out)


# ------------------------------------------------------------------------------------------------
# engine: a ragged batch against the oracle and the engine's own batch-1 runs
# ------------------------------------------------------------------------------------------------
QLENS = (6, 2, 11)


def _ragged_inputs(g, qlens=QLENS, left=False, pad_id=0):
    """One synthetic study per row (its own volume, question and question_ids), padded to the longest prompt."""
    from u2tokenizer_b200.synthetic import synthetic_inputs
    rows = [synthetic_inputs(g, batch=1, frames=2, n_question=n, lt=12, seed=100 + i) for i, n in enumerate(qlens)]
    lens = [r[1].shape[1] for r in rows]
    L = max(lens)
    ids = torch.full((len(rows), L), pad_id, dtype=torch.long)
    mask = torch.zeros(len(rows), L, dtype=torch.long)
    for b, (_, rid, _) in enumerate(rows):
        sl = slice(L - lens[b], L) if left else slice(0, lens[b])
        ids[b, sl] = rid[0]
        mask[b, sl] = 1
    images = torch.cat([r[0] for r in rows])
    qids = torch.cat([r[2] for r in rows])
    return rows, images, ids, qids, mask, lens


def _upto(margins_row, thr, n):
    low = (margins_row[:n] < thr).nonzero()
    return int(low[0]) if len(low) else n


def _engine_family(family):
    if family == "qwen3":
        return tiny_geometry(), dict(bigram=1.0)
    rs = dict(factor=8.0, high_freq_factor=4.0, low_freq_factor=1.0, original_max_position_embeddings=16,
              rope_type="llama3")
    return (tiny_geometry(qk_norm=False, rope_theta=500000.0, rope_scaling=rs, tie_word_embeddings=True, head_dim=32),
            dict(head_tail=1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_engine_ragged_batch_matches_rows_alone(family):
    from oracle import u2_oracle as O
    from u2tokenizer_b200.engine import U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, head_kw = _engine_family(family)
    sd16 = synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **head_kw)
    eng = U2Engine(g, sd16, device=DEV)
    sd = {k: v.float() for k, v in sd16.items()}
    rows, images, ids, qids, _, lens = _ragged_inputs(g)
    n_new = 20
    refs, thr = [], 0.0
    for im, rid, rq in rows:
        with torch.no_grad():
            ref_logits = O.decoder_forward(sd, O.multimodal_embeds(sd, rid, im, rq, g), g)[0]
            refs.append(O.greedy_generate(sd, rid, im, rq, g, max_new_tokens=n_new))
        lg = eng.lm_logits(eng.prefill(eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda()))).float().cpu()
        thr = max(thr, 4.0 * (lg - ref_logits).abs().max().item())
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    for impl in ("tcgen05", "gemv"):
        eng.decode_impl = impl
        alone = [eng.generate_greedy(eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda()), n_new).cpu()
                 for im, rid, rq in rows]
        for use_graph in (False, True):
            got = eng.generate_greedy(emb, n_new, use_graph=use_graph, lengths=lens).cpu()
            assert got.shape == (len(rows), n_new)
            compared = 0
            for b, (ref_ids, margins) in enumerate(refs):
                upto = _upto(margins[0], thr, n_new)
                compared += upto
                assert torch.equal(got[b, :upto], ref_ids[0, :upto]), (impl, use_graph, b, got[b], ref_ids[0])
                assert torch.equal(got[b, :upto], alone[b][0, :upto]), (impl, use_graph, b, got[b], alone[b][0])
            print(f"[{family} {impl} graph={use_graph}] ragged rows identical to the oracle on {compared}/{got.numel()} "
                  f"compared tokens; {sum(torch.equal(got[b], alone[b][0]) for b in range(len(rows)))}/{len(rows)} "
                  f"rows identical to the batch-1 runs")
            if family == "qwen3":
                assert compared >= 0.9 * got.numel(), (compared, thr)


# ------------------------------------------------------------------------------------------------
# surface: model.generate(..., attention_mask=mask)
# ------------------------------------------------------------------------------------------------
def _make_model():
    from u2tokenizer_b200.configuration import U2Qwen3Config
    from u2tokenizer_b200.geometry import Geometry
    from u2tokenizer_b200.modeling import U2Qwen3ForCausalLM
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    cfg = U2Qwen3Config(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, head_dim=32, vocab_size=512, image_size=[16, 64, 64], vit_hidden_size=96,
                        vit_mlp_dim=192, vit_num_layers=2, vit_num_heads=4, u2t_num_layers=2, u2t_top_k=8,
                        num_3d_query_token=8, tie_word_embeddings=False, rms_norm_eps=1e-6)
    model = U2Qwen3ForCausalLM(cfg)
    g = Geometry.from_hf(cfg)
    sd16 = synthetic_state_dict(g, seed=9, device="cpu", dtype=torch.bfloat16, bigram=1.0)
    model.load_state_dict(sd16, strict=False)
    model = model.to(torch.bfloat16).cuda().eval()
    model.generation_config.eos_token_id = None
    return model, g, {k: v.float() for k, v in sd16.items()}


def _surface_refs(model, g, sd, rows, n_new):
    """Per-row oracle ids / margins, the margin threshold from the per-row prefill error, and per-row model calls."""
    from oracle import u2_oracle as O
    refs, alone, thr = [], [], 0.0
    for im, rid, rq in rows:
        with torch.no_grad():
            ref_logits = O.forward_logits(sd, rid, im, rq, g)
            refs.append(O.greedy_generate(sd, rid, im, rq, g, max_new_tokens=n_new))
        lg = model(images=im.cuda(), input_ids=rid.cuda(), question_ids=rq.cuda()).logits.float().cpu()
        thr = max(thr, 4.0 * (lg - ref_logits).abs().max().item())
        alone.append(model.generate(im.cuda(), rid.cuda(), question_ids=rq.cuda(), max_new_tokens=n_new,
                                    do_sample=False).cpu())
    return refs, alone, thr


@pytest.mark.gpu
def test_generate_with_right_and_left_padded_masks():
    model, g, sd = _make_model()
    n_new = 12
    rows, images, ids_r, qids, mask_r, lens = _ragged_inputs(g)
    _, _, ids_l, _, mask_l, _ = _ragged_inputs(g, left=True)
    refs, alone, thr = _surface_refs(model, g, sd, rows, n_new)
    kw = dict(question_ids=qids.cuda(), max_new_tokens=n_new, do_sample=False)
    right = model.generate(images.cuda(), ids_r.cuda(), attention_mask=mask_r.cuda(), **kw).cpu()
    left = model.generate(images.cuda(), ids_l.cuda(), attention_mask=mask_l.cuda(), **kw).cpu()
    assert right.shape == (len(rows), n_new)
    # left padding is normalised to right padding before the splice: the very same computation
    assert torch.equal(left, right)
    for b, (ref_ids, margins) in enumerate(refs):
        upto = _upto(margins[0], thr, n_new)
        assert upto >= n_new // 2, (b, margins[0], thr)
        assert torch.equal(right[b, :upto], ref_ids[0, :upto]), (b, right[b], ref_ids[0])
        assert torch.equal(right[b, :upto], alone[b][0, :upto]), (b, right[b], alone[b][0])
    # max_length keeps HF's meaning: new tokens = max_length - padded width
    ml = model.generate(images.cuda(), ids_r.cuda(), attention_mask=mask_r.cuda(), question_ids=qids.cuda(),
                        max_length=ids_r.shape[1] + 5, do_sample=False).cpu()
    assert torch.equal(ml, right[:, :5])
    # a hole in the mask is refused, as forward() refuses it
    bad = mask_r.clone()
    bad[0, 3] = 0
    with pytest.raises(NotImplementedError):
        model.generate(images.cuda(), ids_r.cuda(), attention_mask=bad.cuda(), **kw)
    short = mask_r.clone()
    short[1, g.num_3d_query_token:] = 0  # <bos> + all but one visual token
    with pytest.raises(ValueError):
        model.generate(images.cuda(), ids_r.cuda(), attention_mask=short.cuda(), **kw)


@pytest.mark.gpu
def test_all_ones_mask_is_bit_identical_to_no_mask():
    model, g, sd = _make_model()
    from u2tokenizer_b200.synthetic import synthetic_inputs
    images, ids, qids = synthetic_inputs(g, batch=3, frames=2, n_question=6, lt=12)
    kw = dict(question_ids=qids.cuda(), max_new_tokens=10, do_sample=False)
    a = model.generate(images.cuda(), ids.cuda(), **kw).cpu()
    b = model.generate(images.cuda(), ids.cuda(), attention_mask=torch.ones_like(ids).cuda(), **kw).cpu()
    assert torch.equal(a, b)


@pytest.mark.gpu
def test_ragged_num_return_sequences_crosses_the_chunk_boundary():
    model, g, sd = _make_model()
    rows, images, ids, qids, mask, lens = _ragged_inputs(g, qlens=(6, 11))
    args = (images.cuda(), ids.cuda())
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=7)
    greedy = model.generate(*args, do_sample=False, **kw).cpu()
    # 2 prompts x 9 samples = 16 + 2 rows; every sample continues from its own prompt's length
    out = model.generate(*args, do_sample=True, top_p=1e-6, num_return_sequences=9, seed=3, **kw).cpu()
    assert out.shape == (18, 7)
    assert torch.equal(out, greedy.repeat_interleave(9, dim=0))


@pytest.mark.gpu
def test_ragged_eos_padding_per_row():
    model, g, sd = _make_model()
    rows, images, ids, qids, mask, lens = _ragged_inputs(g)
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=10, do_sample=False)
    free = model.generate(images.cuda(), ids.cuda(), **kw).cpu()
    eos = int(free[0, 2])
    got = model.generate(images.cuda(), ids.cuda(), eos_token_id=eos, pad_token_id=0, **kw).cpu()
    w = got.shape[1]
    for b in range(free.shape[0]):
        hit = (free[b, :w] == eos).nonzero()
        if len(hit):
            first = int(hit[0])
            assert torch.equal(got[b, :first + 1], free[b, :first + 1]), b
            assert (got[b, first + 1:] == 0).all(), b
        else:
            assert torch.equal(got[b], free[b, :w]), b
    assert (got[0, 3:] == 0).all()


@pytest.mark.gpu
def test_ragged_then_uniform_reuses_the_decode_graph():
    model, g, sd = _make_model()
    from u2tokenizer_b200.synthetic import synthetic_inputs
    rows, images, ids, qids, mask, lens = _ragged_inputs(g)
    kw = dict(max_new_tokens=9, do_sample=False)
    model.generate(images.cuda(), ids.cuda(), question_ids=qids.cuda(), attention_mask=mask.cuda(), **kw)
    st = model.engine()._gen_state
    graph = st["graph"]
    assert graph is not None
    # a uniform batch of the same size and padded width: the same (batch, capacity) -> the same captured step
    u_images, u_ids, u_qids = synthetic_inputs(g, batch=3, frames=2, n_question=ids.shape[1] - g.num_3d_query_token,
                                               lt=12, seed=7)
    assert u_ids.shape == ids.shape
    uni = model.generate(u_images.cuda(), u_ids.cuda(), question_ids=u_qids.cuda(), **kw).cpu()
    assert model.engine()._gen_state is st and st["graph"] is graph
    fresh, _, _ = _make_model()
    want = fresh.generate(u_images.cuda(), u_ids.cuda(), question_ids=u_qids.cuda(), **kw).cpu()
    assert torch.equal(uni, want)
