"""Beam search in generate(): num_beams, length_penalty and early_stopping run inside the captured decode step. The beams
of a prompt are rows of one decode batch; a beam continues another beam's KV cache through an indirection table read by
the decode attention, and HF's per-step selection and finished-hypothesis bookkeeping run as two kernels. The target is
HF generate(inputs_embeds=..., num_beams=K) (GenerationMixin._beam_search): row k of a prompt after a step is HF's
running beam k."""
import pytest
import torch

from common import tiny_geometry

DEV = "cuda"


# ------------------------------------------------------------------------------------------------
# surface (CPU)
# ------------------------------------------------------------------------------------------------
def _beam(kwargs, gc=None, num_beams=4, do_sample=False, n_ret=1, pad=None):
    from u2tokenizer_b200.modeling import U2MetaForCausalLM
    kw = dict(kwargs)
    out = U2MetaForCausalLM._generate_beam_search(kw, gc, num_beams, do_sample, n_ret, pad)
    for k in ("length_penalty", "early_stopping"):
        assert k not in kw
    return out


def test_surface_reads_kwargs_then_generation_config():
    from transformers import GenerationConfig
    b = _beam({})
    assert (b.num_beams, b.length_penalty, b.early_stopping, b.num_return_sequences) == (4, 1.0, False, 1)
    gc = GenerationConfig(num_beams=3, length_penalty=2.0, early_stopping="never")
    b = _beam({}, gc, num_beams=3, n_ret=2, pad=5)
    assert (b.length_penalty, b.early_stopping, b.num_return_sequences, b.pad_token_id) == (2.0, "never", 2, 5)
    b = _beam(dict(length_penalty=-0.5, early_stopping=True), gc)
    assert (b.length_penalty, b.early_stopping) == (-0.5, True)


@pytest.mark.parametrize("kwargs,extra,exc", [
    ({}, dict(do_sample=True), NotImplementedError),
    (dict(num_beam_groups=2), {}, NotImplementedError),
    (dict(constraints=[object()]), {}, NotImplementedError),
    (dict(force_words_ids=[[3]]), {}, NotImplementedError),
    (dict(early_stopping="sometimes"), {}, ValueError),
    (dict(early_stopping=1.0), {}, ValueError),
    (dict(length_penalty="1"), {}, ValueError),
    (dict(length_penalty=float("nan")), {}, ValueError),
    ({}, dict(n_ret=5), ValueError),
    ({}, dict(num_beams=2.0), ValueError),
    ({}, dict(num_beams=0), ValueError),
])
def test_surface_refusals(kwargs, extra, exc):
    with pytest.raises(exc):
        _beam(kwargs, **extra)


def test_generation_config_early_stopping_is_validated():
    from transformers import GenerationConfig
    gc = GenerationConfig()
    gc.early_stopping = "later"
    with pytest.raises(ValueError):
        _beam({}, gc)


def test_num_beams_1_keeps_the_greedy_kwarg_checks():
    # with one beam length_penalty / early_stopping are not consumed: they are refused as before
    from u2tokenizer_b200.modeling import U2MetaForCausalLM
    with pytest.raises(NotImplementedError, match="length_penalty"):
        U2MetaForCausalLM._check_remaining_generate_kwargs({"length_penalty": 2.0})
    with pytest.raises(TypeError, match="early_stopping"):
        U2MetaForCausalLM._check_remaining_generate_kwargs({"early_stopping": True})


def test_beam_params_block_validation():
    from u2tokenizer_b200 import _lib, ops
    blk = ops.beam_params("cpu", num_beams=4, max_new_tokens=8, eos_token_ids=(1, 2, 3), length_penalty=0.5,
                          early_stopping="never")
    p = _lib.BeamParams.from_buffer_copy(bytes(blk.numpy()))
    assert (p.num_beams, p.beams_to_keep, p.early_stopping, p.n_eos, p.length_penalty) == (4, 16, 2, 3, 0.5)
    assert _lib.BeamParams.from_buffer_copy(bytes(ops.beam_params("cpu", num_beams=3, max_new_tokens=2).numpy())
                                            ).beams_to_keep == 6
    for kw in (dict(num_beams=17), dict(num_beams=1), dict(eos_token_ids=tuple(range(9))), dict(early_stopping=1),
               dict(max_new_tokens=0)):
        with pytest.raises(ValueError):
            ops.beam_params("cpu", **{**dict(num_beams=4, max_new_tokens=8), **kw})


# ------------------------------------------------------------------------------------------------
# op: decode attention through the cache indirection table
# ------------------------------------------------------------------------------------------------
def _attn_case(B, Hq, Hkv, dh, Tmax, pos, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    qkv = (torch.randn(B, (Hq + 2 * Hkv) * dh, generator=g) * 0.5).to(DEV, torch.bfloat16)
    kc = (torch.randn(B, Hkv, Tmax, dh, generator=g) * 0.5).to(DEV, torch.bfloat16)
    vc = torch.randn(B, Hkv, Tmax, dh, generator=g).to(DEV, torch.bfloat16)
    # a table as beam search builds it: position t of row b lives in a row whose own position is past t (its slot t is
    # not appended to by this launch), or in row b itself
    pos_t = torch.tensor(pos)
    src = torch.empty(B, Tmax, dtype=torch.int32)
    for t in range(Tmax):
        ok = (pos_t > t).nonzero().flatten()
        pick = ok[torch.randint(0, len(ok), (B,), generator=g)] if len(ok) else torch.arange(B)
        src[:, t] = pick.int()
    return qkv, kc, vc, src.to(DEV), torch.tensor(pos, dtype=torch.int32, device=DEV)


def _gather_reference(q, kc, vc, src, pos, scale):
    """fp32 attention of q [B, Hq, dh] over keys 0..pos[b] of sequence b, key t < pos[b] from row src[b, t]."""
    B, Hq, dh = q.shape
    Hkv = kc.shape[1]
    out = torch.empty(B, Hq, dh, device=q.device)
    for b in range(B):
        T = int(pos[b]) + 1
        rows = src[b, :T].long().clone()
        rows[T - 1] = b
        t = torch.arange(T, device=q.device)
        k = kc[rows, :, t].float()  # [T, Hkv, dh]
        v = vc[rows, :, t].float()
        kk = k.repeat_interleave(Hq // Hkv, dim=1)
        vv = v.repeat_interleave(Hq // Hkv, dim=1)
        p = torch.softmax(torch.einsum("hd,thd->ht", q[b].float(), kk) * scale, dim=-1)
        out[b] = torch.einsum("ht,thd->hd", p, vv)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 2, 4, 8])
@pytest.mark.parametrize("dh,G", [(128, 4), (64, 2), (32, 1)])
def test_fused_decode_attention_indirect_matches_gather_reference(splits, dh, G):
    from u2tokenizer_b200 import ops
    B, Hkv, Tmax = 8, 2, 700
    Hq = Hkv * G
    pos = [5, 699, 31, 32, 300, 1, 517, 64]  # ragged positions
    qkv, kc, vc, src, pos_dev = _attn_case(B, Hq, Hkv, dh, Tmax, pos, seed=dh + splits)
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dh, 2, dtype=torch.float32, device=DEV) / dh))
    kw = dict(B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, inv_freq=inv_freq, scale=dh ** -0.5, pos_dev=pos_dev,
              kv_splits=splits, pos_per_seq=True)
    outs = {}
    for name, table in (("null", None), ("identity", torch.arange(B, dtype=torch.int32, device=DEV)[:, None]
                                         .expand(B, Tmax).contiguous()), ("random", src)):
        k2, v2 = kc.clone(), vc.clone()
        out = torch.empty(B, Hq * dh, device=DEV, dtype=torch.bfloat16)
        ops.decode_attention_fused(qkv, k2, v2, out, kv_src=table, **kw)
        outs[name] = (out, k2, v2)
    assert torch.equal(outs["null"][0], outs["identity"][0])
    out, k2, v2 = outs["random"]
    assert torch.equal(k2, outs["null"][1]) and torch.equal(v2, outs["null"][2])  # the append goes to the row's own slot
    q = torch.empty(B, Hq, dh, device=DEV, dtype=torch.bfloat16)
    # the roped query the kernel attends with, from the unfused rope kernel
    x = qkv.clone()
    ops.rope(x, rows=B, ld=x.shape[1], dh=dh, n_q=Hq, n_k=Hkv, inv_freq=inv_freq, pos0=0, pos_div=1, pos_mod=1,
             pos0_dev=pos_dev, pos0_per_batch=True, rows_per_batch=1, Tmax=Tmax)
    q.copy_(x[:, :Hq * dh].view(B, Hq, dh))
    ref = _gather_reference(q, k2, v2, src, pos, dh ** -0.5)
    err = (out.float().view(B, Hq, dh) - ref).abs().max().item()
    assert err < 2e-2, err
    # a random table gives different outputs than the own rows (it is read at all)
    assert not torch.equal(out, outs["null"][0])


@pytest.mark.gpu
@pytest.mark.parametrize("dh", [32, 64, 128])
def test_gemv_decode_attention_indirect_matches_gather_reference(dh):
    from u2tokenizer_b200 import ops
    B, Hkv, Hq, Tmax = 6, 2, 4, 400
    pos = [0, 399, 31, 200, 77, 128]
    qkv, kc, vc, src, pos_dev = _attn_case(B, Hq, Hkv, dh, Tmax, pos, seed=dh)
    q = qkv[:, :Hq * dh]
    kw = dict(B=B, Hq=Hq, Hkv=Hkv, dh=dh, Tmax=Tmax, T_dev=pos_dev + 1, ldq=qkv.stride(0), ldo=Hq * dh,
              scale=dh ** -0.5, T_per_seq=True)
    outs = []
    for table in (None, torch.arange(B, dtype=torch.int32, device=DEV)[:, None].expand(B, Tmax).contiguous(), src):
        out = torch.empty(B, Hq * dh, device=DEV, dtype=torch.bfloat16)
        ops.decode_attention(q, kc, vc, out, kv_src=table, **kw)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    ref = _gather_reference(q.view(B, Hq, dh), kc, vc, src, pos, dh ** -0.5)
    err = (outs[2].float().view(B, Hq, dh) - ref).abs().max().item()
    assert err < 2e-2, err


# ------------------------------------------------------------------------------------------------
# op: the beam step against HF's own helpers on the same log-probs
# ------------------------------------------------------------------------------------------------
class _HF:
    """The GenerationMixin beam helpers (they only use static methods of the instance)."""

    def __init__(self):
        from transformers.generation.utils import GenerationMixin
        self.g = GenerationMixin.__new__(GenerationMixin)


def _drive(V, K, P, eos, lp, es, max_new, seed):
    """Run our beam kernels and HF's _beam_search helpers step by step on the same log-probs; compare every step."""
    from u2tokenizer_b200 import _lib, ops
    hf = _HF().g
    R, C = P * K, max(2, 1 + len(eos)) * K
    g = torch.Generator(device="cpu").manual_seed(seed)
    blk = ops.beam_params(DEV, num_beams=K, length_penalty=lp, early_stopping=es, max_new_tokens=max_new,
                          eos_token_ids=eos)
    i32 = dict(device=DEV, dtype=torch.int32)
    st = dict(cand_val=torch.empty(R, _lib.BEAM_MAX_KEEP, device=DEV), cand_tok=torch.empty(R, _lib.BEAM_MAX_KEEP, **i32),
              running=torch.full((R,), -1e9, device=DEV), fin_score=torch.full((R,), -1e9, device=DEV),
              fin_info=torch.tensor([0, -1, 0, 0], **i32).repeat(R, 1), flags=torch.tensor([1, 0], **i32).repeat(P, 1),
              rec=torch.zeros(max_new, R, 2, **i32))
    st["running"].view(P, K)[:, 0] = 0
    Tmax = max_new + 4
    kv_src = torch.arange(R, **i32)[:, None].repeat(1, Tmax)
    pos_dev = torch.full((R,), 2, **i32)
    ids = torch.zeros(R, device=DEV, dtype=torch.int64)
    # HF state
    fill = eos[0]
    run_seq = torch.full((P, K, max_new), fill, dtype=torch.int64, device=DEV)
    seqs = run_seq.clone()
    run_scores = torch.zeros(P, K, device=DEV)
    run_scores[:, 1:] = -1e9
    beam_scores = torch.full((P, K), -1e9, device=DEV)
    fin = torch.zeros(P, K, dtype=torch.bool, device=DEV)
    unsat = torch.ones(P, 1, dtype=torch.bool, device=DEV)
    run_bi = torch.full((P, K, max_new), -1, dtype=torch.int32, device=DEV)
    bidx = run_bi.clone()
    top_mask = torch.cat([torch.ones(K, dtype=torch.bool), torch.zeros(C - K, dtype=torch.bool)]).to(DEV)
    eos_t = torch.tensor(eos, device=DEV)
    compared = 0
    kv_ref = kv_src.clone()
    for t in range(max_new):
        logits = torch.randn(R, V, generator=g) * 3
        logits[:, list(eos)] += 4.0  # hypotheses end often
        lpb = ops.log_softmax(logits.to(DEV))
        active = ~st["flags"][:, 1].bool()
        ops.beam_topk(lpb, st["running"], st["flags"], blk, st["cand_val"], st["cand_tok"])
        ops.beam_step(blk, st, ids, kv_src, pos_dev, V=V, step=t)
        # HF
        acc = (lpb.view(P, K, V) + run_scores[:, :, None]).reshape(P, K * V)
        topv, tseq, tbi = hf._get_top_k_continuations(acc, run_seq, run_bi, t, 0, False, C, K, V, P)
        hits = torch.isin(tseq[:, :, t], eos_t) | (t + 1 >= max_new)
        # the selection boundary gaps: the comparison is meaningful only where they exceed fp32 noise
        a_sorted = acc.topk(C + 1, dim=1).values
        gap_ok = ((a_sorted[:, C - 1] - a_sorted[:, C]) > 1e-4)
        run_seq, run_scores, run_bi = hf._get_running_beams_for_next_iteration(topv, tseq, tbi, hits, K)
        seqs, beam_scores, bidx, fin = hf._update_finished_beams(seqs, tseq, beam_scores, topv, bidx, tbi, unsat, fin,
                                                                 hits, top_mask, K, t, 0, lp, es)
        unsat = hf._check_early_stop_heuristic(unsat, run_scores, beam_scores, fin, t + 1, max_new, 0, es, lp)
        got_ids = ids.view(P, K)
        got_run = st["running"].view(P, K)
        got_fin = st["fin_score"].view(P, K)
        info = st["fin_info"].view(P, K, 4)
        for p in range(P):
            if not bool(active[p]) or not bool(gap_ok[p]):
                continue
            compared += 1
            # running beams with real scores; the rest carry -1e9 (every continuation hit a stopping criterion) and tie
            # in fp32, where torch.topk's order is unspecified: they are never continued while a real beam exists
            n = int((run_scores[p] > -1e8).sum())
            assert bool((got_run[p, n:] <= -1e8).all()), (t, p)
            assert torch.equal(got_ids[p, :n], run_seq[p, :n, t]), (t, p, got_ids[p], run_seq[p, :, t])
            assert torch.equal(got_run[p, :n], run_scores[p, :n]), (t, p)
            f = fin[p]
            assert torch.equal(info[p, :, 0].bool(), f), (t, p)
            torch.testing.assert_close(got_fin[p][f], beam_scores[p][f], rtol=1e-6, atol=0)
            assert torch.equal(info[p, :, 1][f], (bidx[p][f] >= 0).sum(-1).int() - 1), (t, p)
            # the parent beams behind the next running rows, and the reordered indirection table
            par = run_bi[p, :n, t] - p * K
            assert torch.equal(st["rec"][t, p * K:p * K + n, 1].long(), par.long()), (t, p)
            nc = 3 if t > 0 else 2  # positions holding K/V: pos_dev + 1 after a decode step, pos_dev at the first pick
            want = kv_ref[p * K + par.long(), :nc]
            assert torch.equal(kv_src[p * K:p * K + n, :nc], want), (t, p)
            assert torch.equal(kv_src[p * K:(p + 1) * K, nc], torch.arange(p * K, (p + 1) * K, **i32)), (t, p)
            # done flag = HF's stopping condition restricted to the prompt
            done = (not bool(unsat[p])) or (es is True and bool(fin[p].all())) or bool(hits[p].all())
            assert bool(st["flags"][p, 1]) == done, (t, p)
        kv_ref = kv_src.clone()
        if bool(st["flags"][:, 1].all()):
            break
    return compared, t


_STEP_CASES = [  # V, K, eos, length_penalty, early_stopping, max_new
    (151936, 4, (7,), 1.0, False, 10),
    (151936, 2, (7, 151935), 0.0, True, 8),
    (151936, 8, (3, 9, 11), 2.0, "never", 6),
    (151936, 16, (5,), -0.5, False, 5),
    (1000, 2, (7,), 1.0, True, 40),
    (1000, 4, (7, 8), 2.0, False, 40),
    (1000, 8, (3, 9, 11), -0.5, "never", 30),
    (1000, 16, (1, 2), 0.0, True, 30),
    (1000, 4, (7,), 0.0, "never", 25),
    (1000, 16, (4, 5, 6), 1.0, False, 20),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", _STEP_CASES, ids=[f"V{c[0]}-K{c[1]}-eos{len(c[2])}-lp{c[3]}-es{c[4]}" for c in _STEP_CASES])
def test_beam_step_matches_hf_helpers(case):
    V, K, eos, lp, es, max_new = case
    P = max(1, 16 // K)
    compared, last = _drive(V, K, P, eos, lp, es, max_new, seed=K * 31 + len(eos))
    assert compared >= P, (compared, last)


# ------------------------------------------------------------------------------------------------
# engine: tiny Qwen3 and Llama against HF generate(num_beams=K) replaying the engine's raw logits
# ------------------------------------------------------------------------------------------------
def _engine_family(family):
    if family == "qwen3":
        return tiny_geometry(), dict(bigram=1.0)
    rs = dict(factor=8.0, high_freq_factor=4.0, low_freq_factor=1.0, original_max_position_embeddings=16,
              rope_type="llama3")
    return (tiny_geometry(qk_norm=False, rope_theta=500000.0, rope_scaling=rs, tie_word_embeddings=True, head_dim=32),
            dict(head_tail=1.0))


def _inputs(g, qlens=(6, 2, 11)):
    from u2tokenizer_b200.synthetic import synthetic_inputs
    rows = [synthetic_inputs(g, batch=1, frames=2, n_question=n, lt=12, seed=100 + i) for i, n in enumerate(qlens)]
    lens = [r[1].shape[1] for r in rows]
    L = max(lens)
    ids = torch.zeros(len(rows), L, dtype=torch.long)
    mask = torch.zeros(len(rows), L, dtype=torch.long)
    for b, (_, rid, _) in enumerate(rows):
        ids[b, :lens[b]] = rid[0]
        mask[b, :lens[b]] = 1
    return rows, torch.cat([r[0] for r in rows]), ids, torch.cat([r[2] for r in rows]), mask, lens


def _replay_model(V, steps):
    """A PreTrainedModel whose forward returns the recorded raw logits of step i at its i-th call."""
    from transformers import GenerationMixin, PretrainedConfig, PreTrainedModel
    from transformers.modeling_outputs import CausalLMOutputWithPast

    class Cfg(PretrainedConfig):
        model_type = "u2_replay"

    class Replay(PreTrainedModel, GenerationMixin):
        config_class = Cfg
        _supports_cache_class = False

        def __init__(self, cfg):
            super().__init__(cfg)
            self.dummy = torch.nn.Parameter(torch.zeros(1))
            self.calls = 0

        def get_input_embeddings(self):
            return None

        def forward(self, input_ids=None, inputs_embeds=None, **kw):
            lg = steps[min(self.calls, len(steps) - 1)]
            self.calls += 1
            return CausalLMOutputWithPast(logits=lg[:, None, :].clone())

        def prepare_inputs_for_generation(self, input_ids, inputs_embeds=None, **kw):
            return dict(input_ids=input_ids, inputs_embeds=inputs_embeds)

    return Replay(Cfg(vocab_size=V, hidden_size=8, num_hidden_layers=1, is_decoder=True)).to(DEV)


def _hf_beam(steps, P, K, V, n_new, eos, lp, es, n_ret, procs_kw):
    m = _replay_model(V, steps)
    emb = torch.zeros(P, 1, 8, device=DEV)
    with torch.no_grad():
        return m.generate(inputs_embeds=emb, num_beams=K, max_new_tokens=n_new, eos_token_id=list(eos),
                          pad_token_id=eos[0], length_penalty=lp, early_stopping=es, num_return_sequences=n_ret,
                          do_sample=False, use_cache=False, **procs_kw)


def _hf_loop(first_logits, next_logits, P, K, V, n_new, eos, lp, es, procs=None, dev=DEV):
    """HF _beam_search step by step through GenerationMixin's own helpers, on logits a callback supplies:
    next_logits(parent_rows [P*K], tokens [P*K]) -> the logits [P*K, V] of the next step for the reordered beams.
    Returns per step (tok, par, real, gap, active) [P, K] / [P] and the final (sequences, scores, beam_indices, finished).
    gap: the smallest difference between consecutive values of the prompt's top beams_to_keep + 1 accumulated scores, so a
    step whose gap exceeds the numerical error of the logits selects the same beams in the same order on any
    implementation; real: running beams with scores above the -1e9 mask; active: the prompt was not done before."""
    hf = _HF().g
    C = max(2, 1 + len(eos)) * K
    fill = eos[0]
    run_seq = torch.full((P, K, n_new), fill, dtype=torch.int64, device=dev)
    seqs = run_seq.clone()
    run_scores = torch.zeros(P, K, device=dev)
    run_scores[:, 1:] = -1e9
    beam_scores = torch.full((P, K), -1e9, device=dev)
    fin = torch.zeros(P, K, dtype=torch.bool, device=dev)
    unsat = torch.ones(P, 1, dtype=torch.bool, device=dev)
    run_bi = torch.full((P, K, n_new), -1, dtype=torch.int32, device=dev)
    bidx = run_bi.clone()
    top_mask = torch.cat([torch.ones(K, dtype=torch.bool), torch.zeros(C - K, dtype=torch.bool)]).to(dev)
    eos_t = torch.tensor(eos, device=dev)
    off = (torch.arange(P, device=dev) * K)[:, None]
    done = torch.zeros(P, dtype=torch.bool, device=dev)
    steps, logits = [], first_logits
    for t in range(n_new):
        lpb = torch.log_softmax(logits.float(), dim=-1)
        if procs is not None:
            lpb = procs(run_seq.reshape(P * K, n_new)[:, :t], lpb)
        acc = (lpb.view(P, K, V) + run_scores[:, :, None]).reshape(P, K * V)
        topv, tseq, tbi = hf._get_top_k_continuations(acc, run_seq, run_bi, t, 0, False, C, K, V, P)
        hits = torch.isin(tseq[:, :, t], eos_t) | (t + 1 >= n_new)
        # the gaps that decide this step: the order of the candidates up to the (K+1)-th one that continues (which ones
        # run on, in which row, and which of the top K finish)
        top = torch.cat([topv, acc.topk(C + 1, dim=1).values[:, C:]], dim=1)
        gap = torch.empty(P, device=dev)
        for p in range(P):
            cont = (~hits[p]).nonzero().flatten()
            m = int(cont[K]) if len(cont) > K else C
            gap[p] = (top[p, :m] - top[p, 1:m + 1]).min()
        run_seq, run_scores, run_bi = hf._get_running_beams_for_next_iteration(topv, tseq, tbi, hits, K)
        seqs, beam_scores, bidx, fin = hf._update_finished_beams(seqs, tseq, beam_scores, topv, bidx, tbi, unsat, fin,
                                                                 hits, top_mask, K, t, 0, lp, es)
        unsat = hf._check_early_stop_heuristic(unsat, run_scores, beam_scores, fin, t + 1, n_new, 0, es, lp)
        steps.append(dict(tok=run_seq[:, :, t].clone(), par=(run_bi[:, :, t] - off).clone(), real=run_scores > -1e8,
                          gap=gap, active=~done))
        done = done | ~unsat[:, 0] | (fin.all(dim=1) & (es is True)) | hits.all(dim=1)
        if bool(done.all()):
            break
        logits = next_logits(run_bi[:, :, t].reshape(-1).long(), run_seq[:, :, t].reshape(-1))
    return steps, (seqs, beam_scores, bidx, fin)


def _hf_procs(eos, device=DEV):
    from transformers.generation.logits_process import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor,
                                                        NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor)
    return LogitsProcessorList([RepetitionPenaltyLogitsProcessor(penalty=1.3), NoRepeatNGramLogitsProcessor(3),
                                MinNewTokensLengthLogitsProcessor(0, 4, list(eos), device=device)])


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_beam_request_matches_hf_beam_search_on_the_engine_logits(family):
    from u2tokenizer_b200.engine import BeamSearch, GenerateRequest, LogitsProcessors, U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, head_kw = _engine_family(family)
    sd16 = synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **head_kw)
    eng = U2Engine(g, sd16, device=DEV)
    rows, images, ids, qids, _, lens = _inputs(g)
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    n_new = 20
    plain = eng.generate_greedy(emb, n_new, lengths=lens).cpu()
    eos = (int(plain[0, 6]), int(plain[1, 9]))
    V = g.vocab_size
    pc = LogitsProcessors(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4, eos_token_ids=eos)
    procs_kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)
    cases = [(4, 1.0, False, 2, None), (2, 0.0, True, 1, None), (4, 2.0, "never", 4, pc), (5, -0.5, False, 3, None)]
    compared = total = 0
    for impl in ("tcgen05", "gemv"):
        eng.decode_impl = impl
        cap = eng._decode_rows()
        for use_graph in (False, True):
            for ragged in (True, False):
                e = emb if ragged else emb[1:2, :lens[1]].contiguous()
                ln = torch.tensor(lens) if ragged else torch.tensor([lens[1]])
                for K, lp, es, n_ret, procs in cases:
                    P = e.shape[0]
                    if P * K > cap:
                        continue
                    bm = BeamSearch(num_beams=K, length_penalty=lp, early_stopping=es, num_return_sequences=n_ret,
                                    pad_token_id=eos[0])
                    lo = []
                    req = GenerateRequest(n_new, list(eos), processors=procs, beam=bm)
                    got = eng._generate(e, req, ln, use_graph, logits_out=lo)
                    want = _hf_beam(lo, P, K, V, n_new, eos, lp, es, n_ret, procs_kw if procs else {}).cpu()
                    # the same selections on the same logits wherever no step of the prompt is a near-tie: HF's
                    # log_softmax and the engine's may differ in the last bit
                    it = iter(lo[1:])
                    steps, _ = _hf_loop(lo[0], lambda par, tok: next(it), P, K, V, n_new, eos, lp, es,
                                        _hf_procs(eos) if procs else None)
                    got = got.cpu()
                    w = min(got.shape[1], want.shape[1])
                    for p in range(P):
                        total += 1
                        if min(float(s["gap"][p]) for s in steps if bool(s["active"][p])) <= 1e-4:
                            continue
                        rows = slice(p * n_ret, (p + 1) * n_ret)
                        assert torch.equal(got[rows, :w], want[rows, :w]), (impl, use_graph, ragged, K, lp, es, p)
                        assert bool((got[rows, w:] == eos[0]).all()) and bool((want[rows, w:] == eos[0]).all())
                        compared += 1
    print(f"[{family}] {compared}/{total} prompts compared (the others have a step with a gap <= 1e-4)")
    assert compared >= 0.75 * total, (compared, total)


def _oracle_beam(O, sd, g, rid, im, rq, K, n_new, eos, lp, es):
    """HF beam search (its own step helpers) over the fp32 oracle decoder, one prompt, on the CPU; the oracle's KV cache
    follows the beams as HF's reorder_cache does."""
    import torch.nn.functional as F
    with torch.no_grad():
        logits, past = O.decoder_forward(sd, O.multimodal_embeds(sd, rid, im, rq, g), g)
        past = [(k.expand(K, -1, -1, -1).contiguous(), v.expand(K, -1, -1, -1).contiguous()) for k, v in past]
        state = dict(past=past)

        def nxt(par, tok):
            pk = [(k.index_select(0, par), v.index_select(0, par)) for k, v in state["past"]]
            lg, state["past"] = O.decoder_forward(sd, F.embedding(tok[:, None], sd["model.embed_tokens.weight"]), g, pk)
            return lg[:, -1]
        return _hf_loop(logits[:, -1].expand(K, -1), nxt, 1, K, g.vocab_size, n_new, eos, lp, es, dev="cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_engine_beams_follow_hf_beam_search_over_the_oracle_decoder(family):
    """The engine's running beams (token and parent of every row at every step, read from its records) and its output
    equal HF beam search over the fp32 oracle decoder, up to the first step whose selection gap is within the numerical
    error of the engine's logits. This is what checks the decode through the KV-cache indirection."""
    from oracle import u2_oracle as O
    from u2tokenizer_b200.engine import BeamSearch, U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, head_kw = _engine_family(family)
    sd16 = synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **head_kw)
    eng = U2Engine(g, sd16, device=DEV)
    sd = {k: v.float() for k, v in sd16.items()}
    rows, images, ids, qids, _, lens = _inputs(g)
    n_new = 16
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    plain = eng.generate_greedy(emb, n_new, lengths=lens).cpu()
    eos = [int(plain[0, 6]), int(plain[2, 9])]
    thr = 0.0
    with torch.no_grad():
        for im, rid, rq in rows:
            ref = O.decoder_forward(sd, O.multimodal_embeds(sd, rid, im, rq, g), g)[0]
            lg = eng.lm_logits(eng.prefill(eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda()))).float().cpu()
            thr = max(thr, 4.0 * (lg - ref).abs().max().item())
    compared_steps = total_steps = finals = 0
    for K, lp, es, n_ret in ((2, 1.0, False, 2), (4, 2.0, "never", 3), (4, 0.0, True, 1)):
        refs = [_oracle_beam(O, sd, g, rid, im, rq, K, n_new, eos, lp, es) for im, rid, rq in rows]
        bm = BeamSearch(num_beams=K, length_penalty=lp, early_stopping=es, num_return_sequences=n_ret,
                        pad_token_id=eos[0])
        for impl in ("tcgen05", "gemv"):
            eng.decode_impl = impl
            cap = eng._decode_rows()
            for ragged in (True, False):
                sel = list(range(len(rows))) if ragged else [1]
                if len(sel) * K > cap:
                    continue
                e = emb if ragged else emb[1:2, :lens[1]].contiguous()
                got = eng.generate(e, n_new, eos_token_id=eos, lengths=lens if ragged else None, beam=bm).cpu()
                rec = eng._gen_state["beam"]["rec"].cpu()
                for p, b in enumerate(sel):
                    steps, (seqs, scores, bidx, fin) = refs[b]
                    tied = False
                    for t, st in enumerate(steps):
                        total_steps += 1
                        if float(st["gap"][0]) <= thr * (t + 1):  # the running scores carry t + 1 steps of error
                            tied = True
                            break
                        real = st["real"][0]
                        mine = rec[t, p * K:(p + 1) * K]
                        assert torch.equal(mine[real, 0].long(), st["tok"][0][real]), (family, impl, K, b, t)
                        assert torch.equal(mine[real, 1].long(), st["par"][0][real].long()), (family, impl, K, b, t)
                        compared_steps += 1
                    fs = scores[0][:n_ret + 1] if n_ret < K else scores[0][:n_ret]
                    if tied or (len(fs) > 1 and float((fs[:-1] - fs[1:]).min()) <= thr * n_new):
                        continue
                    n = int((bidx[0, :n_ret] >= 0).sum(-1).max())
                    want = seqs[0, :n_ret, :n]
                    assert torch.equal(got[p * n_ret:(p + 1) * n_ret, :n], want), (family, impl, K, b, got, want)
                    finals += 1
    print(f"[{family}] thr {thr:.3g}: {compared_steps}/{total_steps} steps and {finals} outputs identical to the oracle")
    assert compared_steps >= 1, (compared_steps, total_steps, finals, thr)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_beam_request_logits_equal_the_oracle_on_each_beams_own_history(family):
    """Teacher-forced through the indirection: the logits the engine computes for row k at step t must be the oracle
    decoder's logits for the prompt followed by row k's own history (backtracked from the engine's records). A wrong
    table entry, a table read one step stale or a wrong copy range hands a row another beam's keys / values, which moves
    its logits by far more than the bf16 error."""
    from oracle import u2_oracle as O
    from u2tokenizer_b200.engine import BeamSearch, GenerateRequest, U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    import torch.nn.functional as F
    g, head_kw = _engine_family(family)
    sd16 = synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **head_kw)
    eng = U2Engine(g, sd16, device=DEV)
    sd = {k: v.float() for k, v in sd16.items()}
    E = sd["model.embed_tokens.weight"]
    rows, images, ids, qids, _, lens = _inputs(g)
    n_new = 14
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    with torch.no_grad():
        prompts = [O.multimodal_embeds(sd, rid, im, rq, g) for im, rid, rq in rows]
        err0 = max((eng.lm_logits(eng.prefill(eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda()))).float().cpu()
                    - O.decoder_forward(sd, pe, g)[0]).abs().max().item() for (im, rid, rq), pe in zip(rows, prompts))
    tol = 4.0 * err0
    for impl in ("tcgen05", "gemv"):
        eng.decode_impl = impl
        for use_graph in (False, True):
            K = 4 if impl == "tcgen05" else 2
            bm = BeamSearch(num_beams=K, length_penalty=1.0, early_stopping="never")
            lo = []
            eng._generate(emb, GenerateRequest(n_new, beam=bm), torch.tensor(lens), use_graph, logits_out=lo)
            lo = [x.cpu() for x in lo]
            rec = eng._gen_state["beam"]["rec"].cpu()
            worst, reparented = 0.0, 0
            for t in range(1, len(lo)):
                for p in range(len(rows)):
                    hist = torch.empty(K, t, dtype=torch.long)
                    for k in range(K):
                        r = k
                        for s in range(t - 1, -1, -1):
                            hist[k, s] = rec[s, p * K + r, 0]
                            r = int(rec[s, p * K + r, 1])
                        reparented += int(rec[t - 1, p * K + k, 1]) != k
                    with torch.no_grad():
                        x = torch.cat([prompts[p].expand(K, -1, -1), F.embedding(hist, E)], dim=1)
                        ref = O.decoder_forward(sd, x, g)[0][:, -1]
                    err = (lo[t][p * K:(p + 1) * K] - ref).abs().max().item()
                    worst = max(worst, err)
                    assert err <= tol, (family, impl, use_graph, t, p, err, tol)
            print(f"[{family} {impl} graph={use_graph}] max |engine - oracle| {worst:.3g} (tol {tol:.3g}) over "
                  f"{len(lo) - 1} steps, {reparented} rows continued another beam")
            assert reparented > 0  # the indirection was exercised


@pytest.mark.gpu
def test_each_prompt_of_a_ragged_batch_equals_the_prompt_alone_across_chunks():
    # 5 prompts x 4 beams: 4 prompts fill the first 16-row chunk, the fifth runs in a second one
    from u2tokenizer_b200.engine import BeamSearch, U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, head_kw = _engine_family("qwen3")
    eng = U2Engine(g, synthetic_state_dict(g, seed=5, device="cpu", dtype=torch.bfloat16, **head_kw), device=DEV)
    rows, images, ids, qids, _, lens = _inputs(g, qlens=(6, 2, 11, 4, 9))
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    plain = eng.generate_greedy(emb, 16, lengths=lens).cpu()
    eos = [int(plain[0, 5]), int(plain[3, 8])]
    bm = BeamSearch(num_beams=4, length_penalty=1.0, early_stopping=False, num_return_sequences=2, pad_token_id=eos[0])
    got = eng.generate(emb, 16, eos_token_id=eos, lengths=lens, beam=bm).cpu()
    scores = eng.last_beam_scores.clone()
    assert got.shape[0] == 10
    for b in range(5):
        alone = eng.generate(emb[b:b + 1, :lens[b]].contiguous(), 16, eos_token_id=eos, beam=bm).cpu()
        w = alone.shape[1]
        assert torch.equal(got[2 * b:2 * b + 2, :w], alone), b
        assert bool((got[2 * b:2 * b + 2, w:] == eos[0]).all()), b
        assert torch.equal(scores[2 * b:2 * b + 2], eng.last_beam_scores), b


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
    model.load_state_dict(synthetic_state_dict(g, seed=9, device="cpu", dtype=torch.bfloat16, bigram=1.0), strict=False)
    model = model.to(torch.bfloat16).cuda().eval()
    model.generation_config.eos_token_id = None
    return model, g


@pytest.mark.gpu
def test_greedy_beam_greedy_keeps_greedy_bit_identical_with_the_same_launches():
    from u2tokenizer_b200 import _lib
    model, g = _make_model()
    rows, images, ids, qids, mask, lens = _inputs(g)
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=12)
    args = (images.cuda(), ids.cuda())
    model.generate(*args, **kw)
    n0 = _lib.launches()
    a = model.generate(*args, **kw).cpu()
    n1 = _lib.launches()
    beams = model.generate(*args, num_beams=4, num_return_sequences=2, eos_token_id=int(a[0, 3]), **kw).cpu()
    assert beams.shape[0] == 6
    model.generate(*args, **kw)
    n2 = _lib.launches()
    b = model.generate(*args, **kw).cpu()
    n3 = _lib.launches()
    fresh, _ = _make_model()
    assert torch.equal(a, b) and torch.equal(a, fresh.generate(*args, **kw).cpu())
    assert n3 - n2 == n1 - n0


@pytest.mark.gpu
def test_generation_config_num_beams_is_honoured():
    model, g = _make_model()
    rows, images, ids, qids, mask, lens = _inputs(g)
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=10)
    args = (images.cuda(), ids.cuda())
    explicit = model.generate(*args, num_beams=3, length_penalty=0.0, **kw).cpu()
    model.generation_config.num_beams = 3
    model.generation_config.length_penalty = 0.0
    assert torch.equal(model.generate(*args, **kw).cpu(), explicit)
    with pytest.raises(ValueError):
        model.generate(*args, num_beams=17, **kw)
