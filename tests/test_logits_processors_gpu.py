"""generate()'s repetition_penalty, no_repeat_ngram_size, bad_words_ids and min_new_tokens / min_length: one kernel
rewrites every step's fp32 logits in place before the argmax or the sampler, from a device-side history of the generated
tokens, inside the captured decode step. The target is HF generate(inputs_embeds=...): the processors see the generated
tokens only, in _get_logits_processor's order."""
import pytest
import torch

from common import tiny_geometry

DEV = "cuda"


def _helper(kwargs, gc=None, L=10, eos=None, V=1000):
    from u2tokenizer_b200.modeling import U2MetaForCausalLM
    kw = dict(kwargs)
    out = U2MetaForCausalLM._generate_logits_processors(kw, gc, L, eos, V)
    for k in ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens", "min_length", "bad_words_ids"):
        assert k not in kw
    return out


def _hf_processors(pc, device=DEV):
    """HF's LogitsProcessorList for an engine.LogitsProcessors, in _get_logits_processor's order (CUDA tensors)."""
    from transformers.generation.logits_process import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor,
                                                        NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor)
    procs = LogitsProcessorList()
    if pc.repetition_penalty != 1.0:
        procs.append(RepetitionPenaltyLogitsProcessor(penalty=float(pc.repetition_penalty)))
    if pc.no_repeat_ngram_size > 0:
        procs.append(NoRepeatNGramLogitsProcessor(pc.no_repeat_ngram_size))
    if pc.bad_words_ids:
        procs.append(NoBadWordsLogitsProcessor([list(w) for w in pc.bad_words_ids],
                                               list(pc.eos_token_ids) if pc.eos_token_ids else None))
    if pc.min_new_tokens > 0 and pc.eos_token_ids:
        procs.append(MinNewTokensLengthLogitsProcessor(0, pc.min_new_tokens, list(pc.eos_token_ids), device=device))
    return procs


# ------------------------------------------------------------------------------------------------
# surface helper (CPU)
# ------------------------------------------------------------------------------------------------
def test_helper_is_none_for_absent_or_neutral_values():
    from transformers import GenerationConfig
    assert _helper({}) is None
    assert _helper({}, GenerationConfig()) is None
    neutral = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, min_length=0, bad_words_ids=None)
    assert _helper(neutral, eos=7) is None
    # min_new_tokens / min_length with no EOS id ban nothing; min_length within the prompt width asks for no new token
    assert _helper(dict(min_new_tokens=5)) is None
    assert _helper(dict(min_length=8), L=10, eos=7) is None


def test_helper_reads_generation_config_and_maps_min_length():
    from transformers import GenerationConfig
    gc = GenerationConfig(repetition_penalty=1.3, no_repeat_ngram_size=3, bad_words_ids=[[5], [6, 7]], min_length=25)
    pc = _helper({}, gc, L=10, eos=[2, 3])
    assert pc.repetition_penalty == 1.3 and pc.no_repeat_ngram_size == 3
    assert pc.bad_words_ids == ((5,), (6, 7))
    assert pc.min_new_tokens == 15 and pc.eos_token_ids == (2, 3)  # min_length counts from the padded prompt width
    # kwargs win over the generation config, min_new_tokens over min_length
    pc = _helper(dict(repetition_penalty=2.0, min_new_tokens=4), gc, L=10, eos=2)
    assert pc.repetition_penalty == 2.0 and pc.min_new_tokens == 4 and pc.eos_token_ids == (2,)
    pc = _helper(dict(min_new_tokens=0, min_length=30), L=10, eos=2)
    assert pc is None
    # one-token bad words equal to an EOS id are dropped (NoBadWordsLogitsProcessor); EOS ids outside the vocabulary
    # can never be picked and are not sent to the kernel
    pc = _helper(dict(bad_words_ids=[[2], [4], [2, 9]], min_new_tokens=3), eos=[2, 5000], V=1000)
    assert pc.bad_words_ids == ((4,), (2, 9)) and pc.eos_token_ids == (2,)
    pc = _helper(dict(min_new_tokens=3), eos=torch.tensor([11, 12]))
    assert pc.eos_token_ids == (11, 12)


@pytest.mark.parametrize("kwargs", [
    dict(repetition_penalty=0.0), dict(repetition_penalty=-1.2), dict(repetition_penalty="1.2"),
    dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=2.0), dict(no_repeat_ngram_size=True),
    dict(min_new_tokens=-1), dict(min_new_tokens=1.5), dict(min_length=-3),
    dict(bad_words_ids=[]), dict(bad_words_ids=[5]), dict(bad_words_ids=[[5], (6,)]), dict(bad_words_ids=[[-1]]),
    dict(bad_words_ids=[[1.0]]), dict(bad_words_ids=[[]]), dict(bad_words_ids=[[3, 1000]]), dict(bad_words_ids=[[7]]),
    dict(bad_words_ids=[[i] for i in range(300)]), dict(bad_words_ids=[[i] * 10 for i in range(1, 250)]),
])
def test_helper_refuses_bad_values(kwargs):
    # [[7]] with EOS 7: nothing is left after the EOS filter, as HF refuses it
    with pytest.raises(ValueError):
        _helper(kwargs, eos=7, V=1000)


@pytest.mark.parametrize("name,value", [("typical_p", 0.9), ("encoder_repetition_penalty", 1.2),
                                        ("suppress_tokens", [3]), ("logits_processor", [object()]),
                                        ("epsilon_cutoff", 3e-4), ("min_p", 0.1),
                                        ("force_words_ids", [[3]]), ("begin_suppress_tokens", [1])])
def test_other_options_still_refused(name, value):
    from u2tokenizer_b200.modeling import U2MetaForCausalLM
    with pytest.raises(NotImplementedError, match=name):
        U2MetaForCausalLM._check_remaining_generate_kwargs({name: value})
    U2MetaForCausalLM._check_remaining_generate_kwargs({"use_cache": True, "typical_p": 1.0})


def test_hf_reference_on_cpu_matches_the_documented_semantics():
    """The reference these tests compare against, on one hand-checked case."""
    from u2tokenizer_b200.engine import LogitsProcessors
    pc = LogitsProcessors(repetition_penalty=2.0, no_repeat_ngram_size=2, min_new_tokens=5, eos_token_ids=(9,),
                          bad_words_ids=((8,), (1, 4)))
    hist = torch.tensor([[1, 2, 1, 2, 3, 1]])
    x = torch.full((1, 10), 3.0)
    x[0, 2] = -3.0
    y = _hf_processors(pc, "cpu")(hist, x.clone())
    # penalised once: 1, 2, 3; banned: 2 (after "1"), 8, 4 ("1" ends the history), EOS 9 (6 < 5 is false: allowed)
    want = torch.tensor([[3.0, 1.5, -float("inf"), 1.5, -float("inf"), 3, 3, 3, -float("inf"), 3]])
    assert torch.equal(y, want)


# ------------------------------------------------------------------------------------------------
# op: the kernel against HF's processors on CUDA, bit for bit
# ------------------------------------------------------------------------------------------------
def _case(B, V, T, seed, n):
    g = torch.Generator(device="cpu").manual_seed(seed)
    logits = (torch.randn(B, V, generator=g) * 4).to(DEV)
    # small alphabets: many duplicates and repeated n-grams
    hist = torch.stack([torch.randint(0, 6 if b % 2 == 0 else min(V, 64), (T,), generator=g) for b in range(B)])
    tail = hist[0, max(0, T - 2):].tolist() if T else []
    bad = [[int(torch.randint(3, V - 1, (1,), generator=g))], [3], [5, 7, 1]]  # no one-token word is an EOS id
    if len(tail) == 2:
        bad += [tail + [11], tail[-1:] + [12]]  # prefixes that end row 0's history
    eos = (V - 1, 2)
    return logits, hist.to(DEV), bad, eos


def _process(logits, hist_full, t, pc, cap=None, step_dev=None):
    from u2tokenizer_b200 import ops
    B, V = logits.shape
    cap = cap or max(t, 1) + 3
    hist = torch.full((B, cap), -7, device=DEV, dtype=torch.int32)
    if t > 1:
        hist[:, :t - 1] = hist_full[:, :t - 1].int()
    ids = hist_full[:, t - 1].clone() if t > 0 else torch.zeros(B, device=DEV, dtype=torch.int64)
    blk = ops.logits_proc_params(DEV, V, repetition_penalty=pc.repetition_penalty,
                                 no_repeat_ngram_size=pc.no_repeat_ngram_size, min_new_tokens=pc.min_new_tokens,
                                 eos_token_ids=pc.eos_token_ids, bad_words_ids=pc.bad_words_ids)
    out = logits.clone()
    ops.logits_process(out, blk, ids, hist, step=t)
    if t > 0:
        assert torch.equal(hist[:, :t].long(), hist_full[:, :t])  # the fed token was appended
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("V", [151936, 1000])
@pytest.mark.parametrize("B", [1, 4, 16])
@pytest.mark.parametrize("penalty,n", [(0.7, 2), (1.3, 3), (2.0, 4)])
def test_kernel_matches_hf_bitwise(V, B, penalty, n):
    from u2tokenizer_b200.engine import LogitsProcessors
    for T in (0, 1, n - 1, n, 800):
        logits, hist, bad, eos = _case(B, V, T, seed=V + B + T + n, n=n)
        pc = LogitsProcessors(repetition_penalty=penalty, no_repeat_ngram_size=n, min_new_tokens=n + 1,
                              eos_token_ids=eos, bad_words_ids=tuple(tuple(w) for w in bad))
        got = _process(logits, hist, T, pc)
        want = _hf_processors(pc)(hist[:, :T], logits.clone())
        assert torch.equal(got, want), (V, B, T, (got != want).nonzero()[:8].tolist())
        assert not torch.equal(got, logits)


@pytest.mark.gpu
def test_kernel_each_processor_alone_matches_hf():
    from u2tokenizer_b200.engine import LogitsProcessors
    logits, hist, bad, eos = _case(4, 151936, 300, seed=1, n=3)
    for pc in (LogitsProcessors(repetition_penalty=1.2), LogitsProcessors(no_repeat_ngram_size=1),
               LogitsProcessors(bad_words_ids=tuple(tuple(w) for w in bad)),
               LogitsProcessors(min_new_tokens=301, eos_token_ids=eos)):
        got = _process(logits, hist, 300, pc)
        assert torch.equal(got, _hf_processors(pc)(hist, logits.clone())), pc


@pytest.mark.gpu
def test_kernel_history_built_step_by_step_through_step_dev():
    from u2tokenizer_b200 import ops
    from u2tokenizer_b200.engine import LogitsProcessors
    B, V, T = 4, 151936, 40
    logits, hist_full, bad, eos = _case(B, V, T, seed=2, n=3)
    pc = LogitsProcessors(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=20, eos_token_ids=eos,
                          bad_words_ids=tuple(tuple(w) for w in bad))
    blk = ops.logits_proc_params(DEV, V, repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=20,
                                 eos_token_ids=eos, bad_words_ids=pc.bad_words_ids)
    hist = torch.zeros(B, T + 4, device=DEV, dtype=torch.int32)
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    ids = torch.zeros(B, device=DEV, dtype=torch.int64)
    for t in range(T + 1):
        step.fill_(t)
        if t > 0:
            ids.copy_(hist_full[:, t - 1])
        out = logits.clone()
        ops.logits_process(out, blk, ids, hist, step_dev=step)
        assert torch.equal(out, _process(logits, hist_full, t, pc)), t
    assert torch.equal(hist[:, :T].long(), hist_full)


@pytest.mark.gpu
def test_captured_kernel_reads_an_overwritten_parameter_block():
    from u2tokenizer_b200 import ops
    from u2tokenizer_b200.engine import LogitsProcessors
    B, V, T = 4, 151936, 60
    logits, hist_full, bad, eos = _case(B, V, T, seed=3, n=2)
    blk = ops.logits_proc_params(DEV, V, repetition_penalty=0.7, no_repeat_ngram_size=2)
    hist = torch.zeros(B, T + 4, device=DEV, dtype=torch.int32)
    hist[:, :T - 1] = hist_full[:, :T - 1].int()
    step = torch.full((1,), T, device=DEV, dtype=torch.int32)
    ids = hist_full[:, T - 1].clone()
    buf = logits.clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.logits_process(buf, blk, ids, hist, step_dev=step)
    pc = LogitsProcessors(repetition_penalty=2.0, no_repeat_ngram_size=4, min_new_tokens=T + 1, eos_token_ids=eos,
                          bad_words_ids=tuple(tuple(w) for w in bad))
    ops.logits_proc_params(DEV, V, repetition_penalty=2.0, no_repeat_ngram_size=4, min_new_tokens=T + 1,
                           eos_token_ids=eos, bad_words_ids=pc.bad_words_ids, out=blk)
    buf.copy_(logits)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(buf, _process(logits, hist_full, T, pc))


# ------------------------------------------------------------------------------------------------
# engine: teacher-forced parity with HF's processors, oracle agreement, constraints hold
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


def _ngram_repeats(row, n):
    seen = set()
    for i in range(len(row) - n + 1):
        gram = tuple(row[i:i + n])
        if gram in seen:
            return True
        seen.add(gram)
    return False


def _contains(row, word):
    return any(tuple(row[i:i + len(word)]) == tuple(word) for i in range(len(row) - len(word) + 1))


def _config_from_plain(plain, n_new):
    """Processors built from what the plain run emits, so that each one has something to do."""
    from u2tokenizer_b200.engine import LogitsProcessors
    r0 = plain[0].tolist()
    eos = (r0[1], r0[3]) if r0[1] != r0[3] else (r0[1], (r0[1] + 1) % 97)
    words = [w for w in ((r0[5],), (r0[6], r0[7])) if not (len(w) == 1 and w[0] in eos)]
    return LogitsProcessors(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=n_new // 2,
                            eos_token_ids=eos, bad_words_ids=tuple(words))


def _check_constraints(ids, pc, n_new):
    for row in ids.tolist():
        assert not _ngram_repeats(row, pc.no_repeat_ngram_size), row
        for w in pc.bad_words_ids:
            assert not _contains(row, w), (row, w)
        assert not any(x in pc.eos_token_ids for x in row[:pc.min_new_tokens]), row


def _oracle_with_processors(O, sd, rid, im, rq, g, n_new, procs):
    """oracle.greedy_generate with HF's processors applied to the fp32 logits, from the ids generated so far; the
    margins are taken after processing."""
    import torch.nn.functional as F
    emb = O.multimodal_embeds(sd, rid, im, rq, g)
    logits, past = O.decoder_forward(sd, emb, g)
    out, margins = torch.zeros(1, 0, dtype=torch.long), []
    for _ in range(n_new):
        last = procs(out, logits[:, -1].float().clone())
        top2 = last.topk(2, dim=-1).values
        margins.append(top2[:, 0] - top2[:, 1])
        nxt = last.argmax(-1)
        out = torch.cat([out, nxt[:, None]], dim=1)
        logits, past = O.decoder_forward(sd, F.embedding(nxt[:, None], sd["model.embed_tokens.weight"]), g, past)
    return out, torch.stack(margins, dim=1)


def _upto(margins_row, thr, n):
    low = (margins_row[:n] < thr).nonzero()
    return int(low[0]) if len(low) else n


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_engine_processed_logits_match_hf_teacher_forced(family):
    from oracle import u2_oracle as O
    from u2tokenizer_b200.engine import U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, head_kw = _engine_family(family)
    sd16 = synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **head_kw)
    eng = U2Engine(g, sd16, device=DEV)
    sd = {k: v.float() for k, v in sd16.items()}
    rows, images, ids, qids, _, lens = _inputs(g)
    n_new = 24
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    plain = eng.generate_greedy(emb, n_new, lengths=lens).cpu()
    pc = _config_from_plain(plain, n_new)
    hf = _hf_processors(pc)
    # margin-aware agreement with the oracle (fp32 weights on the CPU) per row
    refs, thr = [], 0.0
    cpu_procs = _hf_processors(pc, "cpu")
    for im, rid, rq in rows:
        with torch.no_grad():
            ref_logits = O.decoder_forward(sd, O.multimodal_embeds(sd, rid, im, rq, g), g)[0]
            refs.append(_oracle_with_processors(O, sd, rid, im, rq, g, n_new, cpu_procs))
        lg = eng.lm_logits(eng.prefill(eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda()))).float().cpu()
        thr = max(thr, 4.0 * (lg - ref_logits).abs().max().item())
    for impl in ("tcgen05", "gemv"):
        eng.decode_impl = impl
        for use_graph in (False, True):
            for lengths, sel in ((lens, slice(None)), (None, slice(1, 2))):  # ragged rows, then one uniform row
                e = emb if lengths is not None else emb[sel, :lens[1]].contiguous()
                lo, raw = [], []
                got = eng.generate_greedy(e, n_new, use_graph=use_graph, lengths=lengths, processors=pc,
                                          logits_out=lo)
                eng.generate_greedy(e, n_new, use_graph=use_graph, lengths=lengths, force_ids=got, logits_out=raw)
                for t in range(n_new):
                    want = hf(got[:, :t], raw[t].clone())
                    assert torch.equal(lo[t], want), (impl, use_graph, t, (lo[t] != want).nonzero()[:6].tolist())
                    picked = lo[t].gather(1, got[:, t:t + 1]).squeeze(1)
                    assert torch.equal(picked, lo[t].max(dim=1).values), (impl, use_graph, t)
                got = got.cpu()
                _check_constraints(got, pc, n_new)
                if lengths is None:
                    continue
                assert not torch.equal(got, plain), "the processors changed nothing"
                compared = 0
                for b, (ref_ids, margins) in enumerate(refs):
                    upto = _upto(margins[0], thr, n_new)
                    compared += upto
                    assert torch.equal(got[b, :upto], ref_ids[0, :upto]), (impl, use_graph, b, got[b], ref_ids[0])
                print(f"[{family} {impl} graph={use_graph}] identical to the oracle on {compared}/{got.numel()} "
                      f"compared tokens")
                if family == "qwen3":
                    assert compared >= 0.75 * got.numel(), (compared, thr)


# ------------------------------------------------------------------------------------------------
# surface: model.generate(..., repetition_penalty=..., ...)
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
    return model, g


def _hf_kwargs(pc):
    return dict(repetition_penalty=pc.repetition_penalty, no_repeat_ngram_size=pc.no_repeat_ngram_size,
                min_new_tokens=pc.min_new_tokens, bad_words_ids=[list(w) for w in pc.bad_words_ids])


@pytest.mark.gpu
def test_sampled_ragged_rows_across_the_chunk_boundary_keep_every_constraint():
    model, g = _make_model()
    rows, images, ids, qids, mask, lens = _inputs(g, qlens=(6, 11))
    args = (images.cuda(), ids.cuda())
    n_new = 16
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=n_new)
    plain = model.generate(*args, do_sample=False, **kw).cpu()
    pc = _config_from_plain(plain, n_new)
    eos = list(pc.eos_token_ids)
    skw = dict(do_sample=True, num_return_sequences=9, seed=3, eos_token_id=eos, pad_token_id=-1, **_hf_kwargs(pc), **kw)
    out = model.generate(*args, **skw).cpu()
    assert out.shape[0] == 18  # 2 prompts x 9 samples = 16 + 2 rows
    assert out.shape[1] > pc.min_new_tokens
    for row in out.tolist():
        hit = [i for i, x in enumerate(row) if x in eos]
        row = row[:hit[0] + 1] if hit else row
        assert -1 not in row and (not hit or hit[0] >= pc.min_new_tokens), row
        assert not _ngram_repeats(row, pc.no_repeat_ngram_size), row
        assert not any(_contains(row, w) for w in pc.bad_words_ids), row
    assert torch.equal(model.generate(*args, **skw).cpu(), out)


@pytest.mark.gpu
def test_neutral_values_are_bit_identical_with_the_same_launches():
    from u2tokenizer_b200 import _lib
    model, g = _make_model()
    rows, images, ids, qids, mask, lens = _inputs(g)
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=12, do_sample=False)
    args = (images.cuda(), ids.cuda())
    model.generate(*args, **kw)
    n0 = _lib.launches()
    a = model.generate(*args, **kw).cpu()
    n1 = _lib.launches()
    b = model.generate(*args, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, min_length=0,
                       bad_words_ids=None, **kw).cpu()
    n2 = _lib.launches()
    assert torch.equal(a, b)
    assert n2 - n1 == n1 - n0


@pytest.mark.gpu
def test_processors_on_off_on_match_fresh_models():
    model, g = _make_model()
    rows, images, ids, qids, mask, lens = _inputs(g)
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=14, do_sample=False)
    args = (images.cuda(), ids.cuda())
    plain = model.generate(*args, **kw).cpu()
    r0 = plain[0].tolist()
    calls = [dict(repetition_penalty=1.5, no_repeat_ngram_size=2, bad_words_ids=[[r0[2]]]),
             dict(),
             dict(repetition_penalty=0.8, no_repeat_ngram_size=4, min_new_tokens=6, eos_token_id=r0[1],
                  bad_words_ids=[[r0[3], r0[4]]]),
             dict(repetition_penalty=1.5, no_repeat_ngram_size=2, bad_words_ids=[[r0[2]]])]
    got = [model.generate(*args, **c, **kw).cpu() for c in calls]
    for c, out in zip(calls, got):
        fresh, _ = _make_model()
        assert torch.equal(out, fresh.generate(*args, **c, **kw).cpu()), c
    assert torch.equal(got[1], plain) and not torch.equal(got[0], plain) and torch.equal(got[0], got[3])
