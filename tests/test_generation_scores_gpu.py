"""Generation scores on the GPU: the step-indexed row store, the sampler with outputs, the greedy and slot log-probs
against torch; generate(return_dict_in_generate, output_scores, output_logits) against HF generate() replaying the
engine's own logits (Qwen3 and Llama, both decode paths, eager and graphed), compute_transition_scores, chunks and
ragged prompts against each prompt alone, generate_batch(return_logprobs) against generate() alone, and that nothing
changes when the options are off."""
import pytest
import torch

from common import tiny_geometry

DEV = "cuda"
pytestmark = pytest.mark.gpu

# a token whose ascending cumulative probability lies this close to HF's nucleus boundary (1 - top_p) may fall on
# either side of it: the sampler bisects on the scaled logit with __expf sums, HF sorts and sums in torch
NUCLEUS_TOL = 1e-4


def _inv_t(temperature):
    return torch.tensor(1.0, dtype=torch.float32) / torch.tensor(temperature, dtype=torch.float32)


def _hf_kept(x: torch.Tensor, top_k: int, top_p: float):
    """HF's TopKLogitsWarper + TopPLogitsWarper keep mask on scaled logits x [B, V], and the tokens whose ascending
    cumulative probability lies within NUCLEUS_TOL of the nucleus boundary."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    s = x.clone()
    if top_k > 0:
        s = TopKLogitsWarper(top_k)(None, s)
    near = torch.zeros_like(s, dtype=torch.bool)
    if top_p < 1.0:
        srt, idx = torch.sort(s, descending=False)
        cum = srt.softmax(dim=-1).cumsum(dim=-1)
        near.scatter_(1, idx, (cum - (1 - top_p)).abs() < NUCLEUS_TOL)
        s = TopPLogitsWarper(top_p)(None, s)
    return s > -float("inf"), near


# ------------------------------------------------------------------------------------------------
# kernels against torch
# ------------------------------------------------------------------------------------------------
def test_sampler_with_outputs_draws_the_same_ids_and_writes_the_warped_row():
    from u2tokenizer_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(7)
    V, steps = 5003, 3
    boundary = total = 0
    for B in (1, 3, 16):
        logits = torch.randn(B, V, device=DEV, generator=g) * 3
        for temp, k, p in ((1.0, 50, 1.0), (0.7, 0, 0.9), (1.3, 20, 0.8), (0.9, 0, 1.0)):
            for seed in (0, 12345, 2 ** 63 + 11):
                blk = ops.sample_params(DEV, temp, k, p, seed)
                buf = torch.full((steps, B, V), 7.0, device=DEV)
                store = ops.row_store_params(DEV, **ops.row_store_dst(buf))
                for step in range(steps):
                    want = ops.sample_dev(logits, blk, step=step)
                    lp = torch.empty(B, device=DEV)
                    got = ops.sample_out(logits, blk, torch.empty(B, device=DEV, dtype=torch.int64), scores=store,
                                         logprob=lp, step=step)
                    assert torch.equal(got, want), (B, temp, k, p, seed, step)
                    sc = buf[step]
                    x = logits * _inv_t(temp).to(DEV)
                    kept = sc > -float("inf")
                    assert torch.equal(sc[kept], x[kept])
                    assert bool(kept.gather(1, got[:, None]).all())
                    hf, near = _hf_kept(x, k, p)
                    diff = kept != hf
                    assert not bool((diff & ~near).any()), (B, temp, k, p, seed)
                    boundary += int(diff.sum())
                    total += int(hf.sum())
                    ref = torch.log_softmax(sc, dim=-1).gather(1, got[:, None])[:, 0]
                    assert (lp - ref).abs().max().item() < 2e-5
    print(f"kept sets: {boundary} of {total} HF-kept tokens differ, all within {NUCLEUS_TOL} of the nucleus boundary")


def test_sampler_with_outputs_on_slots_is_the_slot_sampler():
    from u2tokenizer_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(2)
    B, V = 6, 3001
    logits = torch.randn(B, V, device=DEV, generator=g) * 3
    slots = ops.slot_state([11, 2 ** 63 + 5, 11, 0, 77, 5], [0, 1, 2, 5, 0, 3], [1000] * B, [0, 4, 9, 1, 300, 2]).to(DEV)
    blk = ops.sample_params(DEV, 0.8, 30, 0.9, 999)
    lp = torch.empty(B, device=DEV)
    got = ops.sample_out(logits, blk, torch.empty(B, device=DEV, dtype=torch.int64), logprob=lp, slots=slots)
    assert torch.equal(got, ops.sample_slots(logits, blk, slots))
    buf = torch.zeros(301, B, V, device=DEV)  # a slot's scores row goes to its own step, the slot's count
    for b, c in enumerate([0, 4, 9, 1, 300, 2]):
        ops.sample_out(logits[b:b + 1], blk, torch.empty(1, device=DEV, dtype=torch.int64),
                       scores=ops.row_store_params(DEV, **ops.row_store_dst(buf[:, b:b + 1])), slots=slots[b:b + 1])
        assert int((buf[:, b].abs().sum(-1) > 0).sum()) == 1
        sc = buf[c, b]
        assert abs(torch.log_softmax(sc, -1)[got[b]].item() - lp[b].item()) < 2e-5, (b, c)


def test_pick_logprob_matches_torch():
    from u2tokenizer_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(3)
    for B, V in ((1, 100), (5, 151936), (16, 3001)):
        logits = torch.randn(B, V, device=DEV, generator=g) * 4
        logits[:, ::7] = -float("inf")  # processors leave -inf entries
        ids = torch.randint(0, V, (B,), device=DEV, generator=g)
        ids[0] = logits[0].argmax()
        got = ops.pick_logprob(logits, ids)
        ref = torch.log_softmax(logits, -1).gather(1, ids[:, None])[:, 0]
        fin = ref > -float("inf")
        assert (got[fin] - ref[fin]).abs().max().item() < 2e-5
        assert bool((got[~fin] == -float("inf")).all())


def test_row_store_writes_the_device_step_and_skips_steps_outside():
    from u2tokenizer_b200 import ops
    src = torch.randn(3, 777, device=DEV)
    buf = torch.zeros(4, 5, 777, device=DEV)
    blk = ops.row_store_params(DEV, **ops.row_store_dst(buf[:, 1:4]))
    step = torch.tensor([2], device=DEV, dtype=torch.int32)
    ops.store_rows(src, blk, step_dev=step)
    ops.store_rows(src * 2, blk, step=0)
    ops.store_rows(src * 3, blk, step=4)  # outside [0, steps): not stored
    want = torch.zeros_like(buf)
    want[2, 1:4], want[0, 1:4] = src, src * 2
    assert torch.equal(buf, want)


def test_slot_update_with_logprobs_is_slot_update_plus_the_logprob_column():
    from u2tokenizer_b200 import ops
    B, W = 7, 6
    params = ops.slot_params(DEV, 3, (7,))
    slots = ops.slot_state([0] * B, range(B), [2, 6, 6, 1, 6, 6, 6], [1, 0, 5, 0, 2, 3, 0], [0, 0, 0, 0, 1, 0, 0])
    ids = torch.tensor([5, 7, 9, 4, 8, 6, 2], device=DEV)
    a_ids, b_ids = ids.clone(), ids.clone()
    a_sl, b_sl = slots.to(DEV), slots.to(DEV)
    a_out, b_out = torch.zeros(B, W, device=DEV, dtype=torch.int64), torch.zeros(B, W, device=DEV, dtype=torch.int64)
    lp_step = torch.arange(B, device=DEV, dtype=torch.float32) - 10
    lp = torch.full((B, W), 0.5, device=DEV)
    ops.slot_update(a_ids, a_sl, a_out, params)
    ops.slot_update(b_ids, b_sl, b_out, params, lp=(lp_step, lp))
    assert torch.equal(a_ids, b_ids) and torch.equal(a_sl, b_sl) and torch.equal(a_out, b_out)
    want = torch.full((B, W), 0.5)
    for b, (c, d) in enumerate(zip([1, 0, 5, 0, 2, 3, 0], [0, 0, 0, 0, 1, 0, 0])):
        if not d:
            want[b, c] = lp_step[b].item()
    assert torch.equal(lp.cpu(), want)


# ------------------------------------------------------------------------------------------------
# generate() against HF generate() replaying the engine's raw logits
# ------------------------------------------------------------------------------------------------
def _family(family):
    if family == "qwen3":
        return tiny_geometry(), dict(bigram=1.0)
    rs = dict(factor=8.0, high_freq_factor=4.0, low_freq_factor=1.0, original_max_position_embeddings=16,
              rope_type="llama3")
    return (tiny_geometry(qk_norm=False, rope_theta=500000.0, rope_scaling=rs, tie_word_embeddings=True),
            dict(head_tail=1.0))


def _inputs(g, qlens=(6, 2, 11)):
    from u2tokenizer_b200.synthetic import synthetic_inputs
    rows = [synthetic_inputs(g, batch=1, frames=2, n_question=n, lt=12, seed=100 + i) for i, n in enumerate(qlens)]
    lens = [r[1].shape[1] for r in rows]
    ids = torch.zeros(len(rows), max(lens), dtype=torch.long)
    for b, (_, rid, _) in enumerate(rows):
        ids[b, :lens[b]] = rid[0]
    return torch.cat([r[0] for r in rows]), ids, torch.cat([r[2] for r in rows]), lens


@pytest.fixture(scope="module", params=["qwen3", "llama"])
def fam(request):
    from u2tokenizer_b200.engine import U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, kw = _family(request.param)
    eng = U2Engine(g, synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **kw), device=DEV)
    images, ids, qids, lens = _inputs(g)
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    plain = eng.generate_greedy(emb, 20, lengths=lens).cpu()
    eos = (int(plain[0, 6]), int(plain[1, 9]))
    return eng, g, emb, lens, eos


def _replay_model(V, steps):
    """A PreTrainedModel whose forward returns the recorded raw logits of step i at its i-th call."""
    from transformers import GenerationMixin, PretrainedConfig, PreTrainedModel
    from transformers.modeling_outputs import CausalLMOutputWithPast

    class Cfg(PretrainedConfig):
        model_type = "u2_scores_replay"

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


def _hf(raw, rows, n_new, eos, **kw):
    m = _replay_model(raw.shape[-1], list(raw))
    with torch.no_grad():
        out = m.generate(inputs_embeds=torch.zeros(rows, 1, 8, device=DEV), max_new_tokens=n_new,
                         eos_token_id=list(eos), pad_token_id=eos[0], use_cache=False, return_dict_in_generate=True,
                         output_scores=True, output_logits=True, **kw)
    return m, out


def _upto_eos(row, eos):
    row = [int(x) for x in row]
    for i, t in enumerate(row):
        if t in eos:
            return i + 1
    return len(row)


PROCS = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4)


@pytest.mark.parametrize("impl", ["tcgen05", "gemv"])
@pytest.mark.parametrize("use_graph", [False, True])
def test_greedy_scores_and_logits_equal_hf_on_the_engine_logits(fam, impl, use_graph):
    from u2tokenizer_b200.engine import GenerateRequest, LogitsProcessors
    eng, g, emb, lens, eos = fam
    eng.decode_impl = impl
    n_new = 20
    for procs in (None, LogitsProcessors(eos_token_ids=eos, **PROCS)):
        lo = []
        req = GenerateRequest(n_new, eos, processors=procs, output_scores=True, output_logits=True)
        ids, scores, logits = eng._generate(emb, req, torch.tensor(lens), use_graph, logits_out=lo)
        # the device store equals the host-side clones of the same steps (logits_out holds the processed logits)
        T = len(lo)
        for t in range(T):
            assert torch.equal(scores[t], lo[t]), t
        assert bool((scores[T:] == 0).all()) and bool((logits[T:] == 0).all())
        if procs is None:
            assert torch.equal(scores[:T], logits[:T])
        m, hf = _hf(logits[:T], len(lens), n_new, eos, **(PROCS if procs else {}))
        ids = ids.cpu()
        for r in range(len(lens)):
            w = _upto_eos(ids[r], eos)
            assert torch.equal(ids[r, :w], hf.sequences[r, :w].cpu()), (r, procs)
            for t in range(w):
                assert torch.equal(hf.logits[t][r], logits[t, r]), (r, t)
                assert torch.equal(hf.scores[t][r], scores[t, r]), (r, t, procs)
        for norm in (False, True):
            mine = m.compute_transition_scores(ids.to(DEV), tuple(scores[:ids.shape[1]]), normalize_logits=norm)
            theirs = m.compute_transition_scores(hf.sequences, hf.scores, normalize_logits=norm)
            for r in range(len(lens)):
                w = _upto_eos(ids[r], eos)
                assert torch.allclose(mine[r, :w], theirs[r, :w], atol=1e-5), (r, norm)


@pytest.mark.parametrize("impl", ["tcgen05", "gemv"])
def test_beam_scores_sequences_scores_and_beam_indices_match_hf(fam, impl):
    from u2tokenizer_b200.engine import BeamSearch, GenerateRequest
    eng, g, emb, lens, eos = fam
    eng.decode_impl = impl
    n_new, K = 20, 4
    bm = BeamSearch(num_beams=K, length_penalty=1.0, early_stopping=False, num_return_sequences=2, pad_token_id=eos[0])
    compared = 0
    for b, use_graph in ((0, False), (1, True), (2, True)):
        e, ln = emb[b:b + 1, :lens[b]].contiguous(), torch.tensor([lens[b]])
        lo = []
        req = GenerateRequest(n_new, eos, beam=bm, output_scores=True, output_logits=True)
        ids, scores, logits = eng._generate(e, req, ln, use_graph, logits_out=lo)
        T = len(lo)
        for t in range(T):
            assert torch.equal(logits[t], lo[t]), t
        m, hf = _hf(torch.stack(lo), 1, n_new, eos, num_beams=K, num_return_sequences=2, do_sample=False)
        w = ids.shape[1]
        if not torch.equal(ids, hf.sequences):
            continue  # a near-tie of two candidates: HF's log_softmax and the engine's may differ in the last bit
        compared += 1
        assert torch.equal(eng.last_beam_indices.long(), hf.beam_indices.long())
        assert torch.allclose(eng.last_beam_scores.to(DEV), hf.sequences_scores, atol=1e-4)
        for t in range(w):
            fin = hf.scores[t] > -1e30
            assert torch.allclose(scores[t][fin], hf.scores[t][fin], atol=1e-5), t
        mine = m.compute_transition_scores(ids, tuple(scores[:w]), eng.last_beam_indices)
        theirs = m.compute_transition_scores(hf.sequences, hf.scores, hf.beam_indices)
        assert torch.allclose(mine, theirs, atol=1e-4)
    assert compared >= 2, compared


def test_sampled_scores_are_hf_warpers_on_the_processed_logits(fam):
    from u2tokenizer_b200.engine import GenerateRequest, LogitsProcessors
    eng, g, emb, lens, eos = fam
    eng.decode_impl = "tcgen05"
    for temp, k, p, procs in ((0.9, 40, 0.9, None), (1.2, 0, 0.8, LogitsProcessors(eos_token_ids=eos, **PROCS))):
        lo = []
        req = GenerateRequest(16, eos, (temp, k, p, 1234), procs, output_scores=True, output_logits=True)
        ids, scores, logits = eng._generate(emb, req, torch.tensor(lens), True, logits_out=lo)
        x_all = torch.stack(lo) * _inv_t(temp).to(DEV)
        for t in range(len(lo)):
            kept = scores[t] > -float("inf")
            assert torch.equal(scores[t][kept], x_all[t][kept]), t
            assert bool(kept.gather(1, ids[:, t:t + 1]).all()), t
            hf, near = _hf_kept(x_all[t], k, p)
            assert not bool(((kept != hf) & ~near).any()), t


# ------------------------------------------------------------------------------------------------
# chunks and ragged prompts: every row's outputs are its prompt's outputs alone
# ------------------------------------------------------------------------------------------------
def test_multi_chunk_beams_and_ragged_rows_equal_each_prompt_alone():
    from u2tokenizer_b200.engine import BeamSearch, U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g, kw = _family("qwen3")
    eng = U2Engine(g, synthetic_state_dict(g, seed=5, device="cpu", dtype=torch.bfloat16, **kw), device=DEV)
    images, ids, qids, lens = _inputs(g, qlens=(6, 2, 11, 4, 9))
    emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    plain = eng.generate_greedy(emb, 16, lengths=lens).cpu()
    eos = (int(plain[0, 5]), int(plain[3, 8]))
    # 5 prompts x 4 beams: a 16-row chunk and a 4-row chunk
    bm = BeamSearch(num_beams=4, length_penalty=1.0, early_stopping=False, num_return_sequences=2, pad_token_id=eos[0])
    got, sc, lg = eng.generate(emb, 16, eos_token_id=eos, lengths=lens, beam=bm, output_scores=True,
                               output_logits=True)
    bi = eng.last_beam_indices.clone()
    for b in range(5):
        alone, a_sc, a_lg = eng.generate(emb[b:b + 1, :lens[b]].contiguous(), 16, eos_token_id=eos, beam=bm,
                                         output_scores=True, output_logits=True)
        w = alone.shape[1]
        assert torch.equal(got[2 * b:2 * b + 2, :w], alone), b
        rb = bi[2 * b:2 * b + 2, :w]
        assert torch.equal(torch.where(rb >= 0, rb - 4 * b, rb), eng.last_beam_indices), b
        rows = slice(4 * b, 4 * b + 4)
        assert torch.allclose(sc[:w, rows], a_sc[:w], atol=1e-5) and torch.allclose(lg[:w, rows], a_lg[:w], atol=1e-5)
    # greedy over the ragged batch: each row up to its first EOS is its prompt alone
    got, sc, lg = eng.generate(emb, 16, eos_token_id=eos, lengths=lens, output_scores=True, output_logits=True)
    for b in range(5):
        alone, a_sc, a_lg = eng.generate(emb[b:b + 1, :lens[b]].contiguous(), 16, eos_token_id=eos,
                                         output_scores=True, output_logits=True)
        w = _upto_eos(alone[0], eos)
        assert torch.equal(got[b, :w], alone[0, :w]), b
        assert torch.allclose(sc[:w, b], a_sc[:w, 0], atol=1e-5) and torch.allclose(lg[:w, b], a_lg[:w, 0], atol=1e-5)


# ------------------------------------------------------------------------------------------------
# the model surface
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
    model.load_state_dict(synthetic_state_dict(g, seed=9, device="cpu", dtype=torch.bfloat16, bigram=1.0), strict=False)
    model = model.to(torch.bfloat16).cuda().eval()
    model.generation_config.eos_token_id = None
    return model, g


def test_model_outputs_wrap_the_same_sequences_with_the_same_launches_when_off():
    from transformers.generation import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput
    from u2tokenizer_b200 import _lib
    model, g = _make_model()
    images, ids, qids, lens = _inputs(g)
    mask = (torch.arange(ids.shape[1])[None] < torch.tensor(lens)[:, None]).long()
    kw = dict(question_ids=qids.cuda(), attention_mask=mask.cuda(), max_new_tokens=12)
    args = (images.cuda(), ids.cuda())
    first = model.generate(*args, **kw)
    eos = int(first[0, 4])
    kw["eos_token_id"] = eos
    model.generate(*args, **kw)
    n0 = _lib.launches()
    a = model.generate(*args, **kw)
    n1 = _lib.launches()
    d = model.generate(*args, return_dict_in_generate=True, **kw)
    n2 = _lib.launches()
    assert isinstance(d, GenerateDecoderOnlyOutput) and d.scores is None and d.logits is None
    assert torch.equal(d.sequences, a) and n2 - n1 == n1 - n0
    full = model.generate(*args, return_dict_in_generate=True, output_scores=True, output_logits=True, **kw)
    assert torch.equal(full.sequences, a)
    assert len(full.scores) == len(full.logits) == a.shape[1]
    assert torch.equal(torch.stack(full.scores), torch.stack(full.logits))  # greedy without processors
    n3 = _lib.launches()
    b = model.generate(*args, **kw)
    n4 = _lib.launches()
    assert torch.equal(a, b) and n4 - n3 == n1 - n0
    lp = model.compute_transition_scores(full.sequences, full.scores, normalize_logits=True)
    ref = torch.stack(full.scores, 1).log_softmax(-1).gather(2, a[:, :, None])[:, :, 0]
    assert torch.allclose(lp, ref, atol=1e-6)
    # beams; the flags come from generation_config too
    model.generation_config.return_dict_in_generate = True
    model.generation_config.output_scores = True
    bo = model.generate(*args, num_beams=4, num_return_sequences=2, **kw)
    assert isinstance(bo, GenerateBeamDecoderOnlyOutput) and bo.logits is None
    assert bo.sequences.shape[0] == 6 and len(bo.scores) == bo.sequences.shape[1] == bo.beam_indices.shape[1]
    assert bo.sequences_scores.shape == (6,)
    ts = model.compute_transition_scores(bo.sequences, bo.scores, bo.beam_indices)
    n_tok = (bo.beam_indices >= 0).sum(1)
    assert torch.allclose(ts.sum(1) / n_tok, bo.sequences_scores, atol=1e-4)  # length_penalty 1
    with pytest.raises(NotImplementedError):
        model.generate(*args, output_attentions=True, **kw)


# ------------------------------------------------------------------------------------------------
# continuous batching: return_logprobs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["greedy", "sampled", "n3", "processors"])
def test_generate_batch_logprobs_equal_transition_scores_of_generate_alone(fam, monkeypatch, mode):
    from u2tokenizer_b200 import _lib
    from u2tokenizer_b200.engine import LogitsProcessors, SlotRequest
    monkeypatch.setenv("U2_ATTN_SPLIT", "2")
    eng, g, emb, lens, eos = fam
    eng.decode_impl = "tcgen05"
    kw, n = {}, 1
    if mode == "sampled":
        kw = dict(do_sample=True, temperature=0.9, top_k=40, top_p=0.95)
    elif mode == "n3":
        kw, n = dict(do_sample=True, temperature=1.1, top_k=0, top_p=0.9), 3
    elif mode == "processors":
        kw = dict(do_sample=True, temperature=0.8, top_k=20, processors=LogitsProcessors(eos_token_ids=eos, **PROCS))
    embeds = [emb[b:b + 1, :lens[b]].contiguous() for b in range(len(lens))] * 2
    news, seeds = [14, 9, 17, 6, 20, 11], [100 + 3 * i for i in range(6)]
    reqs = lambda: (SlotRequest(str(i), embeds[i], news[i], seeds[i]) for i in range(len(embeds)))
    plain = eng.generate_continuous(reqs(), 4, eos_token_id=eos, num_return_sequences=n, **kw)
    n0 = _lib.launches()
    plain2 = eng.generate_continuous(reqs(), 4, eos_token_id=eos, num_return_sequences=n, **kw)
    n1 = _lib.launches()
    out = eng.generate_continuous(reqs(), 4, eos_token_id=eos, num_return_sequences=n, return_logprobs=True, **kw)
    n2 = _lib.launches()
    plain3 = eng.generate_continuous(reqs(), 4, eos_token_id=eos, num_return_sequences=n, **kw)
    n3 = _lib.launches()
    assert plain == plain2 == plain3 and n1 - n0 == n3 - n2
    for i in range(len(embeds)):
        ids, sc = eng.generate(embeds[i], news[i], eos_token_id=eos, seed=seeds[i], num_return_sequences=n,
                               output_scores=True, **kw)[:2]
        for j, (toks, lps) in enumerate(out[str(i)]):
            assert toks == plain[str(i)][j] and len(lps) == len(toks), (i, j)
            w = len(toks)
            assert ids[j, :w].tolist() == toks
            ref = sc[:w, j].log_softmax(-1).gather(1, ids[j, :w, None])[:, 0]
            assert (torch.tensor(lps, device=DEV) - ref).abs().max().item() < 2e-5, (mode, i, j)


def test_generate_batch_surface_fills_logprobs():
    model, g = _make_model()
    images, ids, qids, lens = _inputs(g)
    reqs = [dict(images=images[b:b + 1], input_ids=ids[b, :lens[b]], question_ids=qids[b:b + 1], max_new_tokens=8)
            for b in range(len(lens))]
    plain = model.generate_batch(reqs)
    out = model.generate_batch(reqs, return_logprobs=True)
    for rid, o in out.items():
        assert o.generated_tokens == plain[rid].generated_tokens and plain[rid].logprobs == []
        assert len(o.logprobs) == len(o.generated_tokens) and all(lp <= 0 for lp in o.logprobs)
    with pytest.raises(NotImplementedError):
        model.generate_batch(reqs, output_scores=True)
