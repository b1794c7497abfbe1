"""generate_batch() on the GPU: the slot kernels against their models, every request bit-identical to generate() on
that request alone (greedy, sampled, multi-sample, logits processors; both decode paths, eager and graph), oracle
parity, one captured step per (slots, capacity), cache growth, and the module surface."""
import random

import pytest
import torch

from common import tiny_geometry

DEV = "cuda"
pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
def test_slot_update_matches_the_slot_model():
    from u2tokenizer_b200 import ops
    rnd = random.Random(5)
    B, W, pad, eos = 13, 9, 3, (7, 11)
    params = ops.slot_params(DEV, pad, eos)
    for trial in range(20):
        max_new = [rnd.randint(1, W) for _ in range(B)]
        count = [rnd.randint(0, m - 1) for m in max_new]
        done = [int(rnd.random() < 0.3) for _ in range(B)]
        ids = [rnd.choice([7, 11, 20, 21, 22, 23]) for _ in range(B)]
        lens = [rnd.randint(5, 50) for _ in range(B)]
        out0 = torch.randint(100, 200, (B, W), dtype=torch.int64)
        slots = ops.slot_state([rnd.getrandbits(64) for _ in range(B)], list(range(B)), max_new, count, done).to(DEV)
        t_ids = torch.tensor(ids, device=DEV)
        t_out = out0.to(DEV)
        L = torch.tensor(lens, device=DEV, dtype=torch.int32)
        L1 = L + 1
        with_len = trial % 2 == 0
        ops.slot_update(t_ids, slots, t_out, params, L if with_len else None, L1 if with_len else None)
        f = {k: v.cpu().tolist() for k, v in ops.slot_state_fields(slots).items()}
        w_out = out0.clone()
        for b in range(B):
            c, d, ln = count[b], done[b], lens[b]
            if not d:
                w_out[b, c] = ids[b]
                c += 1
                d = int(ids[b] in eos or c >= max_new[b])
                if not d and with_len:
                    ln += 1
            assert f["count"][b] == c and f["done"][b] == d and f["max_new"][b] == max_new[b], (trial, b)
            assert t_ids[b].item() == (pad if d else ids[b]), (trial, b)
            assert L[b].item() == ln and L1[b].item() == ln + 1, (trial, b)
        assert torch.equal(t_out.cpu(), w_out)


def test_slot_sampler_is_the_sampler_at_the_slot_seed_step_and_row():
    from u2tokenizer_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(2)
    B, V = 6, 3001
    logits = torch.randn(B, V, device=DEV, generator=g) * 3
    seeds = [11, 2 ** 63 + 5, 11, 0, 77, 12345678901]
    rows, counts = [0, 1, 2, 5, 0, 3], [0, 4, 9, 1, 300, 2]
    for temp, k, p in ((1.0, 50, 1.0), (0.7, 0, 0.9), (1.3, 5, 0.5)):
        blk = ops.sample_params(DEV, temp, k, p, 999)  # its seed is not used: the slots carry theirs
        slots = ops.slot_state(seeds, rows, [1000] * B, counts).to(DEV)
        got = ops.sample_slots(logits, blk, slots).cpu()
        for b in range(B):
            rep = logits[b:b + 1].expand(rows[b] + 1, V).contiguous()
            want = ops.sample(rep, temperature=temp, top_k=k, top_p=p, seed=seeds[b], step=counts[b])[rows[b]]
            assert got[b].item() == want.item(), (temp, k, p, b)


def test_slot_processors_are_the_processors_at_each_slot_history_length():
    from u2tokenizer_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(3)
    B, V, cap = 5, 700, 24
    logits = torch.randn(B, V, device=DEV, generator=g)
    hist = torch.randint(0, 40, (B, cap), device=DEV, generator=g, dtype=torch.int32)
    ids = torch.randint(0, 40, (B,), device=DEV, generator=g)
    counts = [0, 1, 5, 17, 24]
    blk = ops.logits_proc_params(DEV, V, repetition_penalty=1.4, no_repeat_ngram_size=2, min_new_tokens=6,
                                 eos_token_ids=(3, 9), bad_words_ids=((5,), (12, 13), (1, 2, 3)))
    slots = ops.slot_state([0] * B, [0] * B, [100] * B, counts).to(DEV)
    got_l, got_h = logits.clone(), hist.clone()
    ops.logits_process_slots(got_l, blk, ids, got_h, slots)
    for b in range(B):
        wl, wh = logits[b:b + 1].clone(), hist[b:b + 1].clone()
        ops.logits_process(wl, blk, ids[b:b + 1].clone(), wh, step=counts[b])
        assert torch.equal(got_l[b], wl[0]), b
        assert torch.equal(got_h[b], wh[0]), b


# ------------------------------------------------------------------------------------------------
# the engine: every request as generate() runs it alone
# ------------------------------------------------------------------------------------------------
QLENS = (6, 2, 11, 4, 9, 1, 14, 3, 7, 12, 5)
NEWS = (24, 9, 17, 30, 5, 21, 12, 26, 8, 15, 19)


def _engine(family="qwen3"):
    from u2tokenizer_b200.engine import U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    if family == "qwen3":
        g, kw = tiny_geometry(), dict(bigram=1.0)
    else:
        rs = dict(factor=8.0, high_freq_factor=4.0, low_freq_factor=1.0, original_max_position_embeddings=16,
                  rope_type="llama3")
        g, kw = (tiny_geometry(qk_norm=False, rope_theta=500000.0, rope_scaling=rs, tie_word_embeddings=True),
                 dict(head_tail=1.0))
    sd16 = synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, **kw)
    return U2Engine(g, sd16, device=DEV), g, sd16


def _studies(g, qlens=QLENS, lt=16):
    from u2tokenizer_b200.synthetic import synthetic_inputs
    return [synthetic_inputs(g, batch=1, frames=2, n_question=n, lt=max(lt, n), seed=200 + i)
            for i, n in enumerate(qlens)]


@pytest.fixture(scope="module")
def tiny():
    eng, g, sd16 = _engine()
    studies = _studies(g)
    embeds = [eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda()) for im, rid, rq in studies]
    return eng, g, embeds


def _cut(row, eos):
    row = [int(x) for x in row]
    for i, t in enumerate(row):
        if t in eos:
            return row[:i + 1]
    return row


def _alone(eng, emb, max_new, eos, mode, seed, n):
    ids = eng.generate(emb, max_new, eos_token_id=eos, seed=seed, num_return_sequences=n, **mode).cpu()
    return [_cut(r, eos) for r in ids]


def _batch(eng, embeds, news, num_slots, eos, mode, seeds, n=1, use_graph=True):
    from u2tokenizer_b200.engine import SlotRequest
    reqs = (SlotRequest(str(i), embeds[i], news[i], seeds[i]) for i in range(len(embeds)))
    return eng.generate_continuous(reqs, num_slots, eos_token_id=eos, num_return_sequences=n, use_graph=use_graph,
                                   **mode)


MODES = {
    "greedy": (dict(), 1),
    "sampled": (dict(do_sample=True, temperature=0.9, top_k=40, top_p=0.95), 1),
    "n3": (dict(do_sample=True, temperature=1.1, top_k=0, top_p=0.9), 3),
}


def _processors():
    from u2tokenizer_b200.engine import LogitsProcessors
    return LogitsProcessors(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=4, eos_token_ids=(),
                            bad_words_ids=((17,), (30, 31)))


@pytest.mark.parametrize("impl", ["tcgen05", "gemv"])
@pytest.mark.parametrize("mode", ["greedy", "sampled", "n3", "processors"])
def test_every_request_is_bit_identical_to_generate_alone(tiny, monkeypatch, impl, mode):
    import dataclasses
    monkeypatch.setenv("U2_ATTN_SPLIT", "2")
    eng, g, embeds = tiny
    eng.decode_impl = impl
    if mode == "processors":
        kw, n = dict(do_sample=True, temperature=0.8, top_k=20), 1
    else:
        kw, n = MODES[mode]
        kw = dict(kw)
    # an EOS id that some requests meet early: request 0's fourth greedy token
    eos = (int(eng.generate(embeds[0], 4)[0, 3]),)
    if mode == "processors":
        kw["processors"] = dataclasses.replace(_processors(), eos_token_ids=eos)
    seeds = [1000 + 7 * i for i in range(len(embeds))]
    want = {str(i): _alone(eng, e, NEWS[i], eos, kw, seeds[i], n) for i, e in enumerate(embeds)}
    if mode == "greedy":
        assert any(len(w[0]) < NEWS[int(i)] for i, w in want.items())  # EOS ends some requests early
    for use_graph in (False, True):
        got = _batch(eng, embeds, NEWS, 4, eos, kw, seeds, n=n, use_graph=use_graph)
        assert sorted(got, key=int) == sorted(want, key=int)
        for rid in want:
            assert got[rid] == want[rid], (impl, mode, use_graph, rid, got[rid], want[rid])
        assert eng.last_continuous["admissions"] == len(embeds)


@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_greedy_requests_match_the_oracle(family):
    from oracle import u2_oracle as O
    eng, g, sd16 = _engine(family)
    sd = {k: v.float() for k, v in sd16.items()}
    studies = _studies(g, qlens=(6, 2, 11, 4, 9))
    n_new = 16
    embeds, refs, thr = [], [], 0.0
    for im, rid, rq in studies:
        with torch.no_grad():
            ref_logits = O.decoder_forward(sd, O.multimodal_embeds(sd, rid, im, rq, g), g)[0]
            refs.append(O.greedy_generate(sd, rid, im, rq, g, max_new_tokens=n_new))
        e = eng.multimodal_embeds(rid.cuda(), im.cuda(), rq.cuda())
        embeds.append(e)
        lg = eng.lm_logits(eng.prefill(e)).float().cpu()
        thr = max(thr, 4.0 * (lg - ref_logits).abs().max().item())
    got = _batch(eng, embeds, [n_new] * len(embeds), 2, (), {}, [0] * len(embeds))
    compared = 0
    for i, (ref_ids, margins) in enumerate(refs):
        low = (margins[0][:n_new] < thr).nonzero()
        upto = int(low[0]) if len(low) else n_new
        compared += upto
        assert got[str(i)][0][:upto] == ref_ids[0, :upto].tolist(), (family, i)
    if family == "qwen3":
        assert compared >= 0.9 * n_new * len(refs), (compared, thr)


def test_one_capture_per_slots_and_capacity_and_growth(tiny, monkeypatch):
    from u2tokenizer_b200.engine import slot_capacity
    monkeypatch.setenv("U2_ATTN_SPLIT", "2")
    eng, g, embeds = tiny
    eng.decode_impl = "tcgen05"
    news = [30] + list(NEWS[1:])  # the largest max_new_tokens first: the capacity never grows
    seeds = list(range(len(embeds)))
    kw = dict(do_sample=True, top_k=30)
    got = _batch(eng, embeds, news, 3, (), kw, seeds)
    assert eng.last_continuous["captures"] == 1 and eng.last_continuous["steps"] > max(news)
    assert all(len(got[str(i)][0]) == news[i] for i in range(len(embeds)))
    # a prompt longer than 128 positions mid-stream: the live slots move to a larger cache, one more capture
    long_im, long_ids, long_q = _studies(g, qlens=(150,), lt=150)[0]
    long_emb = eng.multimodal_embeds(long_ids.cuda(), long_im.cuda(), long_q.cuda())
    assert long_emb.shape[1] > 128
    embeds2 = embeds[:5] + [long_emb] + embeds[5:8]
    news2 = news[:5] + [14] + news[5:8]
    seeds2 = list(range(len(embeds2)))
    got2 = _batch(eng, embeds2, news2, 3, (), kw, seeds2)
    # the step at the first capacity is still captured from the call above; the grown cache adds one capture
    assert eng.last_continuous["captures"] == 1
    assert eng.last_continuous["capacity"] == slot_capacity(long_emb.shape[1], 30) > slot_capacity(128, 30)
    for i, e in enumerate(embeds2):
        assert got2[str(i)] == _alone(eng, e, news2[i], (), kw, seeds2[i], 1), i


def test_requests_that_finish_at_admission(tiny, monkeypatch):
    monkeypatch.setenv("U2_ATTN_SPLIT", "2")
    eng, g, embeds = tiny
    eng.decode_impl = "tcgen05"
    first = int(eng.generate(embeds[1], 1)[0, 0])
    news = [10, 10, 1, 10]
    got = _batch(eng, embeds[:4], news, 2, (first,), {}, [0] * 4)
    assert got["1"] == [[first]]                       # its first token is EOS
    assert len(got["2"][0]) == 1                       # max_new_tokens = 1
    for i in (0, 2, 3):
        assert got[str(i)] == _alone(eng, embeds[i], news[i], (first,), {}, 0, 1), i


# ------------------------------------------------------------------------------------------------
# the module surface
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


def test_generate_batch_matches_generate_rows():
    from u2tokenizer_b200.modeling import GenerationOutput
    model, g = _make_model()
    studies = _studies(g, qlens=(6, 2, 11, 4, 9, 3))
    eos = int(model.generate(studies[0][0].cuda(), studies[0][1].cuda(), question_ids=studies[0][2].cuda(),
                             max_new_tokens=3, do_sample=False)[0, 2])
    model.generation_config.eos_token_id = eos
    model.generation_config.do_sample = True
    model.generation_config.top_p = 0.9
    news = [12, 7, 15, 9, 11, 6]
    pulled = []

    def requests():  # CPU-resident volumes, squeezed shapes, read lazily
        for i, (im, rid, rq) in enumerate(studies):
            pulled.append(i)
            r = dict(images=im[0], input_ids=rid[0], question_ids=rq, max_new_tokens=news[i])
            if i == 4:
                r.update(request_id="study-4", seed=77)
            yield r

    out = model.generate_batch(requests(), num_slots=3, seed=500, pad_token_id=0)
    assert sorted(out) == ["0", "1", "2", "3", "5", "study-4"] and pulled == list(range(6))
    for i, (im, rid, rq) in enumerate(studies):
        rid_key = "study-4" if i == 4 else str(i)
        o = out[rid_key]
        assert isinstance(o, GenerationOutput) and o.request_id == rid_key and o.prompt_ids == rid[0].tolist()
        row = model.generate(im.cuda(), rid.cuda(), question_ids=rq.cuda(), max_new_tokens=news[i],
                             seed=77 if i == 4 else 500 + i, pad_token_id=0)[0].cpu().tolist()
        assert o.generated_tokens == _cut(row, (eos,)), i
    # three samples per request share one prefill; greedy defaults come back with do_sample=False
    out3 = model.generate_batch([dict(images=studies[1][0], input_ids=studies[1][1], question_ids=studies[1][2])],
                                num_slots=4, num_return_sequences=3, max_new_tokens=8, seed=9)
    rows = model.generate(studies[1][0].cuda(), studies[1][1].cuda(), question_ids=studies[1][2].cuda(),
                          max_new_tokens=8, num_return_sequences=3, seed=9).cpu()
    assert out3["0"].generated_tokens == [_cut(r, (eos,)) for r in rows.tolist()]
    with pytest.raises(NotImplementedError):
        model.generate_batch([], num_beams=2)
    with pytest.raises(TypeError):
        model.generate_batch([dict(input_ids=studies[0][1], attention_mask=None)])
