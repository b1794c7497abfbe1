"""Generation scores without a GPU: the output flags of generate() (kwargs, then generation_config), the options that
stay refused, generate_batch()'s return_logprobs and its refusals, GenerationOutput's logprobs default, and HF's
beam_indices rebuilt from the beam records."""
import pytest
import torch

from u2tokenizer_b200.engine import SlotRequest, SlotScheduler, U2Engine
from u2tokenizer_b200.modeling import GenerationOutput, U2MetaForCausalLM


class _Cfg:
    num_beams, do_sample, temperature, top_k, top_p = 1, False, None, None, None
    eos_token_id, pad_token_id, max_length, num_return_sequences = 2, None, 20, None
    repetition_penalty = no_repeat_ngram_size = min_new_tokens = min_length = bad_words_ids = None
    return_dict_in_generate = output_scores = output_logits = False


class _Model(U2MetaForCausalLM):
    def get_model(self):
        return None


def _flags(gc=None, **kw):
    out = U2MetaForCausalLM._generate_output_flags(kw, gc)
    assert not kw, "the flags are consumed"
    return out


def test_output_flags_come_from_kwargs_then_generation_config():
    assert _flags() == (False, False, False)
    assert _flags(return_dict_in_generate=True) == (True, False, False)
    assert _flags(return_dict_in_generate=True, output_scores=True) == (True, True, False)
    assert _flags(return_dict_in_generate=True, output_logits=True) == (True, False, True)
    # HF keeps scores and logits only in a returned dict
    assert _flags(output_scores=True, output_logits=True) == (False, False, False)
    gc = _Cfg()
    gc.return_dict_in_generate, gc.output_scores = True, True
    assert _flags(gc) == (True, True, False)
    assert _flags(gc, output_scores=False, output_logits=True) == (True, False, True)
    assert _flags(gc, return_dict_in_generate=False) == (False, False, False)


@pytest.mark.parametrize("k", ["output_attentions", "output_hidden_states"])
def test_attentions_and_hidden_states_stay_refused(k):
    with pytest.raises(NotImplementedError):
        U2MetaForCausalLM._check_remaining_generate_kwargs({k: True})
    U2MetaForCausalLM._check_remaining_generate_kwargs({k: False})


def _head(gc=None, **kw):
    return _Model()._generate_batch_head(kw, gc or _Cfg(), None, 16, 512)


def test_generate_batch_accepts_return_logprobs_and_refuses_scores():
    assert _head()["return_logprobs"] is False
    assert _head(return_logprobs=True)["return_logprobs"] is True
    gc = _Cfg()
    gc.return_logprobs = True
    assert _head(gc)["return_logprobs"] is True
    for k in ("output_scores", "return_dict_in_generate", "output_logits"):
        with pytest.raises(NotImplementedError):
            _head(**{k: True})


def test_generation_output_defaults_logprobs_to_an_empty_list():
    a, b = GenerationOutput("0", [1, 2], [3, 4]), GenerationOutput("1", [1], [5])
    assert a.logprobs == [] and b.logprobs == [] and a.logprobs is not b.logprobs
    assert GenerationOutput("2", [1], [3], [-0.5]).logprobs == [-0.5]


def test_beam_backtrack_rebuilds_hf_beam_indices():
    """Two prompts of K = 2 beams over 3 steps; rec[s, row] = (token, parent beam) of the running beam in `row` after
    step s. HF's beam_indices: per step the batch-wide row the token was appended to, -1 after the hypothesis ends."""
    i32 = torch.int32
    rec = torch.zeros(3, 4, 2, dtype=i32)
    rec[0, 0], rec[0, 1] = torch.tensor([10, 0]), torch.tensor([11, 0])
    rec[1, 0], rec[1, 1] = torch.tensor([12, 1]), torch.tensor([13, 0])
    rec[0, 2], rec[0, 3] = torch.tensor([20, 0]), torch.tensor([21, 0])
    rec[1, 2], rec[1, 3] = torch.tensor([22, 0]), torch.tensor([23, 1])
    # fin_info per row: (unused, last step, parent beam at the last step, last token)
    info = torch.tensor([[0, 2, 0, 99], [0, 0, 0, 98], [0, 1, 1, 97], [0, 2, 1, 96]], dtype=i32)
    bs = dict(fin_info=info, fin_score=torch.tensor([-1.0, -2.0, -3.0, -4.0]), rec=rec)
    seqs, sc, rows = U2Engine._beam_backtrack(bs, P=2, K=2, n_ret=2, fill=0, row0=6)
    assert seqs == [[11, 12, 99], [98], [21, 97], [21, 23, 96]]
    assert rows == [[6, 7, 6], [6], [8, 9], [8, 9, 9]]
    assert sc.tolist() == [-1.0, -2.0, -3.0, -4.0]


def test_scheduler_passes_per_slot_results_through():
    """With return_logprobs a backend reports (tokens, log-probs) per finished slot; the scheduler only routes it."""
    class Backend:
        def __init__(self):
            self.slot = [None, None]

        def reserve(self, capacity, width):
            pass

        def admit(self, r, slots):
            for s in slots:
                self.slot[s] = [r, 0]

        def step(self):
            for st in self.slot:
                if st is not None and st[1] < st[0].max_new_tokens:
                    st[1] += 1

        def snapshot(self):
            return [None if st is None or st[1] < st[0].max_new_tokens else
                    ([st[0].seed] * st[1], [-0.25 * st[0].seed] * st[1]) for st in self.slot]

        @staticmethod
        def read(h):
            return h

    reqs = [SlotRequest(str(i), torch.empty(1, 4, 0), 3 + i, seed=i + 1) for i in range(3)]
    out = SlotScheduler(Backend(), 2).run(reqs)
    for i in range(3):
        assert out[str(i)] == [([i + 1] * (3 + i), [-0.25 * (i + 1)] * (3 + i))]
