"""generate_batch() host side without a GPU: request parsing and refusals, default ids and seeds, and the slot
scheduler (slot order, n-sample admission, lazy reading of the requests, cache growth) on a fake device backend."""
import pytest
import torch

from u2tokenizer_b200 import engine as E
from u2tokenizer_b200.engine import SlotRequest, SlotScheduler, slot_capacity
from u2tokenizer_b200.modeling import U2MetaForCausalLM


# ------------------------------------------------------------------------------------------------
# request parsing and refusals
# ------------------------------------------------------------------------------------------------
def _req(i, r, seed=100):
    return U2MetaForCausalLM._generate_batch_request(i, r, seed)


def test_request_defaults_ids_and_seeds():
    a = _req(0, dict(input_ids=torch.arange(5)))
    assert a["request_id"] == "0" and a["seed"] == 100 and a["input_ids"].shape == (1, 5)
    assert a["images"] is None and a["max_new_tokens"] is None
    b = _req(3, dict(input_ids=torch.arange(5)[None], images=torch.zeros(2, 4, 8, 8), question_ids=torch.arange(3)))
    assert b["request_id"] == "3" and b["seed"] == 103
    assert b["images"].shape == (1, 2, 4, 8, 8) and b["question_ids"].shape == (1, 3)
    c = _req(7, dict(input_ids=[1, 2], seed=5, request_id="study-9", max_new_tokens=4))
    assert c["request_id"] == "study-9" and c["seed"] == 5 and c["max_new_tokens"] == 4


@pytest.mark.parametrize("bad", [dict(input_ids=[1], attention_mask=[1]), dict(input_ids=[1], num_beams=2),
                                 dict(images=torch.zeros(1, 1, 4, 4, 4))])
def test_request_unknown_or_missing_keys_raise_type_error(bad):
    with pytest.raises(TypeError):
        _req(0, bad)


@pytest.mark.parametrize("bad", [dict(input_ids=torch.zeros(2, 3)), dict(input_ids=[1], max_new_tokens=0),
                                 dict(input_ids=[1], images=torch.zeros(2, 1, 4, 4, 4))])
def test_request_bad_shapes_and_values_raise_value_error(bad):
    with pytest.raises(ValueError):
        _req(0, bad)


class _Cfg:
    num_beams, do_sample, temperature, top_k, top_p = 1, False, None, None, None
    eos_token_id, pad_token_id, max_length, num_return_sequences = 2, None, 20, None
    repetition_penalty = no_repeat_ngram_size = min_new_tokens = min_length = bad_words_ids = None


class _Model(U2MetaForCausalLM):
    def get_model(self):
        return None


def _head(num_slots=None, rows=16, gc=_Cfg(), **kw):
    return _Model()._generate_batch_head(kw, gc, num_slots, rows, 512)


def test_head_defaults_and_generation_config_fallbacks():
    h = _head(seed=11)
    assert h["num_slots"] == 16 and h["n"] == 1 and not h["do_sample"] and h["seed"] == 11
    assert h["eos"] == (2,) and h["pad"] == 2 and h["max_length"] == 20 and h["processors"] is None
    gc = _Cfg()
    gc.do_sample, gc.top_p, gc.repetition_penalty, gc.pad_token_id = True, 0.9, 1.3, 0
    h = _head(num_slots=4, gc=gc, num_return_sequences=3, min_new_tokens=2)
    assert h["do_sample"] and h["top_p"] == 0.9 and h["n"] == 3 and h["pad"] == 0
    assert h["processors"].repetition_penalty == 1.3 and h["processors"].min_new_tokens == 2


def test_head_refusals():
    with pytest.raises(NotImplementedError):
        _head(num_beams=4)
    with pytest.raises(ValueError):
        _head(num_slots=17)
    with pytest.raises(ValueError):
        _head(num_slots=0)
    with pytest.raises(ValueError):
        _head(num_slots=2, do_sample=True, num_return_sequences=3)
    with pytest.raises(ValueError):
        _head(num_return_sequences=2)  # greedy
    with pytest.raises(NotImplementedError):
        _head(output_scores=True)
    with pytest.raises(TypeError):
        _head(bogus=1)
    with pytest.raises(NotImplementedError):
        _head(min_length=30)


# ------------------------------------------------------------------------------------------------
# the scheduler on a fake backend
# ------------------------------------------------------------------------------------------------
class FakeBackend:
    """Slots that generate request-derived tokens: request r emits r.seed * 100 + t at its step t and finishes after
    its max_new_tokens. Snapshots copy the state, like the device copy the real backend enqueues."""

    def __init__(self, S):
        self.S = S
        self.slot = [None] * S   # [request, row j, tokens]
        self.log = []

    def reserve(self, capacity, width):
        self.log.append(("reserve", capacity, width))

    def admit(self, r, slots):
        self.log.append(("admit", r.request_id, tuple(slots)))
        for j, s in enumerate(slots):
            assert self.slot[s] is None or self.slot[s][3], "admitted into a live slot"
            toks = [r.seed * 100 + j]
            self.slot[s] = [r, j, toks, len(toks) >= r.max_new_tokens]

    def step(self):
        for st in self.slot:
            if st is not None and not st[3]:
                st[2].append(st[0].seed * 100 + st[1] + 10 * len(st[2]))
                st[3] = len(st[2]) >= st[0].max_new_tokens

    def snapshot(self):
        return [list(st[2]) if st is not None and st[3] else None for st in self.slot]

    @staticmethod
    def read(h):
        return h


def _reqs(lens, news, log=None):
    for i, (L, n) in enumerate(zip(lens, news)):
        if log is not None:
            log.append(("pull", str(i)))
        yield SlotRequest(str(i), torch.empty(1, L, 0), n, seed=i)


def _want(i, n_new, j=0):
    return [i * 100 + j + 10 * t for t in range(n_new)]


def test_slot_order_and_results():
    be = FakeBackend(3)
    news = [5, 30, 9, 2, 17, 4, 1]
    out = SlotScheduler(be, 3).run(_reqs([10] * 7, news))
    assert sorted(out) == [str(i) for i in range(7)]
    for i, n in enumerate(news):
        assert out[str(i)] == [_want(i, n)]
    admits = [e for e in be.log if e[0] == "admit"]
    assert [a[2] for a in admits[:3]] == [(0,), (1,), (2,)]  # lowest free slot first
    # request 0 (5 tokens) and 3 (2) finish before 2 (9): the refills go to the lowest freed slot
    assert admits[3] == ("admit", "3", (0,))


def test_n_sample_request_waits_for_n_free_slots():
    be = FakeBackend(4)
    sched = SlotScheduler(be, 4, samples=3)
    out = sched.run(_reqs([8] * 3, [40, 3, 6]))
    admits = [e for e in be.log if e[0] == "admit"]
    assert admits[0] == ("admit", "0", (0, 1, 2))
    # request 1 needs 3 slots: only slot 3 is free until request 0's samples finish
    assert admits[1] == ("admit", "1", (0, 1, 2))
    assert all(len(out[str(i)]) == 3 for i in range(3))
    assert out["0"] == [_want(0, 40, j) for j in range(3)]


def test_requests_are_pulled_lazily():
    log = []
    be = FakeBackend(2)
    orig = be.admit
    be.admit = lambda r, s: (log.append(("admit", r.request_id)), orig(r, s))
    SlotScheduler(be, 2).run(_reqs([4] * 6, [50, 3, 3, 3, 3, 3], log))
    held = 0
    for e in log:
        held += 1 if e[0] == "pull" else 0
        if e[0] == "admit":
            held -= 1
        assert held <= 1, log  # at most the one request being admitted is held beyond the slots
    pulls = [e for e in log if e[0] == "pull"]
    assert len(pulls) == 6


def test_capacity_grows_with_a_longer_prompt():
    be = FakeBackend(2)
    sched = SlotScheduler(be, 2)
    out = sched.run(_reqs([100, 60, 300, 20], [10, 10, 7, 12]))
    res = [e for e in be.log if e[0] == "reserve"]
    assert res[0] == ("reserve", slot_capacity(100, 10), 10) == ("reserve", 138, 10)
    assert ("reserve", slot_capacity(300, 10), 10) in res        # the 300-token prompt grows the cache
    assert res[-1] == ("reserve", slot_capacity(300, 12), 12)    # so does a larger max_new_tokens
    assert sched.capacity == 396
    # growth happens before the admission that needs it
    i = be.log.index(("reserve", 394, 10))
    assert be.log[i + 1][:2] == ("admit", "2")
    assert out["3"] == [_want(3, 12)]


def test_duplicate_request_ids_are_refused():
    be = FakeBackend(2)
    reqs = [SlotRequest("a", torch.empty(1, 3, 0), 4), SlotRequest("a", torch.empty(1, 3, 0), 4)]
    with pytest.raises(ValueError, match="duplicate"):
        SlotScheduler(be, 2).run(reqs)


def test_poll_interval_is_a_constant():
    assert isinstance(E.SLOT_POLL_STEPS, int) and E.SLOT_POLL_STEPS >= 1
