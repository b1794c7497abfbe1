"""Host-side logic of the module surface that needs no GPU: argument checks that guard the fused CUDA path."""
import pytest
import torch


def _cls():
    from u2tokenizer_b200.modeling import U2LlamaForCausalLM
    return U2LlamaForCausalLM


def test_right_padded_masks_are_accepted():
    chk = _cls()._check_right_padded
    chk(None)
    chk(torch.ones(3, 7, dtype=torch.long))
    chk(torch.tensor([[1, 1, 1, 0, 0], [1, 1, 1, 1, 1], [1, 0, 0, 0, 0]]))
    chk(torch.tensor([[True, True, False]]))


@pytest.mark.parametrize("mask", [
    torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1]]),   # left padding: the usual HF layout for batched generation
    torch.tensor([[1, 0, 1, 1, 0]]),                   # a hole
    torch.tensor([[0, 0, 0]]),                         # nothing valid
    torch.ones(2, 3, 4),                               # not [batch, tokens]
])
def test_other_masks_are_refused_loudly(mask):
    """The reference hands the mask to HF (u2llama.py:76-87); the fused path has none, so anything that would change the
    result must raise instead of being ignored."""
    with pytest.raises(NotImplementedError):
        _cls()._check_right_padded(mask)


def test_surface_matches_the_reference_call_forms():
    """forward / generate keep the reference's parameter names (u2llama.py:41-55, 90-96; train_stage1.py:244-250 passes
    images, input_ids, labels, attention_mask, question_ids by keyword)."""
    import inspect
    from u2tokenizer_b200.modeling import U2LlamaForCausalLM, U2Qwen3ForCausalLM
    want = ["images", "input_ids", "labels", "attention_mask", "question_ids", "position_ids", "past_key_values",
            "inputs_embeds", "use_cache", "output_attentions", "output_hidden_states", "return_dict"]
    for cls in (U2LlamaForCausalLM, U2Qwen3ForCausalLM):
        names = [n for n in inspect.signature(cls.forward).parameters if n != "self"]
        assert names[:len(want)] == want, names
        gen = [n for n in inspect.signature(cls.generate).parameters if n != "self"]
        assert gen[:2] == ["images", "inputs"] and "question_ids" in gen, gen
        for attr in ("get_model", "prepare_inputs_for_multimodal", "initialize_vision_tokenizer",
                     "prepare_inputs_for_generation", "per_token_logps"):
            assert hasattr(cls, attr), attr


G = 0x9E3779B97F4A7C15  # seed stride between multi-sample chunks


@pytest.mark.parametrize("B, n, cap, beam, rows, seeds", [
    (3, 1, 16, False, [[0, 1, 2]], [0]),
    (20, 1, 16, False, [list(range(16)), [16, 17, 18, 19]], [0, 0]),   # single samples: every chunk keeps the seed
    (2, 9, 16, False, [[0] * 9 + [1] * 7, [1, 1]], [0, G]),           # a prompt's samples may straddle chunks
    (5, 4, 16, True, [[p for p in range(4) for _ in range(4)], [4] * 4], [0, G]),
    (3, 3, 16, True, [[0] * 3 + [1] * 3 + [2] * 3], [0]),
    (20, 1, 8, False, [list(range(8)), list(range(8, 16)), [16, 17, 18, 19]], [0, 0, 0]),
    (5, 3, 8, True, [[0] * 3 + [1] * 3, [2] * 3 + [3] * 3, [4] * 3], [0, G, 2 * G]),  # beams never straddle chunks
])
def test_chunk_plan_maps_rows_to_prompts_and_seeds(B, n, cap, beam, rows, seeds):
    """generate() decodes B prompts x n rows (row b * n + s is row s of prompt b) in chunks of at most cap rows:
    windows of cap rows, or (cap // n) * n rows for beam search; chunk i of a multi-sample request samples with
    seed + 0x9E3779B97F4A7C15 * i."""
    from u2tokenizer_b200.engine import chunk_plan
    plan = chunk_plan(B, n, cap, beam)
    assert [src.tolist() for src, _ in plan] == rows
    assert [off for _, off in plan] == seeds
    assert all(src.dtype == torch.int64 and src.device.type == "cpu" for src, _ in plan)
    width = (cap // n) * n if beam else cap
    assert all(len(src) == width for src, _ in plan[:-1]) and 0 < len(plan[-1][0]) <= width


@pytest.mark.parametrize("eos, want", [(None, ()), (7, (7,)), ([3, 9], (3, 9)), ((4,), (4,)),
                                       (torch.tensor(5), (5,)), (torch.tensor([[1, 2]]), (1, 2))])
def test_eos_ids_takes_every_form_generate_accepts(eos, want):
    from u2tokenizer_b200.engine import GenerateRequest, eos_ids
    assert eos_ids(eos) == want and all(type(e) is int for e in eos_ids(eos))
    assert GenerateRequest(4, eos).eos_token_id == want


def test_generate_request_runs_a_neutral_processor_configuration_as_none():
    from u2tokenizer_b200.engine import GenerateRequest, LogitsProcessors
    assert GenerateRequest(4, processors=LogitsProcessors(min_new_tokens=2)).processors is None  # no EOS id to ban
    pc = LogitsProcessors(repetition_penalty=1.3)
    assert GenerateRequest(4, processors=pc).processors is pc
