"""The mu2-Phi-3 family on the CPU: configuration and geometry (with the Phi-3 variants that are refused), HF Phi3
state-dict keys, the remote-code checkpoint round trip, and the fp32 Phi-3 restatement the GPU tests compare against,
pinned to the installed HF Phi3ForCausalLM across the sliding window (prefill and cached decode)."""
import json
import os
import sys
import types

import pytest
import torch

import phi3_oracle as P3
from common import fp32_sd, tiny_geometry
from u2tokenizer_b200 import checkpoint
from u2tokenizer_b200.configuration import PHI3_MINI_4K, U2Phi3Config
from u2tokenizer_b200.geometry import Geometry
from u2tokenizer_b200.synthetic import param_shapes

WINDOW = 24


def tiny_phi3_geometry(window=WINDOW, **over):
    """E 192, 2 heads of 96 (MHA), I 384: the head_dim and the attention shape of Phi-3-mini, scaled down."""
    kw = dict(qk_norm=False, hidden_size=192, intermediate_size=384, num_attention_heads=2, num_key_value_heads=2,
              head_dim=96, rms_norm_eps=1e-5, rope_theta=1e4, decoder_family="phi3", sliding_window=window)
    kw.update(over)
    return tiny_geometry(**kw)


def tiny_phi3_config(window=WINDOW):
    g = tiny_phi3_geometry(window)
    return U2Phi3Config(hidden_size=g.hidden_size, intermediate_size=g.intermediate_size, num_hidden_layers=2,
                        num_attention_heads=2, num_key_value_heads=2, vocab_size=g.vocab_size, rms_norm_eps=1e-5,
                        sliding_window=window, pad_token_id=0, bos_token_id=1, eos_token_id=2, image_size=g.image_size,
                        patch_size=g.patch_size, u2t_num_layers=g.u2t_num_layers, u2t_top_k=g.u2t_top_k,
                        num_3d_query_token=g.num_3d_query_token, vit_hidden_size=g.vit_hidden, vit_mlp_dim=g.vit_mlp,
                        vit_num_layers=g.vit_layers, vit_num_heads=g.vit_heads, mm_hidden_size=g.vit_hidden)


@pytest.fixture
def package_auto_classes(monkeypatch):
    """The package's "u2phi3" registration, as in a process that never imported the reference's own
    src.model.language_model (whose __init__ registers its u2Phi3Config under the same model_type)."""
    from transformers.models.auto.configuration_auto import CONFIG_MAPPING
    monkeypatch.setitem(CONFIG_MAPPING._extra_content, "u2phi3", U2Phi3Config)


def test_three_class_import(package_auto_classes):
    """The reference's stage-1 import (train_stage1.py:11) with the package in place of src.model.language_model."""
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM, u2LlamaForCausalLM, u2Phi3ForCausalLM, u2Qwen3ForCausalLM
    assert u2Phi3ForCausalLM is U2Phi3ForCausalLM
    assert u2LlamaForCausalLM.config_class.model_type == "u2llama"
    assert u2Qwen3ForCausalLM.config_class.model_type == "u2Qwen3"
    assert u2Phi3ForCausalLM.config_class.model_type == "u2phi3"
    from transformers import AutoConfig, AutoModelForCausalLM
    cfg = AutoConfig.for_model("u2phi3", **{k: v for k, v in PHI3_MINI_4K.items() if k != "num_hidden_layers"},
                               num_hidden_layers=1)
    assert isinstance(cfg, U2Phi3Config)
    assert AutoModelForCausalLM._model_mapping[U2Phi3Config] is U2Phi3ForCausalLM


def test_phi3_mini_geometry():
    g = Geometry.from_hf(U2Phi3Config(**PHI3_MINI_4K))
    assert (g.decoder_family, g.hidden_size, g.head_dim, g.num_attention_heads, g.num_key_value_heads) == \
        ("phi3", 3072, 96, 32, 32)
    assert (g.intermediate_size, g.vocab_size, g.sliding_window, g.window) == (8192, 32064, 2047, 2047)
    assert g.rope_theta == 1e4 and g.rope_scaling is None and not g.qk_norm and not g.tie_word_embeddings
    assert g.rms_norm_eps == 1e-5 and g.decoder_dropout == 0.0
    # the multimodal defaults are those of the other two configs; the tokenizer runs at E / 8 = 384 per head
    assert g.u2t_num_heads == 8 and g.hidden_size // g.u2t_num_heads == 384
    # no window -> None (the kernels' 0)
    g2 = Geometry.from_hf(U2Phi3Config(**dict(PHI3_MINI_4K, sliding_window=None)))
    assert g2.sliding_window is None and g2.window == 0
    # the Llama / Qwen3 geometries are unchanged: no window, separate projections
    from u2tokenizer_b200.configuration import QWEN3_8B, U2Qwen3Config
    gq = Geometry.from_hf(U2Qwen3Config(**QWEN3_8B))
    assert gq.decoder_family == "llama" and gq.sliding_window is None and gq.qk_norm


@pytest.mark.parametrize("over, what", [
    (dict(rope_scaling=dict(rope_type="longrope", short_factor=[1.0] * 48, long_factor=[1.0] * 48,
                            original_max_position_embeddings=4096), max_position_embeddings=131072), "longrope"),
    (dict(partial_rotary_factor=0.75), "partial_rotary_factor"),
])
def test_out_of_scope_variants_raise(over, what):
    with pytest.raises(NotImplementedError, match=what):
        Geometry.from_hf(U2Phi3Config(**dict(PHI3_MINI_4K, **over)))


@pytest.mark.parametrize("field", ["resid_pdrop", "embd_pdrop", "attention_dropout"])
def test_nonzero_dropout_is_refused_for_training(field):
    """Eval mode ignores dropout (as HF does); the training path has none, so a non-zero rate raises there. A zero-dropout
    Phi-3 trains (tests/test_phi3_train_gpu.py)."""
    g = Geometry.from_hf(U2Phi3Config(**dict(PHI3_MINI_4K, **{field: 0.1})))
    assert g.decoder_dropout == 0.1
    from u2tokenizer_b200.train import TrainEngine
    with pytest.raises(NotImplementedError, match="dropout"):
        TrainEngine(g, {}, device="cpu")
    assert Geometry.from_hf(U2Phi3Config(**PHI3_MINI_4K)).decoder_dropout == 0.0


def test_lora_targets_and_streams():
    """PEFT targets on Phi-3 are the four fused linears find_all_linear_names returns; each is a group with one adapter;
    their mask streams are disjoint from the Llama / Qwen3 ones, which do not move."""
    from u2tokenizer_b200.lora import LoraConfig, _resolve_targets
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM
    from u2tokenizer_b200.train import Layout, LoraSpec, lora_groups, lora_stream
    cfg = tiny_phi3_config()
    model = U2Phi3ForCausalLM(cfg)
    found, kinds = _resolve_targets(model, LoraConfig(r=8, target_modules=["qkv_proj", "o_proj", "gate_up_proj",
                                                                           "down_proj"]))
    assert kinds == ("qkv_proj", "o_proj", "gate_up_proj", "down_proj") and len(found) == 8
    with pytest.raises(NotImplementedError):
        _resolve_targets(model, LoraConfig(r=8, target_modules=["embed_tokens"]))
    g = Geometry.from_hf(cfg)
    assert all(len(m) == 1 for _, m in lora_groups(g))
    streams = {lora_stream(g, li, t) for li in range(32) for t in kinds}
    gl = tiny_geometry(qk_norm=False)
    old = {li * 8 + t for li in range(4096) for t in range(7)}
    assert len(streams) == 4 * 32 and not streams & old
    assert [lora_stream(gl, 3, t) for t in ("q_proj", "down_proj")] == [24, 30]
    lay = Layout(g, lora=LoraSpec(r=8, scaling=2.0, dropout=0.0, targets=kinds))
    assert lay.shapes["model.layers.0.self_attn.qkv_proj.lora_B.default.weight"] == (3 * 192, 8)
    assert lay.shapes["model.layers.0.mlp.gate_up_proj.lora_B.default.weight"] == (2 * 384, 8)
    assert "model.layers.0.self_attn.qkv_proj.weight" in lay.frozen_names


def test_state_dict_keys_are_hf_phi3():
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM
    cfg = tiny_phi3_config()
    model = U2Phi3ForCausalLM(cfg)
    sd = model.state_dict()
    shapes = param_shapes(Geometry.from_hf(cfg))
    assert set(sd) == set(shapes)
    assert all(tuple(sd[k].shape) == shapes[k] for k in shapes)
    assert tuple(sd["model.layers.0.self_attn.qkv_proj.weight"].shape) == ((2 + 2 * 2) * 96, 192)
    assert tuple(sd["model.layers.0.mlp.gate_up_proj.weight"].shape) == (2 * 384, 192)
    assert not any(".q_proj." in k or ".gate_proj." in k for k in sd)


def test_remote_code_round_trip(tmp_path, monkeypatch, package_auto_classes):
    import transformers.dynamic_module_utils as dmu
    from transformers import AutoModelForCausalLM
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM
    monkeypatch.setattr(dmu, "HF_MODULES_CACHE", str(tmp_path / "hf_modules"))
    monkeypatch.setattr(sys, "path", list(sys.path))
    cfg = tiny_phi3_config()
    model = U2Phi3ForCausalLM(cfg)
    model.load_state_dict({k: v for k, v in fp32_sd(Geometry.from_hf(cfg), seed=2).items()})
    d = str(tmp_path / "ckpt")
    checkpoint.save_pretrained(model, d)
    cj = json.load(open(os.path.join(d, "config.json")))
    assert cj["auto_map"] == {"AutoConfig": "configuration_u2.u2Config",
                              "AutoModelForCausalLM": "modeling_u2Phi3.u2Phi3ForCausalLM"}
    assert cj["architectures"] == ["u2Phi3ForCausalLM"] and cj["model_type"] == "u2phi3"
    loaded = AutoModelForCausalLM.from_pretrained(d, trust_remote_code=True)
    assert isinstance(loaded, U2Phi3ForCausalLM)
    a, b = model.state_dict(), loaded.state_dict()
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert loaded.config.sliding_window == WINDOW and Geometry.from_hf(loaded.config).decoder_family == "phi3"


def test_plain_phi3_checkpoint_then_initialize_vision_modules(tmp_path):
    """Stage-1 bring-up (train_stage1.py:290-330): a plain Phi-3 checkpoint loads into U2Phi3ForCausalLM, then
    initialize_vision_modules adds the vision tower, projector and mu2-tokenizer."""
    from transformers import Phi3Config, Phi3ForCausalLM
    from u2tokenizer_b200.modeling import U2Phi3ForCausalLM
    g = tiny_phi3_geometry()
    plain = Phi3ForCausalLM(Phi3Config(hidden_size=192, intermediate_size=384, num_hidden_layers=2, num_attention_heads=2,
                                       num_key_value_heads=2, vocab_size=g.vocab_size, sliding_window=WINDOW,
                                       pad_token_id=0, bos_token_id=1, eos_token_id=2))
    d = str(tmp_path / "phi3")
    plain.save_pretrained(d)
    model = U2Phi3ForCausalLM.from_pretrained(d)
    for k, v in plain.state_dict().items():
        assert torch.equal(model.state_dict()[k], v), k
    # the reference's model_args carry the canonical multimodal hyper-parameters (train_stage1.py:46-78)
    from u2tokenizer_b200.configuration import MM_DEFAULTS
    args = types.SimpleNamespace(**MM_DEFAULTS, freeze_vision_tower=False, pretrain_vision_model=None,
                                 pretrain_mm_mlp_adapter=None)
    model.get_model().initialize_vision_modules(args)
    assert model.get_vision_tower() is not None and model.get_u2tokenizer() is not None
    shapes = param_shapes(Geometry.from_hf(model.config))
    sd = model.state_dict()
    assert set(sd) == set(shapes) and all(tuple(sd[k].shape) == shapes[k] for k in shapes)


def _hf_phi3(g, sd):
    from transformers import Phi3Config, Phi3ForCausalLM
    cfg = Phi3Config(hidden_size=g.hidden_size, intermediate_size=g.intermediate_size,
                     num_hidden_layers=g.num_hidden_layers, num_attention_heads=g.num_attention_heads,
                     num_key_value_heads=g.num_key_value_heads, vocab_size=g.vocab_size, rms_norm_eps=g.rms_norm_eps,
                     rope_theta=g.rope_theta, sliding_window=g.sliding_window, max_position_embeddings=4096,
                     pad_token_id=0, bos_token_id=1, eos_token_id=2, attn_implementation="eager")
    m = Phi3ForCausalLM(cfg).eval()
    dec = {k: v for k, v in sd.items() if k.startswith("model.layers.") or k in
           ("model.embed_tokens.weight", "model.norm.weight", "lm_head.weight")}
    res = m.load_state_dict(dec, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return m


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("window", [WINDOW, None])
def test_oracle_matches_hf_phi3(window):
    """Prefill over 40 positions (window 24 crossed) and 12 cached decode steps past it: the restatement and HF
    Phi3ForCausalLM agree to 1e-4 relative error; the window changes the logits (it is not a no-op here)."""
    torch.manual_seed(0)
    g = tiny_phi3_geometry(window)
    sd = fp32_sd(g, seed=11)
    hf = _hf_phi3(g, sd)
    gen = torch.Generator().manual_seed(3)
    emb = torch.randn(2, 52, g.hidden_size, generator=gen) * 0.5
    with torch.no_grad():
        ref = hf(inputs_embeds=emb[:, :40]).logits
        got, past = P3.decoder_forward(sd, emb[:, :40], g)
        assert _rel(got, ref) < 1e-4
        out = hf(inputs_embeds=emb[:, :40], use_cache=True)
        cache = out.past_key_values
        for t in range(40, 52):
            out = hf(inputs_embeds=emb[:, t:t + 1], past_key_values=cache, use_cache=True)
            cache = out.past_key_values
            got, past = P3.decoder_forward(sd, emb[:, t:t + 1], g, past)
            assert _rel(got[:, -1], out.logits[:, -1]) < 1e-4, t
        if window:
            full, _ = P3.decoder_forward(sd, emb[:, :40], tiny_phi3_geometry(None))
            assert _rel(full[:, -1], ref[:, -1]) > 1e-2


def test_full_model_matches_reference_phi3():
    """forward() logits and greedy generate() ids of the reference's own u2Phi3ForCausalLM (imported unmodified, MONAI
    stand-in) equal the Phi-3 restatement's, with the window (24) crossed by the prompt: pins the wrapper, the splice and
    the generate contract. Under transformers 5.5 the reference's generate() raises (reference defect, SURVEY.md F9):
    Phi3ForCausalLM.prepare_inputs_for_generation passes `logits_to_keep`, which u2Phi3ForCausalLM.forward does not
    accept; a test-local subclass drops it."""
    import refshim
    from oracle import u2_oracle as O
    g = tiny_phi3_geometry()
    sd = fp32_sd(g, seed=7)
    from u2tokenizer_b200.synthetic import synthetic_inputs
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=20, lt=24, im_patch_id=g.vocab_size - 2)
    assert ids.shape[1] > WINDOW

    def reference():
        refshim.install()
        from src.model.language_model.u2phi3 import u2Phi3Config, u2Phi3ForCausalLM
        from u2tokenizer_b200.configuration import MM_DEFAULTS

        class Phi3DropsLogitsToKeep(u2Phi3ForCausalLM):
            def forward(self, *a, logits_to_keep=None, **k):
                return super().forward(*a, **k)

        cfg = u2Phi3Config(hidden_size=g.hidden_size, intermediate_size=g.intermediate_size,
                           num_hidden_layers=g.num_hidden_layers, num_attention_heads=g.num_attention_heads,
                           num_key_value_heads=g.num_key_value_heads, vocab_size=g.vocab_size, rms_norm_eps=g.rms_norm_eps,
                           max_position_embeddings=4096, sliding_window=WINDOW, pad_token_id=0, bos_token_id=1,
                           eos_token_id=2, tie_word_embeddings=False)
        for k, v in MM_DEFAULTS.items():
            setattr(cfg, k, v)
        cfg.image_size, cfg.patch_size = g.image_size, g.patch_size
        cfg.u2t_num_layers, cfg.u2t_top_k, cfg.num_3d_query_token = g.u2t_num_layers, g.u2t_top_k, g.num_3d_query_token
        cfg.mm_hidden_size = g.vit_hidden
        torch.manual_seed(0)
        import src.model.multimodal_encoder.vit as refvit
        orig = refvit.ViT.__init__

        def small_init(self, *a, **kw):
            kw.update(hidden_size=g.vit_hidden, mlp_dim=g.vit_mlp, num_layers=g.vit_layers, num_heads=g.vit_heads)
            orig(self, *a, **kw)
        refvit.ViT.__init__ = small_init
        try:
            model = Phi3DropsLogitsToKeep(cfg)
            from src.model.u2tokenizer.builder import build_u2tokenizer_tower
            model.get_model().u2tokenizer = build_u2tokenizer_tower(cfg)
        finally:
            refvit.ViT.__init__ = orig
        res = model.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys, res.unexpected_keys
        assert all("rotary" in k or "inv_freq" in k for k in res.missing_keys), res.missing_keys
        model.eval().float()
        with torch.no_grad():
            logits = model(images=images, input_ids=ids, question_ids=qids).logits
            gen_ids = model.generate(images, ids, question_ids=qids, max_new_tokens=6, do_sample=False)
        return {"logits": logits, "ids": gen_ids[:, -6:]}
    want, _ = refshim.pinned("full_model_phi3", reference)
    with torch.no_grad():
        emb = O.multimodal_embeds(sd, ids, images, qids, g)
        got = P3.decoder_forward(sd, emb, g)[0]
        assert ((got - want["logits"]).abs().max() / want["logits"].abs().max()).item() < 1e-4
        got_ids, _ = P3.greedy_from_embeds(sd, emb, g, 6)
    assert torch.equal(got_ids, want["ids"])
