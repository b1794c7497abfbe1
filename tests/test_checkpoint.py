"""HF remote-code checkpoint layout (SURVEY.md §8f-3): a directory written by `checkpoint.save_pretrained` loads through
`AutoModelForCausalLM.from_pretrained(dir, trust_remote_code=True)` — the call the reference's stage-2 trainer and eval
scripts make (train_stage2.py:145-152, eval/mrg.py:42-45) — with identical keys, tensors and multimodal config."""
import json
import os
import sys

import pytest
import torch

from u2tokenizer_b200 import checkpoint
from u2tokenizer_b200.configuration import U2LlamaConfig, U2Qwen3Config
from u2tokenizer_b200.geometry import Geometry
from u2tokenizer_b200.modeling import U2LlamaForCausalLM, U2Qwen3ForCausalLM
from u2tokenizer_b200.synthetic import synthetic_state_dict

KW = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
          head_dim=32, vocab_size=512, image_size=[16, 64, 64], vit_hidden_size=96, vit_mlp_dim=192, vit_num_layers=2,
          vit_num_heads=4, u2t_num_layers=2, u2t_top_k=8, num_3d_query_token=8, tie_word_embeddings=False,
          rms_norm_eps=1e-6, attn_type="rope", enable_diffts=False)


def build(family):
    cfg = (U2Qwen3Config if family == "qwen3" else U2LlamaConfig)(**KW)
    model = (U2Qwen3ForCausalLM if family == "qwen3" else U2LlamaForCausalLM)(cfg)
    sd = synthetic_state_dict(Geometry.from_hf(cfg), seed=3, device="cpu", dtype=torch.bfloat16)
    res = model.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    return model.to(torch.bfloat16), sd


@pytest.fixture
def hf_modules(tmp_path, monkeypatch):
    """Keep HF's dynamic-module cache inside the test's temp directory."""
    import transformers.dynamic_module_utils as dmu
    cache = tmp_path / "hf_modules"
    monkeypatch.setattr(dmu, "HF_MODULES_CACHE", str(cache))
    monkeypatch.setattr(sys, "path", list(sys.path))
    return cache


@pytest.mark.parametrize("family", ["llama", "qwen3"])
def test_remote_code_round_trip(family, tmp_path, hf_modules):
    from transformers import AutoConfig, AutoModelForCausalLM
    model, sd = build(family)
    d = str(tmp_path / "ckpt")
    checkpoint.save_pretrained(model, d)
    stem, cls = {"llama": ("modeling_u2Llama", "u2LlamaForCausalLM"), "qwen3": ("modeling_u2Qwen3", "u2Qwen3ForCausalLM")}[family]
    cfg_json = json.load(open(os.path.join(d, "config.json")))
    assert cfg_json["auto_map"] == {"AutoConfig": "configuration_u2.u2Config", "AutoModelForCausalLM": f"{stem}.{cls}"}
    assert cfg_json["architectures"] == [cls]
    assert os.path.isfile(os.path.join(d, "configuration_u2.py")) and os.path.isfile(os.path.join(d, stem + ".py"))
    cfg = AutoConfig.from_pretrained(d, trust_remote_code=True)
    # (HF resolves to the remote shim or, when the package already registered the model_type, to the package class:
    #  both are the same implementation)
    assert isinstance(cfg, U2Qwen3Config if family == "qwen3" else U2LlamaConfig)
    assert cfg.attn_type == "rope" and cfg.enable_diffts is False
    assert list(cfg.image_size) == [16, 64, 64] and cfg.num_3d_query_token == 8
    # the shim files themselves import and expose the reference's class names
    from transformers.dynamic_module_utils import get_class_from_dynamic_module
    shim_cls = get_class_from_dynamic_module(f"{stem}.{cls}", d)
    assert shim_cls.__name__ == cls and issubclass(shim_cls, U2Qwen3ForCausalLM if family == "qwen3" else U2LlamaForCausalLM)
    assert shim_cls.config_class.__name__ == "u2Config"
    loaded = AutoModelForCausalLM.from_pretrained(d, trust_remote_code=True, dtype=torch.bfloat16)
    assert isinstance(loaded, U2Qwen3ForCausalLM if family == "qwen3" else U2LlamaForCausalLM)
    a, b = model.state_dict(), loaded.state_dict()
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # the surface the reference's scripts touch right after loading (train_stage1.py:369, u2_arch.py:26-32)
    assert loaded.get_model().mm_projector.proj_out_num == model.get_model().mm_projector.proj_out_num > 0
    assert loaded.get_vision_tower() is not None and loaded.get_u2tokenizer() is not None


def test_reference_config_json_is_understood(tmp_path, hf_modules):
    """A config.json with the reference's own field names (enable_rpe instead of attn_type, extra segmentation fields,
    base_model_tokenizers/Llama-3.2-1B-Instruct/config.json) resolves to the H100 classes once the shims are written."""
    from transformers import AutoConfig
    ref_like = dict(KW)
    ref_like.pop("attn_type")
    ref_like.update(model_type="u2llama", architectures=["u2LlamaForCausalLM"], enable_rpe=True, seg_token_id=32003,
                    segmentation_module=None, mm_projector_type="spp", proj_layer_type="mlp", proj_layer_num=2,
                    auto_map={"AutoConfig": "configuration_u2.u2Config", "AutoModelForCausalLM": "modeling_u2Llama.u2LlamaForCausalLM"})
    d = tmp_path / "ref_ckpt"
    d.mkdir()
    (d / "config.json").write_text(json.dumps(ref_like))
    am = checkpoint.write_remote_code(str(d))
    assert am["AutoModelForCausalLM"] == "modeling_u2Llama.u2LlamaForCausalLM"
    cfg = AutoConfig.from_pretrained(str(d), trust_remote_code=True)
    assert cfg.attn_type == "rma" and cfg.model_type == "u2llama" and cfg.seg_token_id == 32003
    assert Geometry.from_hf(cfg).attn_type == "rma"


def test_load_reference_state_dict_formats(tmp_path):
    from safetensors.torch import save_file
    _, sd = build("qwen3")
    sd = {k: v.contiguous() for k, v in sd.items()}
    # (1) a single pytorch_model.bin, as the reference's trainer writes it (sft_u2Trainer.py:11-30)
    d1 = tmp_path / "bin"
    d1.mkdir()
    torch.save(sd, d1 / "pytorch_model.bin")
    got = checkpoint.load_reference_state_dict(str(d1))
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    # (2) sharded safetensors with an index
    d2 = tmp_path / "sharded"
    d2.mkdir()
    keys = sorted(sd)
    half = len(keys) // 2
    shards = {"model-00001-of-00002.safetensors": keys[:half], "model-00002-of-00002.safetensors": keys[half:]}
    wm = {}
    for name, ks in shards.items():
        save_file({k: sd[k] for k in ks}, str(d2 / name))
        wm.update({k: name for k in ks})
    (d2 / "model.safetensors.index.json").write_text(json.dumps({"metadata": {}, "weight_map": wm}))
    got = checkpoint.load_reference_state_dict(str(d2))
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    # (3) a bare file path
    got = checkpoint.load_reference_state_dict(str(d1 / "pytorch_model.bin"))
    assert set(got) == set(sd)
    with pytest.raises(FileNotFoundError):
        checkpoint.load_reference_state_dict(str(tmp_path))
