"""Checkpoint directories in the reference's HF remote-code layout (SURVEY.md §8f-3).

The reference ships / trains checkpoints as a HuggingFace directory whose ``config.json`` carries an ``auto_map``
pointing at two python files stored next to the weights
(base_model_tokenizers/Llama-3.2-1B-Instruct/config.json:1-8: ``configuration_u2.u2Config`` and
``modeling_u2Llama.u2LlamaForCausalLM``) and loads them with
``AutoModelForCausalLM.from_pretrained(path, trust_remote_code=True)`` (src/train/train_stage2.py:145-152,
eval/mrg.py:42-45). The state-dict keys of those classes are the ones ``modeling.py`` reproduces, so switching a
checkpoint directory to the H100 path means replacing the two python files by thin shims that re-export the classes of
this package under the reference's file and class names; the weights, tokenizer files and ``config.json`` stay as
they are. ``write_remote_code`` does exactly that; ``save_pretrained`` writes a complete directory from a model.
"""
from __future__ import annotations

import json
import os

# family -> (model file stem, model class name in the shim, package class, config package class)
_FAMILIES = {
    "llama": ("modeling_u2Llama", "u2LlamaForCausalLM", "U2LlamaForCausalLM", "U2LlamaConfig"),
    "qwen3": ("modeling_u2Qwen3", "u2Qwen3ForCausalLM", "U2Qwen3ForCausalLM", "U2Qwen3Config"),
    "phi3": ("modeling_u2Phi3", "u2Phi3ForCausalLM", "U2Phi3ForCausalLM", "U2Phi3Config"),
}
_MODEL_TYPES = {"u2llama": "llama", "u2Qwen3": "qwen3", "u2phi3": "phi3"}
_CONFIG_STEM, _CONFIG_CLASS = "configuration_u2", "u2Config"

_CONFIG_SHIM = '''"""Remote-code shim: the configuration class of the H100 path under the reference's name
(replaces the reference's configuration_u2.py in a checkpoint directory)."""
from u2tokenizer_b200.configuration import {cfg} as _Base


class u2Config(_Base):
    pass
'''

_MODEL_SHIM = '''"""Remote-code shim: the H100 implementation under the reference's module / class name
(replaces the reference's {stem}.py in a checkpoint directory; same state-dict keys, same forward / generate)."""
from u2tokenizer_b200.modeling import {pkg_cls} as _Base

from .configuration_u2 import u2Config


class {cls}(_Base):
    config_class = u2Config
'''


def family_of(config_or_model) -> str:
    mt = getattr(getattr(config_or_model, "config", config_or_model), "model_type", "")
    if mt in _MODEL_TYPES:
        return _MODEL_TYPES[mt]
    raise ValueError(f"not a mu2 configuration (model_type={mt!r}; expected one of {sorted(_MODEL_TYPES)})")


def write_remote_code(directory: str, family: str | None = None) -> dict:
    """Write the two shim files into ``directory`` and point ``config.json``'s ``auto_map`` / ``architectures`` at
    them. ``family`` defaults to what ``config.json``'s ``model_type`` says. Returns the ``auto_map`` written."""
    cfg_path = os.path.join(directory, "config.json")
    if not os.path.isfile(cfg_path):
        raise FileNotFoundError(f"{cfg_path}: a checkpoint directory needs a config.json")
    with open(cfg_path) as f:
        cfg = json.load(f)
    if family is None:
        family = _MODEL_TYPES.get(cfg.get("model_type"))
    if family not in _FAMILIES:
        raise ValueError(f"unknown family {family!r} (config.json model_type={cfg.get('model_type')!r})")
    stem, cls, pkg_cls, pkg_cfg = _FAMILIES[family]
    with open(os.path.join(directory, _CONFIG_STEM + ".py"), "w") as f:
        f.write(_CONFIG_SHIM.format(cfg=pkg_cfg))
    with open(os.path.join(directory, stem + ".py"), "w") as f:
        f.write(_MODEL_SHIM.format(stem=stem, pkg_cls=pkg_cls, cls=cls))
    auto_map = {"AutoConfig": f"{_CONFIG_STEM}.{_CONFIG_CLASS}", "AutoModelForCausalLM": f"{stem}.{cls}"}
    cfg["auto_map"] = auto_map
    cfg["architectures"] = [cls]
    with open(cfg_path, "w") as f:
        json.dump(cfg, f, indent=2, sort_keys=True)
        f.write("\n")
    return auto_map


def save_pretrained(model, directory: str, safe_serialization: bool = True) -> None:
    """``model.save_pretrained`` + the remote-code shims: the directory then loads with
    ``AutoModelForCausalLM.from_pretrained(directory, trust_remote_code=True)`` exactly like a reference checkpoint."""
    os.makedirs(directory, exist_ok=True)
    model.save_pretrained(directory, safe_serialization=safe_serialization)
    write_remote_code(directory, family_of(model))


def load_reference_state_dict(path: str) -> dict:
    """Read the tensors of a reference checkpoint file or directory (``pytorch_model.bin`` as written by the
    reference's trainer, src/train/sft_u2Trainer.py:11-30, sharded ``*.safetensors`` / ``*.bin`` with an index, or a
    single file). Keys are returned unchanged: they are the keys this package's modules use."""
    import torch

    def read(fp):
        if fp.endswith(".safetensors"):
            from safetensors.torch import load_file
            return load_file(fp)
        return torch.load(fp, map_location="cpu", weights_only=True)

    if os.path.isfile(path):
        return read(path)
    for index in ("model.safetensors.index.json", "pytorch_model.bin.index.json"):
        ip = os.path.join(path, index)
        if os.path.isfile(ip):
            with open(ip) as f:
                shards = sorted(set(json.load(f)["weight_map"].values()))
            sd = {}
            for s in shards:
                sd.update(read(os.path.join(path, s)))
            return sd
    for single in ("model.safetensors", "pytorch_model.bin"):
        fp = os.path.join(path, single)
        if os.path.isfile(fp):
            return read(fp)
    raise FileNotFoundError(f"no weights found under {path}")
