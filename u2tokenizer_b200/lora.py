"""LoRA on the decoder: a drop-in for the two peft names the reference uses (src/train/train_stage1.py:217-227, 342-359;
evalscipt/ourmodel_ctrate.py:77-110), so that

    from u2tokenizer_b200.lora import LoraConfig, get_peft_model

is the only change its stage-1 and eval code need.

`get_peft_model` rebuilds the targeted decoder linears in PEFT's module layout (`<name>.base_layer`,
`<name>.lora_A.default`, `<name>.lora_B.default`, `<name>.lora_dropout.default`), so `state_dict()` keys and a saved
`model_with_lora.bin` are those of a PEFT model. The modules hold parameters only: a training forward runs on
TrainEngine's LoRA path (train.py), an inference forward / generate() on U2Engine built from the merged weights
W + s B A (computed on the GPU with the GEMM), so LoRA costs nothing per decoded token.
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field
from typing import Optional, Sequence, Union

import torch
import torch.nn as nn

from .train import LORA_TARGETS, PHI3_LORA_TARGETS, LoraSpec, lora_groups, lora_targets

_TARGET_RE = re.compile(r"model\.layers\.(\d+)\.(self_attn|mlp)\.(" + "|".join(LORA_TARGETS + PHI3_LORA_TARGETS) + r")$")


@dataclass
class LoraConfig:
    """The fields of peft.LoraConfig the reference sets. scaling = lora_alpha / r."""
    r: int = 8
    lora_alpha: int = 8
    target_modules: Optional[Union[Sequence[str], str]] = None
    lora_dropout: float = 0.0
    bias: str = "none"
    task_type: Optional[str] = None
    use_rslora: bool = False
    use_dora: bool = False
    modules_to_save: Optional[Sequence[str]] = None
    init_lora_weights: Union[bool, str] = True
    peft_type: str = field(default="LORA", init=False)

    def __post_init__(self):
        if self.bias != "none":
            raise NotImplementedError(f"LoraConfig(bias={self.bias!r}): only bias='none' is supported")
        if self.use_rslora:
            raise NotImplementedError("LoraConfig(use_rslora=True) is not supported")
        if self.use_dora:
            raise NotImplementedError("LoraConfig(use_dora=True) is not supported")
        if self.modules_to_save:
            raise NotImplementedError("LoraConfig(modules_to_save=...) is not supported: set requires_grad on those "
                                      "parameters instead, as the reference does")
        if self.init_lora_weights is not True:
            raise NotImplementedError(f"LoraConfig(init_lora_weights={self.init_lora_weights!r}): only the default "
                                      "initialisation (A kaiming-uniform, B zeros) is supported")
        if isinstance(self.target_modules, (list, tuple, set)):
            self.target_modules = set(self.target_modules)

    @property
    def scaling(self) -> float:
        return self.lora_alpha / self.r


class LoraLinear(nn.Module):
    """PEFT's lora.Linear parameter layout around a decoder nn.Linear. It computes nothing itself."""

    def __init__(self, base: nn.Linear, r: int, lora_alpha: float, lora_dropout: float):
        super().__init__()
        self.base_layer = base
        w = base.weight
        self.lora_A = nn.ModuleDict({"default": nn.Linear(base.in_features, r, bias=False, device=w.device, dtype=w.dtype)})
        self.lora_B = nn.ModuleDict({"default": nn.Linear(r, base.out_features, bias=False, device=w.device, dtype=w.dtype)})
        self.lora_dropout = nn.ModuleDict({"default": nn.Dropout(lora_dropout) if lora_dropout > 0 else nn.Identity()})
        self.scaling = {"default": lora_alpha / r}
        # peft LoraLayer.reset_lora_parameters with init_lora_weights=True
        with torch.no_grad():
            a = torch.empty(r, base.in_features, dtype=torch.float32, device=w.device)
            nn.init.kaiming_uniform_(a, a=math.sqrt(5))
            self.lora_A["default"].weight.copy_(a)
            nn.init.zeros_(self.lora_B["default"].weight)

    def forward(self, *a, **k):
        raise RuntimeError("LoRA parameter container: the computation runs in the CUDA engines, not in this module")


def _matches(name: str, targets) -> bool:
    """peft check_target_module_exists: a regex full match for a string, else an exact or '.'-suffix match."""
    if isinstance(targets, str):
        return re.fullmatch(targets, name) is not None
    return name in targets or any(name.endswith("." + t) for t in targets)


def _resolve_targets(model: nn.Module, config: LoraConfig):
    """Names of the modules `config.target_modules` selects; anything but a decoder q/k/v/o/gate/up/down_proj
    (Phi-3: qkv/o/gate_up/down_proj) raises."""
    if not config.target_modules:
        raise ValueError("LoraConfig.target_modules must name the modules to adapt (the reference passes "
                         "find_all_linear_names(model))")
    found = [n for n, _ in model.named_modules() if n and _matches(n, config.target_modules)]
    if not found:
        raise ValueError(f"Target modules {config.target_modules} not found in the base model")
    from .geometry import Geometry
    g = Geometry.from_hf(model.config)
    targets = lora_targets(g)
    for n in found:
        m = _TARGET_RE.fullmatch(n)
        if not m or m.group(3) not in targets or not isinstance(model.get_submodule(n), nn.Linear):
            raise NotImplementedError(f"LoRA on {n!r} is not supported: only the decoder's {'/'.join(targets)} "
                                      "linears can carry adapters")
    layers = {}
    for n in found:
        m = _TARGET_RE.fullmatch(n)
        layers.setdefault(int(m.group(1)), set()).add(m.group(3))
    kinds = set().union(*layers.values())
    n_layers = model.config.num_hidden_layers
    if len(layers) != n_layers or any(v != kinds for v in layers.values()):
        raise NotImplementedError("LoRA targets must be the same projections on every decoder layer")
    for _, members in lora_groups(g):
        part = kinds.intersection(members)
        if part and len(part) != len(members):
            raise NotImplementedError(f"LoRA on {sorted(part)} without the rest of its fused group {list(members)} is not "
                                      "supported")
    return found, tuple(t for t in targets if t in kinds)


class LoraModel(nn.Module):
    """peft.LoraModel: holds the adapted model as `.model` (state-dict prefix `base_model.model.`)."""

    def __init__(self, model: nn.Module):
        super().__init__()
        self.model = model

    def forward(self, *a, **k):
        return self.model(*a, **k)


class PeftModelForCausalLM(nn.Module):
    """What get_peft_model returns: forward / generate / per_token_logps of the wrapped U2*ForCausalLM, PEFT's parameter
    names, merge_and_unload() and print_trainable_parameters()."""

    def __init__(self, model: nn.Module, config: LoraConfig):
        super().__init__()
        self.peft_config = {"default": config}
        self.active_adapter = "default"
        self.base_model = LoraModel(model)

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self.base_model.model, name)

    def forward(self, *a, **k):
        return self.base_model.model(*a, **k)

    @torch.no_grad()
    def generate(self, *a, **k):
        return self.base_model.model.generate(*a, **k)

    def get_base_model(self):
        return self.base_model.model

    def get_nb_trainable_parameters(self):
        trainable = sum(p.numel() for p in self.parameters() if p.requires_grad)
        return trainable, sum(p.numel() for p in self.parameters())

    def print_trainable_parameters(self):
        trainable, total = self.get_nb_trainable_parameters()
        print(f"trainable params: {trainable:,d} || all params: {total:,d} || trainable%: {100 * trainable / total:.4f}")

    def merge_and_unload(self):
        """Fold s B A into every base weight (on the GPU) and return the plain U2*ForCausalLM without adapter modules."""
        model = self.base_model.model
        merged = merged_weights(model)
        for n, mod in list(model.named_modules()):
            if isinstance(mod, LoraLinear):
                parent, _, child = n.rpartition(".")
                base = mod.base_layer
                base.weight = nn.Parameter(merged[n + ".weight"], requires_grad=base.weight.requires_grad)
                setattr(model.get_submodule(parent), child, base)
        _set_lora(model, None)
        return model


def _set_lora(model: nn.Module, spec: Optional[LoraSpec]):
    """Attach (or drop) the adapter description the engines read; engines built for the other layout are dropped."""
    if spec is None:
        model.__dict__.pop("_u2_lora", None)
    else:
        model.__dict__["_u2_lora"] = spec
    model.__dict__.pop("_u2_train_engine", None)
    model.invalidate_engine()


def merged_weights(model: nn.Module) -> dict:
    """{'<target>.weight': W + s * B @ A} (bf16, on the GEMM: alpha = s, residual = W) for every LoRA module."""
    from . import ops
    out = {}
    for n, mod in model.named_modules():
        if not isinstance(mod, LoraLinear):
            continue
        W = mod.base_layer.weight.detach()
        A, B = mod.lora_A["default"].weight.detach(), mod.lora_B["default"].weight.detach()
        if not W.is_cuda:
            raise RuntimeError("merging LoRA weights runs on CUDA only (model.cuda()); there is no CPU fallback")
        W, A, B = (t.to(torch.bfloat16).contiguous() for t in (W, A, B))
        out_f, in_f = W.shape
        Wm = torch.empty_like(W)
        ops.gemm(B, A, Wm, M=out_f, N=in_f, K=A.shape[0], lda=B.stride(0), ldb=A.stride(0), ldc=in_f, b_mn=True,
                 alpha=mod.scaling["default"], residual=W, ldr=in_f)
        out[n + ".weight"] = Wm
    return out


def merged_state_dict(model: nn.Module) -> dict:
    """The model's state dict in the plain (unadapted) layout with every LoRA target merged: what U2Engine is built from."""
    merged = merged_weights(model)
    sd = {}
    for k, v in model.state_dict().items():
        if ".lora_A." in k or ".lora_B." in k:
            continue
        if ".base_layer." in k:
            k = k.replace(".base_layer.", ".")
            v = merged.get(k, v)
        sd[k] = v
    return sd


def get_peft_model(model: nn.Module, config: LoraConfig) -> PeftModelForCausalLM:
    """peft.get_peft_model for a U2*ForCausalLM: adapters on the targeted decoder linears, their base weights frozen.
    Every other parameter keeps its requires_grad flag."""
    from .modeling import U2MetaForCausalLM
    if not isinstance(model, U2MetaForCausalLM):
        raise NotImplementedError("get_peft_model supports the U2*ForCausalLM models of this package")
    if model.__dict__.get("_u2_lora") is not None:
        raise NotImplementedError("the model already carries LoRA adapters (one adapter per model is supported)")
    if config.r not in (8, 16, 32, 64):
        raise NotImplementedError(f"LoRA rank r={config.r}: the CUDA path supports r in (8, 16, 32, 64)")
    if not 0.0 <= config.lora_dropout < 1.0:
        raise ValueError(f"lora_dropout must lie in [0, 1), got {config.lora_dropout}")
    names, kinds = _resolve_targets(model, config)
    for n in names:
        parent, _, child = n.rpartition(".")
        base = model.get_submodule(n)
        base.weight.requires_grad_(False)
        setattr(model.get_submodule(parent), child, LoraLinear(base, config.r, config.lora_alpha, config.lora_dropout))
    _set_lora(model, LoraSpec(r=config.r, scaling=config.scaling, dropout=float(config.lora_dropout), targets=kinds))
    return PeftModelForCausalLM(model, config)
