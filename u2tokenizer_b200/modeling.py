"""HuggingFace-style module surface of the hot path (the drop-in boundary).

Mirrors the reference classes

    u2LlamaForCausalLM(u2MetaForCausalLM, LlamaForCausalLM)   src/model/language_model/u2llama.py:25-142
    u2Qwen3ForCausalLM (Llama-style contract, SURVEY.md F4)    src/model/language_model/u2qwen3.py:25-145
    u2Phi3ForCausalLM(u2MetaForCausalLM, Phi3ForCausalLM)     src/model/language_model/u2phi3.py:25-140
    u2MetaModel / u2MetaForCausalLM                            src/model/u2_arch.py:10-164

with the same constructor / forward() / generate() / get_model() / initialize_vision_modules() /
initialize_vision_tokenizer() signatures, the same state-dict keys (so reference checkpoints load with
load_state_dict) and the same Auto* registration. The modules below only HOLD parameters; every
forward computation is dispatched to `U2Engine` (hand-written sm_90a kernels behind the C ABI).
Running them without CUDA / without libu2b200.so raises - there is no PyTorch fallback.
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn as nn
from transformers import (AutoConfig, AutoModelForCausalLM, LlamaForCausalLM, LlamaModel, Phi3ForCausalLM, Phi3Model,
                          Qwen3ForCausalLM, Qwen3Model)
from transformers.generation import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput
from transformers.modeling_outputs import CausalLMOutputWithPast

from . import _lib
from .configuration import U2LlamaConfig, U2Phi3Config, U2Qwen3Config
from .geometry import Geometry
from .synthetic import param_shapes


# ------------------------------------------------------------------------------------------------
# parameter containers with the reference's module / parameter names
# ------------------------------------------------------------------------------------------------
class ParamTree(nn.Module):
    """A nested container of nn.Parameters addressed by dotted names (state-dict compatible with the
    reference modules). It computes nothing: `forward` raises."""

    def add_param(self, dotted: str, shape, dtype=None, device=None):
        head, _, rest = dotted.partition(".")
        if not rest:
            self.register_parameter(head, nn.Parameter(torch.zeros(shape, dtype=dtype, device=device)))
            return
        child = self._modules.get(head)
        if child is None:
            child = ParamTree()
            self.add_module(head, child)
        child.add_param(rest, shape, dtype, device)

    def forward(self, *a, **k):
        raise RuntimeError("parameter container: the computation runs in U2Engine (CUDA), not in this module")


class ViT3DTowerParams(ParamTree):
    """Stands where the reference's ViT3DTower stands (multimodal_encoder/vit.py:132-175)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.select_layer = config.vision_select_layer
        self.select_feature = config.vision_select_feature
        self._hidden = getattr(config, "vit_hidden_size", 768)

    @property
    def hidden_size(self):
        return self._hidden


class SpatialPoolingProjectorParams(ParamTree):
    """Stands where SpatialPoolingProjector stands (multimodal_projector/spatial_pooling_projector.py:7-58)."""

    def __init__(self, geom: Geometry):
        super().__init__()
        self._n = geom.tokens_per_frame

    @property
    def proj_out_num(self):
        return self._n


def _build_param_modules(config, which: str, dtype=None, device=None) -> nn.Module:
    g = Geometry.from_hf(config)
    shapes = param_shapes(g)
    prefix = {"vision_tower": "model.vision_tower.", "mm_projector": "model.mm_projector.",
              "u2tokenizer": "model.u2tokenizer."}[which]
    if which == "vision_tower":
        root = ViT3DTowerParams(config)
    elif which == "mm_projector":
        root = SpatialPoolingProjectorParams(g)
    else:
        root = ParamTree()
    for name, shape in shapes.items():
        if name.startswith(prefix):
            root.add_param(name[len(prefix):], shape, dtype, device)
    return root


def build_vision_tower(config, **kw):
    """reference multimodal_encoder/builder.py:4-8"""
    vt = getattr(config, "vision_tower", None)
    if vt is not None and "vit3d" in vt.lower():
        return _build_param_modules(config, "vision_tower", **kw)
    raise ValueError(f"Unknown vision tower: {vt}")


def build_mm_projector(config, **kw):
    """reference multimodal_projector/builder.py:80-99 (only the 'spp' projector is on the hot path)"""
    pt = getattr(config, "mm_projector_type")
    if pt == "spp":
        return _build_param_modules(config, "mm_projector", **kw)
    raise ValueError(f"Unknown projector type: {pt}")


def build_u2tokenizer_tower(config, **kw):
    """reference u2tokenizer/builder.py:3-14"""
    return _build_param_modules(config, "u2tokenizer", **kw)


# ------------------------------------------------------------------------------------------------
# mixins (reference src/model/u2_arch.py)
# ------------------------------------------------------------------------------------------------
class U2MetaModel:
    def __init__(self, config):
        super().__init__(config)
        self.config = config
        if getattr(config, "vision_tower", None) is not None:
            self.vision_tower = build_vision_tower(config)
            self.mm_projector = build_mm_projector(config)
            # the remote-code variant builds the tokenizer from the config too
            # (base_model_tokenizers/.../modeling_u2Llama.py:1728); src/model defers it to
            # initialize_vision_modules - both are supported here.
            if getattr(config, "enable_u2tokenizer", False):
                self.u2tokenizer = build_u2tokenizer_tower(config)

    def get_u2tokenizer(self):
        return getattr(self, "u2tokenizer", None)

    def get_vision_tower(self):
        return getattr(self, "vision_tower", None)

    def initialize_vision_modules(self, model_args):
        """reference u2_arch.py:34-83"""
        c = self.config
        for k in ("image_channel", "image_size", "patch_size", "vision_tower", "vision_select_layer",
                  "vision_select_feature", "mm_projector_type", "proj_layer_type", "proj_layer_num",
                  "proj_pooling_type", "proj_pooling_size", "enable_u2tokenizer", "u2t_num_heads", "u2t_num_layers",
                  "u2t_top_k", "use_multi_scale", "num_3d_query_token", "enable_diffts", "enable_dmtp"):
            setattr(c, k, getattr(model_args, k))
        c.attn_type = getattr(model_args, "attn_type", "rma")
        if self.get_vision_tower() is None:
            self.vision_tower = build_vision_tower(c)
            self.vision_tower.requires_grad_(not model_args.freeze_vision_tower)
        if self.get_u2tokenizer() is None and model_args.enable_u2tokenizer:
            self.u2tokenizer = build_u2tokenizer_tower(c)
        if getattr(model_args, "pretrain_vision_model", None) is not None:
            w = torch.load(model_args.pretrain_vision_model, map_location="cpu")
            w.pop("patch_embedding.cls_token", None)  # unused MONAI buffer in some checkpoints
            self.vision_tower.vision_tower.load_state_dict(w, strict=True)
        c.mm_hidden_size = self.vision_tower.hidden_size
        if getattr(self, "mm_projector", None) is None:
            self.mm_projector = build_mm_projector(c)
        if getattr(model_args, "pretrain_mm_mlp_adapter", None) is not None:
            w = torch.load(model_args.pretrain_mm_mlp_adapter, map_location="cpu")
            self.mm_projector.load_state_dict({k.split("mm_projector.")[1]: v for k, v in w.items() if "mm_projector" in k},
                                              strict=True)


@dataclass
class GenerationOutput:
    """One request's result from generate_batch(), with the field names of HF's continuous-batching output.
    generated_tokens: the new token ids up to and including the first EOS (what generate() returns for the request's
    row before it pads); with num_return_sequences = n > 1, a list of n such lists, sample 0 first.
    logprobs: with generate_batch(return_logprobs=True), one float per generated token (one list per sample when n > 1):
    log_softmax of the scores the token was picked from, at the token; empty otherwise."""
    request_id: str
    prompt_ids: List[int]
    generated_tokens: list
    logprobs: list = field(default_factory=list)


_BATCH_REQUEST_KEYS = ("images", "input_ids", "question_ids", "max_new_tokens", "seed", "request_id")


class U2MetaForCausalLM(ABC):
    @abstractmethod
    def get_model(self):
        ...

    def get_vision_tower(self):
        return self.get_model().get_vision_tower()

    def get_u2tokenizer(self):
        return self.get_model().get_u2tokenizer()

    # ---- engine management --------------------------------------------------------------------
    def engine(self):
        """Build (once) the CUDA engine from this module's current parameters."""
        eng = self.__dict__.get("_u2_engine")
        if eng is not None and self.__dict__.get("_u2_engine_stamp") != self._param_stamp():
            # some parameter changed in place since the engine copied / fused the weights (optimizer step, p.copy_, a
            # re-pointed p.data, a submodule load_state_dict): the fused copies are stale -> rebuild, never serve them
            self.invalidate_engine()
            eng = None
        if eng is None:
            from .engine import U2Engine
            p = next(self.parameters())
            if not p.is_cuda:
                raise RuntimeError("the mu2 hot path runs on CUDA only: move the model to an H100 (model.cuda()); "
                                   "there is no CPU fallback")
            if self.__dict__.get("_u2_lora") is not None:
                from .lora import merged_state_dict
                sd = merged_state_dict(self)   # LoRA: the decode step runs on W + s B A, no per-token adapter work
            else:
                sd = {k: v for k, v in self.state_dict().items()}
            eng = U2Engine(Geometry.from_hf(self.config), sd, device=p.device)
            self.__dict__["_u2_engine"] = eng
            self.__dict__["_u2_engine_stamp"] = self._param_stamp()
            if not self.__dict__.get("_u2_hooks"):
                # submodule.load_state_dict(...) does not pass through this module's load_state_dict override
                for m in self.modules():
                    m.register_load_state_dict_post_hook(lambda mod, keys, root=self: root.invalidate_engine())
                self.__dict__["_u2_hooks"] = True
        return eng

    def _param_stamp(self):
        """(storage address, autograd version counter) of every parameter: in-place updates through the parameter bump
        the counter, `p.data = ...` changes the address. Writers that go through `p.data` IN PLACE (which torch does
        not track) must call invalidate_engine() themselves - parallel.Zero1Step and the training engine do."""
        return tuple((q.data_ptr(), q._version) for q in self.parameters())

    def invalidate_engine(self):
        self.__dict__.pop("_u2_engine", None)
        self.__dict__.pop("_u2_engine_stamp", None)

    # ---- training ---------------------------------------------------------------------------------
    def train_engine(self, **kw):
        """Build (once) the training engine: the parameters move into its flat training-layout buffer and this module's
        nn.Parameters are re-pointed at slices of it (no second copy; the optimizer's in-place updates ARE the engine's
        weights). Group-level requires_grad flags are read from the parameters (freeze_vision_tower / freeze_backbone /
        tune_mm_mlp_adapter of the reference, train_stage1.py:313-332, u2_arch.py:58)."""
        te = self.__dict__.get("_u2_train_engine")
        if te is None:
            from .train import TrainEngine
            p = next(self.parameters())
            if not p.is_cuda:
                raise RuntimeError("the training path runs on CUDA only (model.cuda()); there is no CPU fallback")

            def any_rg(prefix):   # LoRA adapters always train: they do not make their group trainable
                ps = [q for n, q in self.named_parameters() if n.startswith(prefix) and ".lora_" not in n]
                return any(q.requires_grad for q in ps) if ps else False
            flags = dict(vit=any_rg("model.vision_tower."), proj=any_rg("model.mm_projector."), u2t=any_rg("model.u2tokenizer."),
                         dec=any_rg("model.layers.") or any_rg("model.norm."), embed=any_rg("model.embed_tokens."),
                         head=any_rg("lm_head."))
            kw.setdefault("trainable", flags)
            lora = self.__dict__.get("_u2_lora")
            sd = {k.replace(".base_layer.", "."): v for k, v in self.state_dict().items()}
            te = TrainEngine(Geometry.from_hf(self.config), sd, device=p.device, lora=lora, **kw)
            te.bind_module(self)
            self.__dict__["_u2_train_engine"] = te
            self.invalidate_engine()
        return te

    def load_state_dict(self, *a, **k):
        self.invalidate_engine()
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self.invalidate_engine()
        return super()._apply(fn, *a, **k)

    # ---- reference surface ----------------------------------------------------------------------
    def encode_images(self, images):
        """reference u2_arch.py:96-99"""
        return self.engine().encode_images(images)

    def prepare_inputs_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels,
                                      images, question_ids):
        """reference u2_arch.py:101-122 (7 arguments in, 6 values out)."""
        if self.get_vision_tower() is None or images is None or input_ids.shape[1] == 1:
            return input_ids, position_ids, attention_mask, past_key_values, None, labels
        inputs_embeds = self.engine().multimodal_embeds(input_ids, images, question_ids)
        return None, position_ids, attention_mask, past_key_values, inputs_embeds, labels

    def initialize_vision_tokenizer(self, model_args, tokenizer):
        """reference u2_arch.py:124-164"""
        num_new_tokens = model_args.num_new_tokens
        self.resize_token_embeddings(len(tokenizer))
        self.invalidate_engine()
        if num_new_tokens > 0:
            inp = self.get_input_embeddings().weight.data
            out = self.get_output_embeddings().weight.data
            inp[-num_new_tokens:] = inp[:-num_new_tokens].mean(dim=0, keepdim=True)
            out[-num_new_tokens:] = out[:-num_new_tokens].mean(dim=0, keepdim=True)
            for p in self.get_input_embeddings().parameters():
                p.requires_grad = True
            for p in self.get_output_embeddings().parameters():
                p.requires_grad = not model_args.tune_mm_mlp_adapter
        if getattr(model_args, "pretrain_mm_mlp_adapter", None):
            w = torch.load(model_args.pretrain_mm_mlp_adapter, map_location="cpu")
            etw = w["model.embed_tokens.weight"]
            inp = self.get_input_embeddings().weight.data
            if inp.shape == etw.shape:
                inp.copy_(etw)
            elif etw.shape[0] == num_new_tokens:
                inp[-num_new_tokens:] = etw
            else:
                raise ValueError(f"Unexpected embed_tokens_weight shape. Pretrained: {etw.shape}. Current: {inp.shape}. "
                                 f"Numer of new tokens: {num_new_tokens}.")

    @staticmethod
    def _check_right_padded(attention_mask):
        """The fused path has no padding mask: a RIGHT-padded batch is exact under the causal mask (real tokens never
        attend to the pads on their right), anything else (left padding, holes) would silently change the result."""
        if attention_mask is None:
            return
        m = attention_mask.to(torch.bool)
        if m.dim() != 2 or bool((m[:, 1:] & ~m[:, :-1]).any()) or not bool(m[:, 0].all()):
            raise NotImplementedError("attention_mask must be all ones or right-padded (left-padded / sparse masks are "
                                      "not supported by the fused CUDA path)")

    @staticmethod
    def _generate_prompt_rows(input_ids, attention_mask, min_len: int = 1):
        """generate()'s padded batch -> (input_ids with every row's real tokens moved to the front, per-row lengths
        [B] int64 on the CPU). The lengths are None when the mask is absent or all ones (every prompt fills the width).
        A row is right-padded (its ones start at column 0) or left-padded (they end at the last column, as trl's
        collator pads prompts); left padding is rolled to the right BEFORE the visual tokens are spliced at positions
        1..n_vis, so each row sees the positions it would see alone. min_len: <bos> + the visual tokens."""
        if attention_mask is None:
            return input_ids, None
        m = attention_mask.detach().to("cpu", torch.bool)
        if m.dim() != 2 or tuple(m.shape) != tuple(input_ids.shape):
            raise ValueError(f"attention_mask {tuple(m.shape)} does not match input_ids {tuple(input_ids.shape)}")
        if bool(m.all()):
            return input_ids, None
        B, L = m.shape
        lens = m.sum(dim=1)
        col = torch.arange(L)
        right = (m == (col[None, :] < lens[:, None])).all(dim=1)
        left = (m == (col[None, :] >= (L - lens)[:, None])).all(dim=1)
        if not bool((right | left).all()):
            raise NotImplementedError("attention_mask must be all ones, right-padded or left-padded in generate() "
                                      "(masks with holes are not supported by the fused CUDA path)")
        short = (lens < min_len).nonzero().flatten().tolist()
        if short:
            raise ValueError(f"prompt rows {short} have {lens[short].tolist()} tokens: each needs at least {min_len} "
                             "(<bos> + the visual tokens)")
        shift = torch.where(right, torch.zeros_like(lens), L - lens)  # left-padded rows: real tokens start at L - len
        idx = (col[None, :] + shift[:, None]) % L
        ids = input_ids.gather(1, idx.to(input_ids.device))
        return ids, lens

    @staticmethod
    def _generate_logits_processors(kwargs: dict, generation_config, prompt_width: int, eos_token_id, vocab_size: int):
        """generate()'s repetition_penalty, no_repeat_ngram_size, min_new_tokens / min_length and bad_words_ids (popped
        from `kwargs`, else read from `generation_config`) -> a validated engine.LogitsProcessors, or None when every
        value is absent or neutral. HF semantics for generate(inputs_embeds=...): the processors see the generated tokens
        only; min_length counts from the padded prompt width (max(min_length - prompt_width, 0) new tokens) and
        min_new_tokens takes precedence over it; without an EOS id min_new_tokens has nothing to ban. bad_words_ids is
        validated as NoBadWordsLogitsProcessor does, and one-token words equal to an EOS id are dropped first."""
        from .engine import LogitsProcessors, eos_ids

        def opt(name):
            v = kwargs.pop(name, None)
            return getattr(generation_config, name, None) if v is None and generation_config is not None else v

        def count(name, v):
            if v is None:
                return None
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 0:
                raise ValueError(f"`{name}` has to be a non-negative integer, but is {v!r}")
            return int(v)

        pen = opt("repetition_penalty")
        if pen is not None:
            if isinstance(pen, bool) or not isinstance(pen, (int, float, np.floating, np.integer)) or not pen > 0:
                raise ValueError(f"`repetition_penalty` has to be a strictly positive float, but is {pen!r}")
            pen = float(pen)
        ngram = count("no_repeat_ngram_size", opt("no_repeat_ngram_size"))
        min_new = count("min_new_tokens", opt("min_new_tokens"))
        min_len = count("min_length", opt("min_length"))
        if min_new is None:
            min_new = max((min_len or 0) - int(prompt_width), 0)
        eos = eos_ids(eos_token_id)
        bad = opt("bad_words_ids")
        words = ()
        if bad is not None:
            if not isinstance(bad, list) or len(bad) == 0:
                raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bad}.")
            if any(not isinstance(w, list) for w in bad):
                raise ValueError(f"`bad_words_ids` has to be a list of lists, but is {bad}.")
            if any(any(not isinstance(x, (int, np.integer)) or x < 0 for x in w) for w in bad):
                raise ValueError(f"Each list in `bad_words_ids` has to be a list of positive integers, but is {bad}.")
            kept = dict.fromkeys(tuple(int(x) for x in w) for w in bad if all(w != [e] for e in eos))
            if not kept:
                raise ValueError(f"`bad_words_ids` {bad} holds nothing but EOS ids")
            if any(len(w) == 0 for w in kept):
                raise ValueError(f"Each word in `bad_words_ids` needs at least one token, but is {bad}.")
            out = sorted({x for w in kept for x in w if x >= vocab_size})
            if out:
                raise ValueError(f"The model vocabulary size is {vocab_size}, but the following tokens were being "
                                 f"banned: {out}")
            words = tuple(kept)
        # an EOS id outside the vocabulary can never be picked: banning it is a no-op, so it is not sent to the kernel
        eos_in = tuple(dict.fromkeys(e for e in eos if 0 <= e < vocab_size))
        if min_new and len(eos_in) > _lib.LP_MAX_EOS:
            raise ValueError(f"min_new_tokens supports at most {_lib.LP_MAX_EOS} EOS ids, got {len(eos_in)}")
        if len(words) > _lib.LP_MAX_BAD_WORDS or sum(map(len, words)) > _lib.LP_MAX_BAD_TOKENS:
            raise ValueError(f"bad_words_ids holds at most {_lib.LP_MAX_BAD_WORDS} words of {_lib.LP_MAX_BAD_TOKENS} "
                             "tokens in all on the CUDA path")
        pc = LogitsProcessors(repetition_penalty=1.0 if pen is None else pen, no_repeat_ngram_size=ngram or 0,
                              min_new_tokens=min_new if eos_in else 0, eos_token_ids=eos_in if min_new else (),
                              bad_words_ids=words)
        return None if pc.neutral() else pc

    # ---- forward / generate shared by the Llama, Qwen3 and Phi-3 wrappers (reference u2llama.py:41-138) ----
    def _u2_forward(self, images=None, input_ids=None, labels=None, attention_mask=None, question_ids=None,
                    position_ids=None, past_key_values=None, inputs_embeds=None, use_cache=None,
                    output_attentions=None, output_hidden_states=None, return_dict=None, **kwargs):
        if output_attentions or output_hidden_states:
            raise NotImplementedError("attention maps / hidden states are not materialised by the fused path")
        if past_key_values is not None:
            raise NotImplementedError("HF-driven cached decoding is not supported; call generate() "
                                      "(greedy decode runs inside the engine with its own static KV cache)")
        self._check_right_padded(attention_mask)
        if (labels is not None and self.training and torch.is_grad_enabled() and inputs_embeds is None and input_ids is not None
                and any(p.requires_grad for p in self.parameters())):
            # training step (model.train(), reference train_stage1.py:244-250: batch -> model(**batch) -> loss.backward();
            # in eval mode the same call returns loss + logits from the inference path): forward with
            # saved activations on the training engine, backward through ONE autograd node that hands every parameter its
            # gradient (computed by the hand-written backward pass, not by torch autograd)
            te = self.train_engine()
            # gradient_checkpointing_enable() / _disable() set HF's per-module flags; the training tape honours them by
            # recomputing every repeated block in the backward (TrainEngine._segment), from this step on
            te.checkpoint = self.is_gradient_checkpointing
            names, params = zip(*[(n, p) for n, p in self.named_parameters() if p.requires_grad])
            loss = _U2TrainLoss.apply(te, (images, input_ids, question_ids, labels), names, *params)
            if return_dict is False:
                return (loss, None)
            return CausalLMOutputWithPast(loss=loss, logits=None, past_key_values=None)
        eng = self.engine()
        if (inputs_embeds is None and labels is None and images is not None and self.get_vision_tower() is not None
                and input_ids is not None and input_ids.shape[1] != 1):
            # inference-style forward with images: one call into the engine, replayed as a CUDA graph when the shapes repeat
            logits = eng.forward_logits(input_ids, images, question_ids)
            if return_dict is False:
                return (logits,)
            return CausalLMOutputWithPast(loss=None, logits=logits, past_key_values=None)
        if inputs_embeds is None:
            (input_ids, position_ids, attention_mask, past_key_values, inputs_embeds, labels
             ) = self.prepare_inputs_for_multimodal(input_ids, position_ids, attention_mask, past_key_values, labels,
                                                    images, question_ids)
            if inputs_embeds is None:
                inputs_embeds = eng.embed_tokens(input_ids)
        # attention_mask: right-padded batches are exact under the causal mask (real tokens never see the
        # pads to their right); the reference itself drops the mask in generate() (u2llama.py:97-99,123-126)
        hidden = eng.prefill(inputs_embeds.to(torch.bfloat16))
        logits = eng.lm_logits(hidden)
        loss = None
        if labels is not None:
            # HF ForCausalLMLoss (shift by one, mean NLL over labels != -100) on the fused lm_head + log-softmax head:
            # the loss never reads the [B, L, V] logits
            acc = torch.zeros(2, device=hidden.device, dtype=torch.float32)
            shift = labels[:, 1:].to(hidden.device, torch.int64).contiguous()
            eng.token_logps(hidden[:, :-1], shift, nll_acc=acc)
            loss = acc[0] / acc[1]
        if return_dict is False:
            return (loss, logits) if loss is not None else (logits,)
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=None)

    @torch.no_grad()
    def per_token_logps(self, images=None, input_ids=None, question_ids=None, loss_mask=None, attention_mask=None):
        """The log-probability side of `u2DPOTrainer.concatenated_forward` (reference src/train/dpo_u2trainer.py:267-302,
        343-350) without the [B, L, V] logits: labels are `input_ids` rolled left by one, positions whose rolled
        `loss_mask` is 0 contribute 0, the result is rolled back right by one. Returns a dict with `per_token_logps`
        [B, L] fp32, `all_logps` [B] and `mean_logits` (mean of the masked rows' logits, as the trainer logs it)."""
        self._check_right_padded(attention_mask)
        eng = self.engine()
        (_, _, _, _, inputs_embeds, _) = self.prepare_inputs_for_multimodal(input_ids, None, attention_mask, None, None,
                                                                            images, question_ids)
        if inputs_embeds is None:
            inputs_embeds = eng.embed_tokens(input_ids)
        hidden = eng.prefill(inputs_embeds.to(torch.bfloat16))
        ids = input_ids.to(hidden.device, torch.int64)
        if loss_mask is None:
            loss_mask = torch.ones_like(ids)
        labels = torch.roll(ids, shifts=-1, dims=1)
        mask = torch.roll(loss_mask.to(hidden.device), shifts=-1, dims=1).bool()
        labels = labels.masked_fill(~mask, -1)
        logp, _, lsum = eng.token_logps(hidden, labels, want_logit_sum=True)
        ptl = torch.roll(logp, shifts=1, dims=1)
        n = mask.sum().clamp(min=1) * eng.g.vocab_size
        return {"per_token_logps": ptl, "all_logps": ptl.sum(-1), "mean_logits": (lsum * mask).sum() / n}

    @torch.no_grad()
    def _u2_generate(self, images=None, inputs=None, question_ids=None, **kwargs):
        position_ids = kwargs.pop("position_ids", None)
        attention_mask = kwargs.pop("attention_mask", None)
        question_ids = kwargs.pop("question_ids", question_ids)
        if inputs is None:
            inputs = kwargs.pop("input_ids", None)
        if "inputs_embeds" in kwargs:
            raise NotImplementedError("`inputs_embeds` is not supported")
        eng = self.engine()
        # prompts of different lengths: real tokens first, one length per row (the decode runs each row at its own
        # positions); the reference drops the mask here (u2llama.py:97-99) and would decode after the pads
        if inputs is None:
            raise ValueError("generate() needs input_ids")
        splices = images is not None and self.get_vision_tower() is not None and inputs.shape[1] != 1
        n_vis = (eng.g.num_3d_query_token if eng.g.enable_u2tokenizer else eng.g.tokens_per_frame) if splices else 0
        inputs, lengths = self._generate_prompt_rows(inputs, attention_mask, min_len=1 + n_vis)
        if images is not None:
            (inputs, position_ids, attention_mask, _, inputs_embeds, _
             ) = self.prepare_inputs_for_multimodal(inputs, position_ids, attention_mask, None, None, images, question_ids)
            if inputs_embeds is None:
                inputs_embeds = eng.embed_tokens(inputs)
        else:
            inputs_embeds = eng.embed_tokens(inputs)
        gc = getattr(self, "generation_config", None)
        num_beams = kwargs.pop("num_beams", None)
        if num_beams is None:
            num_beams = getattr(gc, "num_beams", None) or 1
        do_sample = kwargs.pop("do_sample", None)
        if do_sample is None:
            do_sample = bool(getattr(gc, "do_sample", False))

        def opt(name, default):
            v = kwargs.pop(name, None)
            if v is None and gc is not None:
                v = getattr(gc, name, None)
            return default if v is None else v
        temperature, top_k, top_p = opt("temperature", 1.0), opt("top_k", 50), opt("top_p", 1.0)
        seed = kwargs.pop("seed", None)
        if seed is None:
            seed = int(torch.initial_seed()) + self.__dict__.setdefault("_u2_sample_calls", 0)
            self.__dict__["_u2_sample_calls"] += 1
        L = inputs_embeds.shape[1]
        max_new = kwargs.pop("max_new_tokens", None)
        if max_new is None:
            max_len = kwargs.pop("max_length", None) or (gc.max_length if gc is not None else 20)
            max_new = max(1, max_len - L)
        from .engine import eos_ids
        eos = kwargs.pop("eos_token_id", None)
        eos = eos_ids(gc.eos_token_id if eos is None and gc is not None else eos)
        pad = kwargs.pop("pad_token_id", None)
        if pad is None and gc is not None:
            pad = gc.pad_token_id
        n_ret = int(opt("num_return_sequences", 1))
        beam = None
        if num_beams != 1:
            beam = self._generate_beam_search(kwargs, gc, num_beams, bool(do_sample), n_ret, pad)
        procs = self._generate_logits_processors(kwargs, gc, L, eos, eng.g.vocab_size)
        return_dict, want_scores, want_logits = self._generate_output_flags(kwargs, gc)
        self._check_remaining_generate_kwargs(kwargs)
        if n_ret > 1 and not do_sample and beam is None:
            raise ValueError("num_return_sequences > 1 needs do_sample=True (greedy decoding is deterministic; HF raises too)")
        ids = eng.generate(inputs_embeds.to(torch.bfloat16), max_new_tokens=max_new, eos_token_id=eos,
                           do_sample=bool(do_sample), temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                           num_return_sequences=n_ret, lengths=lengths, processors=procs, beam=beam,
                           output_scores=want_scores, output_logits=want_logits)
        scores = logits = None
        if want_scores or want_logits:
            ids, scores, logits = ids
        if beam is None:
            ids = self._generate_mask_after_eos(ids, eos, pad)
        if not return_dict:
            return ids
        steps = lambda buf: None if buf is None else tuple(buf[t] for t in range(ids.shape[1]))
        if beam is None:
            return GenerateDecoderOnlyOutput(sequences=ids, scores=steps(scores), logits=steps(logits))
        return GenerateBeamDecoderOnlyOutput(
            sequences=ids, sequences_scores=eng.last_beam_scores.to(ids.device) if want_scores else None,
            scores=steps(scores), logits=steps(logits), beam_indices=eng.last_beam_indices)

    @staticmethod
    def _generate_output_flags(kwargs: dict, generation_config) -> Tuple[bool, bool, bool]:
        """return_dict_in_generate, output_scores and output_logits, popped from `kwargs`, else read from
        `generation_config`. HF keeps scores and logits only in a returned dict, so without it both are False."""
        def flag(name):
            v = kwargs.pop(name, None)
            if v is None and generation_config is not None:
                v = getattr(generation_config, name, None)
            return bool(v)
        return_dict = flag("return_dict_in_generate")
        scores, logits = flag("output_scores"), flag("output_logits")
        return return_dict, scores and return_dict, logits and return_dict

    @staticmethod
    def _generate_mask_after_eos(ids: torch.Tensor, eos, pad) -> torch.Tensor:
        """generate()'s greedy / sampled ids: every position after a row's first EOS becomes pad (eos[0] when pad is
        None), and the columns after the last row's first EOS are dropped, as HF's stopping criteria end the loop."""
        if eos:
            hit = torch.isin(ids, torch.as_tensor(eos, device=ids.device))
            after = (hit.cumsum(dim=1) - hit.long()) > 0  # strictly after the first EOS
            if pad is None:
                pad = eos[0]
            ids = ids.masked_fill(after, pad)
            keep = int((~after).any(dim=0).sum())
            ids = ids[:, :max(keep, 1)]
        return ids  # new tokens only, like HF generate() on inputs_embeds (reference u2llama.py:123-127)

    @torch.no_grad()
    def generate_batch(self, requests, num_slots: Optional[int] = None, **kwargs) -> Dict[str, GenerationOutput]:
        """Continuous batching over many studies: every request runs as if generate() ran it alone, but a decode row
        whose request has finished is refilled with the next queued request instead of idling until its batch ends.
        requests: any iterable of dicts with `images` ([1, C, D, H, W] or [C, D, H, W], CPU or CUDA), `input_ids` ([L]
        or [1, L], unpadded) and optionally `question_ids`, `max_new_tokens`, `seed` and `request_id` (default: the
        request's index as a string); it is read lazily, so only the requests in the decode rows are held.
        num_slots: decode rows in flight (default and maximum: the rows one decode step carries, 16 on the wgmma path).
        kwargs: generate()'s greedy / sampling / num_return_sequences / logits-processor / eos / pad options, and
        return_logprobs (HF's ContinuousBatchingConfig name): each output's `logprobs` then holds the log-prob of every
        generated token, recorded inside the decode step. Request i without a seed samples with seed + i. Returns
        {request_id: GenerationOutput}."""
        eng = self.engine()
        gc = getattr(self, "generation_config", None)
        head = self._generate_batch_head(kwargs, gc, num_slots, eng._decode_rows(), eng.g.vocab_size)
        n_vis = eng.g.num_3d_query_token if eng.g.enable_u2tokenizer else eng.g.tokens_per_frame
        prompts = {}

        def engine_requests():
            from .engine import SlotRequest
            for i, r in enumerate(requests):
                p = self._generate_batch_request(i, r, head["seed"])
                ids, images = p["input_ids"], p["images"]
                if images is not None and self.get_vision_tower() is not None and ids.shape[1] != 1:
                    if ids.shape[1] < 1 + n_vis:
                        raise ValueError(f"request {p['request_id']!r}: {ids.shape[1]} prompt tokens, at least "
                                         f"{1 + n_vis} needed (<bos> + the visual tokens)")
                    emb = eng.multimodal_embeds(ids, images, p["question_ids"])
                else:
                    emb = eng.embed_tokens(ids)
                max_new = p["max_new_tokens"]
                if max_new is None:
                    max_new = head["max_new_tokens"]
                if max_new is None:  # max_length counts the prompt, as in generate()
                    max_new = max(1, head["max_length"] - ids.shape[1])
                prompts[p["request_id"]] = ids[0].tolist()
                yield SlotRequest(p["request_id"], emb.to(torch.bfloat16), int(max_new), p["seed"])

        out = eng.generate_continuous(engine_requests(), head["num_slots"], eos_token_id=head["eos"],
                                      pad_token_id=head["pad"], do_sample=head["do_sample"],
                                      temperature=head["temperature"], top_k=head["top_k"], top_p=head["top_p"],
                                      num_return_sequences=head["n"], processors=head["processors"],
                                      return_logprobs=head["return_logprobs"])
        one = (lambda x: x[0]) if head["n"] == 1 else (lambda x: x)
        if not head["return_logprobs"]:
            return {rid: GenerationOutput(rid, prompts[rid], one(seqs)) for rid, seqs in out.items()}
        return {rid: GenerationOutput(rid, prompts[rid], one([t for t, _ in res]), one([lp for _, lp in res]))
                for rid, res in out.items()}

    def _generate_batch_head(self, kwargs: dict, gc, num_slots, rows: int, vocab_size: int) -> dict:
        """generate_batch()'s options, read and validated by generate()'s helpers and generation_config fallbacks."""
        from .engine import eos_ids
        num_beams = kwargs.pop("num_beams", None)
        if num_beams is None:
            num_beams = getattr(gc, "num_beams", None) or 1
        if num_beams != 1:
            raise NotImplementedError("generate_batch() does not run beam search (num_beams > 1); use generate()")
        do_sample = kwargs.pop("do_sample", None)
        if do_sample is None:
            do_sample = bool(getattr(gc, "do_sample", False))

        def opt(name, default):
            v = kwargs.pop(name, None)
            if v is None and gc is not None:
                v = getattr(gc, name, None)
            return default if v is None else v
        temperature, top_k, top_p = opt("temperature", 1.0), opt("top_k", 50), opt("top_p", 1.0)
        seed = kwargs.pop("seed", None)
        if seed is None:
            seed = int(torch.initial_seed()) + self.__dict__.setdefault("_u2_sample_calls", 0)
            self.__dict__["_u2_sample_calls"] += 1
        max_new = kwargs.pop("max_new_tokens", None)
        max_length = kwargs.pop("max_length", None) or getattr(gc, "max_length", None) or 20
        eos = kwargs.pop("eos_token_id", None)
        eos = eos_ids(gc.eos_token_id if eos is None and gc is not None else eos)
        pad = kwargs.pop("pad_token_id", None)
        if pad is None and gc is not None:
            pad = gc.pad_token_id
        if pad is not None and not isinstance(pad, (int, np.integer)):
            pad = int(torch.as_tensor(pad).reshape(-1)[0])
        n_ret = int(opt("num_return_sequences", 1))
        min_new_set = kwargs.get("min_new_tokens") is not None or getattr(gc, "min_new_tokens", None) is not None
        if not min_new_set and (kwargs.get("min_length") or getattr(gc, "min_length", None) or 0) > 0:
            raise NotImplementedError("generate_batch(): min_length counts each prompt's width; pass min_new_tokens")
        procs = self._generate_logits_processors(kwargs, gc, 0, eos, vocab_size)
        return_logprobs = bool(opt("return_logprobs", False))
        self._check_remaining_generate_kwargs(kwargs)
        if n_ret > 1 and not do_sample:
            raise ValueError("num_return_sequences > 1 needs do_sample=True (greedy decoding is deterministic; HF raises too)")
        S = rows if num_slots is None else num_slots
        if isinstance(S, bool) or not isinstance(S, (int, np.integer)) or not 1 <= S <= rows:
            raise ValueError(f"num_slots={num_slots!r} outside 1..{rows} (the rows one decode step carries)")
        if not 1 <= n_ret <= S:
            raise ValueError(f"num_return_sequences={n_ret} outside 1..num_slots={S}")
        if len(eos) > _lib.LP_MAX_EOS:
            raise ValueError(f"generate_batch() supports at most {_lib.LP_MAX_EOS} EOS ids, got {len(eos)}")
        return dict(num_slots=int(S), n=n_ret, do_sample=bool(do_sample), temperature=temperature, top_k=top_k,
                    top_p=top_p, seed=int(seed), max_new_tokens=max_new, max_length=int(max_length), eos=eos,
                    pad=int(pad) if pad is not None else (eos[0] if eos else 0), processors=procs,
                    return_logprobs=return_logprobs)

    @staticmethod
    def _generate_batch_request(i: int, r, seed: int) -> dict:
        """Request i of generate_batch() -> input_ids [1, L], images [1, C, D, H, W] or None, question_ids, its
        max_new_tokens (None: the call's), its seed (default seed + i) and its id (default str(i))."""
        if not isinstance(r, dict):
            raise TypeError(f"generate_batch(): request {i} must be a dict, got {type(r).__name__}")
        unknown = sorted(set(r) - set(_BATCH_REQUEST_KEYS))
        if unknown:
            raise TypeError(f"generate_batch(): request {i} has unsupported keys {unknown}")
        if r.get("input_ids") is None:
            raise TypeError(f"generate_batch(): request {i} needs input_ids")
        ids = torch.as_tensor(r["input_ids"])
        if ids.dim() == 1:
            ids = ids[None]
        if ids.dim() != 2 or ids.shape[0] != 1 or ids.shape[1] < 1:
            raise ValueError(f"generate_batch(): request {i}: input_ids must be [L] or [1, L], got {tuple(ids.shape)}")
        images = r.get("images")
        if images is not None:
            if images.dim() == 4:
                images = images[None]
            if images.dim() != 5 or images.shape[0] != 1:
                raise ValueError(f"generate_batch(): request {i}: images must be [C, D, H, W] or [1, C, D, H, W], got "
                                 f"{tuple(images.shape)}")
        q = r.get("question_ids")
        if q is not None:
            q = torch.as_tensor(q)
            q = q[None] if q.dim() == 1 else q
        mn = r.get("max_new_tokens")
        if mn is not None and (isinstance(mn, bool) or not isinstance(mn, (int, np.integer)) or mn < 1):
            raise ValueError(f"generate_batch(): request {i}: max_new_tokens must be a positive integer, got {mn!r}")
        s = r.get("seed")
        rid = r.get("request_id")
        return dict(input_ids=ids, images=images, question_ids=q, max_new_tokens=None if mn is None else int(mn),
                    seed=int(seed) + i if s is None else int(s), request_id=str(i) if rid is None else str(rid))

    @staticmethod
    def _generate_beam_search(kwargs: dict, generation_config, num_beams, do_sample: bool, num_return_sequences: int,
                              pad_token_id):
        """num_beams != 1: length_penalty and early_stopping (popped from `kwargs`, else read from `generation_config`)
        -> a validated engine.BeamSearch. Beam sampling, group (diverse) and constrained beam search are refused."""
        from .engine import BeamSearch

        def opt(name, default):
            v = kwargs.pop(name, None)
            if v is None and generation_config is not None:
                v = getattr(generation_config, name, None)
            return default if v is None else v

        if isinstance(num_beams, bool) or not isinstance(num_beams, (int, np.integer)) or num_beams < 1:
            raise ValueError(f"`num_beams` has to be a positive integer, but is {num_beams!r}")
        if do_sample:
            raise NotImplementedError("beam sampling (num_beams > 1 with do_sample=True) is not implemented on the CUDA path")
        if opt("num_beam_groups", 1) != 1:
            raise NotImplementedError("group (diverse) beam search is not implemented on the CUDA path")
        for k in ("constraints", "force_words_ids"):
            if kwargs.pop(k, None):
                raise NotImplementedError(f"constrained beam search ({k}) is not implemented on the CUDA path")
        lp = opt("length_penalty", 1.0)
        if isinstance(lp, bool) or not isinstance(lp, (int, float, np.integer, np.floating)) or not np.isfinite(lp):
            raise ValueError(f"`length_penalty` has to be a finite number, but is {lp!r}")
        es = opt("early_stopping", False)
        if not (es is True or es is False or es == "never"):
            raise ValueError(f"`early_stopping` has to be True, False or 'never', but is {es!r}")
        if num_return_sequences > num_beams:
            raise ValueError(f"`num_return_sequences` ({num_return_sequences}) has to be smaller or equal to "
                             f"`num_beams` ({num_beams}).")
        if pad_token_id is not None and not isinstance(pad_token_id, (int, np.integer)):
            pad_token_id = int(torch.as_tensor(pad_token_id).reshape(-1)[0])
        return BeamSearch(num_beams=int(num_beams), length_penalty=float(lp), early_stopping=es,
                          num_return_sequences=int(num_return_sequences),
                          pad_token_id=None if pad_token_id is None else int(pad_token_id))

    @staticmethod
    def _check_remaining_generate_kwargs(kwargs: dict):
        """Consumes the generate() kwargs left after the supported ones."""
        # options that would change the generated ids and are not implemented on the CUDA path must not be dropped
        # silently; pure output-format / cache switches are accepted
        neutral = {"length_penalty": 1.0, "encoder_repetition_penalty": 1.0, "typical_p": 1.0, "epsilon_cutoff": 0.0,
                   "eta_cutoff": 0.0, "min_p": None, "force_words_ids": None,
                   "suppress_tokens": None, "begin_suppress_tokens": None, "logits_processor": None,
                   "stopping_criteria": None, "prefix_allowed_tokens_fn": None, "penalty_alpha": None,
                   "num_beam_groups": 1, "diversity_penalty": 0.0}
        for k in list(kwargs):
            if k in neutral:
                v = kwargs.pop(k)
                if v is not None and v != neutral[k] and v != [] and v != 0:
                    raise NotImplementedError(f"generate({k}={v!r}) is not implemented on the CUDA path")
            elif k in ("use_cache", "return_dict_in_generate", "output_scores", "output_logits", "output_attentions",
                       "output_hidden_states", "synced_gpus", "streamer", "generation_config", "bos_token_id",
                       "cache_implementation", "tokenizer"):
                v = kwargs.pop(k)
                if k in ("return_dict_in_generate", "output_scores", "output_logits", "output_attentions",
                         "output_hidden_states") and v:
                    raise NotImplementedError(f"generate({k}=True) is not implemented on the CUDA path")
        if kwargs:
            raise TypeError(f"generate() got unsupported arguments {sorted(kwargs)}")


class _U2TrainLoss(torch.autograd.Function):
    """loss = TrainEngine.forward_loss(batch); backward() = TrainEngine.backward(): the bridge that lets
    `model(**batch).loss.backward()` (HF Trainer / accelerate) drive the hand-written backward pass."""

    @staticmethod
    def forward(ctx, te, batch, names, *params):
        images, input_ids, question_ids, labels = batch
        ctx.te, ctx.names, ctx.params = te, names, params
        with torch.no_grad():
            return te.forward_loss(images, input_ids, question_ids, labels)

    @staticmethod
    def backward(ctx, grad_out):
        te = ctx.te
        # autograd keeps the returned views as p.grad (no copy): on the next micro-batch of a gradient-accumulation window
        # those p.grad ARE the matrix slots, so the kernels add into them in place and nothing is handed back for them
        keep = {n for n, p in zip(ctx.names, ctx.params)
                if n in te.lay.mat_off and p.grad is not None and p.grad.data_ptr() == te.grad(n).data_ptr()}
        te.zero_grad(keep=keep)
        te.backward(grad_out.to(torch.float32))
        return (None, None, None, *te.param_grads(ctx.names, keep))


# ------------------------------------------------------------------------------------------------
# concrete classes
# ------------------------------------------------------------------------------------------------
class U2LlamaModel(U2MetaModel, LlamaModel):
    config_class = U2LlamaConfig

    def __init__(self, config):
        super().__init__(config)


class U2LlamaForCausalLM(U2MetaForCausalLM, LlamaForCausalLM):
    config_class = U2LlamaConfig

    def __init__(self, config):
        super(LlamaForCausalLM, self).__init__(config)
        self.model = U2LlamaModel(config)
        self.pretraining_tp = getattr(config, "pretraining_tp", 1)
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()

    def get_model(self):
        return self.model

    def forward(self, images=None, input_ids=None, labels=None, attention_mask=None, question_ids=None,
                position_ids=None, past_key_values=None, inputs_embeds=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, return_dict=None, **kwargs) -> Union[Tuple, CausalLMOutputWithPast]:
        return self._u2_forward(images, input_ids, labels, attention_mask, question_ids, position_ids, past_key_values,
                                inputs_embeds, use_cache, output_attentions, output_hidden_states, return_dict, **kwargs)

    @torch.no_grad()
    def generate(self, images=None, inputs=None, question_ids=None, **kwargs):
        return self._u2_generate(images, inputs, question_ids, **kwargs)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, **kwargs):
        images = kwargs.pop("images", None)
        out = super().prepare_inputs_for_generation(input_ids, past_key_values=past_key_values,
                                                    inputs_embeds=inputs_embeds, **kwargs)
        if images is not None:
            out["images"] = images
        return out


class U2Qwen3Model(U2MetaModel, Qwen3Model):
    config_class = U2Qwen3Config

    def __init__(self, config):
        super().__init__(config)


class U2Qwen3ForCausalLM(U2MetaForCausalLM, Qwen3ForCausalLM):
    """Qwen3 wrapper with the working (Llama-style) contract; the shipped reference u2qwen3.py is
    internally inconsistent (SURVEY.md F4) and cannot serve as the surface."""
    config_class = U2Qwen3Config

    def __init__(self, config):
        super(Qwen3ForCausalLM, self).__init__(config)
        self.model = U2Qwen3Model(config)
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()

    def get_model(self):
        return self.model

    def forward(self, images=None, input_ids=None, labels=None, attention_mask=None, question_ids=None,
                position_ids=None, past_key_values=None, inputs_embeds=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, return_dict=None, **kwargs) -> Union[Tuple, CausalLMOutputWithPast]:
        return self._u2_forward(images, input_ids, labels, attention_mask, question_ids, position_ids, past_key_values,
                                inputs_embeds, use_cache, output_attentions, output_hidden_states, return_dict, **kwargs)

    @torch.no_grad()
    def generate(self, images=None, inputs=None, question_ids=None, **kwargs):
        return self._u2_generate(images, inputs, question_ids, **kwargs)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, **kwargs):
        images = kwargs.pop("images", None)
        out = super().prepare_inputs_for_generation(input_ids, past_key_values=past_key_values,
                                                    inputs_embeds=inputs_embeds, **kwargs)
        if images is not None:
            out["images"] = images
        return out


class U2Phi3Model(U2MetaModel, Phi3Model):
    config_class = U2Phi3Config

    def __init__(self, config):
        super().__init__(config)


class U2Phi3ForCausalLM(U2MetaForCausalLM, Phi3ForCausalLM):
    """Phi-3 wrapper (reference u2phi3.py:25-140): HF Phi3's fused qkv_proj / gate_up_proj state-dict keys and its
    sliding window; the decoder runs on the same CUDA engine as the Llama / Qwen3 wrappers."""
    config_class = U2Phi3Config

    def __init__(self, config):
        super(Phi3ForCausalLM, self).__init__(config)
        self.model = U2Phi3Model(config)
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()

    def get_model(self):
        return self.model

    def forward(self, images=None, input_ids=None, labels=None, attention_mask=None, question_ids=None,
                position_ids=None, past_key_values=None, inputs_embeds=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, return_dict=None, **kwargs) -> Union[Tuple, CausalLMOutputWithPast]:
        return self._u2_forward(images, input_ids, labels, attention_mask, question_ids, position_ids, past_key_values,
                                inputs_embeds, use_cache, output_attentions, output_hidden_states, return_dict, **kwargs)

    @torch.no_grad()
    def generate(self, images=None, inputs=None, question_ids=None, **kwargs):
        return self._u2_generate(images, inputs, question_ids, **kwargs)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, **kwargs):
        images = kwargs.pop("images", None)
        out = super().prepare_inputs_for_generation(input_ids, past_key_values=past_key_values,
                                                    inputs_embeds=inputs_embeds, **kwargs)
        if images is not None:
            out["images"] = images
        return out


# reference-compatible aliases (class names used by the reference's callers / checkpoints)
u2LlamaForCausalLM = U2LlamaForCausalLM
u2Qwen3ForCausalLM = U2Qwen3ForCausalLM
u2Phi3ForCausalLM = U2Phi3ForCausalLM


def register_auto_classes():
    """AutoConfig / AutoModelForCausalLM registration (reference u2llama.py:141-142, u2qwen3.py:144-145,
    u2phi3.py:139-140)."""
    for cfg, mdl in ((U2LlamaConfig, U2LlamaForCausalLM), (U2Qwen3Config, U2Qwen3ForCausalLM),
                     (U2Phi3Config, U2Phi3ForCausalLM)):
        try:
            AutoConfig.register(cfg.model_type, cfg)
        except ValueError:
            pass
        try:
            AutoModelForCausalLM.register(cfg, mdl)
        except ValueError:
            pass


register_auto_classes()
