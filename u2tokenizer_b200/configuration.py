"""Configuration classes of the HF-style surface.

Mirrors the reference's ``u2Config(LlamaConfig)`` (model_type "u2llama",
reference src/model/language_model/u2llama.py:15-16) and ``u2Config(Qwen3Config)`` (model_type
"u2Qwen3", u2qwen3.py:15-16) and ``u2Phi3Config(Phi3Config)`` (model_type "u2phi3", u2phi3.py:15-16). The multimodal hyper-parameters are the ones
``initialize_vision_modules`` copies onto the config (reference src/model/u2_arch.py:35-57); the
canonical values are those of base_model_tokenizers/Llama-3.2-1B-Instruct/config.json:9-44.
"""
from __future__ import annotations

from transformers import LlamaConfig, Phi3Config, Qwen3Config

# canonical multimodal hyper-parameters (reference config.json:9-44, train_stage1.py:46-78)
MM_DEFAULTS = dict(
    image_channel=1,
    image_size=[32, 256, 256],
    patch_size=[4, 16, 16],
    vision_tower="vit3d",
    vision_select_layer=-1,
    vision_select_feature="patch",
    mm_hidden_size=768,
    mm_projector_type="spp",
    proj_layer_type="mlp",
    proj_layer_num=2,
    proj_pooling_type="spatial",
    proj_pooling_size=2,
    enable_u2tokenizer=True,
    u2t_num_heads=8,
    u2t_num_layers=4,
    u2t_top_k=1024,
    use_multi_scale=True,
    num_3d_query_token=256,
    attn_type="rma",
    enable_diffts=True,
    enable_dmtp=True,
    # ViT-B/12 geometry: MONAI ViT defaults used by the reference (vit.py:35-38)
    vit_hidden_size=768,
    vit_mlp_dim=3072,
    vit_num_layers=12,
    vit_num_heads=12,
)


def _apply_mm_defaults(cfg, kwargs):
    for k, v in MM_DEFAULTS.items():
        setattr(cfg, k, kwargs.pop(k, v))
    # remote-code checkpoints carry `enable_rpe` instead of attn_type
    # (base_model_tokenizers/Llama-3.2-1B-Instruct/u2Tokenizer.py:413-425)
    if "enable_rpe" in kwargs:
        cfg.attn_type = "rma" if kwargs.pop("enable_rpe") else cfg.attn_type


class U2LlamaConfig(LlamaConfig):
    model_type = "u2llama"

    def __init__(self, **kwargs):
        mm = {k: kwargs.pop(k) for k in list(kwargs) if k in MM_DEFAULTS or k == "enable_rpe"}
        super().__init__(**kwargs)
        _apply_mm_defaults(self, mm)


class U2Qwen3Config(Qwen3Config):
    model_type = "u2Qwen3"

    def __init__(self, **kwargs):
        mm = {k: kwargs.pop(k) for k in list(kwargs) if k in MM_DEFAULTS or k == "enable_rpe"}
        super().__init__(**kwargs)
        _apply_mm_defaults(self, mm)


class U2Phi3Config(Phi3Config):
    model_type = "u2phi3"

    def __init__(self, **kwargs):
        mm = {k: kwargs.pop(k) for k in list(kwargs) if k in MM_DEFAULTS or k == "enable_rpe"}
        super().__init__(**kwargs)
        _apply_mm_defaults(self, mm)


# public model geometries (model cards; the reference only names the checkpoints, README.md:43-44)
QWEN3_1P7B = dict(hidden_size=2048, intermediate_size=6144, num_hidden_layers=28, num_attention_heads=16,
                  num_key_value_heads=8, head_dim=128, vocab_size=151936, rms_norm_eps=1e-6,
                  rope_theta=1000000.0, max_position_embeddings=40960, tie_word_embeddings=True)
QWEN3_8B = dict(hidden_size=4096, intermediate_size=12288, num_hidden_layers=36, num_attention_heads=32,
                num_key_value_heads=8, head_dim=128, vocab_size=151936, rms_norm_eps=1e-6,
                rope_theta=1000000.0, max_position_embeddings=40960, tie_word_embeddings=False)
LLAMA32_1B = dict(hidden_size=2048, intermediate_size=8192, num_hidden_layers=16, num_attention_heads=32,
                  num_key_value_heads=8, head_dim=64, vocab_size=128256, rms_norm_eps=1e-5,
                  rope_theta=500000.0, max_position_embeddings=131072, tie_word_embeddings=True,
                  rope_scaling=dict(factor=32.0, high_freq_factor=4.0, low_freq_factor=1.0,
                                    original_max_position_embeddings=8192, rope_type="llama3"))
PHI3_MINI_4K = dict(hidden_size=3072, intermediate_size=8192, num_hidden_layers=32, num_attention_heads=32,
                    num_key_value_heads=32, vocab_size=32064, rms_norm_eps=1e-5, rope_theta=10000.0,
                    max_position_embeddings=4096, original_max_position_embeddings=4096, sliding_window=2047,
                    tie_word_embeddings=False, hidden_act="silu", pad_token_id=32000, bos_token_id=1,
                    eos_token_id=32000)
