"""Plain-data description of the hot path's shapes, extracted once from the HF config.

The engine (and, in tests, the oracle) read this flat object instead of poking at
version-dependent HF config attributes (transformers >= 5 moved rope_theta/rope_scaling into
``rope_parameters``).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional


@dataclass
class Geometry:
    # --- vision front (reference src/model/u2_arch.py:35-57) ---
    image_channel: int = 1
    image_size: List[int] = field(default_factory=lambda: [32, 256, 256])
    patch_size: List[int] = field(default_factory=lambda: [4, 16, 16])
    vision_select_feature: str = "patch"
    vit_hidden: int = 768
    vit_mlp: int = 3072
    vit_layers: int = 12
    vit_heads: int = 12
    proj_layer_type: str = "mlp"
    proj_layer_num: int = 2
    proj_pooling_type: str = "spatial"
    proj_pooling_size: int = 2
    # --- mu2-tokenizer ---
    enable_u2tokenizer: bool = True
    u2t_num_heads: int = 8
    u2t_num_layers: int = 4
    u2t_top_k: int = 1024
    use_multi_scale: bool = True
    num_3d_query_token: int = 256
    attn_type: str = "rma"
    enable_diffts: bool = True
    enable_dmtp: bool = True
    # --- decoder ---
    hidden_size: int = 2048
    intermediate_size: int = 6144
    num_hidden_layers: int = 28
    num_attention_heads: int = 16
    num_key_value_heads: int = 8
    head_dim: int = 128
    vocab_size: int = 151936
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1e6
    rope_scaling: Optional[Dict[str, Any]] = None
    qk_norm: bool = True  # Qwen3: per-head RMSNorm on q,k; Llama, Phi-3: none
    tie_word_embeddings: bool = False
    # decoder state-dict naming: "llama" = separate q/k/v_proj and gate/up_proj (Llama and Qwen3), "phi3" = the fused
    # self_attn.qkv_proj [(hq + 2 hkv) dh, E] and mlp.gate_up_proj [gate; up] of HF Phi3 (modeling_phi3.py:54,58-62)
    decoder_family: str = "llama"
    # sliding-window attention (Phi-3): key j is visible from query i iff i - sliding_window < j <= i
    # (HF masking_utils.sliding_window_overlay); None = unlimited
    sliding_window: Optional[int] = None
    # largest of resid_pdrop / embd_pdrop / attention_dropout (Phi-3); eval mode ignores it as HF does, the training
    # path refuses a non-zero value
    decoder_dropout: float = 0.0

    @property
    def window(self) -> int:
        """The sliding window as the kernels take it: 0 = no window."""
        return int(self.sliding_window or 0)

    # derived
    @property
    def grid(self) -> List[int]:
        return [i // p for i, p in zip(self.image_size, self.patch_size)]

    @property
    def n_patches(self) -> int:
        g = self.grid
        return g[0] * g[1] * g[2]

    @property
    def patch_dim(self) -> int:
        p = self.patch_size
        return p[0] * p[1] * p[2] * self.image_channel

    @property
    def tokens_per_frame(self) -> int:
        """SpatialPoolingProjector.proj_out_num (reference spatial_pooling_projector.py:54-58)."""
        if self.proj_pooling_type == "spatial":
            n = 1
            for g in self.grid:
                n *= g // self.proj_pooling_size
            return n
        return self.n_patches // self.proj_pooling_size ** 3

    @classmethod
    def from_hf(cls, config) -> "Geometry":
        rp = getattr(config, "rope_parameters", None) or {}
        rope_theta = rp.get("rope_theta", getattr(config, "rope_theta", 10000.0))
        rs = getattr(config, "rope_scaling", None) or (rp if rp.get("rope_type", "default") != "default" else None)
        if rs is not None and rs.get("rope_type", rs.get("type", "default")) == "default":
            rs = None
        head_dim = getattr(config, "head_dim", None) or config.hidden_size // config.num_attention_heads
        qk_norm = "qwen3" in config.model_type.lower()
        family, window, dropout = "llama", None, 0.0
        if "phi3" in config.model_type.lower():
            family = "phi3"
            rope_type = (rs or {}).get("rope_type", (rs or {}).get("type", "default"))
            if rs is not None:
                raise NotImplementedError(
                    f"Phi-3 rope_type {rope_type!r} (longrope / su: Phi-3-mini-128k, Phi-3.5) is not supported: only the "
                    "default RoPE of the 4k Phi-3 models runs on the CUDA path")
            prf = float(rp.get("partial_rotary_factor", getattr(config, "partial_rotary_factor", 1.0)) or 1.0)
            if prf != 1.0:
                raise NotImplementedError(f"Phi-3 partial_rotary_factor={prf} (Phi-4-mini) is not supported: the CUDA "
                                          "path rotates the whole head")
            window = getattr(config, "sliding_window", None)
            window = int(window) if window else None
            dropout = max(float(getattr(config, k, 0.0) or 0.0) for k in ("resid_pdrop", "embd_pdrop", "attention_dropout"))
        return cls(
            image_channel=config.image_channel, image_size=list(config.image_size),
            patch_size=list(config.patch_size), vision_select_feature=config.vision_select_feature,
            vit_hidden=getattr(config, "vit_hidden_size", 768), vit_mlp=getattr(config, "vit_mlp_dim", 3072),
            vit_layers=getattr(config, "vit_num_layers", 12), vit_heads=getattr(config, "vit_num_heads", 12),
            proj_layer_type=config.proj_layer_type, proj_layer_num=int(config.proj_layer_num),
            proj_pooling_type=config.proj_pooling_type, proj_pooling_size=int(config.proj_pooling_size),
            enable_u2tokenizer=bool(config.enable_u2tokenizer), u2t_num_heads=config.u2t_num_heads,
            u2t_num_layers=config.u2t_num_layers, u2t_top_k=config.u2t_top_k,
            use_multi_scale=bool(config.use_multi_scale), num_3d_query_token=config.num_3d_query_token,
            attn_type=getattr(config, "attn_type", "rma"), enable_diffts=bool(config.enable_diffts),
            enable_dmtp=bool(config.enable_dmtp),
            hidden_size=config.hidden_size, intermediate_size=config.intermediate_size,
            num_hidden_layers=config.num_hidden_layers, num_attention_heads=config.num_attention_heads,
            num_key_value_heads=config.num_key_value_heads, head_dim=head_dim,
            vocab_size=config.vocab_size, rms_norm_eps=config.rms_norm_eps,
            rope_theta=float(rope_theta), rope_scaling=dict(rs) if rs else None, qk_norm=qk_norm,
            tie_word_embeddings=bool(getattr(config, "tie_word_embeddings", False)),
            decoder_family=family, sliding_window=window, decoder_dropout=dropout,
        )
