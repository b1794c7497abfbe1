"""u2tokenizer_b200: a H100-native (sm_90a) implementation of the mu2-LLM hot path.

CT volume -> 3D patch embedding -> ViT3D -> spatial-pooling projector -> mu2-Tokenizer ->
splice into the prompt embeddings -> Qwen3/Llama decoder forward / greedy generate.

The arithmetic lives in hand-written CUDA behind a C ABI (``libu2b200.so``, ``include/u2b200.h``);
this package is the thin host side that mirrors the reference's HuggingFace-style module surface.
"""
__version__ = "0.1.0"
