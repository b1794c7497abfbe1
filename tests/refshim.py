"""Test-only helper: import the REFERENCE modules from a checkout of the reference project, where one is mounted at
REF_ROOT, and otherwise serve their recorded outputs (tests/golden/pins/) so that the pins run everywhere.

MONAI 1.3.0 is neither vendored nor installed, so `monai.networks.blocks.{patchembedding,
transformerblock}` are provided by a small nn.Module restatement registered in sys.modules; the
reference's own vit.py / u2_arch.py / u2llama.py then import unchanged. Never used by product code.

Recording (needs the reference tree): U2_RECORD_PINS=1 python -m pytest tests/test_oracle_pin.py tests/test_oracle_grad_pin.py
"""
import os
import sys
import types

import torch
import torch.nn as nn

REF_ROOT = os.environ.get("U2_REFERENCE_ROOT", "/root/reference")
PIN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pins")


def have_reference() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "src", "model"))


def pinned(key, compute, keep=None):
    """(what the reference computes for `key`, complete?). With the reference tree mounted, `compute()` runs it (and with
    U2_RECORD_PINS=1 stores the result as golden/pins/<key>.pt, reduced by `keep` where the full output would be large);
    without it, the stored copy is returned: complete unless `keep` reduced it."""
    if have_reference():
        out = compute()
        if os.environ.get("U2_RECORD_PINS") == "1":
            os.makedirs(PIN_DIR, exist_ok=True)
            torch.save(keep(out) if keep else out, os.path.join(PIN_DIR, f"{key}.pt"))
        return out, True
    return torch.load(os.path.join(PIN_DIR, f"{key}.pt")), keep is None


class _PatchEmbeddingBlock(nn.Module):
    def __init__(self, in_channels, img_size, patch_size, hidden_size, num_heads, pos_embed, dropout_rate=0.0,
                 spatial_dims=3):
        super().__init__()
        assert pos_embed == "perceptron" and spatial_dims == 3
        self.patch_size = tuple(patch_size)
        n = 1
        for i, p in zip(img_size, patch_size):
            n *= i // p
        pd = in_channels * patch_size[0] * patch_size[1] * patch_size[2]
        self.patch_embeddings = nn.Sequential(nn.Identity(), nn.Linear(pd, hidden_size))
        self.position_embeddings = nn.Parameter(torch.zeros(1, n, hidden_size))
        nn.init.trunc_normal_(self.position_embeddings, std=0.02)

    def forward(self, x):
        b, c, H, W, D = x.shape
        p1, p2, p3 = self.patch_size
        x = x.view(b, c, H // p1, p1, W // p2, p2, D // p3, p3).permute(0, 2, 4, 6, 3, 5, 7, 1)
        x = x.reshape(b, -1, p1 * p2 * p3 * c)
        return self.patch_embeddings(x) + self.position_embeddings


class _SABlock(nn.Module):
    def __init__(self, hidden, heads, qkv_bias=False):
        super().__init__()
        self.h = heads
        self.qkv = nn.Linear(hidden, 3 * hidden, bias=qkv_bias)
        self.out_proj = nn.Linear(hidden, hidden)

    def forward(self, x):
        b, s, e = x.shape
        qkv = self.qkv(x).view(b, s, 3, self.h, e // self.h).permute(2, 0, 3, 1, 4)
        att = (torch.einsum("blxd,blyd->blxy", qkv[0], qkv[1]) * (e // self.h) ** -0.5).softmax(-1)
        return self.out_proj(torch.einsum("bhxy,bhyd->bhxd", att, qkv[2]).permute(0, 2, 1, 3).reshape(b, s, e))


class _MLPBlock(nn.Module):
    def __init__(self, hidden, mlp):
        super().__init__()
        self.linear1 = nn.Linear(hidden, mlp)
        self.linear2 = nn.Linear(mlp, hidden)

    def forward(self, x):
        return self.linear2(torch.nn.functional.gelu(self.linear1(x)))


class _TransformerBlock(nn.Module):
    def __init__(self, hidden_size, mlp_dim, num_heads, dropout_rate=0.0, qkv_bias=False, save_attn=False):
        super().__init__()
        self.mlp = _MLPBlock(hidden_size, mlp_dim)
        self.norm1 = nn.LayerNorm(hidden_size)
        self.attn = _SABlock(hidden_size, num_heads, qkv_bias)
        self.norm2 = nn.LayerNorm(hidden_size)

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


def install():
    """Put /root/reference on sys.path and register the MONAI stand-ins. Returns `src.model`."""
    if not have_reference():
        raise RuntimeError("reference tree not mounted")
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    if "monai.networks.blocks.patchembedding" not in sys.modules:
        for name in ("monai", "monai.networks", "monai.networks.blocks"):
            sys.modules.setdefault(name, types.ModuleType(name))
        pe = types.ModuleType("monai.networks.blocks.patchembedding")
        pe.PatchEmbeddingBlock = _PatchEmbeddingBlock
        tb = types.ModuleType("monai.networks.blocks.transformerblock")
        tb.TransformerBlock = _TransformerBlock
        sys.modules["monai.networks.blocks.patchembedding"] = pe
        sys.modules["monai.networks.blocks.transformerblock"] = tb
    import importlib
    return importlib.import_module("src.model")
