"""fp32 restatement of the Phi-3 decoder (HF transformers models/phi3/modeling_phi3.py) for the tests: the fused
self_attn.qkv_proj / mlp.gate_up_proj weights and the sliding window of masking_utils.sliding_window_overlay
(key j visible from query i iff i - W < j <= i). The vision front and the mu2-tokenizer are the shared oracle's."""
import math

import torch
import torch.nn.functional as F

from oracle import u2_oracle as O


def decoder_forward(sd, inputs_embeds: torch.Tensor, g, past=None, return_hidden: bool = False):
    """Phi-3 decoder stack + lm_head, eager fp32, positions past_len + arange; `past`: list of full-length (k, v) per
    layer [B, Hkv, T, dh] (the window is a mask, the cache keeps every position). Returns (logits, new_past)."""
    b, s, _ = inputs_embeds.shape
    hq, hkv, dh = g.num_attention_heads, g.num_key_value_heads, g.head_dim
    eps, W = g.rms_norm_eps, g.sliding_window
    past_len = 0 if past is None else past[0][0].shape[2]
    dev, dt = inputs_embeds.device, inputs_embeds.dtype
    pos = torch.arange(past_len, past_len + s, dtype=torch.float32, device=dev)
    fr = torch.outer(pos, O.rope_inv_freq(g).to(dev))
    emb = torch.cat((fr, fr), dim=-1)
    cos, sin = emb.cos()[None, None].to(dt), emb.sin()[None, None].to(dt)
    qi = torch.arange(past_len, past_len + s, device=dev)[:, None]
    kj = torch.arange(past_len + s, device=dev)[None, :]
    visible = kj <= qi
    if W:
        visible &= kj > qi - W
    mask = torch.zeros(visible.shape, device=dev, dtype=dt).masked_fill(~visible, float("-inf"))
    x = inputs_embeds
    new_past = []
    for i in range(g.num_hidden_layers):
        lp = f"model.layers.{i}."
        y = O._rms(x, sd[lp + "input_layernorm.weight"], eps)
        qkv = F.linear(y, sd[lp + "self_attn.qkv_proj.weight"])
        q = qkv[..., :hq * dh].view(b, s, hq, dh).transpose(1, 2)
        k = qkv[..., hq * dh:(hq + hkv) * dh].view(b, s, hkv, dh).transpose(1, 2)
        v = qkv[..., (hq + hkv) * dh:].view(b, s, hkv, dh).transpose(1, 2)
        q = q * cos + O._rotate_half(q) * sin
        k = k * cos + O._rotate_half(k) * sin
        if past is not None:
            k = torch.cat((past[i][0], k), dim=2)
            v = torch.cat((past[i][1], v), dim=2)
        new_past.append((k, v))
        kk = k.repeat_interleave(hq // hkv, dim=1)
        vv = v.repeat_interleave(hq // hkv, dim=1)
        att = torch.softmax(q @ kk.transpose(-2, -1) / math.sqrt(dh) + mask, dim=-1)
        o = (att @ vv).transpose(1, 2).reshape(b, s, hq * dh)
        x = x + F.linear(o, sd[lp + "self_attn.o_proj.weight"])
        y = O._rms(x, sd[lp + "post_attention_layernorm.weight"], eps)
        gate, up = F.linear(y, sd[lp + "mlp.gate_up_proj.weight"]).chunk(2, dim=-1)
        x = x + F.linear(up * F.silu(gate), sd[lp + "mlp.down_proj.weight"])
    x = O._rms(x, sd["model.norm.weight"], eps)
    if return_hidden:
        return x, new_past
    w_head = sd["lm_head.weight"] if "lm_head.weight" in sd else sd["model.embed_tokens.weight"]
    return F.linear(x, w_head), new_past


@torch.no_grad()
def greedy_from_embeds(sd, emb: torch.Tensor, g, max_new_tokens: int):
    """Greedy decoding after a prefill on `emb`: new ids [B, n] and the per-step top-1 / top-2 logit margins."""
    logits, past = decoder_forward(sd, emb, g)
    out, margins = [], []
    for _ in range(max_new_tokens):
        last = logits[:, -1]
        top2 = last.topk(2, dim=-1).values
        margins.append(top2[:, 0] - top2[:, 1])
        nxt = last.argmax(-1)
        out.append(nxt)
        logits, past = decoder_forward(sd, F.embedding(nxt[:, None], sd["model.embed_tokens.weight"]), g, past)
    return torch.stack(out, dim=1), torch.stack(margins, dim=1)
