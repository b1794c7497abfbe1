"""LoRA on the decoder (u2tokenizer_b200/lora.py, the LoRA path of train.py, csrc/lora.cu): PEFT's parameter layout and
refusals, the training layout, the three kernels against fp32 torch with the dropout masks rebuilt from the documented
hash, the training engine against autograd through the oracle with the adapter term added, and the reference's
stage-1 / eval flows through the module surface."""
import math

import pytest
import torch
import torch.nn.functional as F

from common import cosine, rel_err, tiny_geometry
from oracle import u2_oracle as O
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict

BF = torch.bfloat16
M32 = 0xFFFFFFFF
TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
IGNORE = ("vision_tower", "mm_projector", "embed_tokens", "lm_head", "seg_projector", "seg_module", "u2tokenizer")


# ------------------------------------------------------------------------------------------------
# the documented mask hash, restated in torch (int64 holding uint32 values)
# ------------------------------------------------------------------------------------------------
def _mul32(h, c):
    return ((h * (c & 0xFFFF)) + (((h * (c >> 16)) & 0xFFFF) << 16)) & M32


def fmix32(h):
    h = h ^ (h >> 16)
    h = _mul32(h, 0x85EBCA6B)
    h = h ^ (h >> 13)
    h = _mul32(h, 0xC2B2AE35)
    return h ^ (h >> 16)


def lora_mask(seed, stream, M, K, p, device="cpu"):
    """D [M, K] fp32: 0 where fmix32(fmix32(key ^ row) ^ col) < floor(p 2^32), else 1 / (1 - p)."""
    if p == 0:
        return torch.ones(M, K, device=device)
    lo, hi = seed & M32, (seed >> 32) & M32
    t = lambda v: torch.tensor(v, dtype=torch.int64, device=device)
    key = fmix32(t(lo) ^ fmix32((t(hi) + _mul32(t(stream), 0x9E3779B9)) & M32))
    rows = torch.arange(M, dtype=torch.int64, device=device)[:, None]
    cols = torch.arange(K, dtype=torch.int64, device=device)[None, :]
    h = fmix32(fmix32(key ^ rows) ^ cols)
    thr = min(math.floor(p * 2 ** 32), M32)
    keep = torch.tensor(1.0 / (1.0 - p), dtype=torch.float32).item()
    return torch.where(h < thr, torch.zeros((), device=device), torch.full((), keep, device=device))


def test_mask_hash_restatement_matches_integer_arithmetic():
    def fm(h):
        h ^= h >> 16
        h = (h * 0x85EBCA6B) & M32
        h ^= h >> 13
        h = (h * 0xC2B2AE35) & M32
        return h ^ (h >> 16)
    seed, stream = 0x123456789ABCDEF1, 8 * 3 + 5
    key = fm((seed & M32) ^ fm(((seed >> 32) + stream * 0x9E3779B9) & M32))
    p = 0.3
    D = lora_mask(seed, stream, 5, 7, p)
    for r in range(5):
        for c in range(7):
            want = 0.0 if fm(fm(key ^ r) ^ c) < math.floor(p * 2 ** 32) else 1 / (1 - p)
            assert abs(float(D[r, c]) - want) < 1e-6


# ------------------------------------------------------------------------------------------------
# CPU: the surface
# ------------------------------------------------------------------------------------------------
def _tiny_model(family="qwen3", device="cpu", tie=False):
    from u2tokenizer_b200.configuration import U2LlamaConfig, U2Qwen3Config
    from u2tokenizer_b200.modeling import U2LlamaForCausalLM, U2Qwen3ForCausalLM
    kw = dict(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
              head_dim=32, vocab_size=512, image_size=[16, 64, 64], vit_hidden_size=96, vit_mlp_dim=192, vit_num_layers=2,
              vit_num_heads=4, u2t_num_layers=2, u2t_top_k=8, num_3d_query_token=8, tie_word_embeddings=tie,
              rms_norm_eps=1e-6, rope_theta=1e6)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(BF)
    try:
        with torch.device(device):
            if family == "qwen3":
                cfg = U2Qwen3Config(**kw)
                model = U2Qwen3ForCausalLM(cfg)
            else:
                cfg = U2LlamaConfig(**kw)
                model = U2LlamaForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)
    return model


def reference_linear_names(model):
    """The reference's find_all_linear_names rule: every nn.Linear whose module name holds none of its ignore keywords."""
    return sorted(n for n, m in model.named_modules()
                  if isinstance(m, torch.nn.Linear) and not any(k in n for k in IGNORE))


@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_peft_state_dict_keys(family):
    from u2tokenizer_b200.lora import LoraConfig, get_peft_model
    model = _tiny_model(family, tie=(family == "llama"))
    before = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    peft = get_peft_model(model, LoraConfig(r=8, lora_alpha=16, target_modules=reference_linear_names(model),
                                            lora_dropout=0.05, bias="none", task_type="CAUSAL_LM"))
    want = {}
    for k, s in before.items():
        parts = k.split(".")
        if len(parts) == 6 and parts[0] == "model" and parts[1] == "layers" and parts[4] in TARGETS and parts[5] == "weight":
            m = "base_model.model." + k[:-len(".weight")]
            want[m + ".base_layer.weight"] = s
            want[m + ".lora_A.default.weight"] = (8, s[1])
            want[m + ".lora_B.default.weight"] = (s[0], 8)
        else:
            want["base_model.model." + k] = s
    got = {k: tuple(v.shape) for k, v in peft.state_dict().items()}
    assert got == want
    n_lora = sum(1 for k in got if ".lora_" in k)
    assert n_lora == 2 * 7 * model.config.num_hidden_layers


def test_target_resolution_and_requires_grad():
    from u2tokenizer_b200.lora import LoraConfig, LoraLinear, get_peft_model
    model = _tiny_model()
    names = reference_linear_names(model)
    assert len(names) == 7 * model.config.num_hidden_layers and all(n.split(".")[-1] in TARGETS for n in names)
    model.get_model().vision_tower.requires_grad_(False)
    flags = {n: p.requires_grad for n, p in model.named_parameters()}
    peft = get_peft_model(model, LoraConfig(r=16, lora_alpha=32, target_modules=names, lora_dropout=0.05))
    assert sorted(n for n, m in model.named_modules() if isinstance(m, LoraLinear)) == names
    for n, p in peft.named_parameters():
        inner = n[len("base_model.model."):]
        if ".lora_" in inner:
            assert p.requires_grad
        elif ".base_layer." in inner:
            assert not p.requires_grad
        else:
            assert p.requires_grad == flags[inner], inner
    a = model.get_submodule(names[0]).lora_A["default"].weight.float()
    bound = 1 / math.sqrt(a.shape[1])   # kaiming_uniform_(a=sqrt(5)) on [r, in]
    assert a.abs().max() <= bound + 1e-3 and a.abs().max() > 0.5 * bound
    assert all(model.get_submodule(n).lora_B["default"].weight.abs().max() == 0 for n in names)
    # the reference's unfreeze loop works as written
    for n, p in peft.named_parameters():
        if any(x in n for x in IGNORE):
            p.requires_grad = True
    assert all(p.requires_grad for n, p in peft.named_parameters() if "vision_tower" in n)
    t, tot = peft.get_nb_trainable_parameters()
    assert 0 < t < tot


@pytest.mark.parametrize("kw,what", [
    (dict(bias="all"), "bias"), (dict(bias="lora_only"), "bias"), (dict(use_rslora=True), "rslora"),
    (dict(use_dora=True), "dora"), (dict(modules_to_save=["lm_head"]), "modules_to_save"),
    (dict(init_lora_weights="gaussian"), "init_lora_weights"), (dict(init_lora_weights=False), "init_lora_weights")])
def test_config_refusals(kw, what):
    from u2tokenizer_b200.lora import LoraConfig
    with pytest.raises(NotImplementedError, match=what):
        LoraConfig(r=8, lora_alpha=16, target_modules=["q_proj"], **kw)


@pytest.mark.parametrize("targets,match", [
    (["lm_head"], "lm_head"), (["wq"], "u2tokenizer"), (["qkv"], "vision_tower"), (["mm_projector"], "mm_projector"),
    (["q_proj"], "fused group"), (["gate_proj"], "fused group")])
def test_target_refusals(targets, match):
    from u2tokenizer_b200.lora import LoraConfig, get_peft_model
    model = _tiny_model()
    with pytest.raises(NotImplementedError, match=match):
        get_peft_model(model, LoraConfig(r=8, lora_alpha=16, target_modules=targets))


def test_rank_and_target_errors():
    from u2tokenizer_b200.lora import LoraConfig, get_peft_model
    with pytest.raises(NotImplementedError, match="rank"):
        get_peft_model(_tiny_model(), LoraConfig(r=4, lora_alpha=8, target_modules=["q_proj", "k_proj", "v_proj"]))
    with pytest.raises(ValueError, match="not found"):
        get_peft_model(_tiny_model(), LoraConfig(r=8, lora_alpha=8, target_modules=["nope"]))


# ------------------------------------------------------------------------------------------------
# CPU: the training layout
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_lora_layout(world):
    from u2tokenizer_b200.train import Layout, LoraSpec, training_order
    g = tiny_geometry()
    L = Layout(g, world_size=world, bucket_elems=50_000, lora=LoraSpec(16, 2.0, 0.05, TARGETS))
    assert len(L.frozen_names) == 7 * g.num_hidden_layers and not set(L.frozen_names) & set(L.mat_off)
    assert L.frozen_total >= sum(L._numel(n) for n in L.frozen_names)
    assert all(n not in ns for ns in L.bucket_names for n in L.frozen_names)
    owned = sorted((i * L.bucket + r * L.piece, i * L.bucket + (r + 1) * L.piece) for r in range(world) for i in range(L.n_buckets))
    assert owned[0][0] == 0 and owned[-1][1] == L.mat_total and all(a[1] == b[0] for a, b in zip(owned[:-1], owned[1:]))
    assert L.mat_used <= L.mat_total
    for li in range(g.num_hidden_layers):
        p = f"model.layers.{li}."
        for pre, grp in (("self_attn.", ("q_proj", "k_proj", "v_proj")), ("mlp.", ("gate_proj", "up_proj"))):
            assert L.adjacent([p + pre + t + ".lora_A.default.weight" for t in grp])
            assert L.adjacent([p + pre + t + ".lora_B.default.weight" for t in grp])
            assert L.adjacent([p + pre + t + ".weight" for t in grp])   # the frozen bases stay fused
        assert L.shapes[p + "mlp.down_proj.lora_A.default.weight"] == (16, g.intermediate_size)
        assert L.shapes[p + "mlp.down_proj.lora_B.default.weight"] == (g.hidden_size, 16)
    # without LoRA: today's layout, no frozen region
    L0, Ln = Layout(g, world_size=world, bucket_elems=50_000), Layout(g, world_size=world, bucket_elems=50_000, lora=None)
    mats, vecs = training_order(g)
    assert L0.mat_names == mats and L0.vec_names == vecs and L0.frozen_total == 0 and not L0.frozen_names
    assert (L0.mat_off, L0.vec_off, L0.bucket, L0.n_buckets, L0.mat_total, L0.vec_total) == \
        (Ln.mat_off, Ln.vec_off, Ln.bucket, Ln.n_buckets, Ln.mat_total, Ln.vec_total)
    # the non-decoder matrices keep their relative order
    assert [n for n in L.mat_names if ".lora_" not in n] == [n for n in mats if n not in L.frozen_names]


# ------------------------------------------------------------------------------------------------
# GPU: the kernels
# ------------------------------------------------------------------------------------------------
def _op_inputs(M, K, r, nA, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn(M, K, device="cuda", generator=g).to(BF)
    A = (torch.randn(nA * r, K, device="cuda", generator=g) * 0.1).to(BF)
    dU = torch.randn(M, nA * r, device="cuda", generator=g).to(BF)
    return X, A, dU


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.0, 0.05, 0.5])
@pytest.mark.parametrize("r", [8, 16, 64])
@pytest.mark.parametrize("nA", [1, 2, 3])
@pytest.mark.parametrize("M", [1, 65, 1000, 4096])
def test_kernels_match_fp32_torch(p, r, nA, M):
    from u2tokenizer_b200 import train_ops as T
    K, s, seed = 200, 1.75, 0x0123456789ABCDEF
    streams = [8 * 5 + j for j in range(nA)]
    X, A, dU = _op_inputs(M, K, r, nA, seed=M + r)
    D = [lora_mask(seed, st, M, K, p, device="cuda") for st in streams]
    Xm = [(D[j] * X.float()).to(BF).float() for j in range(nA)]
    U = T.lora_down(X, A, r, s, p=p, seed=seed, streams=streams)
    for j in range(nA):
        want = s * Xm[j] @ A[j * r:(j + 1) * r].float().T
        got = U[:, j * r:(j + 1) * r].float()
        assert (got - want).abs().max().item() <= 1e-2 * want.abs().max().item() + 1e-3, ("down", j)
    assert torch.equal(U, T.lora_down(X, A, r, s, p=p, seed=seed, streams=streams))   # same seed, same bits
    dA = torch.empty_like(A)
    T.lora_wgrad(dU, X, dA, r, s, p=p, seed=seed, streams=streams)
    want_dA = torch.cat([s * dU[:, j * r:(j + 1) * r].float().T @ Xm[j] for j in range(nA)])
    assert (dA.float() - want_dA).abs().max().item() <= 1e-2 * want_dA.abs().max().item() + 1e-3, "wgrad"
    dA2 = dA.clone()
    T.lora_wgrad(dU, X, dA2, r, s, p=p, seed=seed, streams=streams, accumulate=True)
    assert (dA2.float() - 2 * want_dA).abs().max().item() <= 2e-2 * want_dA.abs().max().item() + 1e-3, "wgrad accumulate"
    dX0 = torch.randn(M, K, device="cuda").to(BF)
    dX = dX0.clone()
    T.lora_dgrad(dU, A, dX, r, s, p=p, seed=seed, streams=streams)
    add = sum(D[j] * (s * dU[:, j * r:(j + 1) * r].float() @ A[j * r:(j + 1) * r].float()) for j in range(nA))
    want_dX = dX0.float() + add
    assert (dX.float() - want_dX).abs().max().item() <= 1e-2 * want_dX.abs().max().item() + 1e-2, "dgrad"


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.05, 0.5])
def test_kernel_mask_bits_rate_and_seed(p):
    """With X = 1, A = I and s = 1 the down-projection returns the masks themselves: they equal the restated hash, the
    dropped fraction lies within 5 sigma of p, another seed gives another mask; the dgrad kernel drops the same elements."""
    from u2tokenizer_b200 import train_ops as T
    M, K, r, nA, seed = 4096, 64, 64, 3, 987654321
    X = torch.ones(M, K, device="cuda", dtype=BF)
    A = torch.eye(r, device="cuda").repeat(nA, 1).to(BF).contiguous()
    streams = [3, 11, 12]
    U = T.lora_down(X, A, r, 1.0, p=p, seed=seed, streams=streams)
    n = M * K
    for j in range(nA):
        want = lora_mask(seed, streams[j], M, K, p, device="cuda").to(BF)
        got = U[:, j * r:(j + 1) * r]
        assert torch.equal(got, want), j
        rate = (got == 0).float().mean().item()
        assert abs(rate - p) < 5 * math.sqrt(p * (1 - p) / n), (rate, p)
    assert not torch.equal(U, T.lora_down(X, A, r, 1.0, p=p, seed=seed + 1, streams=streams))
    # backward mask == forward mask: dX = D o (dU A) with dU = 1 on adapter j only
    for j in range(nA):
        dU = torch.zeros(M, nA * r, device="cuda", dtype=BF)
        dU[:, j * r:(j + 1) * r] = 1
        dX = torch.zeros(M, K, device="cuda", dtype=BF)
        T.lora_dgrad(dU, A, dX, r, 1.0, p=p, seed=seed, streams=streams)
        assert torch.equal(dX == 0, U[:, j * r:(j + 1) * r] == 0), j


# ------------------------------------------------------------------------------------------------
# GPU: the training engine against the oracle's autograd with the adapter term added
# ------------------------------------------------------------------------------------------------
def _lora_sd(g, sd16, r, seed=4, zero_b=False):
    gen = torch.Generator().manual_seed(seed)
    sd = dict(sd16)
    for li in range(g.num_hidden_layers):
        for pre, t in [("self_attn.", t) for t in TARGETS[:4]] + [("mlp.", t) for t in TARGETS[4:]]:
            m = f"model.layers.{li}.{pre}{t}."
            out_f, in_f = sd16[m + "weight"].shape
            sd[m + "lora_A.default.weight"] = ((torch.rand(r, in_f, generator=gen) * 2 - 1) / math.sqrt(in_f)).to(BF)
            b = torch.zeros(out_f, r) if zero_b else torch.randn(out_f, r, generator=gen) * 0.05
            sd[m + "lora_B.default.weight"] = b.to(BF)
    return sd


class _OracleLora:
    """Monkeypatches the oracle's linear so that every adapted decoder linear adds s * B A (D o x)."""

    def __init__(self, monkeypatch, sd, s, p, seed):
        self.sd, self.s, self.p, self.seed = sd, s, p, seed
        orig = O._lin

        def lin(x, sd_, name, bias=True):
            y = orig(x, sd_, name, bias)
            a = name + ".lora_A.default.weight"
            if a not in sd_:
                return y
            parts = name.split(".")
            li, t = int(parts[2]), parts[4]
            x2 = x.reshape(-1, x.shape[-1])
            D = lora_mask(self.seed, li * 8 + TARGETS.index(t), x2.shape[0], x2.shape[1], self.p if self.seed else 0.0,
                          device=x.device)
            u = (D * x2) @ sd_[a].T
            return y + (self.s * u @ sd_[name + ".lora_B.default.weight"].T).view(*y.shape[:-1], -1)
        monkeypatch.setattr(O, "_lin", lin)


def _next_seed(torch_seed):
    torch.manual_seed(torch_seed)
    return int(torch.randint(1, 2 ** 63 - 1, (1,)).item())


ENGINE_CASES = {"qwen3_p0": (dict(), 0.0), "qwen3_p01": (dict(), 0.1), "llama_tied_p0": (
    dict(qk_norm=False, tie_word_embeddings=True, rope_theta=500000.0), 0.0), "llama_tied_p01": (
    dict(qk_norm=False, tie_word_embeddings=True, rope_theta=500000.0), 0.1)}


def _compare_grads(te, ref_g, skip=()):
    L = te.lay
    gmax = max(v.abs().max().item() for v in ref_g.values())
    bad, n_lora = [], 0
    for n in L.mat_names + L.vec_names:
        if n in skip or (n == "lm_head.weight" and te.tied):
            continue
        got = te.grad(n).float().cpu()
        want = ref_g[n].cpu()
        if want.abs().max().item() < 1e-9:
            continue
        n_lora += ".lora_" in n
        e, c = rel_err(got, want), cosine(got, want)
        if not (e < 4e-2 and c > 0.995) and (got - want).abs().max().item() >= 2e-3 * gmax:
            bad.append((n, round(e, 4), round(c, 5)))
    return bad, n_lora


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ENGINE_CASES))
def test_engine_forward_backward_matches_oracle(case, monkeypatch):
    from u2tokenizer_b200.train import LoraSpec, TrainEngine
    over, p = ENGINE_CASES[case]
    g = tiny_geometry(**over)
    r, s = 8, 2.0
    sd16 = synthetic_state_dict(g, seed=21, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    sd16 = _lora_sd(g, sd16, r)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=3, n_question=7, lt=12)
    labels = ids.clone()
    labels[:, :g.num_3d_query_token + 1] = -100
    te = TrainEngine(g, sd16, device="cuda", lora=LoraSpec(r, s, p, TARGETS))
    te.zero_grad()
    torch.manual_seed(123)
    loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    torch.cuda.synchronize()
    seed = _next_seed(123) if p > 0 else 0
    assert te._lora_seed == seed
    _OracleLora(monkeypatch, None, s, p, seed)
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    logits = O.forward_logits(sd, ids.cuda(), images.cuda(), qids.cuda(), g)
    ref = O.causal_lm_loss(logits, labels.cuda())
    ref.backward()
    ref_g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}
    assert abs(float(loss) - float(ref)) < 2e-2 * max(1.0, abs(float(ref))), (float(loss), float(ref))
    bad, n_lora = _compare_grads(te, ref_g)
    assert not bad, bad[:6]
    assert n_lora == 2 * 7 * g.num_hidden_layers


@pytest.mark.gpu
def test_engine_zero_b_is_bit_identical_and_steps_keep_frozen_bases():
    from u2tokenizer_b200.train import LoraSpec, TrainEngine
    g = tiny_geometry()
    sd16 = synthetic_state_dict(g, seed=9, device="cpu", dtype=BF)
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10)
    labels = ids.clone()
    labels[:, :g.num_3d_query_token + 1] = -100
    args = (images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
    plain = TrainEngine(g, sd16, device="cuda")
    te = TrainEngine(g, _lora_sd(g, sd16, 16, zero_b=True), device="cuda", lora=LoraSpec(16, 2.0, 0.1, TARGETS),
                     bucket_elems=50_000)
    assert float(plain.forward_loss(*args)) == float(te.forward_loss(*args))
    L = te.lay
    frozen0 = te.W[L.mat_total + L.vec_total:].clone()
    te.init_optimizer(lr=1e-3, weight_decay=0.01, max_grad_norm=1.0)
    ref_m = torch.nn.Parameter(te.W[:L.mat_total].float().clone())
    ref_v = torch.nn.Parameter(te.W[L.mat_total:L.mat_total + L.vec_total].float().clone())
    opt = torch.optim.AdamW([ref_m, ref_v], lr=1e-3, weight_decay=0.01)
    losses = []
    for it in range(3):
        te.zero_grad()
        losses.append(float(te.forward_backward(*args)))
        ref_m.grad, ref_v.grad = te.Gm.float().clone(), te.Gv.clone()
        torch.nn.utils.clip_grad_norm_([ref_m, ref_v], 1.0)
        opt.step()
        te.optimizer_step()
        assert float((te.opt["m_master"] - ref_m.data).abs().max()) < 2e-5, it
        assert float((te.opt["v_master"] - ref_v.data).abs().max()) < 2e-5, it
        assert torch.equal(te.W[L.mat_total + L.vec_total:], frozen0), it
    b = te.w("model.layers.0.self_attn.q_proj.lora_B.default.weight")
    assert b.abs().max().item() > 0     # B left zero after the first step
    assert losses[2] < losses[0], losses


@pytest.mark.gpu
def test_engine_dpo_step_matches_oracle(monkeypatch):
    from u2tokenizer_b200.train import LoraSpec, TrainEngine
    g = tiny_geometry()
    r, s, p = 8, 2.0, 0.1
    sd16 = synthetic_state_dict(g, seed=31, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    sd16 = _lora_sd(g, sd16, r, seed=6)
    images, ids, qids = synthetic_inputs(g, batch=1, frames=2, n_question=6, lt=10)
    gen = torch.Generator().manual_seed(3)
    n_prompt = ids.shape[1]
    ans = torch.randint(1, g.vocab_size - 16, (2, 9), generator=gen)
    ids2 = torch.cat([ids.expand(2, -1), ans], 1)
    images2, qids2 = images.expand(2, *images.shape[1:]).contiguous(), qids.expand(2, -1).contiguous()
    mask = torch.zeros_like(ids2)
    mask[:, n_prompt:] = 1
    ref_logps = torch.tensor([-30.0, -28.5])
    beta = 0.1
    te = TrainEngine(g, sd16, device="cuda", lora=LoraSpec(r, s, p, TARGETS))
    te.zero_grad()
    torch.manual_seed(7)
    st = te.dpo_forward_backward(images2.cuda(), ids2.cuda(), qids2.cuda(), mask.cuda(), ref_logps.cuda(), beta)
    torch.cuda.synchronize()
    _OracleLora(monkeypatch, None, s, p, _next_seed(7))
    sd = {k: v.float().cuda().requires_grad_(True) for k, v in sd16.items()}
    logits = O.forward_logits(sd, ids2.cuda(), images2.cuda(), qids2.cuda(), g)
    _, allp, _ = O.dpo_per_token_logps(logits, ids2.cuda(), mask.cuda())
    loss = -F.logsigmoid(beta * ((allp[0] - allp[1]) - (ref_logps[0] - ref_logps[1]).cuda()))
    loss.backward()
    assert abs(float(st[0]) - float(loss)) < 2e-2 * max(1.0, float(loss)), (st, float(loss))
    ref_g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}
    bad, n_lora = _compare_grads(te, ref_g)
    assert not bad, bad[:6]
    assert n_lora > 0


# ------------------------------------------------------------------------------------------------
# GPU: the reference's flows through the surface
# ------------------------------------------------------------------------------------------------
def _surface_model(family="qwen3", seed=5):
    from u2tokenizer_b200.geometry import Geometry
    model = _tiny_model(family, device="cuda", tie=(family == "llama"))
    g = Geometry.from_hf(model.config)
    sd16 = synthetic_state_dict(g, seed=seed, device="cpu", dtype=BF)
    sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
    model.load_state_dict(sd16, strict=False)
    model.generation_config.eos_token_id = None
    return model, g


def _peft(model, dropout=0.05):
    from u2tokenizer_b200.lora import LoraConfig, get_peft_model
    return get_peft_model(model, LoraConfig(r=16, lora_alpha=32, target_modules=reference_linear_names(model),
                                            lora_dropout=dropout, bias="none", task_type="CAUSAL_LM"))


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_stage1_flow_trains_and_checkpoint_round_trips(family):
    model, g = _surface_model(family)
    model.requires_grad_(False)               # freeze_backbone
    peft = _peft(model)
    for n, p in peft.named_parameters():    # the reference's unfreeze loop
        if any(x in n for x in IGNORE):
            p.requires_grad = True
    peft.print_trainable_parameters()
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=10)
    labels = ids.clone()
    labels[:, :g.num_3d_query_token + 1] = -100
    batch = dict(images=images.cuda(), input_ids=ids.cuda(), labels=labels.cuda(), question_ids=qids.cuda(),
                 attention_mask=torch.ones_like(ids).cuda())
    peft.train()
    opt = torch.optim.AdamW([p for p in peft.parameters() if p.requires_grad], lr=5e-3)
    bases = {n: p.detach().clone() for n, p in peft.named_parameters() if ".base_layer." in n}
    losses = []
    torch.manual_seed(0)
    for _ in range(4):
        opt.zero_grad(set_to_none=True)
        out = peft(**batch)
        out.loss.backward()
        losses.append(float(out.loss))
        for n, p in peft.named_parameters():
            assert (p.grad is not None) == (p.requires_grad and p.grad is not None), n
        opt.step()
    assert losses[-1] < losses[0], losses
    assert all(torch.equal(p, bases[n]) for n, p in peft.named_parameters() if ".base_layer." in n)
    assert any(p.grad is not None and p.grad.abs().max() > 0 for n, p in peft.named_parameters() if "lora_A" in n)
    # model_with_lora.bin -> a fresh PEFT wrapper, strict=True (evalscipt/ourmodel_ctrate.py:77-110)
    sd = {k: v.detach().cpu().clone() for k, v in peft.state_dict().items()}
    peft.eval()
    with torch.no_grad():
        lg = peft(images=batch["images"], input_ids=batch["input_ids"], question_ids=batch["question_ids"]).logits
    fresh, _ = _surface_model(family, seed=77)
    fresh = _peft(fresh)
    fresh.load_state_dict(sd, strict=True)
    fresh.eval()
    with torch.no_grad():
        lg2 = fresh(images=batch["images"], input_ids=batch["input_ids"], question_ids=batch["question_ids"]).logits
    assert torch.equal(lg, lg2)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen3", "llama"])
def test_generate_on_wrapper_equals_merged_and_oracle(family):
    from u2tokenizer_b200.lora import merged_weights
    model, g = _surface_model(family, seed=9)
    peft = _peft(model, dropout=0.1)
    gen = torch.Generator().manual_seed(2)
    with torch.no_grad():   # trained-looking adapters: B != 0
        for n, p in peft.named_parameters():
            if "lora_B" in n:
                p.copy_((torch.randn(p.shape, generator=gen) * 0.05).to(BF))
    peft.eval()
    images, ids, qids = synthetic_inputs(g, batch=2, frames=2, n_question=6, lt=12)
    kw = dict(question_ids=qids.cuda(), max_new_tokens=6, do_sample=False)
    got = peft.generate(images.cuda(), ids.cuda(), **kw)
    pl = peft.per_token_logps(images=images.cuda(), input_ids=ids.cuda(), question_ids=qids.cuda())
    merged_sd = {k: v.float().cpu() for k, v in merged_weights(model).items()}
    plain = peft.merge_and_unload()
    assert not any(".lora_" in k or ".base_layer." in k for k in plain.state_dict())
    assert type(plain).__name__ in ("U2Qwen3ForCausalLM", "U2LlamaForCausalLM")
    got_m = plain.generate(images.cuda(), ids.cuda(), **kw)
    assert torch.equal(got, got_m)
    pl_m = plain.per_token_logps(images=images.cuda(), input_ids=ids.cuda(), question_ids=qids.cuda())
    assert torch.equal(pl["per_token_logps"], pl_m["per_token_logps"])
    sd = {k: v.float().cpu() for k, v in plain.state_dict().items() if "rotary" not in k}
    for k, v in merged_sd.items():
        assert torch.equal(sd[k], v)
    with torch.no_grad():
        ref_logits = O.forward_logits(sd, ids, images, qids, g)
        ref_ids, margins = O.greedy_generate(sd, ids, images, qids, g, max_new_tokens=6)
        lg = plain(images=images.cuda(), input_ids=ids.cuda(), question_ids=qids.cuda()).logits.float().cpu()
    assert rel_err(lg, ref_logits) < 3e-2 and cosine(lg, ref_logits) > 0.999
    thr = 4.0 * (lg - ref_logits).abs().max().item()
    for b in range(got.shape[0]):
        low = (margins[b] < thr).nonzero()
        upto = int(low[0]) if len(low) else got.shape[1]
        assert torch.equal(got[b, :upto].cpu(), ref_ids[b, :upto]), (got[b], ref_ids[b], margins[b])
