"""The lossless 13-bit packing of the decode-linear weights (u2_dlinear_pack_bf16, csrc/dlinear_wgmma.cu).

CPU: a pure-torch reference packer / unpacker of the unit layout round-trips adversarial units bit for bit, and a
word-level mirror of the kernel's unpack arithmetic (unpack_word) reproduces the bf16 bits from the reference bytes.
GPU: the CUDA packer writes the reference bytes, and ops.dlinear / ops.dlinear_multi on packed weights return exactly
what they return on the bf16 weights."""
import numpy as np
import pytest
import torch

UNIT = 13328
SM_OFF, NIB_OFF, HI_OFF = 16, 16 + 8192, 16 + 8192 + 4096


def _fragment_index():
    """rows, cols [128 threads, 32 words, 2 halves] of the wgmma A-fragment element each packed weight belongs to."""
    t = torch.arange(128).view(128, 1, 1)
    R = torch.arange(32).view(1, 32, 1)
    h = torch.arange(2).view(1, 1, 2)
    w, l = t // 32, t % 32
    mh, ks, r = R // 16, (R // 4) % 4, R % 4
    rows = mh * 64 + w * 16 + l // 4 + 8 * (r % 2)
    cols = ks * 16 + 2 * (l % 4) + 8 * (r // 2) + h
    return rows.expand(128, 32, 2), cols.expand(128, 32, 2)


def _units(w: torch.Tensor) -> torch.Tensor:
    """[units, 128, 64] int64 bf16 bit patterns, tile-major; rows >= N are +0."""
    N, K = w.shape
    T = -(-N // 128)
    bits = torch.zeros(T * 128, K, dtype=torch.int64)
    bits[:N] = w.view(torch.int16).to(torch.int64) & 0xFFFF
    return bits.view(T, 128, K // 64, 64).permute(0, 2, 1, 3).reshape(-1, 128, 64)


def ref_pack(w: torch.Tensor):
    """Reference packer: (bytes uint8 [units * 13328], number of units that do not fit)."""
    units = _units(w)
    U = units.shape[0]
    rows, cols = _fragment_index()
    x = units[:, rows, cols]                                        # [U, 128, 32, 2]
    e = (x >> 7) & 0xFF
    emax = e.view(U, -1).max(dim=1).values
    base = (emax - 31).clamp(min=0).view(U, 1, 1, 1)
    bad = int(((e != 0) & (e <= base)).view(U, -1).any(dim=1).sum())
    c = torch.where(e == 0, torch.zeros_like(e), (e - base) & 31)
    out = torch.zeros(U, UNIT, dtype=torch.uint8)
    out[:, 0:4] = torch.stack([(base.view(U) >> (8 * i)) & 0xFF for i in range(4)], dim=1).to(torch.uint8)
    sm = (((x >> 8) & 0x80) | (x & 0x7F)).view(U, 128, 64)          # byte 2R + h of thread t
    j = torch.arange(64)
    t = torch.arange(128).view(128, 1)
    pos = SM_OFF + ((j // 16) * 128 + t) * 16 + j % 16              # [128, 64]
    out[:, pos.reshape(-1)] = sm.reshape(U, -1).to(torch.uint8)
    R = torch.arange(32).view(1, 1, 32, 1)
    h = torch.arange(2).view(1, 1, 1, 2)
    nib = ((c & 15) << (4 * (R % 4) + 16 * h)).view(U, 128, 8, 4, 2).sum(dim=(3, 4))   # word q = R // 4
    hi = ((c >> 4) << (R % 16 + 16 * h)).view(U, 128, 2, 16, 2).sum(dim=(3, 4))       # word u = R // 16
    q = torch.arange(8)
    for b in range(4):
        out[:, (NIB_OFF + ((q // 4) * 128 + t) * 16 + 4 * (q % 4) + b).reshape(-1)] = \
            ((nib >> (8 * b)) & 0xFF).reshape(U, -1).to(torch.uint8)
        u = torch.arange(2)
        out[:, (HI_OFF + 8 * t + 4 * u + b).reshape(-1)] = ((hi >> (8 * b)) & 0xFF).reshape(U, -1).to(torch.uint8)
    return out.view(-1), bad


def _words(packed: torch.Tensor, U: int):
    """Per unit: base [U], s<<7|m words [U, 128, 16], nibble words [U, 128, 8], high-bit words [U, 128, 2] (uint32)."""
    b = packed.view(U, UNIT).numpy()
    w32 = lambda a: a.copy().view(np.uint32).astype(np.uint64)
    base = w32(b[:, 0:4])[:, 0]
    sm = w32(b[:, SM_OFF:NIB_OFF].reshape(U, 4, 128, 16).transpose(0, 2, 1, 3).reshape(U, 128, 64))
    nib = w32(b[:, NIB_OFF:HI_OFF].reshape(U, 2, 128, 16).transpose(0, 2, 1, 3).reshape(U, 128, 32))
    hi = w32(b[:, HI_OFF:UNIT].reshape(U, 128, 8))
    return base, sm, nib, hi


def _prmt_sign(x, sel):
    """prmt.b32 x, 0, sel (with selector bit 3 = replicate the byte's sign)."""
    out = np.zeros_like(x)
    for n in range(4):
        s = (sel >> (4 * n)) & 0xF
        byte = (x >> np.uint64(8 * (s & 7))) & np.uint64(0xFF)
        if s & 8:
            byte = np.where(byte & np.uint64(0x80), np.uint64(0xFF), np.uint64(0))
        out |= byte << np.uint64(8 * n)
    return out


def kernel_unpack(packed: torch.Tensor, U: int) -> torch.Tensor:
    """Mirror of the kernel's unpack_word: [U, 128 threads, 32 words] bf16x2 fragment words (uint32)."""
    base, sm, nib, hi = _words(packed, U)
    M = np.uint64(0xFFFFFFFF)
    b7 = ((base << np.uint64(7)) * np.uint64(0x10001)) & M
    out = np.zeros((U, 128, 32), dtype=np.uint64)
    for R in range(32):
        i, j = R & 3, R & 15
        n, hw, s = nib[:, :, R >> 2], hi[:, :, R >> 4], sm[:, :, R >> 1]
        ns = ((n << np.uint64(7 - 4 * i)) & M) if i < 2 else (n >> np.uint64(4 * i - 7))
        hs = ((hw << np.uint64(11 - j)) & M) if j <= 11 else (hw >> np.uint64(j - 11))
        c7 = (ns & np.uint64(0x07800780)) | (hs & np.uint64(0x08000800))
        nz = _prmt_sign((c7 + np.uint64(0x7F807F80)) & M, 0xBB99)
        e7 = (c7 + (nz & b7[:, None])) & M
        z = _prmt_sign(s, 0x3322 if R & 1 else 0x1100)
        out[:, :, R] = (z & np.uint64(0x807F807F)) | e7
    return torch.from_numpy(out.astype(np.int64))


def ref_unpack(packed: torch.Tensor, N: int, K: int) -> torch.Tensor:
    """bf16 [N, K] from the packed bytes (through the kernel's arithmetic)."""
    T, KB = -(-N // 128), K // 64
    U = T * KB
    words = kernel_unpack(packed, U)                                  # [U, 128, 32]
    x = torch.stack([words & 0xFFFF, (words >> 16) & 0xFFFF], dim=-1)  # [U, 128, 32, 2]
    rows, cols = _fragment_index()
    units = torch.zeros(U, 128, 64, dtype=torch.int64)
    units[:, rows.reshape(-1), cols.reshape(-1)] = x.reshape(U, -1)
    bits = units.view(T, KB, 128, 64).permute(0, 2, 1, 3).reshape(T * 128, K)[:N]
    return bits.to(torch.int32).to(torch.int16).view(torch.bfloat16)


def _bf16(bits) -> torch.Tensor:
    return torch.as_tensor(np.asarray(bits, dtype=np.uint16).astype(np.int16)).view(torch.bfloat16)


def _gauss(N, K, std, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(N, K, generator=g) * std).to(torch.bfloat16)


def _assert_roundtrip(w):
    packed, bad = ref_pack(w)
    assert bad == 0
    back = ref_unpack(packed, *w.shape)
    assert torch.equal(back.view(torch.int16), w.view(torch.int16))


def test_roundtrip_gaussian_and_ragged_rows():
    _assert_roundtrip(_gauss(256, 128, 0.02))
    _assert_roundtrip(_gauss(200, 192, 1 / 64, seed=1))  # N not a multiple of 128: rows >= N are +0


def test_roundtrip_zeros_subnormals_negative_zero():
    w = _gauss(128, 64, 0.02).view(torch.int16).clone()
    w[0, :8] = _bf16([0x0000, 0x8000, 0x0001, 0x807F, 0x0040, 0x8001, 0x007F, 0x0000]).view(torch.int16)
    _assert_roundtrip(w.view(torch.bfloat16))


def test_roundtrip_window_edges():
    # emax = 140 -> base 109: exponents 110 (c = 1) and 140 (c = 31) are the edges of the window
    e = np.full((128, 64), 125, dtype=np.uint16)
    e[3, 5], e[100, 63], e[64, 0] = 110, 140, 0
    m = (np.arange(128 * 64, dtype=np.uint16).reshape(128, 64) * 37) & 0x7F
    s = (np.arange(128 * 64, dtype=np.uint16).reshape(128, 64) % 3 == 0).astype(np.uint16) << 15
    _assert_roundtrip(_bf16(s | (e << 7) | m))


def test_roundtrip_small_emax_uses_base_zero():
    e = (np.arange(128 * 64, dtype=np.uint16).reshape(128, 64) % 31)  # emax 30 < 31: base 0, codes are the exponents
    packed, bad = ref_pack(_bf16((e << 7) | 0x55))
    assert bad == 0 and int(packed[0]) == 0
    _assert_roundtrip(_bf16((e << 7) | 0x55))


def test_span_of_32_is_not_packable():
    e = np.full((128, 64), 125, dtype=np.uint16)
    e[7, 9], e[8, 9] = 151, 119  # emax 151 -> base 120: exponent 119 (and 120) fall outside
    assert ref_pack(_bf16(e << 7))[1] == 1
    e[8, 9] = 120
    assert ref_pack(_bf16(e << 7))[1] == 1
    e[8, 9] = 121  # span 151 - 121 = 30 fits
    assert ref_pack(_bf16(e << 7))[1] == 0
    # one bad unit of three
    w = torch.cat([_gauss(128, 64, 0.02), _bf16(np.where(np.arange(64) == 0, 151, 119).astype(np.uint16)[None].repeat(128, 0) << 7),
                   _gauss(128, 64, 0.02, seed=3)], dim=1)
    assert ref_pack(w)[1] == 1


def test_roundtrip_inf_nan_inside_window():
    w = _gauss(128, 128, 1e37, seed=5).view(torch.int16).clone()  # exponents near 249: Inf / NaN (255) are in the window
    w[1, 2], w[3, 4], w[5, 6], w[7, 70] = _bf16([0x7F80, 0xFF80, 0x7FC1, 0xFFC1]).view(torch.int16)  # +-Inf, +-NaN payload
    _assert_roundtrip(w.view(torch.bfloat16))


def test_packed_size():
    packed, _ = ref_pack(_gauss(130, 128, 0.02))
    assert packed.numel() == 2 * 2 * UNIT and UNIT == 16 + 128 * 64 * 13 // 8


# ------------------------------------------------------------------------------------------------------------ GPU
QWEN3_8B = [(6144, 4096), (4096, 4096), (24576, 4096), (4096, 12288), (151936, 4096)]


def _dev_weight(N, K, seed, std=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(N, K, device="cuda", generator=g) * (std or K ** -0.5)).to(torch.bfloat16)


def _ws(N, K):
    from u2tokenizer_b200 import ops
    return dict(ws=ops.dlinear_new_ws(ops.dlinear_ws_elems(N, K)),
                counters=torch.zeros((N + 63) // 64 + 8, device="cuda", dtype=torch.int32))


@pytest.mark.gpu
def test_cuda_packer_writes_the_reference_bytes():
    from u2tokenizer_b200 import ops
    for (N, K, std) in [(256, 128, 0.02), (200, 192, 1 / 64), (4096, 256, 0.02)]:
        w = _dev_weight(N, K, 11, std)
        w[0, :4] = torch.tensor([0.0, -0.0, 1e-39, float("inf")], device="cuda").to(torch.bfloat16) if N == 200 else w[0, :4]
        pk = ops.dlinear_pack(w)
        ref, bad = ref_pack(w.cpu())
        if bad:
            assert pk is None
            continue
        assert pk is not None and torch.equal(pk.buf.cpu(), ref)


@pytest.mark.gpu
def test_unpackable_matrix_falls_back_to_bf16():
    from u2tokenizer_b200 import ops
    w = _dev_weight(256, 128, 3)
    w[130, 64] = 1e30  # span > 31 exponents in one unit
    assert ops.dlinear_pack(w) is None
    x = torch.randn(4, 128, device="cuda").to(torch.bfloat16)
    y = torch.empty(4, 256, device="cuda", dtype=torch.bfloat16)
    ops.dlinear(x, w, y, **_ws(256, 128))
    ref = (x.float() @ w.float().t())
    torch.testing.assert_close(y.float(), ref, rtol=2e-2, atol=1e-2 * ref.abs().max().item())


def _both(x, w, pk, out_shape, out_dtype, **kw):
    from u2tokenizer_b200 import ops
    outs = []
    for ww in (w, pk):
        N, K = w.shape
        y = torch.zeros(out_shape, device="cuda", dtype=out_dtype)
        kk = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
        ops.dlinear(x, ww, y, **_ws(N, K), **kk)
        torch.cuda.synchronize()
        outs.append((y, {k: v for k, v in kk.items() if isinstance(v, torch.Tensor)}))
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("N,K", QWEN3_8B + [(3072 * 3, 3072), (8192 * 2, 3072), (3072, 8192), (4160, 4096), (32064, 3072)])
@pytest.mark.parametrize("B", [1, 4, 5, 16])
def test_packed_dlinear_equals_bf16(N, K, B):
    from u2tokenizer_b200 import ops
    w = _dev_weight(N, K, N + K)
    pk = ops.dlinear_pack(w)
    assert pk is not None
    x = (torch.randn(B, K, device="cuda") * 0.5).to(torch.bfloat16)
    res = (torch.randn(B, N, device="cuda") * 0.1).to(torch.bfloat16)
    ssq_in = (torch.rand(16, device="cuda") * K)
    gam = torch.rand(N, device="cuda") + 0.5
    forms = [
        ((B, N), torch.float32, {}),
        ((B, N), torch.bfloat16, dict(ssq_in=ssq_in, eps=1e-6)),
        ((B, N), torch.bfloat16, dict(residual=res, gamma_next=gam, xg=torch.zeros(B, N, device="cuda", dtype=torch.bfloat16),
                                      ssq_out=torch.zeros(16, device="cuda"), ssq_zero=torch.ones(16, device="cuda"))),
    ]
    if N % 2 == 0:
        forms.append(((B, N // 2), torch.bfloat16, dict(ssq_in=ssq_in, eps=1e-6, silu_pair=True)))
    for shape, dt, kw in forms:
        (ya, ta), (yb, tb) = _both(x, w, pk, shape, dt, **kw)
        assert torch.equal(ya, yb), (N, K, B, sorted(kw))
        for k in ta:
            assert torch.equal(ta[k], tb[k]), (N, K, B, k)


@pytest.mark.gpu
def test_packed_dlinear_multi_chain_equals_bf16():
    """o_proj -> gate|up -> down -> next qkv in one launch, Qwen3-8B shapes, packed vs bf16."""
    from u2tokenizer_b200 import ops
    E, I, Q = 4096, 12288, 6144
    B = 4
    wo, wgu, wd, wq = _dev_weight(E, E, 1), _dev_weight(2 * I, E, 2), _dev_weight(E, I, 3), _dev_weight(Q, E, 4)
    pks = [ops.dlinear_pack(t) for t in (wo, wgu, wd, wq)]
    assert all(p is not None for p in pks)
    g2, g1 = torch.rand(E, device="cuda") + 0.5, torch.rand(E, device="cuda") + 0.5
    ctx0 = (torch.randn(B, E, device="cuda") * 0.5).to(torch.bfloat16)
    x0 = (torch.randn(B, E, device="cuda") * 0.5).to(torch.bfloat16)
    results = []
    for ws_list in ((wo, wgu, wd, wq), pks):
        wse = max(ops.dlinear_ws_elems(n, k) for n, k in [(E, E), (2 * I, E), (E, I), (Q, E)])
        ws = ops.dlinear_new_ws(wse, lead=(2,))
        cnt = torch.zeros(2, (2 * I + 63) // 64 + 8, device="cuda", dtype=torch.int32)
        gridbar = torch.zeros(4, device="cuda", dtype=torch.int32)
        step = torch.ones(1, device="cuda", dtype=torch.int32)
        x, ctx = x0.clone(), ctx0.clone()
        xg_a, xg_b = torch.zeros(B, E, device="cuda", dtype=torch.bfloat16), torch.zeros(B, E, device="cuda", dtype=torch.bfloat16)
        act = torch.zeros(B, I, device="cuda", dtype=torch.bfloat16)
        qkv = torch.zeros(B, Q, device="cuda", dtype=torch.bfloat16)
        ssq_a, ssq_b = torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda")
        c0, c1 = dict(ws=ws[0], counters=cnt[0]), dict(ws=ws[1], counters=cnt[1])
        chain = [
            (ctx, ws_list[0], x, dict(residual=x, gamma_next=g2, xg=xg_a, ssq_out=ssq_a, ssq_zero=ssq_b, **c0)),
            (xg_a, ws_list[1], act, dict(ssq_in=ssq_a, eps=1e-6, silu_pair=True, **c1)),
            (act, ws_list[2], x, dict(residual=x, gamma_next=g1, xg=xg_b, ssq_out=ssq_b, ssq_zero=ssq_a, **c0)),
            (xg_b, ws_list[3], qkv, dict(ssq_in=ssq_b, eps=1e-6, **c1)),
        ]
        ops.dlinear_multi(chain, gridbar=gridbar, step_dev=step)
        torch.cuda.synchronize()
        results.append((x, act, qkv, xg_a, xg_b, ssq_b))
    for a, b in zip(*results):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_dlinear_multi_refuses_mixed_weight_formats():
    from u2tokenizer_b200 import ops
    w1, w2 = _dev_weight(256, 128, 1), _dev_weight(128, 128, 2)
    x = torch.randn(2, 128, device="cuda").to(torch.bfloat16)
    y1 = torch.empty(2, 256, device="cuda", dtype=torch.bfloat16)
    y2 = torch.empty(2, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="weight format"):
        ops.dlinear_multi([(x, ops.dlinear_pack(w1), y1, _ws(256, 128)), (x, w2, y2, _ws(256, 128))],
                          gridbar=torch.zeros(4, device="cuda", dtype=torch.int32),
                          step_dev=torch.ones(1, device="cuda", dtype=torch.int32))


# ----------------------------------------------------------------------------------- engine: packed vs bf16 decode
def _engine_8b_widths(layers=2, **over):
    """Qwen3-8B decoder widths (bigram head, so greedy ids have decisive margins) with a reduced layer count."""
    from common import tiny_geometry
    from u2tokenizer_b200.engine import U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g = tiny_geometry(hidden_size=4096, intermediate_size=12288, num_hidden_layers=layers, num_attention_heads=32,
                      num_key_value_heads=8, head_dim=128, vocab_size=151936, **over)
    eng = U2Engine(g, synthetic_state_dict(g, seed=5, device="cuda", dtype=torch.bfloat16, bigram=1.0), device="cuda")
    return g, eng


def _both_formats(eng, fn):
    outs = []
    for bf16 in (False, True):
        eng._decode_bf16 = bf16
        eng._gen_state = None  # a captured decode step holds the weight pointers of its format
        outs.append(fn())
        torch.cuda.synchronize()
    eng._decode_bf16 = False
    return outs


@pytest.mark.gpu
def test_generate_ids_identical_with_packed_and_bf16_weights():
    from u2tokenizer_b200.engine import BeamSearch
    g, eng = _engine_8b_widths()
    assert len(eng._packed) == 4 * g.num_hidden_layers + 1  # every decoder matrix and the head
    gen = torch.Generator(device="cuda").manual_seed(7)
    emb = (torch.randn(4, 24, g.hidden_size, device="cuda", generator=gen) * 0.02).bfloat16()
    greedy = _both_formats(eng, lambda: eng.generate_greedy(emb, 32))
    assert torch.equal(*greedy)
    sampled = _both_formats(eng, lambda: eng.generate(emb, 24, do_sample=True, temperature=0.9, top_k=40, top_p=0.95,
                                                      seed=123))
    assert torch.equal(*sampled)
    beams = _both_formats(eng, lambda: eng.generate(emb[:2], 16, beam=BeamSearch(num_beams=4)))
    assert torch.equal(beams[0], beams[1])


@pytest.mark.gpu
def test_engine_keeps_bf16_for_a_matrix_that_does_not_pack():
    """A layer whose down projection has a unit spanning more than 31 exponents streams bf16 in that layer's launch
    and still generates what the all-bf16 decode step generates."""
    from common import tiny_geometry
    from u2tokenizer_b200.engine import U2Engine
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    g = tiny_geometry(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, head_dim=64, vocab_size=1000)
    sd = synthetic_state_dict(g, seed=9, device="cuda", dtype=torch.bfloat16, bigram=1.0)
    sd["model.layers.1.mlp.down_proj.weight"][3, 7] = 1e20
    eng = U2Engine(g, sd, device="cuda")
    assert (1, "wdown") not in eng._packed and (0, "wdown") in eng._packed
    emb = (torch.randn(3, 10, g.hidden_size, device="cuda") * 0.02).bfloat16()
    a, b = _both_formats(eng, lambda: eng.generate_greedy(emb, 12))
    assert torch.equal(a, b)
