"""Training side of the hot path: forward with saved activations + hand-written backward over the C-ABI kernels.

What the reference gets from `model(**batch)` + HF Trainer / DeepSpeed (src/train/train_stage1.py:244-250,
config/ds_config.json:27-39; src/train/dpo_u2trainer.py:185-359 for stage 2) is done here by

  * `TrainEngine.forward_backward(...)`  - vision tower -> projector -> mu2-tokenizer -> splice -> decoder -> loss head,
    every activation the backward needs kept in HBM, then the backward pass: dgrad / wgrad and the attention
    contractions on the wgmma GEMM (transposed operands, no copies), everything else on train_kernels.cu; with
    `checkpoint` set (HF gradient_checkpointing_enable()) every repeated block keeps only its input and output and is
    recomputed in the backward (`_segment`);
  * flat parameter / gradient buffers in a TRAINING LAYOUT (q|k|v, gate|up, wk|wv adjacent, so that one GEMM produces the
    fused gradient; every reference parameter is a contiguous slice, the nn.Parameters of the HF-style module are
    re-pointed at those slices);
  * `TrainEngine.optimizer_step(...)` - ZeRO-1 over the data-parallel group: bucketed NCCL reduce-scatter of the bf16
    matrix gradients (2e8-element buckets like the reference's DeepSpeed config), fused AdamW on the local 1/W shard
    (fp32 master / m / v), all-gather of the updated bf16 parameters; the small vector parameters (biases, norms,
    relative-bias tables, position / cls / query embeddings: fp32 gradients) are all-reduced and updated replicated.

No arithmetic in torch: torch provides memory, streams, NCCL. There is no CPU path.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from . import train_ops as T
from .engine import REL_MAX, _pad8
from .geometry import Geometry
from .synthetic import param_shapes

BF16, F32 = torch.bfloat16, torch.float32
_VEC_SUFFIX = ("relative_bias", "dynamic_pool.gate_fc.weight", "cls_token", "position_embeddings", "query_tokens")


# LoRA targets of one decoder layer in mask-stream order (u2_lora_desc.stream = layer * 8 + index), grouped as the training
# forward runs them: the members of a group share one input and one fused base GEMM
LORA_TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
LORA_GROUPS = (("self_attn.", ("q_proj", "k_proj", "v_proj")), ("self_attn.", ("o_proj",)), ("mlp.", ("gate_proj", "up_proj")),
               ("mlp.", ("down_proj",)))
# Phi-3 (HF Phi3: fused qkv_proj, [gate; up] gate_up_proj): one adapter per group, on the same four fused GEMMs. Its
# mask streams are PHI3_STREAM_BASE + layer * 4 + index, disjoint from the Llama / Qwen3 streams above
PHI3_LORA_TARGETS = ("qkv_proj", "o_proj", "gate_up_proj", "down_proj")
PHI3_LORA_GROUPS = (("self_attn.", ("qkv_proj",)), ("self_attn.", ("o_proj",)), ("mlp.", ("gate_up_proj",)),
                    ("mlp.", ("down_proj",)))
PHI3_STREAM_BASE = 1 << 24


def lora_targets(g: Geometry) -> Tuple[str, ...]:
    return PHI3_LORA_TARGETS if g.decoder_family == "phi3" else LORA_TARGETS


def lora_groups(g: Geometry):
    return PHI3_LORA_GROUPS if g.decoder_family == "phi3" else LORA_GROUPS


def lora_stream(g: Geometry, layer: int, target: str) -> int:
    """Dropout-mask stream of one adapter (u2_lora_desc.stream, documented in u2b200_train.h)."""
    if g.decoder_family == "phi3":
        return PHI3_STREAM_BASE + layer * 4 + PHI3_LORA_TARGETS.index(target)
    return layer * 8 + LORA_TARGETS.index(target)


@dataclass(frozen=True)
class LoraSpec:
    """LoRA adapters on the decoder linears: rank r, scaling = lora_alpha / r, dropout p, short names of the targets."""
    r: int
    scaling: float
    dropout: float
    targets: Tuple[str, ...]

    def names(self, layer: int, prefix: str, t: str) -> Tuple[str, str, str]:
        """(base weight, lora_A, lora_B) parameter names of target t of a layer (PEFT's module layout)."""
        m = f"model.layers.{layer}.{prefix}{t}."
        return m + "weight", m + "lora_A.default.weight", m + "lora_B.default.weight"


def is_vector_param(name: str, shape) -> bool:
    """Vector class: parameters whose gradient is produced by reductions in fp32 (and that the kernels read as fp32, or
    that are tiny bf16 tables): everything 1-D plus the tables named in _VEC_SUFFIX."""
    return len(shape) == 1 or name.endswith(_VEC_SUFFIX)


def training_order(g: Geometry) -> Tuple[List[str], List[str]]:
    """(matrix names, vector names) in flat-buffer order. Adjacent on purpose: q|k|v, wk|wv, gate|up and their biases."""
    shapes = param_shapes(g)
    mats, vecs = [], []
    # param_shapes lists q,k,v / gate,up (decoder) and wq,wk,wv,dense (tokenizer, weight and bias alternating) in
    # order: splitting into the matrix and the vector class keeps the weights of a fused group adjacent, and their biases
    for n, s in shapes.items():
        (vecs if is_vector_param(n, s) else mats).append(n)
    return mats, vecs


class Layout:
    """Offsets of every parameter in the flat buffers. W (bf16): [matrix region | vector region | frozen region]; Gm
    (bf16): matrix region; V32 / Gv (fp32): vector region. The frozen region holds the base weights of the LoRA targets
    (empty without LoRA): no gradient slot, no optimizer state. With LoRA the matrix region holds the adapters in place
    of those base weights, the A's of a fused group adjacent (q|k|v, gate|up), then its B's."""

    def __init__(self, g: Geometry, world_size: int = 1, bucket_elems: int = 200_000_000, lora: Optional[LoraSpec] = None):
        self.shapes = dict(param_shapes(g))
        mats, vecs = training_order(g)
        self.frozen_names: List[str] = []
        if lora is not None:
            mats = self._lora_order(g, mats, lora)
        self.mat_names, self.vec_names = mats, vecs
        self.mat_off, self.vec_off = {}, {}
        off = 0
        for n in mats:
            self.mat_off[n] = off
            off += (self._numel(n) + 7) // 8 * 8
        self.mat_used = off
        # ZeRO-1 ownership is interleaved by bucket: bucket i is the contiguous region [i * bucket, (i + 1) * bucket) and
        # rank r owns its r-th 1/W slice, so every bucket's reduce-scatter input / all-gather output is a plain view
        W = max(1, world_size)
        self.n_buckets = max(1, (off + bucket_elems - 1) // bucket_elems)
        per = (off + self.n_buckets - 1) // self.n_buckets
        self.bucket = max(8 * W, (per + 8 * W - 1) // (8 * W) * (8 * W))
        self.mat_total = self.n_buckets * self.bucket
        self.piece = self.bucket // W   # elements of one bucket owned by one rank
        self.name_buckets = {}          # matrix name -> buckets its slot intersects
        self.bucket_names = [[] for _ in range(self.n_buckets)]
        for n in mats:
            lo, hi = self.mat_off[n], self.mat_off[n] + self._numel(n)
            bs = list(range(lo // self.bucket, (hi - 1) // self.bucket + 1))
            self.name_buckets[n] = bs
            for b in bs:
                self.bucket_names[b].append(n)
        off = 0
        for n in vecs:
            self.vec_off[n] = off
            off += (self._numel(n) + 7) // 8 * 8
        self.vec_total = max(8, off)
        self.frozen_off = {}
        off = 0
        for n in self.frozen_names:
            self.frozen_off[n] = off
            off += (self._numel(n) + 7) // 8 * 8
        self.frozen_total = off

    def _lora_order(self, g: Geometry, mats: List[str], lora: LoraSpec) -> List[str]:
        """The matrix order with every target's base weight replaced by its adapters (the base moves to frozen_names)."""
        first = {}   # base name of a group's first targeted member -> the group's adapter names (A's, then B's)
        skip = set()
        for li in range(g.num_hidden_layers):
            for pre, members in lora_groups(g):
                tg = [t for t in members if t in lora.targets]
                if not tg:
                    continue
                trip = [lora.names(li, pre, t) for t in tg]
                for base, a, b in trip:
                    out_f, in_f = self.shapes[base]
                    self.shapes[a], self.shapes[b] = (lora.r, in_f), (out_f, lora.r)
                    skip.add(base)
                first[trip[0][0]] = [a for _, a, _ in trip] + [b for _, _, b in trip]
        out = []
        for n in mats:
            if n in skip:
                self.frozen_names.append(n)
                out.extend(first.get(n, ()))
            else:
                out.append(n)
        return out

    def _numel(self, n: str) -> int:
        k = 1
        for d in self.shapes[n]:
            k *= d
        return k

    def adjacent(self, names: Sequence[str]) -> bool:
        if len(names) == 1:
            return True
        tab = next(t for t in (self.mat_off, self.vec_off, self.frozen_off) if names[0] in t)
        for a, b in zip(names[:-1], names[1:]):
            if tab[a] + self._numel(a) != tab[b]:
                return False
        return True


class Var:
    """An activation with its gradient slot (a tape entry's inputs / outputs)."""
    __slots__ = ("v", "g", "ng")

    def __init__(self, v: torch.Tensor, ng: bool = True):
        self.v, self.g, self.ng = v, None, ng


class TrainEngine:
    def __init__(self, geom: Geometry, state_dict: Dict[str, torch.Tensor], device="cuda", world_size: int = 1, rank: int = 0,
                 group=None, trainable: Optional[Dict[str, bool]] = None, bucket_elems: int = 200_000_000,
                 lora: Optional[LoraSpec] = None, checkpoint: bool = False):
        if geom.decoder_dropout:
            # HF applies resid / embd / attention dropout in train mode (modeling_phi3.py); this path has no dropout
            raise NotImplementedError(f"training with decoder dropout {geom.decoder_dropout} (Phi-3 resid_pdrop / "
                                      "embd_pdrop / attention_dropout) is not supported: set them to 0")
        if not torch.cuda.is_available():
            raise RuntimeError("TrainEngine needs a CUDA device: the training path has no CPU implementation")
        from . import _lib
        _lib.load()
        g = self.g = geom
        if g.vision_select_feature != "patch" or g.attn_type not in ("rma", "rope") or g.image_channel != 1:
            raise NotImplementedError("training path: vision_select_feature='patch', attn_type in (rma, rope), 1 channel")
        self.dev = torch.device(device)
        self.world, self.rank, self.group = world_size, rank, group
        self.bucket_elems = bucket_elems
        if lora is not None:
            bad = [t for t in lora.targets if t not in lora_targets(g)]
            if bad or lora.r not in (8, 16, 32, 64) or not 0.0 <= lora.dropout < 1.0:
                raise NotImplementedError(f"LoRA on the training path: targets in {lora_targets(g)}, r in (8, 16, 32, 64), "
                                          f"0 <= dropout < 1 (got {lora})")
        self.lora = lora
        self.lay = Layout(g, world_size=world_size, bucket_elems=bucket_elems, lora=lora)
        L = self.lay
        self.W = torch.zeros(L.mat_total + L.vec_total + L.frozen_total, device=self.dev, dtype=BF16)
        self.V32 = torch.zeros(L.vec_total, device=self.dev, dtype=F32)
        self.Gm = torch.zeros(L.mat_total, device=self.dev, dtype=BF16)
        self.Gv = torch.zeros(L.vec_total, device=self.dev, dtype=F32)
        for n in L.mat_names + L.vec_names + L.frozen_names:
            if n in state_dict:
                self.w(n).copy_(state_dict[n].to(self.dev).view(L.shapes[n]))
            elif n == "lm_head.weight" or ".lora_" in n:
                raise KeyError(n)
        self.tied = g.tie_word_embeddings or "lm_head.weight" not in L.shapes
        self.refresh_vectors()
        # group-level requires_grad (reference: freeze_vision_tower / freeze_backbone / tune_mm_mlp_adapter)
        self.trainable = dict(vit=True, proj=True, u2t=True, dec=True, embed=True, head=True)
        if trainable:
            self.trainable.update(trainable)
        dh = g.hidden_size // g.u2t_num_heads
        self.u2t_inv_freq = (1.0 / (10000 ** (torch.arange(0, dh, 2, dtype=F32) / dh))).to(self.dev)
        from .engine import U2Engine
        self.inv_freq = U2Engine._decoder_inv_freq(self).to(self.dev)
        self.opt = None
        self.tape: List = []
        self.stats = {}
        # gradient exchange overlapped with the backward pass: a bucket's reduce-scatter is issued on the communication
        # stream as soon as the wgrads of every parameter in it have been issued (reference: DeepSpeed overlap_comm,
        # config/ds_config.json:35)
        self.overlap = world_size > 1
        self.comm_stream = torch.cuda.Stream(device=self.dev) if world_size > 1 else None
        self._pending = None
        self._ag_ev = [None] * self.lay.n_buckets   # all-gather completion events of the previous optimizer step
        # Matrix gradients are not zero-filled per step: the first wgrad of a step OVERWRITES its slot (no memset of
        # the 2 bytes / parameter buffer, no accumulating read in the GEMM epilogue), later writers accumulate.
        # _gm_written: names written since zero_grad(); _gm_dirty: names whose slot holds a gradient of any step (a
        # dirty slot that a step does not write is zeroed when its segment's marker fires, see _mark / run_backward).
        self._gm_written = set()
        self._gm_dirty = set()
        self._gm_offs = sorted((L.mat_off[n], n) for n in L.mat_names)
        self._gm_names_cache = {}
        self._lora_seed = 0   # dropout-mask seed of the current forward (0 with p = 0 or outside a training forward)
        # activation checkpointing (HF gradient_checkpointing_enable()): every repeated block of the training tape keeps
        # only its input and output and is recomputed in the backward (see _segment). Read at the start of each training
        # forward; _ckpt is the value the current tape was built with
        self.checkpoint = bool(checkpoint)
        self._ckpt = False

    # =========================================================================================
    # flat-buffer views
    # =========================================================================================
    def _slot(self, n: str):
        L = self.lay
        if n in L.mat_off:
            return L.mat_off[n], L._numel(n), True
        if n in L.frozen_off:
            return L.mat_total + L.vec_total + L.frozen_off[n], L._numel(n), False
        return L.mat_total + L.vec_off[n], L._numel(n), False

    def w(self, n: str) -> torch.Tensor:
        """bf16 parameter view (the module's nn.Parameter aliases this)."""
        off, k, _ = self._slot(n)
        return self.W[off:off + k].view(self.lay.shapes[n])

    def wcat(self, names: Sequence[str]) -> torch.Tensor:
        """Fused 2-D view [sum(out), in] over adjacent matrices."""
        L = self.lay
        assert L.adjacent(names), names
        cols = L.shapes[names[0]][-1]
        k = sum(L._numel(n) for n in names)
        off = self._slot(names[0])[0]
        return self.W[off:off + k].view(k // cols, cols)

    def v32(self, n: str) -> torch.Tensor:
        L = self.lay
        off = L.vec_off[n]
        return self.V32[off:off + L._numel(n)]

    def v32cat(self, names: Sequence[str]) -> torch.Tensor:
        L = self.lay
        assert L.adjacent(names), names
        off = L.vec_off[names[0]]
        return self.V32[off:off + sum(L._numel(n) for n in names)]

    def gm(self, names) -> torch.Tensor:
        """bf16 gradient view of a matrix (or of adjacent matrices, fused)."""
        L = self.lay
        if isinstance(names, str):
            names = [names]
        assert L.adjacent(names), names
        cols = L.shapes[names[0]][-1]
        k = sum(L._numel(n) for n in names)
        off = L.mat_off[names[0]]
        return self.Gm[off:off + k].view(k // cols, cols)

    def gv(self, names) -> torch.Tensor:
        L = self.lay
        if isinstance(names, str):
            names = [names]
        assert L.adjacent(names), names
        off = L.vec_off[names[0]]
        return self.Gv[off:off + sum(L._numel(n) for n in names)]

    def grad(self, n: str) -> torch.Tensor:
        """Gradient of parameter n in its parameter shape: a view of its bf16 slot in Gm (matrices) or its fp32 slot in Gv
        (vectors)."""
        L = self.lay
        buf, off = (self.Gm, L.mat_off[n]) if n in L.mat_off else (self.Gv, L.vec_off[n])
        return buf[off:off + L._numel(n)].view(L.shapes[n])

    def param_grads(self, names: Sequence[str], keep=()) -> List[Optional[torch.Tensor]]:
        """The gradients autograd hands to the module parameters `names` after backward(): matrices get their Gm slot (no
        copy), vectors a view of one bf16 cast of Gv. None for the tied lm_head (its gradient is delivered through
        embed_tokens), for names in `keep` (their p.grad already is the slot, accumulated in place) and for parameters
        without a slot (frozen)."""
        L = self.lay
        gvb = torch.empty(L.vec_total, device=self.dev, dtype=BF16)
        T.cast(self.Gv, gvb)
        out = []
        for n in names:
            if (n == "lm_head.weight" and self.tied) or n in keep:
                out.append(None)
            elif n in L.mat_off:
                out.append(self.grad(n))
            elif n in L.vec_off:
                out.append(gvb[L.vec_off[n]:L.vec_off[n] + L._numel(n)].view(L.shapes[n]))
            else:
                out.append(None)
        return out

    def refresh_vectors(self):
        """fp32 mirrors of the vector parameters (biases, norm weights, bias tables) from their bf16 values."""
        L = self.lay
        T.cast(self.W[L.mat_total:L.mat_total + L.vec_total], self.V32)

    def bind_module(self, model) -> None:
        """Re-point the module's nn.Parameters at the flat buffer (no second copy of the weights); gradients are
        exposed the same way after backward (see param_grads)."""
        sd_names = dict(model.named_parameters())
        for n, p in sd_names.items():
            n = n.replace(".base_layer.", ".")   # a LoRA target's base weight (PEFT module layout)
            if n in self.lay.shapes:
                p.data = self.w(n)
        if self.tied and "lm_head.weight" in sd_names:
            sd_names["lm_head.weight"].data = self.w("model.embed_tokens.weight")

    def zero_grad(self, set_to_zero: bool = False, keep=()):
        """Start a new gradient: the fp32 vector gradients are cleared; the matrix slots are overwritten by their first
        writer of the step (set_to_zero=True also clears them now, e.g. before reading gradients of a partial pass).
        keep: matrix names whose slots already hold a gradient that this pass must ADD to (micro-batch accumulation
        when the module's p.grad aliases the slot)."""
        self.Gv.zero_()
        self._gm_written = set(keep)
        self._gm_dirty.update(keep)
        if set_to_zero:
            assert not keep
            self.Gm.zero_()
            self._gm_dirty = set()

    def _gm_names(self, gw: torch.Tensor):
        """Parameter names covered by a matrix-gradient view (a single matrix or a fused group of adjacent ones)."""
        off = (gw.data_ptr() - self.Gm.data_ptr()) // 2
        key = (off, gw.numel())
        names = self._gm_names_cache.get(key)
        if names is None:
            import bisect
            i = bisect.bisect_left(self._gm_offs, (off, ""))
            names = []
            while i < len(self._gm_offs) and self._gm_offs[i][0] < off + gw.numel():
                names.append(self._gm_offs[i][1])
                i += 1
            assert names and self.lay.mat_off[names[0]] == off, "gradient view does not start at a parameter"
            self._gm_names_cache[key] = names = tuple(names)
        return names

    def _gm_begin_write(self, gw: torch.Tensor) -> bool:
        """Called right before a kernel writes the matrix-gradient view `gw`. Returns True when the kernel has to
        ACCUMULATE (the slot already holds a contribution of this step), False when it may overwrite."""
        names = self._gm_names(gw)
        fresh = [n for n in names if n not in self._gm_written]
        self._gm_written.update(names)
        self._gm_dirty.update(names)
        if len(fresh) == len(names):
            return False
        for n in fresh:   # a fused view after one of its members was written on its own: clear the others, then add
            self.gm(n).zero_()
        return True

    def _gm_clear_stale(self, names):
        """Slots that hold an earlier step's gradient but were not written in this one (a parameter that dropped out of
        the graph) must read as zero before they are reduced / consumed."""
        for n in names:
            if n in self._gm_dirty and n not in self._gm_written:
                self.gm(n).zero_()
                self._gm_dirty.discard(n)

    def wgrad(self, dy: torch.Tensor, x: torch.Tensor, gw: torch.Tensor):
        """gw (+)= dy^T x on the tensor cores; the first write of a step overwrites."""
        T.linear_wgrad(dy, x, gw, accumulate=self._gm_begin_write(gw))

    def _gm_scatter_target(self, name: str) -> torch.Tensor:
        """Gradient slot for a kernel that ADDS into it (embedding scatter): cleared first when this is the step's first
        writer."""
        gw = self.gm(name)
        if not self._gm_begin_write(gw):
            gw.zero_()
        return gw

    # =========================================================================================
    # tape helpers
    # =========================================================================================
    def _acc(self, var: Var, t: torch.Tensor, owned: bool):
        """Deliver a gradient contribution to `var`. owned: nobody else reads `t` afterwards (it may be adopted)."""
        if not var.ng:
            return
        if var.g is None:
            var.g = t if owned else t.clone()
        else:
            T.add_(var.g, t.view(var.g.shape) if t.is_contiguous() else t.contiguous().view(var.g.shape))

    def _backward(self, out: Var, fn):
        """Tape entry of the op that produced `out`: the backward calls fn(out.g) (see _run_tape)."""
        self.tape.append((out, fn))

    def _run_tape(self, tape):
        """Run a tape in reverse. An op's entry (out, fn) runs fn(out.g) only when out received a gradient, and releases
        that gradient right after (a checkpointed segment's recompute relies on every op freeing its output's gradient);
        an entry without an output (marker, segment recompute, loss head) always runs."""
        for out, fn in reversed(tape):
            if out is None:
                fn()
            elif out.g is not None:
                fn(out.g)
                out.g = None

    def _reshape(self, var: Var, shape) -> Var:
        """A Var over a reshaped view of var.v; its gradient is routed back to var."""
        out = Var(var.v.view(shape), var.ng)
        self._backward(out, lambda dy: self._acc(var, dy.view(var.v.shape), owned=True))
        return out

    def _tr(self, group: str) -> bool:
        return bool(self.trainable.get(group, True))

    def _wait_params(self, names: Sequence[str]):
        """The previous step's parameter all-gather runs on the communication stream, bucket by bucket in forward order,
        while this step's forward is already under way: before a segment first reads its weights, make the compute stream
        wait for the buckets that hold them."""
        for n in names:
            for b in self.lay.name_buckets.get(n, ()):
                ev = self._ag_ev[b]
                if ev is not None:
                    torch.cuda.current_stream().wait_event(ev)
                    self._ag_ev[b] = None

    def sync_params(self):
        """Wait for every outstanding parameter all-gather (before anything outside the training forward reads W)."""
        for b, ev in enumerate(self._ag_ev):
            if ev is not None:
                torch.cuda.current_stream().wait_event(ev)
                self._ag_ev[b] = None

    def _mark(self, names: Sequence[str]):
        """Placed on the tape BEFORE the ops of a segment: in the reversed (backward) order it runs right after the
        segment's last gradient kernel has been issued, i.e. when the gradients of `names` are final."""
        names = [n for n in names if n in self.lay.mat_off]
        self._wait_params(names)

        def done():
            self._gm_clear_stale(names)
            if self._pending is None:
                return
            for n in names:
                for b in self.lay.name_buckets[n]:
                    self._pending[b].discard(n)
                    if not self._pending[b] and not self.opt["reduced"][b]:
                        ev = torch.cuda.Event()
                        ev.record()
                        with torch.cuda.stream(self.comm_stream):
                            self.comm_stream.wait_event(ev)
                            self.reduce_bucket(b)
        self.tape.append((None, done))

    def _segment(self, body, x: Var) -> Var:
        """One repeated block (ViT block, SVR layer, TTA layer, decoder layer): out = body(x), body starting with the
        block's _mark. Plain: body's ops go on the tape. Checkpointed: body runs on a local tape that is dropped at once
        (the block's intermediates are freed; only x and out stay alive), and the tape gets one entry that, in the
        backward, runs body(x) again on the same input Vars - same weight views, kernels and arguments, and the LoRA
        dropout seed of this forward, so every value is bit-identical - hands out's gradient to the recomputed output and
        runs the local tape in reverse. External inputs the body closes over (the TTA layers' vis / t_tokens) receive
        their contributions in the plain order, and the block's marker still fires right after its last wgrad."""
        if not self._ckpt:
            return body(x)
        outer, seed = self.tape, self._lora_seed
        self.tape = []
        try:
            out = body(x)
        finally:
            self.tape = outer

        def bwd():
            outer_, seed_ = self.tape, self._lora_seed
            self.tape, self._lora_seed = [], seed
            try:
                out2 = body(x)
                local = self.tape
            finally:
                self.tape, self._lora_seed = outer_, seed_
            out2.g, out.g = out.g, None
            self._run_tape(local)
        self.tape.append((None, bwd))
        return out

    # ---- linear ---------------------------------------------------------------------------------
    def linear(self, x: Var, w: torch.Tensor, gw: Optional[torch.Tensor], bias: Optional[torch.Tensor] = None,
               gbias: Optional[torch.Tensor] = None, residual: Optional[Var] = None, out_rows_pad_zero: bool = False) -> Var:
        """y = x @ w^T + bias (+ residual). gw / gbias: gradient views (None: frozen)."""
        y = ops.linear(x.v, w, bias, residual=residual.v if residual is not None else None)
        out = Var(y, x.ng or gw is not None or (residual is not None and residual.ng))

        def bwd(dy):
            if gw is not None:
                self.wgrad(dy, x.v, gw)
            if gbias is not None:
                T.colsum(dy, gbias)
            if x.ng:
                if x.g is None:
                    x.g = T.linear_dgrad(dy, w)
                else:
                    T.linear_dgrad(dy, w, out=x.g, accumulate=True)
            if residual is not None:
                self._acc(residual, dy, owned=True)
        self._backward(out, bwd)
        return out

    def _param_linear(self, x: Var, weights, biases, group: str, residual: Optional[Var] = None) -> Var:
        """linear() on named parameters: weights / biases one name or a list of adjacent names (one fused GEMM: q|k|v,
        wk|wv, gate|up), biases may be None. Gradient slots only while `group` trains."""
        ws = [weights] if isinstance(weights, str) else weights
        bs = [biases] if isinstance(biases, str) else biases
        gw = gb = None
        if self._tr(group):
            gw, gb = self.gm(ws), (self.gv(bs) if bs else None)
        return self.linear(x, self.wcat(ws), gw, self.v32cat(bs) if bs else None, gb, residual=residual)

    # ---- norms ------------------------------------------------------------------------------------
    def layernorm(self, x: Var, gname: str, bname: str, group: str, eps: float = 1e-5, residual: Optional[Var] = None) -> Var:
        """y = LN(x [+ residual]); the sum is kept for the backward."""
        gamma, beta = self.v32(gname), self.v32(bname)
        if residual is not None:
            s = torch.empty_like(x.v)
            y = ops.layernorm(x.v, gamma, beta, eps, residual=residual.v, sum_out=s)
        else:
            s = x.v
            y = ops.layernorm(x.v, gamma, beta, eps)
        out = Var(y, True)
        dgamma, dbeta = (self.gv(gname), self.gv(bname)) if self._tr(group) else (None, None)

        def bwd(dy):
            if x.ng or (residual is not None and residual.ng) or dgamma is not None:
                pend = x.g if (x.g is not None and residual is None) else None
                dx = T.layernorm_bwd(s, gamma, dy, dres=pend, out=pend, dgamma=dgamma, dbeta=dbeta, eps=eps)
                if pend is None:
                    if residual is not None:
                        self._acc(x, dx, owned=False)
                        self._acc(residual, dx, owned=True)
                    else:
                        self._acc(x, dx, owned=True)
        self._backward(out, bwd)
        return out

    def rmsnorm(self, x: Var, gname: str, group: str, eps: float) -> Var:
        gamma = self.v32(gname)
        y = ops.rmsnorm(x.v, gamma, eps)
        out = Var(y, True)
        dgamma = self.gv(gname) if self._tr(group) else None

        def bwd(dy):
            pend = x.g
            dx = T.rmsnorm_bwd(x.v, gamma, dy, dres=pend, out=pend, dgamma=dgamma, eps=eps)
            if pend is None:
                self._acc(x, dx, owned=True)
        self._backward(out, bwd)
        return out

    # ---- activations --------------------------------------------------------------------------------
    def gelu(self, x: Var) -> Var:
        out = Var(T.gelu(x.v), x.ng)

        def bwd(dy):
            if x.ng:
                self._acc(x, T.gelu_bwd(x.v, dy), owned=True)
        self._backward(out, bwd)
        return out

    def silu_mul(self, gu: Var) -> Var:
        out = Var(ops.silu_mul(gu.v, interleaved=False), gu.ng)

        def bwd(dy):
            if gu.ng:
                self._acc(gu, T.silu_mul_bwd(gu.v, dy), owned=True)
        self._backward(out, bwd)
        return out

    # ---- attention through the GEMM (scores fp32, probabilities bf16 kept for the backward) -----------
    def attention(self, qv: Var, q_view, kv: Var, k_view, vv: Var, v_view, out_shape, scale: float,
                  rel_name: Optional[str] = None, causal: bool = False, group: str = "u2t", recompute: bool = False,
                  window: int = 0) -> Var:
        """q_view / k_view / v_view map the base tensor of a Var (value or gradient, same shape) to the strided 4-D view
        [b, S, heads, dh]. Returns ctx Var [b, Sq, h*dh] (out_shape may pad the token axis: extra rows stay zero).
        window > 0 (causal only): sliding window in the softmax; the backward needs nothing more, P is 0 outside it."""
        q, k, v = q_view(qv.v), k_view(kv.v), v_view(vv.v)
        b, Sq, h, dh = q.shape
        Sk, hk = k.shape[1], k.shape[2]
        G = h // hk
        Skp = _pad8(Sk)
        dev = self.dev
        rel = self.v32(rel_name).view(-1) if rel_name is not None else None
        ctx_full = torch.zeros(out_shape, device=dev, dtype=BF16) if out_shape[1] != Sq else torch.empty(out_shape, device=dev, dtype=BF16)
        ctx = ctx_full[:, :Sq]

        def probs():
            sc = torch.empty(b, h, Sq, Skp, device=dev, dtype=F32)
            p_ = torch.empty(b, h, Sq, Skp, device=dev, dtype=BF16)
            ops.gemm(q, k, sc, M=Sq, N=Sk, K=dh, lda=q.stride(1), ldb=k.stride(1), ldc=Skp, zi=h, zo=b, b_zi_div=G,
                     a_strides=(q.stride(2), q.stride(0)), b_strides=(k.stride(2), k.stride(0)),
                     c_strides=(Sq * Skp, h * Sq * Skp), alpha=scale)
            ops.softmax(sc, p_, n0=b, H=h, S=Sq, n=Sk, in_strides=(h * Sq * Skp, Sq * Skp, Skp),
                        out_strides=(h * Sq * Skp, Sq * Skp, Skp), rel_bias=rel, rel_max=REL_MAX, causal=causal,
                        causal_off=Sk - Sq, zero_pad_to=Skp, window=window if causal else 0)
            return p_
        saved = {}
        if recompute and dh == 64 and h == hk and rel is None and not causal:
            # fused wgmma attention forward (scores never leave the SM); the probabilities are recomputed in the backward
            lse = torch.empty(b, h, Sq, device=dev, dtype=F32)
            ops.flash_attention_d64(q, k, v, ctx, scale, lse=lse)
            saved["lse"] = lse
        else:
            pr0 = probs()
            # ctx = P @ V: V [Sk, dh] is consumed as stored (MN-major B operand: no transposed copy)
            ops.gemm(pr0, v, ctx, M=Sq, N=dh, K=Sk, lda=Skp, ldb=v.stride(1), ldc=ctx.stride(1), zi=h, zo=b, b_zi_div=G,
                     a_strides=(Sq * Skp, h * Sq * Skp), b_strides=(v.stride(2), v.stride(0)), c_strides=(dh, ctx.stride(0)),
                     b_mn=True)
            if not recompute:
                saved["p"] = pr0
            del pr0
        out = Var(ctx_full, qv.ng or kv.ng or vv.ng)
        tr_rel = rel_name is not None and self._tr(group)

        def bwd(dy):
            do = dy[:, :Sq].view(b, Sq, h, dh)
            pr = saved.pop("p", None)
            lse = saved.pop("lse", None)
            if pr is None and lse is not None:
                # P = exp(scale * q.k - lse) straight out of the score GEMM's epilogue (bf16): no fp32 score round trip
                pr = torch.empty(b, h, Sq, Skp, device=dev, dtype=BF16)
                ops.gemm(q, k, pr, M=Sq, N=Sk, K=dh, lda=q.stride(1), ldb=k.stride(1), ldc=Skp, zi=h, zo=b, b_zi_div=G,
                         a_strides=(q.stride(2), q.stride(0)), b_strides=(k.stride(2), k.stride(0)),
                         c_strides=(Sq * Skp, h * Sq * Skp), alpha=scale, epi_op=1, rowvec=lse, rv_strides=(Sq, h * Sq))
            elif pr is None:
                pr = probs()
            # gradient buffers of the operands (first writer allocates; later consumers accumulate)
            fresh = {}
            for var in (qv, kv, vv):
                if id(var) not in fresh and var.ng:
                    fresh[id(var)] = var.g is None
                    if var.g is None:
                        # rows outside the views (ViT padding rows) must read as zero downstream
                        var.g = torch.zeros_like(var.v)
            # dV = P^T @ dO   (per query head, summed over the group for GQA)
            if vv.ng:
                dv = v_view(vv.g)
                self._pt_gemm(pr, do, dv, b, h, hk, Sq, Sk, Skp, dh, 1.0, accumulate=not fresh[id(vv)])
            if lse is not None:
                # dS = P * (dO.V^T - D), D = rowsum(dO * O): formed in the dP GEMM's epilogue, in place of P (bf16)
                D = T.rowdot(do, out.v[:, :Sq].view(b, Sq, h, dh))
                ops.gemm(do, v, pr, M=Sq, N=Sk, K=dh, lda=do.stride(1), ldb=v.stride(1), ldc=Skp, zi=h, zo=b, b_zi_div=G,
                         a_strides=(do.stride(2), do.stride(0)), b_strides=(v.stride(2), v.stride(0)),
                         c_strides=(Sq * Skp, h * Sq * Skp), epi_op=2, rowvec=D, rv_strides=(Sq, h * Sq), mul=pr)
            else:
                dP = torch.empty(b, h, Sq, Skp, device=dev, dtype=F32)
                # dP = dO @ V^T
                ops.gemm(do, v, dP, M=Sq, N=Sk, K=dh, lda=do.stride(1), ldb=v.stride(1), ldc=Skp, zi=h, zo=b, b_zi_div=G,
                         a_strides=(do.stride(2), do.stride(0)), b_strides=(v.stride(2), v.stride(0)),
                         c_strides=(Sq * Skp, h * Sq * Skp))
                # dS = P * (dP - sum(dP * P)) in place of P
                T.softmax_bwd(pr, dP, pr, n0=b, H=h, S=Sq, n=Sk, p_strides=(h * Sq * Skp, Sq * Skp, Skp),
                              dp_strides=(h * Sq * Skp, Sq * Skp, Skp), ds_strides=(h * Sq * Skp, Sq * Skp, Skp),
                              zero_pad_to=Skp)
                del dP
            if tr_rel:
                T.relbias_grad(pr, self.gv(rel_name), n0=b, H=h, S=Sq, n=Sk, strides=(h * Sq * Skp, Sq * Skp, Skp), rel_max=REL_MAX)
            # dQ = scale * dS @ K
            if qv.ng:
                dq = q_view(qv.g)
                accq = not fresh[id(qv)]
                ops.gemm(pr, k, dq, M=Sq, N=dh, K=Sk, lda=Skp, ldb=k.stride(1), ldc=dq.stride(1), zi=h, zo=b, b_zi_div=G,
                         a_strides=(Sq * Skp, h * Sq * Skp), b_strides=(k.stride(2), k.stride(0)),
                         c_strides=(dq.stride(2), dq.stride(0)), alpha=scale, b_mn=True,
                         residual=dq if accq else None, ldr=dq.stride(1) if accq else 0)
            # dK = scale * dS^T @ Q
            if kv.ng:
                dk = k_view(kv.g)
                self._pt_gemm(pr, q, dk, b, h, hk, Sq, Sk, Skp, dh, scale, accumulate=not fresh[id(kv)])
        self._backward(out, bwd)
        return out

    def _pt_gemm(self, p: torch.Tensor, x: torch.Tensor, dst: torch.Tensor, b, h, hk, Sq, Sk, Skp, dh, alpha, accumulate):
        """dst[b, :, hk', :] (+)= alpha * sum over the G query heads of  P[b, h]^T [Sk, Sq] @ x[b, :, h, :] [Sq, dh].
        P^T and x are consumed as stored (both MN-major operands)."""
        G = h // hk
        if G == 1:
            ops.gemm(p, x, dst, M=Sk, N=dh, K=Sq, lda=Skp, ldb=x.stride(1), ldc=dst.stride(1), zi=h, zo=b,
                     a_strides=(Sq * Skp, h * Sq * Skp), b_strides=(x.stride(2), x.stride(0)),
                     c_strides=(dst.stride(2), dst.stride(0)), alpha=alpha, a_mn=True, b_mn=True,
                     residual=dst if accumulate else None, ldr=dst.stride(1) if accumulate else 0)
            return
        if accumulate:
            raise NotImplementedError("accumulating GQA dK / dV into a shared buffer is not needed on this path")
        tmp = torch.empty(b, Sk, h, dh, device=self.dev, dtype=BF16)
        ops.gemm(p, x, tmp, M=Sk, N=dh, K=Sq, lda=Skp, ldb=x.stride(1), ldc=h * dh, zi=h, zo=b,
                 a_strides=(Sq * Skp, h * Sq * Skp), b_strides=(x.stride(2), x.stride(0)), c_strides=(dh, Sk * h * dh),
                 alpha=alpha, a_mn=True, b_mn=True)
        if dst.stride(0) != Sk * dst.stride(1):
            raise ValueError("GQA dK / dV destination must have a uniform token stride over (batch, token)")
        T.group_sum(tmp, dst, rows=b * Sk, heads=hk, G=G, dh=dh, ld_in=h * dh, ld_out=dst.stride(1))

    # =========================================================================================
    # vision front
    # =========================================================================================
    def encode_images(self, frames: torch.Tensor) -> Var:
        """ViT3D tower + spatial pooling projector (reference u2_arch.py:96-99) -> Var [F * tokens_per_frame, E]."""
        g = self.g
        Fr = frames.shape[0]
        Hd, P = g.vit_hidden, g.n_patches
        S = P + 1
        Sp = _pad8(S)
        trv = self._tr("vit")
        v = "model.vision_tower.vision_tower."
        vol = frames.to(device=self.dev, dtype=F32).contiguous().view(Fr, *g.image_size)
        rows = ops.patchify(vol, g.patch_size)
        self._wait_params([v + "patch_embedding.patch_embeddings.1.weight"])
        pe_w, pe_b = self.w(v + "patch_embedding.patch_embeddings.1.weight"), self.v32(v + "patch_embedding.patch_embeddings.1.bias")
        pos = self.w(v + "patch_embedding.position_embeddings").view(P, Hd)
        x0 = torch.empty(Fr, Sp, Hd, device=self.dev, dtype=BF16)
        ops.gemm(rows, pe_w, x0, M=Fr * P, N=Hd, K=g.patch_dim, lda=g.patch_dim, ldb=g.patch_dim, ldc=Hd, bias=pe_b,
                 residual=pos, ldr=Hd, res_row_mod=P, row_remap=(P, Sp, 1))
        ops.vit_frame_rows(x0, self.w(v + "cls_token").view(Hd), Fr, Sp, S)
        x = Var(x0.view(Fr * Sp, Hd), trv)
        self._mark([v + "patch_embedding.patch_embeddings.1.weight"])

        def bwd_embed(dx):
            if not trv:
                return
            dx = dx.view(Fr, Sp, Hd)
            dy = dx[:, 1:1 + P].contiguous().view(Fr * P, Hd)
            self.wgrad(dy, rows, self.gm(v + "patch_embedding.patch_embeddings.1.weight"))
            T.colsum(dy, self.gv(v + "patch_embedding.patch_embeddings.1.bias"))
            T.colsum(dy, self.gv(v + "patch_embedding.position_embeddings"), rows=Fr, cols=P * Hd, ld=P * Hd)
            T.colsum(dx, self.gv(v + "cls_token"), rows=Fr, cols=Hd, ld=Sp * Hd)
        self._backward(x, bwd_embed)

        nh = g.vit_heads
        dh = Hd // nh

        def view_q(i):
            return lambda t: t.view(Fr, Sp, 3, nh, dh)[:, :S, i]

        def block(li, x):
            b = f"{v}blocks.{li}."
            self._mark([b + "attn.qkv.weight", b + "attn.out_proj.weight", b + "mlp.linear1.weight", b + "mlp.linear2.weight"])
            y = self.layernorm(x, b + "norm1.weight", b + "norm1.bias", "vit")
            qb = b + "attn.qkv.bias"
            qkv = self._param_linear(y, b + "attn.qkv.weight", qb if qb in self.lay.shapes else None, "vit")
            ctx = self.attention(qkv, view_q(0), qkv, view_q(1), qkv, view_q(2), (Fr, Sp, Hd), dh ** -0.5, group="vit",
                                 recompute=True)
            ctx = self._reshape(ctx, (Fr * Sp, Hd))
            x = self._param_linear(ctx, b + "attn.out_proj.weight", b + "attn.out_proj.bias", "vit", residual=x)
            y = self.layernorm(x, b + "norm2.weight", b + "norm2.bias", "vit")
            h = self.gelu(self._param_linear(y, b + "mlp.linear1.weight", b + "mlp.linear1.bias", "vit"))
            return self._param_linear(h, b + "mlp.linear2.weight", b + "mlp.linear2.bias", "vit", residual=x)
        for li in range(g.vit_layers):
            x = self._segment(functools.partial(block, li), x)
        y = self.layernorm(x, v + "norm.weight", v + "norm.bias", "vit")
        # drop cls + pooling
        npf = g.tokens_per_frame
        pooled = torch.empty(Fr, npf, Hd, device=self.dev, dtype=BF16)
        seq = g.proj_pooling_type == "sequence"
        ops.spp_pool(y.v, pooled, frames=Fr, grid=g.grid, ps=g.proj_pooling_size, E=Hd, in_frame_stride=Sp, in_off=1, ldx=Hd,
                     sequence=seq)
        z = Var(pooled.view(Fr * npf, Hd), y.ng)

        def bwd_pool(dz):
            if not y.ng:
                return
            dy = torch.empty(Fr * Sp, Hd, device=self.dev, dtype=BF16)
            T.spp_pool_bwd(dz, dy, frames=Fr, grid=g.grid, ps=g.proj_pooling_size, E=Hd, in_frame_stride=Sp, in_off=1, ldx=Hd,
                           rows_per_frame=Sp, sequence=seq)
            self._acc(y, dy, owned=True)
        self._backward(z, bwd_pool)
        # projector MLP
        p = "model.mm_projector.projector."
        n = int(g.proj_layer_num)
        self._mark([k for k in self.lay.mat_names if k.startswith(p)])
        for i in range(n):
            idx = (2 * i if g.proj_layer_type == "mlp" else i) if i else 0
            z = self._param_linear(z, p + f"{idx}.weight", p + f"{idx}.bias", "proj")
            if g.proj_layer_type == "mlp" and i < n - 1:
                z = self.gelu(z)
        return z

    # =========================================================================================
    # mu2-tokenizer
    # =========================================================================================
    def _self_attention(self, x: Var, nb: int, S: int, pre: str, residual: Optional[Var] = None) -> Var:
        """RMA / RoPE self attention over nb sequences of length S (reference rma.py:46-82, rope.py:62-91)."""
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        qkv = self._param_linear(x, [pre + "wq.weight", pre + "wk.weight", pre + "wv.weight"],
                                 [pre + "wq.bias", pre + "wk.bias", pre + "wv.bias"], "u2t")
        if g.attn_type == "rope":
            qkv = self._rope_tok(qkv, rows=nb * S, pos_div=1, pos_mod=S)
        view = lambda i: (lambda t: t.view(nb, S, 3, H, dh)[:, :, i])
        ctx = self.attention(qkv, view(0), qkv, view(1), qkv, view(2), (nb, S, E), 1.0 / math.sqrt(dh),
                             rel_name=(pre + "relative_bias") if g.attn_type == "rma" else None)
        return self._param_linear(self._reshape(ctx, (nb * S, E)), pre + "dense.weight", pre + "dense.bias", "u2t",
                                  residual=residual)

    def _rope_tok(self, qkv: Var, rows: int, pos_div: int, pos_mod: int) -> Var:
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        y = qkv.v.clone()
        ops.rope(y, rows=rows, ld=3 * E, dh=dh, n_q=H, n_k=H, inv_freq=self.u2t_inv_freq, pos_div=pos_div, pos_mod=pos_mod)
        out = Var(y, qkv.ng)

        def bwd(dy):
            if qkv.ng:
                T.rope_bwd(dy, None, rows=rows, ld=3 * E, dh=dh, n_q=H, n_k=H, inv_freq=self.u2t_inv_freq, pos_div=pos_div,
                           pos_mod=pos_mod)
                self._acc(qkv, dy, owned=True)
        self._backward(out, bwd)
        return out

    def _temporal_attention(self, x: Var, B: int, C: int, N: int, pre: str) -> Var:
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        qkv = self._param_linear(x, [pre + "wq.weight", pre + "wk.weight", pre + "wv.weight"],
                                 [pre + "wq.bias", pre + "wk.bias", pre + "wv.bias"], "u2t")
        if g.attn_type == "rope":
            qkv = self._rope_tok(qkv, rows=B * C * N, pos_div=N, pos_mod=C)
        rel = self.v32(pre + "relative_bias").view(-1) if g.attn_type == "rma" else None
        scale = 1.0 / math.sqrt(dh)
        ctxv = torch.empty(B * C * N, E, device=self.dev, dtype=BF16)
        ops.temporal_attention(qkv.v, ctxv, B=B, C_=C, N=N, H=H, dh=dh, scale=scale, rel_bias=rel, rel_max=REL_MAX)
        ctx = Var(ctxv, qkv.ng)
        drel = self.gv(pre + "relative_bias") if (rel is not None and self._tr("u2t")) else None

        def bwd(dctx):
            if qkv.ng:
                dqkv = torch.empty_like(qkv.v)
                T.temporal_attention_bwd(qkv.v, dctx, dqkv, B=B, C_=C, N=N, H=H, dh=dh, scale=scale, rel_bias=rel, drel=drel,
                                         rel_max=REL_MAX)
                self._acc(qkv, dqkv, owned=True)
        self._backward(ctx, bwd)
        return self._param_linear(ctx, pre + "dense.weight", pre + "dense.bias", "u2t")

    def _cross_attention(self, q_in: Var, kv_in: Var, B: int, Sq: int, Sk: int, pre: str, residual: Optional[Var],
                         compress: bool = False) -> Var:
        """MultiHeadCrossAttention (reference tta.py:42-69); compress = LinearAggregation (raw values, no dense)."""
        g = self.g
        E, H = g.hidden_size, g.u2t_num_heads
        dh = E // H
        q = self._param_linear(q_in, pre + "wq.weight", pre + "wq.bias", "u2t")
        qview = lambda t: t.view(B, Sq, H, dh)
        if compress:
            k = self._param_linear(kv_in, pre + "wk.weight", pre + "wk.bias", "u2t")
            kview = lambda t: t.view(B, Sk, H, dh)
            ctx = self.attention(q, qview, k, kview, kv_in, kview, (B, Sq, E), 1.0 / math.sqrt(dh))
            return self._reshape(ctx, (B * Sq, E))
        kvp = self._param_linear(kv_in, [pre + "wk.weight", pre + "wv.weight"], [pre + "wk.bias", pre + "wv.bias"], "u2t")
        kview = lambda i: (lambda t: t.view(B, Sk, 2, H, dh)[:, :, i])
        ctx = self.attention(q, qview, kvp, kview(0), kvp, kview(1), (B, Sq, E), 1.0 / math.sqrt(dh))
        return self._param_linear(self._reshape(ctx, (B * Sq, E)), pre + "dense.weight", pre + "dense.bias", "u2t",
                                  residual=residual)

    def _token_selection_diff(self, x: Var, B: int, Tn: int) -> Var:
        """DifferentiableTokenSelection (reference svr.py:101-117): softmax over the TOKEN axis of W_s X^T, selected =
        weights @ X - and its backward, all on the GEMM + the row softmax kernels."""
        g = self.g
        E = g.hidden_size
        sname = "model.u2tokenizer.svt_module.token_selection.score_net.weight"
        Ws = self.w(sname)
        K = Ws.shape[0]
        Tp = _pad8(Tn)
        tr = self._tr("u2t")
        x3 = x.v.view(B, Tn, E)
        scT = torch.empty(K, B * Tn, device=self.dev, dtype=F32)
        ops.gemm(Ws, x.v, scT, M=K, N=B * Tn, K=E, lda=E, ldb=E, ldc=B * Tn)
        pT = torch.empty(B, K, Tp, device=self.dev, dtype=BF16)
        ops.softmax(scT, pT, n0=B, H=1, S=K, n=Tn, in_strides=(Tn, 0, B * Tn), out_strides=(K * Tp, 0, Tp), zero_pad_to=Tp)
        del scT
        sel = torch.empty(B, K, E, device=self.dev, dtype=BF16)
        ops.gemm(pT, x3, sel, M=K, N=E, K=Tn, lda=Tp, ldb=E, ldc=E, zo=B, a_strides=(0, K * Tp), b_strides=(0, Tn * E),
                 c_strides=(0, K * E), b_mn=True)
        out = Var(sel, x.ng or tr)

        def bwd(ds):
            if x.ng and x.g is None:
                x.g = torch.zeros_like(x.v)
            dx3 = x.g.view(B, Tn, E) if x.ng else None
            dpT = torch.empty(B, K, Tp, device=self.dev, dtype=F32)
            ops.gemm(ds, x3, dpT, M=K, N=Tn, K=E, lda=E, ldb=E, ldc=Tp, zo=B, a_strides=(0, K * E), b_strides=(0, Tn * E),
                     c_strides=(0, K * Tp))
            if x.ng:  # dX += P^T dsel
                ops.gemm(pT, ds, dx3, M=Tn, N=E, K=K, lda=Tp, ldb=E, ldc=E, zo=B, a_strides=(0, K * Tp), b_strides=(0, K * E),
                         c_strides=(0, Tn * E), a_mn=True, b_mn=True, residual=dx3, ldr=E)
            T.softmax_bwd(pT, dpT, pT, n0=B, H=1, S=K, n=Tn, p_strides=(K * Tp, 0, Tp), dp_strides=(K * Tp, 0, Tp),
                          ds_strides=(K * Tp, 0, Tp), zero_pad_to=Tp)
            del dpT
            for bi in range(B):
                dsc = pT[bi]
                if tr:  # dW_s (+)= dsc [K, T] @ X_b [T, E]: the step's first write overwrites the slot, like every wgrad
                    gws = self.gm(sname)
                    acc = self._gm_begin_write(gws)
                    ops.gemm(dsc, x3[bi], gws, M=K, N=E, K=Tn, lda=Tp, ldb=E, ldc=E, b_mn=True, residual=gws if acc else None,
                             ldr=E if acc else 0)
                if x.ng:  # dX_b += dsc^T [T, K] @ W_s [K, E]
                    ops.gemm(dsc, Ws, dx3[bi], M=Tn, N=E, K=K, lda=Tp, ldb=E, ldc=E, a_mn=True, b_mn=True, residual=dx3[bi], ldr=E)
        self._backward(out, bwd)
        return out

    def _token_selection_hard(self, x: Var, B: int, Tn: int) -> Var:
        """TokenSelection (reference svr.py:75-91): the indices carry no gradient (score_net stays without one, as under
        autograd); the selected rows route theirs back."""
        g = self.g
        E, K = g.hidden_size, g.u2t_top_k
        if K > Tn:
            raise RuntimeError(f"selected index k out of range: top_k={K} > {Tn} tokens (torch.topk raises too)")
        Ws = self.w("model.u2tokenizer.svt_module.token_selection.score_net.weight")
        sc = torch.empty(B * Tn, 1, device=self.dev, dtype=F32)
        ops.gemm(x.v, Ws, sc, M=B * Tn, N=1, K=E, lda=E, ldb=E, ldc=1)
        idx = ops.topk_rows(sc.view(B, Tn), K, idx_offset_per_row=Tn)
        out = Var(ops.embed_splice(idx, x.v, None), x.ng)

        def bwd(dy):
            if x.ng:
                if x.g is None:
                    x.g = torch.zeros_like(x.v)
                T.embed_scatter_add(idx, dy, x.g, None)
        self._backward(out, bwd)
        return out

    def _multiscale(self, x: Var, B: int) -> Var:
        g = self.g
        gname = "model.u2tokenizer.svt_module.dynamic_pool.gate_fc.weight"
        gate_w = self.v32(gname) if g.enable_dmtp else None
        K, E = x.v.shape[1], x.v.shape[2]
        y, logits = T.multiscale_pool_fwd(x.v, gate_w, g.enable_dmtp)
        out = Var(y, x.ng)
        dgate = self.gv(gname) if (g.enable_dmtp and self._tr("u2t")) else None

        def bwd(dy):
            if x.ng:
                self._acc(x, T.multiscale_pool_bwd(x.v, dy, gate_w, logits, dgate, g.enable_dmtp), owned=True)
        self._backward(out, bwd)
        return out

    def u2tokenizer(self, v_tokens: Var, B: int, C: int, N: int, t_tokens: Var, Lt: int) -> Var:
        """u2Tokenizer.forward (reference u2Tokenizer.py:40-47) -> Var [B * Q, E]."""
        g = self.g
        E, Q = g.hidden_size, g.num_3d_query_token
        u = "model.u2tokenizer."

        def svr_layer(i, x):
            l = f"{u}svt_module.attention_network.layers.{i}."
            self._mark([k for k in self.lay.mat_names if k.startswith(l)])
            x = self._self_attention(x, B * C, N, l + "spatial_attention.")
            return self._temporal_attention(x, B, C, N, l + "temporal_attention.")
        x = v_tokens
        for i in range(g.u2t_num_layers):
            x = self._segment(functools.partial(svr_layer, i), x)
        self._mark([u + "svt_module.token_selection.score_net.weight"])
        sel = self._token_selection_diff(x, B, C * N) if g.enable_diffts else self._token_selection_hard(x, B, C * N)
        if sel.v.dim() == 2:
            sel = self._reshape(sel, (B, -1, E))
        vis3 = self._multiscale(sel, B) if g.use_multi_scale else sel
        Mv = vis3.v.shape[1]
        vis = self._reshape(vis3, (B * Mv, E))
        tr = self._tr("u2t")
        qtok = self.w(u + "query_tokens").view(Q, E)
        q = Var(qtok.unsqueeze(0).expand(B, Q, E).contiguous().view(B * Q, E), tr)

        def bwd_q(dq):
            if tr:
                T.colsum(dq, self.gv(u + "query_tokens"), rows=B, cols=Q * E, ld=Q * E)
        self._backward(q, bwd_q)
        lin = u + "tta_module.layer_linagg.linear_aggregator."
        self._mark([lin + "wq.weight", lin + "wk.weight"])

        def tta_layer(i, q):
            l = f"{u}tta_module.layers_vt.{i}."
            self._mark([k for k in self.lay.mat_names if k.startswith(l)])
            s = self._self_attention(q, B, Q, l + "self_attention.")
            s = self.layernorm(s, l + "norm_self.weight", l + "norm_self.bias", "u2t", residual=q)
            vx = self._cross_attention(s, vis, B, Q, Mv, l + "visual_cross_attention.", residual=None)
            vx = self.layernorm(vx, l + "norm_cross_v.weight", l + "norm_cross_v.bias", "u2t", residual=s)
            tx = self._cross_attention(vx, t_tokens, B, Q, Lt, l + "text_cross_attention.", residual=None)
            return self.layernorm(tx, l + "norm_cross_t.weight", l + "norm_cross_t.bias", "u2t", residual=vx)
        for i in range(g.u2t_num_layers):
            q = self._segment(functools.partial(tta_layer, i), q)
        return self._cross_attention(q, vis, B, Q, Mv, u + "tta_module.layer_linagg.linear_aggregator.", residual=None, compress=True)

    # =========================================================================================
    # embeddings, splice, decoder, loss heads
    # =========================================================================================
    def embed(self, ids: torch.Tensor) -> Var:
        table = self.w("model.embed_tokens.weight")
        ids = ids.to(self.dev).long().contiguous()
        B, Lx = ids.shape
        out = Var(ops.embed_splice(ids, table, None).view(B * Lx, -1), self._tr("embed"))

        def bwd(dy):
            if self._tr("embed"):
                T.embed_scatter_add(ids, dy.contiguous(), self._gm_scatter_target("model.embed_tokens.weight"), None)
        self._backward(out, bwd)
        return out

    def splice(self, ids: torch.Tensor, vis: Optional[Var], n_vis: int) -> Var:
        """prepare_inputs_for_multimodal's cat (reference u2_arch.py:118-121): visual tokens at positions 1..n_vis."""
        table = self.w("model.embed_tokens.weight")
        ids = ids.to(self.dev).long().contiguous()
        B, Lx = ids.shape
        E = table.shape[1]
        visv = vis.v.view(B, n_vis, E) if vis is not None else None
        out = Var(ops.embed_splice(ids, table, visv).view(B * Lx, E), self._tr("embed") or (vis is not None and vis.ng))

        def bwd(dy):
            dvis = torch.empty(B * n_vis, E, device=self.dev, dtype=BF16) if (vis is not None and vis.ng) else None
            T.embed_scatter_add(ids, dy.contiguous(),
                                self._gm_scatter_target("model.embed_tokens.weight") if self._tr("embed") else None, dvis, n_vis)
            if dvis is not None:
                self._acc(vis, dvis, owned=True)
        self._backward(out, bwd)
        return out

    def decoder(self, x: Var, B: int, Lx: int) -> Var:
        """Qwen3 / Llama / Phi-3 decoder stack (HF modeling_qwen3.py:305-336, modeling_phi3.py per layer), causal (+ the
        Phi-3 sliding window), positions 0..L-1 -> final-norm hidden. Both families run the same four fused GEMMs per layer
        (q|k|v, o, gate|up in halves, down): Phi-3 stores them as single parameters."""
        g = self.g
        E, hq, hkv, dh, I = g.hidden_size, g.num_attention_heads, g.num_key_value_heads, g.head_dim, g.intermediate_size
        nh = hq + 2 * hkv
        eps = g.rms_norm_eps

        def layer(li, x):
            l = f"model.layers.{li}."
            self._mark([k for k in self.lay.mat_names if k.startswith(l)])
            y = self.rmsnorm(x, l + "input_layernorm.weight", "dec", eps)
            qkv = self._rope_dec(self._dec_linear(y, li, 0), l, B, Lx)
            qv = lambda t: t.view(B, Lx, nh, dh)[:, :, :hq]
            kv_ = lambda t: t.view(B, Lx, nh, dh)[:, :, hq:hq + hkv]
            vv_ = lambda t: t.view(B, Lx, nh, dh)[:, :, hq + hkv:]
            ctx = self.attention(qkv, qv, qkv, kv_, qkv, vv_, (B, Lx, hq * dh), 1.0 / math.sqrt(dh), causal=True, group="dec",
                                 window=g.window)
            x = self._dec_linear(self._reshape(ctx, (B * Lx, hq * dh)), li, 1, residual=x)
            y = self.rmsnorm(x, l + "post_attention_layernorm.weight", "dec", eps)
            act = self.silu_mul(self._dec_linear(y, li, 2))
            return self._dec_linear(act, li, 3, residual=x)
        for li in range(g.num_hidden_layers):
            x = self._segment(functools.partial(layer, li), x)
        return self.rmsnorm(x, "model.norm.weight", "dec", eps)

    def _dec_linear(self, x: Var, li: int, gi: int, residual: Optional[Var] = None) -> Var:
        """Fused group gi of lora_groups(g) of decoder layer li (q|k|v, o, gate|up, down). Without adapters: one linear
        (wgrad while the decoder trains). With adapters on (some of) its members: the base output on the frozen weight,
        then for every adapter j  U_j = s (D_j o x) A_j^T (lora_down) and y[:, rows_j] += U_j B_j^T on the GEMM (K = r)."""
        pre, members = lora_groups(self.g)[gi]
        names = [f"model.layers.{li}.{pre}{t}.weight" for t in members]
        lo = self.lora
        tg = [t for t in members if lo is not None and t in lo.targets]
        if not tg:
            return self._param_linear(x, names, None, "dec", residual=residual)
        if len(tg) != len(members):
            raise NotImplementedError(f"LoRA on part of a fused group ({tg} of {members}) is not supported on the training path")
        r, s = lo.r, lo.scaling
        trip = [lo.names(li, pre, t) for t in tg]
        an, bn = [a for _, a, _ in trip], [b for _, _, b in trip]
        A, Wb = self.wcat(an), self.wcat(names)
        Bs = [self.w(b) for b in bn]
        streams = [lora_stream(self.g, li, t) for t in tg]
        p, seed = (lo.dropout, self._lora_seed) if self._lora_seed else (0.0, 0)
        y = ops.linear(x.v, Wb, residual=residual.v if residual is not None else None)
        x2 = x.v.view(-1, x.v.shape[-1])
        U = T.lora_down(x2, A, r, s, p=p, seed=seed, streams=streams)
        y2 = y.view(-1, y.shape[-1])
        M, Ntot = y2.shape
        col = 0
        cols = []
        for j, B in enumerate(Bs):
            n = B.shape[0]
            yj, uj = y2[:, col:col + n], U[:, j * r:(j + 1) * r]
            ops.gemm(uj, B, yj, M=M, N=n, K=r, lda=U.stride(0), ldb=r, ldc=Ntot, residual=yj, ldr=Ntot)
            cols.append((col, n))
            col += n
        out = Var(y, True)

        def bwd(dy):
            dy2 = dy.view(-1, Ntot)
            dU = torch.empty_like(U)
            for j, (c0, n) in enumerate(cols):
                dyj = dy2[:, c0:c0 + n]
                self.wgrad(dyj, U[:, j * r:(j + 1) * r], self.gm(bn[j]))
                T.linear_dgrad(dyj, Bs[j], out=dU[:, j * r:(j + 1) * r])
            gA = self.gm(an)
            T.lora_wgrad(dU, x2, gA, r, s, p=p, seed=seed, streams=streams, accumulate=self._gm_begin_write(gA))
            if x.ng:
                if x.g is None:
                    x.g = T.linear_dgrad(dy, Wb)
                else:
                    T.linear_dgrad(dy, Wb, out=x.g, accumulate=True)
                T.lora_dgrad(dU, A, x.g.view(-1, x2.shape[1]), r, s, p=p, seed=seed, streams=streams)
            if residual is not None:
                self._acc(residual, dy, owned=True)
        self._backward(out, bwd)
        return out

    def _rope_dec(self, qkv_raw: Var, l: str, B: int, Lx: int) -> Var:
        g = self.g
        hq, hkv, dh = g.num_attention_heads, g.num_key_value_heads, g.head_dim
        nqkv = (hq + 2 * hkv) * dh
        qn = self.v32(l + "self_attn.q_norm.weight") if g.qk_norm else None
        kn = self.v32(l + "self_attn.k_norm.weight") if g.qk_norm else None
        y = qkv_raw.v.clone()
        ops.rope(y, rows=B * Lx, ld=nqkv, dh=dh, n_q=hq, n_k=hkv, n_v=0, inv_freq=self.inv_freq, q_norm_w=qn, k_norm_w=kn,
                 eps=g.rms_norm_eps, pos0=0, pos_div=1, pos_mod=Lx)
        out = Var(y, qkv_raw.ng)
        dqn = dkn = None
        if g.qk_norm and self._tr("dec"):
            dqn, dkn = self.gv(l + "self_attn.q_norm.weight"), self.gv(l + "self_attn.k_norm.weight")

        def bwd(dy):
            if qkv_raw.ng:
                T.rope_bwd(dy, qkv_raw.v, rows=B * Lx, ld=nqkv, dh=dh, n_q=hq, n_k=hkv, inv_freq=self.inv_freq, q_norm_w=qn,
                           k_norm_w=kn, eps=g.rms_norm_eps, pos0=0, pos_div=1, pos_mod=Lx, dq_norm_w=dqn, dk_norm_w=dkn)
                self._acc(qkv_raw, dy, owned=True)
        self._backward(out, bwd)
        return out

    def _head_w(self):
        name = "model.embed_tokens.weight" if self.tied else "lm_head.weight"
        return name, self.w(name)

    def logprob_head(self, hidden: Var, labels: torch.Tensor, coef_fn) -> Tuple[torch.Tensor, torch.Tensor]:
        """Fused lm_head + log-softmax statistics forward (the [R, V] logits are not materialised); the backward
        recomputes the logits once in fp32, turns them into dlogits = coef * (softmax - onehot) in place of a bf16 buffer
        and runs the two head GEMMs. coef_fn(logp) -> fp32 [R] (-dLoss/dlogp per row, 0 where unlabelled), called at
        backward time. Returns (logp [R], lse [R])."""
        hname, Wh = self._head_w()
        h2 = hidden.v
        lab = labels.to(self.dev, torch.int64).contiguous().view(-1)
        if not self.tied:
            self._mark([hname])
        logp, lse, _ = ops.lmhead_logprob(h2, Wh, lab, want_lse=True)
        trh = self._tr("head") if not self.tied else (self._tr("head") or self._tr("embed"))

        def bwd():
            coef = coef_fn(logp)
            R, V = h2.shape[0], Wh.shape[0]
            logits = torch.empty(R, V, device=self.dev, dtype=F32)
            ops.gemm(h2, Wh, logits, M=R, N=V, K=h2.shape[1], lda=h2.stride(0), ldb=Wh.stride(0), ldc=V)
            dl = T.ce_bwd(logits, lse, lab.clamp_min(0), coef)
            del logits
            if trh:
                self.wgrad(dl, h2, self.gm(hname))
            if hidden.ng:
                self._acc(hidden, T.linear_dgrad(dl, Wh), owned=True)
        self.tape.append((None, bwd))
        lin = "model.u2tokenizer.tta_module.layer_linagg.linear_aggregator."
        unused = [lin + "wv.weight", lin + "dense.weight"]   # never run by the reference either (tta.py:47-48,62-65)
        if not self.g.enable_diffts:
            unused.append("model.u2tokenizer.svt_module.token_selection.score_net.weight")  # top-k indices carry no gradient
        self._mark(unused)
        return logp, lse

    # =========================================================================================
    # whole-model passes
    # =========================================================================================
    def _forward_hidden(self, images, input_ids, question_ids) -> Tuple[Var, int, int]:
        g = self.g
        input_ids = input_ids.to(self.dev)
        B, Lx = input_ids.shape
        vis = None
        n_vis = 0
        self._mark(["model.embed_tokens.weight"])   # first on the tape = last in the backward: the embedding's gradient
        if images is not None:
            if g.enable_u2tokenizer:
                Bi, C = images.shape[0], images.shape[1]
                feats = self.encode_images(images.reshape(Bi * C, 1, *images.shape[2:]))
                N = g.tokens_per_frame
                if question_ids is None:
                    raise ValueError("question_ids is required when the mu2-tokenizer is enabled")
                Lt = question_ids.shape[1]
                t_tokens = self.embed(question_ids)
                vis = self.u2tokenizer(feats, Bi, C, N, t_tokens, Lt)
                n_vis = g.num_3d_query_token
            else:
                vis = self.encode_images(images)
                n_vis = g.tokens_per_frame
        x = self.splice(input_ids, vis, n_vis)
        return self.decoder(x, B, Lx), B, Lx

    def run_backward(self):
        if self.overlap and self.opt is not None and self.world > 1:
            self._pending = [set(ns) for ns in self.lay.bucket_names]
        else:
            self._pending = None
        self._run_tape(self.tape)
        self.tape = []
        self._pending = None
        self._gm_clear_stale(tuple(self._gm_dirty))   # whatever no marker covered

    def _begin_pass(self, train: bool):
        """Start a forward on an empty tape with fresh fp32 vector mirrors. A training pass draws the LoRA dropout seed (one
        nonzero 63-bit seed from torch's default generator, so torch.manual_seed makes the masks reproducible; the backward
        recomputes the masks from it) and checkpoints when `checkpoint` is set; a no-grad pass runs with neither."""
        self.tape = []
        self.refresh_vectors()
        self._lora_seed = 0
        if train and self.lora is not None and self.lora.dropout > 0:
            self._lora_seed = int(torch.randint(1, 2 ** 63 - 1, (1,)).item())
        self._ckpt = train and bool(self.checkpoint)

    def forward_loss(self, images, input_ids, question_ids, labels) -> torch.Tensor:
        """Forward half of the training step: HF ForCausalLMLoss of `model(images=, input_ids=, question_ids=, labels=)`
        (reference u2llama.py:76-87: shift by one, mean NLL over labels != -100). Keeps the tape for backward()."""
        self._begin_pass(train=True)
        hidden, B, Lx = self._forward_hidden(images, input_ids, question_ids)
        lab = labels.to(self.dev, torch.int64)
        shift = torch.full_like(lab, -100)
        shift[:, :-1] = lab[:, 1:]
        shift = shift.view(-1)
        n_valid = (shift >= 0).sum().clamp(min=1).to(F32)
        self._grad_scale = 1.0

        def coef_fn(logp):
            return (shift >= 0).to(F32) * (self._grad_scale / n_valid)
        logp, _ = self.logprob_head(hidden, torch.where(shift >= 0, shift, torch.full_like(shift, -1)), coef_fn)
        return -(logp.sum() / n_valid)

    def backward(self, grad_scale=1.0):
        """Backward half: gradients go to Gm / Gv - the first matrix write after zero_grad() overwrites its slot, every
        later one (a second backward() before the next zero_grad(): micro-batch accumulation) adds. grad_scale: float or
        a device scalar (the upstream gradient of the loss)."""
        self._grad_scale = grad_scale
        self.run_backward()

    def forward_backward(self, images, input_ids, question_ids, labels, grad_scale=1.0) -> torch.Tensor:
        loss = self.forward_loss(images, input_ids, question_ids, labels)
        self.backward(grad_scale)
        return loss

    def forward_loss_only(self, images, input_ids, question_ids, labels) -> torch.Tensor:
        self._begin_pass(train=False)
        hidden, B, Lx = self._forward_hidden(images, input_ids, question_ids)
        lab = labels.to(self.dev, torch.int64)
        shift = torch.full_like(lab, -1)
        shift[:, :-1] = torch.where(lab[:, 1:] >= 0, lab[:, 1:], torch.full_like(lab[:, 1:], -1))
        hname, Wh = self._head_w()
        logp, _, _ = ops.lmhead_logprob(hidden.v, Wh, shift.view(-1))
        self.tape = []
        return -(logp.sum() / (shift >= 0).sum().clamp(min=1))

    @torch.no_grad()
    def sequence_logps(self, images, input_ids, question_ids, loss_mask) -> torch.Tensor:
        """Summed log-probability of the masked tokens per sequence without gradients (the frozen reference model of the
        DPO step, trl DPOTrainer.compute_ref_log_probs / dpo_u2trainer.py:267-302)."""
        self._begin_pass(train=False)
        hidden, B, Lx = self._forward_hidden(images, input_ids, question_ids)
        labels, mask = _dpo_labels(input_ids.to(self.dev), loss_mask.to(self.dev))
        hname, Wh = self._head_w()
        logp, _, _ = ops.lmhead_logprob(hidden.v, Wh, labels.view(-1))
        self.tape = []
        return (logp.view(B, Lx) * mask).sum(-1)

    def dpo_forward_backward(self, images, input_ids, question_ids, loss_mask, ref_logps: torch.Tensor, beta: float = 0.1):
        """Policy side of the DPO step (reference dpo_u2trainer.py:185-359 + trl sigmoid loss, beta from
        train_stage2.py:83): rows [0, P) are the chosen, [P, 2P) the rejected sequences. ref_logps fp32 [2P] from the frozen
        reference model. Returns the fp32 [3] stats tensor (loss, reward accuracy, reward margin)."""
        self._begin_pass(train=True)
        hidden, B, Lx = self._forward_hidden(images, input_ids, question_ids)
        labels, mask = _dpo_labels(input_ids.to(self.dev), loss_mask.to(self.dev))
        stats = {}

        def coef_fn(logp):
            st, coef = T.dpo_loss(logp.view(B, Lx).contiguous(), ref_logps.to(self.dev, F32).contiguous(),
                                  mask.to(torch.uint8).contiguous(), beta)
            stats["dpo"] = st
            return coef.view(-1)
        self.logprob_head(hidden, labels.view(-1), coef_fn)
        self.run_backward()
        return stats["dpo"]

    # =========================================================================================
    # optimizer: ZeRO-1 over the data-parallel group
    # =========================================================================================
    def init_optimizer(self, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, max_grad_norm: Optional[float] = 1.0,
                       moment_dtype=F32):
        """AdamW state for this rank: fp32 master / m / v of the local 1/W slice of every bucket of the matrix region and of
        the whole (replicated) vector region. Defaults follow the reference's TrainingArguments (train_stage1.py:113-131:
        adamw_torch, lr 1e-4, weight_decay 0) and HF Trainer's max_grad_norm 1.0. moment_dtype=torch.bfloat16 stores the
        matrix region's moments in bf16 (8 instead of 12 bytes of state per parameter): what ONE GPU needs to hold the
        unsharded state of the 8B model; the sharded multi-GPU step keeps fp32."""
        L = self.lay
        pc, nb = L.piece, L.n_buckets
        mm = torch.empty(nb * pc, device=self.dev, dtype=F32)
        for i in range(nb):
            lo = i * L.bucket + self.rank * pc
            T.cast(self.W[lo:lo + pc], mm[i * pc:(i + 1) * pc])
        vm = torch.empty(L.vec_total, device=self.dev, dtype=F32)
        T.cast(self.W[L.mat_total:L.mat_total + L.vec_total], vm)
        self.opt = dict(lr=lr, b1=betas[0], b2=betas[1], eps=eps, wd=weight_decay, clip=max_grad_norm, step=0,
                        m_master=mm, m_m=torch.zeros(nb * pc, device=self.dev, dtype=moment_dtype),
                        m_v=torch.zeros(nb * pc, device=self.dev, dtype=moment_dtype),
                        v_master=vm, v_m=torch.zeros_like(vm), v_v=torch.zeros_like(vm),
                        gshard=torch.empty(nb * pc, device=self.dev, dtype=BF16) if self.world > 1 else None,
                        norm=torch.zeros(2, device=self.dev, dtype=F32), scale=torch.ones(1, device=self.dev, dtype=F32),
                        reduced=[False] * nb)
        return self.opt

    def _grad_piece(self, i: int) -> torch.Tensor:
        """This rank's (averaged) gradient slice of bucket i."""
        L = self.lay
        if self.world > 1:
            return self.opt["gshard"][i * L.piece:(i + 1) * L.piece]
        return self.Gm[i * L.bucket:(i + 1) * L.bucket]

    def reduce_bucket(self, i: int):
        """NCCL reduce-scatter (mean) of bucket i of the bf16 matrix gradients into this rank's slice. Stream-ordered on
        the CURRENT stream: the overlapped schedule calls it on the communication stream as soon as the bucket's last
        wgrad has been issued (see run_backward)."""
        import torch.distributed as dist
        L = self.lay
        if self.world > 1 and not self.opt["reduced"][i]:
            dist.reduce_scatter_tensor(self._grad_piece(i), self.Gm[i * L.bucket:(i + 1) * L.bucket], op=dist.ReduceOp.AVG,
                                       group=self.group)
        self.opt["reduced"][i] = True

    def optimizer_step(self):
        """reduce-scatter (mean) of the bf16 matrix gradients bucket by bucket (those not already reduced during the
        backward) -> global gradient-norm clipping -> fused AdamW on the local slices -> all-gather of the updated bf16
        parameters; the fp32 vector gradients are all-reduced and updated replicated."""
        import torch.distributed as dist
        o = self.opt
        L = self.lay
        W_, pc, nb = self.world, L.piece, L.n_buckets
        o["step"] += 1
        if self.comm_stream is not None:
            torch.cuda.current_stream().wait_stream(self.comm_stream)
        self.sync_params()
        if W_ > 1:
            self.Gv.mul_(1.0 / W_)  # a few MB of fp32: plumbing of the collective (mean), not hot-path arithmetic
            dist.all_reduce(self.Gv, group=self.group)
        for i in range(nb):
            self.reduce_bucket(i)
        scale = None
        if o["clip"] is not None:  # HF Trainer clip_grad_norm_ over the averaged gradients
            o["norm"].zero_()
            for i in range(nb):
                T.sumsq(self._grad_piece(i), o["norm"][0:1])
            T.sumsq(self.Gv, o["norm"][1:2])
            if W_ > 1:
                dist.all_reduce(o["norm"][0:1], group=self.group)
            total = (o["norm"][0] + o["norm"][1]).sqrt()
            o["scale"].copy_((o["clip"] / (total + 1e-6)).clamp(max=1.0).view(1))
            o["grad_norm"] = total
            scale = o["scale"]
        kw = dict(lr=o["lr"], beta1=o["b1"], beta2=o["b2"], eps=o["eps"], weight_decay=o["wd"], step=o["step"], grad_scale=scale)
        for i in range(nb):
            lo = i * L.bucket + self.rank * pc
            sl = slice(i * pc, (i + 1) * pc)
            # index_offset = the slice's offset in the whole matrix region: bf16 moments get the same stochastic rounding
            # for any world size
            T.adamw(o["m_master"][sl], o["m_m"][sl], o["m_v"][sl], self._grad_piece(i), self.W[lo:lo + pc], index_offset=lo,
                    **kw)
            if W_ > 1:
                # all-gather of the updated slice on the communication stream: it overlaps the remaining AdamW launches and
                # the NEXT step's forward, which waits per bucket (_wait_params) right before a segment reads its weights
                ev = torch.cuda.Event()
                ev.record()
                with torch.cuda.stream(self.comm_stream):
                    self.comm_stream.wait_event(ev)
                    dist.all_gather_into_tensor(self.W[i * L.bucket:(i + 1) * L.bucket], self.W[lo:lo + pc], group=self.group)
                    done = torch.cuda.Event()
                    done.record(self.comm_stream)
                self._ag_ev[i] = done
        T.adamw(o["v_master"], o["v_m"], o["v_v"], self.Gv, self.W[L.mat_total:L.mat_total + L.vec_total], param_out_f32=self.V32,
                **kw)
        o["reduced"] = [False] * nb


def _dpo_labels(input_ids: torch.Tensor, loss_mask: torch.Tensor):
    """Labels = input_ids rolled left by one; position l predicts token l + 1 and counts when loss_mask[l + 1] is set
    (reference dpo_u2trainer.py:274-302, non-padding-free branch)."""
    labels = torch.roll(input_ids.long(), shifts=-1, dims=1)
    mask = torch.roll(loss_mask.bool(), shifts=-1, dims=1)
    mask[:, -1] = False
    labels = labels.masked_fill(~mask, -1)
    return labels, mask.to(F32)
