"""Records what the training path computes for a fixed set of passes, so two versions of the package can be compared bit
for bit: TrainEngine.forward_backward plain and checkpointed, LoRA r=16 with dropout 0.05 plain and checkpointed, the
Phi-3 sliding-window geometry, `model(**batch).loss.backward()` over two micro-batches with the vision tower frozen (Qwen3
and tied-embedding Llama), a DPO step, sequence_logps and forward_loss_only, at the tiny test geometries with synthetic
weights and fixed seeds.

For every training case it saves the loss (or the DPO stats), Gm and Gv after the backward, W, the fp32 vector mirror
and the AdamW state after one optimizer_step, and for each pass the number of kernels launched (_lib.launches() delta)
and the trace of its C-ABI calls: entry point, scalar arguments and descriptor fields, with every pointer written as
(flat buffer, byte offset) inside W / Gm / Gv / V32 and otherwise by order of first use in the pass. The module cases
also save every p.grad.

The backward's fp32 atomics make some gradient bits differ from run to run of the same code, so two versions are
compared against two runs of one of them: the traces, launch counts and forward results must be equal, and --compare
prints the largest difference of every tensor that is not.

usage: python tools/train_identity_probe.py --out a.pt [--root TREE]   (TREE: the checkout whose package runs)
       python tools/train_identity_probe.py --compare a.pt b.pt        (exit 1 unless every entry is equal)"""
import argparse
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF = torch.bfloat16
OPT_STATE = ("m_master", "m_m", "m_v", "v_master", "v_m", "v_v", "norm", "scale")


class CallTrace:
    """Stands in for the loaded library: records every call, then makes it."""

    def __init__(self, lib):
        self.lib, self.calls, self.seen, self.bases = lib, [], {}, {}

    def start(self, te):
        self.calls, self.seen = [], {}
        self.bases = {k: getattr(te, k) for k in ("W", "Gm", "Gv", "V32")}

    def __getattr__(self, name):
        fn = getattr(self.lib, name)

        def call(*args):
            self.calls.append((name, tuple(self.arg(a) for a in args)))
            return fn(*args)
        return call

    def arg(self, a):
        if hasattr(a, "_obj"):   # byref(descriptor)
            a = a._obj
        if isinstance(a, C.Structure):
            return tuple((f[0], self.arg(getattr(a, f[0]))) for f in a._fields_)
        if isinstance(a, C.Array):
            return tuple(self.arg(x) for x in a)
        if isinstance(a, int) and a > 1 << 40:   # a device pointer or a stream handle
            for k, t in self.bases.items():
                lo = t.data_ptr()
                if lo <= a < lo + t.numel() * t.element_size():
                    return (k, a - lo)
            return ("ptr", self.seen.setdefault(a, len(self.seen)))
        return a


def record(root):
    sys.path[:0] = [root, os.path.join(root, "tests")]
    from common import tiny_geometry
    from test_lora_gpu import TARGETS, _lora_sd, _surface_model
    from test_phi3 import tiny_phi3_geometry
    from test_train_gpu import _labels
    from u2tokenizer_b200 import _lib
    from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict
    from u2tokenizer_b200.train import LoraSpec, TrainEngine
    _lib.load()
    trace = _lib._lib = CallTrace(_lib._lib)
    res = {}

    def weights(g, seed):
        sd16 = synthetic_state_dict(g, seed=seed, device="cpu", dtype=BF)
        # O(1) query tokens: the TTA attention is not uniform, so its backward carries real values
        sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(BF)
        return sd16

    def sft_batch(g, seed):
        im, ids, q = synthetic_inputs(g, batch=2, frames=2, n_question=30, lt=32, seed=seed)
        return im.cuda(), ids.cuda(), q.cuda(), _labels(ids, g.num_3d_query_token).cuda()

    def dpo_batch(g):
        images, ids, qids = synthetic_inputs(g, batch=1, frames=2, n_question=6, lt=10)
        ans = torch.randint(1, g.vocab_size - 16, (2, 9), generator=torch.Generator().manual_seed(3))
        ids2 = torch.cat([ids.expand(2, -1), ans], 1).cuda()
        mask = torch.zeros_like(ids2)
        mask[:, ids.shape[1]:] = 1
        mask[1, -2:] = 0
        return (images.expand(2, *images.shape[1:]).contiguous().cuda(), ids2, qids.expand(2, -1).contiguous().cuda(),
                mask)

    def timed(rec, key, te, fn):
        trace.start(te)
        n0 = _lib.launches()
        out = fn()
        torch.cuda.synchronize()
        rec[f"launches/{key}"] = _lib.launches() - n0
        rec[f"trace/{key}"] = trace.calls
        return out

    def step_state(rec, te):
        rec["Gm"], rec["Gv"] = te.Gm.cpu(), te.Gv.cpu()
        timed(rec, "optimizer_step", te, te.optimizer_step)
        rec["W"], rec["V32"] = te.W.cpu(), te.V32.cpu()
        for k in OPT_STATE:
            rec[f"opt/{k}"] = te.opt[k].cpu()

    def engine_case(name, te, fn, seed=0):
        rec = res[name] = {}
        te.init_optimizer(lr=1e-3, weight_decay=0.01, max_grad_norm=1.0)
        te.zero_grad()
        torch.manual_seed(seed)   # the LoRA dropout seed of the training forward
        rec["out"] = timed(rec, "pass", te, fn).float().cpu()
        step_state(rec, te)
        print(f"{name}: out {rec['out'].tolist()} launches {rec['launches/pass']} + {rec['launches/optimizer_step']}",
              flush=True)

    g = tiny_geometry()
    a = sft_batch(g, 1)
    for ckpt in (False, True):
        te = TrainEngine(g, weights(g, 22), device="cuda", checkpoint=ckpt)
        engine_case(f"sft/ckpt{int(ckpt)}", te, lambda: te.forward_backward(*a))
    for ckpt in (False, True):
        te = TrainEngine(g, _lora_sd(g, weights(g, 22), 16), device="cuda", lora=LoraSpec(16, 2.0, 0.05, TARGETS),
                         checkpoint=ckpt)
        engine_case(f"lora_r16_p005/ckpt{int(ckpt)}", te, lambda: te.forward_backward(*a), seed=123)
    gp = tiny_phi3_geometry()
    te = TrainEngine(gp, weights(gp, 31), device="cuda")
    ap = sft_batch(gp, 1)
    engine_case("phi3_window", te, lambda: te.forward_backward(*ap))

    images2, ids2, qids2, mask = dpo_batch(g)
    ref_logps = torch.tensor([-30.0, -28.5], device="cuda")
    te = TrainEngine(g, weights(g, 22), device="cuda")
    engine_case("dpo", te, lambda: te.dpo_forward_backward(images2, ids2, qids2, mask, ref_logps, 0.1))
    rec = res["sequence_logps"] = {}
    rec["out"] = timed(rec, "pass", te, lambda: te.sequence_logps(images2, ids2, qids2, mask)).cpu()
    rec = res["forward_loss_only"] = {}
    rec["out"] = timed(rec, "pass", te, lambda: te.forward_loss_only(*a)).cpu()
    del te

    # the HF surface: two accumulated micro-batches (the second adds into the p.grad slots it was handed by the first)
    for family in ("qwen3", "llama"):
        model, gm = _surface_model(family)
        model.get_model().vision_tower.requires_grad_(False)
        model.train()
        te = model.train_engine()
        te.init_optimizer(lr=1e-3, weight_decay=0.01, max_grad_norm=1.0)
        rec = res[f"module_frozen_vit/{family}"] = {}
        model.zero_grad(set_to_none=True)
        for i, seed in enumerate((1, 2)):
            im, ids, q, lab = sft_batch(gm, seed)
            batch = dict(images=im, input_ids=ids, question_ids=q, labels=lab, attention_mask=torch.ones_like(ids))

            def micro_batch():
                loss = model(**batch).loss
                loss.backward()
                return loss.detach()
            rec[f"loss{i}"] = timed(rec, f"micro_batch{i}", te, micro_batch).float().cpu()
        for n, p in model.named_parameters():
            if p.grad is not None:
                rec[f"grad/{n}"] = p.grad.cpu()
        step_state(rec, te)
        print(f"module_frozen_vit/{family}: {sum(k.startswith('grad/') for k in rec)} p.grad, launches "
              f"{rec['launches/micro_batch0']} + {rec['launches/micro_batch1']} + {rec['launches/optimizer_step']}",
              flush=True)
        del model, te
    return res


def compare(a_path, b_path):
    a, b = torch.load(a_path), torch.load(b_path)
    bad = sorted(set(a) ^ set(b))
    for k in sorted(set(a) & set(b)):
        for f in sorted(set(a[k]) | set(b[k])):
            x, y = a[k].get(f), b[k].get(f)
            both = isinstance(x, torch.Tensor) and isinstance(y, torch.Tensor)
            same = torch.equal(x, y) if both else (type(x) is type(y) and x == y)
            if not same:
                bad.append(f"{k}:{f}")
                if both and x.shape == y.shape and x.is_floating_point():
                    d = (x.double() - y.double()).abs().max().item()
                    print(f"  {k}:{f}  max |diff| {d:.3g}  (max |a| {x.double().abs().max().item():.3g})")
    n = sum(len(v) for v in a.values())
    print(f"{len(a)} / {len(b)} cases, {n} entries; differences: {bad if bad else 'none'}")
    return not bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    if not torch.cuda.is_available():
        raise SystemExit("train_identity_probe needs a CUDA device")
    torch.save(record(os.path.abspath(args.root)), args.out)


if __name__ == "__main__":
    main()
