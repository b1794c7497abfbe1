"""LoRA training step of mu2-Qwen3-8B on one GPU at the cfg 4 batch geometry (2 volumes of [8, 32, 256, 256], 512-token
sequences) with the reference's recipe: r = 16, alpha = 32, dropout 0.05 on every decoder q/k/v/o/gate/up/down_proj,
the vision tower, projector, mu2-tokenizer, embed_tokens and lm_head trainable, the decoder's own weights frozen.

Reports peak torch.cuda.max_memory_allocated, the step time (CUDA events, after warm-up) and the share of the LoRA
kernels in a separate torch.profiler run, with the card name and power limit read in the same process. A batch that
does not fit is reported as such and the next smaller one is tried.

--checkpoint on runs the step with activation checkpointing (TrainEngine(checkpoint=True), what
gradient_checkpointing_enable() turns on); --checkpoint both runs the plain and the checkpointed step alternately on the
same engine and reports each (a mode that runs out of memory is reported as not fitting; the batch falls back only when
neither fits).

    python tools/lora_train_probe.py --moments fp32 [--seq 1024] [--checkpoint both] [--out results.json]

The result is printed as one JSON line; --out also writes it to a file.
"""
import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def lora_state(g, sd, r, gen):
    from u2tokenizer_b200.train import LORA_GROUPS
    for li in range(g.num_hidden_layers):
        for pre, members in LORA_GROUPS:
            for t in members:
                m = f"model.layers.{li}.{pre}{t}."
                out_f, in_f = sd[m + "weight"].shape
                a = torch.empty(r, in_f, device="cuda")
                torch.nn.init.kaiming_uniform_(a, a=math.sqrt(5), generator=gen)
                sd[m + "lora_A.default.weight"] = a.to(torch.bfloat16)
                # a trained-looking B: a zero B would leave dA = 0 (the arithmetic is the same either way)
                sd[m + "lora_B.default.weight"] = (torch.randn(out_f, r, device="cuda", generator=gen) * 1e-3).to(torch.bfloat16)


def batch(g, B, frames, seq, n_question, lt):
    from u2tokenizer_b200.synthetic import synthetic_inputs
    images, ids, qids = synthetic_inputs(g, batch=B, frames=frames, n_question=n_question, lt=lt, seed=4321)
    for b in range(B):   # raw depth 64 / 128 / 256 -> 2 / 4 / 8 real frames, the rest zero padding (as bench.py cfg 4)
        images[b, (64, 128, 256)[b % 3] // 32:] = 0
    gen = torch.Generator().manual_seed(99)
    n_prompt = ids.shape[1]
    ans = torch.randint(1, g.vocab_size - 16, (B, seq - n_prompt), generator=gen)
    ids = torch.cat([ids, ans], 1)
    labels = ids.clone()
    labels[:, :n_prompt] = -100
    return [t.cuda() for t in (images, ids, qids, labels)]


def run(B, args, modes):
    from u2tokenizer_b200.configuration import QWEN3_8B, U2Qwen3Config
    from u2tokenizer_b200.geometry import Geometry
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    from u2tokenizer_b200.train import LORA_TARGETS, LoraSpec, TrainEngine
    g = Geometry.from_hf(U2Qwen3Config(**QWEN3_8B))
    sd = synthetic_state_dict(g, seed=0, device="cuda", dtype=torch.bfloat16)
    lora_state(g, sd, 16, torch.Generator(device="cuda").manual_seed(1))
    te = TrainEngine(g, sd, device="cuda", lora=LoraSpec(16, 32 / 16, 0.05, LORA_TARGETS),
                     trainable=dict(vit=True, proj=True, u2t=True, dec=False, embed=True, head=True))
    del sd
    torch.cuda.empty_cache()
    te.init_optimizer(lr=1e-4, weight_decay=0.0, max_grad_norm=1.0,
                      moment_dtype=torch.float32 if args.moments == "fp32" else torch.bfloat16)
    L = te.lay
    n_train = L.mat_used + L.vec_total
    data = batch(g, B, 8, args.seq, 32, 512)
    torch.manual_seed(0)

    def step(ck):
        te.checkpoint = ck
        te.zero_grad()
        loss = te.forward_backward(*data)
        te.optimizer_step()
        return loss
    out = {}
    fit = []
    for ck in modes:
        try:
            for _ in range(args.warmup):
                step(ck)
            torch.cuda.synchronize()
            fit.append(ck)
        except torch.cuda.OutOfMemoryError as e:
            te.tape = []
            out[ck] = dict(batch=B, checkpoint=ck, fits=False, error=str(e).splitlines()[0])
            import gc
            gc.collect()
            torch.cuda.empty_cache()
    if not fit:
        return None, list(out.values())
    times, peaks, loss = {ck: [] for ck in fit}, {ck: 0 for ck in fit}, {}
    for _ in range(args.steps):
        for ck in fit:   # the modes alternate step by step: clock and neighbour drift hit both alike
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss[ck] = step(ck)
            e1.record()
            torch.cuda.synchronize()
            times[ck].append(e0.elapsed_time(e1))
            peaks[ck] = max(peaks[ck], torch.cuda.max_memory_allocated())
    from torch.profiler import ProfilerActivity, profile
    for ck in fit:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(ck)
            torch.cuda.synchronize()
        tot = lora = 0.0
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if e.device_type is not None and "cpu" in str(e.device_type).lower():
                continue
            tot += t
            if "lora_" in e.key:
                lora += t
        ts = times[ck]
        out[ck] = dict(batch=B, checkpoint=ck, fits=True, loss=float(loss[ck]), step_ms_median=sorted(ts)[len(ts) // 2],
                       step_ms=ts, peak_alloc_gib=peaks[ck] / 2 ** 30, frozen_gib=L.frozen_total * 2 / 2 ** 30,
                       trainable_params=n_train, gm_gib=L.mat_total * 2 / 2 ** 30, lora_kernel_share=lora / max(tot, 1e-9),
                       kernel_time_ms=tot / 1e3)
    return fit, [out[ck] for ck in modes if ck in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--moments", choices=("fp32", "bf16"), default="fp32")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--checkpoint", choices=("off", "on", "both"), default="off",
                    help="activation checkpointing of the training tape; both: plain and checkpointed steps alternately")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_train_probe needs a CUDA device")
    modes = {"off": [False], "on": [True], "both": [False, True]}[args.checkpoint]
    res = dict(card=card(), moments=args.moments, seq=args.seq, runs=[])
    t0 = time.time()
    for B in range(args.batch, 0, -1):
        try:
            fit, runs = run(B, args, modes)
        except torch.cuda.OutOfMemoryError as e:
            fit, runs = None, [dict(batch=B, fits=False, error=str(e).splitlines()[0])]
        res["runs"].extend(runs)
        import gc
        gc.collect()
        torch.cuda.empty_cache()
        if fit:
            break
    res["wall_s"] = time.time() - t0
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
