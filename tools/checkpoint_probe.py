"""Activation checkpointing on the full-parameter training step that bench.py's `train_step` line trains on one GPU:
mu2-Qwen3-1.7B (the 8B model's training state does not fit one 80 GB card) at the cfg 4 batch geometry (2 volumes of
[8, 32, 256, 256], 512-token sequences), forward + backward + fused AdamW with fp32 moments, as bench.train_substep
runs it.

The plain and the checkpointed step (TrainEngine.checkpoint, what gradient_checkpointing_enable() turns on) run
alternately on the same engine. Reports per mode the peak torch.cuda.max_memory_allocated of a step and the median step
time (CUDA events, after warm-up), with the card name and power limit read in the same process.

    python tools/checkpoint_probe.py [--steps 6] [--warmup 2] [--out results.json]

The result is printed as one JSON line; --out also writes it to a file.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("checkpoint_probe needs a CUDA device")
    import bench
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    from u2tokenizer_b200.train import TrainEngine
    _, _, spec = bench.make_geometry("cfg4")
    _, geom, _ = bench.make_geometry("cfg2")
    spec = dict(spec, model="mu2-Qwen3-1.7B")
    sd = synthetic_state_dict(geom, seed=0, device="cuda", dtype=torch.bfloat16)
    te = TrainEngine(geom, sd, device="cuda")
    del sd
    torch.cuda.empty_cache()
    te.init_optimizer(lr=4e-6, weight_decay=0.0, max_grad_norm=1.0, moment_dtype=torch.float32)
    data = [t.cuda() for t in bench.train_batch(geom, spec, 0, 1)[:4]]
    state = torch.cuda.memory_allocated()

    def step(ck):
        te.checkpoint = ck
        te.zero_grad()
        loss = te.forward_backward(*data)
        te.optimizer_step()
        return loss
    modes = (False, True)
    for _ in range(args.warmup):
        for ck in modes:
            step(ck)
    times, peaks, loss = {ck: [] for ck in modes}, {ck: 0 for ck in modes}, {}
    for _ in range(args.steps):
        for ck in modes:   # alternating: clock and neighbour drift hit both modes alike
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss[ck] = step(ck)
            e1.record()
            torch.cuda.synchronize()
            times[ck].append(e0.elapsed_time(e1))
            peaks[ck] = max(peaks[ck], torch.cuda.max_memory_allocated())
    runs = [dict(checkpoint=ck, loss=float(loss[ck]), step_ms_median=sorted(times[ck])[len(times[ck]) // 2],
                 step_ms=times[ck], peak_alloc_gib=peaks[ck] / 2 ** 30,
                 activation_peak_gib=(peaks[ck] - state) / 2 ** 30) for ck in modes]
    res = dict(card=card(), model=spec["model"], batch=spec["batch"], frames=spec["frames"], seq=spec["seq"],
               moments="fp32", state_gib=state / 2 ** 30, runs=runs)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
