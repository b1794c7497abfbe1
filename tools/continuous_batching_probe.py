"""Continuous batching against static batches on report generation over a dataset.

Model: the cfg 3 geometry (mu2-Qwen3-8B) with synthetic weights, 256^3 synthetic volumes (8 frames), `--studies`
studies. Each study asks for its own max_new_tokens, drawn from a seeded uniform distribution on [64, 768]: this is an
assumption, since no distribution of real report lengths is available. EOS is off, so every request runs to its
max_new_tokens and the two schedules do the same useful work.

  static      generate() over arrival-order chunks of --slots studies; a chunk runs to its longest request
  continuous  generate_batch(num_slots=--slots)

Both run greedy, in one process, alternating, --repeats times. Prints one JSON line per run and a summary line: wall
time, generated tokens/s, studies/s, mean slot occupancy (generated tokens over decode-step rows), graph captures, the
fraction of studies whose ids agree between the two schedules, and the card's name and power limit. --poll N1,N2,...
adds continuous runs at other polling intervals (engine.SLOT_POLL_STEPS) after the comparison.

    python tools/continuous_batching_probe.py [--studies 64] [--slots 16] [--repeats 3] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers still print; the card is then reported unknown
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--studies", type=int, default=64)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--lo", type=int, default=64)
    ap.add_argument("--hi", type=int, default=768)
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--poll", default="")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("continuous_batching_probe needs a CUDA device")
    import bench
    from u2tokenizer_b200 import engine as E
    from u2tokenizer_b200.synthetic import synthetic_inputs
    cfg, geom, spec = bench.make_geometry(a.workload)
    model = bench.build_model(cfg, geom)
    model.generation_config.eos_token_id = None
    eng = model.engine()
    gen = torch.Generator().manual_seed(2024)
    news = torch.randint(a.lo, a.hi + 1, (a.studies,), generator=gen).tolist()
    studies = [synthetic_inputs(geom, batch=1, frames=spec["frames"], n_question=spec["n_question"], lt=spec["lt"],
                                seed=7000 + i) for i in range(a.studies)]
    useful = sum(news)

    def static():
        out, steps = {}, 0
        for c0 in range(0, a.studies, a.slots):
            idx = list(range(c0, min(a.studies, c0 + a.slots)))
            images = torch.cat([studies[i][0] for i in idx]).cuda()
            ids = torch.cat([studies[i][1] for i in idx]).cuda()
            q = torch.cat([studies[i][2] for i in idx]).cuda()
            n = max(news[i] for i in idx)
            rows = model.generate(images, ids, question_ids=q, max_new_tokens=n, do_sample=False).cpu()
            steps += n - 1
            for r, i in enumerate(idx):
                out[str(i)] = rows[r, :news[i]].tolist()
        return out, dict(steps=steps, captures=None)

    def continuous():
        reqs = (dict(images=im, input_ids=ids, question_ids=q, max_new_tokens=news[i])
                for i, (im, ids, q) in enumerate(studies))
        res = model.generate_batch(reqs, num_slots=a.slots, do_sample=False)
        st = eng.last_continuous
        return {k: v.generated_tokens for k, v in res.items()}, dict(steps=st["steps"], captures=st["captures"])

    def timed(name, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, info = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        decode_rows = info["steps"] * a.slots
        rec = dict(run=name, wall_s=round(dt, 3), tokens_per_s=round(useful / dt, 1),
                   studies_per_s=round(a.studies / dt, 4), decode_steps=info["steps"],
                   occupancy=round((useful - a.studies) / decode_rows, 4), captures=info["captures"],
                   poll=E.SLOT_POLL_STEPS)
        print(json.dumps(rec), flush=True)
        return out, rec

    gpu = card()
    timed("warmup-continuous", continuous)
    timed("warmup-static", static)
    runs, agree = [], []
    for rep in range(a.repeats):
        order = (("static", static), ("continuous", continuous))
        outs = {}
        for name, fn in (order if rep % 2 == 0 else order[::-1]):
            outs[name], rec = timed(name, fn)
            runs.append(rec)
        agree.append(sum(outs["static"][k] == outs["continuous"][k] for k in outs["static"]) / a.studies)
    for p in [int(x) for x in a.poll.split(",") if x]:
        E.SLOT_POLL_STEPS = p
        timed("continuous-poll", continuous)
    med = lambda name, k: sorted(r[k] for r in runs if r["run"] == name)[a.repeats // 2]
    summary = dict(card=gpu, workload=a.workload, studies=a.studies, slots=a.slots,
                   max_new_tokens=f"uniform[{a.lo}, {a.hi}] seed 2024", useful_tokens=useful,
                   static_wall_s=med("static", "wall_s"), continuous_wall_s=med("continuous", "wall_s"),
                   static_tokens_per_s=med("static", "tokens_per_s"),
                   continuous_tokens_per_s=med("continuous", "tokens_per_s"),
                   static_occupancy=med("static", "occupancy"), continuous_occupancy=med("continuous", "occupancy"),
                   speedup=round(med("static", "wall_s") / med("continuous", "wall_s"), 3),
                   ids_agree=min(agree), runs=runs)
    print(json.dumps({k: v for k, v in summary.items() if k != "runs"}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
