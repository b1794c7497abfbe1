"""What the generation-score options cost per decode step.

Model: the cfg 3 geometry (mu2-Qwen3-8B) with synthetic weights; prompts of --prompt token embeddings (the vision front
is not part of the decode step). For B in --batches decode rows and each head (greedy, sampled with top-p 0.9, beam
search with K = 4, i.e. B / 4 prompts), the options run off and one at a time:

  generate()        off, output_scores, output_logits (engine.generate)
  generate_batch()  off, return_logprobs (engine.generate_continuous, B slots, B requests; greedy and sampled only)

A decode step's time is (T(--new) - T(1)) / (--new - 1), where T(n) is the wall time of the call with max_new_tokens =
n, EOS off, closed by a device synchronise: the prefill, the first pick and the host's set-up cancel. All variants
alternate in one process, --repeats times; the median is reported. Prints one JSON line per variant and a summary
with the card's name, power limit and max SM clock, read in the same run.

    python tools/generation_scores_probe.py [--batches 4,16] [--new 256] [--repeats 3] [--out result.json]
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
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers still print; the card is then reported unknown
        return f"unknown ({e})"


HEADS = {"greedy": dict(), "sampled": dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9, seed=1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4,16")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generation_scores_probe needs a CUDA device")
    import bench
    from u2tokenizer_b200.engine import BeamSearch, SlotRequest
    cfg, geom, spec = bench.make_geometry(a.workload)
    eng = bench.build_model(cfg, geom).engine()
    gen = torch.Generator().manual_seed(11)

    def variants(B):
        emb = eng.embed_tokens(torch.randint(0, geom.vocab_size, (B, a.prompt), generator=gen).cuda())
        beam = BeamSearch(num_beams=4)
        out = []
        for head in ("greedy", "sampled", "beam"):
            kw = dict(beam=beam) if head == "beam" else HEADS[head]
            e = emb[:B // 4] if head == "beam" else emb
            for opt in ("off", "output_scores", "output_logits"):
                flags = {} if opt == "off" else {opt: True}
                out.append((head, opt, lambda n, e=e, kw=kw, flags=flags: eng.generate(e, n, **kw, **flags)))
            if head != "beam":
                for opt in ("off", "return_logprobs"):
                    flags = {} if opt == "off" else {opt: True}
                    kw2 = {k: v for k, v in kw.items() if k != "seed"}
                    out.append((head, "batch " + opt, lambda n, kw2=kw2, flags=flags: eng.generate_continuous(
                        (SlotRequest(str(i), emb[i:i + 1], n) for i in range(B)), B, **kw2, **flags)))
        return out

    def call(fn, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(n)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    gpu = card()
    rows = []
    for B in [int(x) for x in a.batches.split(",")]:
        vs = variants(B)
        for _, _, fn in vs:  # warm-up: captures, kernel attributes, allocator
            call(fn, a.new)
            call(fn, 1)
        times = {(h, o): [] for h, o, _ in vs}
        for rep in range(a.repeats):
            for h, o, fn in (vs if rep % 2 == 0 else vs[::-1]):
                times[(h, o)].append((call(fn, a.new) - call(fn, 1)) / (a.new - 1))
        for (h, o), ts in times.items():
            ms = sorted(ts)[len(ts) // 2] * 1e3
            off = sorted(times[(h, "batch off" if o.startswith("batch") else "off")])[len(ts) // 2] * 1e3
            rec = dict(rows=B, head=h, option=o, step_ms=round(ms, 4), vs_off_us=round((ms - off) * 1e3, 1),
                       spread_ms=round((max(ts) - min(ts)) * 1e3, 4))
            rows.append(rec)
            print(json.dumps(rec), flush=True)
    summary = dict(card=gpu, workload=a.workload, new_tokens=a.new, prompt=a.prompt, repeats=a.repeats, runs=rows)
    print(json.dumps(dict(card=gpu, workload=a.workload, new_tokens=a.new)), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
