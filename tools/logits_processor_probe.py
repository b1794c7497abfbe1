"""Cost of generate()'s logits processors (repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=64 and 8 bad
words) in the decode step, at the cfg 3 geometry (mu2-Qwen3-8B, 8 frames of 256^3 per study, 256 new tokens).

Per batch size it reports:
  ms per decode step with the processors off and on: (generate_greedy of N - of 2 new tokens) / (N - 2) on the same
  prompt embeddings, decode graph captured, off / on alternated over --rounds rounds (min and median);
  the processors kernel alone at a history of 768 tokens: CUDA events around --launches back-to-back launches;
  ids: whether the processors changed the greedy ids (they should, on this head).
The weights are synthetic with a bigram-structured head (as tools/ragged_generate_probe.py). B = 16 replicates the 4
studies' prompt embeddings, so only 4 studies go through the vision path.
One JSON line per run, with the GPU name and power limit read in the same run.
usage: python tools/logits_processor_probe.py [--batches 4,16] [--new 256] [--rounds 3] [--launches 200]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from ragged_generate_probe import build_model, gpu_info, timed_ms  # noqa: E402


def processors(vocab):
    from u2tokenizer_b200.engine import LogitsProcessors
    g = torch.Generator().manual_seed(0)
    words = tuple(tuple(int(x) for x in torch.randint(0, vocab, (1 + i % 3,), generator=g)) for i in range(8))
    return LogitsProcessors(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=64,
                            eos_token_ids=(151643, 151645), bad_words_ids=words)


def kernel_us(eng, pc, B, t, launches):
    from dataclasses import asdict
    from u2tokenizer_b200 import ops
    V = eng.g.vocab_size
    logits = torch.randn(B, V, device="cuda")
    hist = torch.randint(0, 2000, (B, t + 8), device="cuda", dtype=torch.int32)
    ids = hist[:, t - 1].long().contiguous()
    step = torch.full((1,), t, device="cuda", dtype=torch.int32)
    blk = eng._param_block("logits processors", ops.logits_proc_params, V, **asdict(pc))
    run = lambda: ops.logits_process(logits, blk, ids, hist, step_dev=step)
    for _ in range(10):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4,16")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logits_processor_probe needs a CUDA device (H100)")
    name, pl = gpu_info()
    cfg, geom, spec = bench.make_geometry("cfg3")
    model = build_model(cfg, geom)
    eng = model.engine()
    pc = processors(geom.vocab_size)
    from u2tokenizer_b200.synthetic import synthetic_inputs
    images, ids, qids = synthetic_inputs(geom, batch=4, frames=spec["frames"], n_question=spec["n_question"],
                                         lt=spec["lt"], seed=500)
    with torch.no_grad():
        emb4 = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    n_new = args.new
    res = dict(probe="logits_processor", gpu=name, power_limit_max_sm_clock=pl, model=spec["model"],
               frames_per_study=spec["frames"], image_size=list(geom.image_size), new_tokens=n_new,
               processors=dict(repetition_penalty=pc.repetition_penalty, no_repeat_ngram_size=pc.no_repeat_ngram_size,
                               min_new_tokens=pc.min_new_tokens, bad_words=len(pc.bad_words_ids)), runs=[])
    for B in [int(x) for x in args.batches.split(",")]:
        emb = emb4.repeat((B + 3) // 4, 1, 1)[:B].contiguous()
        run = lambda n, p: eng.generate_greedy(emb, n, processors=p)
        for p in (None, pc):  # capture the decode graph of both capacities, with and without the processors
            run(n_new, p), run(2, p)
        steps = {"off": [], "on": []}
        for _ in range(args.rounds):
            for key, p in (("off", None), ("on", pc)):
                # best of 2: switching processors or capacity swaps the generation state and re-captures the step
                t_long, _ = timed_ms(lambda: run(n_new, p), 2)
                t_short, _ = timed_ms(lambda: run(2, p), 2)
                steps[key].append((t_long - t_short) / (n_new - 2))
        ids_off, ids_on = run(n_new, None), run(n_new, pc)
        off, on = statistics.median(steps["off"]), statistics.median(steps["on"])
        rec = dict(batch=B, decode_step_ms_off=[round(x, 3) for x in steps["off"]],
                   decode_step_ms_on=[round(x, 3) for x in steps["on"]],
                   median_off_ms=round(off, 3), median_on_ms=round(on, 3),
                   overhead_pct_of_median=round(100 * (on - off) / off, 2),
                   kernel_us_at_t768=round(kernel_us(eng, pc, B, 768, args.launches), 2),
                   ids_changed=not torch.equal(ids_off, ids_on))
        res["runs"].append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
