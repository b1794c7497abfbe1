"""Ragged batch generate() against one call per study at the cfg 3 geometry (mu2-Qwen3-8B, 8 frames of 256^3 per
study, 256 new tokens): B studies whose questions have different lengths (spread over 8..120 tokens) run as ONE
model.generate(..., attention_mask=mask) call, and as B calls of one study each (what an eval loop that asks a
different question per study does without padding).

Per batch size it reports, from CUDA events around whole calls (each shape warmed up first):
  volumes/s of the ragged call and of the per-study calls (best of --reps),
  ms per decode step: (generate_greedy of 256 - of 2 new tokens) / 254 on the same prompt embeddings, for the ragged
  batch and for one study alone (the steady-state step, decode graph captured),
  ids: rows identical to the per-study call, and the tokens identical before the first difference.
The weights are synthetic with a bigram-structured head (synthetic_state_dict(bigram=0.35), as the cfg 3 full-depth
test uses): an i.i.d. random head has top-1 / top-2 margins of the order of the bf16 noise, so its ids would compare nothing.
One JSON line per run, with the GPU name and power limit read in the same run.
usage: python tools/ragged_generate_probe.py [--batches 4,8] [--new 256] [--reps 2]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        pl = f"unknown ({e})"
    return name, pl


def build_model(cfg, geom):
    """bench.build_model with a bigram-structured head (decisive greedy margins)."""
    from u2tokenizer_b200.modeling import U2Qwen3ForCausalLM
    from u2tokenizer_b200.synthetic import synthetic_state_dict
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        with torch.device("cuda"):
            model = U2Qwen3ForCausalLM(cfg)
    finally:
        torch.set_default_dtype(prev)
    sd = synthetic_state_dict(geom, seed=0, device="cuda", dtype=torch.bfloat16, bigram=0.35)
    _, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    del sd
    model.eval()
    model.generation_config.eos_token_id = None
    torch.cuda.empty_cache()
    return model


def timed_ms(fn, reps):
    best, out = None, None
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        best = ms if best is None else min(best, ms)
    return best, out


def studies(geom, spec, B):
    from u2tokenizer_b200.synthetic import synthetic_inputs
    qlens = [round(8 + (120 - 8) * i / max(1, B - 1)) for i in range(B)]
    rows = [synthetic_inputs(geom, batch=1, frames=spec["frames"], n_question=n, lt=spec["lt"], seed=500 + i)
            for i, n in enumerate(qlens)]
    lens = [r[1].shape[1] for r in rows]
    L = max(lens)
    ids = torch.zeros(B, L, dtype=torch.long)
    mask = torch.zeros(B, L, dtype=torch.long)
    for b, (_, rid, _) in enumerate(rows):
        ids[b, :lens[b]] = rid[0]
        mask[b, :lens[b]] = 1
    dev = lambda t: t.cuda()
    rows = [tuple(map(dev, r)) for r in rows]
    batch = (dev(torch.cat([r[0] for r in rows])), dev(ids), dev(torch.cat([r[2] for r in rows])), dev(mask))
    return qlens, lens, rows, batch


def decode_step_ms(eng, emb, lens, n_new):
    """Steady-state decode step: the difference of two generate_greedy calls on the same embeddings."""
    run = lambda n: eng.generate_greedy(emb, n, lengths=lens)
    run(n_new), run(2)  # capture the decode graph for both capacities' first use
    t_long, _ = timed_ms(lambda: run(n_new), 2)
    t_short, _ = timed_ms(lambda: run(2), 2)
    return (t_long - t_short) / (n_new - 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="4,8")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_generate_probe needs a CUDA device (H100)")
    name, pl = gpu_info()
    cfg, geom, spec = bench.make_geometry("cfg3")
    model = build_model(cfg, geom)
    eng = model.engine()
    n_new = args.new
    kw = dict(max_new_tokens=n_new, do_sample=False)
    res = dict(probe="ragged_generate", gpu=name, power_limit_max_sm_clock=pl, model=spec["model"],
               frames_per_study=spec["frames"], image_size=list(geom.image_size), new_tokens=n_new, runs=[])
    for B in [int(x) for x in args.batches.split(",")]:
        qlens, lens, rows, (images, ids, qids, mask) = studies(geom, spec, B)
        ragged = lambda: model.generate(images, ids, question_ids=qids, attention_mask=mask, **kw)
        per_study = lambda: [model.generate(im, rid, question_ids=rq, **kw) for im, rid, rq in rows]
        ragged(), per_study()  # warm-up: kernel attributes, graph captures, allocator
        t_rag, got = timed_ms(ragged, args.reps)
        t_one, alone = timed_ms(per_study, args.reps)
        same_rows, prefix = 0, []
        for b in range(B):
            a, r = got[b].cpu(), alone[b][0].cpu()
            same_rows += int(torch.equal(a, r))
            diff = (a != r).nonzero()
            prefix.append(int(diff[0]) if len(diff) else n_new)
        with torch.no_grad():
            emb = eng.multimodal_embeds(ids, images, qids)
            emb1 = eng.multimodal_embeds(rows[0][1], rows[0][0], rows[0][2])
        step_rag = decode_step_ms(eng, emb, lens, n_new)
        step_one = decode_step_ms(eng, emb1, None, n_new)
        rec = dict(batch=B, question_tokens=qlens, prompt_tokens=lens,
                   ragged_ms=round(t_rag, 1), per_study_ms=round(t_one, 1),
                   ragged_volumes_per_s=round(B / (t_rag / 1e3), 3), per_study_volumes_per_s=round(B / (t_one / 1e3), 3),
                   speedup=round(t_one / t_rag, 2),
                   decode_step_ms_ragged=round(step_rag, 3), decode_step_ms_one_study=round(step_one, 3),
                   rows_identical_to_per_study=f"{same_rows}/{B}", identical_prefix_tokens=prefix)
        res["runs"].append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
