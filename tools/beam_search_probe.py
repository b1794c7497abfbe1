"""Beam search decode step at the cfg 3 geometry (mu2-Qwen3-8B, 8 frames of 256^3 per study, 256 new tokens), against
greedy decoding at the same number of rows: num_beams = 4 with 1 study (4 rows) and 4 studies (16 rows).

Reports, from CUDA events around whole generate calls (each shape warmed up first, decode graphs captured):
  ms per decode step: (a call of --new tokens - a call of 2 tokens) / (--new - 2) on the same prompt embeddings,
  the beam kernels' share of a step: log_softmax + per-row top-k + per-prompt merge on the rows' fp32 logits, timed
  alone over --reps launches, over the beam step time,
  greedy with an identity cache indirection table: the cost of the table-driven attention reads alone,
  the GPU name and power limit, read in the same run.
No EOS id is set, so every call runs its --new steps. The weights are synthetic with a bigram-structured head
(synthetic_state_dict(bigram=0.35), as tools/ragged_generate_probe.py).
usage: python tools/beam_search_probe.py [--new 256] [--beams 4] [--reps 200]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from ragged_generate_probe import build_model, gpu_info, timed_ms  # noqa: E402


def step_ms(run, n_new):
    run(n_new), run(2)
    t_long, _ = timed_ms(lambda: run(n_new), 2)
    t_short, _ = timed_ms(lambda: run(2), 2)
    return (t_long - t_short) / (n_new - 2)


def beam_kernels_ms(eng, rows, K, n_new, reps):
    """The three beam kernels of one step on random logits [rows, V], in the state a generate call leaves."""
    from u2tokenizer_b200 import ops
    st = eng._gen_state
    bs, cache = st["beam"], st["cache"]
    blk = ops.beam_params(eng.dev, num_beams=K, max_new_tokens=n_new)
    logits = torch.randn(rows, eng.g.vocab_size, device=eng.dev) * 3
    ids = torch.zeros(rows, device=eng.dev, dtype=torch.int64)
    # the state at the start of a request; with no EOS id and step 1 < max_new_tokens - 1 no candidate finishes, so the
    # heuristic stays unsatisfied and no prompt becomes done: every timed launch does the full work
    bs["running"].view(-1, K).fill_(-1e9)[:, 0] = 0.0
    bs["fin_score"].fill_(-1e9)
    bs["fin_info"].copy_(torch.tensor([0, -1, 0, 0], dtype=torch.int32).expand(rows, 4))
    bs["flags"].copy_(torch.tensor([1, 0], dtype=torch.int32).expand(rows // K, 2))

    def once():
        lp = ops.log_softmax(logits, bs["lp"])
        ops.beam_topk(lp, bs["running"], bs["flags"], blk, bs["cand_val"], bs["cand_tok"])
        ops.beam_step(blk, bs, ids, cache.kv_src, cache.length_dev, V=eng.g.vocab_size, step=1)
    once()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        once()
    e1.record()
    torch.cuda.synchronize()
    if bool(bs["flags"][:, 1].any()):
        raise RuntimeError("a prompt became done during the timed loop: the timing would miss work")
    return e0.elapsed_time(e1) / reps


def greedy_indirect_step_ms(eng, emb, n_new):
    """Greedy decode with an identity indirection table on every cache: the same ids as greedy, through the attention
    kernels beam search uses (table lookup before each K/V row). Isolates their cost from the beam kernels'."""
    orig = eng.new_cache

    def new_cache(B, L):
        c = orig(B, L)
        c.kv_src = torch.arange(B, device=eng.dev, dtype=torch.int32)[:, None].expand(B, L).contiguous()
        return c
    eng.new_cache = new_cache
    eng._gen_state = None
    try:
        return step_ms(lambda n: eng.generate_greedy(emb, n), n_new)
    finally:
        eng.new_cache = orig
        eng._gen_state = None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--beams", type=int, default=4)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beam_search_probe needs a CUDA device (H100)")
    from u2tokenizer_b200.engine import BeamSearch
    from u2tokenizer_b200.synthetic import synthetic_inputs
    name, pl = gpu_info()
    cfg, geom, spec = bench.make_geometry("cfg3")
    model = build_model(cfg, geom)
    eng = model.engine()
    K, n_new = args.beams, args.new
    im, rid, rq = (t.cuda() for t in synthetic_inputs(geom, batch=1, frames=spec["frames"], n_question=40,
                                                        lt=spec["lt"], seed=500))
    with torch.no_grad():
        emb1 = eng.multimodal_embeds(rid, im, rq)
    res = dict(probe="beam_search", gpu=name, power_limit_max_sm_clock=pl, model=spec["model"],
               frames_per_study=spec["frames"], image_size=list(geom.image_size), new_tokens=n_new, num_beams=K, runs=[])
    bm = BeamSearch(num_beams=K)
    for studies in (1, 16 // K):
        emb = emb1.expand(studies, -1, -1).contiguous()
        rows = studies * K
        beam = step_ms(lambda n: eng.generate(emb, n, beam=bm), n_new)
        kern = beam_kernels_ms(eng, rows, K, n_new, args.reps)
        embr = emb1.expand(rows, -1, -1).contiguous()
        greedy = step_ms(lambda n: eng.generate_greedy(embr, n), n_new)
        indirect = greedy_indirect_step_ms(eng, embr, n_new)
        rec = dict(studies=studies, rows=rows, beam_step_ms=round(beam, 3), greedy_step_ms_same_rows=round(greedy, 3),
                   greedy_step_ms_identity_table=round(indirect, 3), beam_kernels_ms=round(kern, 4),
                   beam_kernels_share_of_step=round(kern / beam, 4))
        res["runs"].append(rec)
        print(json.dumps(rec), file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
