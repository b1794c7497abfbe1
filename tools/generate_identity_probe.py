"""Records what generate() returns for a fixed set of requests, so two versions of the package can be compared bit for
bit: greedy, sampled (one and nine samples per prompt), logits processors and beam search, at batches inside one
decode chunk and across chunk boundaries, under decode_impl "tcgen05" and "gemv", at the tiny test geometry with
synthetic weights and fixed seeds. Every case runs twice (the second call replays the captured decode graph).

For every call it saves the ids, last_beam_scores (beam search) and the number of kernels launched (_lib.launches()
delta); generate_greedy's test hooks (margins, teacher forcing, per-step logits) are recorded too.

usage: python tools/generate_identity_probe.py --out a.pt [--root TREE]   (TREE: the checkout whose package runs)
       python tools/generate_identity_probe.py --compare a.pt b.pt        (exit 1 unless every entry is equal)"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def record(root):
    sys.path[:0] = [root, os.path.join(root, "tests")]
    from common import tiny_geometry
    from u2tokenizer_b200 import _lib
    from u2tokenizer_b200.engine import BeamSearch, LogitsProcessors, U2Engine
    from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict
    g = tiny_geometry()
    eng = U2Engine(g, synthetic_state_dict(g, seed=3, device="cpu", dtype=torch.bfloat16, bigram=1.0), device="cuda")
    images, ids, qids = synthetic_inputs(g, batch=20, frames=2, n_question=8, lt=12, seed=100)
    with torch.no_grad():
        emb = eng.multimodal_embeds(ids.cuda(), images.cuda(), qids.cuda())
    L = emb.shape[1]
    lens = [L - (3 * b) % 7 for b in range(20)]
    res = {}

    def call(name, fn):
        for rep in range(2):
            eng.last_beam_scores = None
            n0 = _lib.launches()
            out = fn()
            torch.cuda.synchronize()
            n = _lib.launches() - n0
            scores = eng.last_beam_scores
            rec = dict(launches=n, scores=None if scores is None else scores.cpu())
            if isinstance(out, tuple):
                rec["ids"], rec["margins"] = out[0].cpu(), out[1].cpu()
            else:
                rec["ids"] = out.cpu()
            res[f"{name}/{rep}"] = rec
            print(f"{name}/{rep}: ids {tuple(rec['ids'].shape)} launches {n}", flush=True)
        return out

    for impl in ("tcgen05", "gemv"):
        eng.decode_impl = impl
        eng._gen_state = None
        n_new = 24
        plain = call(f"{impl}/greedy_b3", lambda: eng.generate(emb[:3], n_new, lengths=lens[:3]))
        eos = [int(plain[0, 5]), int(plain[2, 9])]
        words = ((int(plain[1, 3]),), (int(plain[0, 7]), int(plain[0, 8])))
        pc = LogitsProcessors(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=4, eos_token_ids=tuple(eos),
                              bad_words_ids=words)
        res[f"{impl}/eos"] = dict(ids=torch.tensor(eos))
        call(f"{impl}/greedy_b3_eos", lambda: eng.generate(emb[:3], n_new, eos_token_id=eos, lengths=lens[:3]))
        call(f"{impl}/greedy_b20_eos", lambda: eng.generate(emb, n_new, eos_token_id=eos, lengths=lens))
        # every row of the first chunk (8 or 16 rows) meets one of these early, the last rows may not: the chunks end
        # at different widths and the short ones are padded with the first EOS id
        plain20 = call(f"{impl}/greedy_b20", lambda: eng.generate(emb, n_new, lengths=lens))
        stops = sorted({int(x) for x in plain20[:16 if impl == "tcgen05" else 8, 2]})
        res[f"{impl}/stops"] = dict(ids=torch.tensor(stops))
        call(f"{impl}/greedy_b20_early_stop", lambda: eng.generate(emb, n_new, eos_token_id=stops, lengths=lens))
        call(f"{impl}/sampled_b3", lambda: eng.generate(emb[:3], n_new, eos_token_id=eos, do_sample=True,
                                                         temperature=0.8, top_k=20, top_p=0.9, seed=11, lengths=lens[:3]))
        call(f"{impl}/sampled_b20", lambda: eng.generate(emb, n_new, do_sample=True, temperature=1.2, top_k=0,
                                                          top_p=0.95, seed=12, lengths=lens))
        call(f"{impl}/sampled_n9_b2", lambda: eng.generate(emb[:2], n_new, eos_token_id=eos, do_sample=True, seed=13,
                                                            num_return_sequences=9, lengths=lens[:2]))
        call(f"{impl}/greedy_procs_b3", lambda: eng.generate(emb[:3], n_new, eos_token_id=eos, lengths=lens[:3],
                                                              processors=pc))
        call(f"{impl}/sampled_procs_b3", lambda: eng.generate(emb[:3], n_new, eos_token_id=eos, do_sample=True,
                                                               seed=14, lengths=lens[:3], processors=pc))
        for name, prompts, bm, procs in (
                ("beam_procs_k4_b3", 3, BeamSearch(num_beams=4, length_penalty=1.5, num_return_sequences=2), pc),
                ("beam_k4_n2_b5", 5, BeamSearch(num_beams=4, num_return_sequences=2, pad_token_id=eos[0]), None)):
            call(f"{impl}/{name}", lambda: eng.generate(emb[:prompts], n_new, eos_token_id=eos, lengths=lens[:prompts],
                                                        beam=bm, processors=procs))
        # generate_greedy's hooks: margins (eager steps), teacher forcing and the per-step logits
        lo = []
        call(f"{impl}/greedy_margins_b3", lambda: eng.generate_greedy(emb[:3], 12, lengths=lens[:3],
                                                                      return_margins=True))
        force = plain[:, :12]
        out = eng.generate_greedy(emb[:3], 12, lengths=lens[:3], force_ids=force, logits_out=lo, processors=pc)
        res[f"{impl}/greedy_forced_logits_b3"] = dict(ids=out.cpu(), logits=torch.stack([x.cpu() for x in lo]))
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
    print(f"{len(a)} / {len(b)} entries; differences: {bad if bad else 'none'}")
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
        raise SystemExit("generate_identity_probe needs a CUDA device")
    torch.save(record(os.path.abspath(args.root)), args.out)


if __name__ == "__main__":
    main()
