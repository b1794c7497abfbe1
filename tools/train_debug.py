"""Per-parameter gradient report of TrainEngine against the oracle's autograd (debugging aid; needs a GPU)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from common import cosine, rel_err, tiny_geometry  # noqa: E402
from test_train_gpu import CASES, _labels, _oracle_loss_and_grads  # noqa: E402
from u2tokenizer_b200.synthetic import synthetic_inputs, synthetic_state_dict  # noqa: E402
from u2tokenizer_b200.train import TrainEngine  # noqa: E402

case = sys.argv[1] if len(sys.argv) > 1 else "qwen3_rma_diffts_dmtp"
g = tiny_geometry(**CASES[case])
sd16 = synthetic_state_dict(g, seed=21, device="cpu", dtype=torch.bfloat16)
sd16["model.u2tokenizer.query_tokens"] = (sd16["model.u2tokenizer.query_tokens"].float() * 50).to(torch.bfloat16)
images, ids, qids = synthetic_inputs(g, batch=2, frames=3, n_question=7, lt=12)
labels = _labels(ids, g.num_3d_query_token)
ref_loss, ref_g = _oracle_loss_and_grads(sd16, g, images, ids, qids, labels)
te = TrainEngine(g, sd16, device="cuda")
te.zero_grad()
loss = te.forward_backward(images.cuda(), ids.cuda(), qids.cuda(), labels.cuda())
torch.cuda.synchronize()
print("loss", float(loss), ref_loss)
L = te.lay
for n in L.mat_names + L.vec_names:
    got = te.grad(n).float().cpu()
    want = ref_g.get(n)
    if want is None:
        continue
    want = want.cpu()
    e, c = rel_err(got, want), cosine(got, want)
    flag = "" if (e < 4e-2 and c > 0.995) or want.abs().max() < 1e-9 else "   <<<<"
    print(f"{n:95s} rel {e:9.4g} cos {c:8.5f} |got| {got.abs().max().item():9.3g} |want| {want.abs().max().item():9.3g}{flag}")
