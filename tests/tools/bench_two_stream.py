"""Two-stream retrieval merge (eval/merge_2stream_prob.py --mode s) at the UCF101 split-1 shape: 3783 test x 9537 train
videos, D = 1024 per stream (S3D RGB + S3D flow).  Times, with CUDA events after warm-up:
  * the engine: coclr_sim2_fp32 (both streams into one similarity matrix) and coclr_retrieval_rank, and the whole
    two_stream_retrieval (four centre + normalise calls, sim2, rank);
  * the reference's arithmetic in torch fp32 on the same GPU: two matmuls and an add (and the five topk + any);
and, for context, the reference's merge_sim arithmetic (preprocess, two matmuls, add, five topk + any) on one host
core.  Prints one JSON line with the card name, power limit and SM clock.

  python tests/tools/bench_two_stream.py [--reps 20] [--cpu-reps 1] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_classifier import gpu_info  # noqa: E402
from bench_eval import event_time  # noqa: E402

NQ, NK, D, NCLS, KS = 3783, 9537, 1024, 101, (1, 5, 10, 20, 50)


def reference_merge_sim(te1, tr1, te2, tr2, ql, kl):
    """merge_sim :172-196 after the alignment: preprocess each set, sim1 + sim2, topk + any for each k."""
    def pre(x):
        return F.normalize(x - x.mean(dim=0, keepdim=True), p=2, dim=1)
    sim = pre(te1).matmul(pre(tr1).t()) + pre(te2).matmul(pre(tr2).t())
    return [torch.any(kl[torch.topk(sim, k, dim=1)[1]] == ql.unsqueeze(1), dim=1).float().mean() for k in KS]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-reps", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_two_stream.py measures on a CUDA device; none is available")
    from coclr_b200 import evaluate as EV
    torch.backends.cuda.matmul.allow_tf32 = False       # torch's default: the reference's matmul is fp32
    res = {"gpu": gpu_info(), "Nq": NQ, "Nk": NK, "D1": D, "D2": D, "reps": args.reps}
    g = torch.Generator(device="cuda").manual_seed(0)
    ql = torch.randint(0, NCLS, (NQ,), device="cuda", generator=g)
    kl = torch.randint(0, NCLS, (NK,), device="cuda", generator=g)
    feats = []
    for _ in range(2):
        centers = torch.randn(NCLS, D, device="cuda", generator=g)
        feats.append((centers[ql] + 10 * torch.randn(NQ, D, device="cuda", generator=g),
                      centers[kl] + 10 * torch.randn(NK, D, device="cuda", generator=g)))
    (te1, tr1), (te2, tr2) = feats
    q1, k1, q2, k2 = (EV.center_normalize(x) for x in (te1, tr1, te2, tr2))
    sim = EV.similarity2(q1, k1, q2, k2)
    res["engine/sim2_ms"] = round(event_time(lambda: EV.similarity2(q1, k1, q2, k2), args.reps, 3), 4)
    res["engine/sim2_tflops"] = round(2.0 * NQ * NK * 2 * D / res["engine/sim2_ms"] / 1e9, 2)
    res["engine/rank_ms"] = round(event_time(lambda: EV.retrieval_rank(sim, ql, kl), args.reps, 3), 4)
    res["engine/sim2_plus_rank_ms"] = round(event_time(
        lambda: EV.retrieval_rank(EV.similarity2(q1, k1, q2, k2), ql, kl), args.reps, 3), 4)
    res["engine/total_ms"] = round(event_time(
        lambda: EV.two_stream_retrieval(te1, tr1, te2, tr2, ql, kl), args.reps, 3), 4)
    res["torch_fp32/two_matmuls_add_ms"] = round(event_time(lambda: q1.matmul(k1.t()) + q2.matmul(k2.t()),
                                                            args.reps, 3), 4)
    res["torch_fp32/total_ms"] = round(event_time(lambda: reference_merge_sim(te1, tr1, te2, tr2, ql, kl),
                                                  args.reps, 3), 4)
    res["acc_engine"] = EV.two_stream_retrieval(te1, tr1, te2, tr2, ql, kl)[2]
    res["acc_torch_fp32"] = [float(a) for a in reference_merge_sim(te1, tr1, te2, tr2, ql, kl)]
    res["gpu_after"] = gpu_info()
    torch.set_num_threads(1)
    cpu = [t.cpu() for t in (te1, tr1, te2, tr2, ql, kl)]
    reference_merge_sim(*cpu)
    t0 = time.perf_counter()
    for _ in range(args.cpu_reps):
        acc_cpu = reference_merge_sim(*cpu)
    res["cpu_1core/total_ms"] = round((time.perf_counter() - t0) * 1e3 / args.cpu_reps, 1)
    res["acc_cpu"] = [float(a) for a in acc_cpu]
    line = json.dumps(res, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
