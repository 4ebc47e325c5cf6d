"""Video-level testing on one GPU: feature-extraction throughput of coclr_b200.evaluate (clips/s, videos of mixed
length so that packing and padding are exercised) next to bare engine passes of the same shape, and the retrieval
kernels (centre + normalise, fp32 FFMA similarity, rank) at the UCF101 split-1 shape against the reference's torch
fp32 arithmetic (:689-705: centre, F.normalize, matmul, topk + any for k in 1, 5, 10, 20, 50) on the same device.
CUDA events around warmed-up repetitions; prints one JSON line with the card name, power limit and SM clock.

  python tests/tools/bench_eval.py [--batch 32] [--seq 32] [--img 128] [--videos 95] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_classifier import gpu_info  # noqa: E402


def event_time(fn, reps, warmup):
    """Mean ms of fn() over reps calls after warmup calls, with CUDA events on the current stream."""
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def extraction(args, res):
    from model.classifier import LinearClassifier
    from coclr_b200.evaluate import evaluate, IMAGENET_MEAN, IMAGENET_STD
    model = LinearClassifier(num_class=101, network="s3d", use_dropout=False, use_l2_norm=True,
                             use_final_bn=True).cuda().eval()
    S, HW = args.seq, args.img
    g = torch.Generator(device="cuda").manual_seed(0)
    base = torch.rand(3, 7 * S + S - 1, HW, HW, device="cuda", generator=g)
    # 1-7 clips plus 0..S-1 leftover frames per video, views into one base tensor
    lengths = [(1 + (i * 5) % 7) * S + (i * 11) % S for i in range(args.videos)]
    videos = [(base[:, :T], i % 101, "v%04d" % i) for i, T in enumerate(lengths)]
    clips = sum(T // S for T in lengths)

    def run():
        evaluate(model, videos, S, args.batch)
    ms = event_time(run, args.reps, 1)
    res["extract/videos"] = args.videos
    res["extract/clips"] = clips
    res["extract/passes"] = -(-clips // args.batch)
    res["extract/ms"] = round(ms, 2)
    res["extract/clips_per_s"] = round(clips / ms * 1e3, 1)
    # bare passes: the same plan, one fixed [B, 3, S, H, W] batch, no staging or accumulation
    x = torch.rand(args.batch, 3, S, HW, HW, device="cuda", generator=g)
    norm = (torch.tensor(IMAGENET_MEAN, device="cuda"), torch.tensor(IMAGENET_STD, device="cuda"))
    passes = res["extract/passes"]

    def bare():
        for _ in range(passes):
            model.infer(x, norm=norm)
    ms_b = event_time(bare, args.reps, 2)
    res["extract/bare_passes_ms"] = round(ms_b, 2)
    res["extract/bare_clips_per_s"] = round(passes * args.batch / ms_b * 1e3, 1)
    del model
    torch.cuda.empty_cache()


def torch_retrieval(qf, ql, kf, kl, ks=(1, 5, 10, 20, 50)):
    q = F.normalize(qf - qf.mean(dim=0, keepdim=True), p=2, dim=1)
    k = F.normalize(kf - kf.mean(dim=0, keepdim=True), p=2, dim=1)
    sim = q.matmul(k.t())
    return sim, [torch.any(kl[torch.topk(sim, kk, dim=1)[1]] == ql.unsqueeze(1), dim=1).float().mean() for kk in ks]


def retrieval(args, res):
    from coclr_b200 import evaluate as EV
    torch.backends.cuda.matmul.allow_tf32 = False       # torch's default: the reference's matmul is fp32
    Nq, Nk = 3783, 9537
    for D in (1024, 2048):
        g = torch.Generator(device="cuda").manual_seed(D)
        ql = torch.randint(0, 101, (Nq,), device="cuda", generator=g)
        kl = torch.randint(0, 101, (Nk,), device="cuda", generator=g)
        centers = torch.randn(101, D, device="cuda", generator=g)
        qf = centers[ql] + 2 * torch.randn(Nq, D, device="cuda", generator=g)
        kf = centers[kl] + 2 * torch.randn(Nk, D, device="cuda", generator=g)
        qn, kn = EV.center_normalize(qf), EV.center_normalize(kf)
        sim = EV.similarity(qn, kn)
        key = "retrieval/D%d/" % D
        res[key + "normalize_ms"] = round(event_time(lambda: (EV.center_normalize(qf), EV.center_normalize(kf)),
                                                     args.reps * 5, 2), 4)
        ms = event_time(lambda: EV.similarity(qn, kn), args.reps * 5, 2)
        res[key + "sim_ms"] = round(ms, 4)
        res[key + "sim_tflops"] = round(2.0 * Nq * Nk * D / ms / 1e9, 2)
        res[key + "rank_ms"] = round(event_time(lambda: EV.retrieval_rank(sim, ql, kl), args.reps * 5, 2), 4)
        res[key + "engine_total_ms"] = round(event_time(lambda: EV.retrieval(qf, ql, kf, kl), args.reps * 5, 2), 4)
        res[key + "torch_fp32_total_ms"] = round(event_time(lambda: torch_retrieval(qf, ql, kf, kl), args.reps * 5, 2), 4)
        res[key + "torch_fp32_matmul_ms"] = round(event_time(lambda: torch.matmul(qn, kn.t()), args.reps * 5, 2), 4)
        acc = EV.retrieval(qf, ql, kf, kl)[2]
        tacc = [float(a) for a in torch_retrieval(qf, ql, kf, kl)[1]]
        res[key + "acc_engine"] = acc
        res[key + "acc_torch_fp32"] = tacc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=32)
    ap.add_argument("--img", type=int, default=128)
    ap.add_argument("--videos", type=int, default=95)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a CUDA device; none is available")
    res = {"gpu": gpu_info(), "net": "s3d", "batch": args.batch, "seq_len": args.seq, "img_dim": args.img,
           "reps": args.reps}
    extraction(args, res)
    retrieval(args, res)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res, sort_keys=True)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
