"""Float64 restatements of the reference's video-level test arithmetic (eval/main_classifier.py) in stock PyTorch ops --
TEST INFRASTRUCTURE ONLY.  tests/test_eval_cpu.py pins the rank formula against the reference's topk / any formula;
tests/test_eval_gpu.py and tests/tools/bench_eval.py compare the engine's kernels (csrc/evaluate.cu) with these."""
import torch
import torch.nn.functional as F


def video_means(logits, feats):
    """One video: softmax(logit).mean(0) and feature.mean(0) over its clips (:488, :637), float64."""
    return F.softmax(logits.double(), dim=-1).mean(0), feats.double().mean(0)


def topk_hits(prob, target, ks=(1, 5)):
    """calc_topk_accuracy (utils/utils.py:52-71) per video: [len(ks), Nv] bool."""
    pred = prob.topk(max(ks), dim=1).indices
    return torch.stack([(pred[:, :k] == target.view(-1, 1)).any(1) for k in ks])


def class_rank(prob, target):
    """Classes ranked above the target: higher probability, ties to the lower index; C for a target outside [0, C)."""
    C = prob.shape[1]
    valid = (target >= 0) & (target < C)
    t = torch.where(valid, target, torch.zeros_like(target))
    pt = prob.gather(1, t.view(-1, 1))
    idx = torch.arange(C, device=prob.device).view(1, -1)
    r = ((prob > pt) | ((prob == pt) & (idx < t.view(-1, 1)))).sum(1)
    return torch.where(valid, r, torch.full_like(r, C))


def center_normalize(x):
    """:690-695 in float64."""
    x = x.double()
    return F.normalize(x - x.mean(dim=0, keepdim=True), p=2, dim=1)


def retrieval_sim(test_feature, train_feature):
    """:689-698 in float64: (test normalised, train normalised, sim)."""
    q, k = center_normalize(test_feature), center_normalize(train_feature)
    return q, k, q @ k.t()


def retrieval_topk(sim, test_label, train_label, ks=(1, 5, 10, 20, 50)):
    """:702-705, the reference's formula: [len(ks), Nq] bool."""
    out = []
    for k in ks:
        idx = torch.topk(sim, k, dim=1).indices
        out.append(torch.any(train_label[idx] == test_label.unsqueeze(1), dim=1))
    return torch.stack(out)


def retrieval_rank(sim, test_label, train_label):
    """Rank of each query's best same-label train item in the order (sim descending, index ascending); Nk when there
    is none.  Also returns the rank-deciding gap: the smallest |sim[j] - sim[best]| over the other items j (a query
    whose gap is below the sim error may legitimately rank differently)."""
    Nq, Nk = sim.shape
    same = train_label.view(1, -1) == test_label.view(-1, 1)
    masked = torch.where(same, sim, torch.full_like(sim, -float("inf")))
    best = masked.argmax(1)            # first maximal index: ties to the lower index
    has = same.any(1)
    sb = sim.gather(1, best.view(-1, 1))
    idx = torch.arange(Nk, device=sim.device).view(1, -1)
    rank = ((sim > sb) | ((sim == sb) & (idx < best.view(-1, 1)))).sum(1)
    rank = torch.where(has, rank, torch.full_like(rank, Nk))
    d = (sim - sb).abs()
    d[torch.arange(Nq), best] = float("inf")
    # every other item counts, same-label ones included: a near-tie there can change which item is the best
    return rank, d.min(1).values


def hits_from_rank(rank, n_items, ks=(1, 5, 10, 20, 50)):
    """[len(ks), Nq] bool: rank < k, never for rank == n_items (no same-label item), whatever k."""
    return torch.stack([(rank < k) & (rank < n_items) for k in ks])
