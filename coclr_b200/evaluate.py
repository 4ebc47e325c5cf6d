"""Video-level evaluation of an encoder on the engine: what the reference's eval/main_classifier.py --test computes.

    scores = evaluate(model, videos, seq_len=32, batch_size=32)        # model: model.classifier.LinearClassifier
    scores.feature [Nv, D]   per-video mean of the clips' feat3d          (test_retrieval: feature.mean(0), :637)
    scores.prob    [Nv, C]   per-video mean of softmax(logit) over clips,  (test_10crop: softmax(logit).mean(0), :488,
                             averaged over the views given so far          summarize_probability :533)
    scores.top1, scores.top5 accuracies over the videos (rank of the target class in scores.prob < 1, < 5)
    sim, rank, acc = retrieval(test_feature, test_label, train_feature, train_label)          (:686-706)

and the two-stream merge of the reference's eval/merge_2stream_prob.py:
    fused, (acc1, acc2, acc_fused) = merge_probabilities(prob1, prob2, target)                 (merge_prob :60-101)
    idx = align_two_stream(train_vname1, test_vname1, train_vname2, test_vname2)               (merge_sim :118-170)
    sim, rank, acc = two_stream_retrieval(test1, train1, test2, train2, test_label, train_label)   (:178-196)

`videos` is any iterable of (video, label, vname) with video a float [3, T_total, H, W] tensor in [0, 1] (the
reference's ToTensor output, CPU or CUDA).  A video gives T_total // seq_len consecutive, non-overlapping clips (the
reference's `tr` view, :444-448); frames left over at the end are dropped.

Clips of consecutive videos are packed into passes of exactly `batch_size` clips (`pack_passes`), so one engine plan and
one CUDA graph serve every pass whatever the video lengths: the clips of a pass are staged along T into one device
buffer [3, batch_size * seq_len, H, W], the pass reads them through a strided [batch_size, 3, seq_len, H, W] view of it
with a `batch_index`, and the last pass repeats its first clip as padding (those outputs are discarded).  The model
runs in eval mode, where every clip's result is independent of the others in its pass.  ImageNet normalisation is the
engine's `norm` (applied while packing the input), as in the reference's GPU-side T.Normalize.

The per-video sums, means, ranks and the retrieval arithmetic are the kernels of csrc/evaluate.cu: fixed summation
order, no float atomics, bit-identical from run to run.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np
import torch

from coclr_b200 import lib as L

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
RETRIEVAL_KS = (1, 5, 10, 20, 50)


def clips_of(video, seq_len, num_seq=1):
    """Number of clips a [3, T_total, H, W] video gives (:446): T_total // (seq_len * num_seq)."""
    if num_seq != 1:
        raise ValueError("num_seq must be 1 for video-level testing (the reference squeezes that dimension), got %d"
                         % num_seq)
    if video.dim() != 4 or video.shape[0] != 3:
        raise ValueError("a video is [3, T_total, H, W], got %s" % (list(video.shape),))
    n = video.shape[1] // seq_len
    if n < 1:
        raise ValueError("video of %d frames is shorter than one clip of %d frames" % (video.shape[1], seq_len))
    return n


def pack_passes(clip_counts, batch):
    """Packs the clips of consecutive videos into passes of exactly `batch` clips.

    clip_counts: iterable of clips per video (consumed lazily).  Yields one (segments, slot) per pass:
      segments: [(video, first_clip, n_clips, first_slot)] -- clips first_clip .. first_clip + n_clips - 1 of `video`
                go to pass slots first_slot .. first_slot + n_clips - 1;
      slot:     [batch] list, the video of each pass slot, -1 for padding (only in the last pass).
    Clips keep their order: a video that straddles a pass boundary continues at slot 0 of the next pass."""
    segments, slot = [], []
    for v, n in enumerate(clip_counts):
        c = 0
        while c < n:
            k = min(n - c, batch - len(slot))
            segments.append((v, c, k, len(slot)))
            slot += [v] * k
            c += k
            if len(slot) == batch:
                yield segments, slot
                segments, slot = [], []
    if slot:
        yield segments, slot + [-1] * (batch - len(slot))


@dataclass
class VideoScores:
    """Per-video results of `evaluate` (device tensors, videos in iteration order)."""
    feature: torch.Tensor       # [Nv, D]  mean feat3d over the video's clips (this view)
    view_prob: torch.Tensor     # [Nv, C]  mean softmax(logit) over the video's clips (this view)
    prob: torch.Tensor          # [Nv, C]  mean of view_prob over the views so far
    label: torch.Tensor         # [Nv] int64
    vname: list
    rank: torch.Tensor          # [Nv] int32: classes ranked above the target in prob (ties to the lower index);
    #                             C for a label outside the head's classes [0, C), which scores as a miss
    top1: float
    top5: float
    n_views: int = 1
    views_sum: torch.Tensor = field(default=None, repr=False)


def _int_tensor(values, device, dtype):
    """Small host list -> device tensor without a host synchronisation (pinned staging, async copy)."""
    return torch.tensor(values, dtype=dtype).pin_memory().to(device, non_blocking=True)


class _Accumulators:
    """Per-video sums, grown by doubling as videos arrive."""

    def __init__(self, C, D, device):
        self.C, self.D, self.device, self.cap = C, D, device, 0
        self._grow(64)

    def _grow(self, cap):
        f32 = dict(dtype=torch.float32, device=self.device)
        new = (torch.zeros(cap, self.C, **f32), torch.zeros(cap, self.D, **f32),
               torch.zeros(cap, dtype=torch.int32, device=self.device))
        if self.cap:
            for n, o in zip(new, (self.prob_sum, self.feat_sum, self.count)):
                n[:self.cap].copy_(o)
        self.prob_sum, self.feat_sum, self.count = new
        self.cap = cap

    def ensure(self, nv):
        if nv > self.cap:
            self._grow(max(nv, 2 * self.cap))


@torch.no_grad()
def evaluate(model, videos, seq_len, batch_size, num_seq=1, normalize=True, previous=None):
    """Per-video features and probabilities of `model` (a LinearClassifier, put in eval mode) over `videos`.

    normalize: apply the ImageNet mean / std (the reference's T.Normalize) while packing; False feeds the values as
    they are.  previous: the VideoScores of the earlier views of the same videos (multi-crop testing); the returned
    prob is then the mean of the per-view means over all views so far, in view order.  Labels are any integers: one
    outside the head's classes [0, C) (e.g. retrieval labels of a dataset with more classes than the head) is kept in
    `label` and counts as a miss in top1 / top5, as the reference's calc_topk_accuracy scores it."""
    if num_seq != 1:
        raise ValueError("num_seq must be 1 for video-level testing (the reference squeezes that dimension), got %d"
                         % num_seq)
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    model.eval()
    lib = L.load()
    head = model.final_fc[-1]
    device = head.weight.device
    if device.type != "cuda":
        raise L.CoclrError("coclr_b200 classifiers run on CUDA (sm_90a) only; there is no CPU path")
    Cn, D = head.out_features, model.param['feature_size']
    norm = None
    if normalize:
        norm = (torch.tensor(IMAGENET_MEAN, dtype=torch.float32, device=device),
                torch.tensor(IMAGENET_STD, dtype=torch.float32, device=device))
    acc = _Accumulators(Cn, D, device)
    labels, vnames, held = [], [], {}
    shape = {}

    def counts():
        for v, (video, label, vname) in enumerate(videos):
            n = clips_of(video, seq_len, num_seq)
            hw = tuple(video.shape[2:])
            if shape.setdefault("hw", hw) != hw:
                raise ValueError("every video of one evaluation needs the same H, W: %s then %s" % (shape["hw"], hw))
            labels.append(int(label))
            vnames.append(vname)
            held[v] = video
            acc.ensure(v + 1)
            yield n

    buf = view = full_index = None
    for segments, slot in pack_passes(counts(), batch_size):
        if buf is None:
            H, W = shape["hw"]
            buf = torch.empty(3, batch_size * seq_len, H, W, dtype=torch.float32, device=device)
            thw = seq_len * H * W
            view = buf.as_strided((batch_size, 3, seq_len, H, W), (thw, batch_size * thw, H * W, W, 1))
            full_index = torch.arange(batch_size, dtype=torch.long, device=device)
        for v, c, k, s in segments:
            video = held[v]
            buf[:, s * seq_len:(s + k) * seq_len].copy_(video[:, c * seq_len:(c + k) * seq_len], non_blocking=True)
            if c + k == video.shape[1] // seq_len:
                del held[v]
        valid = sum(1 for s in slot if s >= 0)
        index = full_index if valid == batch_size else _int_tensor(
            [b if b < valid else 0 for b in range(batch_size)], device, torch.long)
        logits, feat = model.infer(view, batch_index=index, batch=batch_size, norm=norm)
        L.check(lib.coclr_video_accumulate(L.dptr(logits), L.dptr(feat), L.dptr(_int_tensor(slot, device, torch.int32)),
                                           L.dptr(acc.prob_sum), L.dptr(acc.feat_sum), L.dptr(acc.count), batch_size,
                                           Cn, D, L.stream_ptr()), "coclr_video_accumulate")
    Nv = len(labels)
    if Nv == 0:
        raise ValueError("no videos to evaluate")
    if previous is not None:
        if previous.vname != vnames:
            raise ValueError("previous views were computed over different videos")
        views_sum, n_views = previous.views_sum.clone(), previous.n_views + 1
    else:
        views_sum, n_views = torch.zeros(Nv, Cn, dtype=torch.float32, device=device), 1
    f32 = dict(dtype=torch.float32, device=device)
    out = VideoScores(feature=torch.empty(Nv, D, **f32), view_prob=torch.empty(Nv, Cn, **f32),
                      prob=torch.empty(Nv, Cn, **f32), label=_int_tensor(labels, device, torch.long), vname=vnames,
                      rank=torch.empty(Nv, dtype=torch.int32, device=device), top1=0.0, top5=0.0, n_views=n_views,
                      views_sum=views_sum)
    hits = torch.zeros(2, dtype=torch.int32, device=device)
    a = L.VideoFinalize(prob_sum=L.dptr(acc.prob_sum), feat_sum=L.dptr(acc.feat_sum), count=L.dptr(acc.count), Nv=Nv,
                        C=Cn, D=D, n_views=n_views, feat_mean=L.dptr(out.feature), prob_mean=L.dptr(out.view_prob),
                        views_sum=L.dptr(views_sum), prob=L.dptr(out.prob), target=L.dptr(out.label),
                        rank=L.dptr(out.rank), hits=L.dptr(hits))
    L.check(lib.coclr_video_finalize(C.byref(a), L.stream_ptr()), "coclr_video_finalize")
    h = hits.tolist()
    out.top1, out.top5 = h[0] / Nv, h[1] / Nv
    return out


def center_normalize(x):
    """F.normalize(x - x.mean(0), dim=1) of a [N, D] fp32 CUDA tensor (:690-695)."""
    x = x.contiguous()
    assert x.dim() == 2 and x.dtype == torch.float32
    y, mean = torch.empty_like(x), torch.empty(x.shape[1], dtype=torch.float32, device=x.device)
    L.check(L.load().coclr_center_normalize(L.dptr(x), L.dptr(y), L.dptr(mean), x.shape[0], x.shape[1],
                                            L.stream_ptr()), "coclr_center_normalize")
    return y


def _gemm_operand(x, D4):
    """x [N, D] fp32 as the similarity kernel reads it: contiguous, 16-byte aligned rows of D4 (a multiple of 4)
    floats.  An input that already is one is used as is; otherwise it is copied, zero-padded to D4 columns (the zero
    products leave every dot product's bits unchanged)."""
    x = x.float().contiguous()
    if x.shape[1] == D4 and x.data_ptr() % 16 == 0:
        return x
    out = torch.zeros(x.shape[0], D4, dtype=torch.float32, device=x.device)
    out[:, :x.shape[1]].copy_(x)
    return out


def similarity(q, k):
    """q [Nq, D] . k [Nk, D]^T on fp32 FFMA, any D (rows are zero-padded to a multiple of 4 where needed)."""
    assert q.dim() == 2 and k.dim() == 2 and q.shape[1] == k.shape[1], (q.shape, k.shape)
    D4 = (q.shape[1] + 3) // 4 * 4
    q, k = _gemm_operand(q, D4), _gemm_operand(k, D4)
    sim = torch.empty(q.shape[0], k.shape[0], dtype=torch.float32, device=q.device)
    L.check(L.load().coclr_sim_fp32(L.dptr(q), L.dptr(k), L.dptr(sim), q.shape[0], k.shape[0], D4,
                                    L.stream_ptr()), "coclr_sim_fp32")
    return sim


def retrieval_rank(sim, test_label, train_label, ks=RETRIEVAL_KS):
    """Per query, the position of its best same-label train item in the order (sim descending, index ascending), Nk
    when there is none; and, for each k, the number of queries with rank < k that have a same-label item (a k above
    Nk, where the reference's topk would raise, counts the queries that have one)."""
    Nq, Nk = sim.shape
    assert len(ks) <= 8
    rank = torch.empty(Nq, dtype=torch.int32, device=sim.device)
    hits = torch.zeros(max(len(ks), 1), dtype=torch.int32, device=sim.device)
    karr = (C.c_int * max(len(ks), 1))(*ks)
    ql = test_label.to(sim.device, torch.long).contiguous()
    kl = train_label.to(sim.device, torch.long).contiguous()
    assert ql.numel() == Nq and kl.numel() == Nk
    L.check(L.load().coclr_retrieval_rank(L.dptr(sim.contiguous()), L.dptr(ql), L.dptr(kl), Nq, Nk, karr, len(ks),
                                          L.dptr(rank), L.dptr(hits), L.stream_ptr()), "coclr_retrieval_rank")
    return rank, hits[:len(ks)]


def retrieval(test_feature, test_label, train_feature, train_label, ks=RETRIEVAL_KS):
    """Nearest-neighbour retrieval of the reference (:686-706): centre each set by its own mean, l2-normalise,
    sim = test . train^T, and a query hits at k when a train item of its label is among its k most similar.
    Returns (sim [Nq, Nk], rank [Nq] int32, [acc for each k]); acc is the fraction of queries that hit."""
    sim = similarity(center_normalize(test_feature.float()), center_normalize(train_feature.float()))
    rank, hits = retrieval_rank(sim, test_label, train_label, ks)
    Nq = sim.shape[0]
    acc = [h / Nq for h in hits.tolist()]
    return sim, rank, acc


def similarity2(q1, k1, q2, k2):
    """q1 . k1^T + q2 . k2^T on fp32 FFMA (coclr_sim2_fp32): each stream has its own width D1, D2 (any values; rows
    are zero-padded to a multiple of 4 where needed).  Bit-identical to similarity(q1, k1) + similarity(q2, k2)."""
    assert q1.dim() == k1.dim() == q2.dim() == k2.dim() == 2, (q1.shape, k1.shape, q2.shape, k2.shape)
    assert q1.shape[1] == k1.shape[1] and q2.shape[1] == k2.shape[1], (q1.shape, k1.shape, q2.shape, k2.shape)
    assert q1.shape[0] == q2.shape[0] and k1.shape[0] == k2.shape[0], (q1.shape, k1.shape, q2.shape, k2.shape)
    D1, D2 = (q1.shape[1] + 3) // 4 * 4, (q2.shape[1] + 3) // 4 * 4
    q1, k1, q2, k2 = _gemm_operand(q1, D1), _gemm_operand(k1, D1), _gemm_operand(q2, D2), _gemm_operand(k2, D2)
    sim = torch.empty(q1.shape[0], k1.shape[0], dtype=torch.float32, device=q1.device)
    L.check(L.load().coclr_sim2_fp32(L.dptr(q1), L.dptr(k1), D1, L.dptr(q2), L.dptr(k2), D2, L.dptr(sim),
                                     q1.shape[0], k1.shape[0], L.stream_ptr()), "coclr_sim2_fp32")
    return sim


def two_stream_retrieval(test1, train1, test2, train2, test_label, train_label, ks=RETRIEVAL_KS):
    """Two-stream nearest-neighbour retrieval of the reference (merge_sim :172-196): centre each of the four sets by
    its own mean and l2-normalise it, sim = test1 . train1^T + test2 . train2^T, and a query hits at k when a train
    item of its label is among its k most similar.  The streams must already be aligned row for row
    (align_two_stream).  Returns (sim [Nq, Nk], rank [Nq] int32, [acc for each k]) as retrieval() does."""
    if test1.shape[0] != test2.shape[0] or train1.shape[0] != train2.shape[0]:
        raise ValueError("the two streams have %d / %d test and %d / %d train rows; align them first"
                         % (test1.shape[0], test2.shape[0], train1.shape[0], train2.shape[0]))
    q1, k1 = center_normalize(test1.float()), center_normalize(train1.float())
    q2, k2 = center_normalize(test2.float()), center_normalize(train2.float())
    sim = similarity2(q1, k1, q2, k2)
    rank, hits = retrieval_rank(sim, test_label, train_label, ks)
    Nq = sim.shape[0]
    acc = [h / Nq for h in hits.tolist()]
    return sim, rank, acc


def merge_probabilities(prob1, prob2, target):
    """Probability fusion of the reference (merge_prob :60-101) on the device (coclr_prob_merge): fused = (prob1 +
    prob2) / 2 in float64 per video, and the accuracies of argmax prob1, argmax prob2 and argmax fused against target
    (ties to the lowest index, as np.argmax; a target outside [0, C) is a miss).  prob1, prob2: [Nv, C] float64 CUDA
    tensors (the reference reads the JSON floats as float64); target: [Nv] integers.
    Returns (fused [Nv, C] float64, (acc1, acc2, acc_fused))."""
    if prob1.dim() != 2 or prob1.shape != prob2.shape or prob1.shape[0] == 0 or prob1.shape[1] == 0:
        raise ValueError("prob1 and prob2 must be two [Nv, C] matrices of the same non-empty shape, got %s and %s"
                         % (list(prob1.shape), list(prob2.shape)))
    if prob1.device.type != "cuda":
        raise L.CoclrError("coclr_b200 runs on CUDA (sm_90a) only; there is no CPU path")
    Nv, Cn = prob1.shape
    p1 = prob1.to(torch.float64).contiguous()
    p2 = prob2.to(p1.device, torch.float64).contiguous()
    t = torch.as_tensor(target).to(p1.device, torch.long).contiguous()
    if t.numel() != Nv:
        raise ValueError("%d targets for %d videos" % (t.numel(), Nv))
    fused = torch.empty_like(p1)
    hits = torch.zeros(3, dtype=torch.int32, device=p1.device)
    L.check(L.load().coclr_prob_merge(L.dptr(p1), L.dptr(p2), L.dptr(t), Nv, Cn, L.dptr(fused), L.dptr(hits),
                                      L.stream_ptr()), "coclr_prob_merge")
    return fused, tuple(h / Nv for h in hits.tolist())


def _vname_array(vnames):
    """The reference's np.squeeze(np.array(vnames)) of a pickled vname list ([[v], ...] as --retrieval writes it, or
    [v, ...]), kept one-dimensional."""
    return np.atleast_1d(np.squeeze(np.array(vnames)))


def align_two_stream(train_vname1, test_vname1, train_vname2, test_vname2):
    """The name alignment of the reference's merge_sim (:118-170), on the host: each of the four vname lists is
    sorted (np.argsort); then, when stream 1 has fewer train videos than stream 2, stream 2's train and test lists
    keep only the names stream 1 has (np.isin), and after that, when stream 1 has more train videos than stream 2,
    stream 1's lists keep only the names stream 2 has.  Both steps run when the first one leaves stream 2 shorter.
    Returns int64 index tensors (train1, test1, train2, test2): row i of the aligned stream s is row idx[i] of its
    input, and stream 1's labels follow stream 1's indices.  Raises ValueError naming the first position where the
    aligned names differ (the reference asserts)."""
    v1tr, v1te = _vname_array(train_vname1), _vname_array(test_vname1)
    v2tr, v2te = _vname_array(train_vname2), _vname_array(test_vname2)
    i1tr, i1te, i2tr, i2te = (np.argsort(v) for v in (v1tr, v1te, v2tr, v2te))
    v1tr, v1te, v2tr, v2te = v1tr[i1tr], v1te[i1te], v2tr[i2tr], v2te[i2te]
    if len(v1tr) < len(v2tr):
        keep_tr, keep_te = np.isin(v2tr, v1tr), np.isin(v2te, v1te)
        v2tr, i2tr, v2te, i2te = v2tr[keep_tr], i2tr[keep_tr], v2te[keep_te], i2te[keep_te]
    if len(v1tr) > len(v2tr):
        keep_tr, keep_te = np.isin(v1tr, v2tr), np.isin(v1te, v2te)
        v1tr, i1tr, v1te, i1te = v1tr[keep_tr], i1tr[keep_tr], v1te[keep_te], i1te[keep_te]
    for split, a, b in (("train", v1tr, v2tr), ("test", v1te, v2te)):
        if len(a) != len(b):
            raise ValueError("after alignment stream 1 has %d %s videos and stream 2 has %d"
                             % (len(a), split, len(b)))
        bad = np.flatnonzero(a != b)
        if len(bad):
            i = int(bad[0])
            raise ValueError("%s video %d differs after alignment: %r in stream 1, %r in stream 2"
                             % (split, i, str(a[i]), str(b[i])))
    return tuple(torch.from_numpy(np.asarray(i, dtype=np.int64)) for i in (i1tr, i1te, i2tr, i2te))
