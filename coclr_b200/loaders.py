"""GPU batch loaders over the reference's LMDB datasets (coclr_b200.datasets): each batch's sampled frames are read
from the map, deduplicated, decoded once on the GPU (coclr_b200.jpeg, `slots=`) and augmented there
(coclr_b200.augment / clf_augment).

Host work of batch i + 1 -- LMDB reads, frame sampling, the header parse, the dedupe and the augmentation plan -- runs
on a background thread while batch i trains (a queue of depth 2); the decode and the augmentation are enqueued on the
consumer's stream.  Closing the loader, or dropping its iterator, stops and joins the thread.

Random draws follow the reference's num_workers=0 loader: item i's frame sampler, then item i's transform, then item
i + 1, from the loader's own random.Random / np.random.RandomState / torch.Generator.  Parity with the reference's
multi-worker streams is not a goal.
"""
import queue
import random
import threading

import numpy as np
import torch

from .jpeg import JpegDecoder, JpegFrameError, parse

_END = object()


class Prefetch:
    """Runs `produce()` (a generator of host-side batches) on a daemon thread, at most `depth` batches ahead."""

    def __init__(self, produce, depth=2):
        self.q = queue.Queue(depth)
        self.stop = threading.Event()
        self.thread = threading.Thread(target=self._run, args=(produce,), daemon=True, name="coclr-lmdb-prefetch")
        self.thread.start()

    def _put(self, item):
        while not self.stop.is_set():
            try:
                self.q.put(item, timeout=0.05)
                return True
            except queue.Full:
                continue
        return False

    def _run(self, produce):
        try:
            for item in produce():
                if not self._put(item):
                    return
            self._put(_END)
        except BaseException as e:                   # handed to the consumer, raised there
            self._put(e)

    def __iter__(self):
        try:
            while True:
                item = self.q.get()
                if item is _END:
                    return
                if isinstance(item, BaseException):
                    raise item
                yield item
        finally:
            self.close()

    def close(self):
        self.stop.set()
        self.thread.join()


def dedupe(refs):
    """refs: [(stream, key, frame)] of every output frame.  Returns (distinct refs in first-use order, slots), where
    slots[j] lists the output frames distinct frame j fills (every output frame exactly once)."""
    first, slots = {}, []
    for o, r in enumerate(refs):
        j = first.setdefault(r, len(first))
        if j == len(slots):
            slots.append([])
        slots[j].append(o)
    return list(first), slots


class _Batches:
    """Common host path: read, sample, dedupe, parse and plan one list of dataset items."""

    def __init__(self, dataset, device, seed):
        self.ds, self.device = dataset, device
        self.py, self.np = random.Random(seed), np.random.RandomState(seed)
        self.tg = torch.Generator().manual_seed(seed)
        self.ds.rng = self.np
        self.dec = JpegDecoder()
        self._live = []

    def _host(self, items, plan_one):
        """items: dataset indices.  plan_one(size, n_frames) draws the item's transform from the size of its first
        sampled frame.  Returns the parsed distinct frames, their slots, the per-item plan samples and the per-item
        frame counts.  ValueError names the database, video and frame of a frame that is missing or cannot be
        decoded, and the video whose frames differ in size from the one its transform was drawn for."""
        refs, samples, counts, cache = [], [], [], {}
        for i in items:
            fi = self.ds.sample(i)
            r = self.ds.refs(i, fi)
            vname = self.ds.video_subset[i][3]
            for s, key in dict.fromkeys((x[0], x[1]) for x in r):
                if (s, key) not in cache:                  # each video read once per batch
                    cache[s, key] = (self.ds.dbs[s].video(vname), vname)
            size = self._parse(cache, [r[0]]).sizes[0]
            samples.append(plan_one(size, len(r)))
            refs += r
            counts.append(len(r))
        distinct, slots = dedupe(refs)
        batch = self._parse(cache, distinct)
        sizes = batch.output_sizes(slots)
        o = 0
        for i, sp, n in zip(items, samples, counts):        # the transform crops every frame by the first one's size
            if any(hw != tuple(sp.size) for hw in sizes[o:o + n]):
                raise ValueError("video %s: its sampled frames differ in size (%s)" % (
                    self.ds.video_subset[i][3], sorted(set(sizes[o:o + n]))))
            o += n
        return batch, slots, samples, counts

    def _parse(self, cache, refs):
        """parse() of the frames refs name, with the database, video and frame in any error."""
        jpegs = []
        for s, key, f in refs:
            video, vname = cache[s, key]
            if not 0 <= f < len(video):
                raise ValueError("%s: video %s has %d frames, frame %d was sampled" % (
                    self.ds.dbs[s].path, vname, len(video), f))
            jpegs.append(video[f])
        try:
            return parse(jpegs)
        except JpegFrameError as e:
            s, key, f = refs[e.frame]
            raise ValueError("%s: video %s frame %d: %s" % (self.ds.dbs[s].path, cache[s, key][1], f,
                                                             e.reason)) from None

    def _decode(self, batch, slots):
        return self.dec(batch, slots=slots)

    def _iterate(self, produce, finish):
        pf = Prefetch(produce)
        self._live.append(pf)
        try:
            for host in pf:
                yield finish(host)
        finally:
            pf.close()
            self._live.remove(pf)

    def close(self):
        """Stop and join every look-ahead thread of this loader."""
        for pf in list(self._live):
            pf.close()


class PretrainBatches(_Batches):
    """Pre-training batches of a *_2CLIP dataset: what main_nce.py / main_coclr.py's synthetic loaders yield -- the
    PretrainAugment output and, per sample, the label (main_nce) or the source id (main_coclr, two_stream=True).

    Order: the reference's DistributedSampler(shuffle=True), randperm(n) of a generator seeded 0 + epoch, padded to a
    multiple of the world size and strided by rank, then batches of batch_size with drop_last.  The reference's
    FastDataLoader builds its sampler iterator once and never calls set_epoch, so it visits the same order every
    epoch; so does this loader."""

    def __init__(self, dataset, batch_size, seq_len, img_dim, device, seed, rank=0, world_size=1, two_stream=False):
        from .augment import AugmentPlan, PretrainAugment
        super().__init__(dataset, device, seed)
        self.B, self.two_stream = batch_size, two_stream
        self.aug = PretrainAugment(seq_len, img_dim, two_stream=two_stream)
        self._Plan = AugmentPlan
        n = len(dataset)
        order = torch.randperm(n, generator=torch.Generator().manual_seed(0)).tolist()
        per = -(-n // world_size)
        order += order[:per * world_size - n]
        self.order = order[rank:per * world_size:world_size]

    def __len__(self):
        return len(self.order) // self.B

    def _targets(self, items):
        if self.two_stream:
            return [self.ds.source_id(i) for i in items]
        return [self.ds.label(i) for i in items]

    def _produce(self):
        for b in range(len(self)):
            items = self.order[b * self.B:(b + 1) * self.B]
            batch, slots, samples, _ = self._host(
                items, lambda hw, n: self.aug.plan([hw], self.py, self.np, self.tg).samples[0])
            yield batch, slots, self._Plan(self.aug, samples), self._targets(items)

    def _finish(self, host):
        batch, slots, plan, targets = host
        frames = self._decode(batch, slots)
        frames = frames.view(self.B, self.aug.frames, *frames.shape[1:])
        y = torch.tensor(targets, dtype=torch.int64).to(self.device, non_blocking=True)
        return self.aug(frames, plan), y

    def __iter__(self):
        return self._iterate(self._produce, self._finish)


class ClassifierBatches(_Batches):
    """Fine-tuning batches (eval/main_classifier.py, mode 'train' or 'val') of UCF101LMDB / HMDB51LMDB / their flow
    classes: ClassifierAugment output and labels.  The order is a seeded shuffle with drop_last (the reference's
    RandomSampler order is not reproduced); the train batch's flip is drawn from `random` as the synthetic loader
    draws it."""

    def __init__(self, dataset, batch_size, seq_len, img_dim, device, seed, mode, num_seq=1):
        from .clf_augment import ClassifierAugment, ClfAugmentPlan
        super().__init__(dataset, device, seed)
        self.B, self.mode = batch_size, mode
        self.aug = ClassifierAugment(mode, seq_len, img_dim, num_seq=num_seq)
        self._Plan = ClfAugmentPlan
        self.shuffle = torch.Generator().manual_seed(seed)

    def __len__(self):
        return len(self.ds) // self.B

    def order(self):
        """This epoch's item order (a new seeded shuffle per epoch)."""
        return torch.randperm(len(self.ds), generator=self.shuffle).tolist()

    def _produce(self):
        order = self.order()
        for b in range(len(self)):
            items = order[b * self.B:(b + 1) * self.B]
            batch, slots, samples, _ = self._host(items, lambda hw, n: self.aug.plan([hw], self.py).samples[0])
            yield batch, slots, self._Plan(self.aug, samples), [self.ds.label(i) for i in items]

    def _finish(self, host):
        batch, slots, plan, targets = host
        frames = self._decode(batch, slots)
        frames = frames.view(self.B, self.aug.frames, *frames.shape[1:])
        if self.mode == 'train':
            flip = random.random() < 0.5                       # transform_train_cuda's T.RandomHorizontalFlip
            for sp in plan.samples:
                sp.flip = flip
        y = torch.tensor(targets, dtype=torch.int64).to(self.device, non_blocking=True)
        return self.aug(frames, plan), y

    def __iter__(self):
        return self._iterate(self._produce, self._finish)


class TestVideos(_Batches):
    """Test and retrieval videos for coclr_b200.evaluate: (video [3, T, D, D], label, vname) with vname the CSV's
    path column (the reference's return_path), `chunk` videos per decode and augmentation launch.  mode 'test' on
    the test split gives the half-overlap windows; retrieval's train split uses mode 'train' (one random clip)."""

    def __init__(self, dataset, seq_len, img_dim, device, seed, view=(5, 0), mode='test', chunk=8, num_seq=1):
        from .clf_augment import ClassifierAugment, ClfAugmentPlan
        super().__init__(dataset, device, seed)
        self.aug = ClassifierAugment(mode, seq_len, img_dim, num_seq=num_seq, view=view)
        self._Plan = ClfAugmentPlan
        self.chunk = chunk

    def __len__(self):
        return len(self.ds)

    def _produce(self):
        n = len(self.ds)
        for i0 in range(0, n, self.chunk):
            items = list(range(i0, min(i0 + self.chunk, n)))
            batch, slots, samples, counts = self._host(
                items, lambda hw, k: self.aug.plan([hw], self.py, lengths=[k]).samples[0])
            info = [(self.ds.label(i), self.ds.video_subset[i][0]) for i in items]
            yield batch, slots, self._Plan(self.aug, samples), info

    def _finish(self, host):
        batch, slots, plan, info = host
        videos = self.aug(self._decode(batch, slots), plan)
        return [(v, label, vname) for v, (label, vname) in zip(videos, info)]

    def __iter__(self):
        for chunk in self._iterate(self._produce, self._finish):
            yield from chunk
