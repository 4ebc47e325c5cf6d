"""Fine-tuning and test augmentation on the GPU: the transforms of the reference's eval/main_classifier.py
(utils/augmentation.py under PIL) as one CUDA kernel (csrc/augment_clf.cu, `coclr_augment_clf`), bit-identical to the
reference's DataLoader tensor for the same random decisions.

    aug = ClassifierAugment('train', seq_len=32, img_dim=128)
    plan = aug.plan(sizes, batch_flip=random.random() < 0.5)   # host only: every draw, in the reference's order
    x = aug(frames, plan)                                      # frames: uint8 [B, T, Hmax, Wmax, 3] on the GPU
    model.set_input_transform(); model(x)                      # x: [B, 3, T, img_dim, img_dim] in [0, 1]

    aug = ClassifierAugment('test', seq_len=32, img_dim=128, view=(aug_idx, flip_idx))
    videos = aug(frames, aug.plan(sizes, lengths=[T0, T1, ...]))   # frames: uint8 [sum(T), Hmax, Wmax, 3]
                                                                    # -> [[3, T0, D, D], [3, T1, D, D], ...]

Recipes (one decision per sample, `consistent=True` throughout):
  train      RandomSizedCrop(224, bottom_area=.2) -> Scale(img_dim) -> ColorJitter(.4, .4, .4, .1, p=.3) -> ToTensor,
             then the batch's T.RandomHorizontalFlip (one draw per batch, in the main process: `batch_flip`)
  val        RandomSizedCrop(224, bottom_area=.2) -> Scale(img_dim) -> ToTensor
  test       RandomHorizontalFlip(command='left' | 'right') -> FiveCrop(224, where=aug_idx) -> Scale((D, D)) ->
             ColorJitter(.2, .2, .2, .1, p=.3) -> ToTensor            (test_10crop; view = (aug_idx, flip_idx))
  retrieval  CenterCrop(224) -> Scale((D, D)) -> ColorJitter(.2, .2, .2, .1, p=.3) -> ToTensor   (test_retrieval)

Only Python's `random` is drawn from (np.random and torch's generator are left alone, as in the reference).
RandomSizedCrop(consistent=True) makes up to 10 attempts; after 10 misses it falls back to Scale(224) (shorter side to
224) and CenterCrop(224), which is one bicubic resize of the whole frame read through a 224 x 224 window.  FiveCrop and
CenterCrop need frames of at least 224 x 224: smaller ones raise ValueError (the reference's FiveCrop raises, and its
CenterCrop would zero-pad).

Train and val run two bicubic resizes, crop -> 224 x 224 and 224 -> img_dim, with a uint8 image in between, as Pillow
does; the test views and retrieval, and img_dim == 224, run one.
"""
import ctypes as C
import math
import random as _random
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch

from .augment import JITTER_OPS, SMEM_LIMIT, hue_shift_byte, resize_taps

CROP = 224                                             # the recipes' crop side
MODES = ("train", "val", "test", "retrieval")
SAMPLE_INTS = 16                                       # int32 words per sample record (coclr_augment_clf_sample_t)
FRAME_LONGS = 4                                        # int64 words per frame record (coclr_augment_clf_frame_t)


def _jitter_ranges(b, c, s, h):
    """ColorJitter._check_input of the reference: [1 - v, 1 + v] (clipped at 0) and [-h, h]."""
    return tuple([max(1 - v, 0), 1 + v] for v in (b, c, s)) + ([0 - h, 0 + h],)


JITTER = {"train": _jitter_ranges(0.4, 0.4, 0.4, 0.1), "test": _jitter_ranges(0.2, 0.2, 0.2, 0.1),
          "retrieval": _jitter_ranges(0.2, 0.2, 0.2, 0.1)}
JITTER_P = 0.3


@dataclass
class ClfSamplePlan:
    """Decisions for one sample (a clip of train / val, a whole video of test / retrieval).

    crop      (x1, y1, w, h): the box, in the (flipped, for src_flip) frame, that the first resize takes to 224
              (train / val) or img_dim (test / retrieval); None with a fallback
    fallback  (scaled_h, scaled_w, y1, x1): RandomSizedCrop's fallback, Scale(224) of the whole frame to
              scaled_h x scaled_w, then CenterCrop(224) at (y1, x1) of it; None when a box fitted
    attempts  RandomSizedCrop attempts drawn (train / val): 1-10, or 10 with a fallback
    jitter    [(op, factor)] in application order, or None; hue_shift the byte added to PIL's H when 'hue' is in it
    src_flip  the test view's flip of the source before the crop
    flip      the train batch's flip of the augmented tensor
    """
    size: Tuple[int, int]
    frames: int
    crop: Optional[Tuple[int, int, int, int]] = None
    fallback: Optional[Tuple[int, int, int, int]] = None
    attempts: int = 0
    jitter: Optional[List[Tuple[str, float]]] = None
    hue_shift: Optional[int] = None
    src_flip: bool = False
    flip: bool = False


class ClfAugmentPlan:
    """Per-sample decisions plus the device tables they compile to (built lazily, once per device)."""

    def __init__(self, aug, samples):
        self.aug = aug
        self.samples = samples
        self._dev = {}

    @property
    def sizes(self):
        return [s.size for s in self.samples]

    @property
    def lengths(self):
        return [s.frames for s in self.samples]

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]

    def tables(self):
        return self.aug._tables(self)

    def to(self, device):
        """Device copy of the tables (cached: a captured graph replays without host work)."""
        device = torch.device(device)
        if device not in self._dev:
            t = self.tables()
            self._dev[device] = {k: (torch.from_numpy(v).to(device) if isinstance(v, np.ndarray) else v)
                                 for k, v in t.items()}
        return self._dev[device]


def scale_size(h, w, size=CROP):
    """Scale(size) with an int size: (h, w) after it; unchanged when the shorter side already is `size`."""
    if (w <= h and w == size) or (h <= w and h == size):
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def center_offset(n, size=CROP):
    """CenterCrop / FiveCrop(5): int(round((n - size) / 2.)), Python's round (half to even)."""
    return int(round((n - size) / 2.))


def five_crop_box(h, w, where, size=CROP):
    """FiveCrop(size, where) of an h x w frame: (x1, y1, size, size).  1 top-left, 2 top-right, 3 bottom-left,
    4 bottom-right (the reference's h - tw, the same for square crops), 5 centre."""
    if size > h or size > w:
        raise ValueError("FiveCrop(%d) of a %d x %d frame: the frame must be at least %d on each side" % (size, h, w, size))
    x1, y1 = {1: (0, 0), 2: (w - size, 0), 3: (0, h - size), 4: (w - size, h - size),
              5: (center_offset(w, size), center_offset(h, size))}[where]
    return (x1, y1, size, size)


def _window_taps(n, scaled, off, out):
    """Taps of output pixels [off, off + out) of a bicubic resize of n pixels to `scaled`: (start, count, coef)."""
    st, cnt, kk = resize_taps(n, scaled)
    return st[off:off + out], cnt[off:off + out], kk[:, off:off + out]


class ClassifierAugment:
    """The transforms of eval/main_classifier.py for one mode: 'train', 'val', 'test' (one crop view,
    view = (aug_idx, flip_idx) of test_10crop) or 'retrieval'.  A train / val sample is num_seq * seq_len frames;
    a test / retrieval sample is a whole video of any length."""

    def __init__(self, mode, seq_len, img_dim=128, num_seq=1, view=(5, 0)):
        if mode not in MODES:
            raise ValueError("mode must be one of %s, got %r" % (", ".join(MODES), mode))
        if seq_len < 1 or img_dim < 1 or num_seq < 1:
            raise ValueError("seq_len, img_dim and num_seq must be positive")
        aug_idx, flip_idx = (int(v) for v in view)
        if aug_idx not in (1, 2, 3, 4, 5) or flip_idx not in (0, 1):
            raise ValueError("view must be (aug_idx in 1..5, flip_idx in 0, 1), got %r" % (tuple(view),))
        self.mode, self.seq_len, self.img_dim, self.num_seq = mode, int(seq_len), int(img_dim), int(num_seq)
        self.view = (aug_idx, flip_idx)
        self.frames = self.num_seq * self.seq_len            # frames per train / val sample
        self.M = CROP if mode in ("train", "val") and self.img_dim != CROP else self.img_dim
        if self.layout(9)[2] > SMEM_LIMIT:
            raise ValueError("img_dim %d does not fit the kernel's shared memory" % img_dim)

    def layout(self, taps):
        """(band_rows, rows, shared bytes) for a first resize of `taps` taps per pixel: two CTAs per SM when the
        frames fit, else one CTA with the rest of the shared memory for the bands."""
        D, M = self.img_dim, self.M
        half, full = (SMEM_LIMIT - 4096) // 2, SMEM_LIMIT - 1024      # 1 KB per CTA is reserved
        if M == D:
            R = max(taps, (half - 3 * D * D) // (3 * D))
            return R, 0, 3 * D * D + 3 * R * D
        fixed = 3 * M * D
        budget = half if fixed + max(3 * D * D, 6 * M * taps) <= half else full
        R = max(taps, (budget - fixed) // (6 * M))
        return R, R, fixed + max(3 * D * D, 6 * M * R)

    # -- host plan ------------------------------------------------------------------------------------------------
    def plan(self, sizes, py_rng=None, lengths=None, batch_flip=False):
        """Draw every decision for len(sizes) samples, sample after sample, in the reference's call order.
        sizes: [(h, w)] of each sample's source frames; py_rng defaults to the `random` module.  lengths: frames of
        each test / retrieval video (default num_seq * seq_len each; train / val samples always have that many).
        batch_flip: the train batch's T.RandomHorizontalFlip decision, which the reference draws in the main
        process (`random.random() < 0.5` per batch), not in the transform."""
        py = _random if py_rng is None else py_rng
        if lengths is None:
            lengths = [self.frames] * len(sizes)
        if len(lengths) != len(sizes):
            raise ValueError("%d lengths for %d samples" % (len(lengths), len(sizes)))
        if self.mode in ("train", "val") and any(int(n) != self.frames for n in lengths):
            raise ValueError("train / val samples have num_seq * seq_len = %d frames" % self.frames)
        if batch_flip and self.mode != "train":
            raise ValueError("batch_flip is the train recipe's flip")
        samples = []
        for hw, n in zip(sizes, lengths):
            h, w = int(hw[0]), int(hw[1])
            if h < 1 or w < 1 or int(n) < 1:
                raise ValueError("source size %r and length %r must be positive" % (tuple(hw), n))
            sp = ClfSamplePlan(size=(h, w), frames=int(n))
            if self.mode in ("train", "val"):
                self._random_sized_crop(sp, py)
                if self.mode == "train":
                    self._jitter(sp, py)
                    sp.flip = bool(batch_flip)
            elif self.mode == "test":
                aug_idx, flip_idx = self.view
                py.random()                      # RandomHorizontalFlip(command): random() < 0 ('left') or < 1
                sp.src_flip = flip_idx == 1
                sp.crop = five_crop_box(h, w, aug_idx)
                self._jitter(sp, py)
            else:
                if h < CROP or w < CROP:
                    raise ValueError("CenterCrop(%d) of a %d x %d frame: the frame must be at least %d on each side"
                                     % (CROP, h, w, CROP))
                sp.crop = (center_offset(w), center_offset(h), CROP, CROP)
                self._jitter(sp, py)
            samples.append(sp)
        return ClfAugmentPlan(self, samples)

    @staticmethod
    def _random_sized_crop(sp, py, bottom_area=0.2):
        """RandomSizedCrop(224, consistent=True): random() < p (= 1), then up to 10 attempts of uniform, uniform,
        random() (swap) and, when the box fits, randint, randint."""
        h, w = sp.size
        py.random()
        for attempt in range(10):
            area = w * h
            target_area = py.uniform(bottom_area, 1) * area
            aspect_ratio = py.uniform(3. / 4, 4. / 3)
            cw = int(round(math.sqrt(target_area * aspect_ratio)))
            ch = int(round(math.sqrt(target_area / aspect_ratio)))
            if py.random() < 0.5:
                cw, ch = ch, cw
            if cw <= w and ch <= h:
                x1 = py.randint(0, w - cw)
                y1 = py.randint(0, h - ch)
                sp.crop, sp.attempts = (x1, y1, cw, ch), attempt + 1
                return
        sh, sw = scale_size(h, w)
        sp.fallback, sp.attempts = (sh, sw, center_offset(sh), center_offset(sw)), 10

    def _jitter(self, sp, py):
        """ColorJitter(p=.3, consistent=True): random() < p, then get_params: b, c, s, h uniforms and a shuffle."""
        if py.random() < JITTER_P:
            ops = [(name, py.uniform(lo, hi)) for name, (lo, hi) in zip(JITTER_OPS, JITTER[self.mode])]
            py.shuffle(ops)
            sp.jitter = ops
            sp.hue_shift = hue_shift_byte(dict(ops)["hue"])

    # -- device tables --------------------------------------------------------------------------------------------
    def first_taps(self, sp):
        """The first resize of a sample as ((x start, count, coef), (y start, count, coef)) over its M x M output;
        starts are coordinates in the (flipped, for src_flip) source frame."""
        M = self.M
        if sp.fallback is not None:
            h, w = sp.size
            sh, sw, y1, x1 = sp.fallback
            return _window_taps(w, sw, x1, CROP), _window_taps(h, sh, y1, CROP)
        x1, y1, cw, ch = sp.crop
        (xs, xn, xk), (ys, yn, yk) = resize_taps(cw, M), resize_taps(ch, M)
        return (xs + x1, xn, xk), (ys + y1, yn, yk)

    def _tables(self, plan):
        """Packs a plan into the kernel's inputs (layouts in include/coclr_b200.h, coclr_augment_clf_t)."""
        NS, D, M, DD = len(plan), self.img_dim, self.M, self.img_dim ** 2
        taps = [self.first_taps(sp) for sp in plan.samples]
        K1 = max(max(tx[2].shape[0], ty[2].shape[0]) for tx, ty in taps)
        coef1 = np.zeros((NS, 2, K1, M), np.int32)
        bounds1 = np.zeros((NS, 2, 2, M), np.int32)
        for i, axes in enumerate(taps):
            for a, (st, n, kk) in enumerate(axes):
                coef1[i, a, :kk.shape[0]] = kk
                bounds1[i, a, 0], bounds1[i, a, 1] = st, n
        rec = np.zeros((NS, SAMPLE_INTS), np.int32)
        op_code = {n: i for i, n in enumerate(JITTER_OPS)}
        for i, sp in enumerate(plan.samples):
            if sp.jitter is not None:
                rec[i, 0] = len(sp.jitter)
                for j, (name, f) in enumerate(sp.jitter):
                    rec[i, 1 + j] = op_code[name]
                    if name != "hue":
                        rec[i, 5 + op_code[name]] = np.float32(f).view(np.int32)
                rec[i, 8] = sp.hue_shift or 0
            rec[i, 9], rec[i, 10], rec[i, 11] = int(sp.flip), int(sp.src_flip), sp.size[1]
        n = np.asarray(plan.lengths, np.int64)
        first = np.concatenate([[0], np.cumsum(n)[:-1]])
        frames = np.zeros((int(n.sum()), FRAME_LONGS), np.int64)
        k = 0
        for i in range(NS):
            t = np.arange(n[i])
            frames[k:k + n[i], 0] = i
            frames[k:k + n[i], 1] = first[i] + t                   # source frame
            frames[k:k + n[i], 2] = 3 * DD * first[i] + t * DD     # sample i is [3, n_i, D, D] at 3 * DD * first_i
            frames[k:k + n[i], 3] = n[i] * DD
            k += n[i]
        t = {"K1": K1, "coef1": coef1, "bounds1": bounds1, "samples": rec, "frames": frames}
        if M != D:
            st, cnt, kk = resize_taps(M, D)
            t["K2"], t["coef2"], t["bounds2"] = kk.shape[0], np.ascontiguousarray(kk), np.stack([st, cnt])
        return t

    # -- launch ---------------------------------------------------------------------------------------------------
    def __call__(self, frames, plan):
        """frames: uint8 channels-last frames contiguous on a CUDA device, either [B, F, Hmax, Wmax, 3] (every sample
        F frames) or [sum of the plan's lengths, Hmax, Wmax, 3] (the samples' frames one after another).  Returns
        [B, 3, F, D, D] float32 for train / val, and a list of [3, T_i, D, D] videos (views into one buffer) for
        test / retrieval."""
        self._validate(frames, plan)
        from . import lib as L
        D = self.img_dim
        Hm, Wm = frames.shape[-3], frames.shape[-2]
        NF = int(np.prod(frames.shape[:-3]))
        dev = plan.to(frames.device)
        R, Y, smem = self.layout(dev["K1"])
        if smem > SMEM_LIMIT:
            raise ValueError("a resize of %d taps per pixel does not fit the kernel's shared memory" % dev["K1"])
        total = sum(plan.lengths)
        out = torch.empty(3 * total * D * D, dtype=torch.float32, device=frames.device)
        a = L.AugmentClf()
        a.src, a.NF, a.Hmax, a.Wmax, a.n_frames = L.dptr(frames), NF, Hm, Wm, total
        a.frames, a.samples = L.dptr(dev["frames"]), L.dptr(dev["samples"])
        a.M, a.D, a.K1, a.band_rows, a.rows = self.M, D, dev["K1"], R, Y
        a.coef1, a.bounds1 = L.dptr(dev["coef1"]), L.dptr(dev["bounds1"])
        if self.M != D:
            a.K2, a.coef2, a.bounds2 = dev["K2"], L.dptr(dev["coef2"]), L.dptr(dev["bounds2"])
        a.out = L.dptr(out)
        L.check(L.load().coclr_augment_clf(C.byref(a), L.stream_ptr()), "coclr_augment_clf")
        if self.mode in ("train", "val"):
            return out.view(len(plan), 3, self.frames, D, D)
        videos, off = [], 0
        for n in plan.lengths:
            videos.append(out[off:off + 3 * n * D * D].view(3, n, D, D))
            off += 3 * n * D * D
        return videos

    def _validate(self, frames, plan):
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise ValueError("frames must be a uint8 tensor")
        if frames.dim() not in (4, 5) or frames.shape[-1] != 3 or not frames.is_contiguous():
            raise ValueError("frames must be contiguous [B, F, H, W, 3] or [N, H, W, 3] (channels last), got %s"
                             % (tuple(frames.shape),))
        if not isinstance(plan, ClfAugmentPlan) or plan.aug.mode != self.mode or plan.aug.img_dim != self.img_dim \
                or plan.aug.frames != self.frames or plan.aug.view != self.view:
            raise ValueError("plan was not made by a ClassifierAugment of this mode / seq_len / img_dim / view")
        if len(plan) < 1:
            raise ValueError("plan has no samples")
        if frames.dim() == 5:
            if frames.shape[0] != len(plan):
                raise ValueError("plan has %d samples, frames %d" % (len(plan), frames.shape[0]))
            if any(n != frames.shape[1] for n in plan.lengths):
                raise ValueError("frames per sample is %d, the plan's lengths are %s" % (frames.shape[1], plan.lengths))
        elif frames.shape[0] != sum(plan.lengths):
            raise ValueError("%d frames for the plan's %d" % (frames.shape[0], sum(plan.lengths)))
        Hm, Wm = frames.shape[-3], frames.shape[-2]
        for h, w in plan.sizes:
            if h > Hm or w > Wm:
                raise ValueError("source size (%d, %d) exceeds the frame buffer (%d, %d)" % (h, w, Hm, Wm))
        if not frames.is_cuda:
            raise ValueError("frames must be on a CUDA device")
