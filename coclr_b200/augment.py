"""Pre-training augmentation on the GPU: the reference's `get_transform('train')` of main_nce.py / main_coclr.py
(utils/augmentation.py under PIL) as one CUDA kernel (csrc/augment.cu, `coclr_augment`), bit-identical to the
reference's DataLoader tensor for the same random decisions.

    aug = PretrainAugment(seq_len=32, img_dim=128)            # two_stream=True for main_coclr.py
    plan = aug.plan(sizes)                                    # host only: every random draw, in the reference's order
    x = aug(frames, plan)                                     # frames: uint8 [B, 2T, Hmax, Wmax, 3] on the GPU
    model.set_input_transform(); model(x)                     # x: [B, 3, 2T, img_dim, img_dim] in [0, 1]

The recipe is TransformController([TwoClipTransform(base, null, p=.3), OneClipTransform(base, null)], [.5, .5]),
null = RandomSizedCrop + flip and base = RandomSizedCrop, RandomApply(ColorJitter(.4, .4, .4, .1), .8),
RandomGray(.2), RandomApply(GaussianBlur([.1, 2.]), .5), flip.  `plan` consumes Python `random`, `np.random` and
torch's CPU generator (RandomApply's torch.rand(1)) exactly as the reference does, so seeding the three the same way
gives the decisions the reference makes for the same samples, one sample after another.

Everything Pillow computes in double (bicubic coefficients, box-blur radius and weights) is computed here, on the
host, with the same operations in the same order; the kernel then runs only integer and explicitly rounded float /
double arithmetic.
"""
import ctypes as C
import math
import random as _random
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np
import torch

PRECISION_BITS = 22                   # Resample.c: 32 - 8 - 2
JITTER_OPS = ("brightness", "contrast", "saturation", "hue")
JITTER_RANGES = ((0.6, 1.4), (0.6, 1.4), (0.6, 1.4), (-0.1, 0.1))    # ColorJitter(.4, .4, .4, .1)
SMEM_LIMIT = 227 * 1024               # opt-in shared memory per block on sm_90


# ----------------------------------------------------------------------------------------------------------------------
# Pillow's tables
# ----------------------------------------------------------------------------------------------------------------------

def _bicubic(x):
    """Resample.c bicubic_filter (a = -0.5), elementwise in double."""
    x = np.abs(x)
    near = ((-0.5 + 2.0) * x - (-0.5 + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * -0.5
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def resize_taps(in_size, out_size):
    """Resample.c precompute_coeffs + normalize_coeffs_8bpc for a bicubic resize of [0, in_size) to out_size.
    Returns (start [out], count [out], coef [K, out] int32) with K = 2 * ceil(support) + 1; coef[k, o] weighs
    source pixel start[o] + k."""
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 2.0 * filterscale
    K = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    ss = 1.0 / filterscale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    w = np.zeros((K, out_size))
    ww = np.zeros(out_size)
    for k in range(K):                                   # left to right, as the C loop sums
        live = k < xmax
        w[k] = np.where(live, _bicubic((k + xmin - center + 0.5) * ss), 0.0)
        ww = np.where(live, ww + w[k], ww)
    w = np.where(ww != 0.0, w / np.where(ww != 0.0, ww, 1.0), w)
    kk = np.where(w < 0, np.trunc(-0.5 + w * (1 << PRECISION_BITS)), np.trunc(0.5 + w * (1 << PRECISION_BITS)))
    return xmin.astype(np.int32), xmax.astype(np.int32), kk.astype(np.int32)


def box_blur_weights(sigma):
    """ImageFilter.GaussianBlur(radius=sigma) -> BoxBlur.c: the fractional box radius of _gaussian_blur_radius(sigma, 3)
    in float32 (double where C promotes), then ImagingHorizontalBoxBlur's integer radius and 24-bit weights.
    Returns (radius, ww, fw)."""
    f32 = np.float32
    radius = f32(sigma)
    sigma2 = radius * radius / f32(3)
    L = f32(math.sqrt(12.0 * float(sigma2) + 1.0))
    l = f32(math.floor((float(L) - 1.0) / 2.0))
    a = (f32(2) * l + f32(1)) * (l * (l + f32(1)) - f32(3) * sigma2)
    a = a / (f32(6) * (sigma2 - (l + f32(1)) * (l + f32(1))))
    fr = l + a
    r = int(fr)
    ww = int(f32(1 << 24) / (fr * f32(2) + f32(1)))
    fw = ((1 << 24) - (r * 2 + 1) * ww) // 2
    return r, ww, fw


def hue_shift_byte(hue_factor):
    """torchvision adjust_hue: np.int32(hue_factor * 255).astype(np.uint8)."""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


# ----------------------------------------------------------------------------------------------------------------------
# The plan: every random decision of the reference transform, drawn in its order
# ----------------------------------------------------------------------------------------------------------------------

@dataclass
class ClipPlan:
    """Decisions for one augmented clip (one call of `base` or `null`)."""
    half: int                                          # source half the clip reads: frames [half*S, (half+1)*S)
    base: bool                                         # True: base transform, False: null transform
    crop: Optional[Tuple[int, int, int, int]]          # (x1, y1, w, h), or None: the box did not fit, whole frame
    jitter: Optional[List[Tuple[str, float]]] = None   # [(op, factor)] in application order, or None
    hue_shift: Optional[int] = None                    # byte added to PIL's H (mod 256) when jitter has 'hue'
    gray: Optional[List[int]] = None                   # channel replicated in each frame, or None
    blur_sigma: Optional[float] = None
    flip: bool = False


@dataclass
class SamplePlan:
    two_clip: bool                                     # TwoClipTransform (True) or OneClipTransform
    size: Tuple[int, int]                              # (h, w) of the sample's source frames
    clips: List[ClipPlan] = field(default_factory=list)


class AugmentPlan:
    """Per-sample decisions plus the device tables they compile to (built lazily, once per device)."""

    def __init__(self, aug, samples):
        self.aug = aug
        self.samples = samples
        self._dev = {}

    @property
    def sizes(self):
        return [s.size for s in self.samples]

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


def _rand_apply(p, gen):
    """torchvision RandomApply.forward: skip when p < torch.rand(1)."""
    return not (p < torch.rand(1, generator=gen))


class PretrainAugment:
    """get_transform('train') of main_nce.py (two_stream=False: clips of seq_len frames) or main_coclr.py
    (two_stream=True: each clip is seq_len rgb frames then seq_len flow frames, transformed together)."""

    def __init__(self, seq_len, img_dim=128, two_stream=False):
        if seq_len < 1 or img_dim < 1:
            raise ValueError("seq_len and img_dim must be positive")
        self.seq_len, self.img_dim, self.two_stream = int(seq_len), int(img_dim), bool(two_stream)
        self.S = self.seq_len * (2 if two_stream else 1)   # frames one transform call sees (the reference's seq_len)
        self.frames = 2 * self.S                           # source frames per sample
        if self.smem_bytes(self.img_dim) > SMEM_LIMIT:
            raise ValueError("img_dim %d does not fit the kernel's shared-memory frame" % img_dim)

    @staticmethod
    def band_rows(d, taps=0):
        """Source rows per horizontal resize band: at least one output row's taps and one frame plane (the band
        doubles as the blur's second plane), else what leaves room for two CTAs per SM."""
        return max(d, taps, ((SMEM_LIMIT - 4096) // 2 - 3 * d * d) // (3 * d))   # 1 KB per CTA is reserved

    @staticmethod
    def smem_bytes(d, taps=0):
        return 3 * d * d + 3 * d * PretrainAugment.band_rows(d, taps)

    # -- host plan ------------------------------------------------------------------------------------------------
    def plan(self, sizes, py_rng=None, np_rng=None, torch_gen=None):
        """Draw every decision for len(sizes) samples, sample after sample, in the reference's call order.
        sizes: [(h, w)] of each sample's source frames.  py_rng defaults to the `random` module, np_rng to
        `np.random`, torch_gen to torch's default CPU generator."""
        py = _random if py_rng is None else py_rng
        npr = np.random if np_rng is None else np_rng
        samples = []
        for hw in sizes:
            h, w = int(hw[0]), int(hw[1])
            if h < 1 or w < 1:
                raise ValueError("source size %r: sides must be positive" % (tuple(hw),))
            idx = py.choices(range(2), weights=[0.5, 0.5])[0]
            if idx == 0:                                              # TwoClipTransform(p=0.3)
                b1 = py.random() < 0.3
                b2 = py.random() < 0.3
                sp = SamplePlan(True, (h, w))
                sp.clips.append(self._clip(0, b1, h, w, py, npr, torch_gen))
                sp.clips.append(self._clip(1, b2, h, w, py, npr, torch_gen))
            else:                                                     # OneClipTransform
                first_base = py.random() < 0.5
                half = 0 if py.random() < 0.5 else 1
                sp = SamplePlan(False, (h, w))
                sp.clips.append(self._clip(half, first_base, h, w, py, npr, torch_gen))
                sp.clips.append(self._clip(half, not first_base, h, w, py, npr, torch_gen))
            samples.append(sp)
        return AugmentPlan(self, samples)

    def _clip(self, half, base, h, w, py, npr, gen):
        c = ClipPlan(half=half, base=base, crop=self._crop(h, w, py))
        if base:
            if _rand_apply(0.8, gen):                                 # RandomApply([ColorJitter], p=.8)
                py.random()                                           # ColorJitter(p=1.0): random() < 1.0
                ops = [(name, py.uniform(lo, hi)) for name, (lo, hi) in zip(JITTER_OPS, JITTER_RANGES)]
                py.shuffle(ops)
                c.jitter = ops
                c.hue_shift = hue_shift_byte(dict(ops)["hue"])
            if py.random() < 0.2:                                     # RandomGray(p=.2): one draw per clip,
                c.gray = [int(npr.choice(3)) for _ in range(self.S)]  # one channel per frame
            if _rand_apply(0.5, gen):                                 # RandomApply([GaussianBlur], p=.5)
                c.blur_sigma = py.uniform(0.1, 2.0)
        c.flip = py.random() < 0.5                                    # RandomHorizontalFlip: one draw per clip
        return c

    @staticmethod
    def _crop(h, w, py):
        """RandomSizedCrop(consistent=False, bottom_area=.2), first attempt only (that branch always returns)."""
        py.random()                                                   # random() < p (= 1.0)
        area = w * h
        target_area = py.uniform(0.2, 1) * area
        aspect_ratio = py.uniform(3. / 4, 4. / 3)
        cw = int(round(math.sqrt(target_area * aspect_ratio)))
        ch = int(round(math.sqrt(target_area / aspect_ratio)))
        if py.random() < 0.5:
            cw, ch = ch, cw
        if cw <= w and ch <= h:
            x1 = py.randint(0, w - cw)
            y1 = py.randint(0, h - ch)
            return (x1, y1, cw, ch)
        return None

    # -- device tables --------------------------------------------------------------------------------------------
    def _tables(self, plan):
        """Packs a plan into the kernel's inputs (layouts in include/coclr_b200.h, coclr_augment_t)."""
        B, D, S = len(plan), self.img_dim, self.S
        taps = []
        for sp in plan.samples:
            h, w = sp.size
            for c in sp.clips:
                x1, y1, cw, ch = c.crop if c.crop is not None else (0, 0, w, h)
                taps.append((resize_taps(cw, D), x1, resize_taps(ch, D), y1))
        K = max(max(tx[2].shape[0], ty[2].shape[0]) for tx, _, ty, _ in taps)
        coef = np.zeros((B * 2, 2, K, D), np.int32)
        bounds = np.zeros((B * 2, 2, 2, D), np.int32)
        for i, (tx, x1, ty, y1) in enumerate(taps):
            for a, ((st, n, kk), off) in enumerate(((tx, x1), (ty, y1))):
                coef[i, a, :kk.shape[0]] = kk
                bounds[i, a, 0] = st + off
                bounds[i, a, 1] = n
        rec = np.zeros((B * 2, CLIP_INTS), np.int32)
        gray = np.full((B * 2, S), -1, np.int8)
        op_code = {n: i for i, n in enumerate(JITTER_OPS)}
        for i, c in enumerate(cl for sp in plan.samples for cl in sp.clips):
            rec[i, 0] = c.half * S
            if c.jitter is not None:
                rec[i, 1] = len(c.jitter)
                for j, (name, f) in enumerate(c.jitter):
                    rec[i, 2 + j] = op_code[name]
                    if name != "hue":
                        rec[i, 6 + op_code[name]] = np.float32(f).view(np.int32)
                rec[i, 9] = c.hue_shift or 0          # a chain without hue leaves the shift unused
            if c.blur_sigma is not None:
                r, ww, fw = box_blur_weights(c.blur_sigma)
                rec[i, 10], rec[i, 11], rec[i, 12] = r, ww, fw
            else:
                rec[i, 10] = -1
            rec[i, 13] = int(c.flip)
            if c.gray is not None:
                gray[i] = c.gray
        return {"K": K, "coef": coef, "bounds": bounds, "clips": rec, "gray": gray}

    # -- launch ---------------------------------------------------------------------------------------------------
    def __call__(self, frames, plan, sizes=None):
        """frames: uint8 [B, 2S, Hmax, Wmax, 3] contiguous on a CUDA device (S = seq_len, or 2 * seq_len with
        two_stream).  Returns [B, 3, 2S, D, D] float32, or with two_stream the reference's (seq1, seq2), each
        [B, 3, 2 * seq_len, D, D]."""
        self._validate(frames, plan, sizes)
        from . import lib as L
        B, F, Hm, Wm, _ = frames.shape
        D, S = self.img_dim, self.S
        dev = plan.to(frames.device)
        if self.smem_bytes(D, dev["K"]) > SMEM_LIMIT:
            raise ValueError("a resize of %d taps per pixel does not fit the kernel's shared memory" % dev["K"])
        if self.two_stream:       # seq1 and seq2 as two contiguous [B, 3, S, D, D] halves of one buffer
            out = torch.empty(2, B, 3, S, D, D, dtype=torch.float32, device=frames.device)
            strides = (3 * S * D * D, B * 3 * S * D * D, S * D * D)
        else:
            out = torch.empty(B, 3, 2 * S, D, D, dtype=torch.float32, device=frames.device)
            strides = (3 * 2 * S * D * D, S * D * D, 2 * S * D * D)
        a = L.Augment()
        a.src, a.B, a.F, a.Hmax, a.Wmax = L.dptr(frames), B, F, Hm, Wm
        a.S, a.D, a.K, a.band_rows = S, D, dev["K"], self.band_rows(D, dev["K"])
        a.clips, a.coef, a.bounds, a.gray = (L.dptr(dev[k]) for k in ("clips", "coef", "bounds", "gray"))
        a.out = L.dptr(out)
        a.out_batch_stride, a.out_clip_stride, a.out_chan_stride = strides
        L.check(L.load().coclr_augment(C.byref(a), L.stream_ptr()), "coclr_augment")
        if self.two_stream:
            return out[0], out[1]
        return out

    def _validate(self, frames, plan, sizes):
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise ValueError("frames must be a uint8 tensor")
        if frames.dim() != 5 or frames.shape[-1] != 3 or not frames.is_contiguous():
            raise ValueError("frames must be contiguous [B, F, H, W, 3] (channels last), got %s" % (tuple(frames.shape),))
        if frames.shape[1] != self.frames:
            raise ValueError("frames per sample must be %d (2 x %d%s), got %d" % (
                self.frames, self.seq_len, " x 2 streams" if self.two_stream else "", frames.shape[1]))
        if not isinstance(plan, AugmentPlan) or plan.aug.S != self.S or plan.aug.img_dim != self.img_dim:
            raise ValueError("plan was not made by a PretrainAugment of this seq_len / img_dim / two_stream")
        if len(plan) != frames.shape[0]:
            raise ValueError("plan has %d samples, frames %d" % (len(plan), frames.shape[0]))
        if sizes is not None and [tuple(int(v) for v in s) for s in sizes] != [tuple(s) for s in plan.sizes]:
            raise ValueError("sizes differ from the sizes the plan was drawn for")
        Hm, Wm = frames.shape[2], frames.shape[3]
        for h, w in plan.sizes:
            if h < 1 or w < 1 or h > Hm or w > Wm:
                raise ValueError("source size (%d, %d) is empty or exceeds the frame buffer (%d, %d)" % (h, w, Hm, Wm))
        if not frames.is_cuda:
            raise ValueError("frames must be on a CUDA device")


CLIP_INTS = 16   # int32 words per clip record (coclr_augment_clip_t)
