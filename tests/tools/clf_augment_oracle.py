"""numpy restatement of the classifier augmentation (coclr_b200.clf_augment, csrc/augment_clf.cu): the first bicubic
resize read through a sample's tap tables (crop box, fallback window, or a flipped frame's window), the second resize
224 -> img_dim with a uint8 image in between, the jitter chain and the flip.  It is the CPU check that the host tables
reproduce Pillow, and the statement the kernel mirrors.  Frames are uint8 [H, W, 3] arrays; the per-pixel arithmetic is
tests/tools/augment_oracle.py's.
"""
import numpy as np

import augment_oracle as O


def _hpass(img, taps):
    st, n, kk = taps
    out = np.empty((img.shape[0], len(st), 3), np.uint8)
    for x in range(len(st)):
        acc = np.full((img.shape[0], 3), 1 << 21, np.int64)
        for k in range(n[x]):
            acc += img[:, st[x] + k, :].astype(np.int64) * int(kk[k, x])
        out[:, x] = np.clip(acc >> 22, 0, 255)
    return out


def resample(img, xtaps, ytaps):
    """One Pillow resize pair of passes (horizontal over every source row, then vertical), uint8 after each."""
    return _hpass(_hpass(img, xtaps).transpose(1, 0, 2), ytaps).transpose(1, 0, 2).copy()


def first_resize(aug, sp, frame):
    """The sample's first resize of one source frame [h, w, 3] (its top-left sp.size) -> [M, M, 3]."""
    h, w = sp.size
    f = frame[:h, :w]
    if sp.src_flip:
        f = f[:, ::-1]
    xt, yt = aug.first_taps(sp)
    return resample(np.ascontiguousarray(f), xt, yt)


def frame(aug, sp, src):
    """One output frame, uint8 [D, D, 3]: first resize, second resize when there are two, jitter, flip."""
    x = first_resize(aug, sp, src)
    if aug.M != aug.img_dim:
        x = O.resize(x, aug.img_dim)
    if sp.jitter is not None:
        x = O.jitter(x, [(n, sp.hue_shift if n == "hue" else v) for n, v in sp.jitter])
    return O.flip(x) if sp.flip else x


def sample(aug, sp, frames):
    """A sample's frames [n, h, w, 3] -> uint8 [n, D, D, 3] (to_tensor of it is the reference's [3, n, D, D])."""
    return np.stack([frame(aug, sp, f) for f in frames])
