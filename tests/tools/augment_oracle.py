"""numpy restatement of the Pillow / torchvision arithmetic behind the reference's pre-training augmentation
(utils/augmentation.py).  It is the CPU check that the host tables of coclr_b200.augment (bicubic coefficients,
box-blur weights) reproduce Pillow, and the statement the CUDA kernel (csrc/augment.cu) mirrors operation by
operation.  Every function takes and returns uint8 [H, W, 3] arrays.

Sources of the arithmetic (Pillow 12, libImaging): Resample.c (bicubic, 22-bit fixed point), Blend.c (float32
blend, truncate, clamp), Convert.c (L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16, RGB <-> HSV in float / double),
BoxBlur.c (extended box blur, 24-bit fixed point); ImageEnhance (degenerate images), ImageStat (mean).
"""
import numpy as np

from coclr_b200 import augment as A


def resize(img, d):
    """Image.resize((d, d), BICUBIC) of the whole image: horizontal pass, then vertical, uint8 in between."""
    h, w = img.shape[:2]
    (xs, xn, xc), (ys, yn, yc) = A.resize_taps(w, d), A.resize_taps(h, d)
    tmp = np.empty((h, d, 3), np.uint8)
    for x in range(d):
        acc = np.full((h, 3), 1 << 21, np.int64)
        for k in range(xn[x]):
            acc += img[:, xs[x] + k, :].astype(np.int64) * int(xc[k, x])
        tmp[:, x] = np.clip(acc >> 22, 0, 255)
    out = np.empty((d, d, 3), np.uint8)
    for y in range(d):
        acc = np.full((d, 3), 1 << 21, np.int64)
        for k in range(yn[y]):
            acc += tmp[ys[y] + k].astype(np.int64) * int(yc[k, y])
        out[y] = np.clip(acc >> 22, 0, 255)
    return out


def luma(img):
    i = img.astype(np.int64)
    return ((i[..., 0] * 19595 + i[..., 1] * 38470 + i[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def blend(deg, img, factor):
    """Image.blend(deg, img, factor): float32 d + f * (x - d), truncated, clamped to [0, 255]."""
    a = np.float32(factor)
    d = deg.astype(np.float32)
    t = d + a * (img.astype(np.float32) - d)           # float32 throughout, no contraction in numpy
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.trunc(np.clip(t, 0, 255)))).astype(np.uint8)


def brightness(img, f):
    return blend(np.zeros_like(img), img, f)


def contrast(img, f):
    s, n = int(luma(img).astype(np.int64).sum()), img.shape[0] * img.shape[1]
    mean = (2 * s + n) // (2 * n)                      # int(s / n + 0.5), exactly
    return blend(np.full_like(img, mean), img, f)


def saturation(img, f):
    return blend(np.repeat(luma(img)[..., None], 3, axis=2), img, f)


def rgb_to_hsv(img):
    """Convert.c rgb2hsv: float32 intermediates, double where the C source promotes."""
    r, g, b = (img[..., c].astype(np.int32) for c in range(3))
    mx, mn = np.maximum(np.maximum(r, g), b), np.minimum(np.minimum(r, g), b)
    cr = (mx - mn).astype(np.float32)
    ok = mx != mn
    crs = np.where(ok, cr, np.float32(1))
    s = np.where(ok, cr / np.where(ok, mx, 1).astype(np.float32), np.float32(0)).astype(np.float32)
    rc, gc, bc = ((mx - c).astype(np.float32) / crs for c in (r, g, b))
    h = np.where(r == mx, (bc - gc).astype(np.float32),
                 np.where(g == mx, ((2.0 + rc.astype(np.float64)) - bc).astype(np.float32),
                          ((4.0 + gc.astype(np.float64)) - rc).astype(np.float32)))
    h = np.fmod(h.astype(np.float64) / 6.0 + 1.0, 1.0).astype(np.float32)
    uh = np.clip((h.astype(np.float64) * 255.0).astype(np.int64), 0, 255)
    us = np.clip((s.astype(np.float64) * 255.0).astype(np.int64), 0, 255)
    return np.stack([np.where(ok, uh, 0), np.where(ok, us, 0), mx], -1).astype(np.uint8)


def _round_half_away(x):
    return np.where(x >= 0, np.floor(x + 0.5), -np.floor(-x + 0.5))


def hsv_to_rgb(hsv):
    """Convert.c hsv2rgb."""
    h, s, v = (hsv[..., c].astype(np.float64) for c in range(3))
    hh = h * 6.0 / 255.0
    i = np.floor(hh).astype(np.int64)
    f = (hh - i.astype(np.float32).astype(np.float64)).astype(np.float32)
    fs = (s.astype(np.float32).astype(np.float64) / 255.0).astype(np.float32)
    vf = v.astype(np.float32).astype(np.float64)
    p = np.clip(_round_half_away(vf * (1.0 - fs.astype(np.float64))), 0, 255).astype(np.uint8)
    q = np.clip(_round_half_away(vf * (1.0 - (fs * f).astype(np.float64))), 0, 255).astype(np.uint8)
    t = np.clip(_round_half_away(vf * (1.0 - fs.astype(np.float64) * (1.0 - f.astype(np.float64)))), 0, 255).astype(np.uint8)
    v8 = hsv[..., 2]
    i = i % 6
    sel = [(v8, t, p), (q, v8, p), (p, v8, t), (p, q, v8), (t, p, v8), (v8, p, q)]
    out = np.empty(hsv.shape, np.uint8)
    for c in range(3):
        ch = np.select([i == k for k in range(6)], [sel[k][c] for k in range(6)])
        out[..., c] = np.where(hsv[..., 1] == 0, v8, ch)
    return out


def hue(img, shift):
    """torchvision adjust_hue on PIL: HSV, H += shift (mod 256), back to RGB.  `shift` is the byte
    np.int32(hue_factor * 255).astype(np.uint8)."""
    hsv = rgb_to_hsv(img)
    hsv[..., 0] = (hsv[..., 0].astype(np.int32) + int(shift)) & 255
    return hsv_to_rgb(hsv)


def _box_pass(a, r, ww, fw, axis):
    """One BoxBlur.c line pass along `axis` with clamped edges: (ww * window + fw * (two far pixels) + 2^23) >> 24."""
    n = a.shape[axis]
    idx = np.arange(n)
    take = lambda o: np.take(a, np.clip(idx + o, 0, n - 1), axis=axis).astype(np.uint64)
    s = sum(take(o) for o in range(-r, r + 1))
    out = (np.uint64(ww) * s + np.uint64(fw) * (take(-r - 1) + take(r + 1)) + np.uint64(1 << 23)) >> np.uint64(24)
    return out.astype(np.uint8)


def blur(img, sigma):
    """ImageFilter.GaussianBlur(sigma): three horizontal then three vertical extended-box passes."""
    r, ww, fw = A.box_blur_weights(sigma)
    for axis in (1, 1, 1, 0, 0, 0):
        img = _box_pass(img, r, ww, fw, axis)
    return img


def gray(img, channel):
    return np.repeat(img[..., channel:channel + 1], 3, axis=2)


def flip(img):
    return img[:, ::-1].copy()


JITTER = {"brightness": brightness, "contrast": contrast, "saturation": saturation}


def jitter(img, ops):
    """ops: [(name, value)] in application order; value is the factor, or the hue shift byte for 'hue'."""
    for name, v in ops:
        img = hue(img, v) if name == "hue" else JITTER[name](img, v)
    return img


def to_tensor(frames):
    """ToTensor of each frame stacked along dim 1: uint8 [F, H, W, 3] -> float32 [3, F, H, W] = x / 255."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(frames)).permute(3, 0, 1, 2).float().div(255)


def crop_resize(img, crop, d):
    if crop is not None:
        x1, y1, w, h = crop
        img = img[y1:y1 + h, x1:x1 + w]
    return resize(img, d)


def clip(frames, c, d):
    """One ClipPlan applied to its S source frames [S, H, W, 3] -> [S, d, d, 3]."""
    out = []
    for j, f in enumerate(frames):
        f = crop_resize(f, c.crop, d)
        if c.jitter is not None:
            f = jitter(f, [(n, c.hue_shift if n == "hue" else v) for n, v in c.jitter])
        if c.gray is not None:
            f = gray(f, c.gray[j])
        if c.blur_sigma is not None:
            f = blur(f, c.blur_sigma)
        out.append(flip(f) if c.flip else f)
    return np.stack(out)


def sample(aug, sp, frames):
    """One SamplePlan on one sample's frames [2S, h, w, 3]: the uint8 frames of the loader tensor in output order
    ([2S, d, d, 3]: q clip then k clip)."""
    S = aug.S
    return np.concatenate([clip(frames[c.half * S:(c.half + 1) * S], c, aug.img_dim) for c in sp.clips])
