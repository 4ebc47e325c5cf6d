"""Writes tests/golden/augment.npz by running the UNMODIFIED reference utils/augmentation.py ($COCLR_REFERENCE)
under Pillow / torchvision on small smooth-plus-noise sources.

Three groups of cases, every output stored as uint8 (the stored bytes / 255 in float32 are asserted here to be the
reference's ToTensor output bit for bit):
  op_*      one PIL operation on one frame (op_img unless the case stores its own op<i>_src): crop + bicubic resize (downscale, upscale, one axis unchanged, the whole
            frame as when the crop does not fit, 320x240 -> 128), brightness / contrast / saturation, hue (wrapping
            shifts included), GaussianBlur, the gray channel split and the flip
  chain_*   the ColorJitter chain (torchvision's functional ops, as the reference's Lambdas call them) in 8 orders
  nce_*     the whole get_transform('train') recipe of main_nce.py (seq_len 2, img_dim 24), 16 samples
  coclr_*   the same for main_coclr.py (two streams: seq_len 2, so 8 source frames per sample; img_dim 24), 16 samples
For the recipe samples the file holds the three seeds (random, np.random, torch), each sample's source index, the
output, the first draw of each generator after the call, and, recorded by wrapping RandomSizedCrop.__call__ and
Image.crop (behaviour and draws unchanged), each clip's first source frame and crop box (-1s: no crop).

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_augment.py
"""
import importlib.util
import os
import random
import sys

import numpy as np
import PIL
import torch
import torchvision
from PIL import Image, ImageFilter
from torchvision import transforms
import torchvision.transforms.functional as TF

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402

OUT = os.path.join(HERE, "augment.npz")


def load_reference_augmentation():
    path = os.path.join(REF, "utils", "augmentation.py")
    spec = importlib.util.spec_from_file_location("reference_augmentation", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def source(rng, h, w, frames=None, block=2):
    """Smooth colour fields plus a little noise on block x block cells (so that every op has work to do and rounding
    is exercised, while the file stays small)."""
    def one():
        hb, wb = -(-h // block), -(-w // block)
        y, x = np.mgrid[0:hb, 0:wb] * block
        ph = rng.uniform(0, 6.3, 6)
        fx, fy = rng.uniform(3, 12, 2) * block / 2
        img = np.stack([128 + 110 * np.sin(x / fx + ph[c]) * np.cos(y / fy + ph[c + 3]) for c in range(3)], -1)
        img = np.clip(img + rng.integers(-6, 7, (hb, wb, 3)), 0, 255).astype(np.uint8)
        return np.ascontiguousarray(img.repeat(block, 0).repeat(block, 1)[:h, :w])
    return one() if frames is None else np.stack([one() for _ in range(frames)])


def get_transform(A, seq_len, img_dim):
    """main_nce.py / main_coclr.py get_transform('train') with the reference's classes (seq_len is the value the
    reference passes: args.seq_len for main_nce.py, 2 * args.seq_len for main_coclr.py)."""
    null = transforms.Compose([
        A.RandomSizedCrop(size=img_dim, consistent=False, seq_len=seq_len, bottom_area=0.2),
        A.RandomHorizontalFlip(consistent=False, seq_len=seq_len),
        A.ToTensor(),
    ])
    base = transforms.Compose([
        A.RandomSizedCrop(size=img_dim, consistent=False, seq_len=seq_len, bottom_area=0.2),
        transforms.RandomApply([A.ColorJitter(0.4, 0.4, 0.4, 0.1, p=1.0, consistent=False, seq_len=seq_len)], p=0.8),
        A.RandomGray(p=0.2, seq_len=seq_len),
        transforms.RandomApply([A.GaussianBlur([.1, 2.], seq_len=seq_len)], p=0.5),
        A.RandomHorizontalFlip(consistent=False, seq_len=seq_len),
        A.ToTensor(),
    ])
    return A.TransformController([A.TwoClipTransform(base, null, seq_len=seq_len, p=0.3),
                                  A.OneClipTransform(base, null, seq_len=seq_len)], weights=[0.5, 0.5])


def as_u8(t):
    """uint8 bytes whose float32 / 255 is exactly t (asserted)."""
    u = torch.round(t * 255).to(torch.uint8)
    assert torch.equal(u.float().div(255), t)
    return u.numpy()


def op_cases(A, rng):
    cases = []     # (name, params, src, out)
    to = lambda im: np.array(im)
    # crop + resize: (source h, w), box (x1, y1, w, h), output side
    for (h, w), box, d in [((240, 320), (0, 0, 320, 240), 128),     # the whole frame, 4:3 -> square (no-fit branch)
                           ((48, 64), (5, 3, 50, 40), 32),           # downscale
                           ((30, 40), (7, 4, 21, 17), 48),           # upscale
                           ((60, 45), (0, 0, 45, 60), 64),           # whole frame, upscale
                           ((64, 64), (9, 2, 32, 50), 32),           # width unchanged
                           ((70, 50), (3, 11, 41, 40), 40),          # height unchanged
                           ((97, 143), (0, 0, 143, 97), 32)]:        # odd sizes, whole frame
        im = source(rng, h, w, block=4 if h > 200 else 2 if h > 90 else 1)
        x1, y1, cw, ch = box
        out = Image.fromarray(im).crop((x1, y1, x1 + cw, y1 + ch)).resize((d, d), Image.BICUBIC)
        cases.append(("resize", [x1, y1, cw, ch, d], im, to(out)))
    im = source(rng, 32, 32, block=1)
    for name, fn in (("brightness", TF.adjust_brightness), ("contrast", TF.adjust_contrast),
                     ("saturation", TF.adjust_saturation)):
        for f in (0.6, 0.6000000000000001, 1.0, 1.4, 1.3999999999999997, 0.8123, 1.2345):
            cases.append((name, [f], im, to(fn(Image.fromarray(im), f))))
    for f in (-0.1, 0.1, -0.09999, 0.0999, -0.05, 0.03, -0.003, 0.0):
        cases.append(("hue", [f], im, to(TF.adjust_hue(Image.fromarray(im), f))))
    for s in (0.1, 0.3, 1.0, 2.0, 0.7321, 1.618):
        cases.append(("blur", [s], im, to(Image.fromarray(im).filter(ImageFilter.GaussianBlur(radius=s)))))
    gray = A.RandomGray(p=1.0)
    for c in range(3):
        seed = next(s for s in range(100) if np.random.RandomState(s).choice(3) == c)
        np.random.seed(seed)
        cases.append(("gray", [c], im, to(gray.grayscale(Image.fromarray(im)))))
    cases.append(("flip", [], im, to(Image.fromarray(im).transpose(Image.FLIP_LEFT_RIGHT))))
    return cases, im


def chain_cases(rng):
    fns = {"brightness": TF.adjust_brightness, "contrast": TF.adjust_contrast,
           "saturation": TF.adjust_saturation, "hue": TF.adjust_hue}
    orders = [("brightness", "contrast", "saturation", "hue"), ("hue", "contrast", "brightness", "saturation"),
              ("saturation", "hue", "contrast", "brightness"), ("contrast", "saturation", "hue", "brightness"),
              ("hue", "saturation", "brightness", "contrast"), ("brightness", "hue", "saturation", "contrast"),
              ("saturation", "brightness", "hue", "contrast"), ("contrast", "hue", "brightness", "saturation")]
    out = []
    for order in orders:
        f = {"brightness": rng.uniform(0.6, 1.4), "contrast": rng.uniform(0.6, 1.4),
             "saturation": rng.uniform(0.6, 1.4), "hue": rng.uniform(-0.1, 0.1)}
        im = source(rng, 32, 32, block=1)
        pil = Image.fromarray(im)
        for name in order:
            pil = fns[name](pil, f[name])
        out.append((order, [f[n] for n in order], im, np.array(pil)))
    return out


def recipe_cases(A, rng, two_stream, n, seq_len, img_dim, sizes, seed0):
    S = 2 * seq_len if two_stream else seq_len
    tf = get_transform(A, S, img_dim)
    srcs = [source(rng, h, w, 2 * S) for h, w in sizes]
    log = []
    orig_rsc, orig_crop = A.RandomSizedCrop.__call__, Image.Image.crop

    def rsc(self, imgmap):
        boxes = []
        Image.Image.crop = lambda im, box=None: (boxes.append(box), orig_crop(im, box))[1]
        try:
            res = orig_rsc(self, imgmap)
        finally:
            Image.Image.crop = orig_crop
        start = next(i for i, p in enumerate(current) if p is imgmap[0])
        x1, y1, x2, y2 = boxes[0] if boxes else (-1, -1, -2, -2)
        log.append([start, x1, y1, x2 - x1, y2 - y1])
        return res

    A.RandomSizedCrop.__call__ = rsc
    seeds, which, outs, after, clips = [], [], [], [], []
    try:
        for i in range(n):
            s = (seed0 + i, seed0 + 100 + i, seed0 + 200 + i)
            random.seed(s[0]); np.random.seed(s[1]); torch.manual_seed(s[2])
            src = srcs[i % len(srcs)]
            current = [Image.fromarray(f) for f in src]
            del log[:]
            seq = tf(list(current))
            if two_stream:      # lmdb_dataset.py: seq1 = seq[:2T], seq2 = seq[2T:], each stacked along dim 1
                y = torch.stack([torch.stack(seq[:S], 1), torch.stack(seq[S:], 1)])
            else:
                y = torch.stack(seq, 1)
            after.append([random.random(), np.random.random(), float(torch.rand(1))])
            seeds.append(s); which.append(i % len(srcs)); outs.append(as_u8(y)); clips.append(list(log))
            assert len(log) == 2
    finally:
        A.RandomSizedCrop.__call__ = orig_rsc
    return srcs, np.array(seeds), np.array(which), np.stack(outs), np.array(after), np.array(clips, np.int32)


def main():
    assert REF, "set COCLR_REFERENCE to a checkout of the reference"
    A = load_reference_augmentation()
    rng = np.random.default_rng(20261017)
    d = {"versions": np.array(["Pillow " + PIL.__version__, "torchvision " + torchvision.__version__,
                               "numpy " + np.__version__, "torch " + torch.__version__])}
    ops, d["op_img"] = op_cases(A, rng)
    d["op_names"] = np.array([o[0] for o in ops])
    for i, (name, params, src, out) in enumerate(ops):
        d["op%d_params" % i], d["op%d_out" % i] = np.array(params, np.float64), out
        if src is not d["op_img"]:                 # the colour, blur, gray and flip cases all read op_img
            d["op%d_src" % i] = src
    chains = chain_cases(rng)
    d["chain_orders"] = np.array([c[0] for c in chains])
    d["chain_factors"] = np.array([c[1] for c in chains], np.float64)
    d["chain_src"] = np.stack([c[2] for c in chains])
    d["chain_out"] = np.stack([c[3] for c in chains])
    for tag, two, T, D, sizes, seed0 in (("nce", False, 2, 24, [(36, 48), (40, 30), (24, 32), (50, 64)], 1000),
                                         ("coclr", True, 2, 24, [(36, 48), (28, 36), (24, 20), (44, 52)], 5000)):
        srcs, seeds, which, outs, after, clips = recipe_cases(A, rng, two, 16, T, D, sizes, seed0)
        d[tag + "_meta"] = np.array([T, D])
        for j, s in enumerate(srcs):
            d["%s_src%d" % (tag, j)] = s
        d[tag + "_seeds"], d[tag + "_which"], d[tag + "_out"] = seeds, which, outs
        d[tag + "_after"], d[tag + "_clips"] = after, clips
    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
