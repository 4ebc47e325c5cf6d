"""Writes tests/golden/clf_augment.npz by running the UNMODIFIED reference utils/augmentation.py and utils/transforms.py
($COCLR_REFERENCE) under Pillow / torchvision: the transforms of eval/main_classifier.py.

The reference's Scale tests `collections.Iterable`, which Python 3.10 moved to collections.abc; the alias is set
before the module is loaded (its code is run as it is).  Every output is stored as uint8; the stored bytes / 255 in
float32 are asserted here to be the reference's ToTensor output bit for bit.  Sources are at least 224 on each side.

Every source is a window of one stored image `base` (uint8 [480, 480, 3], smooth colour fields plus noise on 8 x 8
cells): `op_src` / `chain_at` / `src_at` give (y, x, h, w) of each, and frame t of recipe source k starts `src_step`
* t further down and right.  Arrays that are equal are stored once, in the pool `img<j>`.

  op_*      one resize chain on one frame (source window `op_src[i]`), with its 224 x 224 intermediate and output
            (indices `op_mid[i]`, `op_out[i]` into the pool).  An intermediate that is a plain window of the source
            (FiveCrop, CenterCrop, a 224-exact box) is not stored (`op_mid[i]` = -1): the reference's crop box is,
            as `op_box[i]` ([x1, y1, x2, y2] in the flipped frame for a flipped view).
              crop  -> resize 224 -> Scale(D), D in 32, 128, 224, and a 224-exact box      (params x1, y1, w, h, D)
              fallback: RandomSizedCrop(224, consistent=True) seeded to miss 10 times, on a wide, a tall and a
              224-high frame, then Scale(D)                                                 (params seed, D)
              center: CenterCrop(224) with odd margins, then Scale((D, D))                  (params D)
              five:   RandomHorizontalFlip(command) -> FiveCrop(224, where) -> Scale((D, D)) (params where, flip, D)
  chain_*   ColorJitter chains (torchvision's functional ops, as the reference's Lambdas call them) at the test
            strength (.2) and the train strength (.4), 8 orders each, on 32 x 32 windows
  train_*, val_*, test<a><f>_*, retrieval_*   whole recipes (seq_len 2, img_dim 32): per sample the random seed, the
            source index, the length, the output, the first draw of random / np.random / torch after the call, and
            the first Image.crop box of the call with the size of the image it cropped ([x1, y1, x2, y2, w, h]).  Train
            samples also hold the batch flip decision of utils/transforms.RandomHorizontalFlip (seed
            `train_flip_seeds`), whose output is asserted here to be the stored output mirrored.

Run in the build container only:  COCLR_REFERENCE=<checkout> python tests/golden/make_golden_clf_augment.py
"""
import collections
import collections.abc
import importlib.util
import os
import random
import sys

import numpy as np
import PIL
import torch
import torchvision
from PIL import Image
import torchvision.transforms.functional as TF
from torchvision import transforms

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402
from make_golden_augment import as_u8, source  # noqa: E402

OUT = os.path.join(HERE, "clf_augment.npz")
T, D = 2, 32                                   # recipe samples: seq_len, img_dim
BASE = 480                                     # side of the image every source is a window of
SRC_AT = [(0, 0, 240, 320), (40, 60, 256, 341), (100, 200, 300, 227)]   # recipe sources (y, x, h, w)
SRC_STEP = (7, 11)                             # frame t of a recipe source is its window moved down 7t, right 11t
VIEWS = [(a, f) for f in (0, 1) for a in (5, 1, 2, 3, 4)]


def window(base, at):
    y, x, h, w = at
    return np.ascontiguousarray(base[y:y + h, x:x + w])


def recipe_source(base, k, frames=3):
    y, x, h, w = SRC_AT[k]
    return np.stack([window(base, (y + SRC_STEP[0] * t, x + SRC_STEP[1] * t, h, w)) for t in range(frames)])


def load(rel, name):
    collections.Iterable = collections.abc.Iterable
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, *rel.split("/")))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def pil(frames):
    return [Image.fromarray(f) for f in frames]


def np_frames(imgs):
    return np.stack([np.array(i) for i in imgs])


def fallback_seed(A, h, w, start):
    """First seed from `start` at which RandomSizedCrop(224, consistent=True) misses all 10 attempts on h x w."""
    im = [Image.new("RGB", (w, h))]
    for s in range(start, start + 100000):
        random.seed(s)
        r = random.Random(s)
        r.random()
        hit = False
        for _ in range(10):
            area = w * h
            ta = r.uniform(0.2, 1) * area
            ar = r.uniform(3. / 4, 4. / 3)
            cw, ch = int(round((ta * ar) ** .5)), int(round((ta / ar) ** .5))
            if r.random() < 0.5:
                cw, ch = ch, cw
            if cw <= w and ch <= h:
                hit = True
                break
        if not hit:
            random.seed(s)
            assert A.RandomSizedCrop(size=224, consistent=True, bottom_area=0.2)(im)[0].size == (224, 224)
            return s
    raise RuntimeError("no fallback seed")


def recorded_crop(fn):
    """Runs fn() and returns (its result, the box of its first Image.crop call)."""
    orig, boxes = Image.Image.crop, []
    Image.Image.crop = lambda im, box=None: (boxes.append(tuple(box)), orig(im, box))[1]
    try:
        return fn(), boxes[0] if boxes else None
    finally:
        Image.Image.crop = orig


def op_cases(A, base):
    cases = []     # (name, params, source window, mid, out, crop box of the reference)
    for at, box, d in [((0, 0, 240, 320), (37, 11, 250, 201), 32), ((0, 0, 240, 320), (37, 11, 250, 201), 128),
                       ((0, 0, 240, 320), (37, 11, 250, 201), 224), ((13, 17, 240, 320), (60, 5, 131, 149), 64),
                       ((31, 40, 240, 320), (41, 9, 224, 224), 48)]:
        im = Image.fromarray(window(base, at))
        x1, y1, cw, ch = box
        mid = im.crop((x1, y1, x1 + cw, y1 + ch)).resize((224, 224), Image.BICUBIC)   # RandomSizedCrop's resize
        out = A.Scale(d)([mid])[0]
        cases.append(("crop", [x1, y1, cw, ch, d], at, np.array(mid), np.array(out), (x1, y1, x1 + cw, y1 + ch)))
    for at, d in [((0, 0, 240, 480), 64), ((0, 0, 480, 240), 32), ((50, 0, 224, 480), 48)]:
        im = Image.fromarray(window(base, at))
        s = fallback_seed(A, at[2], at[3], 0)
        random.seed(s)
        mid, box = recorded_crop(lambda: A.RandomSizedCrop(size=224, consistent=True, bottom_area=0.2)([im])[0])
        out = A.Scale(d)([mid])[0]
        cases.append(("fallback", [s, d], at, np.array(mid), np.array(out), box))
    for at, d in [((5, 9, 240, 321), 32), ((100, 50, 227, 300), 64)]:
        im = Image.fromarray(window(base, at))
        mid, box = recorded_crop(lambda: A.CenterCrop(size=(224, 224))([im])[0])
        out = A.Scale(size=(d, d))([mid])[0]
        cases.append(("center", [d], at, np.array(mid), np.array(out), box))
    at = (200, 100, 243, 325)
    im = Image.fromarray(window(base, at))
    for flip in (0, 1):
        for where in (1, 2, 3, 4, 5):
            random.seed(where)
            f = A.RandomHorizontalFlip(command='right' if flip else 'left')([im])
            mid, box = recorded_crop(lambda: A.FiveCrop(size=(224, 224), where=where)(f)[0])
            out = A.Scale(size=(D, D))([mid])[0]
            cases.append(("five", [where, flip, D], at, np.array(mid), np.array(out), box))
    return cases


def chain_cases(rng, base):
    fns = {"brightness": TF.adjust_brightness, "contrast": TF.adjust_contrast,
           "saturation": TF.adjust_saturation, "hue": TF.adjust_hue}
    orders = [("brightness", "contrast", "saturation", "hue"), ("hue", "contrast", "brightness", "saturation"),
              ("saturation", "hue", "contrast", "brightness"), ("contrast", "saturation", "hue", "brightness"),
              ("hue", "saturation", "brightness", "contrast"), ("brightness", "hue", "saturation", "contrast"),
              ("saturation", "brightness", "hue", "contrast"), ("contrast", "hue", "brightness", "saturation")]
    out = []
    for v in (0.2, 0.4):
        for j, order in enumerate(orders):
            f = {"brightness": rng.uniform(1 - v, 1 + v), "contrast": rng.uniform(1 - v, 1 + v),
                 "saturation": rng.uniform(1 - v, 1 + v), "hue": rng.uniform(-0.1, 0.1)}
            at = (int(rng.integers(0, BASE - 32)), int(rng.integers(0, BASE - 32)), 32, 32)
            im = window(base, at)
            p = Image.fromarray(im)
            for name in order:
                p = fns[name](p, f[name])
            out.append((v, order, [f[n] for n in order], at, np.array(p)))
    return out


def recipe(A, Tt, mode, view=None):
    """The reference's transform of `mode` (eval/main_classifier.py get_transform, test_10crop, test_retrieval)."""
    if mode == "train":
        return transforms.Compose([A.RandomSizedCrop(size=224, consistent=True, bottom_area=0.2), A.Scale(D),
                                   A.ColorJitter(0.4, 0.4, 0.4, 0.1, p=0.3, consistent=True), A.ToTensor()])
    if mode == "val":
        return transforms.Compose([A.RandomSizedCrop(size=224, consistent=True, bottom_area=0.2), A.Scale(D),
                                   A.ToTensor()])
    if mode == "test":
        aug_idx, flip_idx = view
        return transforms.Compose([A.RandomHorizontalFlip(command='left' if flip_idx == 0 else 'right'),
                                   A.FiveCrop(size=(224, 224), where=aug_idx), A.Scale(size=(D, D)),
                                   A.ColorJitter(0.2, 0.2, 0.2, 0.1, p=0.3, consistent=True), A.ToTensor()])
    return transforms.Compose([A.CenterCrop(size=(224, 224)), A.Scale(size=(D, D)),
                               A.ColorJitter(0.2, 0.2, 0.2, 0.1, p=0.3, consistent=True), A.ToTensor()])


def recipe_cases(A, srcs, mode, n, seed0, lengths, view=None):
    tf = recipe(A, T, mode, view)
    orig_crop = Image.Image.crop
    seeds, which, lens, outs, after, boxes = [], [], [], [], [], []
    for i in range(n):
        s = (seed0 + i, seed0 + 100 + i, seed0 + 200 + i)
        random.seed(s[0]); np.random.seed(s[1]); torch.manual_seed(s[2])
        k, L = i % len(srcs), lengths[i % len(lengths)]
        log = []

        def crop(im, box=None):
            log.append(list(box) + list(im.size))
            return orig_crop(im, box)
        Image.Image.crop = crop
        try:
            seq = tf(pil(srcs[k][:L]))
        finally:
            Image.Image.crop = orig_crop
        y = torch.stack(seq, 1)                        # the dataset's stack along dim 1: [3, L, D, D]
        after.append([random.random(), np.random.random(), float(torch.rand(1))])
        seeds.append(s); which.append(k); lens.append(L); outs.append(as_u8(y).reshape(-1)); boxes.append(log[0])
    return (np.array(seeds), np.array(which), np.array(lens), np.concatenate(outs), np.array(after),
            np.array(boxes, np.int32))


def main():
    assert REF, "set COCLR_REFERENCE to a checkout of the reference"
    A = load("utils/augmentation.py", "reference_augmentation")
    Tt = load("utils/transforms.py", "reference_transforms")
    rng = np.random.default_rng(20261018)
    d = {"versions": np.array(["Pillow " + PIL.__version__, "torchvision " + torchvision.__version__,
                               "numpy " + np.__version__, "torch " + torch.__version__])}
    base = source(rng, BASE, BASE, block=8)
    d["base"] = base
    pool = []

    def put(a):
        for j, b in enumerate(pool):
            if b.shape == a.shape and np.array_equal(b, a):
                return j
        pool.append(a)
        return len(pool) - 1

    ops = op_cases(A, base)
    d["op_names"] = np.array([o[0] for o in ops])
    d["op_src"] = np.array([o[2] for o in ops], np.int64)
    d["op_box"] = np.array([o[5] for o in ops], np.int64)
    op_mid, op_out = [], []
    for i, (name, params, at, mid, out, box) in enumerate(ops):
        d["op%d_params" % i] = np.array(params, np.int64)
        src = window(base, at)
        if params[1:2] == [1] and name == "five":
            src = src[:, ::-1]
        x1, y1, x2, y2 = box
        plain = name in ("center", "five") or (name == "crop" and params[2:4] == [224, 224])
        if plain:                                  # the intermediate is the window the reference cut
            assert np.array_equal(mid, src[y1:y2, x1:x2]), (i, name)
        op_mid.append(-1 if plain else put(mid))
        op_out.append(put(out))
    d["op_mid"], d["op_out"] = np.array(op_mid), np.array(op_out)
    for j, a in enumerate(pool):
        d["img%d" % j] = a
    chains = chain_cases(rng, base)
    d["chain_strength"] = np.array([c[0] for c in chains])
    d["chain_orders"] = np.array([c[1] for c in chains])
    d["chain_factors"] = np.array([c[2] for c in chains], np.float64)
    d["chain_at"] = np.array([c[3] for c in chains], np.int64)
    d["chain_out"] = np.stack([c[4] for c in chains])
    srcs = [recipe_source(base, k) for k in range(len(SRC_AT))]
    d["src_at"], d["src_step"] = np.array(SRC_AT, np.int64), np.array(SRC_STEP, np.int64)
    d["meta"] = np.array([T, D])
    tags = [("train", "train", None, 6, 1000, [T]), ("val", "val", None, 4, 2000, [T])]
    tags += [("test%d%d" % v, "test", v, 3, 3000 + 10 * j, [2, 1, 1]) for j, v in enumerate(VIEWS)]
    tags += [("retrieval", "retrieval", None, 3, 4000, [1, 2, 1])]
    for tag, mode, view, n, seed0, lengths in tags:
        seeds, which, lens, out, after, boxes = recipe_cases(A, srcs, mode, n, seed0, lengths, view)
        d[tag + "_seeds"], d[tag + "_which"], d[tag + "_len"], d[tag + "_out"] = seeds, which, lens, out
        d[tag + "_after"], d[tag + "_box"] = after, boxes
    # the train batch flip (utils/transforms.RandomHorizontalFlip in the main process) of each train sample
    fl, fseeds = [], []
    out = torch.from_numpy(d["train_out"]).float().div(255).view(len(d["train_seeds"]), 3, T, D, D)
    for i in range(out.shape[0]):
        random.seed(7000 + i)
        y = Tt.RandomHorizontalFlip()(out[i:i + 1])
        flipped = not torch.equal(y, out[i:i + 1])
        assert torch.equal(y, out[i:i + 1].flip(-1) if flipped else out[i:i + 1])
        fseeds.append(7000 + i); fl.append(int(flipped))
    assert 0 < sum(fl) < len(fl)
    d["train_flip_seeds"], d["train_flip"] = np.array(fseeds), np.array(fl)
    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
