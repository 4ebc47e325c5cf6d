"""Host side of the classifier augmentation (coclr_b200.clf_augment) against tests/golden/clf_augment.npz, written by the
unmodified reference utils/augmentation.py under Pillow / torchvision (tests/golden/make_golden_clf_augment.py):

  * the plans' decisions and draw counts: every recipe sample's crop box (or fallback window), and the first draw of
    random, np.random and torch after it (so the plan draws from `random` exactly as the reference, and from nothing
    else);
  * the fallback windows of Scale(224) + CenterCrop(224), FiveCrop's boxes and the round-half-even offsets;
  * the numpy restatement of the kernel's arithmetic (tests/tools/clf_augment_oracle.py: the two resizes through the
    host tables, jitter, flip) against every fixture output, intermediates included;
  * the ValueErrors of malformed plans and inputs.
"""
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200 import clf_augment as CA  # noqa: E402
from coclr_b200.augment import hue_shift_byte  # noqa: E402
import augment_oracle as AO  # noqa: E402
import clf_augment_oracle as O  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "clf_augment.npz"))
T, D = (int(v) for v in G["meta"])
TAGS = ["train", "val"] + ["test%d%d" % (a, f) for f in (0, 1) for a in (5, 1, 2, 3, 4)] + ["retrieval"]


def aug_for(tag, d=D):
    if tag.startswith("test"):
        return CA.ClassifierAugment("test", T, d, view=(int(tag[4]), int(tag[5])))
    return CA.ClassifierAugment(tag, T, d)


def window(at):
    """A source: the window (y, x, h, w) of the fixture's base image."""
    y, x, h, w = (int(v) for v in at)
    return np.ascontiguousarray(G["base"][y:y + h, x:x + w])


def recipe_source(k):
    """Recipe source k, uint8 [3, h, w, 3]: frame t is its window moved src_step * t down and right."""
    y, x, h, w = (int(v) for v in G["src_at"][k])
    dy, dx = (int(v) for v in G["src_step"])
    return np.stack([window((y + dy * t, x + dx * t, h, w)) for t in range(3)])


def recipe_outputs(tag):
    """The fixture's per-sample uint8 outputs [n, D, D, 3]."""
    out, off = [], 0
    for n in G[tag + "_len"]:
        k = 3 * int(n) * D * D
        out.append(G[tag + "_out"][off:off + k].reshape(3, int(n), D, D).transpose(1, 2, 3, 0))
        off += k
    return out


def seeded_plan(tag, i, py_rng=None):
    """Seeds the three generators as the fixture did for sample i and draws its plan (from `random` itself unless
    py_rng is given)."""
    s = G[tag + "_seeds"][i]
    random.seed(int(s[0])); np.random.seed(int(s[1])); torch.manual_seed(int(s[2]))
    k, n = int(G[tag + "_which"][i]), int(G[tag + "_len"][i])
    src = recipe_source(k)
    return aug_for(tag).plan([src.shape[1:3]], py_rng, lengths=[n]), src[:n]


def expected_box(sp):
    """The first Image.crop of the reference call, as [x1, y1, x2, y2, w, h] of the image it cropped."""
    h, w = sp.size
    if sp.fallback is not None:
        sh, sw, y1, x1 = sp.fallback
        return [x1, y1, x1 + 224, y1 + 224, sw, sh]
    x1, y1, cw, ch = sp.crop
    return [x1, y1, x1 + cw, y1 + ch, w, h]


@pytest.mark.parametrize("tag", TAGS)
def test_plan_decisions_and_draws(tag):
    for i in range(len(G[tag + "_seeds"])):
        plan, _ = seeded_plan(tag, i)
        sp = plan[0]
        assert expected_box(sp) == list(G[tag + "_box"][i]), (tag, i)
        after = [random.random(), np.random.random(), float(torch.rand(1))]
        assert after == list(G[tag + "_after"][i]), (tag, i)     # random drawn as the reference; np / torch untouched
        assert sp.src_flip == (tag.startswith("test") and tag[5] == "1")
        assert not sp.flip
        if tag == "val":
            assert sp.jitter is None


def test_plan_uses_the_given_generator_only():
    random.seed(12345); np.random.seed(1); torch.manual_seed(1)
    before = (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state())
    plan = aug_for("train").plan([(240, 320)] * 4, random.Random(99), batch_flip=True)
    assert random.getstate() == before[0] and np.array_equal(np.random.get_state()[1], before[1])
    assert torch.equal(torch.get_rng_state(), before[2])
    random.seed(99)
    ref = aug_for("train").plan([(240, 320)] * 4)
    for a, b in zip(plan, ref):
        assert (a.crop, a.fallback, a.jitter, a.attempts) == (b.crop, b.fallback, b.jitter, b.attempts)
        assert a.flip and not b.flip


def test_jitter_draws_at_both_strengths():
    """ColorJitter(p=.3): one random(), then four uniforms in b, c, s, h order and a shuffle."""
    for mode, (lo, hi) in (("train", (0.6, 1.4)), ("retrieval", (0.8, 1.2))):
        aug = CA.ClassifierAugment(mode, 1, 32)
        hits = 0
        for seed in range(100):
            r, ref = random.Random(seed), random.Random(seed)
            sp = aug.plan([(240, 320)], r)[0]
            if mode == "train":                          # RandomSizedCrop's draws come first
                CA.ClassifierAugment._random_sized_crop(CA.ClfSamplePlan((240, 320), 1), ref)
            else:
                assert sp.crop == (48, 8, 224, 224)
            if ref.random() < 0.3:
                f = [ref.uniform(lo, hi), ref.uniform(lo, hi), ref.uniform(lo, hi), ref.uniform(-0.1, 0.1)]
                ops = list(zip(("brightness", "contrast", "saturation", "hue"), f))
                ref.shuffle(ops)
                assert sp.jitter == ops and sp.hue_shift == hue_shift_byte(f[3])
                hits += 1
            else:
                assert sp.jitter is None
            assert r.random() == ref.random()
        assert 10 < hits < 60


def test_fallback_windows_and_offsets():
    assert CA.center_offset(321) == 48 and CA.center_offset(323) == 50      # 48.5 -> 48, 49.5 -> 50: half to even
    assert CA.center_offset(227) == 2 and CA.center_offset(229) == 2 and CA.center_offset(224) == 0
    assert CA.scale_size(240, 320) == (224, 298)                             # int(224 * 320 / 240)
    assert CA.scale_size(600, 240) == (560, 224)
    assert CA.scale_size(224, 500) == (224, 500)                             # shorter side already 224: no resize
    assert CA.scale_size(300, 300) == (224, 224)
    for where, box in ((1, (0, 0)), (2, (101, 0)), (3, (0, 19)), (4, (101, 19)), (5, (50, 10))):
        assert CA.five_crop_box(243, 325, where) == box + (224, 224)
    for i, name in enumerate(G["op_names"]):
        if name == "fallback":
            seed, d = (int(v) for v in G["op%d_params" % i])
            src = op_src(i)
            sp = CA.ClassifierAugment("val", 1, d).plan([src.shape[:2]], random.Random(seed))[0]
            sh, sw, y1, x1 = sp.fallback
            assert sp.crop is None and sp.attempts == 10
            assert (sh, sw) == CA.scale_size(*src.shape[:2]) and (y1, x1) == (CA.center_offset(sh), CA.center_offset(sw))


def test_small_frames_raise():
    with pytest.raises(ValueError):
        CA.ClassifierAugment("test", 2, 32, view=(1, 0)).plan([(223, 400)])
    with pytest.raises(ValueError):
        CA.ClassifierAugment("retrieval", 2, 32).plan([(300, 200)])
    with pytest.raises(ValueError):
        CA.ClassifierAugment("test", 2, 32, view=(6, 0))
    with pytest.raises(ValueError):
        CA.ClassifierAugment("val", 2, 32).plan([(240, 320)], batch_flip=True)
    with pytest.raises(ValueError):
        CA.ClassifierAugment("train", 2, 32).plan([(240, 320)], lengths=[3])


def test_call_validates_before_launch():
    aug = CA.ClassifierAugment("train", 2, 32)
    plan = aug.plan([(240, 320)] * 2, random.Random(0))
    ok = torch.zeros(2, 2, 240, 320, 3, dtype=torch.uint8)
    for bad in (ok.float(), ok[..., :2], ok[:1], torch.zeros(2, 3, 240, 320, 3, dtype=torch.uint8),
                torch.zeros(2, 2, 200, 320, 3, dtype=torch.uint8), ok.transpose(2, 3)):
        with pytest.raises(ValueError):
            aug(bad, plan)
    with pytest.raises(ValueError):
        CA.ClassifierAugment("val", 2, 32)(ok, plan)
    with pytest.raises(ValueError):
        aug(ok, plan)                                    # a CPU tensor
    vid = CA.ClassifierAugment("retrieval", 2, 32)
    vplan = vid.plan([(240, 320)] * 2, random.Random(0), lengths=[3, 2])
    with pytest.raises(ValueError):
        vid(torch.zeros(6, 240, 320, 3, dtype=torch.uint8), vplan)   # 5 frames expected


def case_plan(name, p, src_hw):
    """A hand-built plan for a per-op case: (aug, sample plan)."""
    if name == "crop":
        x1, y1, cw, ch, d = (int(v) for v in p)
        return CA.ClassifierAugment("val", 1, d), CA.ClfSamplePlan(src_hw, 1, crop=(x1, y1, cw, ch))
    if name == "fallback":
        seed, d = (int(v) for v in p)
        aug = CA.ClassifierAugment("val", 1, d)
        return aug, aug.plan([src_hw], random.Random(seed))[0]
    if name == "center":
        aug = CA.ClassifierAugment("retrieval", 1, int(p[0]))
        h, w = src_hw
        return aug, CA.ClfSamplePlan(src_hw, 1, crop=(CA.center_offset(w), CA.center_offset(h), 224, 224))
    where, flip, d = (int(v) for v in p)
    aug = CA.ClassifierAugment("test", 1, d, view=(where, flip))
    return aug, CA.ClfSamplePlan(src_hw, 1, crop=CA.five_crop_box(*src_hw, where), src_flip=bool(flip))


def op_src(i):
    return window(G["op_src"][i])


def op_images(i, sp):
    """(the 224 x 224 intermediate, the output) of per-op case i.  An intermediate the fixture does not store is the
    window the reference cut (op_box, in the flipped frame for a flipped view); the plan must name the same box."""
    want = G["img%d" % G["op_out"][i]]
    if G["op_mid"][i] >= 0:
        return G["img%d" % G["op_mid"][i]], want
    x1, y1, x2, y2 = (int(v) for v in G["op_box"][i])
    assert sp.crop == (x1, y1, x2 - x1, y2 - y1), (i, sp.crop)
    src = op_src(i)[:, ::-1] if sp.src_flip else op_src(i)
    return np.ascontiguousarray(src[y1:y2, x1:x2]), want


def test_op_cases_through_the_oracle():
    for i, name in enumerate(G["op_names"]):
        src = op_src(i)
        aug, sp = case_plan(str(name), G["op%d_params" % i], src.shape[:2])
        mid, want = op_images(i, sp)
        first = O.first_resize(aug, sp, src)
        if aug.M == 224:
            assert np.array_equal(first, mid), (i, name)               # the 224 x 224 intermediate
            assert np.array_equal(AO.resize(first, aug.img_dim), want), (i, name)
        else:                                                          # one resize, straight to img_dim
            assert np.array_equal(first, want), (i, name)
            crop = CA.ClassifierAugment("retrieval", 1, 224)          # the 224 window itself: identity taps
            assert np.array_equal(O.first_resize(crop, sp, src), mid), (i, name)


def test_jitter_chains_through_the_oracle():
    for order, f, at, want in zip(G["chain_orders"], G["chain_factors"], G["chain_at"], G["chain_out"]):
        src = window(at)
        ops = [(str(n), float(v)) for n, v in zip(order, f)]
        got = AO.jitter(src, [(n, hue_shift_byte(v) if n == "hue" else v) for n, v in ops])
        assert np.array_equal(got, want), tuple(order)


@pytest.mark.parametrize("tag", ["train", "val", "test50", "test21", "test41", "retrieval"])
def test_recipes_through_the_oracle(tag):
    want = recipe_outputs(tag)
    for i in range(len(want)):
        plan, src = seeded_plan(tag, i)
        assert np.array_equal(O.sample(plan.aug, plan[0], src), want[i]), (tag, i)


def test_train_batch_flip():
    """utils/transforms.RandomHorizontalFlip in the main process: random() < .5 per batch (the fixture's generator
    asserts that a flip mirrors the tensor)."""
    fl = [bool(f) for f in G["train_flip"]]
    assert any(fl) and not all(fl)
    for seed, f in zip(G["train_flip_seeds"], fl):
        assert (random.Random(int(seed)).random() < 0.5) == f
