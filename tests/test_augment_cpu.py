"""The pre-training augmentation's host side (coclr_b200.augment) against the reference's PIL pipeline, without a GPU.

tests/golden/augment.npz comes from the unmodified reference utils/augmentation.py (make_golden_augment.py).  Here:
  * the plan, under each recorded sample's seeds, makes the reference's decisions: the same source half and the same
    crop box (or no crop) for both clips, and leaves `random`, `np.random` and torch's generator where the reference
    left them;
  * the host tables (bicubic coefficients, box-blur weights, hue shift byte), run through the numpy restatement of the
    kernel's arithmetic (tests/tools/augment_oracle.py), give every per-op case, every jitter chain and every
    whole-recipe sample bit for bit;
  * malformed input raises ValueError before anything reaches the device.
"""
import os
import random
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200 import augment as A  # noqa: E402
import augment_oracle as O  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "augment.npz"))
RECIPES = {"nce": False, "coclr": True}


def recipe(tag):
    T, D = (int(v) for v in G[tag + "_meta"])
    aug = A.PretrainAugment(T, D, two_stream=RECIPES[tag])
    srcs = [G["%s_src%d" % (tag, j)] for j in range(int(G[tag + "_which"].max()) + 1)]
    return aug, srcs


def seeded_plan(aug, size, seeds):
    py, npr, gen = random.Random(int(seeds[0])), np.random.RandomState(int(seeds[1])), torch.Generator()
    gen.manual_seed(int(seeds[2]))
    plan = aug.plan([size], py, npr, gen)
    return plan, (py.random(), npr.random_sample(), float(torch.rand(1, generator=gen)))


def op_src(i):
    return G["op%d_src" % i] if ("op%d_src" % i) in G.files else G["op_img"]


@pytest.mark.parametrize("tag", sorted(RECIPES))
def test_plan_decisions_and_draw_order(tag):
    aug, srcs = recipe(tag)
    for i, seeds in enumerate(G[tag + "_seeds"]):
        h, w = srcs[G[tag + "_which"][i]].shape[1:3]
        plan, after = seeded_plan(aug, (h, w), seeds)
        assert after == tuple(G[tag + "_after"][i]), (tag, i)
        for c, rec in zip(plan[0].clips, G[tag + "_clips"][i]):
            assert c.half * aug.S == rec[0], (tag, i)
            assert c.crop == (None if rec[1] < 0 else tuple(int(v) for v in rec[1:])), (tag, i)


def test_plan_defaults_to_global_generators():
    aug, srcs = recipe("nce")
    seeds = G["nce_seeds"][0]
    random.seed(int(seeds[0])); np.random.seed(int(seeds[1])); torch.manual_seed(int(seeds[2]))
    aug.plan([srcs[G["nce_which"][0]].shape[1:3]])
    assert (random.random(), np.random.random(), float(torch.rand(1))) == tuple(G["nce_after"][0])


def test_plan_covers_every_branch():
    """The fixture's samples reach every decision the recipe has, so the comparisons above are not vacuous."""
    seen = set()
    for tag in RECIPES:
        aug, srcs = recipe(tag)
        for i, seeds in enumerate(G[tag + "_seeds"]):
            sp = seeded_plan(aug, srcs[G[tag + "_which"][i]].shape[1:3], seeds)[0][0]
            seen.add("two_clip" if sp.two_clip else "one_clip")
            for c in sp.clips:
                seen |= {k for k, on in (("base", c.base), ("null", not c.base), ("no_crop", c.crop is None),
                                         ("crop", c.crop is not None), ("jitter", c.jitter), ("gray", c.gray),
                                         ("blur", c.blur_sigma is not None), ("flip", c.flip)) if on}
    assert seen == {"two_clip", "one_clip", "base", "null", "no_crop", "crop", "jitter", "gray", "blur", "flip"}, seen


def test_ops_through_host_tables():
    for i, name in enumerate(G["op_names"]):
        p, src, want = G["op%d_params" % i], op_src(i), G["op%d_out" % i]
        if name == "resize":
            x1, y1, w, h, d = (int(v) for v in p)
            got = O.crop_resize(src, (x1, y1, w, h), d)
        elif name == "hue":
            got = O.hue(src, A.hue_shift_byte(float(p[0])))
        elif name == "blur":
            got = O.blur(src, float(p[0]))
        elif name == "gray":
            got = O.gray(src, int(p[0]))
        elif name == "flip":
            got = O.flip(src)
        else:
            got = O.JITTER[name](src, float(p[0]))
        assert np.array_equal(got, want), (i, name, p)


def test_jitter_chains():
    orders = [tuple(o) for o in G["chain_orders"]]
    assert len(set(orders)) >= 6 and any(o.index("hue") < o.index("contrast") for o in orders)
    for order, f, src, want in zip(orders, G["chain_factors"], G["chain_src"], G["chain_out"]):
        ops = [(n, A.hue_shift_byte(v) if n == "hue" else v) for n, v in zip(order, f)]
        assert np.array_equal(O.jitter(src, ops), want), order


@pytest.mark.parametrize("tag", sorted(RECIPES))
def test_whole_recipe_through_plan(tag):
    aug, srcs = recipe(tag)
    for i, seeds in enumerate(G[tag + "_seeds"]):
        src = srcs[G[tag + "_which"][i]]
        plan, _ = seeded_plan(aug, src.shape[1:3], seeds)
        got = O.sample(aug, plan[0], src)                          # [2S, D, D, 3]
        want = G[tag + "_out"][i]
        if aug.two_stream:                                         # [2, 3, S, D, D] -> [2S, D, D, 3]
            want = np.concatenate([want[0], want[1]], axis=1)
        assert np.array_equal(got, want.transpose(1, 2, 3, 0)), (tag, i)
    assert torch.equal(O.to_tensor(np.arange(256, dtype=np.uint8).reshape(1, 1, 256, 1).repeat(3, 3))[0, 0, 0],
                       torch.arange(256, dtype=torch.uint8).float().div(255))


def test_resize_taps_match_pillow_shape_rules():
    for n, d in ((320, 128), (128, 128), (45, 128), (1920, 128), (7, 3)):
        st, cnt, kk = A.resize_taps(n, d)
        assert kk.shape == (int(np.ceil(2 * max(n / d, 1.0))) * 2 + 1, d)
        assert (np.diff(st) >= 0).all() and (np.diff(st + cnt) >= 0).all()
        assert st.min() >= 0 and (st + cnt).max() <= n and (cnt <= kk.shape[0]).all()


def test_validation():
    aug = A.PretrainAugment(2, 24)
    plan = aug.plan([(20, 30), (10, 10)], random.Random(0), np.random.RandomState(0), torch.Generator())
    good = torch.zeros(2, 4, 20, 30, 3, dtype=torch.uint8)
    with pytest.raises(ValueError):
        aug(good.float(), plan)                                     # dtype
    with pytest.raises(ValueError):
        aug(good.permute(0, 1, 4, 2, 3).contiguous(), plan)         # channels first
    with pytest.raises(ValueError):
        aug(good.transpose(2, 3), plan)                             # not contiguous
    with pytest.raises(ValueError):
        aug(torch.zeros(2, 6, 20, 30, 3, dtype=torch.uint8), plan)  # F != 2T
    with pytest.raises(ValueError):
        A.PretrainAugment(2, 24, two_stream=True)(good, plan)      # F != 4T
    with pytest.raises(ValueError):
        aug(good[:, :, :19].contiguous(), plan)                     # a source taller than the buffer
    with pytest.raises(ValueError):
        aug(good[:1].contiguous(), plan)                            # plan for another batch size
    with pytest.raises(ValueError):
        aug(good, plan, sizes=[(20, 30), (10, 11)])                 # sizes other than the plan's
    with pytest.raises(ValueError):
        aug(good, plan)                                             # not on a CUDA device
    with pytest.raises(ValueError):
        aug.plan([(0, 30)])
    with pytest.raises(ValueError):
        A.PretrainAugment(2, 256)                                   # frame does not fit shared memory
