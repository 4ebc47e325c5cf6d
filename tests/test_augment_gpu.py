"""The pre-training augmentation kernel (csrc/augment.cu via coclr_b200.augment) against the reference's PIL pipeline:
every output is compared bit for bit with tests/golden/augment.npz, written by the unmodified reference
utils/augmentation.py under Pillow / torchvision (tests/golden/make_golden_augment.py).

  * per-op cases (crop + resize, brightness, contrast, saturation, hue, blur, gray, flip) and the jitter chains, each
    run as a one-frame clip whose other steps are off;
  * the 16 whole-recipe samples of main_nce.py and of main_coclr.py (two streams), in one batch of mixed source sizes,
    also reversed, one by one, and next to a 720 x 540 batch mate: a sample's bits depend on nothing else;
  * a source taller than one resize band (the horizontal pass runs in several bands), against the numpy restatement;
  * a CUDA-graph replay equals the eager call;
  * main_nce.py and main_coclr.py train a few steps with --gpu-augment.
"""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200 import augment as A  # noqa: E402
import augment_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(ROOT, "tests", "golden", "augment.npz"))
DEV = torch.device("cuda", 0)


def as_float(u8):
    return torch.from_numpy(np.ascontiguousarray(u8)).float().div(255)


def run_clip(src, clip, d):
    """One clip of one frame through the kernel: src uint8 [h, w, 3] -> [d, d, 3] uint8-valued float / 255."""
    aug = A.PretrainAugment(1, d)
    h, w = src.shape[:2]
    frames = torch.from_numpy(np.stack([src, src])[None]).to(DEV)
    other = A.ClipPlan(half=1, base=False, crop=None)
    plan = A.AugmentPlan(aug, [A.SamplePlan(True, (h, w), [clip, other])])
    out = aug(frames, plan)
    return out[0, :, 0].permute(1, 2, 0).cpu()


def op_src(i):
    return G["op%d_src" % i] if ("op%d_src" % i) in G.files else G["op_img"]


def test_ops_bit_identical():
    for i, name in enumerate(G["op_names"]):
        p, src, want = G["op%d_params" % i], op_src(i), G["op%d_out" % i]
        c = A.ClipPlan(half=0, base=True, crop=None)
        d = src.shape[0]
        if name == "resize":
            x1, y1, w, h, d = (int(v) for v in p)
            c.crop = (x1, y1, w, h)
        elif name == "hue":
            c.jitter, c.hue_shift = [("hue", float(p[0]))], A.hue_shift_byte(float(p[0]))
        elif name == "blur":
            c.blur_sigma = float(p[0])
        elif name == "gray":
            c.gray = [int(p[0])]
        elif name == "flip":
            c.flip = True
        else:
            c.jitter = [(str(name), float(p[0]))]
        assert torch.equal(run_clip(src, c, d), as_float(want)), (i, name, p)


def test_jitter_chains_bit_identical():
    for order, f, src, want in zip(G["chain_orders"], G["chain_factors"], G["chain_src"], G["chain_out"]):
        ops = [(str(n), float(v)) for n, v in zip(order, f)]
        c = A.ClipPlan(half=0, base=True, crop=None, jitter=ops, hue_shift=A.hue_shift_byte(dict(ops)["hue"]))
        assert torch.equal(run_clip(src, c, src.shape[0]), as_float(want)), tuple(order)


def recipe_batch(tag, order, extra=None):
    """The recipe's fixture samples in `order` as one batch (sources top-left in a shared buffer), plus optional
    (size, frames) batch mates appended; returns the per-sample outputs in the fixture's layout."""
    T, D = (int(v) for v in G[tag + "_meta"])
    two = tag == "coclr"
    aug = A.PretrainAugment(T, D, two_stream=two)
    srcs = [G["%s_src%d" % (tag, G[tag + "_which"][i])] for i in order] + [f for _, f in (extra or [])]
    Hm, Wm = max(s.shape[1] for s in srcs), max(s.shape[2] for s in srcs)
    buf = np.zeros((len(srcs), aug.frames, Hm, Wm, 3), np.uint8)
    for k, s in enumerate(srcs):
        buf[k, :, :s.shape[1], :s.shape[2]] = s
    samples = []
    for i in order:
        s = G[tag + "_seeds"][i]
        gen = torch.Generator().manual_seed(int(s[2]))
        plan = aug.plan([srcs[len(samples)].shape[1:3]], random.Random(int(s[0])), np.random.RandomState(int(s[1])), gen)
        samples += plan.samples
    for k in range(len(order), len(srcs)):
        samples += aug.plan([srcs[k].shape[1:3]], random.Random(k), np.random.RandomState(k), torch.Generator()).samples
    out = aug(torch.from_numpy(buf).to(DEV), A.AugmentPlan(aug, samples))
    if two:
        out = torch.stack(out, 1)                 # [B, 2, 3, S, D, D], the fixture's per-sample [2, 3, S, D, D]
    return out.cpu()[:len(order)]


@pytest.mark.parametrize("tag", ["nce", "coclr"])
def test_recipe_bit_identical_in_any_batch(tag):
    n = len(G[tag + "_seeds"])
    want = as_float(G[tag + "_out"])
    got = recipe_batch(tag, list(range(n)))
    for i in range(n):
        assert torch.equal(got[i], want[i]), (tag, i)
    assert torch.equal(recipe_batch(tag, list(range(n))[::-1]), want.flip(0))
    for i in (0, n - 1):
        assert torch.equal(recipe_batch(tag, [i])[0], want[i])
    rng = np.random.default_rng(1)
    F = (4 if tag == "coclr" else 2) * int(G[tag + "_meta"][0])
    big = rng.integers(0, 256, (F, 720, 540, 3), dtype=np.uint8)
    assert torch.equal(recipe_batch(tag, [3, 5], extra=[((720, 540), big)]), want[[3, 5]])


def test_tall_source_in_bands():
    """A 720-row source resized whole to 128 needs several horizontal-pass bands (at most band_rows rows each)."""
    rng = np.random.default_rng(2)
    y, x = np.mgrid[0:720, 0:540]
    src = np.stack([128 + 100 * np.sin(x / 17.0 + c) * np.cos(y / 23.0) for c in range(3)], -1)
    src = np.clip(src + rng.integers(-20, 21, src.shape), 0, 255).astype(np.uint8)
    assert A.PretrainAugment.band_rows(128) < 720
    for crop in (None, (31, 7, 400, 650)):
        c = A.ClipPlan(half=0, base=True, crop=crop, blur_sigma=1.3, flip=True)
        want = O.flip(O.blur(O.crop_resize(src, crop, 128), 1.3))
        assert torch.equal(run_clip(src, c, 128), as_float(want)), crop


def test_graph_replay_equals_eager():
    aug = A.PretrainAugment(4, 64)
    g = torch.Generator(device=DEV).manual_seed(0)
    frames = torch.randint(0, 256, (6, 8, 120, 160, 3), dtype=torch.uint8, device=DEV, generator=g)
    plan = aug.plan([(120, 160), (100, 150), (120, 97), (64, 64), (33, 160), (120, 160)],
                    random.Random(7), np.random.RandomState(7), torch.Generator().manual_seed(7))
    eager = aug(frames, plan)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        aug(frames, plan)                         # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = aug(frames, plan)
    captured.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)


def _run(script, args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, script)] + args, cwd=cwd, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


@pytest.mark.parametrize("script", ["main_nce.py", "main_coclr.py"])
def test_drivers_train_with_gpu_augment(tmp_path, script):
    args = ["--synthetic", "--gpu-augment", "--batch_size", "4", "--seq_len", "8", "--img_dim", "64", "--moco-k", "16",
            "--steps-per-epoch", "5", "--print_freq", "1", "--net", "s3d", "--epochs", "1", "--source-size", "120", "160"]
    out = _run(script, args, str(tmp_path))
    losses = [float(l.split("loss ")[1].split()[0]) for l in out.splitlines() if "loss " in l]
    assert "finished" in out and len(losses) >= 5 and all(np.isfinite(losses)), out[-2000:]
