"""The classifier augmentation kernel (csrc/augment_clf.cu via coclr_b200.clf_augment) against the reference's PIL
transforms of eval/main_classifier.py: every output is compared bit for bit with tests/golden/clf_augment.npz, written by
the unmodified reference utils/augmentation.py under Pillow / torchvision (tests/golden/make_golden_clf_augment.py).

  * per-op cases (crop -> 224 -> D at D = 32, 128, 224, a 224-exact crop, the fallback on a wide, a tall and a 224-high
    frame, CenterCrop with odd margins, every FiveCrop position with both flips), each with its 224 x 224 intermediate
    (the same plan run at img_dim 224), and the jitter chains at both strengths;
  * the whole-recipe samples of train (with and without the batch flip), val, the ten test views and retrieval, in one
    launch per recipe: in order, reversed, one by one, and next to a batch mate of another source size; the test and
    retrieval videos have different lengths in one launch;
  * a CUDA-graph replay equals the eager call;
  * LinearClassifier.set_input_transform gives forward() the engine's fused normalisation;
  * eval/main_classifier.py --synthetic --gpu-augment fine-tunes (ft, last) with validation and runs --test --ten_crop
    and --test --retrieval, writing the reference's files.
"""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200 import clf_augment as CA  # noqa: E402
from coclr_b200.augment import hue_shift_byte  # noqa: E402
import test_clf_augment_cpu as CPU  # noqa: E402

pytestmark = pytest.mark.gpu
G = CPU.G
T, D = CPU.T, CPU.D
DEV = torch.device("cuda", 0)


def u8(t):
    """Kernel output (x / 255 floats) back to the uint8 it encodes, asserting it is exactly such a value."""
    u = torch.round(t * 255).to(torch.uint8)
    assert torch.equal(u.float().div(255), t)
    return u


def run_one(aug, sp, src):
    """One one-frame sample through the kernel: src uint8 [h, w, 3] -> uint8 [D, D, 3] (numpy)."""
    if aug.mode in ("train", "val"):
        frames = torch.from_numpy(np.ascontiguousarray(src)[None, None]).to(DEV)
    else:
        frames = torch.from_numpy(np.ascontiguousarray(src)[None]).to(DEV)
    x = aug(frames, CA.ClfAugmentPlan(aug, [sp]))[0]
    return u8(x[:, 0].permute(1, 2, 0).cpu()).numpy()


def test_ops_bit_identical():
    for i, name in enumerate(G["op_names"]):
        src = CPU.op_src(i)
        aug, sp = CPU.case_plan(str(name), G["op%d_params" % i], src.shape[:2])
        mid, want = CPU.op_images(i, sp)
        assert np.array_equal(run_one(aug, sp, src), want), (i, name)
        if aug.mode == "val":                                      # the intermediate: the same window at 224
            at224 = CA.ClassifierAugment("val", 1, 224)
        else:
            at224 = CA.ClassifierAugment(aug.mode, 1, 224, view=aug.view)
        assert np.array_equal(run_one(at224, sp, src), mid), (i, name)


def test_jitter_chains_bit_identical():
    for order, f, at, want in zip(G["chain_orders"], G["chain_factors"], G["chain_at"], G["chain_out"]):
        src = CPU.window(at)
        ops = [(str(n), float(v)) for n, v in zip(order, f)]
        aug = CA.ClassifierAugment("retrieval", 1, src.shape[0])
        sp = CA.ClfSamplePlan(src.shape[:2], 1, crop=(0, 0, src.shape[1], src.shape[0]), jitter=ops,
                              hue_shift=hue_shift_byte(dict(ops)["hue"]))
        assert np.array_equal(run_one(aug, sp, src), want), tuple(order)


def recipe_run(tag, order, extra=None, batch_flip=False):
    """The recipe's fixture samples in `order` in one launch (sources top-left in a shared buffer), plus optional
    (size, frames) batch mates; returns their uint8 outputs [n, D, D, 3]."""
    aug = CPU.aug_for(tag)
    video = aug.mode in ("test", "retrieval")
    srcs = [CPU.recipe_source(int(G[tag + "_which"][i]))[:int(G[tag + "_len"][i])] for i in order]
    srcs += [f for _, f in (extra or [])]
    Hm, Wm = max(s.shape[1] for s in srcs), max(s.shape[2] for s in srcs)
    samples = []
    for i in order:
        s = G[tag + "_seeds"][i]
        k, n = int(G[tag + "_which"][i]), int(G[tag + "_len"][i])
        samples += aug.plan([CPU.recipe_source(k).shape[1:3]], random.Random(int(s[0])), lengths=[n],
                            batch_flip=batch_flip).samples
    for k in range(len(order), len(srcs)):
        samples += aug.plan([srcs[k].shape[1:3]], random.Random(k), lengths=[srcs[k].shape[0]]).samples
    if video:
        buf = np.zeros((sum(s.shape[0] for s in srcs), Hm, Wm, 3), np.uint8)
        off = 0
        for s in srcs:
            buf[off:off + s.shape[0], :s.shape[1], :s.shape[2]] = s
            off += s.shape[0]
    else:
        buf = np.zeros((len(srcs), aug.frames, Hm, Wm, 3), np.uint8)
        for k, s in enumerate(srcs):
            buf[k, :, :s.shape[1], :s.shape[2]] = s
    out = aug(torch.from_numpy(buf).to(DEV), CA.ClfAugmentPlan(aug, samples))
    out = out if video else list(out)
    return [u8(o.permute(1, 2, 3, 0).cpu()).numpy() for o in out[:len(order)]]


@pytest.mark.parametrize("tag", CPU.TAGS)
def test_recipe_bit_identical_in_any_batch(tag):
    want = CPU.recipe_outputs(tag)
    n = len(want)
    got = recipe_run(tag, list(range(n)))
    for i in range(n):
        assert np.array_equal(got[i], want[i]), (tag, i)
    for i, g in zip(range(n)[::-1], recipe_run(tag, list(range(n))[::-1])):
        assert np.array_equal(g, want[i]), (tag, "reversed", i)
    for i in (0, n - 1):
        assert np.array_equal(recipe_run(tag, [i])[0], want[i]), (tag, "alone", i)
    rng = np.random.default_rng(1)
    big = rng.integers(0, 256, (T, 480, 641, 3), dtype=np.uint8)
    mates = recipe_run(tag, [n - 1, 0], extra=[((480, 641), big)])
    assert np.array_equal(mates[0], want[n - 1]) and np.array_equal(mates[1], want[0]), tag


def test_train_batch_flip_bit_identical():
    n = len(G["train_seeds"])
    got = recipe_run("train", list(range(n)), batch_flip=True)
    want = CPU.recipe_outputs("train")
    for i in range(n):
        assert np.array_equal(got[i], want[i][:, :, ::-1]), i


@pytest.mark.parametrize("mode", ["train", "test"])
def test_graph_replay_equals_eager(mode):
    g = torch.Generator(device=DEV).manual_seed(0)
    sizes = [(240, 320), (300, 227), (224, 500), (256, 256)]
    if mode == "train":
        aug = CA.ClassifierAugment("train", 4, 64)
        frames = torch.randint(0, 256, (4, 4, 300, 500, 3), dtype=torch.uint8, device=DEV, generator=g)
        plan = aug.plan(sizes, random.Random(7), batch_flip=True)
        call = lambda: aug(frames, plan)                                   # noqa: E731
    else:
        aug = CA.ClassifierAugment("test", 4, 64, view=(2, 1))
        frames = torch.randint(0, 256, (5 + 9 + 1 + 4, 300, 500, 3), dtype=torch.uint8, device=DEV, generator=g)
        plan = aug.plan(sizes, random.Random(7), lengths=[5, 9, 1, 4])
        call = lambda: torch.cat([v.reshape(-1) for v in aug(frames, plan)])   # noqa: E731
    eager = call()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()                                    # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = call()
    captured.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured, eager)


def test_set_input_transform_fuses_normalisation():
    from model.classifier import LinearClassifier
    import classifier_oracle as CO
    m = LinearClassifier(num_class=51, network="s3d", use_dropout=False, use_final_bn=True, use_l2_norm=True)
    m.load_state_dict(CO.classifier_state("s3d", 51, False, True, seed=4), strict=False)
    m = m.to(DEV).eval()
    x = torch.rand(2, 3, 8, 64, 64, device=DEV)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    norm = (torch.tensor(mean, device=DEV), torch.tensor(std, device=DEV))
    with torch.no_grad():
        plain = torch.cat(m(x), 1)
        m.set_input_transform(mean, std)
        fused = torch.cat(m(x), 1)
        want = torch.cat(m.infer(x, norm=norm), 1)
        torch_norm = torch.cat(m.infer((x - norm[0].view(1, 3, 1, 1, 1)) / norm[1].view(1, 3, 1, 1, 1)), 1)
        m.set_input_transform(None)
        assert torch.equal(torch.cat(m(x), 1), plain)
    assert float(torch_norm.abs().max()) > 0
    assert torch.equal(fused, want)
    assert float((fused - torch_norm).abs().max()) <= 1e-4 * float(torch_norm.abs().max())
    assert float((fused - plain).abs().max()) > 1e-3 * float(torch_norm.abs().max())


def _cli(cwd, *extra):
    cmd = [sys.executable, os.path.join(ROOT, "eval", "main_classifier.py"), "--synthetic", "--gpu-augment",
           "--net", "s3d", "--dataset", "hmdb51", "--batch_size", "4", "--seq_len", "8", "--img_dim", "64",
           "--synthetic-videos", "6", "--source-size", "240", "320"] + list(extra)
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


@pytest.mark.parametrize("what", ["ft", "last"])
def test_cli_finetune_with_gpu_augment(tmp_path, what):
    out = _cli(str(tmp_path), "--train_what", what, "--epochs", "1", "--steps-per-epoch", "4", "--print_freq", "1")
    losses = [float(l.split("loss ")[1].split()[0]) for l in out.splitlines() if "loss " in l]
    assert len(losses) >= 4 and all(np.isfinite(losses)), out[-2000:]
    assert "Epoch: [0]\tLoss:" in out and "finished" in out
    best = [os.path.join(dp, f) for dp, _, fs in os.walk(str(tmp_path)) for f in fs if f == "model_best.pth.tar"]
    epoch = [os.path.join(dp, f) for dp, _, fs in os.walk(str(tmp_path)) for f in fs if f == "epoch0.pth.tar"]
    assert len(epoch) == 1 and len(best) <= 1


def _checkpoint(tmp_path):
    from model.classifier import LinearClassifier
    torch.manual_seed(0)
    m = LinearClassifier(num_class=51, network="s3d", use_dropout=False, use_final_bn=True, use_l2_norm=True)
    path = os.path.join(str(tmp_path), "model", "epoch2.pth.tar")
    os.makedirs(os.path.dirname(path))
    torch.save({"epoch": 2, "state_dict": m.state_dict()}, path)
    return path


def test_cli_ten_crop_with_gpu_augment(tmp_path):
    path = _checkpoint(tmp_path)
    out = _cli(str(tmp_path), "--test", path, "--ten_crop")
    assert out.count("Aug type:") == 10 and "Test using 10 crop" in out
    for t in ("center", "five", "ten"):
        with open(path + "-prob-%s.json" % t) as fp:
            stat = json.load(fp)
        assert len(stat) == 6 and all(len(v["mean_prob"][0]) == 51 for v in stat.values())


def test_cli_retrieval_with_gpu_augment(tmp_path):
    path = _checkpoint(tmp_path)
    out = _cli(str(tmp_path), "--test", path, "--retrieval")
    assert "Computing test set feature" in out and "Computing train set feature" in out
    d = os.path.join(os.path.dirname(path), "feature")
    for split in ("test", "train"):
        f = torch.load(os.path.join(d, "hmdb51_%s_feature.pth.tar" % split))
        assert f.shape == (6, 1024) and bool(torch.isfinite(f).all())
        assert os.path.exists(os.path.join(d, "hmdb51_%s_vname.pkl" % split))
    assert torch.load(os.path.join(d, "hmdb51_sim.pth.tar")).shape == (6, 6)
    assert len([l for l in out.splitlines() if "NN acc = " in l]) == 5
