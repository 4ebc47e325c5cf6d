"""Repeated-frame decoding and the LMDB batch loaders on the H100: a slot decode is bit-identical to decoding the
expanded frame list, the loaders reproduce the reference's transformed batches and test views
(tests/golden/datasets.npz) bit for bit,
and the three drivers train and test from a fixture database through --data-root / --split-root."""
import glob
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "tools"))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, ROOT)

import dataset_fixture as F  # noqa: E402
from coclr_b200 import datasets as D  # noqa: E402
from coclr_b200 import loaders as LD  # noqa: E402
from coclr_b200.jpeg import JpegDecoder  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "datasets.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def dirs(tmp_path_factory, golden):
    jpegs = F.pool_from_arrays(golden["pool_data"], golden["pool_off"])
    return F.write(str(tmp_path_factory.mktemp("fixture")), F.spec(), jpegs)


def _slots(n_distinct, n_out, seed):
    r = np.random.RandomState(seed)
    owner = np.concatenate([np.arange(n_distinct), r.randint(0, n_distinct, n_out - n_distinct)])
    perm = r.permutation(n_out)
    slots = [[] for _ in range(n_distinct)]
    for o, j in zip(perm, owner):
        slots[j].append(int(o))
    expanded = [None] * n_out
    for j, s in enumerate(slots):
        for o in s:
            expanded[o] = j
    return slots, expanded


def test_slot_decode_matches_expanded(golden):
    jpegs = F.pool_from_arrays(golden["pool_data"], golden["pool_off"])[:20]
    torch.cuda.set_device(0)
    slots, expanded = _slots(len(jpegs), 57, 0)
    dec = JpegDecoder()
    want = dec(dec.parse([jpegs[j] for j in expanded]))
    batch = dec.parse(jpegs)
    got = dec(batch, slots=slots)
    assert torch.equal(got, want)
    assert batch.sample_sizes(3, slots) == [(F.H, F.W)] * 3
    small = JpegDecoder(work_limit=int(batch.frames["blocks"].max()) * 128 * 3)     # several passes
    assert torch.equal(small(batch, slots=slots), want)
    out = torch.zeros(57, F.H + 3, F.W + 5, 3, dtype=torch.uint8, device="cuda")
    dec(batch, out=out, slots=slots)
    assert torch.equal(out[:, :F.H, :F.W], want) and int(out[:, F.H:].max()) == 0
    with pytest.raises(ValueError, match="exactly once"):
        dec(batch, slots=[[0]] + slots[1:])
    with pytest.raises(ValueError, match="entries"):
        dec(batch, slots=slots[1:])


def test_slot_decode_under_graph_capture(golden):
    jpegs = F.pool_from_arrays(golden["pool_data"], golden["pool_off"])[:12]
    slots, expanded = _slots(len(jpegs), 30, 1)
    dec = JpegDecoder()
    batch = dec.parse(jpegs)
    want = dec(batch, slots=slots)
    out = torch.zeros_like(want)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            dec(batch, out=out, check=False, slots=slots)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want) and int(dec.graph_status.abs().sum()) == 0


def _loader(case, dirs, golden):
    import make_golden_datasets as G
    idx = golden["idx_" + case].tolist()
    name = {"nce": "UCF101LMDB_2CLIP", "coclr": "UCF101_2STREAM_LMDB_2CLIP", "clf": "UCF101LMDB"}[case]
    kw = G.class_kwargs(name, dirs[0], dirs[1], "train", 1)
    kw["return_label"] = True
    ds = getattr(D, name)(**kw)
    dev = torch.device("cuda")
    if case == "clf":
        import make_golden_clf_augment as CA
        ld = LD.ClassifierBatches(ds, len(idx), G.NF, CA.D, dev, seed=G.TRANSFORM_SEED, mode="train")
        ld.order = lambda: idx
    else:
        ld = LD.PretrainBatches(ds, len(idx), G.NF, G.IMG, dev, seed=G.TRANSFORM_SEED, two_stream=case == "coclr")
        ld.order = idx
    return ld


@pytest.mark.parametrize("case", ["nce", "coclr", "clf"])
def test_loader_matches_reference(case, dirs, golden):
    ld = _loader(case, dirs, golden)
    if case == "clf":
        import random
        random.seed(0)
        flip = random.random() < 0.5
        random.seed(0)
    it = iter(ld)
    x, y = next(it)
    it.close()
    want = torch.from_numpy(golden["out_" + case])
    if case == "coclr":
        x = torch.stack(list(x))
    if case == "clf" and flip:
        want = want.flip(-1)                         # the train batch's flip, drawn from `random` per batch
    assert torch.equal(x.cpu(), want)
    assert y.cpu().tolist() == golden["target_" + case].tolist()
    assert not [t for t in threading.enumerate() if t.name == "coclr-lmdb-prefetch"]


@pytest.mark.parametrize("case,chunk", [("test50", 8), ("test21", 2)])
def test_test_videos_match_reference(case, chunk, dirs, golden):
    """TestVideos (the --test loader) against test_10crop's transform of the reference's mode-'test' dataset: the
    half-overlap windows, the per-video lengths of a chunked plan, the slots across videos and the flip / five-crop
    of the view, bit for bit."""
    import make_golden_clf_augment as CA
    import make_golden_datasets as G
    view = dict((c, v) for c, v, _ in G.TEST_VIEWS)[case]
    kw = G.class_kwargs("UCF101LMDB", dirs[0], dirs[1], "test", 1)
    ds = D.UCF101LMDB(return_label=True, **kw)
    ds.video_subset = [ds.video_subset[i] for i in golden["idx_" + case].tolist()]
    tv = LD.TestVideos(ds, G.NF, CA.D, torch.device("cuda"), seed=G.TRANSFORM_SEED, view=view, chunk=chunk)
    got = list(tv)
    assert [v.shape[1] for v, _, _ in got] == golden["len_" + case].tolist()
    assert [label for _, label, _ in got] == golden["target_" + case].tolist()
    assert [vname for _, _, vname in got] == [r[0] for r in ds.video_subset]
    want = torch.from_numpy(golden["out_" + case]).float().div(255)
    assert torch.equal(torch.cat([v for v, _, _ in got], 1).cpu(), want)


def test_loader_threads_stop_on_close(dirs, golden):
    ld = _loader("nce", dirs, golden)
    ld.order = list(range(len(ld.ds))) * 4
    it = iter(ld)
    next(it)
    assert [t for t in threading.enumerate() if t.name == "coclr-lmdb-prefetch"]
    ld.close()
    assert not [t for t in threading.enumerate() if t.name == "coclr-lmdb-prefetch"]


def _run(script, args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, script)] + args, cwd=cwd, env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_drivers_end_to_end(tmp_path, dirs):
    data = ["--data-root", dirs[0], "--split-root", dirs[1]]
    small = data + ["--batch_size", "2", "--seq_len", "8", "--img_dim", "64", "--print_freq", "1", "--epochs", "1"]
    out = _run("main_nce.py", small + ["--dataset", "ucf101-2clip", "--moco-k", "16"], str(tmp_path))
    assert "Training from ep 0 to ep 1 finished" in out and "[0][1/2]" in out and "nan" not in out.lower()
    out = _run("main_coclr.py", small + ["--dataset", "ucf101-2stream-2clip", "--moco-k", "16"], str(tmp_path))
    assert "finished" in out and "[0][1/2]" in out
    out = _run("eval/main_classifier.py", small + ["--dataset", "ucf101", "--train_what", "ft"], str(tmp_path))
    assert "Training from ep 0 to ep 1 finished" in out
    ck = glob.glob(str(tmp_path / "log-eval-linclr" / "*" / "model" / "epoch0.pth.tar"))
    assert len(ck) == 1
    _run("eval/main_classifier.py", data + ["--dataset", "ucf101", "--seq_len", "8", "--img_dim", "64", "--test", ck[0],
                                            "--ten_crop", "--batch_size", "2"], str(tmp_path))
    ds = D.UCF101LMDB(root=os.path.join(dirs[1], "ucf101"), db_path=os.path.join(dirs[0], F.RGB), mode="test",
                      num_frames=8)
    paths = [r[0] for r in ds.video_subset]
    for title in ("center", "five", "ten"):
        with open(os.path.join(os.path.dirname(ck[0]), "epoch0.pth.tar-prob-%s.json" % title)) as f:
            assert sorted(json.load(f)) == sorted(paths)
    _run("eval/main_classifier.py", data + ["--dataset", "ucf101", "--seq_len", "8", "--img_dim", "64", "--test", ck[0],
                                            "--retrieval", "--batch_size", "2"], str(tmp_path))
    assert glob.glob(os.path.join(os.path.dirname(ck[0]), "feature", "ucf101_test_feature.pth.tar"))
