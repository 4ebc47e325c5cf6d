"""JPEG decoding on the GPU (coclr_b200.jpeg, csrc/jpeg.cu) against Pillow, bit for bit:

  * every case of tests/golden/jpeg.npz (Pillow's output of its own encodes), decoded as one mixed batch (sizes,
    samplings, grayscale, restart intervals, optimised and 16-bit tables, a stripped DHT) in two orders;
  * freshly encoded frames against live Pillow, when its libjpeg is the fixture's;
  * a sentinel-filled `out=` is untouched outside each frame's h x w x 3 bytes, also when a small workspace makes the
    call run in passes;
  * a repeat call and a CUDA-graph replay give identical bytes;
  * a frame with corrupted entropy-coded data behind valid headers gets the status the oracle gives it (checked on the
    CPU first), and its neighbours stay exact;
  * decode -> PretrainAugment and decode -> ClassifierAugment equal the same augmentation of Pillow-decoded frames;
  * main_nce.py, main_coclr.py and eval/main_classifier.py train two steps with --synthetic --gpu-augment --jpeg.
"""
import hashlib
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200.jpeg import JpegDecoder  # noqa: E402
import jpeg_cases as JC  # noqa: E402
import jpeg_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(ROOT, "tests", "golden", "jpeg.npz"))
NAMES = [str(n) for n in G["names"]]
RAWS = [G["data"][G["offsets"][i]:G["offsets"][i + 1]].tobytes() for i in range(len(NAMES))]


def _matches_fixture(i, img):
    h, w = (int(v) for v in G["sizes"][i])
    if img.shape != (h, w, 3):
        return False
    if str(G["sha256"][i]):
        return hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest() == str(G["sha256"][i])
    want = G["pixels"][G["pixel_offsets"][i]:G["pixel_offsets"][i + 1]].reshape(h, w, 3)
    return np.array_equal(img, want)


def _frames(out, batch):
    o = out.cpu().numpy()
    return [o[i, :h, :w] for i, (h, w) in enumerate(batch.sizes)]


@pytest.mark.parametrize("order", ["fixture", "shuffled"])
def test_fixture_bit_identical(order):
    idx = list(range(len(NAMES)))
    if order == "shuffled":
        random.Random(7).shuffle(idx)
    dec = JpegDecoder()
    batch = dec.parse([RAWS[i] for i in idx])
    out = dec(batch)
    bad = [NAMES[i] for i, img in zip(idx, _frames(out, batch)) if not _matches_fixture(i, img)]
    assert not bad, bad


def test_live_pillow():
    if features.version("jpg") != str(G["versions"][1]):
        pytest.skip("Pillow's libjpeg %s is not the fixture's %s" % (features.version("jpg"), G["versions"][1]))
    raws = []
    for k, (h, w, ss, q) in enumerate([(240, 320, 2, 75), (240, 320, 2, 90), (241, 323, 1, 60), (99, 131, 0, 85),
                                       (2, 3, 2, 75), (4, 6, 1, 95), (63, 65, 2, 100)]):
        raws.append(JC.encode(JC.field(h, w, 1000 + k, noise=8.0 + 4 * k), quality=q, subsampling=ss))
    raws.append(JC.encode(JC.field(77, 91, 1100, gray=True), quality=70, restart_marker_rows=2))
    dec = JpegDecoder()
    batch = dec.parse(raws)
    got = _frames(dec(batch), batch)
    for k, r in enumerate(raws):
        assert np.array_equal(got[k], JC.pillow_decode(r)), k


def test_out_sentinel_and_passes():
    raws = [RAWS[NAMES.index(n)] for n in ("s420_7x9_q75", "s444_241x323_q75", "gray_33x47", "rst_blocks3_s420_33x47",
                                           "s422_1x1_q75", "q90_s420_240x320")]
    for limit in (1 << 30, 1800 * 128):            # one pass; then a workspace of one 240 x 320 4:2:0 frame
        dec = JpegDecoder(work_limit=limit)
        batch = dec.parse(raws)
        out = torch.full((len(raws), 250, 330, 3), 0xAB, dtype=torch.uint8, device="cuda")
        dec(batch, out=out)
        o = out.cpu().numpy()
        for i, (h, w) in enumerate(batch.sizes):
            assert np.array_equal(o[i, :h, :w], JC.pillow_decode(raws[i])), (limit, i)
            mask = np.ones(o.shape[1:], bool)
            mask[:h, :w] = False
            assert (o[i][mask] == 0xAB).all(), (limit, i)


def test_more_frames_than_one_grid_holds():
    """70000 frames fit the workspace at once, but a pass holds at most 65535 (the grids' y and z limit)."""
    raws = [RAWS[NAMES.index("gray_rst_7x9")], RAWS[NAMES.index("s444_1x1_q75")]] * 35000
    dec = JpegDecoder()
    batch = dec.parse(raws)
    assert batch.work_bytes <= dec.work_limit
    out = dec(batch)
    o = out.cpu().numpy()
    want = [JC.pillow_decode(r) for r in raws[:2]]
    assert (o[0::2, :7, :9] == want[0]).all() and (o[1::2, :1, :1] == want[1]).all()


def test_repeat_and_graph_replay():
    dec = JpegDecoder()
    batch = dec.parse(RAWS)
    first = torch.zeros(len(RAWS), 241, 323, 3, dtype=torch.uint8, device="cuda")
    dec(batch, out=first)
    out = torch.zeros_like(first)
    dec(batch, out=out, check=False)
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    out.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            dec(batch, out=out, check=False)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    out.zero_()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    assert int(dec.graph_status.abs().sum()) == 0
    other = dec.parse([RAWS[i] for i in reversed(range(len(RAWS)))])
    scratch = torch.zeros_like(first)
    dec(other, out=scratch)                         # an eager call between replays leaves the captured batch alone
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first) and not torch.equal(scratch, first)
    with pytest.raises(ValueError, match="already holds a captured decode"):
        with torch.cuda.stream(s):
            with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
                dec(batch, out=out, check=False)


def _corrupt():
    """Two frames with valid headers and broken entropy-coded data: the second half of the segment cut off (the scan
    ends early), and a run of FF 00 (all-one bits: no code of Pillow's tables) in the middle."""
    raw = RAWS[NAMES.index("q90_s420_240x320")]
    p = O.parse(raw)
    b0, b1 = p["ecs"]
    cut = raw[:b0 + (b1 - b0) // 2] + b"\xff\xd9"
    mid = b0 + (b1 - b0) // 3
    ones = raw[:mid] + b"\xff\x00" * 16 + raw[mid + 32:]
    return [cut, ones]


def test_corrupted_frame_status():
    bad = _corrupt()
    want = []
    for r in bad:                                  # the oracle decides the expected status before the GPU sees it
        _, st = O.decode(r)
        assert st != O.ST_OK
        want.append(st)
    good = [RAWS[NAMES.index(n)] for n in ("s420_240x320_q75", "gray_241x323", "rst_rows1_s422_240x320")]
    raws = [good[0], bad[0], good[1], bad[1], good[2]]
    dec = JpegDecoder()
    batch = dec.parse(raws)
    out = dec(batch, check=False)
    st = dec.status.cpu().numpy()
    assert list(st) == [0, want[0], 0, want[1], 0], st
    got = _frames(out, batch)
    for k in (0, 2, 4):
        assert np.array_equal(got[k], JC.pillow_decode(raws[k])), k
    with pytest.raises(ValueError, match="frame 1"):
        dec(batch)


def _restart_corrupt():
    """Two frames with restart markers (one per MCU row) and broken entropy-coded data: 20 bytes cut from the end of
    the fifth interval (it ends before its last block), and the third RSTn renumbered (out of sequence)."""
    import re
    raw = RAWS[NAMES.index("rst_rows1_s422_240x320")]
    ms = [m.start() for m in re.finditer(rb"\xff[\xd0-\xd7]", raw)]
    k = ms[4]
    cut = raw[:k - 20] + raw[k:]
    k = ms[2]
    renumbered = raw[:k + 1] + bytes([0xD0 + ((raw[k + 1] - 0xD0 + 3) & 7)]) + raw[k + 2:]
    return [cut, renumbered]


def test_corrupted_restart_interval_status():
    """A bad restart interval stops the frame's whole warp; its neighbours stay exact."""
    bad = _restart_corrupt()
    want = [O.decode(r)[1] for r in bad]           # the oracle decides the expected statuses first
    assert want == [O.ST_EARLY_END, O.ST_BAD_RESTART]
    good = [RAWS[NAMES.index(n)] for n in ("rst_rows1_s422_240x320", "s420_240x320_q75", "rst_blocks3_s420_33x47")]
    raws = [good[0], bad[0], good[1], bad[1], good[2]]
    dec = JpegDecoder()
    batch = dec.parse(raws)
    out = dec(batch, check=False)
    assert list(dec.status.cpu().numpy()) == [0, want[0], 0, want[1], 0]
    got = _frames(out, batch)
    for k in (0, 2, 4):
        assert np.array_equal(got[k], JC.pillow_decode(raws[k])), k


def _video_jpegs(n, h, w, seed, ss=2):
    return [JC.encode(JC.field(h, w, seed + i), quality=80, subsampling=ss) for i in range(n)]


def test_decode_then_pretrain_augment():
    from coclr_b200.augment import PretrainAugment
    B, T = 2, 4
    aug = PretrainAugment(T, 64)
    raws = _video_jpegs(B * 2 * T, 96, 128, 300)
    dec = JpegDecoder()
    batch = dec.parse(raws)
    frames = dec(batch)
    ref = torch.from_numpy(np.stack([JC.pillow_decode(r) for r in raws])).cuda()
    assert torch.equal(frames, ref)
    plan = aug.plan(batch.sample_sizes(B), random.Random(1), np.random.RandomState(1), torch.Generator().manual_seed(1))
    x = aug(frames.view(B, 2 * T, *frames.shape[1:]), plan)
    y = aug(ref.view(B, 2 * T, *ref.shape[1:]), plan)
    assert torch.equal(x, y)


def test_decode_then_classifier_augment():
    from coclr_b200.clf_augment import ClassifierAugment
    B, T = 2, 4
    aug = ClassifierAugment("train", T, 64)
    raws = _video_jpegs(B * T, 240, 320, 400, ss=1)
    dec = JpegDecoder()
    batch = dec.parse(raws)
    frames = dec(batch)
    ref = torch.from_numpy(np.stack([JC.pillow_decode(r) for r in raws])).cuda()
    assert torch.equal(frames, ref)
    plan = aug.plan(batch.sample_sizes(B), random.Random(2))
    x = aug(frames.view(B, T, *frames.shape[1:]), plan)
    y = aug(ref.view(B, T, *ref.shape[1:]), plan)
    assert torch.equal(x, y)


def _run(cmd, cwd):
    r = subprocess.run([sys.executable] + cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=900, env=dict(os.environ, PYTHONPATH=ROOT))
    assert r.returncode == 0, r.stdout[-4000:]
    losses = [float(l.split("loss ")[1].split()[0]) for l in r.stdout.splitlines() if "loss " in l]
    assert len(losses) >= 2 and all(np.isfinite(losses)), r.stdout[-2000:]


@pytest.mark.parametrize("script", ["main_nce.py", "main_coclr.py"])
def test_pretrain_drivers_with_jpeg(tmp_path, script):
    _run([os.path.join(ROOT, script), "--synthetic", "--gpu-augment", "--jpeg", "--batch_size", "4", "--seq_len", "8",
          "--img_dim", "64", "--moco-k", "16", "--steps-per-epoch", "2", "--print_freq", "1", "--net", "s3d",
          "--epochs", "1", "--source-size", "120", "160"], str(tmp_path))


def test_classifier_driver_with_jpeg(tmp_path):
    _run([os.path.join(ROOT, "eval", "main_classifier.py"), "--synthetic", "--gpu-augment", "--jpeg", "--net", "s3d",
          "--dataset", "hmdb51", "--batch_size", "4", "--seq_len", "8", "--img_dim", "64", "--synthetic-videos", "6",
          "--source-size", "120", "160", "--train_what", "ft", "--epochs", "1", "--steps-per-epoch", "2",
          "--print_freq", "1"], str(tmp_path))
