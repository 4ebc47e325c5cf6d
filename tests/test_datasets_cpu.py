"""The LMDB reader, the msgpack subset, the reference's datasets (against tests/golden/datasets.npz) and the batch
dedupe, on the CPU."""
import json
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))

import dataset_fixture as F  # noqa: E402
import lmdb_writer as W  # noqa: E402
from coclr_b200 import datasets as D  # noqa: E402
from coclr_b200 import lmdb_read as R  # noqa: E402
from coclr_b200.loaders import dedupe  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "datasets.npz")


def _items(n, vsize=lambda i: i % 13, klen=9):
    rng = np.random.RandomState(n)
    return {(b"%0*d" % (klen, i)): rng.bytes(vsize(i)) for i in range(n)}


def _check(db, items):
    for k, v in items.items():
        assert bytes(db.get(k)) == v
    assert db.get(b"missing") is None and db.get(b"") is None and db.get(b"\xff" * 12) is None


def test_single_leaf(tmp_path):
    items = _items(20)
    db = R.open(W.write(str(tmp_path / "a"), items) and str(tmp_path / "a"))
    assert db.depth == 1 and db.entries == 20
    _check(db, items)


def test_three_levels(tmp_path):
    items = _items(21000, klen=64)
    db = R.open(W.write(str(tmp_path / "a"), items))
    assert db.depth >= 3
    _check(db, items)


def test_overflow_values_and_page_sizes(tmp_path):
    items = _items(40, vsize=lambda i: 3 + 997 * i)                      # up to ~39 KB: many overflow pages
    for psize in (1024, 4096, 16384):
        path = W.write(str(tmp_path / ("f%d" % psize)), items, psize=psize, subdir=False)
        assert os.path.isfile(path)
        db = R.open(path)                                                # the file layout (subdir=False)
        assert db.psize == psize
        _check(db, items)


def test_stale_meta_ignored(tmp_path):
    items = _items(50)
    db = R.open(W.write(str(tmp_path / "a"), items, stale_meta=True, stale_root=99999))
    _check(db, items)


def test_meta_page_bytes(tmp_path):
    """A hand-assembled environment: meta pages at the documented offsets, one leaf page."""
    ps = 4096
    buf = bytearray(3 * ps)
    for slot, txnid in ((0, 5), (1, 4)):
        o = slot * ps
        struct.pack_into("<QHHHH", buf, o, slot, 0, 0x08, 0, 0)
        struct.pack_into("<IIQQ", buf, o + 16, 0xBEEFC0DE, 1, 0, 3 * ps)
        struct.pack_into("<IHHQQQQQ", buf, o + 40, ps, 0, 0, 0, 0, 0, 0, 2 ** 64 - 1)           # dbs[0]
        struct.pack_into("<IHHQQQQQ", buf, o + 88, 0, 0, 1, 0, 1, 0, 1, 2 if txnid == 5 else 2 ** 64 - 1)
        struct.pack_into("<QQ", buf, o + 136, 2, txnid)
    o = 2 * ps
    node = struct.pack("<HHHH", 5, 0, 0, 3) + b"key" + b"value"
    upper = ps - len(node)
    struct.pack_into("<QHHHH", buf, o, 2, 0, 0x02, 18, upper)
    struct.pack_into("<H", buf, o + 16, upper)
    buf[o + upper:o + ps] = node
    p = tmp_path / "data.mdb"
    p.write_bytes(bytes(buf))
    db = R.open(str(tmp_path))                                          # a directory means path/data.mdb
    assert bytes(db.get(b"key")) == b"value" and db.get(b"kex") is None
    # the same bytes from the writer
    ref = bytes(open(W.write(str(tmp_path / "w"), {b"key": b"value"}), "rb").read())
    assert ref[2 * ps:] == bytes(buf[2 * ps:])


def test_rejections(tmp_path):
    path = W.write(str(tmp_path / "a"), _items(300, vsize=lambda i: 2000), subdir=False)
    data = open(path, "rb").read()
    cut = tmp_path / "cut"
    cut.write_bytes(data[:len(data) - 4096 - 100])
    with pytest.raises(ValueError, match="cut"):
        db = R.open(str(cut))
        for k in _items(300):
            db.get(k)
    bad = bytearray(data)
    struct.pack_into("<I", bad, 16, 0x12345678)
    (tmp_path / "magic").write_bytes(bytes(bad))
    with pytest.raises(ValueError, match="magic"):
        R.open(str(tmp_path / "magic"))
    (tmp_path / "tiny").write_bytes(b"\0" * 10)
    with pytest.raises(ValueError, match="tiny"):
        R.open(str(tmp_path / "tiny"))
    sub = W.write(str(tmp_path / "s"), {b"a": b"x" * 48, b"b": b"y"}, node_flags={b"a": 0x02})
    db = R.open(sub)
    assert bytes(db.get(b"b")) == b"y"
    with pytest.raises(ValueError, match="sub-databases"):
        db.get(b"a")


def _norm(x):
    if isinstance(x, list):
        return [_norm(y) for y in x]
    return bytes(x) if isinstance(x, memoryview) else x


@pytest.mark.parametrize("bin_type", [False, True])
def test_unpack_against_msgpack(bin_type):
    msgpack = pytest.importorskip("msgpack")
    frames = [bytes([i]) * (i * 37) for i in range(40)] + [b"x" * 70000]
    values = [frames, [b"%09d" % i for i in range(20)], 20, 0, 127, 128, 70000, 2 ** 33, -1, -33, -200, -40000,
              -2 ** 40, [b"Apply Eye/v_ApplyEye_g01_c01", b"k"], list(range(300)), [None, True, False]]
    for v in values:
        packed = msgpack.packb(v, use_bin_type=bin_type)
        assert W.pack(v, bin_type) == packed
        got = R.unpack(packed)
        if not bin_type:                                   # str8, which the old raw spec never writes
            assert bytes(R.unpack(b"\xd9\x03abc")) == b"abc"
        assert _norm(got) == v


def test_unpack_rejects_truncated():
    with pytest.raises(ValueError):
        R.unpack(W.pack([b"abc" * 100])[:-5])


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def fixture_dirs(tmp_path_factory, golden):
    jpegs = F.pool_from_arrays(golden["pool_data"], golden["pool_off"])
    return F.write(str(tmp_path_factory.mktemp("fixture")), F.spec(), jpegs, bin_type=False)


def _make(name, mode, ds, window, dirs):
    import make_golden_datasets as G
    kw = G.class_kwargs(name, dirs[0], dirs[1], mode, ds)
    if window:
        kw["window"] = True
    return getattr(D, name)(**kw)


def _cases():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_datasets as G
    return G.cases()


@pytest.mark.parametrize("case", _cases(), ids=lambda c: "%s-%s-ds%d%s" % (c[0], c[1], c[2], "-window" * c[3]))
def test_subsets_and_samplers(case, golden, fixture_dirs):
    import make_golden_datasets as G
    key = G.case_key(*case)
    d = _make(*case, fixture_dirs)
    assert [list(r) for r in d.video_subset] == json.loads(str(golden["subsets"]))[key]
    d.rng = np.random.RandomState(G.SAMPLE_SEED)
    want = json.loads(str(golden["samples"]))[key]
    assert len(d) == len(want)
    for i in range(len(d)):
        out = d[i]
        frames = out[0] if isinstance(out, tuple) else out
        assert len(frames) == len(want[i]) * len(d.dbs)
    d.rng = np.random.RandomState(G.SAMPLE_SEED)
    assert [d.sample(i).tolist() for i in range(len(d))] == want


def test_item_contents(golden, fixture_dirs):
    """__getitem__ returns the sampled JPEGs in transform order, with the reference's label / source id."""
    jpegs = F.pool_from_arrays(golden["pool_data"], golden["pool_off"])
    sp = F.spec()
    d = _make("UCF101_2STREAM_LMDB_2CLIP", "train", 1, False, fixture_dirs)
    d.rng = np.random.RandomState(0)
    frames, source, label = d[2]
    d.rng = np.random.RandomState(0)
    fi = d.sample(2)
    vname = d.video_subset[2][3]
    rgb = [jpegs[i] for i in sp["dbs"][F.RGB]["videos"][vname]]
    flow = [jpegs[i] for i in sp["dbs"][F.FLOW]["videos"][vname]]
    T = 4
    want = [rgb[f] for f in fi[:T]] + [flow[f] for f in fi[:T]] + [rgb[f] for f in fi[T:]] + [flow[f] for f in fi[T:]]
    assert [bytes(f) for f in frames] == want
    assert label == d.classes.index(d.video_subset[2][2])
    assert source == json.loads(sp["files"]["ucf101/video_source.json"])[vname.split("/")[-1][:-4]]


def test_dedupe_plans(fixture_dirs):
    d = _make("UCF101LMDB", "test", 1, False, fixture_dirs)
    refs = []
    for i in range(len(d)):
        refs += d.refs(i, d.sample(i))
    distinct, slots = dedupe(refs)
    assert sorted(o for s in slots for o in s) == list(range(len(refs)))
    assert len(distinct) == len(set(refs)) < len(refs)
    for r, s in zip(distinct, slots):
        assert all(refs[o] == r for o in s)


def _jpeg(h, w, progressive=False):
    import io
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.full((h, w, 3), 90, np.uint8)).save(b, "JPEG", quality=75, progressive=progressive)
    return b.getvalue()


def test_loader_host_rejects_mixed_sizes_and_bad_frames(tmp_path):
    """A video whose sampled frames differ in size, or with a frame the decoder rejects, raises ValueError naming the
    video (the transform is drawn from the first frame's size; nothing is cropped from unwritten memory)."""
    import torch
    from coclr_b200.loaders import ClassifierBatches
    split = tmp_path / "split"
    split.mkdir()
    (split / "ClassInd.txt").write_text("1, A\n")
    (split / "test_split01.csv").write_text("/d/A/v_A_g01_c01/,8\n/d/A/v_A_g02_c01/,8\n/d/A/v_A_g03_c01/,8\n")
    a, b = _jpeg(224, 240), _jpeg(224, 256)
    videos = {"A/v_A_g01_c01": [a, b] * 4, "A/v_A_g02_c01": [a] * 7 + [_jpeg(224, 240, progressive=True)],
              "A/v_A_g03_c01": [a] * 8}
    db = str(tmp_path / "db.lmdb")
    W.write_videos(db, videos, sorted(videos))
    ds = D.UCF101LMDB(root=str(split), db_path=db, mode="test", num_frames=8)
    ld = ClassifierBatches(ds, 1, 8, 32, torch.device("cpu"), seed=0, mode="val")
    plan_one = lambda hw, n: ld.aug.plan([hw], ld.py).samples[0]              # noqa: E731
    with pytest.raises(ValueError, match="v_A_g01_c01: its sampled frames differ in size"):
        ld._host([0], plan_one)
    with pytest.raises(ValueError, match="db.lmdb: video A/v_A_g02_c01 frame 7: progressive$"):
        ld._host([1], plan_one)
    batch, slots, samples, counts = ld._host([2], plan_one)
    assert len(batch) == 8 and slots == [[o] for o in range(8)] and counts == [8]


def test_retrieval_reads_split_one(fixture_dirs):
    """test_retrieval reads split 1 whatever --which_split says, with num_seq * seq_len frames; test_10crop reads
    --which_split."""
    import torch
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "eval"))
    import main_classifier as MC
    args = MC.parse_args(["--data-root", fixture_dirs[0], "--split-root", fixture_dirs[1], "--which_split", "2",
                          "--seq_len", "4", "--dataset", "ucf101"])
    cpu = torch.device("cpu")
    for mode, want in (("retrieval", 1), ("test", 2)):
        for split in ("test", "train"):
            tv = MC.test_videos(args, split, cpu, mode=mode)
            assert tv.ds.which_split == want and tv.ds.num_frames == 4
            assert tv.ds.mode == ("test" if split == "test" else "train")
