"""TV-L1 flow databases without a GPU: the float64 oracle (tests/tools/flow_oracle.py) recovers a known translation,
the grey and quantisation references match their formulas and Pillow, the streaming LMDB writer round-trips through
lmdb_read (overflow values, a 3-level tree, both msgpack families) with every page referenced exactly once, and the
flow tool refuses bad arguments."""
import io
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "tools"))
sys.path.insert(0, ROOT)

import flow_oracle as O  # noqa: E402
import lmdb_writer  # noqa: E402
from coclr_b200 import lmdb_read, lmdb_write  # noqa: E402

TOOL = os.path.join(ROOT, "tools", "make_flow_lmdb.py")


def test_oracle_recovers_subpixel_translation():
    d = (0.6, -0.35)
    a, b = O.texture(48, 64, 3), O.texture(48, 64, 3, d)
    flow, iters = O.tvl1(a, b)
    epe = np.hypot(flow[0] - d[0], flow[1] - d[1])[4:-4, 4:-4]
    assert epe.mean() < 0.05 and epe.max() < 0.1, (epe.mean(), epe.max())
    assert iters.shape == (len(O.sizes(48, 64)), O.WARPS) and (iters >= 1).all() and (iters <= O.MAX_ITERS).all()


def test_oracle_identical_frames_give_zero():
    a = O.texture(37, 53, 1)
    flow, iters = O.tvl1(a, a)
    assert np.abs(flow).max() == 0.0 and (iters == 1).all()


def test_pyramid_sizes():
    assert O.sizes(240, 320) == [(240, 320), (120, 160), (60, 80), (30, 40)]
    assert O.sizes(256, 340) == [(256, 340), (128, 170), (64, 85), (32, 43), (16, 22)]
    assert O.sizes(37, 53) == [(37, 53), (19, 27)]
    assert O.sizes(12, 400) == [(12, 400)]
    w, r = O.gaussian_taps()
    assert r == 4 and abs(w.sum() - 1) < 1e-15


def test_quantise_reference_formula():
    f = np.array([-25, -20, -19.99, -0.08, -0.0784, 0, 0.0784, 0.08, 19.9, 20, 31, np.float32(1) / 3],
                 np.float32)
    flow = np.stack([f, -f]).reshape(1, 2, 1, -1)
    q = O.quantise(flow)[0, 0]
    for c, vals in ((0, f), (1, -f)):
        want = [min(255, max(0, int(np.floor((float(np.float32(v)) + 20) * 255 / 40 + 0.5)))) for v in vals]
        assert q[:, c].tolist() == want
    assert (q[:, 2] == 128).all()


def test_grey_reference_matches_formula_and_pillow():
    from PIL import Image
    r = np.random.RandomState(0)
    rgb = r.randint(0, 256, (61, 47, 3)).astype(np.uint8)
    rgb[0, :6] = [[0, 0, 0], [255, 255, 255], [255, 0, 0], [0, 255, 0], [0, 0, 255], [1, 2, 3]]
    g = O.grey(rgb)
    R, G, B = (rgb[..., c].astype(np.int64) for c in range(3))
    assert np.array_equal(g, (19595 * R + 38470 * G + 7471 * B + 0x8000) >> 16)
    assert np.array_equal(g, np.asarray(Image.fromarray(rgb).convert("L")))


# --- the streaming LMDB writer ----------------------------------------------------------------------------------------

def _pages(path, psize):
    """Walk the tree from the current meta page; returns {page number: times referenced} and the file's page count."""
    data = open(path, "rb").read()
    metas = [lmdb_read.META.unpack_from(data, s * psize + lmdb_read.PAGEHDR) for s in (0, 1)]
    m = max(metas, key=lambda m: m[-1])
    root, last = m[19], m[20]
    seen = {}

    def visit(pg):
        seen[pg] = seen.get(pg, 0) + 1
        off = pg * psize
        flags, lower = struct.unpack_from("<HH", data, off + 10)
        ptrs = struct.unpack_from("<%dH" % ((lower - 16) // 2), data, off + 16)
        for p in ptrs:
            lo, hi, nflags, ks = struct.unpack_from("<HHHH", data, off + p)
            if flags & lmdb_read.P_BRANCH:
                visit(lo | hi << 16 | nflags << 32)
            elif nflags & lmdb_read.F_BIGDATA:
                ov = struct.unpack_from("<Q", data, off + p + 8 + ks)[0]
                n = struct.unpack_from("<I", data, ov * psize + 12)[0]
                for q in range(ov, ov + n):
                    seen[q] = seen.get(q, 0) + 1

    if root != lmdb_read.INVALID:
        visit(root)
    assert len(data) == (last + 1) * psize
    return seen, last + 1


@pytest.mark.parametrize("psize", [4096, 512])
def test_writer_round_trip_across_overflow_threshold(tmp_path, psize):
    nodemax = (((psize - 16) // 2) & ~1) - 2
    items = {}
    for i, n in enumerate([0, 1, nodemax - 8 - 9 - 1, nodemax - 8 - 9, nodemax - 8 - 9 + 1, psize - 16, psize - 15,
                           3 * psize, 100000]):
        items[b"%09d" % i] = bytes(np.random.RandomState(i).randint(0, 256, n).astype(np.uint8))
    with lmdb_write.Writer(str(tmp_path / "db"), psize=psize) as w:
        for k in sorted(items):
            w.put(k, items[k])
    db = lmdb_read.open(str(tmp_path / "db"))
    for k, v in items.items():
        assert bytes(db.get(k)) == v, k
    assert db.get(b"000000099") is None and db.entries == len(items)
    seen, npages = _pages(str(tmp_path / "db" / "data.mdb"), psize)
    assert sorted(seen) == list(range(2, npages)) and set(seen.values()) == {1}


def test_writer_three_level_tree_matches_fixture_writer(tmp_path):
    psize = 512
    items = {b"k%07d" % i: b"v" * (i % 50) for i in range(3000)}
    items[b"k0000007"] = b"x" * 2000                                     # one overflow value among them
    with lmdb_write.Writer(str(tmp_path / "new"), psize=psize) as w:
        for k in sorted(items):
            w.put(k, items[k])
    assert w.depth >= 3
    lmdb_writer.write(str(tmp_path / "fixture"), items, psize=psize)
    new, fix = lmdb_read.open(str(tmp_path / "new")), lmdb_read.open(str(tmp_path / "fixture"))
    assert (new.depth, new.entries) == (fix.depth, fix.entries)
    for k, v in items.items():
        assert bytes(new.get(k)) == v == bytes(fix.get(k))
    for k in (b"", b"a", b"k", b"k0000000\x00", b"z"):
        assert new.get(k) is None
    seen, npages = _pages(str(tmp_path / "new" / "data.mdb"), psize)
    assert sorted(seen) == list(range(2, npages)) and set(seen.values()) == {1}


@pytest.mark.parametrize("bin_type", [True, False])
def test_writer_msgpack_families(tmp_path, bin_type):
    frames = [b"", b"\xff\xd8" * 10, bytes(range(256)) * 300]
    value = lmdb_write.pack(frames, bin_type)
    assert value == lmdb_writer.pack(frames, bin_type)
    assert lmdb_write.bin_family(value) is bin_type
    assert lmdb_write.bin_family(lmdb_write.pack([b"000000001"], bin_type)) is bin_type
    assert lmdb_write.bin_family(lmdb_write.pack([], bin_type)) is None
    for obj in (None, True, False, 0, 127, 128, 70000, 1 << 40, -1, -33, -40000, [1, [2, b"x"]]):
        assert lmdb_write.pack(obj, bin_type) == lmdb_writer.pack(obj, bin_type)
    with lmdb_write.Writer(str(tmp_path / "db")) as w:
        w.put(b"000000000", value)
        w.put(b"__vlen__", lmdb_write.pack([3, 0, 70000], bin_type))
    db = lmdb_read.open(str(tmp_path / "db"))
    assert [bytes(f) for f in lmdb_read.unpack(db.get(b"000000000"))] == frames
    assert lmdb_read.unpack(db.get(b"__vlen__")) == [3, 0, 70000]


def test_writer_refuses_out_of_order_keys_and_existing_files(tmp_path):
    w = lmdb_write.Writer(str(tmp_path / "db"))
    w.put(b"b", b"1")
    for k in (b"a", b"b"):
        with pytest.raises(ValueError, match="increasing"):
            w.put(k, b"2")
    with pytest.raises(ValueError, match="key length"):
        w.put(b"", b"2")
    w.put(b"c", b"3")
    w.close()
    db = lmdb_read.open(str(tmp_path / "db"))
    assert bytes(db.get(b"b")) == b"1" and bytes(db.get(b"c")) == b"3"
    with pytest.raises(FileExistsError):
        lmdb_write.Writer(str(tmp_path / "db"))


def test_unfinished_writer_leaves_no_valid_meta(tmp_path):
    w = lmdb_write.Writer(str(tmp_path / "db"))
    w.put(b"a", b"x" * 10000)
    w.abort()
    with pytest.raises(ValueError):
        lmdb_read.open(str(tmp_path / "db"))


def test_empty_database(tmp_path):
    lmdb_write.Writer(str(tmp_path / "db")).close()
    db = lmdb_read.open(str(tmp_path / "db"))
    assert db.get(b"a") is None and db.entries == 0


# --- the tool's arguments ---------------------------------------------------------------------------------------------

def _tool(*args):
    return subprocess.run([sys.executable, TOOL] + list(args), capture_output=True, text=True, cwd=ROOT)


def test_tool_argument_errors(tmp_path):
    r = _tool()
    assert r.returncode == 2 and "--rgb" in r.stderr
    r = _tool("--rgb", str(tmp_path / "missing"), "--out", str(tmp_path / "o"))
    assert r.returncode == 2 and "does not exist" in r.stderr
    rgb = tmp_path / "rgb"
    lmdb_writer.write_videos(str(rgb), {"a/v": [b"x"]}, ["a/v"])
    (tmp_path / "exists").mkdir()
    r = _tool("--rgb", str(rgb), "--out", str(tmp_path / "exists"))
    assert r.returncode == 2 and "exists" in r.stderr
    r = _tool("--rgb", str(rgb), "--out", str(tmp_path / "o"), "--pairs", "0")
    assert r.returncode == 2 and "--pairs" in r.stderr
    assert not (tmp_path / "o").exists()


def test_tool_encode_constants():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_flow_lmdb as M
    from PIL import Image
    frame = np.full((16, 24, 3), 128, np.uint8)
    frame[..., 0] = np.arange(24, dtype=np.uint8) * 10
    b = io.BytesIO()
    Image.fromarray(frame).save(b, "JPEG", quality=95, subsampling=0)
    assert (M.QUALITY, M.SUBSAMPLING) == (95, 0) and M.encode(frame) == b.getvalue()


def test_tool_takes_the_frame_family_from_keys():
    """The reference's converter writes `__order__` as Python str (str family under every msgpack) and the keys and
    frames as bytes (bin under msgpack >= 1.0, str under 0.6.2): the flow frames follow the keys."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_flow_lmdb as M
    order = lmdb_write.pack(["c/v1", "c/v0"])
    assert lmdb_write.bin_family(order) is False
    assert M.frame_family(lmdb_write.pack([b"000000000", b"000000001"], True)) is True
    assert M.frame_family(lmdb_write.pack([b"000000000", b"000000001"], False)) is False
    assert M.frame_family(lmdb_write.pack([], True)) is True
