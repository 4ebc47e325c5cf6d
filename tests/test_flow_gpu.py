"""TV-L1 flow on the H100 (coclr_b200.flow) against the float64 oracle (tests/tools/flow_oracle.py): the grey
conversion bit for bit against Pillow, each solver stage at odd sizes, full solves, translation recovery, bit-identical
results in any batch or chunking, the quantisation bit for bit against numpy, and the flow database tool end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "tools"))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, ROOT)

import flow_oracle as O  # noqa: E402
from coclr_b200 import flow  # noqa: E402

pytestmark = pytest.mark.gpu
SIZES = [(37, 53), (61, 47)]


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _smooth_flow(P, h, w, seed, amp):
    """Seeded smooth flows [P, 2, h, w] of magnitude up to about amp px."""
    r = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.zeros((P, 2, h, w))
    for p in range(P):
        for c in range(2):
            fx, fy, ph = r.uniform(8, 30), r.uniform(8, 30), r.uniform(0, 6.3)
            out[p, c] = amp * np.sin(x / fx + ph) * np.cos(y / fy) + r.uniform(-amp / 2, amp / 2)
    return out.astype(np.float32)


def _pairs(P, h, w, seed, max_shift=1.5):
    """P texture pairs, each a translation by its own seeded sub-pixel shift; float32 [P, h, w] x 2 and the shifts."""
    r = np.random.RandomState(seed)
    shifts = r.uniform(-max_shift, max_shift, (P, 2))
    i0 = np.stack([O.texture(h, w, seed * 1000 + p) for p in range(P)]).astype(np.float32)
    i1 = np.stack([O.texture(h, w, seed * 1000 + p, tuple(shifts[p])) for p in range(P)]).astype(np.float32)
    return i0, i1, shifts


def test_grey_matches_pillow():
    from PIL import Image
    r = np.random.RandomState(0)
    rgb = r.randint(0, 256, (5, 37, 53, 3)).astype(np.uint8)
    big = torch.zeros(5, 40, 60, 3, dtype=torch.uint8, device="cuda")
    big[:, :37, :53] = torch.from_numpy(rgb).cuda()
    for src in (torch.from_numpy(rgb).cuda(), big[:, :37, :53]):       # packed, and strided rows / frames
        g = flow.grey(src).cpu().numpy()
        assert g.dtype == np.float32 and g.shape == (5, 37, 53)
        for i in range(5):
            assert np.array_equal(g[i], np.asarray(Image.fromarray(rgb[i]).convert("L"), np.float32))


@pytest.mark.parametrize("h,w", SIZES)
def test_zoom_out_matches_oracle(h, w, diag):
    x = np.stack([O.texture(h, w, s) for s in range(3)]).astype(np.float32)
    hc, wc = O.sizes(h, w)[1]
    got = flow.zoom_out(torch.from_numpy(x).cuda(), hc, wc).cpu().numpy()
    err = max(_rel(got[p], O.zoom_out(x[p].astype(np.float64), hc, wc)) for p in range(3))
    diag["flow/zoom_out/%dx%d" % (h, w)] = err
    assert err < 1e-5, err


@pytest.mark.parametrize("h,w", SIZES)
def test_zoom_in_matches_oracle(h, w, diag):
    hc, wc = O.sizes(h, w)[1]
    u = _smooth_flow(3, hc, wc, 1, 2.0)
    got = flow.zoom_in(torch.from_numpy(u).cuda(), h, w).cpu().numpy()
    err = max(_rel(got[p], O.zoom_in(u[p].astype(np.float64), h, w)) for p in range(3))
    diag["flow/zoom_in/%dx%d" % (h, w)] = err
    assert err < 1e-5, err


@pytest.mark.parametrize("h,w", SIZES)
def test_warp_matches_oracle(h, w, diag):
    i0, i1, _ = _pairs(3, h, w, 2)
    u = _smooth_flow(3, h, w, 3, 4.0)          # reaches past the borders
    got = flow.warp(torch.from_numpy(i0).cuda(), torch.from_numpy(i1).cuda(), torch.from_numpy(u).cuda())
    got = got.cpu().numpy()
    errs = {}
    for p in range(3):
        want = O.warp(i0[p].astype(np.float64), i1[p].astype(np.float64), u[p].astype(np.float64))
        for name, g, wv in zip(("i1x", "i1y", "wx", "wy", "g", "rhoc"), got[:, p], want):
            errs[name] = max(errs.get(name, 0.0), _rel(g, wv))
    diag["flow/warp/%dx%d" % (h, w)] = errs
    assert max(errs.values()) < 1e-5, errs


@pytest.mark.parametrize("h,w", SIZES)
def test_one_iteration_matches_oracle(h, w, diag):
    P = 3
    i0, i1, _ = _pairs(P, h, w, 4)
    u0 = _smooth_flow(P, h, w, 5, 1.5)
    warped = flow.warp(torch.from_numpy(i0).cuda(), torch.from_numpy(i1).cuda(), torch.from_numpy(u0).cuda())
    r = np.random.RandomState(6)
    u = (u0 + r.normal(0, 0.2, u0.shape)).astype(np.float32)
    p = r.uniform(-0.5, 0.5, (P, 4, h, w)).astype(np.float32)
    ug, pg = torch.from_numpy(u).cuda(), torch.from_numpy(p).cuda()
    iters = flow.iterate(warped, ug, pg, 1)
    assert iters.cpu().tolist() == [1] * P
    wv = warped.cpu().numpy().astype(np.float64)
    eu = ep = 0.0
    for k in range(P):
        un, pn, _ = O.iteration(wv[2, k], wv[3, k], wv[4, k], wv[5, k], u[k].astype(np.float64),
                                p[k].astype(np.float64))
        eu, ep = max(eu, _rel(ug[k].cpu().numpy(), un)), max(ep, _rel(pg[k].cpu().numpy(), pn))
    diag["flow/iteration/%dx%d" % (h, w)] = {"u": eu, "p": ep}
    assert eu < 1e-5 and ep < 1e-5, (eu, ep)


@pytest.mark.parametrize("h,w", [(37, 53), (61, 47), (96, 128)])
def test_full_solve_matches_oracle(h, w, diag):
    P = 3
    i0, i1, _ = _pairs(P, h, w, 7)
    got, iters = flow.tvl1(torch.from_numpy(i0).cuda(), torch.from_numpy(i1).cuda())
    got, iters = got.cpu().numpy(), iters.cpu().numpy()
    assert iters.shape == (P, len(O.sizes(h, w)), flow.WARPS)
    d, it_diff = [], 0
    for k in range(P):
        want, wit = O.tvl1(i0[k], i1[k])
        d.append(np.hypot(*(got[k] - want)).ravel())
        it_diff = max(it_diff, int(np.abs(iters[k] - wit).max()))
    d = np.concatenate(d)
    mean, p99 = float(d.mean()), float(np.percentile(d, 99))
    diag["flow/solve/%dx%d" % (h, w)] = {"mean": mean, "p99": p99, "max": float(d.max()), "iters_diff": it_diff}
    assert mean < 0.01 and p99 < 0.1, (mean, p99)


def test_translation_recovery():
    d = (0.6, -0.35)
    i0 = torch.from_numpy(O.texture(48, 64, 3).astype(np.float32)).cuda()[None]
    i1 = torch.from_numpy(O.texture(48, 64, 3, d).astype(np.float32)).cuda()[None]
    f, _ = flow.tvl1(i0, i1)
    f = f[0].cpu().numpy()
    epe = np.hypot(f[0] - d[0], f[1] - d[1])[4:-4, 4:-4]
    assert epe.mean() < 0.05 and epe.max() < 0.1, (epe.mean(), epe.max())
    z, it = flow.tvl1(i0, i0)
    assert float(z.abs().max()) == 0.0 and (it == 1).all()


def test_batch_invariance():
    P, h, w = 37, 45, 61
    i0, i1, _ = _pairs(P, h, w, 8, max_shift=2.5)
    i1[5] = i0[5]                                       # a pair that converges at once next to ones that do not
    a, b = torch.from_numpy(i0).cuda(), torch.from_numpy(i1).cuda()
    f, it = flow.tvl1(a, b)
    f2, it2 = flow.tvl1(a, b)
    assert torch.equal(f, f2) and torch.equal(it, it2)
    assert int(it.max()) > int(it.min())                 # the pairs really stop at different iterations
    for k in range(P):
        fk, ik = flow.tvl1(a[k:k + 1], b[k:k + 1])
        assert torch.equal(fk[0], f[k]) and torch.equal(ik[0], it[k]), k
    for c in range(0, P, 5):
        fc, ic = flow.tvl1(a[c:c + 5], b[c:c + 5])
        assert torch.equal(fc, f[c:c + 5]) and torch.equal(ic, it[c:c + 5]), c


def test_quantise_bit_exact():
    r = np.random.RandomState(9)
    f = r.uniform(-26, 26, (4, 2, 29, 31)).astype(np.float32)
    edges = (np.arange(256, dtype=np.float32) - np.float32(0.5)) / np.float32(6.375) - np.float32(20)
    f.reshape(-1)[:256] = edges
    f.reshape(-1)[256:512] = np.nextafter(edges, np.float32(-np.inf))
    f.reshape(-1)[512:515] = [0.0, -0.0, 1e-30]
    got = flow.quantise(torch.from_numpy(f).cuda()).cpu().numpy()
    assert np.array_equal(got, O.quantise(f))


# --- the tool ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def built(tmp_path_factory):
    import dataset_fixture as F
    import shutil
    root = str(tmp_path_factory.mktemp("flowdb"))
    data, split = F.write(root, F.spec(), F.pool(), bin_type=False)
    out = os.path.join(data, F.FLOW)
    shutil.rmtree(out)                                   # the fixture's stand-in flow database: rebuilt by the tool
    rgb = os.path.join(data, F.RGB)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_flow_lmdb.py"), "--rgb", rgb, "--out", out,
                        "--pairs", "7"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert "pairs/s" in r.stdout
    return data, split, rgb, out


def test_tool_writes_the_flow_database(built):
    import make_flow_lmdb as M
    from coclr_b200 import lmdb_read, lmdb_write
    from coclr_b200.jpeg import JpegDecoder
    _, _, rgb, out = built
    src, db = lmdb_read.open(rgb), lmdb_read.open(out)
    for k in (b"__keys__", b"__len__", b"__order__"):
        assert bytes(db.get(k)) == bytes(src.get(k))
    keys = [bytes(k) for k in lmdb_read.unpack(src.get(b"__keys__"))]
    assert lmdb_write.bin_family(db.get(b"__order__")) is False
    vlen = lmdb_read.unpack(db.get(b"__vlen__"))
    dec = JpegDecoder()
    checked = 0
    for k, n in zip(keys, vlen):
        frames = [bytes(f) for f in lmdb_read.unpack(src.get(k))]
        stored = [bytes(f) for f in lmdb_read.unpack(db.get(k))]
        assert n == len(stored) == max(len(frames) - 1, 0), k
        if not stored:
            assert bytes(db.get(k)) == b"\x90"
            continue
        assert lmdb_write.bin_family(db.get(k)) is False
        g = flow.grey(dec(dec.parse(frames)))
        f, _ = flow.tvl1(g[:-1], g[1:])
        q = flow.quantise(f).cpu().numpy()
        assert [M.encode(x) for x in q] == stored, k
        checked += 1
    assert checked >= 10


def test_tool_is_deterministic_and_refuses(built, tmp_path):
    _, _, rgb, out = built
    again = str(tmp_path / "again")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_flow_lmdb.py"), "--rgb", rgb, "--out", again],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    with open(os.path.join(out, "data.mdb"), "rb") as a, open(os.path.join(again, "data.mdb"), "rb") as b:
        assert a.read() == b.read()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_flow_lmdb.py"), "--rgb", rgb, "--out", again],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 2 and "exists" in r.stderr


def test_tool_refuses_mixed_sizes_and_bad_frames(tmp_path):
    import io
    import lmdb_writer
    import make_flow_lmdb as M
    from PIL import Image

    def jpeg(h, w):
        b = io.BytesIO()
        Image.fromarray(np.full((h, w, 3), 90, np.uint8)).save(b, "JPEG")
        return b.getvalue()

    lmdb_writer.write_videos(str(tmp_path / "mixed"), {"c/ok": [jpeg(32, 32)] * 3, "c/mixed": [jpeg(32, 32),
                             jpeg(32, 48)]}, ["c/ok", "c/mixed"])
    with pytest.raises(M.Refused, match="c/mixed.*differ in size"):
        M.build(str(tmp_path / "mixed"), str(tmp_path / "o1"), 4)
    assert not (tmp_path / "o1").exists()
    lmdb_writer.write_videos(str(tmp_path / "bad"), {"c/bad": [jpeg(32, 32), b"not a jpeg"]}, ["c/bad"])
    with pytest.raises(M.Refused, match="c/bad.*cannot decode"):
        M.build(str(tmp_path / "bad"), str(tmp_path / "o2"), 4)
    assert not (tmp_path / "o2").exists()


def test_two_stream_loader_reads_the_built_database(built):
    import make_golden_datasets as G
    from coclr_b200 import datasets as D
    from coclr_b200 import loaders as LD
    data, split, _, _ = built
    kw = G.class_kwargs("UCF101_2STREAM_LMDB_2CLIP", data, split, "train", 1)
    ds = D.UCF101_2STREAM_LMDB_2CLIP(**kw)
    ld = LD.PretrainBatches(ds, 2, G.NF, G.IMG, torch.device("cuda"), seed=G.TRANSFORM_SEED, two_stream=True)
    it = iter(ld)
    x, _ = next(it)
    it.close()
    x = torch.stack(list(x))
    assert x.is_cuda and x.numel() > 0 and torch.isfinite(x).all()


def test_coclr_trains_on_the_built_database(built, tmp_path):
    data, split, _, _ = built
    args = ["--data-root", data, "--split-root", split, "--batch_size", "2", "--seq_len", "8", "--img_dim", "64",
            "--print_freq", "1", "--epochs", "1", "--dataset", "ucf101-2stream-2clip", "--moco-k", "16"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main_coclr.py")] + args, cwd=str(tmp_path),
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "finished" in r.stdout and "[0][1/2]" in r.stdout


def _jpeg(h, w, value=90):
    import io
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.full((h, w, 3), value, np.uint8)).save(b, "JPEG")
    return b.getvalue()


def _reference_layout_db(path, videos, bin_type):
    """An RGB database as the reference's converter writes it: keys and frames as bytes (`bin_type` picks the family
    of the msgpack that wrote them), `__order__` as a list of Python str (the str family under every msgpack)."""
    from coclr_b200 import lmdb_write
    order = sorted(videos)
    keys = ["%09d" % i for i in range(len(order))]
    with lmdb_write.Writer(path) as w:
        for k, name in zip(keys, order):
            w.put(k.encode(), lmdb_write.pack(videos[name], bin_type))
        w.put(b"__keys__", lmdb_write.pack([k.encode() for k in keys], bin_type))
        w.put(b"__len__", lmdb_write.pack(len(keys), bin_type))
        w.put(b"__order__", lmdb_write.pack(order, bin_type))
        w.put(b"__vlen__", lmdb_write.pack([len(videos[n]) for n in order], bin_type))


@pytest.mark.parametrize("bin_type", [True, False])
def test_tool_keeps_the_frame_family_with_a_str_order(tmp_path, bin_type):
    import make_flow_lmdb as M
    from coclr_b200 import lmdb_read, lmdb_write
    videos = {"c/a": [_jpeg(32, 40, v) for v in (60, 70, 80)], "c/b": [_jpeg(32, 40, 50)], "c/c": []}
    rgb, out = str(tmp_path / "rgb"), str(tmp_path / "flow")
    _reference_layout_db(rgb, videos, bin_type)
    src = lmdb_read.open(rgb)
    assert lmdb_write.bin_family(src.get(b"__order__")) is False
    assert lmdb_write.bin_family(src.get(b"000000000")) is bin_type
    M.build(rgb, out, 4, log=lambda *_: None)
    db = lmdb_read.open(out)
    assert lmdb_write.bin_family(db.get(b"000000000")) is bin_type          # c/a: two flow frames
    assert len(lmdb_read.unpack(db.get(b"000000000"))) == 2
    assert bytes(db.get(b"000000001")) == bytes(db.get(b"000000002")) == b"\x90"
    assert lmdb_read.unpack(db.get(b"__vlen__")) == [2, 0, 0]
    assert bytes(db.get(b"__order__")) == bytes(src.get(b"__order__"))


def test_tool_refuses_an_undecodable_single_frame(tmp_path):
    import make_flow_lmdb as M
    rgb = str(tmp_path / "rgb")
    _reference_layout_db(rgb, {"c/ok": [_jpeg(32, 32)] * 2, "c/one": [b"not a jpeg"]}, True)
    with pytest.raises(M.Refused, match="c/one.*cannot decode"):
        M.build(rgb, str(tmp_path / "o"), 4)
    assert not (tmp_path / "o").exists()


def test_batches_beyond_one_launch():
    """More pairs than one launch's grid takes (flow.MAX_BATCH) are solved in chunks with the same result; 32 x 32
    has two scales, so the flow upsampling runs over the whole batch too."""
    P, h, w = flow.MAX_BATCH + 3, 32, 32
    base = torch.from_numpy(O.texture(h, w, 12).astype(np.float32)).cuda()
    i0 = base.expand(P, h, w).contiguous()
    i1 = i0.clone()
    moved = [0, 40000, P - 1]
    for j, k in enumerate(moved):
        i1[k] = torch.from_numpy(O.texture(h, w, 12, (0.4 + 0.3 * j, -0.5)).astype(np.float32)).cuda()
    f, it = flow.tvl1(i0, i1)
    for k in moved:
        fk, ik = flow.tvl1(i0[k:k + 1], i1[k:k + 1])
        assert torch.equal(fk[0], f[k]) and torch.equal(ik[0], it[k]), k
        assert float(f[k].abs().max()) > 0.1
    still = torch.ones(P, dtype=torch.bool, device="cuda")
    still[moved] = False
    assert float(f[still].abs().max()) == 0.0 and bool((it[still] == 1).all())
    q = flow.quantise(f)
    assert torch.equal(q[moved[1]], flow.quantise(f[moved[1]:moved[1] + 1])[0])
    g = flow.grey(torch.zeros(P, 2, 3, 3, dtype=torch.uint8, device="cuda"))
    assert g.shape == (P, 2, 3) and float(g.abs().max()) == 0.0
