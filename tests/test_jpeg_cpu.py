"""Host side of the JPEG decoder (coclr_b200.jpeg), without a GPU:

  * the numpy oracle (tests/tools/jpeg_oracle.py, the statement the kernels mirror) equals Pillow's
    `Image.open(BytesIO(raw)).convert('RGB')` bit for bit on every case of tests/golden/jpeg.npz (samplings, sizes with
    edge MCUs and odd chroma widths, qualities 1-100, optimised tables, restart markers, grayscale, metadata segments,
    16-bit quant tables, a stripped DHT), and on live Pillow when its libjpeg is the fixture's;
  * the C parser (coclr_jpeg_parse) equals the oracle's parse on every case, stores each distinct table once, and
    gives each rejected kind its reason;
  * the record layouts agree with include/coclr_b200.h, and the batch helpers check their inputs.
"""
import ctypes as C
import hashlib
import os
import re
import struct
import sys

import numpy as np
import pytest
from PIL import Image, features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200 import jpeg as J  # noqa: E402
import jpeg_cases as JC  # noqa: E402
import jpeg_oracle as O  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "jpeg.npz"))
NAMES = [str(n) for n in G["names"]]
RAWS = [G["data"][G["offsets"][i]:G["offsets"][i + 1]].tobytes() for i in range(len(NAMES))]


def _fixture_ok(i, img):
    h, w = (int(v) for v in G["sizes"][i])
    if img.shape != (h, w, 3):
        return False
    if str(G["sha256"][i]):
        return hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest() == str(G["sha256"][i])
    return np.array_equal(img, G["pixels"][G["pixel_offsets"][i]:G["pixel_offsets"][i + 1]].reshape(h, w, 3))


@pytest.mark.parametrize("i", range(len(NAMES)), ids=NAMES)
def test_oracle_equals_fixture(i):
    img, st = O.decode(RAWS[i])
    assert st == O.ST_OK
    assert _fixture_ok(i, img)


def test_fixture_covers_the_cases():
    kinds = {"s444", "s422", "s420", "optimize", "rst_blocks", "rst_rows", "gray", "meta", "qtables16", "nodht",
             "q100_noise"}
    assert all(any(n.startswith(k) for n in NAMES) for k in kinds)
    assert {"q%d" % q for q in JC.QUALITIES} <= {n.split("_")[0] for n in NAMES}
    assert all(any(n.endswith("_%dx%d_q75" % hw) for n in NAMES) for hw in JC.SIZES)
    q16 = RAWS[NAMES.index("qtables16_s420_33x47")]
    assert b"\xff\xc1" in q16 and q16[q16.index(b"\xff\xdb") + 4] >> 4 == 1      # SOF1 and a 16-bit DQT
    assert b"\xff\xc4" not in RAWS[NAMES.index("nodht_s420_33x47")]
    assert re.search(rb"\xff[\xd0-\xd7]", RAWS[NAMES.index("rst_rows1_s422_240x320")])


def test_oracle_equals_live_pillow():
    if features.version("jpg") != str(G["versions"][1]):
        pytest.skip("Pillow's libjpeg %s is not the fixture's %s" % (features.version("jpg"), G["versions"][1]))
    for name, raw in JC.cases():
        img, st = O.decode(raw)
        assert st == O.ST_OK and np.array_equal(img, JC.pillow_decode(raw)), name


def _c_parse(raws):
    return J.parse(raws)


def test_c_parser_equals_oracle():
    batch = _c_parse(RAWS)
    f = batch.frames
    block0 = 0
    for i, raw in enumerate(RAWS):
        p = O.parse(raw)
        geo, mx, my = O.geometry(p)
        assert (f["h"][i], f["w"][i], f["ncomp"][i], f["hs"][i], f["vs"][i], f["restart"][i]) == \
            (p["h"], p["w"], p["ncomp"], p["hs"], p["vs"], p["restart"]), NAMES[i]
        assert (f["mcus_x"][i], f["mcus_y"][i]) == (mx, my)
        assert f["blocks"][i] == sum(g[0] * g[1] for g in geo) and f["block0"][i] == block0
        block0 += int(f["blocks"][i])
        off = batch.offsets[i]
        assert (f["ecs_begin"][i] - off, f["ecs_end"][i] - off) == p["ecs"], NAMES[i]
        for c, comp in enumerate(p["comps"]):
            assert list(batch.quant["q"][f["qt"][i][c]]) == list(comp["q"])
            for key, t in (("dc", comp["dc"]), ("ac", comp["ac"])):
                h = batch.huff[f[key][i][c]]
                assert list(h["bits"]) == t[0] and list(h["val"][:h["nval"]]) == t[1], (NAMES[i], key, c)
    assert batch.work_bytes == 128 * block0


def test_tables_stored_once():
    raws = [RAWS[NAMES.index("s420_33x47_q75")]] * 5 + [RAWS[NAMES.index("gray_33x47")]]
    b = _c_parse(raws)
    assert len(b.quant) == 2 and len(b.huff) == 4
    assert len({tuple(b.frames["qt"][i]) for i in range(5)}) == 1


def test_huffman_lookahead_tables():
    """The derived tables decode every code of every table to its symbol (the kernel's fast and slow paths)."""
    b = _c_parse(RAWS)
    for h in b.huff:
        bits, vals = list(h["bits"]), list(h["val"][:h["nval"]])
        for (l, code), sym in O._codes(bits, vals).items():
            if l <= 9:
                e = int(h["look"][code << (9 - l)])
                assert (e >> 8, e & 255) == (l, sym)
            else:
                assert int(h["look"][code >> (l - 9)]) == 0
                assert code <= h["maxcode"][l] and h["val"][(code + h["valoff"][l]) & 255] == sym


def test_many_distinct_tables_grow_the_arrays():
    img = JC.field(16, 16, 3)
    raws = [JC.encode(img, quality=q) for q in range(5, 95, 7)]
    b = _c_parse(raws)
    assert len(b.quant) == 2 * len(raws)


# ----------------------------------------------------------------------------------------------------------------------
# rejections
# ----------------------------------------------------------------------------------------------------------------------

BASE = RAWS[NAMES.index("s420_33x47_q75")]


def _segments(raw):
    """[(marker, bytes of the whole segment)] up to SOS, then the rest."""
    out, pos = [], 2
    while raw[pos + 1] != 0xDA:
        L = (raw[pos + 2] << 8) | raw[pos + 3]
        out.append((raw[pos + 1], raw[pos:pos + 2 + L]))
        pos += 2 + L
    return out, raw[pos:]


def _with(raw, marker, fn):
    segs, rest = _segments(raw)
    return raw[:2] + b"".join(fn(s) if m == marker else s for m, s in segs) + rest


def _sof(raw, fn):
    return _with(raw, 0xC0, lambda s: s[:4] + fn(bytearray(s[4:])))


def _encode_mode(mode, **kw):
    b = __import__("io").BytesIO()
    Image.new(mode, (24, 16), (10, 20, 30, 40)[:len(mode)] if len(mode) > 1 else 50).save(b, "JPEG", **kw)
    return b.getvalue()


def _sampling(s, h, v):
    s[7] = (h << 4) | v
    return bytes(s)


def _ids(s, ids):
    for k, c in enumerate(ids):
        s[6 + 3 * k] = c
    return bytes(s)


def _precision(s):
    s[0] = 12
    return bytes(s)


def _rgb_ids(raw):
    raw = bytearray(_sof(raw, lambda s: _ids(s, b"RGB")))
    k = raw.index(b"\xff\xda")
    raw[k + 5], raw[k + 7], raw[k + 9] = b"RGB"
    return bytes(raw)


def _overfull_dht(raw):
    """The first DHT (DC 0: 0 1 5 codes of lengths 1-3) with 2 1 3 codes instead: more than fit in 2 bits."""
    k = raw.index(b"\xff\xc4")
    assert raw[k + 5:k + 8] == b"\x00\x01\x05"
    return raw[:k + 5] + b"\x02\x01\x03" + raw[k + 8:]


def _all_ones_dht(raw):
    """The first DHT replaced by a DC table of one 2-bit and six 3-bit codes: its last code, 111, is all ones, which
    libjpeg refuses (Pillow raises on it)."""
    k = raw.index(b"\xff\xc4")
    L = (raw[k + 2] << 8) | raw[k + 3]
    seg = b"\xff\xc4\x00\x1a\x00" + bytes([0, 1, 6] + [0] * 13) + bytes(range(7))
    return raw[:k] + seg + raw[k + 2 + L:]


def _no_jfif(raw):
    segs, rest = _segments(raw)
    return raw[:2] + b"".join(s for m, s in segs if m != 0xE0) + rest


ADOBE0 = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"   # APP14, transform 0 (RGB)
REJECTS = {
    "progressive": (lambda: _encode_mode("RGB", progressive=True), O.PROGRESSIVE),
    "cmyk": (lambda: _encode_mode("CMYK"), O.COMPONENTS),
    "truncated_header": (lambda: BASE[:100], O.TRUNCATED),
    "truncated_scan": (lambda: BASE[:-40], O.NO_EOI),
    "no_soi": (lambda: BASE[2:], O.NO_SOI),
    "empty": (lambda: b"", O.NO_SOI),
    "arithmetic": (lambda: _with(BASE, 0xC0, lambda s: s[:1] + b"\xc9" + s[2:]), O.ARITHMETIC),
    "lossless": (lambda: _with(BASE, 0xC0, lambda s: s[:1] + b"\xc3" + s[2:]), O.SOF_KIND),
    "hierarchical": (lambda: _with(BASE, 0xC0, lambda s: s[:1] + b"\xc5" + s[2:]), O.SOF_KIND),
    "precision12": (lambda: _sof(BASE, _precision), O.PRECISION),
    "sampling_1x2": (lambda: _sof(BASE, lambda s: _sampling(s, 1, 2)), O.SAMPLING),
    "sampling_4x1": (lambda: _sof(BASE, lambda s: _sampling(s, 4, 1)), O.SAMPLING),
    "rgb_ids": (lambda: _no_jfif(_rgb_ids(BASE)), O.RGB),
    "adobe_rgb": (lambda: _no_jfif(BASE[:2] + ADOBE0 + BASE[2:]), O.RGB),
    "no_sof": (lambda: _with(BASE, 0xC0, lambda s: b""), O.NO_SOF),
    "no_sos": (lambda: BASE[:BASE.index(b"\xff\xda")] + b"\xff\xd9", O.NO_SOS),
    "no_eoi": (lambda: BASE[:-2], O.NO_EOI),
    "two_scans": (lambda: BASE[:-2] + BASE[BASE.index(b"\xff\xda"):], O.MULTI_SCAN),
    "missing_dqt": (lambda: _with(BASE, 0xDB, lambda s: b""), O.BAD_TABLE),
    "bad_dht": (lambda: _overfull_dht(BASE), O.BAD_TABLE),
    "all_ones_code": (lambda: _all_ones_dht(BASE), O.BAD_TABLE),
    "bad_length": (lambda: BASE[:4] + b"\x00\x01" + BASE[6:], O.BAD_SEGMENT),
}


@pytest.mark.parametrize("name", sorted(REJECTS))
def test_rejections(name):
    make, reason = REJECTS[name]
    raw = make()
    with pytest.raises(O.Reject) as e:
        O.parse(raw)
    assert e.value.reason == reason, (name, O.REASONS[e.value.reason])
    with pytest.raises(ValueError, match="frame 1: " + re.escape(J.REASONS[reason])):
        J.parse([BASE, raw, BASE])


def test_rejection_cases_are_what_they_say():
    with pytest.raises(OSError):
        JC.pillow_decode(REJECTS["all_ones_code"][0]())
    assert b"\xff\xc2" in REJECTS["progressive"][0]()
    cmyk = REJECTS["cmyk"][0]()
    assert cmyk[cmyk.index(b"\xff\xc0") + 9] == 4                       # four components


def test_gray_in_three_channels_and_grayscale_sampling():
    raw = RAWS[NAMES.index("gray_33x47")]
    img, _ = O.decode(raw)
    assert (img[..., 0] == img[..., 1]).all() and (img[..., 1] == img[..., 2]).all()
    b = J.parse([raw])
    assert b.frames["ncomp"][0] == 1 and (b.frames["hs"][0], b.frames["vs"][0]) == (1, 1)


# ----------------------------------------------------------------------------------------------------------------------
# layouts and helpers
# ----------------------------------------------------------------------------------------------------------------------

def test_record_sizes_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "coclr_b200.h")).read()
    for name in ("coclr_jpeg_frame_t", "coclr_jpeg_quant_t", "coclr_jpeg_huff_t", "coclr_jpeg_t",
                 "coclr_jpeg_parse", "coclr_jpeg_decode", "coclr_jpeg_work_bytes"):
        assert name in hdr
    assert (J.FRAME.itemsize, J.QUANT.itemsize, J.HUFF.itemsize) == (112, 128, 1456)
    assert C.sizeof(J.L.Jpeg) == 96
    assert [J.REASONS[getattr(O, k)] for k in ("PROGRESSIVE", "RGB")] == ["progressive", "RGB colour transform"]
    defines = dict((k, int(v)) for k, v in re.findall(r"#define COCLR_JPEG_(\w+) (\d+)", hdr))
    assert defines["BAD_SEGMENT"] == O.BAD_SEGMENT == len(J.REASONS) - 1
    assert (defines["ST_BAD_CODE"], defines["ST_EARLY_END"], defines["ST_BAD_RESTART"]) == \
        (O.ST_BAD_CODE, O.ST_EARLY_END, O.ST_BAD_RESTART)


def test_sample_sizes():
    raws = [RAWS[NAMES.index("s420_7x9_q75")]] * 4 + [RAWS[NAMES.index("s420_33x47_q75")]] * 2
    b = J.parse(raws)
    assert b.sizes[:2] == [(7, 9), (7, 9)]
    assert b.sample_sizes(3) == [(7, 9), (7, 9), (33, 47)]
    with pytest.raises(ValueError, match="sample 1"):
        b.sample_sizes(2)
    with pytest.raises(ValueError, match="do not split"):
        b.sample_sizes(4)


def test_decode_needs_a_parsed_batch():
    with pytest.raises(ValueError, match="JpegBatch"):
        J.JpegDecoder()([BASE])


def test_corrupted_entropy_data_status_in_the_oracle():
    """A segment cut short reports an early end; a run of one-bits reports an impossible code; a restart marker out
    of sequence reports a bad restart."""
    p = O.parse(BASE)
    b0, b1 = p["ecs"]
    assert O.decode(BASE[:b0 + (b1 - b0) // 2] + b"\xff\xd9")[1] == O.ST_EARLY_END
    assert O.decode(BASE[:b0 + 10] + b"\xff\x00" * 16 + BASE[b0 + 42:])[1] == O.ST_BAD_CODE
    rst = RAWS[NAMES.index("rst_blocks3_s420_33x47")]
    k = rst.index(b"\xff\xd1")
    assert O.decode(rst[:k + 1] + b"\xd5" + rst[k + 2:])[1] == O.ST_BAD_RESTART
    assert struct.pack(">H", 0xFFD9) == rst[-2:]
