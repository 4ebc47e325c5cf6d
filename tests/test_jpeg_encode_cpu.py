"""JPEG encoding without a GPU: the numpy oracle (tests/tools/jpeg_encode_oracle.py) against Pillow byte for byte over
the case grid, the library's header writer against Pillow's headers, the settings it refuses, and the golden file
against a fresh run of its generator."""
import os
import sys

import numpy as np
import pytest
from PIL import features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from coclr_b200 import jpeg  # noqa: E402
import jpeg_encode_cases as JE  # noqa: E402
import jpeg_encode_oracle as O  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_encode.npz"))
LIVE = features.version("jpg") == str(G["versions"][1])


def _library():
    from coclr_b200 import lib
    if not os.path.exists(lib.library_path()):
        pytest.skip("libcoclr_b200.so is not built")


@pytest.mark.skipif(not LIVE, reason="Pillow's libjpeg is not the one the golden file was made with")
@pytest.mark.parametrize("large", [False, True])
def test_oracle_matches_pillow(large):
    cases = [c for c in JE.cases() if ("1080x1920" in c[0]) == large]
    bad = [name for name, img, q, s in cases if O.encode(img, q, s) != JE.pillow(img, q, s)]
    assert not bad, bad


def test_oracle_matches_golden():
    """The oracle against the stored files, whatever Pillow is installed."""
    import hashlib
    bad = []
    for i, (name, img, q, s) in enumerate(JE.cases()):
        raw = O.encode(img, q, s)
        if hashlib.sha256(raw).hexdigest() != str(G["sha256"][i]) or len(raw) != G["lengths"][i]:
            bad.append(name)
    assert not bad, bad


def test_extreme_blocks_reach_the_worst_codes():
    """The grid's checkerboards at quality 100 make the largest coefficients: 10-bit AC magnitudes and 0xFF bytes."""
    img = JE.frame("checker", 16, 16, 0)
    scan, _ = O.coefficients(img, 100, 0)
    assert np.abs(scan[:, 1:]).max() >= 512
    assert b"\xff\x00" in O.encode(img, 100, 0)


def test_header_matches_pillow():
    _library()
    bad = []
    for h, w in [(1, 1), (8, 8), (17, 33), (240, 320), (256, 340), (1080, 1920)]:
        for q in JE.QUALITIES:
            for s in JE.SUBSAMPLINGS:
                want = O.header(h, w, q, s)
                if jpeg.encode_header(h, w, q, s) != want:
                    bad.append((h, w, q, s))
                if LIVE and h * w <= 256 * 340 and JE.pillow(JE.frame("zero", h, w, 0), q, s)[:len(want)] != want:
                    bad.append(("pillow", h, w, q, s))
    assert not bad, bad
    assert len(jpeg.encode_header(65500, 65500, 75, 2)) == jpeg.HEADER_BYTES


@pytest.mark.parametrize("args", [(0, 8, 75, 2), (8, 0, 75, 2), (65501, 8, 75, 2), (8, 65501, 75, 2),
                                  (8, 8, 0, 2), (8, 8, 101, 2), (8, 8, 75, 3), (8, 8, 75, -1), (8, 8, 75.0, 2)])
def test_header_refuses(args):
    _library()
    with pytest.raises(ValueError):
        jpeg.encode_header(*args)


def test_sizes_are_worst_case_bounds():
    _library()
    from coclr_b200 import lib as L
    lib = L.load()
    for h, w, s in [(1, 1, 0), (240, 320, 0), (256, 340, 2), (1080, 1920, 1)]:
        hs, vs = O.SAMPLING[s]
        blocks = -(-w // (8 * hs)) * -(-h // (8 * vs)) * (hs * vs + 2)
        assert lib.coclr_jpeg_encode_max_bytes(h, w, s) == 623 + 2 * (-(-blocks * 1660 // 8)) + 2
        assert lib.coclr_jpeg_encode_work_bytes(2, h, w, s) > lib.coclr_jpeg_encode_work_bytes(1, h, w, s) > 0
    assert lib.coclr_jpeg_encode_max_bytes(0, 8, 2) == 0 and lib.coclr_jpeg_encode_work_bytes(1, 8, 8, 3) == 0


@pytest.mark.skipif(not LIVE, reason="Pillow's libjpeg is not the one the golden file was made with")
def test_golden_matches_generator():
    import make_golden_jpeg_encode as M
    fresh = M.arrays()
    for k in ("names", "quality", "subsampling", "lengths", "sha256", "data", "offsets"):
        assert np.array_equal(fresh[k], G[k]), k
