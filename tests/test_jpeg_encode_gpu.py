"""JPEG encoding on the GPU (coclr_b200.jpeg.JpegEncoder, csrc/jpeg_encode.cu) against Pillow, byte for byte:

  * every case of tests/golden/jpeg_encode.npz (sizes 1x1 .. 1920x1080, qualities 1 .. 100, 4:4:4 / 4:2:2 / 4:2:0,
    smooth, noise, 0/255 checkerboards and stripes, constant and flow-like frames), and live Pillow when its libjpeg
    is the fixture's;
  * a frame gives the same bytes alone, in a batch of 37, from a strided view and across work_limit passes;
  * two runs are identical; JpegDecoder decodes the files as Pillow does;
  * every ValueError is raised before a launch.
"""
import hashlib
import io
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image, features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coclr_b200 import lib as L  # noqa: E402
from coclr_b200.jpeg import JpegDecoder, JpegEncoder  # noqa: E402
import jpeg_encode_cases as JE  # noqa: E402

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_encode.npz"))
LIVE = features.version("jpg") == str(G["versions"][1])


def _golden(i, raw):
    if len(raw) != G["lengths"][i]:
        return False
    if G["offsets"][i + 1] > G["offsets"][i]:
        return raw == G["data"][G["offsets"][i]:G["offsets"][i + 1]].tobytes()
    return hashlib.sha256(raw).hexdigest() == str(G["sha256"][i])


def _groups():
    """Cases grouped by (shape, quality, subsampling): one batch per group."""
    groups = {}
    for i, (name, img, q, s) in enumerate(JE.cases()):
        groups.setdefault((img.shape, q, s), []).append((i, name, img))
    return groups


def test_golden_and_live_pillow():
    bad = []
    for (shape, q, s), items in _groups().items():
        frames = torch.from_numpy(np.stack([img for _, _, img in items])).cuda()
        out = JpegEncoder(q, s)(frames)
        for (i, name, img), raw in zip(items, out):
            if not _golden(i, raw):
                bad.append(name)
            elif LIVE and shape[0] * shape[1] <= 256 * 340 and raw != JE.pillow(img, q, s):
                bad.append("live " + name)
    assert not bad, bad


def test_batch_view_and_passes():
    h, w = 61, 47
    frames = [JE.frame(JE.CONTENTS[i % len(JE.CONTENTS)], h, w, 500 + i) for i in range(37)]
    want = [JE.pillow(f, 90, 2) for f in frames]
    enc = JpegEncoder(quality=90, subsampling=2)
    batch = torch.from_numpy(np.stack(frames)).cuda()
    assert [enc(batch[i:i + 1])[0] for i in (0, 17, 36)] == [want[i] for i in (0, 17, 36)]
    assert enc(batch) == want
    # a crop of a larger tensor, every other frame: rows and frames strided
    big = torch.zeros(74, h + 5, w + 9, 3, dtype=torch.uint8, device="cuda")
    big[::2, 3:3 + h, 4:4 + w] = batch
    view = big[::2, 3:3 + h, 4:4 + w]
    assert view.stride(1) != 3 * w
    assert enc(view) == want
    lib = L.load()
    small = JpegEncoder(quality=90, subsampling=2, work_limit=lib.coclr_jpeg_encode_work_bytes(3, h, w, 2))
    assert small(batch) == want
    assert enc(batch) == enc(batch)                  # a second run, the same bytes
    assert JpegEncoder(quality=90, subsampling=2)(batch[:0]) == []


def test_decoder_round_trip():
    frames = [JE.frame(c, 240, 320, 700 + k) for k, c in enumerate(JE.CONTENTS)]
    for q, s in [(75, 2), (95, 0), (50, 1)]:
        raws = JpegEncoder(q, s)(torch.from_numpy(np.stack(frames)).cuda())
        dec = JpegDecoder()
        batch = dec.parse(raws)
        got = dec(batch).cpu().numpy()
        for k, r in enumerate(raws):
            assert np.array_equal(got[k], np.asarray(Image.open(io.BytesIO(r)).convert("RGB"))), (q, s, k)


def test_refuses_before_launch():
    launches = L.LAUNCHES
    ok = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device="cuda")
    enc = JpegEncoder()
    bad = [ok.cpu(), ok.float(), ok[0], ok[..., :2], ok.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)[..., :1],
           torch.zeros(1, 8, 8, 3, 2, dtype=torch.uint8, device="cuda")[..., 0],
           torch.zeros(1, 0, 8, 3, dtype=torch.uint8, device="cuda"),
           torch.zeros(1, 8, 0, 3, dtype=torch.uint8, device="cuda"),
           torch.zeros(1, 65501, 1, 3, dtype=torch.uint8, device="cuda"),
           torch.zeros(1, 1, 65501, 3, dtype=torch.uint8, device="cuda"), [ok]]
    for x in bad:
        with pytest.raises(ValueError):
            enc(x)
    for kw in [dict(quality=0), dict(quality=101), dict(quality=7.5), dict(subsampling=3), dict(subsampling=-1)]:
        with pytest.raises(ValueError):
            JpegEncoder(**kw)
    assert L.LAUNCHES == launches
