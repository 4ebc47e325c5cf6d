"""JPEG test cases, encoded by Pillow: smooth fields plus noise at every sampling, size and quality the decoder must
match, and the encoder options that change the bitstream (optimised tables, restart markers, metadata segments,
16-bit quant tables, grayscale, a default-table JPEG with its DHT stripped).  `cases()` is deterministic for one
Pillow / libjpeg version."""
import io

import numpy as np
from PIL import Image

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 47), (240, 320), (241, 323)]
QUALITIES = [1, 10, 50, 75, 90, 95, 100]
SUBSAMPLING = {0: "444", 1: "422", 2: "420"}


def field(h, w, seed, noise=12.0, gray=False):
    """A smooth colour field plus Gaussian noise, uint8 [h, w, 3] (or [h, w])."""
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    ch = [128 + 90 * np.sin(xx / (9.0 + 4 * c) + c) * np.cos(yy / (11.0 + 3 * c) - 2 * c) for c in range(3)]
    img = np.clip(np.stack(ch, -1) + r.normal(0, noise, (h, w, 3)), 0, 255).astype(np.uint8)
    return img[..., 0] if gray else img


def encode(img, **kw):
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", **kw)
    return b.getvalue()


def pillow_decode(raw):
    """The reference datasets' pil_from_raw_rgb."""
    return np.asarray(Image.open(io.BytesIO(raw)).convert("RGB"))


def strip_dht(raw):
    """The same JPEG without its DHT segments (libjpeg then uses the Annex K tables, which Pillow's default encoder
    wrote)."""
    out, pos = bytearray(raw[:2]), 2
    while pos < len(raw):
        m = raw[pos + 1]
        if m == 0xDA:
            out += raw[pos:]
            break
        L = (raw[pos + 2] << 8) | raw[pos + 3]
        if m != 0xC4:
            out += raw[pos:pos + 2 + L]
        pos += 2 + L
    return bytes(out)


def cases():
    """[(name, jpeg bytes)]: every size at every sampling (quality 75), every quality at two samplings, and the
    option cases.  Not the full cross product."""
    out = []
    seed = 0
    for ss, tag in SUBSAMPLING.items():
        for h, w in SIZES:
            seed += 1
            out.append(("s%s_%dx%d_q75" % (tag, h, w), encode(field(h, w, seed), quality=75, subsampling=ss)))
    for q in QUALITIES:
        for ss, (h, w) in ((2, (33, 47)), (0, (15, 17))):
            seed += 1
            out.append(("q%d_s%s_%dx%d" % (q, SUBSAMPLING[ss], h, w),
                        encode(field(h, w, seed, noise=40.0 if q == 100 else 12.0), quality=q, subsampling=ss)))
    out.append(("q100_noise_s420_64x96", encode(field(64, 96, 101, noise=60.0), quality=100, subsampling=2)))
    out.append(("q100_noise_s444_57x83", encode(field(57, 83, 102, noise=60.0), quality=100, subsampling=0)))
    out.append(("q90_s420_240x320", encode(field(240, 320, 103), quality=90, subsampling=2)))
    out.append(("optimize_s420_241x323", encode(field(241, 323, 104), quality=80, subsampling=2, optimize=True)))
    out.append(("optimize_s422_33x47", encode(field(33, 47, 105), quality=60, subsampling=1, optimize=True)))
    out.append(("rst_blocks3_s420_33x47", encode(field(33, 47, 106), quality=75, subsampling=2,
                                                 restart_marker_blocks=3)))
    out.append(("rst_rows1_s422_240x320", encode(field(240, 320, 107), quality=75, subsampling=1,
                                                 restart_marker_rows=1)))
    out.append(("rst_blocks1_s444_15x17", encode(field(15, 17, 108), quality=90, subsampling=0,
                                                 restart_marker_blocks=1)))
    out.append(("gray_33x47", encode(field(33, 47, 109, gray=True), quality=75)))
    out.append(("gray_241x323", encode(field(241, 323, 110, gray=True), quality=90)))
    out.append(("gray_rst_7x9", encode(field(7, 9, 111, gray=True), quality=50, restart_marker_blocks=2)))
    exif = Image.Exif()
    exif[0x010E] = "synthetic frame"
    icc = bytes(range(256)) * 8
    out.append(("meta_exif_icc_comment_33x47", encode(field(33, 47, 112), quality=75, exif=exif.tobytes(),
                                                      icc_profile=icc, comment=b"frame 0")))
    qt = [[min(1 + (i * 7) % 400, 400) for i in range(64)], [min(2 + (i * 11) % 300, 300) for i in range(64)]]
    out.append(("qtables16_s420_33x47", encode(field(33, 47, 113, noise=40.0), qtables=qt, subsampling=2)))
    out.append(("qtables8_s444_16x16", encode(field(16, 16, 114), qtables=[[3] * 64, [5] * 64], subsampling=0)))
    out.append(("nodht_s420_33x47", strip_dht(encode(field(33, 47, 115), quality=75, subsampling=2))))
    out.append(("nodht_gray_15x17", strip_dht(encode(field(15, 17, 116, gray=True), quality=75))))
    return out
