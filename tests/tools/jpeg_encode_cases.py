"""JPEG encoder test frames: seeded uint8 [h, w, 3] contents at the sizes, qualities and samplings the encoder must
match Pillow on.  `cases()` is a fixed list of (name, frame, quality, subsampling), not the full cross product:

  * every size x sampling x content at quality 75 or 95 (alternating), the sizes being 1x1 .. 256x340;
  * every quality x sampling x content at 37x53;
  * the extreme contents (0/255 checkerboards and stripes) at quality 100 on every size and sampling;
  * one 1080x1920 flow-like frame per sampling at quality 95.
"""
import io

import numpy as np

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33), (37, 53), (61, 47), (240, 320), (256, 340)]
QUALITIES = [1, 10, 50, 75, 90, 95, 100]
SUBSAMPLINGS = [0, 1, 2]
CONTENTS = ["smooth", "noise", "checker", "stripes", "zero", "full", "flow"]


def frame(content, h, w, seed):
    """A uint8 [h, w, 3] frame: a smooth colour field, N(128, 60) noise, 0/255 one-pixel checkerboard or vertical
    stripes (the largest coefficients: long codes and 0xFF bytes), constant 0 or 255, or a flow-like frame (smooth R
    and G, B = 128, as make_flow_lmdb stores)."""
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    if content == "smooth":
        ch = [128 + 100 * np.sin(xx / (7.0 + 3 * c) + c) * np.cos(yy / (9.0 + 2 * c) - c) for c in range(3)]
        return np.clip(np.stack(ch, -1), 0, 255).astype(np.uint8)
    if content == "noise":
        return np.clip(r.normal(128, 60, (h, w, 3)), 0, 255).astype(np.uint8)
    if content == "checker":
        c = ((yy + xx) % 2 * 255).astype(np.uint8)
        return np.stack([c, 255 - c, c], -1)
    if content == "stripes":
        c = (xx % 2 * 255).astype(np.uint8)
        return np.stack([c, c, 255 - c], -1)
    if content == "zero":
        return np.zeros((h, w, 3), np.uint8)
    if content == "full":
        return np.full((h, w, 3), 255, np.uint8)
    if content == "flow":
        fx, fy = r.uniform(8, 40, 2)
        u = 128 + 60 * np.sin(xx / fx + r.uniform(0, 6)) * np.cos(yy / fy)
        v = 128 + 50 * np.cos(xx / fy - yy / fx)
        return np.stack([np.clip(u, 0, 255), np.clip(v, 0, 255), np.full((h, w), 128.0)], -1).astype(np.uint8)
    raise ValueError(content)


def pillow(img, quality, subsampling):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", quality=quality, subsampling=subsampling)
    return b.getvalue()


def cases(large=True):
    """[(name, frame, quality, subsampling)]; large=False leaves out the 1080x1920 frames."""
    out = []
    seed = 0
    for (h, w) in SIZES:
        for ss in SUBSAMPLINGS:
            for k, c in enumerate(CONTENTS):
                seed += 1
                q = (75, 95)[(k + ss) % 2]
                out.append(("%s_%dx%d_q%d_s%d" % (c, h, w, q, ss), frame(c, h, w, seed), q, ss))
            for c in ("checker", "stripes"):
                out.append(("%s_%dx%d_q100_s%d" % (c, h, w, ss), frame(c, h, w, 0), 100, ss))
    for q in QUALITIES:
        for ss in SUBSAMPLINGS:
            for c in CONTENTS:
                seed += 1
                out.append(("%s_37x53_q%d_s%d_b" % (c, q, ss), frame(c, 37, 53, seed), q, ss))
    if large:
        for ss in SUBSAMPLINGS:
            out.append(("flow_1080x1920_q95_s%d" % ss, frame("flow", 1080, 1920, 9000 + ss), 95, ss))
    return out
