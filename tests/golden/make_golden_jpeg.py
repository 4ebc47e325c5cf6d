"""Writes tests/golden/jpeg.npz: the Pillow-encoded JPEGs of tests/tools/jpeg_cases.py and what Pillow's decoder makes
of them (`Image.open(BytesIO(raw)).convert('RGB')`), with the Pillow and libjpeg versions they came from.  Outputs of
at most 48 x 48 pixels are stored whole, larger ones as the SHA-256 of their uint8 [h, w, 3] bytes.

    python tests/golden/make_golden_jpeg.py
"""
import hashlib
import os
import sys

import numpy as np
import PIL
from PIL import features

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import jpeg_cases as JC  # noqa: E402

STORE_PIXELS = 48 * 48


def main():
    cases = JC.cases()
    names = [n for n, _ in cases]
    raws = [r for _, r in cases]
    offsets = np.zeros(len(raws) + 1, np.int64)
    offsets[1:] = np.cumsum([len(r) for r in raws])
    pix, pix_off, sha, sizes = [], [0], [], []
    for r in raws:
        img = JC.pillow_decode(r)
        sizes.append(img.shape[:2])
        if img.shape[0] * img.shape[1] <= STORE_PIXELS:
            pix.append(img.reshape(-1))
            sha.append("")
        else:
            sha.append(hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest())
        pix_off.append(pix_off[-1] + (img.size if sha[-1] == "" else 0))
    np.savez_compressed(
        os.path.join(HERE, "jpeg.npz"),
        names=np.array(names), data=np.frombuffer(b"".join(raws), np.uint8), offsets=offsets,
        sizes=np.array(sizes, np.int32), pixels=np.concatenate(pix), pixel_offsets=np.array(pix_off, np.int64),
        sha256=np.array(sha), versions=np.array([PIL.__version__, features.version("jpg")]))
    print("wrote %d cases" % len(names))


if __name__ == "__main__":
    main()
