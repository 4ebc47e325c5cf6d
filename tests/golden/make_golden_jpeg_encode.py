"""Writes tests/golden/jpeg_encode.npz: Pillow's JPEG files of the frames of tests/tools/jpeg_encode_cases.py (each
case's name, quality and subsampling; the frames are regenerated from their seeds), with the Pillow and libjpeg
versions they came from.  Files of at most STORE_BYTES are stored whole, larger ones as their length and SHA-256.

    python tests/golden/make_golden_jpeg_encode.py
"""
import hashlib
import os
import sys

import numpy as np
import PIL
from PIL import features

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import jpeg_encode_cases as JE  # noqa: E402

STORE_BYTES = 8192


def arrays():
    names, quality, subsampling, lengths, sha, stored = [], [], [], [], [], []
    for name, img, q, s in JE.cases():
        raw = JE.pillow(img, q, s)
        names.append(name)
        quality.append(q)
        subsampling.append(s)
        lengths.append(len(raw))
        sha.append(hashlib.sha256(raw).hexdigest())
        stored.append(raw if len(raw) <= STORE_BYTES else b"")
    offsets = np.zeros(len(stored) + 1, np.int64)
    offsets[1:] = np.cumsum([len(r) for r in stored])
    return dict(names=np.array(names), quality=np.array(quality, np.int32),
                subsampling=np.array(subsampling, np.int32), lengths=np.array(lengths, np.int64),
                sha256=np.array(sha), data=np.frombuffer(b"".join(stored), np.uint8), offsets=offsets,
                versions=np.array([PIL.__version__, features.version("jpg")]))


def main():
    a = arrays()
    np.savez_compressed(os.path.join(HERE, "jpeg_encode.npz"), **a)
    print("wrote %d cases, %d bytes stored" % (len(a["names"]), a["data"].size))


if __name__ == "__main__":
    main()
