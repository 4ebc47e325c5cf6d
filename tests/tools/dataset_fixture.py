"""A tiny seeded copy of the reference's dataset layout for the dataset tests and the golden generator.

spec() describes it: the split files (UCF101 with 'index, name' ClassInd lines, HMDB51 and K400 with bare names, one
with a space), the videos of every database as indices into a pool of small Pillow JPEGs, and each database's
`__order__`.  RGB and flow lengths differ, the UCF101 flow database misses one video and the K400 val RGB database
another (so K400_LMDB_2CLIP is read in train mode only), and the
lengths cover filtered, padded and multi-window videos.  write(root, spec, pool) puts it on disk:
root/split/{ucf101,hmdb51,k400}/ and root/data/ in the drivers' --data-root layout.
"""
import io
import json
import os
import random

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

POOL, H, W = 48, 224, 240
LENGTHS = [2, 5, 9, 14, 23, 30, 4, 17]
UCF_CLASSES = ["Apply Eye", "Bowling", "Cutting"]
K400_CLASSES = ["air drumming", "abseiling"]
RGB = "UCF101/ucf101_frame.lmdb"
FLOW = "UCF101/ucf101_tvl1_frame.lmdb"
HRGB = "HMDB51/hmdb51_frame.lmdb"
HFLOW = "HMDB51/hmdb51_tvl1_frame.lmdb"
KRGB = "kinetics400-256/frame_full/lmdb/k400_frame_%s.lmdb"
KFLOW = "kinetics400-256/tvl1_flow/lmdb/k400_tvl1_frame_%s.lmdb"


def pool(n=POOL, h=H, w=W, seed=0):
    """n distinct small JPEGs (Pillow, quality 75, 4:2:0): smooth colour fields plus a little noise."""
    from PIL import Image
    r = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = []
    for _ in range(n):
        fx, fy, ph = r.uniform(10, 40, 3), r.uniform(10, 40, 3), r.uniform(0, 6.3, 3)
        img = np.stack([128 + 90 * np.sin(xx / fx[c] + ph[c]) * np.cos(yy / fy[c]) for c in range(3)], -1)
        img = np.clip(img + r.normal(0, 4, img.shape), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(img).save(b, "JPEG", quality=75)
        out.append(b.getvalue())
    return out


def _frames(rng, n):
    start, step = rng.randrange(POOL), rng.choice([1, 5, 7, 11])
    return [(start + step * t) % POOL for t in range(n)]


def spec(seed=0):
    rng = random.Random(seed)
    files, dbs = {}, {}
    files["ucf101/ClassInd.txt"] = "".join("%d, %s\n" % (i + 1, c) for i, c in enumerate(UCF_CLASSES))
    files["hmdb51/ClassInd.txt"] = "".join("%s\n" % c for c in UCF_CLASSES)
    files["k400/ClassInd.txt"] = "".join("%s\n" % c for c in K400_CLASSES)
    k = 0
    rgb, flow, source = {}, {}, {}
    for split, per in (("train", 3), ("test", 2)):
        rows = []
        for ci, c in enumerate(UCF_CLASSES):
            tag = c.replace(" ", "")
            for v in range(per):
                g = 1 + v + (0 if split == "train" else 10)
                vid = "v_%s_g%02d_c%02d" % (tag, g, 1 + (v % 2))
                name = "%s/%s" % (c, vid)
                n = LENGTHS[k % len(LENGTHS)]
                k += 1
                rows.append("/data/UCF101/frame/%s/%s/,%d" % (c, vid, n))
                rgb[name] = _frames(rng, n)
                flow[name] = _frames(rng, max(1, n - (k % 3)))
                source.setdefault(vid[:-4], len(source))
        for i in (1, 2):
            files["ucf101/%s_split%02d.csv" % (split, i)] = "\n".join(rows if i == 1 else rows[::-1]) + "\n"
            files["hmdb51/%s_split%02d.csv" % (split, i)] = files["ucf101/%s_split%02d.csv" % (split, i)]
    files["ucf101/video_source.json"] = json.dumps(source)
    names = sorted(rgb)
    del flow[names[3]]                              # a video only the RGB database has
    for path, videos in ((RGB, rgb), (FLOW, flow), (HRGB, rgb), (HFLOW, flow)):
        order = sorted(videos)
        random.Random(len(path)).shuffle(order)
        dbs[path] = {"videos": videos, "order": order}
    ksource = {}
    for split in ("train", "val"):
        rows, kr, kf = [], {}, {}
        for c in K400_CLASSES + ["not a class"]:
            for v in range(3):
                vid = "%s%d_%06d_%06d" % ("xyz"[v], k, 10 * v, 10 * v + 10)
                n = LENGTHS[k % len(LENGTHS)] + 3
                k += 1
                rows.append("/data/kinetics400-256/%s_split/%s/%s,%d" % (split, c, vid, n))
                name = "%s/%s" % (c, vid)
                kr[name] = _frames(rng, n)
                kf[name] = _frames(rng, n - (k % 2))
                ksource.setdefault(name, len(ksource))
        files["k400/%s_split.csv" % split] = "\n".join(rows) + "\n"
        if split == "val":                          # a video only the flow database has: 2-stream drops it
            del kr[sorted(kr)[1]]
        for path, videos in ((KRGB % split, kr), (KFLOW % split, kf)):
            order = sorted(videos)
            random.Random(len(path) + len(split)).shuffle(order)
            dbs[path] = {"videos": videos, "order": order}
    files["k400/video_source.json"] = json.dumps(ksource)
    return {"files": files, "dbs": dbs}


def write(root, sp, jpegs, bin_type=True):
    """Split files under root/split, databases under root/data (lmdb_writer)."""
    import sys
    sys.path.insert(0, HERE)
    import lmdb_writer
    for rel, text in sp["files"].items():
        p = os.path.join(root, "split", rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            f.write(text)
    for rel, db in sp["dbs"].items():
        videos = {n: [jpegs[i] for i in idx] for n, idx in db["videos"].items()}
        lmdb_writer.write_videos(os.path.join(root, "data", rel), videos, db["order"], bin_type=bin_type)
    return os.path.join(root, "data"), os.path.join(root, "split")


def pool_to_arrays(jpegs):
    off = np.zeros(len(jpegs) + 1, np.int64)
    off[1:] = np.cumsum([len(j) for j in jpegs])
    return np.frombuffer(b"".join(jpegs), np.uint8), off


def pool_from_arrays(data, off):
    data = bytes(data)
    return [data[off[i]:off[i + 1]] for i in range(len(off) - 1)]
