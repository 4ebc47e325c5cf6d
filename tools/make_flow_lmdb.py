"""Build a TV-L1 flow LMDB from an RGB frame LMDB in the reference's layout, on the GPU.

    python tools/make_flow_lmdb.py --rgb ucf101_frame.lmdb --out ucf101_tvl1_frame.lmdb [--pairs 64]

Every video of the RGB database (keys '%09d', in key order) is decoded on the GPU (coclr_b200.jpeg), converted to
grey, and its N - 1 consecutive frame pairs are solved with coclr_b200.flow.tvl1 in chunks of at most --pairs pairs.
The flow is quantised to 8-bit frames on the GPU (coclr_b200.flow.LAYOUT) and each chunk is JPEG-encoded there too
(coclr_b200.jpeg.JpegEncoder, QUALITY, SUBSAMPLING), byte-identical to `encode`, Pillow's encoder: only the JPEG bytes
come back to the host.  The video's list of JPEGs is stored under the same key, then `__keys__`, `__len__` and
`__order__` as the RGB database has them and `__vlen__` with the flow frame counts (N - 1) in `__keys__` order.  The flow frames use the msgpack family (str or bin) of the RGB database's
byte strings, `__keys__` and frames, so a reader of the RGB database reads this one.  A one-frame video gets an empty
list.

Refused, with a message: an existing --out, a video whose frames differ in size and a frame that cannot be decoded
(both name the video).  A refused or failed run removes the partial output.
"""
import argparse
import io
import os
import shutil
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

QUALITY = 95          # Pillow JPEG quality of a stored flow frame
SUBSAMPLING = 0       # 4:4:4: the two flow channels are not smoothed by chroma subsampling


class Refused(Exception):
    pass


def encode(frame):
    """One uint8 [H, W, 3] flow frame as the JPEG bytes the database stores."""
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(frame).save(b, "JPEG", quality=QUALITY, subsampling=SUBSAMPLING)
    return b.getvalue()


def solve_video(dec, enc, jpegs, pairs, name, stats):
    """The JPEG files of one video's N - 1 quantised flow frames; stats["encode_s"] gains the encode time."""
    import torch
    from coclr_b200 import flow
    from coclr_b200.jpeg import JpegFrameError
    n = len(jpegs)
    if n == 0:
        return []
    try:
        batch = dec.parse(jpegs)
    except JpegFrameError as e:
        raise Refused("video %s: cannot decode %s" % (name, e))
    sizes = sorted(set(batch.sizes))
    if len(sizes) != 1:
        raise Refused("video %s: its frames differ in size: %s" % (name, ", ".join("%dx%d" % s for s in sizes)))
    try:
        rgb = dec(batch)
    except ValueError as e:
        raise Refused("video %s: cannot decode %s" % (name, e))
    if n == 1:                                      # decoded all the same: a bad single frame is refused too
        return []
    grey = flow.grey(rgb)
    out = []
    for a in range(0, n - 1, pairs):
        b = min(a + pairs, n - 1)
        f, _ = flow.tvl1(grey[a:b], grey[a + 1:b + 1])
        q = flow.quantise(f)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out += enc(q)                               # synchronises: the files are on the host when it returns
        stats["encode_s"] += time.perf_counter() - t0
    return out


def frame_family(keys_value):
    """True when the RGB database stores byte strings in msgpack's bin family, False for the str family, judged from
    `__keys__`.  The keys and the frames are byte strings, so they share a family: msgpack >= 1.0 writes bin and
    msgpack 0.6.2's `dumps` writes str.  `__order__` is no guide: the converter writes it as a list of Python str,
    which every msgpack stores as str.  A database without videos gets bin."""
    from coclr_b200 import lmdb_write
    bt = lmdb_write.bin_family(keys_value)
    return True if bt is None else bt


def build(rgb_path, out_path, pairs, log=print):
    """Write the flow database of rgb_path to out_path (which must not exist); returns the run's figures."""
    import torch
    from coclr_b200 import lmdb_read, lmdb_write
    from coclr_b200.jpeg import JpegDecoder, JpegEncoder
    if os.path.exists(out_path):
        raise Refused("%s exists; remove it or choose another --out" % out_path)
    src = lmdb_read.open(rgb_path)
    special = {k: src.get(k) for k in (b"__keys__", b"__len__", b"__order__")}
    missing = [k.decode() for k, v in special.items() if v is None]
    if missing:
        raise Refused("%s: not a frame database in the reference's layout (no %s)" % (rgb_path, ", ".join(missing)))
    keys = [bytes(k) for k in lmdb_read.unpack(special[b"__keys__"])]
    order = [bytes(k).decode() for k in lmdb_read.unpack(special[b"__order__"])]
    bt = frame_family(special[b"__keys__"])
    if not torch.cuda.is_available():
        raise Refused("no CUDA device: the flow is computed on the GPU")
    dec = JpegDecoder()
    enc = JpegEncoder(QUALITY, SUBSAMPLING)
    vlen, stats = {}, {"videos": 0, "pairs": 0, "solve_s": 0.0, "encode_s": 0.0}
    t_start = time.perf_counter()
    writer = lmdb_write.Writer(out_path)
    try:
        for key in sorted(set(keys)):
            raw = src.get(key)
            if raw is None:
                raise Refused("%s: key %s is listed in __keys__ but not stored" % (rgb_path, key.decode()))
            i = int(key)
            name = "%s (key %s)" % (order[i] if 0 <= i < len(order) else "?", key.decode())
            t0, e0 = time.perf_counter(), stats["encode_s"]
            files = solve_video(dec, enc, [bytes(f) for f in lmdb_read.unpack(raw)], pairs, name, stats)
            stats["solve_s"] += time.perf_counter() - t0 - (stats["encode_s"] - e0)
            writer.put(key, lmdb_write.pack(files, bt))
            vlen[key] = len(files)
            stats["videos"] += 1
            stats["pairs"] += len(files)
        writer.put(b"__keys__", special[b"__keys__"])
        writer.put(b"__len__", special[b"__len__"])
        writer.put(b"__order__", special[b"__order__"])
        writer.put(b"__vlen__", lmdb_write.pack([vlen[k] for k in keys], bt))
        writer.close()
    except BaseException:
        writer.abort()
        shutil.rmtree(out_path, ignore_errors=True)
        raise
    wall = time.perf_counter() - t_start
    stats["pairs_per_s"] = stats["pairs"] / wall if wall > 0 else 0.0
    log("videos %d  pairs %d  pairs/s %.1f  solve %.1f s  encode %.1f s (GPU, synchronised)"
        % (stats["videos"], stats["pairs"], stats["pairs_per_s"], stats["solve_s"], stats["encode_s"]))
    return stats


def main(argv=None):
    ap = argparse.ArgumentParser(description="Build a TV-L1 flow LMDB from an RGB frame LMDB on the GPU.")
    ap.add_argument("--rgb", required=True, help="the RGB frame database (directory with data.mdb, or the file)")
    ap.add_argument("--out", required=True, help="the flow database to create (a directory; must not exist)")
    ap.add_argument("--pairs", type=int, default=64, help="frame pairs per solve (default 64)")
    args = ap.parse_args(argv)
    if args.pairs < 1:
        ap.error("--pairs must be >= 1")
    if not os.path.exists(args.rgb):
        ap.error("--rgb %s does not exist" % args.rgb)
    if os.path.exists(args.out):
        ap.error("--out %s exists; remove it or choose another path" % args.out)
    try:
        build(args.rgb, args.out, args.pairs)
    except Refused as e:
        ap.exit(2, "%s: error: %s\n" % (ap.prog, e))
    return 0


if __name__ == "__main__":
    sys.exit(main())
