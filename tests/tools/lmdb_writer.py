"""Writes LMDB data files by LMDB 0.9's on-disk layout (64-bit little-endian), for test fixtures: a bulk-loaded B+tree
with values too large for a node in overflow pages, exactly as `coclr_b200.lmdb_read` expects to find them.

    write(path, {b'key': b'value', ...})                 # path/data.mdb (subdir=True) or path itself
    pack(obj, bin_type=True)                             # the msgpack subset of the reference's values

Test-only knobs build the files the reader must reject or see through: `psize`, a stale meta (`stale_meta`: the
other meta slot holds an older txnid whose root is `stale_root`), and `node_flags` (extra leaf node flags per key).
"""
import os
import struct

PAGEHDR = 16
P_BRANCH, P_LEAF, P_OVERFLOW, P_META = 0x01, 0x02, 0x04, 0x08
F_BIGDATA = 0x01
INVALID = (1 << 64) - 1
META = struct.Struct("<IIQQ" + "IHHQQQQQ" * 2 + "QQ")


def _even(n):
    return n + (n & 1)


class _Pages:
    def __init__(self, psize):
        self.psize, self.pages = psize, [None, None]

    def add(self, data):
        self.pages.append(data)
        return len(self.pages) - 1

    def reserve(self, n):
        first = len(self.pages)
        self.pages.extend([b""] * n)
        return first


def _page(psize, pgno, flags, nodes):
    """A branch or leaf page from [(node bytes)] in key order."""
    buf = bytearray(psize)
    upper = psize
    ptrs = []
    for nb in nodes:
        upper -= _even(len(nb))
        buf[upper:upper + len(nb)] = nb
        ptrs.append(upper)
    lower = PAGEHDR + 2 * len(ptrs)
    assert lower <= upper, "page overflow"
    struct.pack_into("<QHHHH", buf, 0, pgno, 0, flags, lower, upper)
    struct.pack_into("<%dH" % len(ptrs), buf, PAGEHDR, *ptrs)
    return bytes(buf)


def write(path, items, psize=4096, subdir=True, stale_meta=False, stale_root=INVALID, node_flags=None):
    """Write `items` (dict of bytes -> bytes) as an LMDB environment; returns the data file's path."""
    node_flags = node_flags or {}
    nodemax = (((psize - PAGEHDR) // 2) & ~1) - 2              # mdb.c me_nodemax with MDB_MINKEYS = 2
    pages = _Pages(psize)
    keys = sorted(items)
    overflow_pages = 0
    leaves, cur, used = [], [], 0
    for k in keys:
        v = bytes(items[k])
        flags = node_flags.get(k, 0)
        if 8 + len(k) + len(v) > nodemax:                    # value goes to overflow pages
            n = (PAGEHDR + len(v) + psize - 1) // psize
            first = pages.reserve(n)
            blob = bytearray(n * psize)
            struct.pack_into("<QHHI", blob, 0, first, 0, P_OVERFLOW, n)
            blob[PAGEHDR:PAGEHDR + len(v)] = v
            for i in range(n):
                pages.pages[first + i] = bytes(blob[i * psize:(i + 1) * psize])
            overflow_pages += n
            data, flags = struct.pack("<Q", first), flags | F_BIGDATA
        else:
            data = v
        node = struct.pack("<HHHH", len(v) & 0xffff, len(v) >> 16, flags, len(k)) + k + data
        need = _even(len(node)) + 2
        if cur and used + need > psize - PAGEHDR:
            leaves.append(cur)
            cur, used = [], 0
        cur.append((k, node))
        used += need
    if cur:
        leaves.append(cur)
    level = []
    for nodes in leaves:
        pg = pages.reserve(1)
        pages.pages[pg] = _page(psize, pg, P_LEAF, [n for _, n in nodes])
        level.append((nodes[0][0], pg))
    depth, branch_pages = (1 if level else 0), 0
    while len(level) > 1:
        nxt, cur, used = [], [], 0
        for i, (k, pg) in enumerate(level):
            key = b"" if not cur else k                          # a branch page's first key is empty
            node = struct.pack("<HHHH", pg & 0xffff, (pg >> 16) & 0xffff, pg >> 32, len(key)) + key
            need = _even(len(node)) + 2
            if cur and used + need > psize - PAGEHDR:
                nxt.append(cur)
                node = struct.pack("<HHHH", pg & 0xffff, (pg >> 16) & 0xffff, pg >> 32, 0)
                cur, used, need = [], 0, 10
            cur.append((k, node))
            used += need
        nxt.append(cur)
        level = []
        for nodes in nxt:
            pg = pages.reserve(1)
            pages.pages[pg] = _page(psize, pg, P_BRANCH, [n for _, n in nodes])
            level.append((nodes[0][0], pg))
            branch_pages += 1
        depth += 1
    root = level[0][1] if level else INVALID
    last = len(pages.pages) - 1
    for slot in (0, 1):
        current = slot == 1
        txnid = 2 if current else 1
        r = root if (current or not stale_meta) else stale_root
        if not stale_meta and not current:
            txnid = 1                                            # an older, identical commit
        buf = bytearray(psize)
        struct.pack_into("<QHHHH", buf, 0, slot, 0, P_META, 0, 0)
        META.pack_into(buf, PAGEHDR, 0xBEEFC0DE, 1, 0, (last + 1) * psize,
                       psize, 0, 0, 0, 0, 0, 0, INVALID,
                       0, 0, depth, branch_pages, len(leaves), overflow_pages, len(keys), r,
                       last, txnid)
        pages.pages[slot] = bytes(buf)
    if subdir:
        os.makedirs(path, exist_ok=True)
        path = os.path.join(path, "data.mdb")
    with open(path, "wb") as f:
        for p in pages.pages:
            f.write(p)
    return path


def pack(obj, bin_type=True):
    """msgpack of None / bool / int / bytes / str / list: byte strings as bin (msgpack >= 1.0) or, bin_type=False, as
    str (msgpack 0.6.2's dumps, what the reference's converter wrote)."""
    out = []
    _pack(obj, bin_type, out)
    return b"".join(out)


def _pack(o, bt, out):
    if o is None:
        out.append(b"\xc0")
    elif o is True or o is False:
        out.append(b"\xc3" if o else b"\xc2")
    elif isinstance(o, int):
        if 0 <= o < 128:
            out.append(bytes([o]))
        elif -32 <= o < 0:
            out.append(bytes([o & 0xff]))
        elif o >= 0:
            for t, f in ((0xcc, ">B"), (0xcd, ">H"), (0xce, ">I"), (0xcf, ">Q")):
                if o < 1 << (8 * struct.calcsize(f)):
                    out.append(bytes([t]) + struct.pack(f, o))
                    break
        else:
            for t, f in ((0xd0, ">b"), (0xd1, ">h"), (0xd2, ">i"), (0xd3, ">q")):
                if o >= -(1 << (8 * struct.calcsize(f) - 1)):
                    out.append(bytes([t]) + struct.pack(f, o))
                    break
    elif isinstance(o, (bytes, bytearray, memoryview, str)):
        b = o.encode() if isinstance(o, str) else bytes(o)
        n = len(b)
        if bt and not isinstance(o, str):
            head = (bytes([0xc4, n]) if n < 256 else b"\xc5" + struct.pack(">H", n) if n < 65536
                    else b"\xc6" + struct.pack(">I", n))
        else:
            # msgpack's old raw spec (use_bin_type=False) has no str8: fixstr, str16, str32
            head = (bytes([0xa0 | n]) if n < 32 else b"\xda" + struct.pack(">H", n) if n < 65536
                    else b"\xdb" + struct.pack(">I", n))
        out.append(head + b)
    elif isinstance(o, (list, tuple)):
        n = len(o)
        out.append(bytes([0x90 | n]) if n < 16 else b"\xdc" + struct.pack(">H", n) if n < 65536
                   else b"\xdd" + struct.pack(">I", n))
        for x in o:
            _pack(x, bt, out)
    else:
        raise TypeError(type(o))


def write_videos(path, videos, order, bin_type=True, **kw):
    """A database in the reference converter's layout: `videos` maps a video name ('class/video') to its list of JPEG
    byte strings, `order` is the shuffled name list (`__order__`); video order[i] is stored under '%09d' % i.  The
    special keys hold the reference's `__keys__` (per-video keys in sorted-name order), `__len__`, `__order__` and
    `__vlen__` (frame counts in `__keys__` order)."""
    vid = {n: "%09d" % i for i, n in enumerate(order)}
    names = sorted(videos)
    items = {vid[n].encode(): pack(list(videos[n]), bin_type) for n in names}
    keys = [vid[n].encode() for n in names]
    items[b"__keys__"] = pack(keys, bin_type)
    items[b"__len__"] = pack(len(keys), bin_type)
    items[b"__order__"] = pack([n.encode() for n in order], bin_type)
    items[b"__vlen__"] = pack([len(videos[n]) for n in names], bin_type)
    return write(path, items, **kw)
