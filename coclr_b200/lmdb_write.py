"""Streaming writer of LMDB data files in LMDB 0.9's on-disk layout (64-bit little-endian), the layout `lmdb_read`
parses and py-lmdb reads, for databases far larger than memory.

    with lmdb_write.Writer(path) as db:      # a directory (path/data.mdb) or, subdir=False, the data file itself
        db.put(b'000000000', pack([...]))    # keys in strictly increasing byte order
    pack(obj, bin_type=True)                 # the msgpack subset of the reference's values

Values too large for a leaf node go to overflow pages, written at once; a leaf page is written when it is full.  Only
each leaf page's first key and page number stay in memory; the branch levels and the two meta pages are written at
`close()` (the meta pages last, into the file's first two pages), so a file whose `close()` did not run has no valid
meta page and is never mistaken for a complete database.
"""
import os
import struct

PAGEHDR = 16
P_BRANCH, P_LEAF, P_OVERFLOW, P_META = 0x01, 0x02, 0x04, 0x08
F_BIGDATA = 0x01
INVALID = (1 << 64) - 1
MAGIC, VERSION = 0xBEEFC0DE, 1
META = struct.Struct("<IIQQ" + "IHHQQQQQ" * 2 + "QQ")    # MDB_meta after the page header
MAX_KEY = 511                                            # mdb.c MDB_MAXKEYSIZE


def _even(n):
    return n + (n & 1)


def _page(psize, pgno, flags, nodes):
    """A branch or leaf page from its node byte strings in key order."""
    buf = bytearray(psize)
    upper = psize
    ptrs = []
    for nb in nodes:
        upper -= _even(len(nb))
        buf[upper:upper + len(nb)] = nb
        ptrs.append(upper)
    lower = PAGEHDR + 2 * len(ptrs)
    struct.pack_into("<QHHHH", buf, 0, pgno, 0, flags, lower, upper)
    struct.pack_into("<%dH" % len(ptrs), buf, PAGEHDR, *ptrs)
    return buf


def _branch_node(pgno, key):
    return struct.pack("<HHHH", pgno & 0xffff, (pgno >> 16) & 0xffff, pgno >> 32, len(key)) + key


class Writer:
    """Writes one LMDB environment front to back.  `put` takes keys in strictly increasing order (ValueError
    otherwise); `close` finishes the file.  An existing data file is refused."""

    def __init__(self, path, subdir=True, psize=4096):
        if psize < 512 or psize & (psize - 1):
            raise ValueError("page size must be a power of two >= 512, got %d" % psize)
        if subdir:
            os.makedirs(path, exist_ok=True)
            path = os.path.join(path, "data.mdb")
        self.path, self.psize = path, psize
        self.nodemax = (((psize - PAGEHDR) // 2) & ~1) - 2     # mdb.c me_nodemax with MDB_MINKEYS = 2
        self._f = open(path, "xb")
        self._f.write(bytes(2 * psize))                         # the meta pages, written at close()
        self._next = 2                                          # next page number
        self._leaf, self._used = [], 0                          # nodes of the leaf page being filled
        self._leaves = []                                       # (first key, page number) of every written leaf
        self._last = None
        self.entries = self.overflow_pages = self.branch_pages = 0
        self.depth = 0

    def __enter__(self):
        return self

    def __exit__(self, exc_type, *_):
        if exc_type is None:
            self.close()
        else:
            self.abort()

    def abort(self):
        """Close the file without finishing it: its meta pages stay zero, so no reader takes it for a database."""
        if self._f is not None:
            self._f.close()
            self._f = None

    def _write(self, data):
        self._f.write(data)
        self._next += len(data) // self.psize

    def put(self, key, value):
        key, value = bytes(key), bytes(value)
        if not 0 < len(key) <= MAX_KEY:
            raise ValueError("key length must be 1 .. %d bytes, got %d" % (MAX_KEY, len(key)))
        if self._last is not None and key <= self._last:
            raise ValueError("keys must arrive in strictly increasing order: %r after %r" % (key, self._last))
        if len(value) >= 1 << 32:
            raise ValueError("value of %d bytes is too large" % len(value))
        self._last = key
        flags = 0
        if 8 + len(key) + len(value) > self.nodemax:           # the value goes to overflow pages, written now
            n = (PAGEHDR + len(value) + self.psize - 1) // self.psize
            first = self._next
            self._write(struct.pack("<QHHI", first, 0, P_OVERFLOW, n) + value +
                        bytes(n * self.psize - PAGEHDR - len(value)))
            self.overflow_pages += n
            data, flags = struct.pack("<Q", first), F_BIGDATA
        else:
            data = value
        node = struct.pack("<HHHH", len(value) & 0xffff, len(value) >> 16, flags, len(key)) + key + data
        need = _even(len(node)) + 2
        if self._leaf and self._used + need > self.psize - PAGEHDR:
            self._flush_leaf()
        self._leaf.append((key, node))
        self._used += need
        self.entries += 1

    def _flush_leaf(self):
        pg = self._next
        self._write(_page(self.psize, pg, P_LEAF, [n for _, n in self._leaf]))
        self._leaves.append((self._leaf[0][0], pg))
        self._leaf, self._used = [], 0

    def close(self):
        """Write the last leaf, the branch levels and the meta pages; returns the data file's path."""
        if self._f is None:
            return self.path
        if self._leaf:
            self._flush_leaf()
        level = self._leaves
        self.depth = 1 if level else 0
        while len(level) > 1:
            groups, cur, used = [], [], 0
            for k, pg in level:
                node = _branch_node(pg, k if cur else b"")      # a branch page's first key is empty
                need = _even(len(node)) + 2
                if cur and used + need > self.psize - PAGEHDR:
                    groups.append(cur)
                    node = _branch_node(pg, b"")
                    cur, used, need = [], 0, _even(len(node)) + 2
                cur.append((k, node))
                used += need
            groups.append(cur)
            level = []
            for nodes in groups:
                pg = self._next
                self._write(_page(self.psize, pg, P_BRANCH, [n for _, n in nodes]))
                level.append((nodes[0][0], pg))
                self.branch_pages += 1
            self.depth += 1
        root = level[0][1] if level else INVALID
        last = self._next - 1
        for slot in (0, 1):
            buf = bytearray(self.psize)
            struct.pack_into("<QHHHH", buf, 0, slot, 0, P_META, 0, 0)
            META.pack_into(buf, PAGEHDR, MAGIC, VERSION, 0, (last + 1) * self.psize,
                           self.psize, 0, 0, 0, 0, 0, 0, INVALID,
                           0, 0, self.depth, self.branch_pages, len(self._leaves), self.overflow_pages,
                           self.entries, root, last, slot + 1)
            self._f.seek(slot * self.psize)
            self._f.write(buf)
        self._f.flush()
        os.fsync(self._f.fileno())
        self._f.close()
        self._f = None
        return self.path


def pack(obj, bin_type=True):
    """msgpack of None / bool / int / bytes / str / list: byte strings in the bin family (msgpack >= 1.0) or,
    bin_type=False, the str family (msgpack 0.6.2's `dumps`, which the reference's converter ran)."""
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
            t, f = next((t, f) for t, f in ((0xcc, ">B"), (0xcd, ">H"), (0xce, ">I"), (0xcf, ">Q"))
                        if o < 1 << (8 * struct.calcsize(f)))
            out.append(bytes([t]) + struct.pack(f, o))
        else:
            t, f = next((t, f) for t, f in ((0xd0, ">b"), (0xd1, ">h"), (0xd2, ">i"), (0xd3, ">q"))
                        if o >= -(1 << (8 * struct.calcsize(f) - 1)))
            out.append(bytes([t]) + struct.pack(f, o))
    elif isinstance(o, (bytes, bytearray, memoryview, str)):
        b = o.encode() if isinstance(o, str) else bytes(o)
        n = len(b)
        if bt and not isinstance(o, str):
            head = (bytes([0xc4, n]) if n < 256 else b"\xc5" + struct.pack(">H", n) if n < 65536
                    else b"\xc6" + struct.pack(">I", n))
        else:   # msgpack's old raw family (use_bin_type=False) has no str8: fixstr, str16, str32
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
        raise TypeError("cannot pack %s" % type(o).__name__)


def bin_family(view):
    """True when the msgpack value `view` (an array of byte strings, or a byte string) stores its byte strings in the
    bin family, False for the str family, None when it holds none."""
    v = memoryview(view).cast("B")
    pos = 0
    if len(v) and (0x90 <= v[0] <= 0x9f or v[0] in (0xdc, 0xdd)):
        if v[0] <= 0x9f and v[0] == 0x90:
            return None
        pos = 1 if v[0] <= 0x9f else 3 if v[0] == 0xdc else 5
    if pos >= len(v):
        return None
    b = v[pos]
    if b in (0xc4, 0xc5, 0xc6):
        return True
    if 0xa0 <= b <= 0xbf or b in (0xd9, 0xda, 0xdb):
        return False
    return None
