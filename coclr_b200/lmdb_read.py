"""Read-only access to the reference's LMDB video databases with nothing beyond the standard library.

    db = lmdb_read.open(path)            # a directory (path/data.mdb) or the data file itself; the lock file is unused
    view = db.get(b'000000042')          # memoryview into the map, or None
    frames = lmdb_read.unpack(view)      # [memoryview of each frame's JPEG bytes]

The on-disk format is LMDB 0.9's (mdb.c) for a 64-bit little-endian build, which is what py-lmdb writes: a B+tree of
fixed-size pages.  Pages 0 and 1 hold the two meta records; the one with the larger txnid is current.  Only the main
database of a plain (no sub-databases, no duplicate keys) environment is read.  Every page and value is bounds-checked
against the file, so a damaged file raises ValueError naming the file, never a crash.

`unpack` decodes the msgpack subset the reference's values use.  Its converter ran msgpack 0.6.2, whose `dumps` writes
byte strings as the str family; files written with msgpack >= 1.0 use the bin family.  Both come back as memoryviews
(byte strings), so neither the `lmdb` nor the `msgpack` package is needed.
"""
import builtins
import mmap
import os
import struct

PAGEHDR = 16
P_BRANCH, P_LEAF, P_OVERFLOW, P_META, P_LEAF2 = 0x01, 0x02, 0x04, 0x08, 0x20
F_BIGDATA, F_SUBDATA, F_DUPDATA = 0x01, 0x02, 0x04
MAGIC, VERSION = 0xBEEFC0DE, 1
META = struct.Struct("<IIQQ" + "IHHQQQQQ" * 2 + "QQ")    # MDB_meta after the page header
NODE = struct.Struct("<HHHH")                            # lo, hi, flags, ksize
INVALID = (1 << 64) - 1
MAX_DEPTH = 64


class Reader:
    """One memory-mapped LMDB data file.  `get` returns zero-copy views, valid while the reader is open."""

    def __init__(self, path):
        self.path = path
        with builtins.open(path, "rb") as f:
            size = os.fstat(f.fileno()).st_size
            if size < 2 * PAGEHDR + META.size:
                raise ValueError("%s: not an LMDB data file (%d bytes)" % (path, size))
            self._map = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
        self.mem = memoryview(self._map)
        metas = [self._meta(0, 0)]
        psize = metas[0][0]
        if psize < 256 or psize & (psize - 1):
            raise ValueError("%s: invalid page size %d" % (path, psize))
        self.psize = psize
        self._page(1)
        metas.append(self._meta(psize, 1))
        _, flags, depth, entries, root, txnid = max(metas, key=lambda m: m[-1])
        if flags & 0x04:                                  # MDB_DUPSORT on the main database
            raise ValueError("%s: duplicate-sort databases are not supported" % path)
        self.depth, self.entries, self.root = depth, entries, root

    def _meta(self, off, pgno):
        if off + PAGEHDR + META.size > len(self.mem):
            raise ValueError("%s: meta page runs past the end of the file" % self.path)
        if not struct.unpack_from("<H", self.mem, off + 10)[0] & P_META:
            raise ValueError("%s: page %d is not a meta page" % (self.path, pgno))
        m = META.unpack_from(self.mem, off + PAGEHDR)
        magic, version = m[0], m[1]
        if magic != MAGIC:
            raise ValueError("%s: bad magic 0x%08x (not an LMDB file)" % (self.path, magic))
        if version != VERSION:
            raise ValueError("%s: unsupported LMDB data version %d" % (self.path, version))
        # m[4:12]: dbs[0] (free list), m[12:20]: dbs[1] (main) = pad, flags, depth, branch, leaf, overflow, entries, root
        main = m[12:20]
        return m[4], main[1], main[2], main[6], main[7], m[21]   # dbs[0].pad is the page size; txnid is last

    def _page(self, pgno):
        off = pgno * self.psize
        if pgno >= INVALID or off + self.psize > len(self.mem):
            raise ValueError("%s: page %d runs past the end of the file" % (self.path, pgno))
        return off

    def _nodes(self, off):
        lower, upper = struct.unpack_from("<HH", self.mem, off + 12)
        if lower < PAGEHDR or lower > upper or upper > self.psize or lower & 1:
            raise ValueError("%s: page %d has an invalid header" % (self.path, off // self.psize))
        n = (lower - PAGEHDR) >> 1
        return struct.unpack_from("<%dH" % n, self.mem, off + PAGEHDR)

    def _node(self, off, ptr):
        if ptr + NODE.size > self.psize:
            raise ValueError("%s: node runs past page %d" % (self.path, off // self.psize))
        lo, hi, flags, ks = NODE.unpack_from(self.mem, off + ptr)
        k0 = off + ptr + NODE.size
        if ptr + NODE.size + ks > self.psize:
            raise ValueError("%s: key runs past page %d" % (self.path, off // self.psize))
        return lo, hi, flags, self.mem[k0:k0 + ks], k0 + ks

    def get(self, key):
        """The value stored under `key` (bytes), as a memoryview into the map, or None."""
        key = bytes(key)
        if self.root == INVALID:
            return None
        pgno = self.root
        for _ in range(MAX_DEPTH):
            off = self._page(pgno)
            flags = struct.unpack_from("<H", self.mem, off + 10)[0]
            ptrs = self._nodes(off)
            if flags & P_LEAF2:
                raise ValueError("%s: duplicate-sort (LEAF2) pages are not supported" % self.path)
            if flags & P_BRANCH:
                if not ptrs:
                    raise ValueError("%s: empty branch page %d" % (self.path, pgno))
                lo_i, hi_i = 1, len(ptrs) - 1             # last child whose key <= key; key 0 is the empty key
                child = 0
                while lo_i <= hi_i:
                    mid = (lo_i + hi_i) >> 1
                    if bytes(self._node(off, ptrs[mid])[3]) <= key:
                        child, lo_i = mid, mid + 1
                    else:
                        hi_i = mid - 1
                lo, hi, nflags, _, _ = self._node(off, ptrs[child])
                pgno = lo | hi << 16 | nflags << 32
                continue
            if not flags & P_LEAF:
                raise ValueError("%s: page %d is neither a branch nor a leaf" % (self.path, pgno))
            lo_i, hi_i = 0, len(ptrs) - 1
            while lo_i <= hi_i:
                mid = (lo_i + hi_i) >> 1
                lo, hi, nflags, k, d0 = self._node(off, ptrs[mid])
                k = bytes(k)
                if k < key:
                    lo_i = mid + 1
                elif k > key:
                    hi_i = mid - 1
                else:
                    return self._value(off, lo | hi << 16, nflags, d0)
            return None
        raise ValueError("%s: tree deeper than %d levels" % (self.path, MAX_DEPTH))

    def _value(self, off, size, flags, d0):
        if flags & (F_SUBDATA | F_DUPDATA):
            raise ValueError("%s: sub-databases and duplicate data are not supported" % self.path)
        if flags & F_BIGDATA:
            if d0 + 8 > off + self.psize:
                raise ValueError("%s: overflow reference runs past page %d" % (self.path, off // self.psize))
            ov = self._page(struct.unpack_from("<Q", self.mem, d0)[0])
            if not struct.unpack_from("<H", self.mem, ov + 10)[0] & P_OVERFLOW:
                raise ValueError("%s: value points at a page that is not an overflow page" % self.path)
            d0 = ov + PAGEHDR
            if d0 + size > len(self.mem):
                raise ValueError("%s: value of %d bytes runs past the end of the file" % (self.path, size))
        elif d0 + size > off + self.psize:
            raise ValueError("%s: value runs past page %d" % (self.path, off // self.psize))
        return self.mem[d0:d0 + size]

    def close(self):
        """Unmap the file; views that `get` returned must no longer be in use."""
        self.mem.release()
        self._map.close()


def open(path):  # noqa: A001 -- mirrors lmdb.open(path, subdir=os.path.isdir(path), readonly=True, lock=False)
    """Open an LMDB environment read-only: a directory means path/data.mdb, a file means path itself."""
    return Reader(os.path.join(path, "data.mdb") if os.path.isdir(path) else path)


def unpack(view):
    """Decode one msgpack value (the subset of the reference's files): nil, bool, ints, arrays, and the str and bin
    families as memoryviews."""
    view = memoryview(view).cast("B")
    obj, end = _unpack(view, 0)
    if end != len(view):
        raise ValueError("msgpack value has %d trailing bytes" % (len(view) - end))
    return obj


_FIXED = {0xcc: "<B", 0xcd: ">H", 0xce: ">I", 0xcf: ">Q", 0xd0: ">b", 0xd1: ">h", 0xd2: ">i", 0xd3: ">q"}
_RAW = {0xd9: ">B", 0xda: ">H", 0xdb: ">I", 0xc4: ">B", 0xc5: ">H", 0xc6: ">I"}      # str8/16/32, bin8/16/32
_ARR = {0xdc: ">H", 0xdd: ">I"}


def _take(v, pos, n):
    if pos + n > len(v):
        raise ValueError("msgpack value is truncated")
    return pos + n


def _unpack(v, pos):
    end = _take(v, pos, 1)
    b = v[pos]
    if b <= 0x7f:
        return b, end
    if b >= 0xe0:
        return b - 0x100, end
    if 0xa0 <= b <= 0xbf:
        n = b & 0x1f
        return v[end:_take(v, end, n)], end + n
    if 0x90 <= b <= 0x9f:
        return _array(v, end, b & 0x0f)
    if b == 0xc0:
        return None, end
    if b in (0xc2, 0xc3):
        return b == 0xc3, end
    if b in _FIXED:
        fmt = _FIXED[b]
        p = _take(v, end, struct.calcsize(fmt))
        return struct.unpack_from(fmt, v, end)[0], p
    if b in _RAW:
        fmt = _RAW[b]
        p = _take(v, end, struct.calcsize(fmt))
        n = struct.unpack_from(fmt, v, end)[0]
        return v[p:_take(v, p, n)], p + n
    if b in _ARR:
        fmt = _ARR[b]
        p = _take(v, end, struct.calcsize(fmt))
        return _array(v, p, struct.unpack_from(fmt, v, end)[0])
    raise ValueError("msgpack type 0x%02x is not used by the reference's databases" % b)


def _array(v, pos, n):
    out = []
    for _ in range(n):
        x, pos = _unpack(v, pos)
        out.append(x)
    return out, pos
