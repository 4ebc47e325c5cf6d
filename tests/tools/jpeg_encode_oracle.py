"""A numpy JPEG encoder with the arithmetic of Pillow's libjpeg(-turbo) baseline path, written from the algorithm
libjpeg documents (ITU T.81, the IJG's jfdctint / jccolor / jcsample / jchuff descriptions), as the reference that
csrc/jpeg_encode.cu is tested against.

    raw = encode(rgb, quality=75, subsampling=2)      # == Image.fromarray(rgb).save(b, "JPEG", quality=.., subsampling=..)

Forward path: fixed-point RGB -> YCbCr (16 fraction bits), edge replication to whole blocks, 2:1 downsampling with
libjpeg's alternating bias, the ISLOW forward DCT (13 constant bits, 2 pass-1 bits), quantisation by rounded division
against 8 q, then sequential Huffman coding with the Annex K tables, 0xFF stuffing and 1-bit padding.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# ITU T.81 Annex K.1 / K.2: the example luminance and chrominance quant tables, natural order
STD_QUANT = np.array([
    [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
     14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99],
    [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
     47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32])

# ITU T.81 Annex K.3: (bits, values) of DC 0, AC 0, DC 1, AC 1
DC_BITS = [[0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]]
DC_VALS = [list(range(12))] * 2
AC_BITS = [[0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]]
AC_VALS = [
    [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
     0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
     0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
     0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
     0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
     0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
     0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
     0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa],
    [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
     0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
     0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
     0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
     0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
     0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
     0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
     0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa]]
SAMPLING = {0: (1, 1), 1: (2, 1), 2: (2, 2)}      # Pillow's subsampling -> luma (h, v) factors; chroma is 1 x 1


def quant_tables(quality):
    """libjpeg's jpeg_set_quality(quality, force_baseline=TRUE): [2, 64] natural order."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((STD_QUANT * scale + 50) // 100, 1, 255)


def huff_codes(bits, vals):
    """symbol -> (code, length) of a canonical table."""
    tab, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            tab[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return tab


def _lut(bits, vals):
    code, size = np.zeros(256, np.int64), np.zeros(256, np.int64)
    for s, (c, l) in huff_codes(bits, vals).items():
        code[s], size[s] = c, l
    return code, size


LUTS = [(_lut(DC_BITS[t], DC_VALS[t]), _lut(AC_BITS[t], AC_VALS[t])) for t in range(2)]


def header(h, w, quality=75, subsampling=2):
    """The bytes before the entropy-coded segment: SOI, JFIF APP0, DQT 0, DQT 1, SOF0, DHT DC0 AC0 DC1 AC1, SOS."""
    hs, vs = SAMPLING[subsampling]
    qt = quant_tables(quality)
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    for t in range(2):
        out += bytes([0xff, 0xdb, 0, 67, t]) + bytes(int(v) for v in qt[t][ZIGZAG])
    out += bytes([0xff, 0xc0, 0, 17, 8, h >> 8, h & 255, w >> 8, w & 255, 3,
                  1, (hs << 4) | vs, 0, 2, 0x11, 1, 3, 0x11, 1])
    for t in range(2):
        for cls, bits, vals in ((0, DC_BITS[t], DC_VALS[t]), (1, AC_BITS[t], AC_VALS[t])):
            n = 3 + 16 + len(vals)
            out += bytes([0xff, 0xc4, n >> 8, n & 255, (cls << 4) | t]) + bytes(bits) + bytes(vals)
    out += bytes([0xff, 0xda, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    return bytes(out)


def ycc(rgb):
    """jccolor's fixed-point conversion: int64 Y, Cb, Cr planes."""
    R, G, B = (rgb[..., i].astype(np.int64) for i in range(3))
    fix = lambda v: int(v * 65536 + 0.5)                                       # noqa: E731
    y = (fix(0.299) * R + fix(0.587) * G + fix(0.114) * B + 32768) >> 16
    cb = (-fix(0.16874) * R - fix(0.33126) * G + fix(0.5) * B + (128 << 16) + 32767) >> 16
    cr = (fix(0.5) * R - fix(0.41869) * G - fix(0.08131) * B + (128 << 16) + 32767) >> 16
    return y, cb, cr


def chroma_plane(p, hs, vs, cw, ch):
    """A chroma plane downsampled to cw x ch blocks of samples.  Columns: the input is replicated to 2 cw * 8 (h2)
    before downsampling.  Rows: the input is replicated to whole row groups; the downsampled plane's last real row is
    then replicated down to the block boundary."""
    h, w = p.shape
    if hs == 1:
        return np.pad(p, ((0, ch * 8 - h), (0, cw * 8 - w)), mode="edge")
    rows = -(-h // vs) * vs
    x = np.pad(p, ((0, rows - h), (0, cw * 16 - w)), mode="edge")
    if vs == 2:
        s = x[0::2, 0::2] + x[0::2, 1::2] + x[1::2, 0::2] + x[1::2, 1::2]
        d = (s + np.tile([1, 2], cw * 4)[None]) >> 2
    else:
        s = x[:, 0::2] + x[:, 1::2]
        d = (s + np.tile([0, 1], cw * 4)[None]) >> 1
    return np.pad(d, ((0, ch * 8 - d.shape[0]), (0, 0)), mode="edge")


# jfdctint's constants: FIX(x) = round(x * 2^13)
_F = {k: int(v * 8192 + 0.5) for k, v in dict(
    c0298=0.298631336, c0390=0.390180644, c0541=0.541196100, c0765=0.765366865, c0899=0.899976223,
    c1175=1.175875602, c1501=1.501321110, c1847=1.847759065, c1961=1.961570560, c2053=2.053119869,
    c2562=2.562915447, c3072=3.072711026).items()}


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct1(d, last):
    F = _F
    t0, t7, t1, t6 = d[0] + d[7], d[0] - d[7], d[1] + d[6], d[1] - d[6]
    t2, t5, t3, t4 = d[2] + d[5], d[2] - d[5], d[3] + d[4], d[3] - d[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = [None] * 8
    if last:
        o[0], o[4], s = _descale(t10 + t11, 2), _descale(t10 - t11, 2), 15
    else:
        o[0], o[4], s = (t10 + t11) << 2, (t10 - t11) << 2, 11
    z1 = (t12 + t13) * F["c0541"]
    o[2] = _descale(z1 + t13 * F["c0765"], s)
    o[6] = _descale(z1 - t12 * F["c1847"], s)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F["c1175"]
    t4, t5, t6, t7 = t4 * F["c0298"], t5 * F["c2053"], t6 * F["c3072"], t7 * F["c1501"]
    z1, z2 = -z1 * F["c0899"], -z2 * F["c2562"]
    z3, z4 = -z3 * F["c1961"] + z5, -z4 * F["c0390"] + z5
    o[7], o[5] = _descale(t4 + z1 + z3, s), _descale(t5 + z2 + z4, s)
    o[3], o[1] = _descale(t6 + z2 + z3, s), _descale(t7 + z1 + z4, s)
    return o


def fdct(b):
    """ISLOW forward DCT of int64 [..., 8, 8] samples minus 128; outputs scaled by 8 as libjpeg's."""
    r = np.stack(_fdct1([b[..., :, i] for i in range(8)], False), -1)
    return np.stack(_fdct1([r[..., i, :] for i in range(8)], True), -2)


def quantise(c, q):
    q = q.astype(np.int64) * 8
    a = (np.abs(c) + (q >> 1)) // q
    return np.where(c < 0, -a, a)


def _blocks(p, bh, bw):
    return p[:bh * 8, :bw * 8].reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3)


def coefficients(rgb, quality=75, subsampling=2):
    """Quantised int64 coefficient blocks in scan order, natural order within a block: [mcus_y * mcus_x * (hs vs
    + 2), 64], with the luma dummy blocks of a partial last MCU column / row."""
    h, w, _ = rgb.shape
    hs, vs = SAMPLING[subsampling]
    qt = quant_tables(quality)
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    wb, hb = -(-w // 8), -(-h // 8)                 # real luma blocks
    Y, Cb, Cr = ycc(rgb)
    yp = np.pad(Y, ((0, hb * 8 - h), (0, wb * 8 - w)), mode="edge")
    yc = quantise(fdct(_blocks(yp, hb, wb) - 128).reshape(hb, wb, 64), qt[0])
    luma = np.zeros((my * vs, mx * hs, 64), np.int64)
    luma[:hb, :wb] = yc
    luma[:hb, wb:, 0] = yc[:, wb - 1:wb, 0]          # right dummies: the last real block's DC, no AC
    for by in range(hb, my * vs):                   # bottom dummies: the DC of the MCU's previous block
        for bx in range(mx * hs):
            m = bx // hs
            luma[by, bx, 0] = luma[by - 1, m * hs + hs - 1, 0]
    chroma = []
    for p in (Cb, Cr):
        d = chroma_plane(p, hs, vs, mx, my)
        chroma.append(quantise(fdct(_blocks(d, my, mx) - 128).reshape(my, mx, 64), qt[1]))
    lum = luma.reshape(my, vs, mx, hs, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, vs * hs, 64)
    scan = np.concatenate([lum, chroma[0][:, :, None], chroma[1][:, :, None]], 2)
    return scan.reshape(-1, 64), hs * vs


def _nbits(v):
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while np.any(a >> n):
        n += (a >> n) > 0
    return n


def entropy_segment(scan, luma_per_mcu):
    """The entropy-coded segment of scan-order blocks (stuffed, padded), without the EOI."""
    nb = scan.shape[0]
    bpm = luma_per_mcu + 2
    comp = np.minimum(np.maximum(np.arange(nb) % bpm - luma_per_mcu + 1, 0), 2)
    zz = scan[:, ZIGZAG]
    dc = zz[:, 0]
    pred = np.zeros(nb, np.int64)
    for c in range(3):                              # DC prediction from the component's previous block
        idx = np.nonzero(comp == c)[0]
        pred[idx[1:]] = dc[idx[:-1]]
    table = np.minimum(comp, 1)
    keys, codes, lens = [], [], []

    def add(key, code, length):
        keys.append(key)
        codes.append(code)
        lens.append(length)

    diff = dc - pred
    s = _nbits(diff)
    b = np.arange(nb)
    for t in range(2):
        m = table == t
        (dcc, dcs), _ = LUTS[t]
        add(b[m] * 256 + 0, dcc[s[m]], dcs[s[m]])
    add(b * 256 + 1, np.where(diff < 0, diff - 1, diff) & ((1 << s) - 1), s)
    blk, pos = np.nonzero(zz[:, 1:])
    pos = pos + 1
    v = zz[blk, pos]
    first = np.ones(len(blk), bool)
    first[1:] = blk[1:] != blk[:-1]
    prev = np.where(first, 0, np.concatenate([[0], pos[:-1]]))
    run = pos - prev - 1
    nz = run // 16
    rs = ((run % 16) << 4) | _nbits(v)
    tb = table[blk]
    for t in range(2):
        _, (acc, acs) = LUTS[t]
        m = tb == t
        zr = np.repeat(np.nonzero(m)[0], nz[m])     # ZRLs before the coefficient
        add(blk[zr] * 256 + pos[zr] * 3 + 2, np.full(len(zr), acc[0xF0]), np.full(len(zr), acs[0xF0]))
        add(blk[m] * 256 + pos[m] * 3 + 3, acc[rs[m]], acs[rs[m]])
    sz = _nbits(v)
    add(blk * 256 + pos * 3 + 4, np.where(v < 0, v - 1, v) & ((1 << sz) - 1), sz)
    last = np.full(nb, 0)
    np.maximum.at(last, blk, pos)
    eob = np.nonzero(last < 63)[0]
    for t in range(2):
        _, (acc, acs) = LUTS[t]
        e = eob[table[eob] == t]
        add(e * 256 + 255, np.full(len(e), acc[0x00]), np.full(len(e), acs[0x00]))
    keys, codes, lens = (np.concatenate(a).astype(np.int64) for a in (keys, codes, lens))
    order = np.argsort(keys, kind="stable")
    codes, lens = codes[order], lens[order]
    j = np.arange(16)
    bits = (codes[:, None] >> np.maximum(lens[:, None] - 1 - j, 0)) & 1
    bits = bits[j[None] < lens[:, None]]
    pad = (-len(bits)) % 8
    raw = np.packbits(np.concatenate([bits, np.ones(pad, np.int64)]).astype(np.uint8))
    ff = np.nonzero(raw == 0xFF)[0]
    return np.insert(raw, ff + 1, 0).tobytes()


def encode(rgb, quality=75, subsampling=2):
    """The complete JPEG file of a uint8 [h, w, 3] frame."""
    rgb = np.asarray(rgb, np.uint8)
    h, w, _ = rgb.shape
    scan, lpm = coefficients(rgb, quality, subsampling)
    return header(h, w, quality, subsampling) + entropy_segment(scan, lpm) + b"\xff\xd9"
