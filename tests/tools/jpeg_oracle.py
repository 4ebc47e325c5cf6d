"""numpy restatement of the JPEG decoder (coclr_b200.jpeg, csrc/jpeg.cu): the header parse with its reject reasons,
sequential Huffman decoding with byte unstuffing and restart markers, libjpeg's ISLOW integer IDCT, fancy upsampling
and the fixed-point YCbCr -> RGB conversion.  It is held to Pillow's `Image.open(BytesIO(raw)).convert('RGB')` bit
for bit, and it is the statement the kernels mirror.
"""
import numpy as np

# reject reasons (coclr_b200.h, COCLR_JPEG_*)
OK, NO_SOI, TRUNCATED, PROGRESSIVE, ARITHMETIC, SOF_KIND, PRECISION, COMPONENTS, RGB, SAMPLING, NO_SOF, NO_SOS, \
    NO_EOI, MULTI_SCAN, BAD_TABLE, BAD_SEGMENT = range(16)
REASONS = ("ok", "no SOI marker", "truncated segment", "progressive", "arithmetic coding", "lossless or hierarchical",
           "sample precision is not 8 bits", "component count is not 1 or 3", "RGB colour transform",
           "unsupported sampling", "no SOF before SOS", "no SOS", "no EOI", "more than one scan",
           "missing or invalid table", "malformed segment")
# status of a decoded frame (coclr_jpeg_decode)
ST_OK, ST_BAD_CODE, ST_EARLY_END, ST_BAD_RESTART = 0, 1, 2, 3

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)   # zigzag index -> natural index

# Annex K.3 tables (libjpeg's jstdhuff.c): (bits[1..16], values) for DC/AC luminance (slot 0) and chrominance (1)
STD_DC = {0: ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
          1: ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))}
_AC_LUM_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a343536"
    "3738393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a9293949596979899"
    "9aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5"
    "f6f7f8f9fa")
_AC_CHR_VALS = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a"
    "35363738393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a9293949596"
    "9798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4"
    "f5f6f7f8f9fa")
STD_AC = {0: ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], list(_AC_LUM_VALS)),
          1: ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], list(_AC_CHR_VALS))}
assert len(STD_AC[0][1]) == 162 and len(STD_AC[1][1]) == 162


class Reject(Exception):
    def __init__(self, reason):
        super().__init__(REASONS[reason])
        self.reason = reason


def huff_valid(bits, vals, is_dc):
    """libjpeg jpeg_make_d_derived_tbl's checks: at most 256 symbols, the codes of each length fit and none is all
    ones, DC symbols <= 15."""
    if sum(bits) > 256 or len(vals) != sum(bits):
        return False
    code = 0
    for l in range(1, 17):
        code += bits[l - 1]
        if code >= (1 << l):
            return False
        code <<= 1
    return not (is_dc and any(v > 15 for v in vals))


def parse(raw):
    """Parse one JPEG; raises Reject.  Returns a dict: h, w, ncomp, hs, vs (luma sampling, 1 1 for grayscale),
    restart, ecs (begin, end) byte range of the entropy-coded segment, and per component its quant table (64 ints,
    natural order) and its DC and AC tables (bits, values)."""
    raw = bytes(raw)
    n = len(raw)
    if n < 2 or raw[0] != 0xFF or raw[1] != 0xD8:
        raise Reject(NO_SOI)
    pos = 2
    qt, dht = {}, {}
    restart = 0
    sof = None
    jfif = adobe = False
    adobe_transform = 0
    scan = None
    while True:
        while pos < n and raw[pos] != 0xFF:        # libjpeg skips garbage before a marker
            pos += 1
        while pos < n and raw[pos] == 0xFF:        # and fill bytes
            pos += 1
        if pos >= n:
            raise Reject(NO_EOI if scan is not None else (NO_SOF if sof is None else NO_SOS))
        m = raw[pos]
        pos += 1
        if m == 0xD9:
            if scan is None:
                raise Reject(NO_SOF if sof is None else NO_SOS)
            break
        if 0xD0 <= m <= 0xD7 or m == 0x01:         # parameterless
            continue
        if pos + 2 > n:
            raise Reject(TRUNCATED)
        L = (raw[pos] << 8) | raw[pos + 1]
        if L < 2:
            raise Reject(BAD_SEGMENT)
        if pos + L > n:
            raise Reject(TRUNCATED)
        seg = raw[pos + 2:pos + L]
        pos += L
        if m == 0xDA:
            if scan is not None:
                raise Reject(MULTI_SCAN)
            if sof is None:
                raise Reject(NO_SOF)
            if len(seg) < 1 or len(seg) != 1 + 2 * seg[0] + 3:
                raise Reject(BAD_SEGMENT)
            ns = seg[0]
            if ns != len(sof["comps"]):
                raise Reject(MULTI_SCAN)
            sel = []
            for i in range(ns):
                cid, t = seg[1 + 2 * i], seg[2 + 2 * i]
                idx = [c[0] for c in sof["comps"]]
                if cid not in idx or idx.index(cid) != i:
                    raise Reject(BAD_SEGMENT)
                sel.append((t >> 4, t & 15))
            comps = []
            for i, (td, ta) in enumerate(sel):
                tq = sof["comps"][i][3]
                if td > 3 or ta > 3 or tq not in qt:
                    raise Reject(BAD_TABLE)
                dc = dht.get((0, td)) or (STD_DC.get(td))
                ac = dht.get((1, ta)) or (STD_AC.get(ta))
                if dc is None or ac is None:
                    raise Reject(BAD_TABLE)
                if not huff_valid(dc[0], dc[1], True) or not huff_valid(ac[0], ac[1], False):
                    raise Reject(BAD_TABLE)
                comps.append({"q": list(qt[tq]), "dc": (list(dc[0]), list(dc[1])), "ac": (list(ac[0]), list(ac[1]))})
            begin = pos
            while True:                             # the segment ends at the first marker other than RSTn
                j = raw.find(b"\xff", pos)
                if j < 0 or j + 1 >= n:
                    raise Reject(NO_EOI)
                k = j + 1
                while k < n and raw[k] == 0xFF:
                    k += 1
                if k >= n:
                    raise Reject(NO_EOI)
                if raw[k] == 0 or 0xD0 <= raw[k] <= 0xD7:
                    pos = k + 1
                    continue
                pos = j
                break
            scan = {"comps": comps, "ecs": (begin, pos)}
            continue
        if m in (0xC0, 0xC1):
            if sof is not None:
                raise Reject(BAD_SEGMENT)
            if len(seg) < 6:
                raise Reject(BAD_SEGMENT)
            P, Y, X, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if len(seg) != 6 + 3 * nf:
                raise Reject(BAD_SEGMENT)
            if P != 8:
                raise Reject(PRECISION)
            if nf not in (1, 3):
                raise Reject(COMPONENTS)
            if Y == 0 or X == 0:
                raise Reject(BAD_SEGMENT)
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
            if any(c[3] > 3 for c in comps) or any(not (1 <= c[1] <= 4 and 1 <= c[2] <= 4) for c in comps):
                raise Reject(BAD_SEGMENT)
            if len({c[0] for c in comps}) != nf:             # duplicate component ids
                raise Reject(BAD_SEGMENT)
            sof = {"h": Y, "w": X, "comps": comps}
        elif m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise Reject(PROGRESSIVE if m == 0xC2 else (ARITHMETIC if m == 0xCA else SOF_KIND))
        elif m in (0xC3, 0xC5, 0xC7):
            raise Reject(SOF_KIND)
        elif m in (0xC9, 0xCB, 0xCD, 0xCF, 0xCC):
            raise Reject(ARITHMETIC)
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                sz = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + sz > len(seg):
                    raise Reject(BAD_SEGMENT)
                q = np.zeros(64, np.int64)
                for k in range(64):
                    q[ZIGZAG[k]] = ((seg[i + 1 + 2 * k] << 8) | seg[i + 2 + 2 * k]) if pq else seg[i + 1 + k]
                qt[tq] = q
                i += 1 + sz
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise Reject(BAD_SEGMENT)
                tc, th = seg[i] >> 4, seg[i] & 15
                bits = list(seg[i + 1:i + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or i + 17 + cnt > len(seg):
                    raise Reject(BAD_SEGMENT)
                dht[(tc, th)] = (bits, list(seg[i + 17:i + 17 + cnt]))
                i += 17 + cnt
        elif m == 0xDD:
            if len(seg) != 2:
                raise Reject(BAD_SEGMENT)
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            if len(seg) >= 14 and seg[:5] == b"JFIF\0":
                jfif = True
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe, adobe_transform = True, seg[11]
        elif m == 0xDC:                             # DNL
            raise Reject(BAD_SEGMENT)
        # other APPn, COM and unknown markers: skipped
    comps = sof["comps"]
    hs = vs = 1
    if len(comps) == 3:
        if not jfif:
            if adobe and adobe_transform == 0:
                raise Reject(RGB)
            if not adobe and [c[0] for c in comps] == [82, 71, 66]:
                raise Reject(RGB)
        samp = [(c[1], c[2]) for c in comps]
        if samp[1] != (1, 1) or samp[2] != (1, 1) or samp[0] not in ((1, 1), (2, 1), (2, 2)):
            raise Reject(SAMPLING)
        hs, vs = samp[0]
    return {"h": sof["h"], "w": sof["w"], "ncomp": len(comps), "hs": hs, "vs": vs, "restart": restart,
            "ecs": scan["ecs"], "comps": scan["comps"]}


# ----------------------------------------------------------------------------------------------------------------------
# entropy decoding
# ----------------------------------------------------------------------------------------------------------------------

def _codes(bits, vals):
    """{(length, code): symbol}."""
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[(l, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return out


class _Bits:
    """MSB-first bit reader over data[pos:end] with FF 00 unstuffing; past a marker it yields zeros (as libjpeg
    does) and counts how many zero bits it made up."""

    def __init__(self, data, pos, end):
        self.d, self.pos, self.end = data, pos, end
        self.acc, self.n, self.fake = 0, 0, 0
        self.marker = False

    def _fill(self):
        if not self.marker and self.pos < self.end:
            c = self.d[self.pos]
            if c == 0xFF:
                k = self.pos + 1
                while k < self.end and self.d[k] == 0xFF:
                    k += 1
                if k < self.end and self.d[k] == 0:
                    self.pos = k + 1
                else:
                    self.marker = True
                    return self._fill()
            else:
                self.pos += 1
            self.acc = (self.acc << 8) | c
        else:
            self.acc <<= 8
            self.fake += 8
        self.n += 8

    def get(self, k):
        while self.n < k:
            self._fill()
        self.n -= k
        v = (self.acc >> self.n) & ((1 << k) - 1)
        self.acc &= (1 << self.n) - 1
        return v

    def overrun(self):
        """True when bits past the segment's real data were consumed."""
        return self.fake > 0 and self.n < self.fake

    def restart(self):
        """Drop the buffered bits and read the next marker; returns the RSTn number or -1."""
        self.acc, self.n, self.fake = 0, 0, 0
        k = self.pos
        while True:                                # libjpeg's next_marker: skip data bytes and FF 00 pairs
            while k < self.end and self.d[k] != 0xFF:
                k += 1
            while k < self.end and self.d[k] == 0xFF:
                k += 1
            if k >= self.end or self.d[k] != 0:
                break
            k += 1
        if k >= self.end or not (0xD0 <= self.d[k] <= 0xD7):
            return -1
        self.pos, self.marker = k + 1, False
        return self.d[k] - 0xD0


def _decode(bits, codes):
    code = 0
    for l in range(1, 17):
        code = (code << 1) | bits.get(1)
        s = codes.get((l, code))
        if s is not None:
            return s
    return None


def _extend(r, s):
    return r - (1 << s) + 1 if s and r < (1 << (s - 1)) else r


def geometry(p):
    """Per component (blocks_w, blocks_h, h_samp, v_samp) and the MCU grid (mcus_x, mcus_y)."""
    h, w = p["h"], p["w"]
    if p["ncomp"] == 1:
        bw, bh = -(-w // 8), -(-h // 8)
        return [(bw, bh, 1, 1)], bw, bh
    hs, vs = p["hs"], p["vs"]
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    return [(mx * hs, my * vs, hs, vs), (mx, my, 1, 1), (mx, my, 1, 1)], mx, my


def entropy_decode(raw, p):
    """Raw (not dequantised) coefficients per component, int64 [blocks_h, blocks_w, 64] in natural order, and the
    status (ST_*)."""
    raw = bytes(raw)
    geo, mx, my = geometry(p)
    coef = [np.zeros((g[1], g[0], 64), np.int64) for g in geo]
    dcc = [_codes(*c["dc"]) for c in p["comps"]]
    acc = [_codes(*c["ac"]) for c in p["comps"]]
    b0, b1 = p["ecs"]
    bits = _Bits(raw, b0, b1)
    pred = [0] * len(geo)
    ri, nmcu, next_rst = p["restart"], mx * my, 0
    for m in range(nmcu):
        if ri and m and m % ri == 0:
            if bits.overrun():
                return coef, ST_EARLY_END
            if bits.restart() != next_rst:
                return coef, ST_BAD_RESTART
            next_rst = (next_rst + 1) & 7
            pred = [0] * len(geo)
        mrow, mcol = divmod(m, mx)
        for c, (bw, bh, hc, vc) in enumerate(geo):
            for v in range(vc):
                for u in range(hc):
                    blk = coef[c][mrow * vc + v, mcol * hc + u]
                    s = _decode(bits, dcc[c])
                    if s is None:
                        return coef, ST_BAD_CODE
                    pred[c] += _extend(bits.get(s), s) if s else 0
                    blk[0] = pred[c]
                    k = 1
                    while k < 64:
                        rs = _decode(bits, acc[c])
                        if rs is None:
                            return coef, ST_BAD_CODE
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            blk[ZIGZAG[min(k, 63)]] = _extend(bits.get(s), s)
                        elif r != 15:
                            break
                        else:
                            k += 15
                        k += 1
    if bits.overrun():
        return coef, ST_EARLY_END
    return coef, ST_OK


# ----------------------------------------------------------------------------------------------------------------------
# IDCT, upsampling, colour
# ----------------------------------------------------------------------------------------------------------------------

F0298, F0390, F0541, F0765, F0899, F1175, F1501, F1847, F1961, F2053, F2562, F3072 = (
    2446, 3196, 4433, 6270, 7373, 9633, 12299, 15137, 16069, 16819, 20995, 25172)


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7):
    """jidctint.c's butterfly on int64 arrays; returns the eight outputs before descaling (scaled by 2^13)."""
    z1 = (x2 + x6) * F0541
    t2 = z1 - x6 * F1847
    t3 = z1 + x2 * F0765
    t0 = (x0 + x4) << 13
    t1 = (x0 - x4) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o0, o1, o2, o3 = x7, x5, x3, x1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F1175
    o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
    z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    return (t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3)


def idct(coef, q):
    """ISLOW IDCT of raw coefficient blocks [..., 64] (natural order) with quant table q [64]; uint8 [..., 8, 8]."""
    x = (coef.astype(np.int64) * np.asarray(q, np.int64)).reshape(coef.shape[:-1] + (8, 8))   # [.., row v, col u]
    cols = _idct_1d(*[x[..., k, :] for k in range(8)])                  # pass 1 over columns
    ws = np.stack([(c + (1 << 10)) >> 11 for c in cols], axis=-2)      # DESCALE(., 13 - 2)
    rows = _idct_1d(*[ws[..., :, k] for k in range(8)])                 # pass 2 over rows
    out = np.stack([(r + (1 << 17)) >> 18 for r in rows], axis=-1)     # DESCALE(., 13 + 2 + 3)
    return np.clip(out + 128, 0, 255).astype(np.uint8)


def plane(blocks):
    """[bh, bw, 8, 8] -> [bh * 8, bw * 8]."""
    bh, bw = blocks.shape[:2]
    return blocks.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample(c, hs, vs, h, w):
    """libjpeg's fancy upsampling of a chroma plane to the luma grid, [h, w] (int64).  c: the padded component plane;
    only its downsampled_width x downsampled_height samples are read."""
    cw, ch = -(-w // hs), -(-h // vs)
    c = c[:ch, :cw].astype(np.int64)
    if hs == 1:
        return c[:h, :w]
    if cw <= 2:                                  # too narrow for the fancy filter: libjpeg replicates
        return np.repeat(np.repeat(c, hs, 1), vs, 0)[:h, :w]
    if vs == 1:
        left = np.concatenate([c[:, :1], c[:, :-1]], 1)
        right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
        out = np.empty((ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * c + left + 1) >> 2
        out[:, 1::2] = (3 * c + right + 2) >> 2
        out[:, 0] = c[:, 0]
        out[:, -1] = c[:, -1]
        return out[:h, :w]
    up = np.concatenate([c[:1], c[:-1]], 0)
    down = np.concatenate([c[1:], c[-1:]], 0)
    rows = np.empty((2 * ch, cw), np.int64)
    rows[0::2] = 3 * c + up
    rows[1::2] = 3 * c + down
    left = np.concatenate([rows[:, :1], rows[:, :-1]], 1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], 1)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    out[:, 0] = (4 * rows[:, 0] + 8) >> 4
    out[:, -1] = (4 * rows[:, -1] + 7) >> 4
    return out[:h, :w]


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c ycc_rgb_convert on int64 planes; uint8 [h, w, 3]."""
    cb, cr = cb - 128, cr - 128
    r = y + ((_fix(1.40200) * cr + 32768) >> 16)
    g = y + ((-_fix(0.34414) * cb + 32768 - _fix(0.71414) * cr) >> 16)
    b = y + ((_fix(1.77200) * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(raw, p=None):
    """uint8 [h, w, 3] and the status; the frame's pixels are meaningful only when the status is ST_OK."""
    p = parse(raw) if p is None else p
    coef, st = entropy_decode(raw, p)
    planes = [plane(idct(c, comp["q"])) for c, comp in zip(coef, p["comps"])]
    h, w = p["h"], p["w"]
    if p["ncomp"] == 1:
        y = planes[0][:h, :w]
        return np.repeat(y[:, :, None], 3, 2), st
    y = planes[0][:h, :w].astype(np.int64)
    cb = upsample(planes[1], p["hs"], p["vs"], h, w)
    cr = upsample(planes[2], p["hs"], p["vs"], h, w)
    return ycc_to_rgb(y, cb, cr), st
