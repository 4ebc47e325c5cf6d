"""JPEG decoding on the GPU: the reference datasets' `pil_from_raw_rgb` (`Image.open(BytesIO(raw)).convert('RGB')`)
as CUDA kernels (csrc/jpeg.cu), bit-identical to Pillow's libjpeg-turbo decoder; and JPEG encoding on the GPU
(`JpegEncoder`, csrc/jpeg_encode.cu), byte-identical to Pillow's `Image.save(buf, "JPEG", quality=, subsampling=)`.

    dec = JpegDecoder()
    batch = dec.parse(jpegs)                  # host only: one bytes object per frame; ValueError names a bad frame
    frames = dec(batch)                       # uint8 [N, Hmax, Wmax, 3] on the GPU; frame i fills its top-left h x w
    x = aug(frames.view(B, F, *frames.shape[1:]), aug.plan(batch.sample_sizes(B)))

Decodable: sequential Huffman JPEGs (SOF0 / SOF1) with 8-bit samples, grayscale or YCbCr with 4:4:4, 4:2:2 or 4:2:0
sampling, with or without restart markers, DHT segments (the Annex K tables stand in for missing ones) and 16-bit
quant tables.  Anything else (progressive, arithmetic, CMYK, RGB-coded, other samplings, truncated input) is rejected
by `parse` with its reason, before anything is launched.
"""
import ctypes as C

import numpy as np
import torch

from . import lib as L

REASONS = ("ok", "no SOI marker", "truncated segment", "progressive", "arithmetic coding", "lossless or hierarchical",
           "sample precision is not 8 bits", "component count is not 1 or 3 (CMYK / YCCK)", "RGB colour transform",
           "unsupported sampling", "no SOF before SOS", "no SOS", "no EOI", "more than one scan",
           "missing or invalid table", "malformed segment")                  # COCLR_JPEG_* of coclr_b200.h
STATUS = ("ok", "invalid Huffman code", "entropy-coded data ends early", "missing restart marker")   # COCLR_JPEG_ST_*

I4, I8 = np.int32, np.int64
FRAME = np.dtype([("reason", I4), ("h", I4), ("w", I4), ("ncomp", I4), ("hs", I4), ("vs", I4), ("restart", I4),
                  ("mcus_x", I4), ("mcus_y", I4), ("qt", I4, 3), ("dc", I4, 3), ("ac", I4, 3), ("pad", I4, 2),
                  ("ecs_begin", I8), ("ecs_end", I8), ("blocks", I8), ("block0", I8)])     # coclr_jpeg_frame_t
QUANT = np.dtype([("q", np.uint16, 64)])                                                   # coclr_jpeg_quant_t
HUFF = np.dtype([("look", np.uint16, 512), ("maxcode", I4, 18), ("valoff", I4, 18), ("val", np.uint8, 256),
                 ("bits", np.uint8, 16), ("nval", I4), ("pad", I4, 3)])                   # coclr_jpeg_huff_t


class JpegFrameError(ValueError):
    """`parse`'s error: `frame` is the index of the first frame that cannot be decoded, `reason` why."""

    def __init__(self, frame, reason, more=""):
        super().__init__("frame %d: %s%s" % (frame, reason, more))
        self.frame, self.reason = frame, reason


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


class JpegBatch:
    """Parsed headers of N frames: the concatenated bytes, per-frame records (FRAME) and the distinct tables."""

    def __init__(self, data, offsets, frames, quant, huff):
        self.data, self.offsets, self.frames, self.quant, self.huff = data, offsets, frames, quant, huff

    def __len__(self):
        return len(self.frames)

    @property
    def sizes(self):
        """[(h, w)] of every frame."""
        return [(int(h), int(w)) for h, w in zip(self.frames["h"], self.frames["w"])]

    @property
    def work_bytes(self):
        """Workspace a single pass over the whole batch needs: 128 bytes per 8 x 8 block."""
        return int(self.frames["blocks"].sum()) * 128

    def sample_sizes(self, B, slots=None):
        """[(h, w)] of B samples of N / B consecutive frames each; ValueError when a sample's frames differ.  With
        `slots` (as given to JpegDecoder), of the output frames that decode writes."""
        sizes = self.sizes if slots is None else self.output_sizes(slots)
        n = len(sizes)
        if B < 1 or n % B:
            raise ValueError("%d frames do not split into %d samples" % (n, B))
        F = n // B
        for b in range(B):
            s = set(sizes[b * F:(b + 1) * F])
            if len(s) != 1:
                raise ValueError("sample %d: its frames have different sizes %s" % (b, sorted(s)))
        return [sizes[b * F] for b in range(B)]

    def output_sizes(self, slots):
        """[(h, w)] of every output frame when frame i is written to output frames slots[i] (JpegDecoder's
        `slots=`), for `sample_sizes`-style checks on the expanded batch."""
        begin, flat = slot_arrays(slots, len(self))
        out = [None] * len(flat)
        for i, hw in enumerate(self.sizes):
            for o in flat[begin[i]:begin[i + 1]]:
                out[o] = hw
        return out


def slot_arrays(slots, n):
    """`slots` (one list of output frame indices per parsed frame) as the int32 (slot_begin [n + 1], slots) of
    coclr_jpeg_t; ValueError unless every output frame 0 .. len - 1 is written exactly once."""
    if len(slots) != n:
        raise ValueError("slots has %d entries for %d frames" % (len(slots), n))
    begin = np.zeros(n + 1, np.int32)
    begin[1:] = np.cumsum([len(s) for s in slots])
    flat = np.array([o for s in slots for o in s], np.int32).reshape(-1)
    if not np.array_equal(np.sort(flat), np.arange(len(flat))):
        raise ValueError("slots must write every output frame 0 .. %d exactly once" % (len(flat) - 1))
    return begin, flat


def parse(jpegs):
    """Host-only header parse of a list of JPEG byte strings (no device needed).  Raises ValueError naming the first
    frame that cannot be decoded and why."""
    n = len(jpegs)
    offsets = np.zeros(n + 1, np.int64)
    offsets[1:] = np.cumsum([len(j) for j in jpegs])
    data = np.frombuffer(b"".join(bytes(j) for j in jpegs), np.uint8) if n else np.zeros(0, np.uint8)
    data = data if data.size else np.zeros(1, np.uint8)
    frames = np.zeros(n, FRAME)
    lib = L.load()
    nq, nh = C.c_int(0), C.c_int(0)
    quant, huff = np.zeros(4, QUANT), np.zeros(8, HUFF)
    for _ in range(2):                               # a second call when the batch has more distinct tables
        rc = lib.coclr_jpeg_parse(_ptr(data), _ptr(offsets), n, _ptr(frames), _ptr(quant), len(quant), C.byref(nq),
                                  _ptr(huff), len(huff), C.byref(nh))
        if rc < 0:
            raise L.CoclrError("coclr_jpeg_parse failed with code %d" % rc)
        if rc == 0:
            break
        quant, huff = np.zeros(max(nq.value, 1), QUANT), np.zeros(max(nh.value, 1), HUFF)
    bad = np.nonzero(frames["reason"])[0]
    if len(bad):
        i = int(bad[0])
        more = " (and %d more)" % (len(bad) - 1) if len(bad) > 1 else ""
        raise JpegFrameError(i, REASONS[frames["reason"][i]], more)
    return JpegBatch(data, offsets, frames, quant[:nq.value], huff[:nh.value])


def _align(n, a=256):
    return (n + a - 1) // a * a


class JpegDecoder:
    """Decodes parsed batches on the current CUDA device.  The bytes, records and tables go up in one copy from a
    pinned staging buffer; the staging buffer, the device copy, the workspace and the status array grow on demand and
    are reused, so a steady stream of batches allocates nothing but (without `out=`) the output.

    work_limit caps the workspace (bytes): a batch whose blocks need more is decoded in passes of consecutive frames
    within one call.

    CUDA graphs: a call under stream capture stages its batch in buffers of its own (a pinned staging buffer sized by
    the eager calls before it, a device copy, a workspace and `graph_status`), which later eager calls never touch.
    Every replay therefore decodes the captured batch again.  One decoder holds one captured decode; capture another
    with another JpegDecoder."""

    def __init__(self, work_limit=1 << 30):
        self.work_limit = int(work_limit)
        self._stage = None                          # pinned host staging buffer of eager calls
        self._graph_stage = None                    # pinned staging buffer reserved for a captured call
        self._copied = None                         # event after the last copy out of self._stage
        self._dev = None                            # device copy of the staged bytes
        self._work = None
        self._status = None
        self._graph = None                          # the captured call's buffers, kept alive for its replays
        self.status = None                          # int32 [N] of the last call, on the device (COCLR_JPEG_ST_*)
        self.graph_status = None                    # int32 [N] each replay of the captured call writes

    parse = staticmethod(parse)

    def __call__(self, batch, out=None, check=True, slots=None):
        """Decode `batch` into out (uint8 [N, >= Hmax, >= Wmax, 3] on the GPU, rows and frames strided; only each
        frame's top-left h x w x 3 bytes are written) or a new [N, Hmax, Wmax, 3] tensor.  check=True reads the
        status back (one synchronisation) and raises ValueError naming the frames with invalid entropy-coded data;
        check=False leaves it in `self.status` on the device.

        slots: one list of output frame indices per parsed frame; frame i is decoded once and written to each of
        slots[i], so N becomes the number of output frames (every one written exactly once)."""
        if not isinstance(batch, JpegBatch):
            raise ValueError("decode takes the JpegBatch of JpegDecoder.parse")
        n = len(batch)
        if slots is not None:
            slot_begin, slot_list = slot_arrays(slots, n)
            n_out = len(slot_list)
        else:
            slot_begin = slot_list = None
            n_out = n
        dev = torch.device("cuda", torch.cuda.current_device())
        hm = max((h for h, _ in batch.sizes), default=1)
        wm = max((w for _, w in batch.sizes), default=1)
        if out is None:
            out = torch.empty(n_out, hm, wm, 3, dtype=torch.uint8, device=dev)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or not out.is_cuda or out.dim() != 4 or
              out.shape[0] != n_out or out.shape[1] < hm or out.shape[2] < wm or out.shape[3] != 3 or
              out.stride(3) != 1 or out.stride(2) != 3):
            raise ValueError("out must be a CUDA uint8 [%d, >= %d, >= %d, 3] tensor with packed pixels"
                             % (n_out, hm, wm))
        if n == 0:
            return out

        # one staging image: bytes | records | quant tables | Huffman tables [| slot_begin | slots], each 256-aligned
        parts = [batch.data.view(np.uint8), batch.frames.view(np.uint8), batch.quant.view(np.uint8),
                 batch.huff.view(np.uint8)]
        if slots is not None:
            parts += [slot_begin.view(np.uint8), slot_list.view(np.uint8)]
        offs, total = [], 0
        for a in parts:
            offs.append(total)
            total = _align(total + a.nbytes)
        need = max(min(batch.work_bytes, self.work_limit), int(batch.frames["blocks"].max()) * 128)
        capturing = torch.cuda.is_current_stream_capturing()
        if capturing:
            if check:
                raise ValueError("check=True reads the status back, which a captured call cannot; pass check=False")
            if self._graph is not None:
                raise ValueError("this decoder already holds a captured decode; capture another with another "
                                 "JpegDecoder")
            if self._graph_stage is None or self._graph_stage.numel() < total:
                raise ValueError("the staging buffer cannot be pinned under graph capture; decode a batch at least "
                                 "this large once before capturing")
            stage = self._graph_stage
            dbuf = torch.empty(total, dtype=torch.uint8, device=dev)          # from the graph's memory pool
            work = torch.empty(need, dtype=torch.uint8, device=dev)
            status = torch.empty(n, dtype=torch.int32, device=dev)
            self._graph = (stage, dbuf, work, status)
            self.graph_status = status
        else:
            if self._stage is None or self._stage.numel() < total:
                size = _align(total * 5 // 4, 1 << 20)
                self._stage = torch.empty(size, dtype=torch.uint8, pin_memory=True)
                self._dev = torch.empty(size, dtype=torch.uint8, device=dev)
                self._copied = None
                if self._graph is None:
                    self._graph_stage = torch.empty(size, dtype=torch.uint8, pin_memory=True)
            if self._copied is not None:
                self._copied.synchronize()          # the previous copy out of the staging buffer has finished
            stage, dbuf = self._stage, self._dev
            if self._work is None or self._work.numel() < need:
                self._work = torch.empty(need, dtype=torch.uint8, device=dev)
            if self._status is None or self._status.numel() < n:
                self._status = torch.empty(max(n, 64), dtype=torch.int32, device=dev)
            work, status = self._work, self._status[:n]
        host = stage.numpy()
        for a, o in zip(parts, offs):
            host[o:o + a.nbytes] = a
        dbuf[:total].copy_(stage[:total], non_blocking=True)
        if not capturing:
            self._copied = torch.cuda.Event()
            self._copied.record()
        self.status = status

        base = dbuf.data_ptr()
        p = L.Jpeg()
        p.n = n
        p.data, p.frames, p.quant, p.huff = (base + o for o in offs[:4])
        p.frames_host = _ptr(batch.frames)
        p.out = L.dptr(out)
        p.frame_stride, p.row_stride = out.stride(0), out.stride(1)
        p.status = L.dptr(status)
        p.work, p.work_bytes = L.dptr(work), work.numel()
        if slots is None:
            L.check(L.load().coclr_jpeg_decode(C.byref(p), L.stream_ptr()), "coclr_jpeg_decode")
        else:
            sl = L.JpegSlots()
            sl.slot_begin, sl.slots = base + offs[4], base + offs[5]
            sl.slot_begin_host, sl.slots_host = _ptr(slot_begin), _ptr(slot_list)
            sl.n_out = n_out
            L.check(L.load().coclr_jpeg_decode_slots(C.byref(p), C.byref(sl), L.stream_ptr()),
                    "coclr_jpeg_decode_slots")
        if check:
            st = status.cpu().numpy()
            bad = np.nonzero(st)[0]
            if len(bad):
                raise ValueError("invalid entropy-coded data: " + ", ".join(
                    "frame %d: %s" % (int(i), STATUS[st[i]] if st[i] < len(STATUS) else st[i]) for i in bad[:8]) +
                    (" (and %d more)" % (len(bad) - 8) if len(bad) > 8 else ""))
        return out


MAX_SIDE = 65500                                     # COCLR_JPEG_MAX_SIDE
HEADER_BYTES = 623                                   # COCLR_JPEG_HEADER_BYTES


def _settings(quality, subsampling):
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
        raise ValueError("quality must be an integer 1 .. 100, got %r" % (quality,))
    if isinstance(subsampling, bool) or subsampling not in (0, 1, 2):
        raise ValueError("subsampling must be 0 (4:4:4), 1 (4:2:2) or 2 (4:2:0), got %r" % (subsampling,))


def encode_header(h, w, quality=75, subsampling=2):
    """Host only: the bytes every encoded h x w file starts with (SOI through SOS), as Pillow writes them."""
    _settings(quality, subsampling)
    if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
        raise ValueError("frame sides must be 1 .. %d, got %d x %d" % (MAX_SIDE, h, w))
    buf = np.zeros(HEADER_BYTES, np.uint8)
    n = L.load().coclr_jpeg_encode_header(h, w, int(quality), int(subsampling), _ptr(buf))
    if n != HEADER_BYTES:
        raise L.CoclrError("coclr_jpeg_encode_header failed with code %d" % n)
    return buf.tobytes()


class JpegEncoder:
    """Encodes uint8 RGB frames on the current CUDA device into JPEG files byte-identical to Pillow's
    `Image.fromarray(frame).save(buf, "JPEG", quality=quality, subsampling=subsampling)` (csrc/jpeg_encode.cu).

        enc = JpegEncoder(quality=95, subsampling=0)
        files = enc(frames)          # CUDA uint8 [N, H, W, 3] (rows and frames may be strided) -> list of N bytes

    Defaults are Pillow's: quality 75, 4:2:0.  work_limit caps the workspace (bytes): a batch that needs more is
    encoded in passes of consecutive frames within one call, with the same bytes.  The output buffer holds every
    file's worst case (coclr_jpeg_encode_max_bytes).  A call reads back the file offsets, then the files' bytes (one
    copy each, into a pinned buffer).  Device and pinned buffers grow on demand and are reused."""

    def __init__(self, quality=75, subsampling=2, work_limit=1 << 30):
        _settings(quality, subsampling)
        self.quality, self.subsampling = int(quality), int(subsampling)
        self.work_limit = int(work_limit)
        self._work = self._out = self._offsets = self._host = None

    @staticmethod
    def _grow(buf, n, **kw):
        return buf if buf is not None and buf.numel() >= n else torch.empty(max(n, 1), dtype=torch.uint8, **kw)

    def __call__(self, frames):
        if (not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or not frames.is_cuda or
                frames.dim() != 4 or frames.shape[3] != 3 or frames.stride(3) != 1 or frames.stride(2) != 3):
            raise ValueError("frames must be a CUDA uint8 [N, H, W, 3] tensor with packed pixels")
        n, h, w, _ = frames.shape
        if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
            raise ValueError("frame sides must be 1 .. %d, got %d x %d" % (MAX_SIDE, h, w))
        if n == 0:
            return []
        lib = L.load()
        dev = frames.device
        q, s = self.quality, self.subsampling
        max_bytes = lib.coclr_jpeg_encode_max_bytes(h, w, s)
        work = min(lib.coclr_jpeg_encode_work_bytes(n, h, w, s),
                   max(self.work_limit, lib.coclr_jpeg_encode_work_bytes(1, h, w, s)))
        with torch.cuda.device(dev):
            self._work = self._grow(self._work, work, device=dev)
            self._out = self._grow(self._out, n * max_bytes, device=dev)
            if self._offsets is None or self._offsets.numel() < n + 1:
                self._offsets = torch.empty(max(n + 1, 64), dtype=torch.int64, device=dev)
            p = L.JpegEncode(n, h, w, q, s, L.dptr(frames), frames.stride(0), frames.stride(1), L.dptr(self._out),
                             self._out.numel(), L.dptr(self._offsets), L.dptr(self._work), self._work.numel())
            L.check(lib.coclr_jpeg_encode(C.byref(p), L.stream_ptr()), "coclr_jpeg_encode")
            offs = self._offsets[:n + 1].cpu().numpy()
            total = int(offs[-1])
            self._host = self._grow(self._host, total, pin_memory=True)
            self._host[:total].copy_(self._out[:total], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        data = self._host[:total].numpy().tobytes()
        return [data[offs[i]:offs[i + 1]] for i in range(n)]


class JpegVideoPool:
    """Seeded stand-in for the reference LMDB's values: `n_videos` videos, each a list of `n_frames` JPEG byte strings
    (Pillow, `quality`, 4:2:0) of h x w frames, a smooth colour field plus noise.  Encoded once, at construction."""

    def __init__(self, n_videos, n_frames, h, w, seed=0, quality=90):
        import io
        from PIL import Image
        r = np.random.RandomState(seed)
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        self.videos = []
        for _ in range(n_videos):
            fx, fy, ph = r.uniform(6, 30, 3), r.uniform(6, 30, 3), r.uniform(0, 6.3, 3)
            base = np.stack([128 + 90 * np.sin(xx / fx[c] + ph[c]) * np.cos(yy / fy[c]) for c in range(3)], -1)
            video = []
            for t in range(n_frames):
                img = np.clip(np.roll(base, t, axis=1) + r.normal(0, 8, base.shape), 0, 255).astype(np.uint8)
                b = io.BytesIO()
                Image.fromarray(img).save(b, "JPEG", quality=quality)
                video.append(b.getvalue())
            self.videos.append(video)

    def __len__(self):
        return len(self.videos)

    def frames(self, picks):
        """The frames of videos `picks`, one video after another (a batch of len(picks) samples)."""
        return [f for i in picks for f in self.videos[i]]
