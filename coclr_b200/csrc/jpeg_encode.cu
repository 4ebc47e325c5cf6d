// JPEG encoding, byte-identical to Pillow's libjpeg(-turbo) baseline encoder (coclr_b200.h, coclr_jpeg_encode*): a host
// header writer, then per pass seven kernels (transform, count, scan, emit, tile count, scans, scatter), each of which
// writes its result in full before the next reads it, so the bytes do not depend on scheduling.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "coclr_b200.h"
#include "jpeg_tables.cuh"

namespace coclr {
namespace {

// ---------------------------------------------------------------------------------------------------------------------
// host: settings, header, sizes
// ---------------------------------------------------------------------------------------------------------------------

// ITU T.81 Annex K.1 / K.2 quant tables, natural order
const uint8_t kStdQuant[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40, 57,
     69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
     81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
     99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

constexpr int kBlockBits = 11 + 11 + 63 * (16 + 10);   // a block's worst case: DC code + bits, 63 x (AC code + bits)
constexpr int kTileBytes = 1024;                        // the stuffing kernels' tile: 256 threads x 4 bytes
constexpr int kHeaderAlloc = 624;

bool settings_ok(int h, int w, int subsampling) {
  return h >= 1 && w >= 1 && h <= COCLR_JPEG_MAX_SIDE && w <= COCLR_JPEG_MAX_SIDE && subsampling >= 0 &&
         subsampling <= 2;
}

struct Geometry {                 // one frame's block layout
  int hs, vs, lpm, bpm;           // luma sampling, luma blocks and blocks per MCU
  int mx, my, wb, hb;             // MCU grid; real luma blocks per row and column
  int64_t blocks;                 // blocks per frame (dummies included)
  int64_t words;                  // 32-bit words of the unstuffed segment's worst case (+1 spare)
  int64_t tiles;                  // kTileBytes tiles of that
};

Geometry geometry(int h, int w, int subsampling) {
  Geometry g;
  g.hs = subsampling ? 2 : 1;
  g.vs = subsampling == 2 ? 2 : 1;
  g.lpm = g.hs * g.vs;
  g.bpm = g.lpm + 2;
  g.mx = (w + 8 * g.hs - 1) / (8 * g.hs);
  g.my = (h + 8 * g.vs - 1) / (8 * g.vs);
  g.wb = (w + 7) / 8;
  g.hb = (h + 7) / 8;
  g.blocks = (int64_t)g.mx * g.my * g.bpm;
  g.words = (g.blocks * kBlockBits + 7 + 31) / 32 + 1;
  g.tiles = (g.words * 4 + kTileBytes - 1) / kTileBytes;
  return g;
}

inline int64_t align256(int64_t b) { return (b + 255) / 256 * 256; }

struct Layout {                   // a pass's workspace: each region holds its frames one after another
  int64_t coef, bits, stream, tiles, frame;   // byte offsets of the regions
  int64_t bytes;
};

Layout layout(const Geometry& g, int nf) {
  Layout l;
  l.coef = 0;
  l.bits = align256(l.coef + (int64_t)nf * g.blocks * 128);
  l.stream = align256(l.bits + (int64_t)nf * g.blocks * 8);
  l.tiles = align256(l.stream + (int64_t)nf * g.words * 4);
  l.frame = align256(l.tiles + (int64_t)nf * g.tiles * 8);
  l.bytes = align256(l.frame + (int64_t)nf * 2 * 8);
  return l;
}

struct Header {                   // the file header and where its tables are, passed to the kernels by value
  uint8_t b[kHeaderAlloc];
  int dqt[2];                     // offsets of the zigzag quant values of tables 0 and 1
  int bits[4], vals[4];           // offsets of the DHT counts and symbols of DC0, AC0, DC1, AC1
};

int write_header(int h, int w, int quality, int subsampling, Header* hd) {
  if (!settings_ok(h, w, subsampling) || quality < 1 || quality > 100) return COCLR_E_ARG;
  uint8_t* o = hd->b;
  int n = 0;
  auto put = [&](int v) { o[n++] = (uint8_t)v; };
  put(0xFF), put(0xD8);
  const uint8_t app0[18] = {0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  for (int i = 0; i < 18; ++i) put(app0[i]);
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;    // libjpeg's jpeg_quality_scaling
  for (int t = 0; t < 2; ++t) {
    put(0xFF), put(0xDB), put(0), put(67), put(t);
    hd->dqt[t] = n;
    for (int k = 0; k < 64; ++k) {
      int q = ((int)kStdQuant[t][kZigzag[k]] * scale + 50) / 100;
      put(q < 1 ? 1 : (q > 255 ? 255 : q));                               // baseline: at most 255
    }
  }
  const int hs = subsampling ? 2 : 1, vs = subsampling == 2 ? 2 : 1;
  const uint8_t sof[19] = {0xFF, 0xC0, 0, 17, 8, (uint8_t)(h >> 8), (uint8_t)h, (uint8_t)(w >> 8), (uint8_t)w, 3,
                           1, (uint8_t)((hs << 4) | vs), 0, 2, 0x11, 1, 3, 0x11, 1};
  for (int i = 0; i < 19; ++i) put(sof[i]);
  for (int t = 0; t < 2; ++t)
    for (int ac = 0; ac < 2; ++ac) {
      const int nv = ac ? 162 : 12, len = 3 + 16 + nv;
      put(0xFF), put(0xC4), put(len >> 8), put(len & 255), put((ac << 4) | t);
      hd->bits[2 * t + ac] = n;
      for (int i = 0; i < 16; ++i) put(ac ? kStdAcBits[t][i] : kStdDcBits[t][i]);
      hd->vals[2 * t + ac] = n;
      for (int i = 0; i < nv; ++i) put(ac ? kStdAcVal[t][i] : kStdDcVal[i]);
    }
  const uint8_t sos[14] = {0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
  for (int i = 0; i < 14; ++i) put(sos[i]);
  return n;                                                                 // COCLR_JPEG_HEADER_BYTES
}

// ---------------------------------------------------------------------------------------------------------------------
// device
// ---------------------------------------------------------------------------------------------------------------------

struct Pass {                     // what every kernel of a pass reads
  const uint8_t* rgb;             // the pass's first frame
  int64_t frame_stride, row_stride;
  int h, w;
  int hs, vs, lpm, bpm, mx, my, wb, hb;
  int64_t blocks, words, tiles;
  int16_t* coef;                  // [nf][blocks][64], zigzag
  int64_t* bits;                  // [nf][blocks]: bit counts, then (scanned) bit offsets
  uint32_t* stream;               // [nf][words]: the unstuffed segment, stream byte order
  int64_t* tile_ff;               // [nf][tiles]: 0xFF bytes per tile, then (scanned) offsets
  int64_t* frame;                 // [nf][2]: total bits, total 0xFF bytes
  int64_t* offsets;               // the call's [n + 1], at the pass's first frame
  uint8_t* out;
  int nf, first;
};

// libjpeg's jccolor: FIX(x) = round(x * 2^16), ONE_HALF for Y, ONE_HALF - 1 and CBCR_OFFSET for Cb and Cr
__device__ __forceinline__ int to_ycc(int c, int r, int g, int b) {
  if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int pixel(const Pass& p, const uint8_t* f, int c, int y, int x) {
  const uint8_t* q = f + (int64_t)y * p.row_stride + 3 * x;
  return to_ycc(c, __ldg(q), __ldg(q + 1), __ldg(q + 2));
}

// sample (y, x) of component c's plane, whole blocks: the image's edges are replicated (the luma and the input of
// the chroma downsampling to whole blocks / row groups; a downsampled 4:2:0 chroma plane's last row to whole blocks),
// and 2:1 downsampling adds libjpeg's alternating bias (h2v1: 0, 1, ...; h2v2: 1, 2, ...)
__device__ __forceinline__ int sample(const Pass& p, const uint8_t* f, int c, int y, int x) {
  const int H = p.h, W = p.w;
  if (c == 0 || p.hs == 1) return pixel(p, f, c, min(y, H - 1), min(x, W - 1));
  const int x0 = min(2 * x, W - 1), x1 = min(2 * x + 1, W - 1);
  if (p.vs == 1) {
    const int r = min(y, H - 1);
    return (pixel(p, f, c, r, x0) + pixel(p, f, c, r, x1) + (x & 1)) >> 1;
  }
  const int cy = min(y, (H + 1) / 2 - 1);
  const int r0 = 2 * cy, r1 = min(2 * cy + 1, H - 1);
  return (pixel(p, f, c, r0, x0) + pixel(p, f, c, r0, x1) + pixel(p, f, c, r1, x0) + pixel(p, f, c, r1, x1) + 1 +
          (x & 1)) >> 2;
}

// jfdctint's butterfly on one row (last = false: outputs scaled by 2^2) or column (last = true: the final scale 8).
// int32 is exact: with samples in -128..127 every intermediate, bounded as a linear form of the 64 samples plus its
// rounding terms, is below 2^23.4 in the row pass and 2^28.4 in the column pass (|output| <= 8194).
__device__ __forceinline__ void fdct_1d(const int* d, int* o, bool last) {
  const int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
            F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
  const int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
  const int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  const int s = last ? 15 : 11, half = 1 << (s - 1);
  if (last) {
    o[0] = (t10 + t11 + 2) >> 2;
    o[4] = (t10 - t11 + 2) >> 2;
  } else {
    o[0] = (t10 + t11) * 4;
    o[4] = (t10 - t11) * 4;
  }
  int z1 = (t12 + t13) * F0541;
  o[2] = (z1 + t13 * F0765 + half) >> s;
  o[6] = (z1 - t12 * F1847 + half) >> s;
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * F1175;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 = z3 * -F1961 + z5;
  z4 = z4 * -F0390 + z5;
  o[7] = (t4 * F0298 + z1 + z3 + half) >> s;
  o[5] = (t5 * F2053 + z2 + z4 + half) >> s;
  o[3] = (t6 * F3072 + z2 + z3 + half) >> s;
  o[1] = (t7 * F1501 + z1 + z4 + half) >> s;
}

// ---- transform: 32 blocks per CTA, 8 threads per block ---------------------------------------------------------------

constexpr int kTxBlocks = 32;

__global__ void __launch_bounds__(8 * kTxBlocks) jpeg_enc_transform_kernel(Pass p, Header hd) {
  __shared__ int ws[kTxBlocks][64];
  __shared__ __align__(16) int16_t zz[kTxBlocks][64];
  __shared__ uint8_t izz[64];                      // natural index -> zigzag position
  __shared__ uint16_t q8[2][64];                   // 8 q, natural order
  const int t = threadIdx.x;
  if (t < 64) izz[kZigzagDev[t]] = (uint8_t)t;
  __syncthreads();
  if (t < 128) q8[t >> 6][t & 63] = (uint16_t)(8 * hd.b[hd.dqt[t >> 6] + izz[t & 63]]);
  const int bl = t >> 3, j = t & 7;
  const int64_t gb = (int64_t)blockIdx.x * kTxBlocks + bl;
  const bool valid = gb < p.blocks;
  const uint8_t* f = p.rgb + (int64_t)blockIdx.y * p.frame_stride;
  int c = 0, by = 0, bx = 0;
  bool dc_only = false;
  if (valid) {
    const int64_t mcu = gb / p.bpm;
    const int k = (int)(gb - mcu * p.bpm);
    const int my = (int)(mcu / p.mx), mx = (int)(mcu - (int64_t)my * p.mx);
    if (k < p.lpm) {
      const int v = k / p.hs, u = k - v * p.hs;
      by = my * p.vs + v;
      bx = mx * p.hs + u;
      if (by >= p.hb) {           // below the image: the DC of the MCU's previous block (the row above's last)
        dc_only = true;
        by -= 1;
        bx = min(mx * p.hs + p.hs - 1, p.wb - 1);
      } else if (bx >= p.wb) {    // right of the image: the DC of the row's last real block
        dc_only = true;
        bx = p.wb - 1;
      }
    } else {
      c = k - p.lpm + 1;
      by = my;
      bx = mx;
    }
    int d[8], o[8];
    for (int i = 0; i < 8; ++i) d[i] = sample(p, f, c, by * 8 + j, bx * 8 + i) - 128;
    fdct_1d(d, o, false);                          // row j
    for (int i = 0; i < 8; ++i) ws[bl][j * 8 + i] = o[i];
  }
  __syncthreads();
  if (valid) {
    int d[8], o[8];
    for (int r = 0; r < 8; ++r) d[r] = ws[bl][r * 8 + j];
    fdct_1d(d, o, true);                           // column j
    const int tq = c ? 1 : 0;
    for (int r = 0; r < 8; ++r) {
      const int n = r * 8 + j, qv = q8[tq][n];
      const int a = (abs(o[r]) + (qv >> 1)) / qv;  // rounded division, sign kept (jcdctmgr's quantize)
      zz[bl][izz[n]] = (int16_t)((dc_only && n) ? 0 : (o[r] < 0 ? -a : a));
    }
  }
  __syncthreads();
  const int64_t b0 = (int64_t)blockIdx.x * kTxBlocks;
  const int nblk = (int)min((int64_t)kTxBlocks, p.blocks - b0);
  for (int i = t; i < nblk * 8; i += blockDim.x)   // 16 bytes per thread
    reinterpret_cast<int4*>(p.coef + ((int64_t)blockIdx.y * p.blocks + b0) * 64)[i] =
        reinterpret_cast<const int4*>(zz)[i];
}

// ---- Huffman: count, then emit -------------------------------------------------------------------------------------

constexpr int kHuffThreads = 256;
constexpr int kRow = 66;                           // int16 per staged block: 33 words, so rows fall in distinct banks

// the four tables of the header (DC0, AC0, DC1, AC1) as (length << 16) | code per symbol
__device__ void derive_tables(const Header& hd, uint32_t (*ehuf)[256]) {
  const int t = threadIdx.x;
  for (int i = t; i < 4 * 256; i += blockDim.x) ehuf[i >> 8][i & 255] = 0;
  __syncthreads();
  if (t < 4) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
      for (int i = 0; i < hd.b[hd.bits[t] + l - 1]; ++i, ++k, ++code)
        ehuf[t][hd.b[hd.vals[t] + k]] = ((uint32_t)l << 16) | (uint32_t)code;
      code <<= 1;
    }
  }
  __syncthreads();
}

struct Counter {
  int64_t n = 0;
  __device__ void put(uint32_t v, int len) { n += len; }
};

struct Writer {                   // MSB-first bits ORed into 32-bit words of stream byte order
  uint32_t* words;
  int64_t pos;                    // stream bit of acc's oldest pending bit
  uint64_t acc = 0;               // the low n bits are pending
  int n = 0;
  __device__ void word(uint32_t v, int len) {      // v's top len bits at pos
    const int64_t w = pos >> 5;
    const int s = (int)(pos & 31);
    atomicOr(words + w, __byte_perm(v >> s, 0, 0x0123));
    if (s && s + len > 32) atomicOr(words + w + 1, __byte_perm(v << (32 - s), 0, 0x0123));
    pos += len;
  }
  __device__ void put(uint32_t v, int len) {
    acc = (acc << len) | v;
    n += len;
    if (n >= 32) {
      n -= 32;
      word((uint32_t)(acc >> n), 32);
    }
  }
  __device__ void flush() {
    if (n) word((uint32_t)(acc << (32 - n)), n);
    n = 0;
  }
};

__device__ __forceinline__ int nbits(int v) { return 32 - __clz(abs(v)); }

// libjpeg's encode_one_block: the DC difference, then run/size codes with ZRL for runs over 15 and EOB
template <class Sink>
__device__ __forceinline__ void code_block(const int16_t* z, int pred, const uint32_t* dct, const uint32_t* act,
                                           Sink& s) {
  const int d = z[0] - pred, ds = nbits(d);
  s.put(dct[ds] & 0xFFFF, dct[ds] >> 16);
  if (ds) s.put((uint32_t)(d < 0 ? d - 1 : d) & ((1u << ds) - 1), ds);
  uint64_t nz = 0;
  for (int k = 1; k < 64; ++k) nz |= (uint64_t)(z[k] != 0) << k;
  int last = 0;
  while (nz) {
    const int k = __ffsll((long long)nz) - 1;
    nz &= nz - 1;
    int r = k - last - 1;
    for (; r > 15; r -= 16) s.put(act[0xF0] & 0xFFFF, act[0xF0] >> 16);
    const int v = z[k], vs = nbits(v);
    const uint32_t e = act[(r << 4) | vs];
    s.put(e & 0xFFFF, e >> 16);
    s.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << vs) - 1), vs);
    last = k;
  }
  if (last < 63) s.put(act[0] & 0xFFFF, act[0] >> 16);
}

// kEmit false: each block's bit count into p.bits; true: its codes at the (scanned) bit offset p.bits holds
template <bool kEmit>
__global__ void __launch_bounds__(kHuffThreads) jpeg_enc_huff_kernel(Pass p, Header hd) {
  __shared__ uint32_t ehuf[4][256];
  __shared__ int16_t blk[kHuffThreads * kRow];
  derive_tables(hd, ehuf);
  const int t = threadIdx.x;
  const int64_t b0 = (int64_t)blockIdx.x * kHuffThreads;
  const int nblk = (int)min((int64_t)kHuffThreads, p.blocks - b0);
  const int16_t* coef = p.coef + (int64_t)blockIdx.y * p.blocks * 64;
  {                                                // stage the CTA's blocks: 16 bytes per load, coalesced
    const int4* src = reinterpret_cast<const int4*>(coef + b0 * 64);
    for (int i = t; i < nblk * 8; i += kHuffThreads) {
      const int4 v = src[i];
      int* dst = reinterpret_cast<int*>(blk + (i >> 3) * kRow + (i & 7) * 8);
      dst[0] = v.x, dst[1] = v.y, dst[2] = v.z, dst[3] = v.w;
    }
  }
  __syncthreads();
  if (t >= nblk) return;
  const int64_t gb = b0 + t;
  const int64_t mcu = gb / p.bpm;
  const int k = (int)(gb - mcu * p.bpm);
  int64_t prev = -1;                               // the component's previous block in scan order
  if (k > 0 && k < p.lpm) prev = gb - 1;
  else if (mcu > 0) prev = k == 0 ? gb - p.bpm + p.lpm - 1 : gb - p.bpm;
  const int pred = prev < 0 ? 0 : coef[prev * 64];
  const int tab = k < p.lpm ? 0 : 2;
  int64_t* bits = p.bits + (int64_t)blockIdx.y * p.blocks;
  if (!kEmit) {
    Counter s;
    code_block(blk + t * kRow, pred, ehuf[tab], ehuf[tab + 1], s);
    bits[gb] = s.n;
  } else {
    Writer s;
    s.words = p.stream + (int64_t)blockIdx.y * p.words;
    s.pos = bits[gb];
    code_block(blk + t * kRow, pred, ehuf[tab], ehuf[tab + 1], s);
    if (gb == p.blocks - 1) {                      // the last block pads the last byte with 1-bits
      const int pad = (int)((8 - (s.pos + s.n) % 8) % 8);
      if (pad) s.put((1u << pad) - 1, pad);
    }
    s.flush();
  }
}

// ---- scans ----------------------------------------------------------------------------------------------------------

// exclusive scan over the CTA of NT threads; *total gets the sum
template <int NT>
__device__ int64_t block_scan(int64_t v, int64_t* sums, int64_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int64_t s = lane < NT / 32 ? sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < NT / 32) sums[lane] = s;
  }
  __syncthreads();
  const int64_t r = x - v + (warp ? sums[warp - 1] : 0);
  *total = sums[NT / 32 - 1];
  __syncthreads();
  return r;
}

constexpr int kScanThreads = 1024;

// per frame (blockIdx.x): data[f * count, (f + 1) * count) scanned in place (exclusive); the sum into total[2 f]
__global__ void __launch_bounds__(kScanThreads) jpeg_enc_scan_kernel(int64_t* data, int64_t count, int64_t* total) {
  __shared__ int64_t sums[kScanThreads / 32];
  int64_t* d = data + (int64_t)blockIdx.x * count;
  int64_t carry = 0;
  for (int64_t i0 = 0; i0 < count; i0 += kScanThreads) {
    const int64_t i = i0 + threadIdx.x;
    const int64_t v = i < count ? d[i] : 0;
    int64_t sum;
    const int64_t e = block_scan<kScanThreads>(v, sums, &sum);
    if (i < count) d[i] = carry + e;
    carry += sum;
  }
  if (threadIdx.x == 0) total[2 * blockIdx.x] = carry;
}

constexpr int kTileThreads = kTileBytes / 4;

// the 0xFF bytes of each tile of each frame's segment (0 for tiles past its end)
__global__ void __launch_bounds__(kTileThreads) jpeg_enc_tile_kernel(Pass p) {
  __shared__ int64_t sums[kTileThreads / 32];
  const int64_t nbytes = (p.frame[2 * blockIdx.y] + 7) / 8;
  const int64_t tile0 = (int64_t)blockIdx.x * kTileBytes, b = tile0 + 4 * threadIdx.x;
  if (tile0 >= nbytes) {
    if (threadIdx.x == 0) p.tile_ff[(int64_t)blockIdx.y * p.tiles + blockIdx.x] = 0;
    return;
  }
  const uint8_t* s = reinterpret_cast<const uint8_t*>(p.stream + (int64_t)blockIdx.y * p.words);
  int ff = 0;
  for (int i = 0; i < 4; ++i) ff += b + i < nbytes && s[b + i] == 0xFF;
  int64_t total;
  block_scan<kTileThreads>(ff, sums, &total);
  if (threadIdx.x == 0) p.tile_ff[(int64_t)blockIdx.y * p.tiles + blockIdx.x] = total;
}

// the pass's file sizes (header, stuffed segment, EOI) scanned into the call's packed offsets
__global__ void __launch_bounds__(kScanThreads) jpeg_enc_offsets_kernel(Pass p) {
  __shared__ int64_t sums[kScanThreads / 32];
  int64_t carry = p.first ? 0 : p.offsets[0];
  for (int f0 = 0; f0 < p.nf; f0 += kScanThreads) {
    const int f = f0 + threadIdx.x;
    const int64_t len = f < p.nf ? COCLR_JPEG_HEADER_BYTES + (p.frame[2 * f] + 7) / 8 + p.frame[2 * f + 1] + 2 : 0;
    int64_t sum;
    const int64_t e = block_scan<kScanThreads>(len, sums, &sum);
    if (f < p.nf) p.offsets[f] = carry + e;
    carry += sum;
  }
  if (threadIdx.x == 0) p.offsets[p.nf] = carry;
}

// stuffed bytes of each tile, the header (tile 0) and EOI
__global__ void __launch_bounds__(kTileThreads) jpeg_enc_scatter_kernel(Pass p, Header hd) {
  __shared__ int64_t sums[kTileThreads / 32];
  const int fr = blockIdx.y;
  const int64_t nbytes = (p.frame[2 * fr] + 7) / 8;
  const int64_t tile0 = (int64_t)blockIdx.x * kTileBytes;
  uint8_t* out = p.out + p.offsets[fr];
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < COCLR_JPEG_HEADER_BYTES; i += blockDim.x) out[i] = hd.b[i];
    if (threadIdx.x == 0) {
      const int64_t end = p.offsets[fr + 1] - p.offsets[fr];
      out[end - 2] = 0xFF;
      out[end - 1] = 0xD9;
    }
  }
  if (tile0 >= nbytes) return;
  const int64_t b = tile0 + 4 * threadIdx.x;
  const uint8_t* s = reinterpret_cast<const uint8_t*>(p.stream + (int64_t)fr * p.words);
  uint32_t v = 0;
  int ff = 0, n = 0;
  for (int i = 0; i < 4 && b + i < nbytes; ++i, ++n) {
    const uint32_t c = s[b + i];
    v |= c << (8 * i);
    ff += c == 0xFF;
  }
  int64_t total;
  int64_t o = block_scan<kTileThreads>(ff, sums, &total) + p.tile_ff[(int64_t)fr * p.tiles + blockIdx.x] + b +
              COCLR_JPEG_HEADER_BYTES;
  for (int i = 0; i < n; ++i) {
    const uint8_t c = (uint8_t)(v >> (8 * i));
    out[o++] = c;
    if (c == 0xFF) out[o++] = 0;
  }
}

bool args_ok(const coclr_jpeg_encode_t* p, const Geometry& g) {
  if (!p || p->n < 0 || !settings_ok(p->h, p->w, p->subsampling) || p->quality < 1 || p->quality > 100) return false;
  if (p->n == 0) return true;
  if (!p->rgb || !p->out || !p->offsets || !p->work || reinterpret_cast<uintptr_t>(p->work) % 256) return false;
  if (p->row_stride < 3 * (int64_t)p->w) return false;
  if (p->n > 1 && p->frame_stride < (int64_t)(p->h - 1) * p->row_stride + 3 * p->w) return false;
  const size_t max_bytes = coclr_jpeg_encode_max_bytes(p->h, p->w, p->subsampling);
  if (p->out_bytes / (size_t)p->n < max_bytes) return false;
  return (size_t)layout(g, 1).bytes <= p->work_bytes;
}

}  // namespace
}  // namespace coclr

extern "C" int coclr_jpeg_encode_header(int h, int w, int quality, int subsampling, uint8_t* out) {
  using namespace coclr;
  if (!out) return COCLR_E_ARG;
  Header hd;
  const int n = write_header(h, w, quality, subsampling, &hd);
  if (n < 0) return n;
  memcpy(out, hd.b, n);
  return n;
}

extern "C" size_t coclr_jpeg_encode_max_bytes(int h, int w, int subsampling) {
  using namespace coclr;
  if (!settings_ok(h, w, subsampling)) return 0;
  const Geometry g = geometry(h, w, subsampling);
  // every byte of the unstuffed segment may be 0xFF and gain a 0x00
  return COCLR_JPEG_HEADER_BYTES + 2 * (size_t)((g.blocks * kBlockBits + 7) / 8) + 2;
}

extern "C" size_t coclr_jpeg_encode_work_bytes(int n, int h, int w, int subsampling) {
  using namespace coclr;
  if (n < 0 || !settings_ok(h, w, subsampling)) return 0;
  return (size_t)layout(geometry(h, w, subsampling), n > 0 ? n : 1).bytes;
}

extern "C" int coclr_jpeg_encode(const coclr_jpeg_encode_t* a, coclr_stream_t stream) {
  using namespace coclr;
  if (!a || !settings_ok(a->h, a->w, a->subsampling)) return COCLR_E_ARG;
  const Geometry g = geometry(a->h, a->w, a->subsampling);
  if (!args_ok(a, g)) return COCLR_E_ARG;
  if (a->n == 0) return COCLR_OK;
  Header hd;
  write_header(a->h, a->w, a->quality, a->subsampling, &hd);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // frames per pass: as many as the workspace holds (one always does), at most 65535 (grid y)
  int per = 1, hi = a->n < 65535 ? a->n : 65535;
  while (per < hi) {
    const int mid = per + (hi - per + 1) / 2;
    if ((size_t)layout(g, mid).bytes <= a->work_bytes) per = mid;
    else hi = mid - 1;
  }
  uint8_t* work = static_cast<uint8_t*>(a->work);
  for (int f0 = 0; f0 < a->n; f0 += per) {
    const int nf = a->n - f0 < per ? a->n - f0 : per;
    const Layout l = layout(g, nf);
    Pass p;
    p.rgb = a->rgb + (int64_t)f0 * a->frame_stride;
    p.frame_stride = a->frame_stride;
    p.row_stride = a->row_stride;
    p.h = a->h;
    p.w = a->w;
    p.hs = g.hs, p.vs = g.vs, p.lpm = g.lpm, p.bpm = g.bpm, p.mx = g.mx, p.my = g.my, p.wb = g.wb, p.hb = g.hb;
    p.blocks = g.blocks, p.words = g.words, p.tiles = g.tiles;
    p.coef = reinterpret_cast<int16_t*>(work + l.coef);
    p.bits = reinterpret_cast<int64_t*>(work + l.bits);
    p.stream = reinterpret_cast<uint32_t*>(work + l.stream);
    p.tile_ff = reinterpret_cast<int64_t*>(work + l.tiles);
    p.frame = reinterpret_cast<int64_t*>(work + l.frame);
    p.offsets = a->offsets + f0;
    p.out = a->out;
    p.nf = nf;
    p.first = f0 == 0;
    const unsigned bx_tx = (unsigned)((g.blocks + kTxBlocks - 1) / kTxBlocks);
    const unsigned bx_h = (unsigned)((g.blocks + kHuffThreads - 1) / kHuffThreads);
    if (cudaMemsetAsync(p.stream, 0, (size_t)nf * g.words * 4, st) != cudaSuccess) return COCLR_E_LAUNCH;
    jpeg_enc_transform_kernel<<<dim3(bx_tx, nf), 8 * kTxBlocks, 0, st>>>(p, hd);
    jpeg_enc_huff_kernel<false><<<dim3(bx_h, nf), kHuffThreads, 0, st>>>(p, hd);
    jpeg_enc_scan_kernel<<<nf, kScanThreads, 0, st>>>(p.bits, g.blocks, p.frame);
    jpeg_enc_huff_kernel<true><<<dim3(bx_h, nf), kHuffThreads, 0, st>>>(p, hd);
    jpeg_enc_tile_kernel<<<dim3((unsigned)g.tiles, nf), kTileThreads, 0, st>>>(p);
    jpeg_enc_scan_kernel<<<nf, kScanThreads, 0, st>>>(p.tile_ff, g.tiles, p.frame + 1);
    jpeg_enc_offsets_kernel<<<1, kScanThreads, 0, st>>>(p);
    jpeg_enc_scatter_kernel<<<dim3((unsigned)g.tiles, nf), kTileThreads, 0, st>>>(p, hd);
    if (cudaGetLastError() != cudaSuccess) return COCLR_E_LAUNCH;
  }
  return COCLR_OK;
}
