// JPEG decoding, bit-identical to Pillow's libjpeg-turbo (coclr_b200.h, coclr_jpeg_*): a host header parser, then per
// pass three kernels: Huffman decoding (one warp per frame), dequantise + ISLOW IDCT, fancy upsampling + YCbCr -> RGB.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "coclr_b200.h"
#include "jpeg_tables.cuh"

namespace coclr {
namespace {

// ---------------------------------------------------------------------------------------------------------------------
// host: header parser
// ---------------------------------------------------------------------------------------------------------------------

struct HuffSrc {                  // a table as the DHT states it
  bool defined = false;
  uint8_t bits[16];
  uint8_t val[256];
  int nval = 0;
};

// libjpeg jpeg_make_d_derived_tbl's checks: the codes of each length fit, none all ones; DC symbols at most 15
bool huff_valid(const HuffSrc& t, bool dc) {
  int code = 0;
  for (int l = 1; l <= 16; ++l) {
    code += t.bits[l - 1];
    if (code >= (1 << l)) return false;          // as libjpeg: no code may be all ones
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < t.nval; ++i)
      if (t.val[i] > 15) return false;
  return true;
}

void derive(const HuffSrc& t, coclr_jpeg_huff_t* d) {
  memset(d, 0, sizeof(*d));
  memcpy(d->bits, t.bits, 16);
  memcpy(d->val, t.val, t.nval);
  d->nval = t.nval;
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    const int n = t.bits[l - 1];
    d->valoff[l] = k - code;
    for (int i = 0; i < n; ++i, ++code, ++k)
      if (l <= 9)
        for (int s = 0; s < (1 << (9 - l)); ++s) d->look[(code << (9 - l)) | s] = (uint16_t)((l << 8) | t.val[k]);
    d->maxcode[l] = n ? code - 1 : -1;
    code <<= 1;
  }
  d->maxcode[0] = d->maxcode[17] = -1;
}

struct Tables {                   // the batch's distinct tables
  coclr_jpeg_quant_t* quant;
  int max_quant, n_quant = 0;
  coclr_jpeg_huff_t* huff;
  int max_huff, n_huff = 0;
  std::vector<coclr_jpeg_quant_t> q;
  std::vector<HuffSrc> h;

  int add_quant(const uint16_t* qv) {
    for (int i = 0; i < (int)q.size(); ++i)
      if (!memcmp(q[i].q, qv, 128)) return i;
    coclr_jpeg_quant_t t;
    memcpy(t.q, qv, 128);
    q.push_back(t);
    if (n_quant < max_quant) quant[n_quant] = t;
    return n_quant++;
  }
  int add_huff(const HuffSrc& s) {
    for (int i = 0; i < (int)h.size(); ++i)
      if (h[i].nval == s.nval && !memcmp(h[i].bits, s.bits, 16) && !memcmp(h[i].val, s.val, s.nval)) return i;
    h.push_back(s);
    if (n_huff < max_huff) derive(s, &huff[n_huff]);
    return n_huff++;
  }
};

inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

int parse_frame(const uint8_t* d, int64_t n, int64_t base, Tables& tabs, coclr_jpeg_frame_t* f) {
  if (n < 2 || d[0] != 0xFF || d[1] != 0xD8) return COCLR_JPEG_NO_SOI;
  int64_t pos = 2;
  uint16_t qt[4][64];
  bool qdef[4] = {false, false, false, false};
  HuffSrc dht[2][4];
  int restart = 0;
  bool have_sof = false, have_scan = false, jfif = false, adobe = false;
  int adobe_transform = 0;
  int h = 0, w = 0, nf = 0;
  int cid[3] = {0, 0, 0}, samp_h[3] = {0, 0, 0}, samp_v[3] = {0, 0, 0}, tq[3] = {0, 0, 0};
  for (;;) {
    while (pos < n && d[pos] != 0xFF) ++pos;   // libjpeg skips garbage before a marker, then fill bytes
    while (pos < n && d[pos] == 0xFF) ++pos;
    if (pos >= n) return have_scan ? COCLR_JPEG_NO_EOI : (have_sof ? COCLR_JPEG_NO_SOS : COCLR_JPEG_NO_SOF);
    const int m = d[pos++];
    if (m == 0xD9) {
      if (!have_scan) return have_sof ? COCLR_JPEG_NO_SOS : COCLR_JPEG_NO_SOF;
      break;
    }
    if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
    if (pos + 2 > n) return COCLR_JPEG_TRUNCATED;
    const int L = be16(d + pos);
    if (L < 2) return COCLR_JPEG_BAD_SEGMENT;
    if (pos + L > n) return COCLR_JPEG_TRUNCATED;
    const uint8_t* s = d + pos + 2;
    const int len = L - 2;
    pos += L;
    if (m == 0xDA) {
      if (have_scan) return COCLR_JPEG_MULTI_SCAN;
      if (!have_sof) return COCLR_JPEG_NO_SOF;
      if (len < 1 || len != 1 + 2 * s[0] + 3) return COCLR_JPEG_BAD_SEGMENT;
      if (s[0] != nf) return COCLR_JPEG_MULTI_SCAN;
      for (int i = 0; i < nf; ++i) {
        int at = -1;
        for (int j = 0; j < nf; ++j)
          if (cid[j] == s[1 + 2 * i]) at = j;
        if (at != i) return COCLR_JPEG_BAD_SEGMENT;
        const int td = s[2 + 2 * i] >> 4, ta = s[2 + 2 * i] & 15;
        if (td > 3 || ta > 3 || !qdef[tq[i]]) return COCLR_JPEG_BAD_TABLE;
        HuffSrc t[2] = {dht[0][td], dht[1][ta]};
        for (int c = 0; c < 2; ++c) {
          const int slot = c ? ta : td;
          if (!t[c].defined) {              // libjpeg falls back to the Annex K tables for slots 0 and 1
            if (slot > 1) return COCLR_JPEG_BAD_TABLE;
            memcpy(t[c].bits, c ? kStdAcBits[slot] : kStdDcBits[slot], 16);
            t[c].nval = c ? 162 : 12;
            memcpy(t[c].val, c ? kStdAcVal[slot] : kStdDcVal, t[c].nval);
            t[c].defined = true;
          }
          if (!huff_valid(t[c], c == 0)) return COCLR_JPEG_BAD_TABLE;
        }
        f->qt[i] = tabs.add_quant(qt[tq[i]]);
        f->dc[i] = tabs.add_huff(t[0]);
        f->ac[i] = tabs.add_huff(t[1]);
      }
      f->ecs_begin = base + pos;
      for (;;) {                            // the segment ends at the first marker other than RSTn
        const uint8_t* ff = (const uint8_t*)memchr(d + pos, 0xFF, (size_t)(n - pos));
        if (!ff || ff + 1 >= d + n) return COCLR_JPEG_NO_EOI;
        int64_t k = ff - d + 1;
        while (k < n && d[k] == 0xFF) ++k;
        if (k >= n) return COCLR_JPEG_NO_EOI;
        if (d[k] == 0 || (d[k] >= 0xD0 && d[k] <= 0xD7)) {
          pos = k + 1;
          continue;
        }
        pos = ff - d;
        break;
      }
      f->ecs_end = base + pos;
      have_scan = true;
      continue;
    }
    if (m == 0xC0 || m == 0xC1) {
      if (have_sof || len < 6) return COCLR_JPEG_BAD_SEGMENT;
      const int P = s[0];
      h = be16(s + 1);
      w = be16(s + 3);
      nf = s[5];
      if (len != 6 + 3 * nf) return COCLR_JPEG_BAD_SEGMENT;
      if (P != 8) return COCLR_JPEG_PRECISION;
      if (nf != 1 && nf != 3) return COCLR_JPEG_COMPONENTS;
      if (h == 0 || w == 0) return COCLR_JPEG_BAD_SEGMENT;
      for (int i = 0; i < nf; ++i) {
        cid[i] = s[6 + 3 * i];
        samp_h[i] = s[7 + 3 * i] >> 4;
        samp_v[i] = s[7 + 3 * i] & 15;
        tq[i] = s[8 + 3 * i];
        if (tq[i] > 3 || samp_h[i] < 1 || samp_h[i] > 4 || samp_v[i] < 1 || samp_v[i] > 4)
          return COCLR_JPEG_BAD_SEGMENT;
        for (int j = 0; j < i; ++j)
          if (cid[j] == cid[i]) return COCLR_JPEG_BAD_SEGMENT;
      }
      have_sof = true;
    } else if (m == 0xC2 || m == 0xC6) {
      return m == 0xC2 ? COCLR_JPEG_PROGRESSIVE : COCLR_JPEG_SOF_KIND;
    } else if (m == 0xCA) {
      return COCLR_JPEG_ARITHMETIC;
    } else if (m == 0xCE || m == 0xC3 || m == 0xC5 || m == 0xC7) {
      return COCLR_JPEG_SOF_KIND;
    } else if (m == 0xC9 || m == 0xCB || m == 0xCD || m == 0xCF || m == 0xCC) {
      return COCLR_JPEG_ARITHMETIC;
    } else if (m == 0xDB) {
      for (int i = 0; i < len;) {
        const int pq = s[i] >> 4, t = s[i] & 15, sz = pq ? 128 : 64;
        if (pq > 1 || t > 3 || i + 1 + sz > len) return COCLR_JPEG_BAD_SEGMENT;
        for (int k = 0; k < 64; ++k)
          qt[t][kZigzag[k]] = (uint16_t)(pq ? be16(s + i + 1 + 2 * k) : s[i + 1 + k]);
        qdef[t] = true;
        i += 1 + sz;
      }
    } else if (m == 0xC4) {
      for (int i = 0; i < len;) {
        if (i + 17 > len) return COCLR_JPEG_BAD_SEGMENT;
        const int tc = s[i] >> 4, th = s[i] & 15;
        int cnt = 0;
        for (int k = 0; k < 16; ++k) cnt += s[i + 1 + k];
        if (tc > 1 || th > 3 || cnt > 256 || i + 17 + cnt > len) return COCLR_JPEG_BAD_SEGMENT;
        HuffSrc& t = dht[tc][th];
        t.defined = true;
        memcpy(t.bits, s + i + 1, 16);
        memcpy(t.val, s + i + 17, cnt);
        t.nval = cnt;
        i += 17 + cnt;
      }
    } else if (m == 0xDD) {
      if (len != 2) return COCLR_JPEG_BAD_SEGMENT;
      restart = be16(s);
    } else if (m == 0xE0) {
      if (len >= 14 && !memcmp(s, "JFIF\0", 5)) jfif = true;
    } else if (m == 0xEE) {
      if (len >= 12 && !memcmp(s, "Adobe", 5)) {
        adobe = true;
        adobe_transform = s[11];
      }
    } else if (m == 0xDC) {
      return COCLR_JPEG_BAD_SEGMENT;         // DNL
    }                                         // other APPn, COM, unknown markers: skipped
  }
  int hs = 1, vs = 1;
  if (nf == 3) {
    if (!jfif && ((adobe && adobe_transform == 0) || (!adobe && cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B')))
      return COCLR_JPEG_RGB;
    const bool luma_ok = (samp_h[0] == 1 && samp_v[0] == 1) || (samp_h[0] == 2 && (samp_v[0] == 1 || samp_v[0] == 2));
    if (!luma_ok || samp_h[1] != 1 || samp_v[1] != 1 || samp_h[2] != 1 || samp_v[2] != 1) return COCLR_JPEG_SAMPLING;
    hs = samp_h[0];
    vs = samp_v[0];
  }
  f->h = h;
  f->w = w;
  f->ncomp = nf;
  f->hs = hs;
  f->vs = vs;
  f->restart = restart;
  f->mcus_x = (w + 8 * hs - 1) / (8 * hs);
  f->mcus_y = (h + 8 * vs - 1) / (8 * vs);
  f->blocks = (int64_t)f->mcus_x * f->mcus_y * (nf == 1 ? 1 : hs * vs + 2);
  return COCLR_JPEG_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// device
// ---------------------------------------------------------------------------------------------------------------------

// component c: its sampling and blocks per row, and its first block within the frame
__host__ __device__ inline int comp_hs(const coclr_jpeg_frame_t& f, int c) { return (f.ncomp == 1 || c) ? 1 : f.hs; }
__host__ __device__ inline int comp_vs(const coclr_jpeg_frame_t& f, int c) { return (f.ncomp == 1 || c) ? 1 : f.vs; }
__host__ __device__ inline int comp_bw(const coclr_jpeg_frame_t& f, int c) { return f.mcus_x * comp_hs(f, c); }
__host__ __device__ inline int64_t comp_first(const coclr_jpeg_frame_t& f, int c) {
  const int64_t luma = (int64_t)f.mcus_x * f.mcus_y * comp_hs(f, 0) * comp_vs(f, 0);
  return c == 0 ? 0 : luma + (c - 1) * (int64_t)f.mcus_x * f.mcus_y;
}

// ---- entropy decoding: one warp per frame, lane 0 decodes, the warp stores each block -------------------------------

constexpr int kEntropyWarps = 4;

struct Bits {                     // MSB-first bit reader over [p, end) with FF 00 unstuffing
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;                   // the low n bits are the stream's next bits
  int n;
  int fake;                       // zero bits made up past the data (libjpeg feeds zeros after a marker)
  bool marker;                    // p is at the marker that ends the data

  __device__ void fill() {        // to at least 57 bits
    while (n <= 56) {
      uint32_t c = 0;
      if (!marker && p < end) {
        c = __ldg(p);
        if (c == 0xFF) {
          const uint8_t* q = p + 1;
          while (q < end && __ldg(q) == 0xFF) ++q;
          if (q < end && __ldg(q) == 0) {
            p = q + 1;
          } else {
            marker = true;
            continue;
          }
        } else {
          ++p;
        }
      } else {
        fake += 8;
      }
      acc = (acc << 8) | c;
      n += 8;
    }
  }
  __device__ uint32_t peek(int k) const { return (uint32_t)(acc >> (n - k)) & ((1u << k) - 1); }
  __device__ uint32_t get(int k) {
    const uint32_t v = peek(k);
    n -= k;
    return v;
  }
  __device__ bool overrun() const { return n < fake; }   // bits past the real data were consumed
  // drops the buffered bits and reads the next marker as libjpeg's next_marker does; returns RSTn's n, or -1
  __device__ int restart() {
    acc = 0;
    n = fake = 0;
    const uint8_t* k = p;
    for (;;) {
      while (k < end && __ldg(k) != 0xFF) ++k;
      while (k < end && __ldg(k) == 0xFF) ++k;
      if (k >= end || __ldg(k) != 0) break;
      ++k;
    }
    if (k >= end) return -1;
    const int m = __ldg(k);
    if (m < 0xD0 || m > 0xD7) return -1;
    p = k + 1;
    marker = false;
    return m - 0xD0;
  }
};

struct SmemHuff {                 // the prefix of coclr_jpeg_huff_t the decoder reads
  uint16_t look[512];
  int maxcode[18];
  int valoff[18];
  uint8_t val[256];
};
constexpr int kSmemHuffInts = sizeof(SmemHuff) / 4;

// the symbol, or -1 for a bit pattern that is no code; needs n >= 16
__device__ __forceinline__ int huff_decode(Bits& b, const SmemHuff& t) {
  const int e = t.look[b.peek(9)];
  if (e) {
    b.n -= e >> 8;
    return e & 255;
  }
  for (int l = 10; l <= 16; ++l) {
    const int code = (int)b.peek(l);
    if (code <= t.maxcode[l]) {
      b.n -= l;
      return t.val[(code + t.valoff[l]) & 255];
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(uint32_t r, int s) {
  return r < (1u << (s - 1)) ? (int)r - (1 << s) + 1 : (int)r;
}

// one block into out (zeroed); returns 0 or COCLR_JPEG_ST_BAD_CODE
__device__ __forceinline__ int decode_block(Bits& b, const SmemHuff& dct, const SmemHuff& act, int& pred,
                                            int16_t* out) {
  if (b.n < 32) b.fill();
  const int s = huff_decode(b, dct);
  if (s < 0) return COCLR_JPEG_ST_BAD_CODE;
  if (s) pred += extend(b.get(s), s);
  out[0] = (int16_t)pred;
  for (int k = 1; k < 64; ++k) {
    if (b.n < 32) b.fill();
    const int rs = huff_decode(b, act);
    if (rs < 0) return COCLR_JPEG_ST_BAD_CODE;
    const int r = rs >> 4, sz = rs & 15;
    if (sz) {
      k += r;
      out[kZigzagDev[k < 63 ? k : 63]] = (int16_t)extend(b.get(sz), sz);   // libjpeg clamps a run past 63 too
    } else {
      if (r != 15) break;
      k += 15;
    }
  }
  return 0;
}

__global__ void __launch_bounds__(32 * kEntropyWarps) jpeg_entropy_kernel(coclr_jpeg_t p, int f0, int f1) {
  __shared__ SmemHuff tabs[kEntropyWarps][6];     // per warp: DC and AC table of each component
  __shared__ __align__(16) int16_t blk[kEntropyWarps][64];
  __shared__ int slots[kEntropyWarps][6], preds[kEntropyWarps][3];   // shared, not indexed registers (no local memory)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fi = f0 + blockIdx.x * kEntropyWarps + warp;
  if (fi >= f1) return;
  const coclr_jpeg_frame_t& fr = p.frames[fi];
  const coclr_jpeg_frame_t f = fr;
  int16_t* ws = reinterpret_cast<int16_t*>(p.work) + (f.block0 - p.frames[f0].block0) * 64;

  // table slot of (component, DC/AC): a table the frame uses twice is loaded once
  SmemHuff* T = tabs[warp];
  int* slot = slots[warp];
  int* pred = preds[warp];
  for (int t = 0; t < 2 * f.ncomp; ++t) {
    const int idx = (t & 1) ? fr.ac[t >> 1] : fr.dc[t >> 1];   // indexed: read from the record, not a copy
    int st = t;
    for (int u = 0; u < t; ++u)
      if (((u & 1) == (t & 1)) && ((u & 1) ? fr.ac[u >> 1] : fr.dc[u >> 1]) == idx) {
        st = u;
        break;
      }
    if (lane == 0) slot[t] = st;
    if (st == t) {
      const int* g = reinterpret_cast<const int*>(&p.huff[idx]);
      int* s = reinterpret_cast<int*>(&T[t]);
      for (int i = lane; i < kSmemHuffInts; i += 32) s[i] = __ldg(g + i);
    }
  }
  reinterpret_cast<int*>(blk[warp])[lane] = 0;
  if (lane < 3) pred[lane] = 0;
  __syncwarp();

  Bits b;
  b.p = p.data + f.ecs_begin;
  b.end = p.data + f.ecs_end;
  b.acc = 0;
  b.n = b.fake = 0;
  b.marker = false;
  int status = 0, next_rst = 0;
  const int nmcu = f.mcus_x * f.mcus_y;
  for (int m = 0; m < nmcu && !status; ++m) {
    if (lane == 0 && f.restart && m && m % f.restart == 0) {
      if (b.overrun()) {
        status = COCLR_JPEG_ST_EARLY_END;
      } else if (b.restart() != next_rst) {
        status = COCLR_JPEG_ST_BAD_RESTART;
      } else {
        next_rst = (next_rst + 1) & 7;
        pred[0] = pred[1] = pred[2] = 0;
      }
    }
    status = __shfl_sync(0xffffffffu, status, 0);   // the whole warp leaves on a bad restart, not lane 0 alone
    const int mrow = m / f.mcus_x, mcol = m - mrow * f.mcus_x;
    for (int c = 0; c < f.ncomp && !status; ++c) {
      const int hc = comp_hs(f, c), vc = comp_vs(f, c), bw = comp_bw(f, c);
      const int64_t c0 = comp_first(f, c);
      for (int v = 0; v < vc && !status; ++v)
        for (int u = 0; u < hc && !status; ++u) {
          if (lane == 0 && !status)
            status = decode_block(b, T[slot[2 * c]], T[slot[2 * c + 1]], pred[c], blk[warp]);
          status = __shfl_sync(0xffffffffu, status, 0);
          __syncwarp();
          if (!status) {
            const int64_t bi = c0 + (int64_t)(mrow * vc + v) * bw + (mcol * hc + u);
            int* src = reinterpret_cast<int*>(blk[warp]);
            reinterpret_cast<int*>(ws + bi * 64)[lane] = src[lane];
            src[lane] = 0;
          }
          __syncwarp();
        }
    }
  }
  if (lane == 0) {
    if (!status && b.overrun()) status = COCLR_JPEG_ST_EARLY_END;
    p.status[fi] = status;
  }
}

// ---- dequantise + ISLOW IDCT: 32 blocks per CTA, 8 threads per block -----------------------------------------------

constexpr int kIdctBlocks = 32;

// jidctint.c's butterfly: x[0..7] in, the eight outputs scaled by 2^13 out (int32 as libjpeg's JLONG on these ranges)
__device__ __forceinline__ void idct_1d(const int* x, int* o) {
  const int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
            F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
  int z1 = (x[2] + x[6]) * F0541;
  const int t2 = z1 - x[6] * F1847;
  const int t3 = z1 + x[2] * F0765;
  const int t0 = (x[0] + x[4]) * 8192;
  const int t1 = (x[0] - x[4]) * 8192;
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  int o0 = x[7], o1 = x[5], o2 = x[3], o3 = x[1];
  z1 = o0 + o3;
  int z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const int z5 = (z3 + z4) * F1175;
  o0 *= F0298;
  o1 *= F2053;
  o2 *= F3072;
  o3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 = z3 * -F1961 + z5;
  z4 = z4 * -F0390 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  o[0] = t10 + o3;
  o[7] = t10 - o3;
  o[1] = t11 + o2;
  o[6] = t11 - o2;
  o[2] = t12 + o1;
  o[5] = t12 - o1;
  o[3] = t13 + o0;
  o[4] = t13 - o0;
}

__global__ void __launch_bounds__(8 * kIdctBlocks) jpeg_idct_kernel(coclr_jpeg_t p, int f0) {
  __shared__ __align__(16) int16_t coef[kIdctBlocks][64];
  __shared__ int wsp[kIdctBlocks][64];
  __shared__ __align__(16) uint8_t pix[kIdctBlocks][64];
  __shared__ uint16_t q[3][64];
  const coclr_jpeg_frame_t& f = p.frames[f0 + blockIdx.y];
  const int64_t nb = f.blocks;
  const int64_t b0 = (int64_t)blockIdx.x * kIdctBlocks;
  if (b0 >= nb) return;
  const int ncomp = f.ncomp;
  const int64_t c1 = comp_first(f, 1), c2 = comp_first(f, 2);
  int16_t* ws = reinterpret_cast<int16_t*>(p.work) + (f.block0 - p.frames[f0].block0) * 64;
  const int t = threadIdx.x;
  for (int i = t; i < ncomp * 64; i += blockDim.x) q[i >> 6][i & 63] = p.quant[f.qt[i >> 6]].q[i & 63];
  const int nblk = nb - b0 < kIdctBlocks ? (int)(nb - b0) : kIdctBlocks;
  {                                               // 16 bytes per thread: the CTA's 32 blocks
    const int bl = t >> 3;
    if (bl < nblk)
      reinterpret_cast<int4*>(coef[bl])[t & 7] = reinterpret_cast<const int4*>(ws + (b0 + bl) * 64)[t & 7];
  }
  __syncthreads();
  const int bl = t >> 3, j = t & 7;
  const int64_t gb = b0 + bl;
  const int c = ncomp == 1 ? 0 : (gb >= c2 ? 2 : (gb >= c1 ? 1 : 0));
  int x[8], o[8];
  if (bl < nblk) {                                // pass 1: column j
    bool ac = false;
    for (int r = 0; r < 8; ++r) {
      x[r] = (int)coef[bl][r * 8 + j] * (int)q[c][r * 8 + j];
      ac |= r && x[r];
    }
    if (!ac) {                                    // libjpeg's DC-only shortcut gives the same values
      for (int r = 0; r < 8; ++r) wsp[bl][r * 8 + j] = x[0] * 4;
    } else {
      idct_1d(x, o);
      for (int r = 0; r < 8; ++r) wsp[bl][r * 8 + j] = (o[r] + (1 << 10)) >> 11;
    }
  }
  __syncthreads();
  if (bl < nblk) {                                // pass 2: row j
    for (int k = 0; k < 8; ++k) x[k] = wsp[bl][j * 8 + k];
    idct_1d(x, o);
    for (int k = 0; k < 8; ++k) pix[bl][j * 8 + k] = (uint8_t)min(max(((o[k] + (1 << 17)) >> 18) + 128, 0), 255);
  }
  __syncthreads();
  if (t < nblk * 4)                               // block b's samples over the first 64 of its 128 bytes
    reinterpret_cast<int4*>(ws + (b0 + (t >> 2)) * 64)[t & 3] = reinterpret_cast<const int4*>(pix[t >> 2])[t & 3];
}

// ---- fancy upsampling + colour conversion, one thread per output pixel ----------------------------------------------

// sample (y, x) of component c (the IDCT's output: 64 bytes at the start of each 128-byte block)
__device__ __forceinline__ int sample(const uint8_t* ws, const coclr_jpeg_frame_t& f, int c, int y, int x) {
  const int64_t bi = comp_first(f, c) + (int64_t)(y >> 3) * comp_bw(f, c) + (x >> 3);
  return ws[bi * 128 + (y & 7) * 8 + (x & 7)];
}

// libjpeg's upsampled chroma at luma pixel (y, x): h2v1 / h2v2 fancy, or replication when the chroma is at most two
// samples wide; cw, ch: the chroma's real (downsampled) width and height
__device__ __forceinline__ int chroma(const uint8_t* ws, const coclr_jpeg_frame_t& f, int c, int y, int x, int cw,
                                      int ch) {
  const int hs = f.hs, vs = f.vs;
  if (hs == 1) return sample(ws, f, c, y, x);
  const int cy = vs == 2 ? y >> 1 : y, cx = x >> 1;
  if (cw <= 2) return sample(ws, f, c, cy, cx);
  const bool right = x & 1;                       // the second output of the pair leans on the next column
  const int ox = right ? cx + 1 : cx - 1;
  const bool edge = ox < 0 || ox >= cw;
  if (vs == 1) {
    const int a = sample(ws, f, c, cy, cx);
    if (edge) return a;
    return (3 * a + sample(ws, f, c, cy, ox) + (right ? 2 : 1)) >> 2;
  }
  const int oy = min(max((y & 1) ? cy + 1 : cy - 1, 0), ch - 1);
  const int s0 = 3 * sample(ws, f, c, cy, cx) + sample(ws, f, c, oy, cx);
  if (edge) return (4 * s0 + (right ? 7 : 8)) >> 4;
  const int s1 = 3 * sample(ws, f, c, cy, ox) + sample(ws, f, c, oy, ox);
  return (3 * s0 + s1 + (right ? 7 : 8)) >> 4;
}

constexpr int kColourX = 32, kColourY = 8;

__global__ void __launch_bounds__(kColourX * kColourY) jpeg_colour_kernel(coclr_jpeg_t p, coclr_jpeg_slots_t sl,
                                                                           int f0) {
  const int fi = f0 + blockIdx.z;
  const coclr_jpeg_frame_t& fr = p.frames[fi];
  const int x = blockIdx.x * kColourX + threadIdx.x, y = blockIdx.y * kColourY + threadIdx.y;
  const int h = fr.h, w = fr.w;
  if (x >= w || y >= h) return;
  const coclr_jpeg_frame_t f = fr;
  const uint8_t* ws = reinterpret_cast<const uint8_t*>(p.work) + (f.block0 - p.frames[f0].block0) * 128;
  const int Y = sample(ws, f, 0, y, x);
  uint8_t r8 = (uint8_t)Y, g8 = r8, b8 = r8;
  if (f.ncomp != 1) {
    const int cw = (w + f.hs - 1) / f.hs, ch = (h + f.vs - 1) / f.vs;
    const int cb = chroma(ws, f, 1, y, x, cw, ch) - 128, cr = chroma(ws, f, 2, y, x, cw, ch) - 128;
    // jdcolor.c: FIX(1.40200), FIX(1.77200), -FIX(0.71414), -FIX(0.34414) with ONE_HALF, 16-bit shift
    r8 = (uint8_t)min(max(Y + ((91881 * cr + 32768) >> 16), 0), 255);
    g8 = (uint8_t)min(max(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16), 0), 255);
    b8 = (uint8_t)min(max(Y + ((116130 * cb + 32768) >> 16), 0), 255);
  }
  // the output frames this frame was sampled into: one store per slot, no second pass over the output
  const int s0 = sl.slot_begin ? sl.slot_begin[fi] : fi, s1 = sl.slot_begin ? sl.slot_begin[fi + 1] : fi + 1;
  const int64_t pix = (int64_t)y * p.row_stride + 3 * x;
  for (int s = s0; s < s1; ++s) {
    uint8_t* out = p.out + (sl.slot_begin ? sl.slots[s] : s) * p.frame_stride + pix;
    out[0] = r8;
    out[1] = g8;
    out[2] = b8;
  }
}

inline bool args_ok(const coclr_jpeg_t* p) {
  if (!p || p->n < 0 || (p->n && (!p->data || !p->frames || !p->frames_host || !p->quant || !p->huff || !p->out ||
                                  !p->status || !p->work)))
    return false;
  if (reinterpret_cast<uintptr_t>(p->work) % 16) return false;
  for (int i = 0; i < p->n; ++i) {
    const coclr_jpeg_frame_t& f = p->frames_host[i];
    if (f.reason != COCLR_JPEG_OK || (size_t)f.blocks * 128 > p->work_bytes) return false;
    if ((int64_t)(f.w * 3) > p->row_stride || (int64_t)(f.h - 1) * p->row_stride + 3 * f.w > p->frame_stride)
      return false;
  }
  return true;
}

// every output frame in [0, n_out) is written by exactly one slot
inline bool slots_ok(const coclr_jpeg_t* p, const coclr_jpeg_slots_t& s) {
  if (!s.slot_begin) return true;
  if (!s.slots || !s.slot_begin_host || !s.slots_host || s.n_out < 0 || s.slot_begin_host[0] != 0 ||
      s.slot_begin_host[p->n] != s.n_out || (s.n_out && p->frame_stride > INT64_MAX / s.n_out))
    return false;
  std::vector<char> seen(s.n_out, 0);
  for (int i = 0; i < p->n; ++i) {
    if (s.slot_begin_host[i + 1] < s.slot_begin_host[i]) return false;
    for (int k = s.slot_begin_host[i]; k < s.slot_begin_host[i + 1]; ++k) {
      const int o = s.slots_host[k];
      if (o < 0 || o >= s.n_out || seen[o]) return false;
      seen[o] = 1;
    }
  }
  return true;
}

}  // namespace
}  // namespace coclr

extern "C" int coclr_jpeg_parse(const uint8_t* data, const int64_t* offsets, int n, coclr_jpeg_frame_t* frames,
                                coclr_jpeg_quant_t* quant, int max_quant, int* n_quant,
                                coclr_jpeg_huff_t* huff, int max_huff, int* n_huff) {
  using namespace coclr;
  if (n < 0 || (n && (!data || !offsets || !frames)) || !n_quant || !n_huff || max_quant < 0 || max_huff < 0)
    return COCLR_E_ARG;
  Tables tabs;
  tabs.quant = quant;
  tabs.max_quant = quant ? max_quant : 0;
  tabs.huff = huff;
  tabs.max_huff = huff ? max_huff : 0;
  int64_t block0 = 0;
  for (int i = 0; i < n; ++i) {
    if (offsets[i + 1] < offsets[i]) return COCLR_E_ARG;
    coclr_jpeg_frame_t* f = &frames[i];
    memset(f, 0, sizeof(*f));
    f->reason = parse_frame(data + offsets[i], offsets[i + 1] - offsets[i], offsets[i], tabs, f);
    if (f->reason != COCLR_JPEG_OK) {
      const int reason = f->reason;
      memset(f, 0, sizeof(*f));
      f->reason = reason;
    }
    f->block0 = block0;
    block0 += f->blocks;
  }
  *n_quant = tabs.n_quant;
  *n_huff = tabs.n_huff;
  return (tabs.n_quant > tabs.max_quant || tabs.n_huff > tabs.max_huff) ? 1 : COCLR_OK;
}

extern "C" size_t coclr_jpeg_work_bytes(const coclr_jpeg_t* p) {
  size_t blocks = 0;
  for (int i = 0; p && p->frames_host && i < p->n; ++i) blocks += (size_t)p->frames_host[i].blocks;
  return blocks * 128;
}

extern "C" int coclr_jpeg_decode(const coclr_jpeg_t* p, coclr_stream_t stream) {
  return coclr_jpeg_decode_slots(p, nullptr, stream);
}

extern "C" int coclr_jpeg_decode_slots(const coclr_jpeg_t* p, const coclr_jpeg_slots_t* s, coclr_stream_t stream) {
  using namespace coclr;
  coclr_jpeg_slots_t sl{};
  if (s) sl = *s;
  if (!args_ok(p) || !slots_ok(p, sl)) return COCLR_E_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const coclr_jpeg_frame_t* F = p->frames_host;
  const int kMaxPassFrames = 65535;               // the IDCT and colour grids put the pass's frames in y and z
  for (int f0 = 0; f0 < p->n;) {                  // a pass: consecutive frames whose blocks fit the workspace
    int f1 = f0;
    int64_t max_blocks = 0;
    int max_h = 0, max_w = 0;
    while (f1 < p->n && f1 - f0 < kMaxPassFrames &&
           (size_t)(F[f1].block0 + F[f1].blocks - F[f0].block0) * 128 <= p->work_bytes) {
      max_blocks = max(max_blocks, F[f1].blocks);
      max_h = max(max_h, F[f1].h);
      max_w = max(max_w, F[f1].w);
      ++f1;
    }
    const int nf = f1 - f0;
    jpeg_entropy_kernel<<<(nf + kEntropyWarps - 1) / kEntropyWarps, 32 * kEntropyWarps, 0, st>>>(*p, f0, f1);
    jpeg_idct_kernel<<<dim3((unsigned)((max_blocks + kIdctBlocks - 1) / kIdctBlocks), nf), 8 * kIdctBlocks, 0, st>>>(
        *p, f0);
    jpeg_colour_kernel<<<dim3((max_w + kColourX - 1) / kColourX, (max_h + kColourY - 1) / kColourY, nf),
                         dim3(kColourX, kColourY), 0, st>>>(*p, sl, f0);
    if (cudaGetLastError() != cudaSuccess) return COCLR_E_LAUNCH;
    f0 = f1;
  }
  return COCLR_OK;
}
