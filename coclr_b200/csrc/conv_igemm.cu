// Implicit-GEMM 3-D convolution on wgmma tensor cores (sm_90a): forward, data-gradient and
// weight-gradient kernels plus the weight packer.
//
// Replaces nn.Conv3d + the statistics half of nn.BatchNorm3d of the reference
// (backbone/s3dg.py:8-28 BasicConv3d, :30-65 STConv3d; model/pretrain.py:52,54) and the cuDNN
// dgrad / wgrad that loss.backward() (main_nce.py:330) dispatches.
//
// Design (see DESIGN.md section 3):
//  * every activation a conv consumes lives in HBM as a pair of channels-last 16-bit planes (hi, lo) with
//    hi + lo == the fp32 value to ~22 bits (fp16 pair) -- written once by the BatchNorm-apply/ReLU/split
//    kernel (or the pooling kernel) that finalises the producer's output;
//  * producer warps only generate addresses: 16-byte cp.async (LDGSTS) copies with hardware zero-fill for
//    padding land 128 pixels x 64 K-elements straight in 128B-swizzled shared-memory tiles; weights arrive
//    pre-split and pre-swizzled through one bulk (TMA-engine) copy per stage;
//  * two consumer warpgroups (64 pixel rows each) issue wgmma (M=64, N<=128, K=16) for the three products
//    hi*lo, lo*hi, hi*hi into one fp32 register accumulator (fp32-equivalent result), or hi*hi only in
//    single-pass mode;
//  * the accumulator goes through shared memory 32 columns at a time; four of the consumer warps then make
//    coalesced stores and accumulate the per-channel sum / sum-of-squares that train-mode BatchNorm needs.
#include "common.cuh"
#include "coclr_b200.h"
#include "conv_tma.h"

namespace coclr {

static constexpr int kTileM = 128;      // pixels per tile (two warpgroups of M = 64)
static constexpr int kChunkK = 64;      // K elements per pipeline stage (one 128B swizzle row)
static constexpr int kProducerWarps = 8;       // weight-gradient kernel: 256 threads gather 64 rows x 2 operands
static constexpr int kFwdProducerWarps = 4;    // forward / dgrad kernel: 128 threads gather 128 rows
static constexpr int kMmaWarps = 8;     // two consumer warpgroups: MMA, then the epilogue
static constexpr int kEpiWarps = 4;     // consumer warps that store a tile (32 rows each)
static constexpr int kMaxBN = 128;      // output columns per tile (register accumulator: 64 fp32 per thread)
static constexpr int kAccChunks = kMaxBN / 32;
// warp roles: [0,8) MMA + epilogue, [8,12) producers, 12 weight loader
static constexpr int kThreads = (kMmaWarps + kFwdProducerWarps + 1) * 32;
static constexpr int kWgradThreads = (kMmaWarps + kProducerWarps) * 32;
static constexpr int kStagePitch = 33;  // floats per staged row (conflict-free transpose)
static constexpr int kMaxStages = 6;

// Decompose destination pixel m into the source-space base coordinates used by the gather.
COCLR_DEVINL void row_coords(const coclr_geom_t& G, int Td, int Hd, int Wd, int M, int m, int& b, int& t, int& y,
                             int& x) {
  if (m >= M) {
    b = -1;
    t = y = x = 0;
    return;
  }
  int xx, yy, tt;
  if (((Wd & (Wd - 1)) | (Hd & (Hd - 1)) | (Td & (Td - 1))) == 0) {  // power-of-two grid: shifts, no division
    const int sw = __ffs(Wd) - 1, sh = __ffs(Hd) - 1, st = __ffs(Td) - 1;
    xx = m & (Wd - 1);
    int r = m >> sw;
    yy = r & (Hd - 1);
    r >>= sh;
    tt = r & (Td - 1);
    b = r >> st;
  } else {
    xx = m % Wd;
    int r = m / Wd;
    yy = r % Hd;
    r /= Hd;
    tt = r % Td;
    b = r / Td;
  }
  if (!G.transposed) {
    t = tt * G.st - G.pt;
    y = yy * G.sh - G.ph;
    x = xx * G.sw - G.pw;
  } else {
    t = tt + G.pt;
    y = yy + G.ph;
    x = xx + G.pw;
  }
}

// Issue the cp.async copies of NI*kRowStride rows x 64 K-columns [kbase, kbase+64) of the implicit operand into one
// swizzled [rows][128 B] block (hi plane) and its lo twin.  Thread (ck, r0) owns the 16-byte chunk ck
// (8 consecutive K elements) of rows r0 + kRowStride*i.  K index k = tap*C + channel, C % 8 == 0.
// Position of one 16-byte K granule in (tap, channel) space; kept per thread and advanced incrementally so the
// pipelined loops never divide.
struct TapPos {
  int k0, ta, ya, xa, ci;
};
COCLR_DEVINL TapPos tap_of(const coclr_src_t& S, const coclr_geom_t& G, int k0) {
  TapPos p;
  p.k0 = k0;
  const int tap = k0 / S.C;
  p.ci = k0 - tap * S.C;
  const int khw = G.kh * G.kw;
  p.ta = tap / khw;
  const int rem = tap - p.ta * khw;
  p.ya = rem / G.kw;
  p.xa = rem - p.ya * G.kw;
  return p;
}
COCLR_DEVINL void tap_advance(TapPos& p, const coclr_src_t& S, const coclr_geom_t& G, int step) {
  p.k0 += step;
  p.ci += step;
  while (p.ci >= S.C) {
    p.ci -= S.C;
    if (++p.xa == G.kw) {
      p.xa = 0;
      if (++p.ya == G.kh) {
        p.ya = 0;
        ++p.ta;
      }
    }
  }
}

template <bool kLo, int NI, int kRowStride = 32>
COCLR_DEVINL void gather_block_async(const coclr_src_t& S, const coclr_geom_t& G, int Kreal, const TapPos& tp, int ck,
                                     int r0, const int* rb, const int* rt, const int* ry, const int* rx,
                                     uint32_t blk_hi, uint32_t blk_lo) {
  // This runs once per (row, K chunk) in warps that share their issue slots with everything else on the SM: for
  // narrow layers (N <= 64) the MMAs of a chunk take ~600 cycles, so the address arithmetic is kept to 32-bit pixel
  // indices (host side guarantees B*T*H*W < 2^31) and one widening multiply per row.
  const bool kvalid = tp.k0 < Kreal;
  const int ta = tp.ta, ya = tp.ya, xa = tp.xa;
  const uint16_t* hi = reinterpret_cast<const uint16_t*>(S.hi) + (S.coff + tp.ci);
  const uint16_t* lo = reinterpret_cast<const uint16_t*>(S.lo) + (S.coff + tp.ci);
  const int HW = S.H * S.W;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    bool in = kvalid && rb[i] >= 0;
    int ts, ys, xs;
    if (!G.transposed) {
      ts = rt[i] + ta;
      ys = ry[i] + ya;
      xs = rx[i] + xa;
    } else {
      ts = rt[i] - ta;
      ys = ry[i] - ya;
      xs = rx[i] - xa;
      if (G.st == 2) { in = in && !(ts & 1); ts >>= 1; }   // arithmetic shifts keep negatives negative
      if (G.sh == 2) { in = in && !(ys & 1); ys >>= 1; }
      if (G.sw == 2) { in = in && !(xs & 1); xs >>= 1; }
    }
    in = in && ((unsigned)ts < (unsigned)S.T) && ((unsigned)ys < (unsigned)S.H) && ((unsigned)xs < (unsigned)S.W);
    const int pix = in ? (rb[i] * S.T + ts) * HW + ys * S.W + xs : 0;
    const size_t off = (size_t)(unsigned)pix * (unsigned)S.ld;
    const uint32_t dst = swz128_offset((uint32_t)(r0 + kRowStride * i), (uint32_t)ck);
    const uint32_t nbytes = in ? 16u : 0u;
    cp_async16(blk_hi + dst, hi + off, nbytes);
    if constexpr (kLo) cp_async16(blk_lo + dst, lo + off, nbytes);
  }
}

// ------------------------------------------------------------------------------------------------
// forward / dgrad kernel
// ------------------------------------------------------------------------------------------------
struct ConvSmemLayout {
  uint32_t a_bytes;      // per copy (hi or lo)
  uint32_t b_bytes;      // per copy
  uint32_t stage_bytes;  // all copies of A and B of one stage
  uint32_t stages;
  uint32_t off_stage;    // [128 rows][kStagePitch] fp32: one 32-column chunk of the accumulator for the epilogue
  uint32_t off_stats;    // float [epilogue warps][2][n_tiles*BN + 4]: per-warp BN-statistic partial sums
  uint32_t off_bars;
  uint32_t total;
};

// per-warp BatchNorm statistic tables cover all output channels when those are few (flushed once per CTA), else one
// N-tile (flushed after every tile: wide layers -- ResNet2d3d-50 has up to 2048 channels -- have few pixel tiles)
static constexpr int kStatTableMaxCols = 512;
__host__ __device__ inline int stat_table_cols(int BN, int n_tiles) {
  return n_tiles * BN <= kStatTableMaxCols ? n_tiles * BN : BN;
}

__host__ __device__ inline ConvSmemLayout conv_smem_layout(int BN, int n_tiles, int npass, int want_stats) {
  ConvSmemLayout L;
  const uint32_t copies = npass > 1 ? 2u : 1u;
  L.a_bytes = kTileM * 128u;
  L.b_bytes = (uint32_t)BN * 128u;
  L.stage_bytes = copies * (L.a_bytes + L.b_bytes);
  const uint32_t stat_bytes = want_stats ? kEpiWarps * 2u * (uint32_t)(stat_table_cols(BN, n_tiles) + 4) * 4u : 0u;
  const uint32_t fixed = kEpiWarps * 32u * kStagePitch * 4u + stat_bytes + 256u;
  const uint32_t budget = 227u * 1024u - 1024u /*alignment slack*/ - fixed;
  uint32_t st = budget / L.stage_bytes;
  if (st > (uint32_t)kMaxStages) st = kMaxStages;
  L.stages = st;
  L.off_stage = L.stages * L.stage_bytes;
  L.off_stats = L.off_stage + kEpiWarps * 32u * kStagePitch * 4u;
  L.off_bars = (L.off_stats + stat_bytes + 15u) & ~15u;
  L.total = L.off_bars + 256u + 1024u;
  return L;
}

// Transposed (dgrad) pass of a temporally strided conv: a tap only meets every other output frame, so for a tile that
// lies inside ONE frame (Hd*Wd % 128 == 0) and K chunks that lie inside one tap (C % 64 == 0) whole chunks are zero.
// Bit kc of the returned mask = chunk kc contributes nothing to this tile; producers, weight loader and MMA warpgroups all
// derive the same mask and skip those chunks.  0 when the shortcut does not apply.
COCLR_DEVINL uint64_t zero_chunk_mask(const coclr_conv_t& P, int nkc, int m_tile) {
  if (!P.g.transposed || P.g.st != 2 || (P.src.C & 63) || ((P.Hd * P.Wd) % kTileM) || nkc > 64) return 0ull;
  const int tt = ((m_tile * kTileM) / (P.Hd * P.Wd)) % P.Td + P.g.pt;
  const int chunks_per_plane = (P.src.C >> 6) * P.g.kh * P.g.kw;   // K chunks that share one temporal tap
  uint64_t mask = 0ull;
  int ta = 0, left = chunks_per_plane;
  for (int kc = 0; kc < nkc; ++kc) {
    const int ts = tt - ta;
    if (ts < 0 || (ts & 1) || (ts >> 1) >= P.src.T) mask |= 1ull << kc;
    if (--left == 0) { left = chunks_per_plane; ++ta; }
  }
  if (mask == (nkc >= 64 ? ~0ull : ((1ull << nkc) - 1ull))) mask &= ~1ull;  // keep one chunk: it zero-fills the accumulator
  return mask;
}

template <int kNPass>
__global__ void __launch_bounds__(kThreads, 1) conv_igemm_kernel(const coclr_conv_t P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr bool kLo = kNPass > 1;
  const int M = P.B * P.Td * P.Hd * P.Wd;
  const int nkc = (P.Kreal + kChunkK - 1) / kChunkK;
  const int m_tiles = (M + kTileM - 1) / kTileM;
  const int total_tiles = m_tiles * P.n_tiles;
  const ConvSmemLayout L = conv_smem_layout(P.BN, P.n_tiles, kNPass, P.stats_sum != nullptr);
  const uint32_t nstages = L.stages;

  float* stage_buf = reinterpret_cast<float*>(smem + L.off_stage);
  float* wstats = reinterpret_cast<float*>(smem + L.off_stats);
  const bool stats_per_tile = P.n_tiles * P.BN > kStatTableMaxCols;
  const int stat_cols = stat_table_cols(P.BN, P.n_tiles) + 4;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L.off_bars);  // [kMaxStages]
  uint64_t* empty_bar = full_bar + kMaxStages;                           // [kMaxStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&full_bar[s], kFwdProducerWarps * 32 + 1);  // every producer thread (async, via cp.async) + the weight loader
      mbar_init(&empty_bar[s], kMmaWarps);               // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  if (P.stats_sum != nullptr) {
    for (int i = threadIdx.x; i < kEpiWarps * 2 * stat_cols; i += kThreads) wstats[i] = 0.f;
  }
  __syncthreads();

  if (warp >= kMmaWarps && warp < kMmaWarps + kFwdProducerWarps) {
    // ===================== A-operand producers (address generation + cp.async only) =====================
    const int pt = threadIdx.x - kMmaWarps * 32;  // 0..127
    const int ck = pt & 7;
    const int r0 = pt >> 3;  // 0..15; rows r0 + 16*i
    const uint32_t smem_base = smem_u32(smem);
    uint32_t stage = 0, phase = 0;
    const TapPos tap0 = tap_of(P.src, P.g, ck * 8);  // this thread's K granule in chunk 0 (the only division)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int m_tile = tile / P.n_tiles;
      int rb[8], rt[8], ry[8], rx[8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        row_coords(P.g, P.Td, P.Hd, P.Wd, M, m_tile * kTileM + r0 + 16 * i, rb[i], rt[i], ry[i], rx[i]);
      TapPos tp = tap0;
      const uint64_t zmask = zero_chunk_mask(P, nkc, m_tile);
      for (int kc = 0; kc < nkc; ++kc) {
        if ((zmask >> kc) & 1ull) {
          tap_advance(tp, P.src, P.g, kChunkK);
          continue;
        }
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        const uint32_t sa = smem_base + stage * L.stage_bytes;
        gather_block_async<kLo, 8, 16>(P.src, P.g, P.Kreal, tp, ck, r0, rb, rt, ry, rx, sa, sa + L.a_bytes);
        tap_advance(tp, P.src, P.g, kChunkK);
        // asynchronous arrival when this thread's copies have landed: the producer never waits for data
        cp_async_mbar_arrive_noinc(&full_bar[stage]);
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (warp == kMmaWarps + kFwdProducerWarps) {
    // ===================== weight loader (bulk copies) =====================
    if (elect_one()) {
      const uint32_t copies = kLo ? 2u : 1u;
      const uint32_t bytes = copies * L.b_bytes;
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_tile = tile % P.n_tiles;
        const uint64_t zmask = zero_chunk_mask(P, nkc, tile / P.n_tiles);
        for (int kc = 0; kc < nkc; ++kc) {
          if ((zmask >> kc) & 1ull) continue;
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sb = smem + stage * L.stage_bytes + copies * L.a_bytes;
          const uint8_t* src =
              reinterpret_cast<const uint8_t*>(P.wpk) + ((size_t)n_tile * nkc + kc) * (size_t)(2u * L.b_bytes);
          mbar_arrive_expect_tx(&full_bar[stage], bytes);
          bulk_g2s(sb, src, bytes, &full_bar[stage]);
          if (++stage == nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < kMmaWarps) {
    // ===================== MMA (two warpgroups of 64 rows), then the epilogue =====================
    const int wg = warp >> 2;
    const int tid_wg = threadIdx.x & 127;
    const bool bf16 = P.a_bf16 != 0;
    const uint32_t a_row_off = (uint32_t)wg * 64u * 128u;   // this warpgroup's 64 rows of the A tile
    float* my_stage = stage_buf + warp * 32 * kStagePitch;
    float acc[16 * kAccChunks];
    uint32_t stage = 0, phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int m_tile = tile / P.n_tiles;
      const int n_tile = tile % P.n_tiles;
      const uint64_t zmask = zero_chunk_mask(P, nkc, m_tile);
#pragma unroll
      for (int i = 0; i < 16 * kAccChunks; ++i) acc[i] = 0.f;
      for (int kc = 0; kc < nkc; ++kc) {
        if ((zmask >> kc) & 1ull) continue;
        mbar_wait_spin(&full_bar[stage], phase);
        fence_proxy_async_smem();   // cp.async (generic proxy) data -> wgmma (async proxy)
        const uint32_t sa = smem_u32(smem + stage * L.stage_bytes);
        const uint32_t sb = sa + (kLo ? 2u : 1u) * L.a_bytes;
        const uint64_t a_hi = make_smem_desc(sa + a_row_off, 16, 1024);
        const uint64_t b_hi = make_smem_desc(sb, 16, 1024);
        if constexpr (kLo) {
          const uint64_t a_lo = make_smem_desc(sa + L.a_bytes + a_row_off, 16, 1024);
          const uint64_t b_lo = make_smem_desc(sb + L.b_bytes, 16, 1024);
          const uint64_t ad[3] = {a_hi, a_lo, a_hi}, bd[3] = {b_lo, b_hi, b_hi};   // small products first
          wgmma_stage<kAccChunks, 0, 0>(acc, ad, bd, 3, 2u, 2u, 512u, P.BN, bf16);
        } else {
          const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_hi, b_hi, b_hi};
          wgmma_stage<kAccChunks, 0, 0>(acc, ad, bd, 1, 2u, 2u, 512u, P.BN, bf16);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);   // this warp's reads of the stage are complete
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
      const int row_base = m_tile * kTileM + warp * 32;
      const int rows_here = min(32, M - row_base);
      // store mapping after the transpose: lane = (row group rg, column quad cq); one 16-byte store per lane covers
      // 4 rows x 128 B per warp instruction
      const int rg = lane >> 3, cq = lane & 7;
#pragma unroll
      for (int c = 0; c < kAccChunks; ++c) {
        const int c0 = c * 32;
        if (c0 >= P.BN) break;
        named_bar_sync(2, kMmaWarps * 32);   // the previous chunk's readers are done with the staging tile
        acc_chunk_to_smem<kAccChunks>(acc, c, stage_buf, kStagePitch, wg, tid_wg);
        named_bar_sync(2, kMmaWarps * 32);
        if (warp >= kEpiWarps) continue;
        const int colq = n_tile * P.BN + c0 + cq * 4;  // first of this lane's 4 output channels
        float us[4] = {1.f, 1.f, 1.f, 1.f};
        if (P.wunscale != nullptr) {
          const float4 u4 = __ldg(reinterpret_cast<const float4*>(P.wunscale + n_tile * P.BN + c0 + cq * 4));
          us[0] = u4.x; us[1] = u4.y; us[2] = u4.z; us[3] = u4.w;
        }
        if (P.out_scale != nullptr) {
          const float os = __ldg(P.out_scale);
          us[0] *= os; us[1] *= os; us[2] *= os; us[3] *= os;
        }
        float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
        const bool full_quad = colq + 3 < P.N;
        if (colq < P.N) {
          // read-modify-write destinations: issue all 8 loads of this chunk before the first store (the compiler
          // must otherwise keep each load behind the previous store)
          float4 old[8];
          if (P.accumulate && full_quad) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int r = it * 4 + rg;
              old[it] = (r < rows_here)
                            ? *reinterpret_cast<const float4*>(P.dst + (size_t)(row_base + r) * P.dst_ld + P.dst_coff + colq)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int r = it * 4 + rg;
            if (r < rows_here) {
              const float* sp = my_stage + r * kStagePitch + cq * 4;
              float4 val = make_float4(sp[0] * us[0], sp[1] * us[1], sp[2] * us[2], sp[3] * us[3]);
              float* d = P.dst + (size_t)(row_base + r) * P.dst_ld + P.dst_coff + colq;
              if (full_quad) {
                if (P.accumulate) {
                  val.x += old[it].x; val.y += old[it].y; val.z += old[it].z; val.w += old[it].w;
                }
                *reinterpret_cast<float4*>(d) = val;
              } else {
                const float vv[4] = {val.x, val.y, val.z, val.w};
                for (int k = 0; k < 4; ++k)
                  if (colq + k < P.N) d[k] = P.accumulate ? d[k] + vv[k] : vv[k];
              }
              s1[0] += val.x; s1[1] += val.y; s1[2] += val.z; s1[3] += val.w;
              s2[0] = fmaf(val.x, val.x, s2[0]); s2[1] = fmaf(val.y, val.y, s2[1]);
              s2[2] = fmaf(val.z, val.z, s2[2]); s2[3] = fmaf(val.w, val.w, s2[3]);
            }
          }
        }
        if (P.stats_sum != nullptr) {
          // column sums over the warp's 32 rows: combine the 4 row groups, then one owner lane per column quad
          // accumulates into this warp's private fp32 table (no atomics; flushed in fp64 at the end)
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            s1[k] += __shfl_xor_sync(0xffffffffu, s1[k], 8);
            s1[k] += __shfl_xor_sync(0xffffffffu, s1[k], 16);
            s2[k] += __shfl_xor_sync(0xffffffffu, s2[k], 8);
            s2[k] += __shfl_xor_sync(0xffffffffu, s2[k], 16);
          }
          if (rg == 0 && colq < P.N) {
            float* ws = wstats + (size_t)warp * 2 * stat_cols;
            const int tc = stats_per_tile ? c0 + cq * 4 : colq;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              ws[tc + k] += s1[k];
              ws[stat_cols + tc + k] += s2[k];
            }
          }
        }
        __syncwarp();
      }
      if (warp < kEpiWarps && stats_per_tile && P.stats_sum != nullptr) {
        named_bar_sync(1, kEpiWarps * 32);
        for (int c = threadIdx.x; c < P.BN; c += kEpiWarps * 32) {
          double a = 0.0, b = 0.0;
#pragma unroll
          for (int w = 0; w < kEpiWarps; ++w) {
            float* ws = wstats + (size_t)w * 2 * stat_cols;
            a += (double)ws[c];
            b += (double)ws[stat_cols + c];
            ws[c] = 0.f;
            ws[stat_cols + c] = 0.f;
          }
          if (n_tile * P.BN + c < P.N) {
            atomicAdd(&P.stats_sum[n_tile * P.BN + c], a);
            atomicAdd(&P.stats_sq[n_tile * P.BN + c], b);
          }
        }
        named_bar_sync(1, kEpiWarps * 32);
      }
    }
    if (warp < kEpiWarps && P.stats_sum != nullptr && !stats_per_tile) {
      named_bar_sync(1, kEpiWarps * 32);
      for (int c = threadIdx.x; c < P.N; c += kEpiWarps * 32) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int w = 0; w < kEpiWarps; ++w) {
          a += (double)wstats[(size_t)w * 2 * stat_cols + c];
          b += (double)wstats[(size_t)w * 2 * stat_cols + stat_cols + c];
        }
        atomicAdd(&P.stats_sum[c], a);
        atomicAdd(&P.stats_sq[c], b);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// weight-gradient kernel: D[cout (128 rows, 64 per warpgroup), kcol (<=128)] = sum over pixels dY[px, cout] * A[px, kcol]
// both operands are MN-major (the 64-element swizzle rows run along cout / kcol, pixels are K).
// ------------------------------------------------------------------------------------------------
static constexpr int kWgPx = 64;  // pixels per pipeline stage

struct WgradSmemLayout {
  uint32_t dy_bytes;   // per copy: 2 blocks of [64 px][128 B]
  uint32_t a_bytes;    // per copy: nblk blocks
  uint32_t stage_bytes;
  uint32_t stages;
  uint32_t off_bars;
  uint32_t total;
};
__host__ __device__ inline WgradSmemLayout wgrad_smem_layout(int BNk, int npass) {
  WgradSmemLayout L;
  const uint32_t copies = npass > 1 ? 2u : 1u;
  L.dy_bytes = 2u * kWgPx * 128u;
  L.a_bytes = (uint32_t)(BNk / 64) * kWgPx * 128u;
  L.stage_bytes = copies * (L.dy_bytes + L.a_bytes);
  uint32_t st = (227u * 1024u - 2048u) / L.stage_bytes;
  if (st > (uint32_t)kMaxStages) st = kMaxStages;
  L.stages = st;
  L.off_bars = L.stages * L.stage_bytes;
  L.total = L.off_bars + 256u + 1024u;
  return L;
}

__host__ __device__ inline int wgrad_bnk(int Kreal) {
  // width of one K-column tile: multiple of 64, at most kMaxBN, balanced over the tiles
  int kt = (Kreal + kMaxBN - 1) / kMaxBN;
  int w = (Kreal + kt - 1) / kt;
  return ((w + 63) / 64) * 64;
}

template <int kNPass>
__global__ void __launch_bounds__(kWgradThreads, 1) conv_wgrad_kernel(const coclr_wgrad_t P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr bool kLo = kNPass > 1;
  const int M = P.B * P.Td * P.Hd * P.Wd;
  const int taps = P.g.kt * P.g.kh * P.g.kw;
  const int Kreal = taps * P.src.C;
  const int BNk = wgrad_bnk(Kreal);
  const int k_tiles = (Kreal + BNk - 1) / BNk;
  const int c_tiles = (P.Cout + 127) / 128;
  const WgradSmemLayout L = wgrad_smem_layout(BNk, kNPass);
  const uint32_t nstages = L.stages;
  // Cout <= 64 in split-precision mode: the hi and the lo plane of dY are the two 64-row halves of the M = 128 tile
  // ([dY_hi; dY_lo] x A_hi, then x A_lo: 2 instructions per K step instead of 3 on a half-empty tile, and the lo x lo
  // term comes for free); rows 64..127 hold the dY_lo products of channels 0..63 and are added by the epilogue
  const bool stack_m = kLo && P.Cout <= 64;

  // work item: (split, c_tile, k_tile)
  int w = blockIdx.x;
  const int k_tile = w % k_tiles;
  w /= k_tiles;
  const int c_tile = w % c_tiles;
  const int split = w / c_tiles;
  const int chunks_total = (M + kWgPx - 1) / kWgPx;
  const int chunks_per = (chunks_total + P.splits - 1) / P.splits;
  const int ch_begin = split * chunks_per;
  const int ch_end = min(chunks_total, ch_begin + chunks_per);
  const int nch = max(0, ch_end - ch_begin);

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L.off_bars);  // [kMaxStages]
  uint64_t* empty_bar = full_bar + kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&full_bar[s], kProducerWarps * 32);
      mbar_init(&empty_bar[s], kMmaWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= kMmaWarps) {
    const int pt = threadIdx.x - kMmaWarps * 32;
    const int ck = pt & 7;
    const int r0 = pt >> 3;  // rows r0 + 32*i, i < 2
    const uint32_t smem_base = smem_u32(smem);
    uint32_t stage = 0, phase = 0;
    coclr_geom_t ident;
    ident.kt = ident.kh = ident.kw = 1;
    ident.st = ident.sh = ident.sw = 1;
    ident.pt = ident.ph = ident.pw = 0;
    ident.transposed = 0;
    // the K granules this thread copies are the same for every pixel chunk: decompose them once
    TapPos tp_dy[2], tp_a[kMaxBN / 64];
#pragma unroll
    for (int blk = 0; blk < 2; ++blk) tp_dy[blk] = tap_of(P.dy, ident, c_tile * 128 + blk * 64 + ck * 8);
#pragma unroll
    for (int blk = 0; blk < kMaxBN / 64; ++blk) tp_a[blk] = tap_of(P.src, P.g, k_tile * BNk + blk * 64 + ck * 8);
    for (int ch = ch_begin; ch < ch_begin + nch; ++ch) {
      int rb[2], rt[2], ry[2], rx[2];    // source-space bases for the activation gather
      int qb[2], qt[2], qy[2], qx[2];    // plain destination coordinates for dY
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int m = ch * kWgPx + r0 + 32 * i;
        row_coords(ident, P.Td, P.Hd, P.Wd, M, m, qb[i], qt[i], qy[i], qx[i]);
        rb[i] = qb[i];
        rt[i] = qt[i] * P.g.st - P.g.pt;
        ry[i] = qy[i] * P.g.sh - P.g.ph;
        rx[i] = qx[i] * P.g.sw - P.g.pw;
      }
      mbar_wait(&empty_bar[stage], phase ^ 1u);
      const uint32_t s_dy = smem_base + stage * L.stage_bytes;
      const uint32_t s_a = s_dy + (kLo ? 2u : 1u) * L.dy_bytes;
      // dY: 2 blocks of 64 output channels (stacked mode: block 0 = hi plane, block 1 = lo plane of channels 0..63)
      if (stack_m) {
        gather_block_async<kLo, 2>(P.dy, ident, P.dy.C, tp_dy[0], ck, r0, qb, qt, qy, qx, s_dy, s_dy + kWgPx * 128);
      } else {
#pragma unroll
        for (int blk = 0; blk < 2; ++blk) {
          gather_block_async<kLo, 2>(P.dy, ident, P.dy.C, tp_dy[blk], ck, r0, qb, qt, qy, qx,
                                     s_dy + blk * (kWgPx * 128), s_dy + L.dy_bytes + blk * (kWgPx * 128));
        }
      }
#pragma unroll
      for (int blk = 0; blk < kMaxBN / 64; ++blk) {
        if (blk < BNk / 64)
          gather_block_async<kLo, 2>(P.src, P.g, Kreal, tp_a[blk], ck, r0, rb, rt, ry, rx,
                                     s_a + blk * (kWgPx * 128), s_a + L.a_bytes + blk * (kWgPx * 128));
      }
      cp_async_mbar_arrive_noinc(&full_bar[stage]);
      if (++stage == nstages) { stage = 0; phase ^= 1u; }
    }
  } else {
    // ===================== MMA: warpgroup wg owns cout rows [64 wg, 64 wg + 64) of the tile =====================
    const int wg = warp >> 2;
    const bool bf16 = P.dy_bf16 != 0;
    float acc[16 * kAccChunks];
#pragma unroll
    for (int i = 0; i < 16 * kAccChunks; ++i) acc[i] = 0.f;
    uint32_t stage = 0, phase = 0;
    for (int ch = 0; ch < nch; ++ch) {
      mbar_wait_spin(&full_bar[stage], phase);
      fence_proxy_async_smem();   // cp.async (generic proxy) data -> wgmma (async proxy)
      const uint32_t s_dy = smem_u32(smem + stage * L.stage_bytes) + (uint32_t)wg * (kWgPx * 128);
      const uint32_t s_a = smem_u32(smem + stage * L.stage_bytes) + (kLo ? 2u : 1u) * L.dy_bytes;
      // MN-major: LBO = stride between 64-element MN blocks (64 px * 128 B), SBO = 8-pixel group stride
      const uint64_t a_hi = make_smem_desc(s_dy, kWgPx * 128, 1024);
      const uint64_t b_hi = make_smem_desc(s_a, kWgPx * 128, 1024);
      const uint32_t b_step = (kWgPx * 128) >> 4;
      // one K=16 step = 16 pixels = 2 swizzle atoms = 2048 B -> +128 in descriptor units
      if constexpr (kLo) {
        const uint64_t a_lo = make_smem_desc(s_dy + L.dy_bytes, kWgPx * 128, 1024);
        const uint64_t b_lo = make_smem_desc(s_a + L.a_bytes, kWgPx * 128, 1024);
        const uint64_t ad[3] = {a_hi, stack_m ? a_hi : a_lo, a_hi}, bd[3] = {b_lo, b_hi, b_hi};
        wgmma_stage<kAccChunks, 1, 1>(acc, ad, bd, stack_m ? 2 : 3, 128u, 128u, b_step, BNk, bf16);
      } else {
        const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_hi, b_hi, b_hi};
        wgmma_stage<kAccChunks, 1, 1>(acc, ad, bd, 1, 128u, 128u, b_step, BNk, bf16);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == nstages) { stage = 0; phase ^= 1u; }
    }
    const int tw = threadIdx.x & 127;
    if (stack_m) {
      // dY_lo rows (warpgroup 1) join the dY_hi rows via smem
      float* xs = reinterpret_cast<float*>(smem);
      named_bar_sync(1, kMmaWarps * 32);   // MMAs done
      if (wg == 1) {
#pragma unroll
        for (int i = 0; i < 16 * kAccChunks; ++i) xs[i * 128 + tw] = acc[i];
      }
      named_bar_sync(1, kMmaWarps * 32);
      if (wg == 0) {
#pragma unroll
        for (int i = 0; i < 16 * kAccChunks; ++i) acc[i] += xs[i * 128 + tw];
      }
    }
    if (nch > 0 && !(stack_m && wg == 1)) {
      // fp32 atomics into dW[cout, cin, tap], one per element when splits == 1
      const int row0 = 64 * wg + 16 * (tw >> 5) + ((tw & 31) >> 2);
      const int col0 = 2 * (tw & 3);
      const float os = P.out_scale != nullptr ? __ldg(P.out_scale) : 1.f;
#pragma unroll
      for (int c = 0; c < kAccChunks; ++c) {
        if (c * 32 >= BNk) break;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
          const int n = c_tile * 128 + row0 + 8 * ((r >> 1) & 1);   // output channel
          const int k = k_tile * BNk + c * 32 + col0 + 8 * (r >> 2) + (r & 1);
          if (n < P.Cout && k < Kreal) {
            const int tap = k / P.src.C;
            const int ci = k - tap * P.src.C;
            if (ci < P.Cin_real) atomicAdd(P.dw + ((size_t)n * P.Cin_real + ci) * taps + tap, acc[16 * c + r] * os);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// weight packer: one CTA per packed row
// ------------------------------------------------------------------------------------------------
template <bool kBf16>
COCLR_DEVINL void pack_row(const coclr_pack_t& P, int N, int BN, int Kreal, int nkc, int row, float* red) {
  const int n_tile = row / BN;
  const int rin = row - n_tile * BN;
  const int n = n_tile * BN + rin;  // tiles are contiguous in n
  const int Kpad = nkc * kChunkK;
  auto wval = [&](int k) -> float {
    if (n >= N || k >= Kreal) return 0.f;
    const int tap = k / P.Cpad;
    const int c = k - tap * P.Cpad;
    if (P.mode == 0) {
      if (c >= P.Cin) return 0.f;
      return P.w[((size_t)n * P.Cin + c) * P.taps + tap];
    } else {
      if (c >= P.Cout) return 0.f;
      return P.w[((size_t)c * P.Cin + n) * P.taps + tap];
    }
  };
  float mx = 0.f;
  for (int k = threadIdx.x; k < Kreal; k += blockDim.x) mx = fmaxf(mx, fabsf(wval(k)));
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    float m2 = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
    if (threadIdx.x == 0) red[0] = m2;
  }
  __syncthreads();
  mx = red[0];
  float scale = 1.f, unscale = 1.f;
  if (mx > 0.f && isfinite(mx)) {
    int e;
    frexpf(mx, &e);  // mx = f * 2^e, f in [0.5, 1)
    e = max(-100, min(100, e));
    scale = ldexpf(1.f, -e);
    unscale = ldexpf(1.f, e);
  }
  if (threadIdx.x == 0) P.unscale[row] = unscale;
  uint8_t* base = reinterpret_cast<uint8_t*>(P.wpk);
  for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
    const float v = wval(k) * scale;
    uint16_t hi, lo;
    split2<kBf16>(v, hi, lo);
    const int kc = k / kChunkK;
    const int kk = k - kc * kChunkK;
    const size_t img = ((size_t)n_tile * nkc + kc) * 2;
    const uint32_t off = swz128_offset((uint32_t)rin, (uint32_t)(kk >> 3)) + (uint32_t)(kk & 7) * 2u;
    *reinterpret_cast<uint16_t*>(base + (img + 0) * (size_t)BN * 128 + off) = hi;
    *reinterpret_cast<uint16_t*>(base + (img + 1) * (size_t)BN * 128 + off) = lo;
  }
}

template <bool kBf16>
__global__ void pack_weights_kernel(const coclr_pack_t P, int N, int BN, int n_tiles, int Kreal, int nkc) {
  __shared__ float red[32];
  pack_row<kBf16>(P, N, BN, Kreal, nkc, blockIdx.x, red);
}

__host__ __device__ inline void tile_plan_hd(int N, int* BN, int* n_tiles) {
  int nt = (N + kMaxBN - 1) / kMaxBN;
  int w = (N + nt - 1) / nt;
  *BN = ((w + 31) / 32) * 32;
  *n_tiles = nt;
}

// All weights of an encoder in ONE launch: CTA r packs global row r; row_start[i] = first row of table entry i
// (ascending, row_start[n] = total rows).  Replaces ~100 launches per encoder pass.
__global__ void pack_weights_batch_kernel(const coclr_pack_t* __restrict__ table, const int* __restrict__ row_start,
                                          int n) {
  __shared__ float red[32];
  __shared__ coclr_pack_t P;
  __shared__ int s_first;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n - 1;              // last entry whose first row is <= blockIdx.x
    const int r = (int)blockIdx.x;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (row_start[mid] <= r) lo = mid; else hi = mid - 1;
    }
    P = table[lo];
    s_first = row_start[lo];
  }
  __syncthreads();
  const int N = P.mode == 0 ? P.Cout : P.Cin;
  const int Kreal = P.taps * P.Cpad;
  int BN, nt;
  tile_plan_hd(N, &BN, &nt);
  const int nkc = (Kreal + kChunkK - 1) / kChunkK;
  const int row = (int)blockIdx.x - s_first;
  if (P.bf16) pack_row<true>(P, N, BN, Kreal, nkc, row, red);
  else pack_row<false>(P, N, BN, Kreal, nkc, row, red);
}

static inline void tile_plan(int N, int* BN, int* n_tiles) { tile_plan_hd(N, BN, n_tiles); }

}  // namespace coclr

using namespace coclr;

extern "C" size_t coclr_conv_packed_bytes(int N, int Kreal, int* BN_out, int* n_tiles_out) {
  int BN, nt;
  tile_plan(N, &BN, &nt);
  if (BN_out) *BN_out = BN;
  if (n_tiles_out) *n_tiles_out = nt;
  const int nkc = (Kreal + kChunkK - 1) / kChunkK;
  return (size_t)nt * nkc * 2 * BN * 128;
}

extern "C" int coclr_pack_weights(const coclr_pack_t* p, coclr_stream_t stream) {
  if (!p || !p->w || !p->wpk || !p->unscale) return COCLR_E_ARG;
  const int N = p->mode == 0 ? p->Cout : p->Cin;
  const int Kreal = p->taps * p->Cpad;
  int BN, nt;
  tile_plan(N, &BN, &nt);
  const int nkc = (Kreal + kChunkK - 1) / kChunkK;
  cudaStream_t s = (cudaStream_t)stream;
  if (p->bf16)
    pack_weights_kernel<true><<<nt * BN, 128, 0, s>>>(*p, N, BN, nt, Kreal, nkc);
  else
    pack_weights_kernel<false><<<nt * BN, 128, 0, s>>>(*p, N, BN, nt, Kreal, nkc);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

extern "C" int coclr_pack_weights_batch(const coclr_pack_t* table_dev, const int* row_start_dev, int n, int total_rows,
                                        coclr_stream_t stream) {
  if (!table_dev || !row_start_dev || n < 1 || total_rows < 1) return COCLR_E_ARG;
  pack_weights_batch_kernel<<<total_rows, 128, 0, (cudaStream_t)stream>>>(table_dev, row_start_dev, n);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

static bool src_ok(const coclr_src_t& s, int need_lo) {
  if (!s.hi || (need_lo && !s.lo)) return false;
  if (s.T < 1 || s.H < 1 || s.W < 1) return false;
  if (s.C % 8 != 0 || s.ld % 8 != 0 || s.coff % 8 != 0) return false;  // 16-byte cp.async granules
  if (((uintptr_t)s.hi & 15) || ((uintptr_t)s.lo & 15)) return false;
  return true;
}

template <int NP>
static int launch_conv(const coclr_conv_t& P, int num_sms, cudaStream_t s) {
  const int M = P.B * P.Td * P.Hd * P.Wd;
  const int m_tiles = (M + kTileM - 1) / kTileM;
  const int total = m_tiles * P.n_tiles;
  const ConvSmemLayout L = conv_smem_layout(P.BN, P.n_tiles, NP, P.stats_sum != nullptr);
  if (L.stages < 2) return COCLR_E_ARG;
  cudaError_t e = cudaFuncSetAttribute(conv_igemm_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total);
  if (e != cudaSuccess) return COCLR_E_LAUNCH;
  const int grid = total < num_sms ? total : num_sms;
  conv_igemm_kernel<NP><<<grid, kThreads, L.total, s>>>(P);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

extern "C" int coclr_conv_igemm(const coclr_conv_t* p, int num_sms, coclr_stream_t stream) {
  if (!p || !p->wpk || !p->dst) return COCLR_E_ARG;
  if (!src_ok(p->src, p->npass > 1)) return COCLR_E_ARG;
  if (p->BN % 32 != 0 || p->BN > kMaxBN || p->BN < 32 || p->n_tiles < 1) return COCLR_E_ARG;
  if (p->a_bf16 != p->b_bf16) return COCLR_E_ARG;   // wgmma takes one 16-bit format for both operands
  if (p->dst_ld % 4 != 0 || p->dst_coff % 4 != 0 || ((uintptr_t)p->dst & 15)) return COCLR_E_ARG;  // 16-byte stores
  if (p->Kreal != p->g.kt * p->g.kh * p->g.kw * p->src.C) return COCLR_E_ARG;
  if ((p->g.st != 1 && p->g.st != 2) || (p->g.sh != 1 && p->g.sh != 2) || (p->g.sw != 1 && p->g.sw != 2))
    return COCLR_E_ARG;
  if (num_sms <= 0) return COCLR_E_ARG;
  if ((long long)p->B * p->src.T * p->src.H * p->src.W >= (1ll << 31)) return COCLR_E_ARG;  // 32-bit pixel indices
  cudaStream_t s = (cudaStream_t)stream;
  // TMA-staged kernel first (conv_tma.cu); shapes it does not cover run on the cp.async gather kernel below
  const int rc = coclr::conv_tma_try(*p, num_sms, s);
  if (rc <= 0) return rc;
  return p->npass > 1 ? launch_conv<3>(*p, num_sms, s) : launch_conv<1>(*p, num_sms, s);
}

template <int NP>
static int launch_wgrad(const coclr_wgrad_t& P, cudaStream_t s) {
  const int taps = P.g.kt * P.g.kh * P.g.kw;
  const int Kreal = taps * P.src.C;
  const int BNk = wgrad_bnk(Kreal);
  const int k_tiles = (Kreal + BNk - 1) / BNk;
  const int c_tiles = (P.Cout + 127) / 128;
  const WgradSmemLayout L = wgrad_smem_layout(BNk, NP);
  if (L.stages < 2) return COCLR_E_ARG;
  cudaError_t e = cudaFuncSetAttribute(conv_wgrad_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total);
  if (e != cudaSuccess) return COCLR_E_LAUNCH;
  const int grid = k_tiles * c_tiles * P.splits;
  conv_wgrad_kernel<NP><<<grid, kWgradThreads, L.total, s>>>(P);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

extern "C" int coclr_conv_wgrad(const coclr_wgrad_t* p, coclr_stream_t stream) {
  if (!p || !p->dw) return COCLR_E_ARG;
  if (!src_ok(p->src, p->npass > 1) || !src_ok(p->dy, p->npass > 1)) return COCLR_E_ARG;
  if (p->splits < 1 || p->g.transposed) return COCLR_E_ARG;
  if (p->dy_bf16 != p->src_bf16) return COCLR_E_ARG;   // wgmma takes one 16-bit format for both operands
  if ((long long)p->B * p->src.T * p->src.H * p->src.W >= (1ll << 31) ||
      (long long)p->B * p->dy.T * p->dy.H * p->dy.W >= (1ll << 31))
    return COCLR_E_ARG;  // 32-bit pixel indices
  cudaStream_t s = (cudaStream_t)stream;
  // TMA-staged kernel first (wgrad_tma.cu: stride-1 "same" convolutions); everything else on the gather kernel
  const int rc = coclr::wgrad_tma_try(*p, s);
  if (rc <= 0) return rc;
  return p->npass > 1 ? launch_wgrad<3>(*p, s) : launch_wgrad<1>(*p, s);
}
