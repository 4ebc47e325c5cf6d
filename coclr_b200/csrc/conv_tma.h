// Tile plan of the TMA-staged convolution kernel (conv_tma.cu), shared between the host planner and the kernel; the
// stage driver and the epilogue that both convolution kernels (conv_tma.cu, conv_igemm.cu) run on their register
// accumulators; and the instance dispatch of every wgmma kernel's launcher.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "coclr_b200.h"
#include "common.cuh"

namespace coclr {

// Output side of a convolution tile plan: the 128 rows of a tile in box order (dim 0 fastest) and the coordinates of
// each epilogue block's 32-row sub-box in the output tensor map.
struct ConvOut {
  int obox[4];         // tile extent per dim (rows are in this box order)
  int o_mul[4];        // tile index -> output-map coordinate
  int oext[4];         // output extent per dim (edge rows are excluded from the statistics)
  int sub[4][4];       // output coordinate offsets of each epilogue block's 32-row sub-box
  int n_tiles_n, BN, N;
  int stage_bufs;      // staging buffers per epilogue block: 1 or 2 of kConvStageBytes
};

static constexpr uint32_t kConvStageBytes = 4096;  // 32 rows x 32 fp32 columns per staging block and buffer
static constexpr uint32_t kConvEpiBarEnd = 5;      // named barriers 1-4: the warp pairs of staging blocks 0-3
static constexpr int kConvEpiThreads = 256;        // two consumer warpgroups of 64 tile rows each: warps 4-11
static constexpr int kConvFirstEpiWarp = 4;

// Epilogue of the two consumer warpgroups (warps 4-11) of a convolution kernel (consumer warp cwarp = warp - 4 = 0..7, warpgroup cwarp / 4 holds
// tile rows 64 (cwarp / 4) .. + 63 of the wgmma accumulator):
//  * each thread scales its accumulator fragment in registers (column factor wunscale[col] * out_scale) and writes it,
//    32 columns at a time, with st.shared.v2 into the 128B-swizzled staging block of its 32 tile rows.  Staging block
//    blk belongs to warps 2 blk and 2 blk + 1 (the same warpgroup), which meet at their own named barrier and take
//    alternate chunks for the rest, so neither warpgroup waits for the other between tiles;
//  * a chunk's warp writes it with ONE cp.async.bulk.tensor store (or add-reduction, for gradient accumulation) per 32
//    rows x 32 channels: edge clipping and channel slices of wider buffers are properties of the output tensor map;
//  * and accumulates the BatchNorm statistics of its valid rows in ascending row order.  Per column it sums d = x - x0
//    and d^2 in fp32, where x0 is the first value of the column this warp sees, and converts exactly in double when the
//    sums leave the CTA:  sum x = sum d + n x0,  sum x^2 = sum d^2 + 2 x0 sum d + n x0^2,  so that var = E[x^2] - mean^2
//    (formed in double by the finalize step) does not lose the variance of channels whose spread is small against their
//    mean to fp32 rounding of the raw sums (nn.BatchNorm3d is two-pass).  Launches with one N tile add the four blocks'
//    sums once per CTA; with several, each block flushes them after every tile.
//    kStatTable (the gather kernel) keeps its own summation order instead: per block and column, plain fp32 sums of the
//    four row groups r % 4 (rows in ascending order each), combined as (g0 + g1) + (g2 + g3), added into a per-block fp32
//    column table in shared memory across the CTA's tiles, and the four blocks' tables summed in double.  The table
//    covers all output channels when there are at most kStatTableMaxCols of them (flushed once per CTA), else one N tile
//    (flushed after every tile).
// The staging area at `stage` (shared-memory address) holds 4 blocks x stage_bufs x kConvStageBytes, 1024-byte aligned.
static constexpr int kStatTableMaxCols = 512;
__host__ __device__ inline int stat_table_cols(int BN, int n_tiles) {
  return n_tiles * BN <= kStatTableMaxCols ? n_tiles * BN : BN;
}

template <int kBN, bool kStatTable = false>
struct ConvEpilogue {
  static constexpr int kChunks = kBN / 32;
  float s1[kChunks], s2[kChunks], x0[kChunks];
  uint32_t x0_set = 0u;
  int nrows = 0;
  float* tab = nullptr;   // kStatTable: [4 blocks][2][stat_table_cols + 4] fp32, zeroed before the first tile

  COCLR_DEVINL ConvEpilogue() {
#pragma unroll
    for (int i = 0; i < kChunks; ++i) s1[i] = s2[i] = x0[i] = 0.f;
  }
  COCLR_DEVINL explicit ConvEpilogue(float* stat_tab) : ConvEpilogue() { tab = stat_tab; }

  // Args (the kernel's parameters) provides wunscale, out_scale, stats_sum, stats_sq and accumulate; they are read from
  // parameter space where they are used, and nothing but the statistics is held in registers through the MMA loop.
  // One tile: idx = tile index per output dim, acc = this thread's accumulator fragment.
  template <class Args>
  COCLR_DEVINL void tile(const Args& P, const ConvOut& O, const CUtensorMap* map_out, uint32_t stage,
                         const float (&acc)[kBN / 2], const int (&idx)[4], int n_tile) {
    const bool want_stats = P.stats_sum != nullptr;
    const int cwarp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0) - kConvFirstEpiWarp;
    const int lane = (int)threadIdx.x & 31;
    const int blk = cwarp >> 1;
    const uint32_t pair_bar = 1u + (uint32_t)blk;
    const uint32_t frow = 16u * (uint32_t)(cwarp & 1) + ((uint32_t)lane >> 2);   // this thread's first row in the block
    const uint32_t my_stage = stage + (uint32_t)blk * (uint32_t)O.stage_bufs * kConvStageBytes;
    // the bulk-tensor stores of a warp are issued, committed and waited for by ONE thread (bulk async-groups are
    // per-thread state); elect.sync is deterministic for a given member mask, so every call elects the same lane
    const bool leader = elect_one();
    const float oscale = P.out_scale != nullptr ? __ldg(P.out_scale) : 1.f;
    // Chunks go through the block's staging buffers in rounds: with two buffers a round holds two chunks, one per
    // buffer, else one.  Both warps of the pair write every chunk of the round; then chunk c is stored and summed by
    // warp 2 blk + (c & 1), so the two warps take the statistics of a round's two chunks at the same time.
    bool valid = true;
    int oc[4];
    int r = blk * 32 + lane;   // row r of the tile: box-relative position (rows are in box order, dim 1 fastest)
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int ri = d < 3 ? r % O.obox[d] : r;
      if (d < 3) r /= O.obox[d];
      const int o = idx[d] * O.o_mul[d];
      valid = valid && (o + ri < O.oext[d]);
      oc[d] = o + O.sub[blk][d];
    }
    const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int kq = 0; kq < kChunks; ++kq) {
      const int col0 = n_tile * kBN + kq * 32;
      if (col0 < O.N) {
        const uint32_t h = O.stage_bufs == 2 ? (uint32_t)kq & 1u : 0u;   // this chunk's buffer
        if (h == 0u) {
          // a round starts: the stores of the last round have read both buffers (each warp waits for its own) and
          // both warps are done with its statistics
          if (leader) bulk_wait_group_read<0>();
          named_bar_sync(pair_bar, 64);
        }
        const uint32_t buf = my_stage + h * kConvStageBytes;
        // this thread's part of the chunk, scaled by the column's weight unscale and the output scale:
        // acc[16 kq + 4 g + 2 h + e] = row frow + 8 h, column 8 g + 2 (lane % 4) + e
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const uint32_t cl = 8u * (uint32_t)g + 2u * ((uint32_t)lane & 3u);
          float f0 = oscale, f1 = oscale;
          if (P.wunscale != nullptr) {
            f0 = __ldg(P.wunscale + col0 + cl) * oscale;
            f1 = __ldg(P.wunscale + col0 + cl + 1) * oscale;
          }
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const uint32_t row = frow + 8u * (uint32_t)hr;
            st_shared_v2(buf + row * 128u + ((((cl >> 2) ^ row) & 7u) << 4) + ((cl & 3u) << 2),
                         acc[16 * kq + 4 * g + 2 * hr] * f0, acc[16 * kq + 4 * g + 2 * hr + 1] * f1);
          }
        }
        const bool round_end = h == 1u || O.stage_bufs == 1 || kq + 1 == kChunks || col0 + 32 >= O.N;
        if (!round_end) continue;
        fence_proxy_async_smem();
        named_bar_sync(pair_bar, 64);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          // the round's chunks: kq, and kq - 1 when kq went into the second buffer; chunk c belongs to warp c & 1
          if (!(c == kq || (c == kq - 1 && h == 1u)) || (c & 1) != (cwarp & 1)) continue;
          const uint32_t cbuf = my_stage + (O.stage_bufs == 2 ? (uint32_t)c & 1u : 0u) * kConvStageBytes;
          const int ccol0 = n_tile * kBN + c * 32;
          if (leader) {
            if (P.accumulate) tma_reduce_add_5d(map_out, cbuf, ccol0, oc[0], oc[1], oc[2], oc[3]);
            else tma_store_5d(map_out, cbuf, ccol0, oc[0], oc[1], oc[2], oc[3]);
            bulk_commit_group();
          }
          if constexpr (kStatTable) {
            const int col = ccol0 + lane;
            if (want_stats && col < O.N) {
              // lane j sums column j of the block's valid rows r, row group r % 4 by row group
              const uint32_t cchunk = (uint32_t)lane >> 2, cword = ((uint32_t)lane & 3u) << 2;
              float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
              for (uint32_t r = 0; r < 32; ++r) {
                if ((vmask >> r) & 1u) {
                  const float v = ld_shared_f32(cbuf + r * 128u + ((cchunk ^ (r & 7u)) << 4) + cword);
                  a[r & 3u] += v;
                  b[r & 3u] = fmaf(v, v, b[r & 3u]);
                }
              }
              const int stat_cols = stat_table_cols(kBN, O.n_tiles_n) + 4;
              float* ws = tab + (size_t)blk * 2 * stat_cols;
              const int tc = O.n_tiles_n * kBN > kStatTableMaxCols ? c * 32 + lane : col;
              ws[tc] += (a[0] + a[1]) + (a[2] + a[3]);
              ws[stat_cols + tc] += (b[0] + b[1]) + (b[2] + b[3]);
            }
          } else if (want_stats && vmask != 0u) {
            // lane j sums column j over the block's valid rows, reading the swizzled block back (conflict-free)
            float a = 0.f, b = 0.f;
            const uint32_t cchunk = (uint32_t)lane >> 2, cword = ((uint32_t)lane & 3u) << 2;
            if (!((x0_set >> c) & 1u)) {
              const uint32_t r0 = (uint32_t)__ffs((int)vmask) - 1u;
              x0[c] = ld_shared_f32(cbuf + r0 * 128u + ((cchunk ^ (r0 & 7u)) << 4) + cword);
              x0_set |= 1u << c;
            }
            const float xs = x0[c];
#pragma unroll 8
            for (uint32_t r = 0; r < 32; ++r) {
              if ((vmask >> r) & 1u) {
                const float d = ld_shared_f32(cbuf + r * 128u + ((cchunk ^ (r & 7u)) << 4) + cword) - xs;
                a += d;
                b = fmaf(d, d, b);
              }
            }
            s1[c] += a;
            s2[c] += b;
          }
        }
      }
    }
    if constexpr (kStatTable) {
      if (want_stats && O.n_tiles_n * kBN > kStatTableMaxCols) {
        // wide layers: the four blocks' sums of this N tile leave the CTA now
        const int ct = (int)threadIdx.x - kConvFirstEpiWarp * 32;
        const int stat_cols = kBN + 4;
        named_bar_sync(kConvEpiBarEnd, kConvEpiThreads);
        for (int c = ct; c < kBN; c += kConvEpiThreads) {
          double a = 0.0, b = 0.0;
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            float* ws = tab + (size_t)w * 2 * stat_cols;
            a += (double)ws[c];
            b += (double)ws[stat_cols + c];
            ws[c] = 0.f;
            ws[stat_cols + c] = 0.f;
          }
          if (n_tile * kBN + c < O.N) {
            atomicAdd(&P.stats_sum[n_tile * kBN + c], a);
            atomicAdd(&P.stats_sq[n_tile * kBN + c], b);
          }
        }
        named_bar_sync(kConvEpiBarEnd, kConvEpiThreads);
      }
      return;
    }
    nrows += __popc(vmask);
    if (want_stats && O.n_tiles_n > 1) {
#pragma unroll
      for (int kq = 0; kq < kChunks; ++kq) {
        const int col = n_tile * kBN + kq * 32 + lane;
        if ((kq & 1) == (cwarp & 1) && col < O.N) {
          const double n = (double)nrows, xd = (double)x0[kq];
          atomicAdd(&P.stats_sum[col], (double)s1[kq] + n * xd);
          atomicAdd(&P.stats_sq[col], (double)s2[kq] + xd * (2.0 * (double)s1[kq] + n * xd));
        }
        s1[kq] = s2[kq] = 0.f;
      }
      x0_set = 0u;
      nrows = 0;
    }
  }

  // After the last tile: every consumer thread calls this once.
  template <class Args>
  COCLR_DEVINL void finish(const Args& P, const ConvOut& O, uint8_t* stage) {
    const int ct = (int)threadIdx.x - kConvFirstEpiWarp * 32;   // thread index among the consumers
    const int cwarp = ct >> 5, lane = ct & 31, blk = cwarp >> 1;
    const bool leader = elect_one();
    if (leader) bulk_wait_group_read<0>();
    if constexpr (kStatTable) {
      if (P.stats_sum != nullptr && O.n_tiles_n * kBN <= kStatTableMaxCols) {
        const int stat_cols = O.n_tiles_n * kBN + 4;
        named_bar_sync(kConvEpiBarEnd, kConvEpiThreads);
        for (int c = ct; c < O.N; c += kConvEpiThreads) {
          double a = 0.0, b = 0.0;
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            a += (double)tab[(size_t)w * 2 * stat_cols + c];
            b += (double)tab[(size_t)w * 2 * stat_cols + stat_cols + c];
          }
          atomicAdd(&P.stats_sum[c], a);
          atomicAdd(&P.stats_sq[c], b);
        }
      }
    } else if (P.stats_sum != nullptr && O.n_tiles_n == 1) {
      // combine the four blocks' column sums in shared memory (the staging blocks are free now), one fp64 atomic per
      // channel and CTA
      double* tab = reinterpret_cast<double*>(stage);   // [4 blocks][2][128] = 8 KB of the staging blocks
      named_bar_sync(kConvEpiBarEnd, kConvEpiThreads);
#pragma unroll
      for (int kq = 0; kq < kChunks; ++kq) {
        if ((kq & 1) != (cwarp & 1)) continue;
        const double n = (double)nrows, xd = (double)x0[kq];
        tab[(blk * 2 + 0) * 128 + kq * 32 + lane] = (double)s1[kq] + n * xd;
        tab[(blk * 2 + 1) * 128 + kq * 32 + lane] = (double)s2[kq] + xd * (2.0 * (double)s1[kq] + n * xd);
      }
      named_bar_sync(kConvEpiBarEnd, kConvEpiThreads);
      for (int c = ct; c < O.N; c += kConvEpiThreads) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          a += tab[(w * 2 + 0) * 128 + c];
          b += tab[(w * 2 + 1) * 128 + c];
        }
        atomicAdd(&P.stats_sum[c], a);
        atomicAdd(&P.stats_sq[c], b);
      }
    }
    if (leader) bulk_wait_group<0>();   // all global writes of this thread's bulk stores are complete
  }
};

// The K loop of a convolution tile on two fresh register blocks: stage s + 1 is issued into the other block before
// stage s is waited for and retired, so one stage is always in flight.  issue(t, rel) waits for the next stage's
// operands, issues it into t and records in rel the slots to release once it has completed; it returns false after the
// tile's last stage.  retire(t, rel) adds the completed block t into the accumulator and releases rel's slots.
template <int kBN, class Rel, class Issue, class Retire>
COCLR_DEVINL void run_stages(Issue&& issue, Retire&& retire) {
  float t0[kBN / 2], t1[kBN / 2];
  Rel rel0, rel1;
  if (!issue(t0, rel0)) return;
  while (true) {
    if (!issue(t1, rel1)) {
      wgmma_wait<0>();
      retire(t0, rel0);
      return;
    }
    wgmma_wait<1>();
    retire(t0, rel0);
    if (!issue(t0, rel0)) {
      wgmma_wait<0>();
      retire(t1, rel1);
      return;
    }
    wgmma_wait<1>();
    retire(t1, rel1);
  }
}

// Kernel instances are picked from run-time values, one compile-time parameter at a time:
// with_int<V...>(v, f) calls f(std::integral_constant<int, V>()) for the V that equals v, and returns false when none
// does.
template <int... Vs, class F>
inline bool with_int(int v, F&& f) {
  return ((v == Vs && (f(std::integral_constant<int, Vs>()), true)) || ...);
}

// Launches kernel with `smem` bytes of dynamic shared memory; COCLR_E_LAUNCH when that much cannot be granted.
template <class... Params, class... Args>
inline int launch_with_smem(void (*kernel)(Params...), int grid, int threads, uint32_t smem, cudaStream_t stream,
                            const Args&... args) {
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return COCLR_E_LAUNCH;
  kernel<<<grid, threads, smem, stream>>>(args...);
  return COCLR_OK;
}

// One TMA slab load of the activation planes: its origin relative to the tile origin (logical dims 1..4 of the tensor
// map), and the taps of the reuse dimension it serves.  Shift j reads the slab j rows of that dimension further on and
// belongs to tap[j] (kt-major, as in the weight tensor): the convolution multiplies it with packed K chunk
// tap[j] * nc + channel_chunk, the weight gradient makes it N block j.
struct TmaSlabType {
  int d[4];
  int nshift;
  int tap[8];
};

struct TmaPlan {
  ConvOut out;
  int ntiles[4];       // tiles per logical dim (dim 0 fastest)
  int a_mul[4];        // tile index -> A-map coordinate
  int m_tiles, total_tiles;
  int nc;              // 64-channel K chunks per tap
  int nkc;             // K chunks of the packed weight image (taps * nc)
  int n_types;         // slab types per channel chunk
  int sel_dim;         // >= 0: the tile index in this dim selects the ONE slab type of the tile
  int a_c0_step;       // channel coordinate step per chunk
  TmaSlabType type[4];
  int slab_bytes;      // one plane of a slab
  int plane_stride;    // slab_bytes rounded up to the 1024-byte swizzle atom
  int shift_bytes;
  int a_slots, a_slot_bytes;
  int b_slots, b_tile_bytes, b_resident;
  uint32_t off_b, off_stage, off_bars, total;
};

struct TmaArgs {
  TmaPlan plan;
  const void* wpk;
  const float* wunscale;
  const float* out_scale;
  double* stats_sum;
  double* stats_sq;
  int accumulate;
  int a_bf16, b_bf16;
};

int conv_tma_try(const coclr_conv_t& P, int num_sms, cudaStream_t stream);

// host-side description of a tiled tensor map (up to 5 dims; dim 0 = channels, unit stride) over one or two planes
struct MapSpec {
  void* base[2];
  uint64_t dims[5];
  uint64_t strides[4];   // bytes, dims 1..4
  uint32_t box[5];
  int elem_bytes;
};
// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda); plane `which`; false when unavailable
bool encode_map(CUtensorMap* m, const MapSpec& s, int which, int rank = 5, bool swizzle = true);
// The hi map, and the lo map when there are several passes (else a copy of the hi map, which the kernel never reads).
bool encode_maps(CUtensorMap* hi, CUtensorMap* lo, const MapSpec& s, int npass);
// A dense channels-last plane at base(s) + coff elements, pixels ld elements apart, as a 5-D tensor map: dim 0 the c
// channels, dims 1..4 the logical extents ext (dim 1 fastest, each dim's stride the previous one's times its extent).
// pitch > 0: dim 2 advances pitch pixels although dim 1 holds only ext[0] of them (the window map's rows).
MapSpec plane_map(const void* hi, const void* lo, int coff, int elem_bytes, int ld, int c, const int (&ext)[4],
                  const int (&box)[5], int pitch = 0);

// How the TMA kernels see the activation planes of a launch.  A tile covers a box of destination pixels; its halo slab
// is that box extended along the kind's reuse dimension (logical dim 1 for the rows, 2 for the frames) by the taps
// that read it.
enum SlabKind {
  kSlabNone,     // not on the TMA kernels
  kSlabFlat,     // 1x1x1: the pixels as one flat dimension [C, M, 1, 1, 1], one tap
  kSlabWindow,   // space-to-depth stem (1,kh,kw): [64, W, H, T, B] over 64/kw-channel pixels, see slab_kind
  kSlabRows,     // (1,kh,kw): [C, W, H, T, B]; one slab type per dx, the kh taps of dy share it
  kSlabFrames,   // (kt,1,1): [C, H*W, 1, T, B]; the kt taps of dt share one slab
  kSlabParity,   // (kt,1,1) at temporal stride 2: [C, H*W, 2, T/2, B]; one slab type per frame parity
};
// The kind of a spatially unstrided convolution of source S onto a Td x Hd x Wd grid.  Each planner adds its own limits.
SlabKind slab_kind(const coclr_geom_t& g, const coclr_src_t& S, int Td, int Hd, int Wd);
// Fills the kind's slab types (the data gradient's, g.transposed, mirrored: taps reversed, origins reflected) and
// returns how many there are, 0 when a frame parity has no taps.
int slab_types(SlabKind kind, const coclr_geom_t& g, TmaSlabType (&type)[4]);
// The source planes of a kind as one tensor map over B clips onto a destination Wd pixels wide, loaded 64 channels x
// the slab of a tile box whose types serve up to `reuse` taps each.
MapSpec slab_map(SlabKind kind, const coclr_geom_t& g, const coclr_src_t& S, int B, int Wd, const int (&tile)[4],
                 int reuse);

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int pymod(int a, int b) { return ((a % b) + b) % b; }

// TMA-staged weight gradient (wgrad_tma.cu): 0 = launched, < 0 = error, 1 = shape not covered (caller falls back)
int wgrad_tma_try(const coclr_wgrad_t& P, cudaStream_t stream);

}  // namespace coclr
