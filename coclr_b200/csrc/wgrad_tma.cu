// TMA-staged weight gradient on wgmma tensor cores (sm_90a): the cuDNN wgrad reached through loss.backward()
// (reference main_nce.py:330) for the stride-1 (1,k,k) / (k,1,1) / 1x1x1 convolutions of the backbones
// (backbone/s3dg.py:11-13,39-42; backbone/resnet_2d3d.py).  Same C ABI as the gather kernel in conv_igemm.cu
// (coclr_conv_wgrad dispatches here first; strided convs and the space-to-depth stem stay on the gather kernel).
//
//   dW[cout, tap, cin] += sum over pixels  dY[px, cout] * X[px + tap, cin]
//
// as a GEMM whose reduction dimension is the PIXEL: both operands are MN-major (a pixel is one 128-byte row of
// 64 channels), which is exactly what a cp.async.bulk.tensor tile load of channels-last planes with the 128B
// swizzle leaves in shared memory -- no thread computes an address:
//
//  * a work item is (pixel range, group of 64-cout blocks, column group).  Per 64-pixel tile it loads the dY blocks
//    [64 px][64 cout] of its cout group and ONE halo slab of X: the tile plus the rows the other taps of the reuse
//    dimension (dy of a (1,3,3) conv, dt of a (k,1,1) conv) need.  The taps are whole 8-row swizzle atoms apart
//    (tile rows are a multiple of 8 pixels), so they are the N blocks of ONE B operand whose block stride is the tap
//    shift: one K step of N = 64 * kh columns multiplies the dY tile with all kh taps at once, and each slab byte
//    fetched from L2 is used kh times (the gather kernel re-fetches every tap);
//  * 1x1x1 convs: the N blocks are up to four 64-channel tiles loaded next to each other;
//  * convolution padding and ragged tile edges are the TMA unit's out-of-bounds zero fill (a zero dY row or a zero X
//    row contributes nothing);
//  * split precision (3 passes over fp16 hi / lo planes) as everywhere; Cout <= 64: hi and lo dY planes are the two
//    64-row halves of the M = 128 tile (2 products per K step instead of 3, lo x lo included);
//  * the pixel range is split over CTAs; every CTA ends with its [cout, columns] register accumulator going to a
//    workspace (summed by one reduction launch) or, without one, with fp32 atomics into dW.
//
// Warp roles (288 threads): 0-7 two MMA warpgroups (64-cout block wg of the item each) + epilogue, 8 loader.
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "coclr_b200.h"
#include "conv_tma.h"

namespace coclr {

static constexpr int kWgMmaWarps = 8;
static constexpr int kWgThreads = (kWgMmaWarps + 1) * 32;
static constexpr int kWgAccChunks = 8;               // N <= 256: 128 fp32 accumulator registers per thread
static constexpr int kWgTilePx = 64;                 // pixels per pipeline stage (4 K steps of 16)
static constexpr int kWgBlockBytes = kWgTilePx * 128;  // one [64 px][64 ch] operand block
static constexpr int kWgMaxStages = 4;

struct WgType {
  int d[4];        // slab origin relative to the tile origin (logical dims 1..4 of the X map)
  int nblk;        // N blocks served by this slab (taps of the reuse dimension)
  int tap[8];      // tap index (kt-major, as in the weight tensor) of each block
};

struct WgPlan {
  int ntiles[4];     // pixel tiles per logical dim (dim 0 fastest)
  int box[4];        // tile extent per dim
  int total_tiles;
  int n_types;       // slab types (one per tap of the non-reuse dimension)
  int nc;            // 64-channel chunks of the input
  int n_cgroups;     // column groups per type: nc (slab mode) or ceil(nc / nload) (block mode)
  int nload;         // X loads per stage and plane (block mode: up to 4 channel chunks; slab mode: 1)
  WgType type[4];
  int slab_bytes;    // one X load (a multiple of 1024)
  int lbo_bytes;     // distance between consecutive N blocks
  int N;             // columns of one MMA = 64 * blocks (the widest slab type; a type with fewer taps uses 64 * nblk)
  int win_c, win_kw; // window mode (space-to-depth stem): a 64-element block is win_kw pixels of win_c channels
  int mb;            // 64-cout blocks per item, one per MMA warpgroup (stacked: 2 = hi / lo plane of the one block)
  int m_groups;      // cout groups
  int m_tiles;       // M = 128 tiles per item (always 1: two warpgroups of 64 rows)
  int stacked;
  int planes;        // 1 (single pass) or 2 (hi / lo)
  int splits, tiles_per_split;
  int stages;
  uint32_t stage_bytes, off_x, off_bars, total;
  int taps, C, Cin_real, Cout;
};

struct WgArgs {
  WgPlan plan;
  float* dw;
  const float* out_scale;
  float* ws;            // partial accumulators [item][column][row] (see the epilogue), or nullptr: fp32 atomics into dw
  int dy_bf16, src_bf16;
};

// column of a work item's accumulator -> (tap, input channel)
struct WgCol {
  int tap, c;
};
COCLR_DEVINL WgCol wg_col(const WgPlan& L, const WgType& T, int cg, int col) {
  const int blk = col >> 6;
  WgCol r;
  if (L.win_c) {                      // window mode: a block is a kernel row, its 64 elements are (dx, channel)
    const int within = col & 63;
    const int dx = within / L.win_c;
    r.tap = T.tap[blk] * L.win_kw + dx;
    r.c = within - dx * L.win_c;
  } else if (L.nload > 1 || T.nblk == 1) {   // block mode: a block is a channel chunk of the single tap
    r.tap = T.tap[0];
    r.c = (cg * L.nload + blk) * 64 + (col & 63);
  } else {                            // slab mode: a block is a tap of the reuse dimension
    r.tap = T.tap[blk];
    r.c = cg * 64 + (col & 63);
  }
  return r;
}

__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_tma_kernel(const __grid_constant__ CUtensorMap map_dy_hi, const __grid_constant__ CUtensorMap map_dy_lo,
                 const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                 const WgArgs P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const WgPlan& L = P.plan;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // work item: column group fastest (items that share a dY tile run at the same time: L2 hits), then cout group, split
  int w = blockIdx.x;
  const int n_cols = L.n_types * L.n_cgroups;
  const int colg = w % n_cols;
  w /= n_cols;
  const int mg = w % L.m_groups;
  const int split = w / L.m_groups;
  const int type_i = colg / L.n_cgroups;
  const int cg = colg - type_i * L.n_cgroups;
  const int t_begin = split * L.tiles_per_split;
  const int t_end = min(L.total_tiles, t_begin + L.tiles_per_split);
  const int ntile = max(0, t_end - t_begin);

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L.off_bars);
  uint64_t* empty_bar = full_bar + kWgMaxStages;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kWgMaxStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kWgMmaWarps);   // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();
  const WgType& T = L.type[type_i];
  const int Nt = L.nload > 1 ? L.N : 64 * T.nblk;     // columns of this item's MMAs
  const uint32_t dy_plane_bytes = (uint32_t)L.mb * kWgBlockBytes;
  const uint32_t x_plane_bytes = (uint32_t)L.nload * (uint32_t)L.slab_bytes;

  if (warp == kWgMmaWarps) {
    // ===================== loader =====================
    if (elect_one()) {
      tma_prefetch_desc(&map_dy_hi);
      tma_prefetch_desc(&map_x_hi);
      if (L.planes > 1) {
        tma_prefetch_desc(&map_dy_lo);
        tma_prefetch_desc(&map_x_lo);
      }
      const uint32_t dy_loads = L.stacked ? 2u : (uint32_t)(L.mb * L.planes);
      const uint32_t bytes = dy_loads * kWgBlockBytes + (uint32_t)L.planes * x_plane_bytes;
      const uint32_t smem_base = smem_u32(smem);
      uint32_t stage = 0, phase = 0;
      for (int t = t_begin; t < t_begin + ntile; ++t) {
        int m = t, o[4];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          o[d] = (m % L.ntiles[d]) * L.box[d];
          m /= L.ntiles[d];
        }
        o[3] = m * L.box[3];
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        mbar_arrive_expect_tx(&full_bar[stage], bytes);
        const uint32_t s_dy = smem_base + stage * L.stage_bytes;
        const uint32_t s_x = s_dy + L.off_x;
        if (L.stacked) {
          tma_load_5d(s_dy, &map_dy_hi, &full_bar[stage], 0, o[0], o[1], o[2], o[3]);
          tma_load_5d(s_dy + kWgBlockBytes, &map_dy_lo, &full_bar[stage], 0, o[0], o[1], o[2], o[3]);
        } else {
          for (int b = 0; b < L.mb; ++b) {
            const int c0 = (mg * L.mb + b) * 64;
            tma_load_5d(s_dy + b * kWgBlockBytes, &map_dy_hi, &full_bar[stage], c0, o[0], o[1], o[2], o[3]);
            if (L.planes > 1)
              tma_load_5d(s_dy + dy_plane_bytes + b * kWgBlockBytes, &map_dy_lo, &full_bar[stage], c0, o[0], o[1], o[2],
                          o[3]);
          }
        }
        for (int j = 0; j < L.nload; ++j) {
          const int c0 = (cg * L.nload + j) * 64;    // block mode: chunks past C are zero-filled
          const uint32_t dst = s_x + j * L.slab_bytes;
          tma_load_5d(dst, &map_x_hi, &full_bar[stage], c0, o[0] + T.d[0], o[1] + T.d[1], o[2] + T.d[2], o[3] + T.d[3]);
          if (L.planes > 1)
            tma_load_5d(dst + x_plane_bytes, &map_x_lo, &full_bar[stage], c0, o[0] + T.d[0], o[1] + T.d[1], o[2] + T.d[2],
                        o[3] + T.d[3]);
        }
        if (++stage == (uint32_t)L.stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // ===================== MMA: warpgroup wg multiplies dY block wg (stacked: plane wg) with the X slab =====================
    const int wg = warp >> 2;
    const int tw = threadIdx.x & 127;
    const bool active = L.stacked || wg < L.mb;
    const bool bf16 = P.dy_bf16 != 0;
    float acc[16 * kWgAccChunks];
#pragma unroll
    for (int i = 0; i < 16 * kWgAccChunks; ++i) acc[i] = 0.f;
    uint32_t stage = 0, phase = 0;
    for (int it = 0; it < ntile; ++it) {
      mbar_wait_spin(&full_bar[stage], phase);
      if (active) {
        const uint32_t s_dy = smem_u32(smem + stage * L.stage_bytes);
        const uint32_t s_x = s_dy + L.off_x;
        // MN-major: LBO = stride between 64-element MN blocks, SBO = stride between 8-pixel groups (one swizzle atom);
        // one K = 16 step = 16 pixels = 2048 bytes = +128 descriptor units
        const uint64_t b_hi = make_smem_desc(s_x, (uint32_t)L.lbo_bytes, 1024);
        const uint64_t b_lo = make_smem_desc(s_x + x_plane_bytes, (uint32_t)L.lbo_bytes, 1024);
        const uint32_t b_step = (uint32_t)L.lbo_bytes >> 4;
        const uint64_t a_hi = make_smem_desc(s_dy + (uint32_t)wg * kWgBlockBytes, kWgBlockBytes, 1024);
        const uint64_t a_lo = make_smem_desc(s_dy + dy_plane_bytes + (uint32_t)wg * kWgBlockBytes, kWgBlockBytes, 1024);
        if (L.planes == 1) {
          const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_hi, b_hi, b_hi};
          wgmma_stage<kWgAccChunks, 1, 1>(acc, ad, bd, 1, 128u, 128u, b_step, Nt, bf16);
        } else if (L.stacked) {
          const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_lo, b_hi, b_hi};
          wgmma_stage<kWgAccChunks, 1, 1>(acc, ad, bd, 2, 128u, 128u, b_step, Nt, bf16);
        } else {
          const uint64_t ad[3] = {a_hi, a_lo, a_hi}, bd[3] = {b_lo, b_hi, b_hi};   // small products first
          wgmma_stage<kWgAccChunks, 1, 1>(acc, ad, bd, 3, 128u, 128u, b_step, Nt, bf16);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == (uint32_t)L.stages) { stage = 0; phase ^= 1u; }
    }
    // ===================== epilogue =====================
    // with a workspace: the accumulator goes to ws[item][column][row] with plain stores and wgrad_reduce_kernel sums the
    // pixel splits into dW; without one: fp32 atomics straight into dW[cout, cin, tap]
    const float os = P.out_scale != nullptr ? __ldg(P.out_scale) : 1.f;
    const int R = 128;
    const int row0 = 64 * wg + 16 * (tw >> 5) + ((tw & 31) >> 2);
    const int col0 = 2 * (tw & 3);
#pragma unroll
    for (int c = 0; c < kWgAccChunks; ++c) {
      if (c * 32 >= Nt) break;
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        const int row = row0 + 8 * ((r >> 1) & 1);      // row of the item's M = 128 tile
        const int col = c * 32 + col0 + 8 * (r >> 2) + (r & 1);
        const float v = acc[16 * c + r];
        if (P.ws != nullptr) {
          P.ws[((size_t)blockIdx.x * L.N + col) * R + row] = v;
        } else if (ntile > 0) {
          int n;
          if (L.stacked) {
            n = row & 63;
          } else {
            n = (mg * L.mb) * 64 + row;
            if ((row >> 6) >= L.mb) n = L.Cout;          // the second warpgroup of an odd last block has no rows
          }
          if (n < L.Cout) {
            const WgCol k = wg_col(L, T, cg, col);
            if (k.c < L.Cin_real) atomicAdd(P.dw + ((size_t)n * L.Cin_real + k.c) * L.taps + k.tap, v * os);
          }
        }
      }
    }
  }
}

// dW[cout, cin, tap] += out_scale * sum over pixel splits of ws[item][column][row]; grid (columns x rows, column group x
// cout group); consecutive threads read consecutive rows.  Every dW element belongs to exactly one thread.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const WgArgs P) {
  const WgPlan& L = P.plan;
  const int n_cols = L.n_types * L.n_cgroups;
  const int colg = blockIdx.y % n_cols, mg = blockIdx.y / n_cols;
  const int type_i = colg / L.n_cgroups, cg = colg - type_i * L.n_cgroups;
  const int rows = L.stacked ? 64 : L.mb * 64;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int col = idx / rows, r = idx - col * rows;
  if (col >= (L.nload > 1 ? L.N : 64 * L.type[type_i].nblk)) return;
  const int n = L.stacked ? r : mg * L.mb * 64 + r;
  const WgCol k = wg_col(L, L.type[type_i], cg, col);
  if (n >= L.Cout || k.c >= L.Cin_real) return;
  const int R = 128 * L.m_tiles;
  const size_t per_split = (size_t)L.m_groups * n_cols * L.N * R;
  const float* src = P.ws + ((size_t)(mg * n_cols + colg) * L.N + col) * R + r;
  float acc = 0.f;
  for (int s = 0; s < L.splits; ++s) {
    acc += src[(size_t)s * per_split];
    if (L.stacked) acc += src[(size_t)s * per_split + 64];
  }
  const float os = P.out_scale != nullptr ? __ldg(P.out_scale) : 1.f;
  P.dw[((size_t)n * L.Cin_real + k.c) * L.taps + k.tap] += acc * os;
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int wg_ceil_div(int a, int b) { return (a + b - 1) / b; }

static int wg_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

static long wg_ws_floats(const WgPlan& L) {
  return (long)L.n_types * L.n_cgroups * L.m_groups * L.splits * L.N * 128 * L.m_tiles;
}

// with_ws: plan for the workspace epilogue (one wave of CTAs, no atomics); otherwise for the atomic epilogue
static bool wgrad_tma_plan(const coclr_wgrad_t& P, bool with_ws, WgPlan& L, MapSpec& DY, MapSpec& X) {
  const coclr_geom_t& g = P.g;
  const coclr_src_t& S = P.src;
  const coclr_src_t& D = P.dy;
  memset(&L, 0, sizeof(L));
  if (P.npass != 1 && P.npass != 3) return false;
  if (g.transposed || g.sh != 1 || g.sw != 1 || (g.st != 1 && g.st != 2)) return false;
  if (D.T != P.Td || D.H != P.Hd || D.W != P.Wd) return false;
  // window kind (the space-to-depth stem, see conv_tma.cu): the kw taps of a kernel row are kw consecutive pixels of
  // 64 / kw channels = one 128-byte run, read through a tensor map whose pixel stride is smaller than its inner extent
  const bool window = g.kt == 1 && g.kw > 1 && S.C * g.kw == 64 && S.ld == S.C && S.coff == 0 && g.pw == 0 &&
                      g.st == 1 && S.W >= P.Wd + g.kw - 1 && S.H == P.Hd && S.T == P.Td;
  const bool tstride = g.st == 2 && g.kh == 1 && g.kw == 1 && g.kt > 1;
  if (g.st == 2 && !tstride) return false;
  if (!window && !tstride && (S.T != P.Td || S.H != P.Hd || S.W != P.Wd)) return false;   // else "same" convs only
  if (S.C % 8 || D.C % 8 || S.ld % 8 || D.ld % 8 || S.coff % 8 || D.coff % 8) return false;
  if (P.npass > 1 && (!S.lo || !D.lo)) return false;
  if (((uintptr_t)S.hi | (uintptr_t)D.hi | (uintptr_t)S.lo | (uintptr_t)D.lo) & 15) return false;
  if (g.kt > 8 || g.kh > 8 || g.kw > 4) return false;
  const long M = (long)P.B * P.Td * P.Hd * P.Wd;
  if (M >= (1l << 31) || P.Cin_real > S.C || P.Cout > D.C) return false;
  L.taps = g.kt * g.kh * g.kw;
  L.C = S.C;
  L.Cin_real = P.Cin_real;
  L.Cout = P.Cout;
  L.planes = P.npass > 1 ? 2 : 1;
  L.nc = wg_ceil_div(S.C, 64);
  const long ldx = (long)S.ld * 2, ldd = (long)D.ld * 2;
  DY.elem_bytes = X.elem_bytes = 2;
  DY.base[0] = (void*)((const uint16_t*)D.hi + D.coff);
  DY.base[1] = D.lo ? (void*)((const uint16_t*)D.lo + D.coff) : nullptr;
  X.base[0] = (void*)((const uint16_t*)S.hi + S.coff);
  X.base[1] = S.lo ? (void*)((const uint16_t*)S.lo + S.coff) : nullptr;
  for (int d = 0; d < 4; ++d) L.ntiles[d] = L.box[d] = 1;
  int reuse = 1;       // taps served by one slab
  if (L.taps == 1) {
    // ---- 1x1x1: flat pixels, up to four channel chunks next to each other ----
    L.box[0] = kWgTilePx;
    L.ntiles[0] = wg_ceil_div((int)M, kWgTilePx);
    for (MapSpec* m : {&DY, &X}) {
      const long ld = m == &DY ? ldd : ldx;
      m->dims[0] = m == &DY ? D.C : S.C; m->dims[1] = M; m->dims[2] = m->dims[3] = m->dims[4] = 1;
      m->strides[0] = ld; m->strides[1] = m->strides[2] = m->strides[3] = (uint64_t)ld * M;
      m->box[0] = 64; m->box[1] = kWgTilePx; m->box[2] = m->box[3] = m->box[4] = 1;
    }
    L.n_types = 1;
    L.type[0].nblk = 1;
    L.type[0].tap[0] = 0;
    L.nload = L.nc < 4 ? L.nc : (L.nc % 4 == 0 ? 4 : (L.nc % 3 == 0 ? 3 : 4));
    L.n_cgroups = wg_ceil_div(L.nc, L.nload);
    L.slab_bytes = kWgBlockBytes;
    L.lbo_bytes = kWgBlockBytes;
    L.N = 64 * L.nload;
  } else if (window) {
    // ---- space-to-depth stem: (1, kh, kw) over 64/kw-channel pixels; ONE slab serves all kh * kw taps: its blocks are
    // the kernel rows, the 64 elements of a block the kw pixels x channels of that row ----
    static const int kNw[2] = {8, 16}, kNh[2] = {8, 4};
    int best = -1;
    long best_px = 0;
    for (int v = 0; v < 2; ++v) {
      const long px = (long)wg_ceil_div(P.Wd, kNw[v]) * kNw[v] * wg_ceil_div(P.Hd, kNh[v]) * kNh[v];
      if (best < 0 || px < best_px) { best = v; best_px = px; }
    }
    const int nw = kNw[best], nh = kNh[best];
    if (2 * (long)P.Wd * P.Hd < best_px || g.kh > 4) return false;
    L.box[0] = nw; L.box[1] = nh;
    L.ntiles[0] = wg_ceil_div(P.Wd, nw); L.ntiles[1] = wg_ceil_div(P.Hd, nh); L.ntiles[2] = P.Td; L.ntiles[3] = P.B;
    DY.dims[0] = D.C; DY.dims[1] = P.Wd; DY.dims[2] = P.Hd; DY.dims[3] = P.Td; DY.dims[4] = P.B;
    DY.strides[0] = ldd; DY.strides[1] = ldd * P.Wd; DY.strides[2] = ldd * P.Wd * P.Hd;
    DY.strides[3] = ldd * P.Wd * P.Hd * P.Td;
    DY.box[0] = 64; DY.box[1] = nw; DY.box[2] = nh; DY.box[3] = DY.box[4] = 1;
    X.dims[0] = 64; X.dims[1] = P.Wd; X.dims[2] = S.H; X.dims[3] = S.T; X.dims[4] = P.B;
    X.strides[0] = ldx; X.strides[1] = ldx * S.W; X.strides[2] = ldx * S.W * S.H; X.strides[3] = ldx * S.W * S.H * S.T;
    X.box[0] = 64; X.box[1] = nw; X.box[2] = nh + g.kh - 1; X.box[3] = X.box[4] = 1;
    reuse = g.kh;
    L.n_types = 1;
    L.type[0].d[1] = -g.ph;
    L.type[0].nblk = g.kh;
    for (int j = 0; j < g.kh; ++j) L.type[0].tap[j] = j;
    L.nc = 1;
    L.nload = 1;
    L.n_cgroups = 1;
    L.win_c = S.C;
    L.win_kw = g.kw;
    L.slab_bytes = nw * (nh + g.kh - 1) * 128;
    L.lbo_bytes = nw * 128;
    L.N = 64 * g.kh;
  } else if (g.kt == 1) {
    // ---- (1, kh, kw): tiles of nw x nh pixels, one slab type per dx, the kh taps of a column share the slab ----
    static const int kNw[3] = {16, 8, 32}, kNh[3] = {4, 8, 2};
    int best = -1;
    long best_px = 0;
    for (int v = 0; v < 3; ++v) {      // least padding first, then the wider rows
      const long px = (long)wg_ceil_div(P.Wd, kNw[v]) * kNw[v] * wg_ceil_div(P.Hd, kNh[v]) * kNh[v];
      if (best < 0 || px < best_px) { best = v; best_px = px; }
    }
    const int nw = kNw[best], nh = kNh[best];
    if (2 * (long)P.Wd * P.Hd < best_px) return false;       // more than half of every tile would be padding
    L.box[0] = nw; L.box[1] = nh;
    L.ntiles[0] = wg_ceil_div(P.Wd, nw); L.ntiles[1] = wg_ceil_div(P.Hd, nh); L.ntiles[2] = P.Td; L.ntiles[3] = P.B;
    for (MapSpec* m : {&DY, &X}) {
      const long ld = m == &DY ? ldd : ldx;
      m->dims[0] = m == &DY ? D.C : S.C; m->dims[1] = P.Wd; m->dims[2] = P.Hd; m->dims[3] = P.Td; m->dims[4] = P.B;
      m->strides[0] = ld; m->strides[1] = ld * P.Wd; m->strides[2] = ld * P.Wd * P.Hd;
      m->strides[3] = ld * P.Wd * P.Hd * P.Td;
      m->box[0] = 64; m->box[1] = nw; m->box[2] = nh; m->box[3] = m->box[4] = 1;
    }
    X.box[2] = nh + g.kh - 1;
    reuse = g.kh;
    L.n_types = g.kw;
    for (int xa = 0; xa < g.kw; ++xa) {
      WgType& t = L.type[xa];
      t.d[0] = xa - g.pw;
      t.d[1] = -g.ph;
      t.nblk = g.kh;
      for (int j = 0; j < g.kh; ++j) t.tap[j] = j * g.kw + xa;
    }
    L.nload = 1;
    L.n_cgroups = L.nc;
    L.slab_bytes = nw * (nh + g.kh - 1) * 128;
    L.lbo_bytes = nw * 128;
    L.N = 64 * g.kh;
  } else if (g.kh == 1 && g.kw == 1) {
    // ---- (kt, 1, 1): the pixels of a frame are one flat dimension; tiles of npx pixels x nt frames ----
    const int HW = P.Hd * P.Wd;
    static const int kNpx[4] = {16, 8, 32, 64}, kNt[4] = {4, 8, 2, 1};
    int best = -1;
    long best_px = 0;
    for (int v = 0; v < 4; ++v) {
      const long px = (long)wg_ceil_div(HW, kNpx[v]) * kNpx[v] * wg_ceil_div(P.Td, kNt[v]) * kNt[v];
      if (best < 0 || px < best_px) { best = v; best_px = px; }
    }
    const int npx = kNpx[best], nt = kNt[best];
    if (2 * (long)HW * P.Td < best_px) return false;
    L.box[0] = npx; L.box[2] = nt;
    L.ntiles[0] = wg_ceil_div(HW, npx); L.ntiles[2] = wg_ceil_div(P.Td, nt); L.ntiles[3] = P.B;
    DY.dims[0] = D.C; DY.dims[1] = HW; DY.dims[2] = 1; DY.dims[3] = P.Td; DY.dims[4] = P.B;
    DY.strides[0] = ldd; DY.strides[1] = ldd * HW; DY.strides[2] = ldd * HW; DY.strides[3] = ldd * HW * P.Td;
    DY.box[0] = 64; DY.box[1] = npx; DY.box[2] = 1; DY.box[3] = nt; DY.box[4] = 1;
    L.nload = 1;
    L.n_cgroups = L.nc;
    L.lbo_bytes = npx * 128;
    if (!tstride) {
      X.dims[0] = S.C; X.dims[1] = HW; X.dims[2] = 1; X.dims[3] = S.T; X.dims[4] = P.B;
      X.strides[0] = ldx; X.strides[1] = ldx * HW; X.strides[2] = ldx * HW; X.strides[3] = ldx * HW * S.T;
      X.box[0] = 64; X.box[1] = npx; X.box[2] = 1; X.box[3] = nt + g.kt - 1; X.box[4] = 1;
      reuse = g.kt;
      L.n_types = 1;
      WgType& t = L.type[0];
      t.d[2] = -g.pt;
      t.nblk = g.kt;
      for (int j = 0; j < g.kt; ++j) t.tap[j] = j;
    } else {
      // temporal stride 2 (the stem's (7,1,1) conv): input frame 2 * t' - pt + dt = 2 * (t' + sh) + par; the X map
      // splits the frames by parity, [C, HW, 2, T / 2, B], and there is one slab type per parity
      if (S.H != P.Hd || S.W != P.Wd || S.T % 2 != 0 || (S.T + 2 * g.pt - g.kt) / 2 + 1 != P.Td) return false;
      X.dims[0] = S.C; X.dims[1] = HW; X.dims[2] = 2; X.dims[3] = S.T / 2; X.dims[4] = P.B;
      X.strides[0] = ldx; X.strides[1] = ldx * HW; X.strides[2] = ldx * HW * 2; X.strides[3] = ldx * HW * S.T;
      L.n_types = 2;
      for (int par = 0; par < 2; ++par) {
        WgType& t = L.type[par];
        t.nblk = 0;
        for (int dt = 0; dt < g.kt; ++dt) {
          const int rel = dt - g.pt;
          if ((((rel % 2) + 2) % 2) != par) continue;
          const int sh = (rel - par) / 2;            // exact
          if (t.nblk == 0) t.d[2] = sh;               // taps of one parity are consecutive shifts
          t.tap[t.nblk++] = dt;
        }
        t.d[1] = par;
        if (t.nblk == 0) return false;
        if (t.nblk > reuse) reuse = t.nblk;
      }
      X.box[0] = 64; X.box[1] = npx; X.box[2] = 1; X.box[3] = nt + reuse - 1; X.box[4] = 1;
    }
    L.slab_bytes = npx * (nt + reuse - 1) * 128;
    L.N = 64 * reuse;
  } else {
    return false;
  }
  if (L.N > 256 || reuse > 4) return false;
  L.total_tiles = L.ntiles[0] * L.ntiles[1] * L.ntiles[2] * L.ntiles[3];
  // ---- cout blocks per item: one per MMA warpgroup, as many as shared memory (>= 2 stages) allows ----
  const int cout_blocks = wg_ceil_div(P.Cout, 64);
  L.stacked = (P.npass > 1 && P.Cout <= 64 && getenv("COCLR_WGRAD_NOSTACK") == nullptr) ? 1 : 0;
  const uint32_t x_bytes = (uint32_t)L.planes * L.nload * L.slab_bytes;
  const uint32_t budget = 227u * 1024u - 2048u;
  int mb = cout_blocks < 2 ? cout_blocks : 2;
  if (L.stacked) mb = 2;
  for (;; --mb) {
    if (mb < 1) return false;
    const int m_tiles = 1;
    const uint32_t dy_bytes = (uint32_t)(L.stacked ? 1 : L.planes) * mb * kWgBlockBytes;
    const uint32_t stage = dy_bytes + x_bytes;
    if (2 * stage <= budget) {
      L.mb = mb;
      L.m_tiles = m_tiles;
      L.off_x = dy_bytes;
      L.stage_bytes = stage;
      break;
    }
    if (L.stacked) return false;
  }
  L.m_groups = L.stacked ? 1 : wg_ceil_div(cout_blocks, L.mb);
  int st = (int)(budget / L.stage_bytes);
  L.stages = st > kWgMaxStages ? kWgMaxStages : st;
  L.off_bars = (uint32_t)L.stages * L.stage_bytes;
  L.total = L.off_bars + 256u + 1024u;
  // ---- pixel splits: one wave of CTAs.  Atomic epilogue: every CTA ends with Cout x N fp32 atomics, measured to
  // dominate once a CTA has fewer than ~16 tiles (and with more than ~74 splits on the same dW); workspace epilogue:
  // plain stores, 4 tiles per CTA are enough to amortise the prologue ----
  const int items = L.n_types * L.n_cgroups * L.m_groups;
  int splits = wg_num_sms() / items;
  if (!with_ws && splits > wg_num_sms() / 2) splits = wg_num_sms() / 2;   // CTAs adding to the same dW elements
  const int min_tiles = with_ws ? 4 : 16;
  const int max_splits = L.total_tiles / min_tiles > 0 ? L.total_tiles / min_tiles : 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  { const char* e = getenv("COCLR_WGRAD_SPLITS"); if (e && atoi(e) > 0) splits = atoi(e); }
  L.tiles_per_split = wg_ceil_div(L.total_tiles, splits);
  L.splits = wg_ceil_div(L.total_tiles, L.tiles_per_split);
  return true;
}

static int g_wgrad_tma = -1;

int wgrad_tma_try(const coclr_wgrad_t& P, cudaStream_t stream) {
  if (g_wgrad_tma < 0) {
    const char* e = getenv("COCLR_WGRAD_TMA");
    g_wgrad_tma = (e && e[0] == '0') ? 0 : 1;
  }
  if (!g_wgrad_tma) return 1;
  WgArgs args;
  MapSpec DY, X;
  bool with_ws = P.ws != nullptr;
  if (!wgrad_tma_plan(P, with_ws, args.plan, DY, X)) return 1;
  if (with_ws && (wg_ws_floats(args.plan) > P.ws_floats || ((uintptr_t)P.ws & 15))) {
    with_ws = false;                                   // workspace too small: atomic epilogue
    if (!wgrad_tma_plan(P, false, args.plan, DY, X)) return 1;
  }
  args.ws = with_ws ? P.ws : nullptr;
  CUtensorMap m_dy_hi, m_dy_lo, m_x_hi, m_x_lo;
  if (!encode_map(&m_dy_hi, DY, 0) || !encode_map(&m_x_hi, X, 0)) return 1;
  if (P.npass > 1) {
    if (!encode_map(&m_dy_lo, DY, 1) || !encode_map(&m_x_lo, X, 1)) return 1;
  } else {
    m_dy_lo = m_dy_hi;
    m_x_lo = m_x_hi;
  }
  const WgPlan& L = args.plan;
  args.dw = P.dw;
  args.out_scale = P.out_scale;
  args.dy_bf16 = P.dy_bf16;
  args.src_bf16 = P.src_bf16;
  if (getenv("COCLR_TMA_DEBUG"))
    fprintf(stderr, "coclr wgrad_tma: tiles %d box %dx%dx%dx%d types %d cgroups %d nload %d N %d mb %d m_groups %d "
            "stacked %d stages %d stage_bytes %u splits %d\n", L.total_tiles, L.box[0], L.box[1], L.box[2],
            L.box[3], L.n_types, L.n_cgroups, L.nload, L.N, L.mb, L.m_groups, L.stacked, L.stages, L.stage_bytes,
            L.splits);
  cudaError_t e = cudaFuncSetAttribute(wgrad_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total);
  if (e != cudaSuccess) return COCLR_E_LAUNCH;
  const int grid = L.n_types * L.n_cgroups * L.m_groups * L.splits;
  wgrad_tma_kernel<<<grid, kWgThreads, L.total, stream>>>(m_dy_hi, m_dy_lo, m_x_hi, m_x_lo, args);
  if (args.ws != nullptr) {
    const int rows = L.stacked ? 64 : L.mb * 64;
    const dim3 rgrid((L.N * rows + 255) / 256, L.n_types * L.n_cgroups * L.m_groups);
    wgrad_reduce_kernel<<<rgrid, 256, 0, stream>>>(args);
  }
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

}  // namespace coclr

extern "C" void coclr_set_wgrad_tma(int enabled) { coclr::g_wgrad_tma = enabled ? 1 : 0; }

// 1 when coclr_conv_wgrad would run this shape on the TMA-staged kernel; info[8] = {tile pixels dim 0, dim 1, dim 2,
// columns per MMA, cout blocks per item, pipeline stages, pixel splits, work items}
extern "C" int coclr_wgrad_tma_plan(const coclr_wgrad_t* p, int* info) {
  if (!p) return 0;
  coclr::WgPlan L;
  coclr::MapSpec DY, X;
  if (!coclr::wgrad_tma_plan(*p, p->ws != nullptr, L, DY, X)) return 0;
  if (info) {
    info[0] = L.box[0]; info[1] = L.box[1]; info[2] = L.box[2]; info[3] = L.N; info[4] = L.mb; info[5] = L.stages;
    info[6] = L.splits; info[7] = L.n_types * L.n_cgroups * L.m_groups * L.splits;
  }
  return 1;
}

// workspace (in floats) with which coclr_conv_wgrad replaces the fp32 atomics of this shape by plain stores + one
// reduction launch; 0 when the shape does not run on the TMA-staged kernel
extern "C" long coclr_wgrad_ws_floats(const coclr_wgrad_t* p) {
  if (!p) return 0;
  coclr::WgPlan L;
  coclr::MapSpec DY, X;
  if (!coclr::wgrad_tma_plan(*p, true, L, DY, X)) return 0;
  return coclr::wg_ws_floats(L);
}
