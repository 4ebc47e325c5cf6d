// TMA-staged weight gradient on wgmma tensor cores (sm_90a): the cuDNN wgrad reached through loss.backward()
// (reference main_nce.py:330) for the stride-1 (1,k,k) / (k,1,1) / 1x1x1 convolutions of the backbones
// (backbone/s3dg.py:11-13,39-42; backbone/resnet_2d3d.py).  Same C ABI as the gather kernel in conv_igemm.cu
// (coclr_conv_wgrad dispatches here first when the call brings a large enough workspace; spatially strided convs
// and calls without a workspace stay on the gather kernel).
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
//  * the pixel range is split over CTAs; every CTA ends with plain stores of its [cout, columns] register
//    accumulator into the workspace, and one reduction launch sums the splits into dW (no atomics).
//
// Warp roles (384 threads, three warpgroups): 0 loader, 1-3 idle (warpgroup 0 gives its registers to the consumers),
// 4-11 two MMA warpgroups (64-cout block wg of the item each) + epilogue.
#include <cuda.h>
#include <string.h>

#include <type_traits>
#include <utility>

#include "common.cuh"
#include "coclr_b200.h"
#include "conv_tma.h"

namespace coclr {

static constexpr int kWgThreads = 12 * 32;
static constexpr int kWgFirstMmaWarp = 4;            // warpgroup 0 loads, warpgroups 1-2 compute
static constexpr uint32_t kWgLoaderRegs = 40, kWgMmaRegs = 232;   // 128 x 40 + 256 x 232 <= 64 Ki registers
static constexpr int kWgTilePx = 64;                 // pixels per pipeline stage (4 K steps of 16)
static constexpr int kWgBlockBytes = kWgTilePx * 128;  // one [64 px][64 ch] operand block
static constexpr int kWgMaxStages = 4;

struct WgPlan {
  int ntiles[4];     // pixel tiles per logical dim (dim 0 fastest)
  int box[4];        // tile extent per dim
  int total_tiles;
  int n_types;       // slab types (one per tap of the non-reuse dimension)
  int nc;            // 64-channel chunks of the input
  int n_cgroups;     // column groups per type: nc (slab mode) or ceil(nc / nload) (block mode)
  int nload;         // X loads per stage and plane (block mode: up to 4 channel chunks; slab mode: 1)
  TmaSlabType type[4];
  int slab_bytes;    // one X load (a multiple of 1024)
  int lbo_bytes;     // distance between consecutive N blocks
  int N;             // columns of one MMA = 64 * blocks (the widest slab type; a type with fewer taps uses 64 * nshift)
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
  float* ws;            // partial accumulators [item][column][row] (see the epilogue)
  int dy_bf16, src_bf16;
};

// column of a work item's accumulator -> (tap, input channel)
struct WgCol {
  int tap, c;
};
COCLR_DEVINL WgCol wg_col(const WgPlan& L, const TmaSlabType& T, int cg, int col) {
  const int blk = col >> 6;
  WgCol r;
  if (L.win_c) {                      // window mode: a block is a kernel row, its 64 elements are (dx, channel)
    const int within = col & 63;
    const int dx = within / L.win_c;
    r.tap = T.tap[blk] * L.win_kw + dx;
    r.c = within - dx * L.win_c;
  } else if (L.nload > 1 || T.nshift == 1) {   // block mode: a block is a channel chunk of the single tap
    r.tap = T.tap[0];
    r.c = (cg * L.nload + blk) * 64 + (col & 63);
  } else {                            // slab mode: a block is a tap of the reuse dimension
    r.tap = T.tap[blk];
    r.c = cg * 64 + (col & 63);
  }
  return r;
}

// An item's kN columns are multiplied in sub-blocks, one wgmma group each; a sub-block starts on a 64-column block
// boundary (an MN-major operand has no other column offsets).  Widths: 64 for kN = 64 (one group per stage, not
// pipelined), 2 x 64 for kN = 128, 128 + 64 for kN = 192 and 4 x 64 for kN = 256.  The pipelined forms have an even
// number of sub-blocks, so each keeps its fresh block from stage to stage, and the accumulator (kN / 2 registers) plus
// the two fresh blocks stay within 192 registers per thread.
__host__ __device__ constexpr int wg_nsub(int n) { return n == 64 ? 1 : (n == 256 ? 4 : 2); }
__host__ __device__ constexpr int wg_sub_cols(int n, int j) { return n == 192 && j == 0 ? 128 : 64; }
__host__ __device__ constexpr int wg_sub_col0(int n, int j) { return j == 0 ? 0 : wg_sub_col0(n, j - 1) + wg_sub_cols(n, j - 1); }

template <int P, class A, class B>
COCLR_DEVINL auto& wg_pick(A& a, B& b) {
  if constexpr (P == 0) return a;
  else return b;
}
// f(0) && f(1) && ... with compile-time arguments
template <class F, int... Q>
COCLR_DEVINL bool wg_static_all(F&& f, std::integer_sequence<int, Q...>) {
  return (f(std::integral_constant<int, Q>{}) && ...);
}

// kN = the plan's L.N (64, 128, 192 or 256); kNProd = products per K step: 1 (single pass), 2 (Cout <= 64, hi / lo dY
// planes stacked over the two warpgroups), 3 (three passes); kBf16 = the 16-bit format of the planes.
template <int kN, int kNProd, bool kBf16>
__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_tma_kernel(const __grid_constant__ CUtensorMap map_dy_hi, const __grid_constant__ CUtensorMap map_dy_lo,
                 const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                 const WgArgs P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const WgPlan& L = P.plan;
  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);   // provably warp-uniform role branches for ptxas

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
      mbar_init(&empty_bar[s], 128u * (uint32_t)L.mb);   // one arrival per thread of every consumer warpgroup with work
    }
    mbar_fence_init();
  }
  __syncthreads();
  const TmaSlabType& T = L.type[type_i];
  const uint32_t dy_plane_bytes = (uint32_t)L.mb * kWgBlockBytes;
  const uint32_t x_plane_bytes = (uint32_t)L.nload * (uint32_t)L.slab_bytes;

  if (warp < kWgFirstMmaWarp) {
    setmaxnreg_dec<kWgLoaderRegs>();   // warpgroup 0: the loader warp 0, and warps 1-3 idle
    // ===================== loader =====================
    if (warp == 0 && elect_one()) {
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
    setmaxnreg_inc<kWgMmaRegs>();
    // ===================== MMA: warpgroup wg multiplies dY block wg (stacked: plane wg) with the X slab =====================
    const int wg = (warp - kWgFirstMmaWarp) >> 2;
    // L.mb == 1 (one 64-cout block, not stacked): warpgroup 2 has no rows; the empty barriers count only warpgroup 1
    if (wg >= L.mb) return;
    const int tw = threadIdx.x & 127;
    constexpr int kNSub = wg_nsub(kN);                  // sub-blocks (wgmma groups) per stage
    static_assert(kNSub == 1 || kNSub % 2 == 0, "a sub-block keeps its fresh block from stage to stage");
    constexpr int kT0 = wg_sub_cols(kN, 0) / 2, kT1 = wg_sub_cols(kN, kNSub == 1 ? 0 : 1) / 2;
    const uint32_t smem_base = smem_u32(smem);
    float acc[kN / 2];
#pragma unroll
    for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
    float t0[kT0], t1[kT1];
    // Issues sub-block j of the tile in stage slot s into t.  The products and their order per column are those of one
    // full-width stage: dY_hi X_lo, dY_lo X_hi, dY_hi X_hi (stacked: this warpgroup's plane X_lo, X_hi), 4 K steps each.
    auto issue = [&](auto jc, uint32_t s, auto& t) {
      constexpr int j = decltype(jc)::value;
      const uint32_t s_dy = smem_base + s * L.stage_bytes;
      // MN-major: LBO = stride between 64-element MN blocks, SBO = stride between 8-pixel groups (one swizzle atom);
      // one K = 16 step = 16 pixels = 2048 bytes = +128 descriptor units
      const uint32_t s_x = s_dy + L.off_x + (uint32_t)(wg_sub_col0(kN, j) / 64) * (uint32_t)L.lbo_bytes;
      const uint64_t b_hi = make_smem_desc(s_x, (uint32_t)L.lbo_bytes, 1024);
      const uint64_t b_lo = make_smem_desc(s_x + x_plane_bytes, (uint32_t)L.lbo_bytes, 1024);
      const uint64_t a_hi = make_smem_desc(s_dy + (uint32_t)wg * kWgBlockBytes, kWgBlockBytes, 1024);
      if constexpr (kNProd == 1) {
        const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_hi, b_hi, b_hi};
        wgmma_stage_issue<wg_sub_cols(kN, j), kBf16, 1, 1, 1>(t, ad, bd, 128u, 128u);
      } else if constexpr (kNProd == 2) {
        const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_lo, b_hi, b_hi};
        wgmma_stage_issue<wg_sub_cols(kN, j), kBf16, 2, 1, 1>(t, ad, bd, 128u, 128u);
      } else {
        const uint64_t a_lo = make_smem_desc(s_dy + dy_plane_bytes + (uint32_t)wg * kWgBlockBytes, kWgBlockBytes, 1024);
        const uint64_t ad[3] = {a_hi, a_lo, a_hi}, bd[3] = {b_lo, b_hi, b_hi};   // small products first
        wgmma_stage_issue<wg_sub_cols(kN, j), kBf16, 3, 1, 1>(t, ad, bd, 128u, 128u);
      }
    };
    // Adds a completed sub-block j into the accumulator (once per stage and column: the precision contract)
    auto fold = [&](auto jc, auto& t) {
      constexpr int j = decltype(jc)::value;
      constexpr int c0 = wg_sub_col0(kN, j) / 2;
      acc_fence(t);
#pragma unroll
      for (int i = 0; i < wg_sub_cols(kN, j) / 2; ++i) acc[c0 + i] += t[i];
    };
    // Group q + 1 is issued before group q is waited for and folded, so one group is always in flight while a
    // warpgroup folds, releases a stage and waits on the next full barrier.  A stage is released after its last
    // sub-block has been folded; every consumer thread arrives (an arrival under `lane == 0` would be a
    // thread-dependent branch inside the wgmma pipeline, which ptxas answers by serialising every wgmma).
    uint32_t stage = 0, phase = 0;   // the stage being folded
    // Waits for the stage after the one being folded and issues its first sub-block into t
    auto issue_next_tile = [&](auto& t) {
      uint32_t ns = stage + 1, np = phase;
      if (ns == (uint32_t)L.stages) { ns = 0; np ^= 1u; }
      mbar_wait_spin(&full_bar[ns], np);
      issue(std::integral_constant<int, 0>{}, ns, t);
    };
    // Folds sub-block j and, after the stage's last one, releases the stage
    auto retire = [&](auto qc) {
      constexpr int j = decltype(qc)::value;
      fold(qc, wg_pick<j & 1>(t0, t1));
      if constexpr (j == kNSub - 1) {
        mbar_arrive(&empty_bar[stage]);
        if (++stage == (uint32_t)L.stages) { stage = 0; phase ^= 1u; }
      }
    };
    // Sub-block q of a stage: issues the group after it, waits for it and retires it.  Only a stage's last sub-block can
    // be the item's last group: the loop ends there, in a branch that waits for everything (ptxas has to see that no
    // group is left in flight on any path).
    int tiles_left = ntile - 1;   // tiles whose first group is not issued yet
    auto step = [&](auto qc) -> bool {
      constexpr int q = decltype(qc)::value;
      if constexpr (q + 1 < kNSub) {
        issue(std::integral_constant<int, q + 1>{}, stage, wg_pick<(q + 1) & 1>(t0, t1));
      } else {
        if (tiles_left == 0) {
          wgmma_wait<0>();
          retire(qc);
          return false;
        }
        issue_next_tile(wg_pick<(q + 1) & 1>(t0, t1));
        --tiles_left;
      }
      wgmma_wait<1>();
      retire(qc);
      return true;
    };
    if constexpr (kNSub == 1) {
      for (int it = 0; it < ntile; ++it) {
        mbar_wait_spin(&full_bar[stage], phase);
        issue(std::integral_constant<int, 0>{}, stage, t0);
        wgmma_wait<0>();
        retire(std::integral_constant<int, 0>{});
      }
    } else if (ntile > 0) {
      mbar_wait_spin(&full_bar[0], 0);
      issue(std::integral_constant<int, 0>{}, 0u, t0);
      while (wg_static_all(step, std::make_integer_sequence<int, kNSub>{})) {
      }
    }
    // ===================== epilogue =====================
    // the accumulator goes to ws[item][column][row] with plain stores; wgrad_reduce_kernel sums the pixel splits into dW
    // (and drops the columns of taps an item does not have: the 3-tap parity of the temporally strided stem conv runs
    // at the 4-tap width kN; its 4th block reads frames inside the slab, which is sized for 4 taps)
    const int R = 128;
    const int row0 = 64 * wg + 16 * (tw >> 5) + ((tw & 31) >> 2);
    const int col0 = 2 * (tw & 3);
#pragma unroll
    for (int c = 0; c < kN / 32; ++c) {
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        const int row = row0 + 8 * ((r >> 1) & 1);      // row of the item's M = 128 tile
        const int col = c * 32 + col0 + 8 * (r >> 2) + (r & 1);
        P.ws[((size_t)blockIdx.x * kN + col) * R + row] = acc[16 * c + r];
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
  if (col >= (L.nload > 1 ? L.N : 64 * L.type[type_i].nshift)) return;
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

// Of the tile shapes (w[v], h[v]), the first that pads a W x H grid least; false when even that one would make more
// than half of every tile padding.
template <int n>
static bool least_padding(const int (&w)[n], const int (&h)[n], int W, int H, int& bw, int& bh) {
  long best_px = 0;
  for (int v = 0; v < n; ++v) {
    const long px = (long)ceil_div(W, w[v]) * w[v] * ceil_div(H, h[v]) * h[v];
    if (v == 0 || px < best_px) { best_px = px; bw = w[v]; bh = h[v]; }
  }
  return 2 * (long)W * H >= best_px;
}

static bool wgrad_tma_plan(const coclr_wgrad_t& P, WgPlan& L, MapSpec& DY, MapSpec& X) {
  const coclr_geom_t& g = P.g;
  const coclr_src_t& S = P.src;
  const coclr_src_t& D = P.dy;
  memset(&L, 0, sizeof(L));
  if (P.npass != 1 && P.npass != 3) return false;
  if (g.transposed) return false;
  const SlabKind kind = slab_kind(g, S, P.Td, P.Hd, P.Wd);
  if (kind == kSlabNone || D.T != P.Td || D.H != P.Hd || D.W != P.Wd) return false;
  // "same" convolutions only, but for the window's padded rows and the strided conv's input frames
  if (kind != kSlabWindow && kind != kSlabParity && (S.T != P.Td || S.H != P.Hd || S.W != P.Wd)) return false;
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
  L.nc = ceil_div(S.C, 64);
  L.nload = 1;
  L.n_cgroups = L.nc;
  for (int d = 0; d < 4; ++d) L.ntiles[d] = L.box[d] = 1;
  int ext[4];          // the output grid in the logical dims of the kind
  if (kind == kSlabFlat) {
    // flat pixels, up to four channel chunks next to each other
    L.box[0] = kWgTilePx;
    L.ntiles[0] = ceil_div((int)M, kWgTilePx);
    L.nload = L.nc < 4 ? L.nc : (L.nc % 4 == 0 ? 4 : (L.nc % 3 == 0 ? 3 : 4));
    L.n_cgroups = ceil_div(L.nc, L.nload);
    ext[0] = (int)M; ext[1] = ext[2] = ext[3] = 1;
  } else if (kind == kSlabWindow || kind == kSlabRows) {
    // tiles of nw x nh pixels; the window's blocks are the kernel rows, the 64 elements of a block the kw pixels x
    // channels of that row, so ONE slab serves all kh * kw taps
    static const int kNw[3] = {16, 8, 32}, kNh[3] = {4, 8, 2};          // least padding first, then the wider rows
    static const int kWinNw[2] = {8, 16}, kWinNh[2] = {8, 4};
    int nw, nh;
    const bool fits = kind == kSlabWindow ? least_padding(kWinNw, kWinNh, P.Wd, P.Hd, nw, nh) && g.kh <= 4
                                          : least_padding(kNw, kNh, P.Wd, P.Hd, nw, nh);
    if (!fits) return false;
    L.box[0] = nw; L.box[1] = nh;
    L.ntiles[0] = ceil_div(P.Wd, nw); L.ntiles[1] = ceil_div(P.Hd, nh); L.ntiles[2] = P.Td; L.ntiles[3] = P.B;
    if (kind == kSlabWindow) {
      L.win_c = S.C;
      L.win_kw = g.kw;
    }
    ext[0] = P.Wd; ext[1] = P.Hd; ext[2] = P.Td; ext[3] = P.B;
  } else {
    // tiles of npx pixels x nt frames; temporal stride 2 (the stem's (7,1,1) conv) reads the input frames by parity
    static const int kNpx[4] = {16, 8, 32, 64}, kNt[4] = {4, 8, 2, 1};
    const int HW = P.Hd * P.Wd;
    int npx, nt;
    if (!least_padding(kNpx, kNt, HW, P.Td, npx, nt)) return false;
    if (kind == kSlabParity &&
        (S.H != P.Hd || S.W != P.Wd || S.T % 2 != 0 || (S.T + 2 * g.pt - g.kt) / 2 + 1 != P.Td))
      return false;
    L.box[0] = npx; L.box[2] = nt;
    L.ntiles[0] = ceil_div(HW, npx); L.ntiles[2] = ceil_div(P.Td, nt); L.ntiles[3] = P.B;
    ext[0] = HW; ext[1] = 1; ext[2] = P.Td; ext[3] = P.B;
  }
  L.n_types = slab_types(kind, g, L.type);
  if (L.n_types == 0) return false;
  int reuse = 0;       // taps served by one slab
  for (int i = 0; i < L.n_types; ++i) reuse = L.type[i].nshift > reuse ? L.type[i].nshift : reuse;
  DY = plane_map(D.hi, D.lo, D.coff, 2, D.ld, D.C, ext, {64, L.box[0], L.box[1], L.box[2], L.box[3]});
  X = slab_map(kind, g, S, P.B, P.Wd, L.box, reuse);
  L.slab_bytes = 128 * (int)(X.box[1] * X.box[2] * X.box[3] * X.box[4]);
  L.lbo_bytes = 128 * L.box[0];
  L.N = 64 * (kind == kSlabFlat ? L.nload : reuse);
  if (L.N > 256 || reuse > 4) return false;
  L.total_tiles = L.ntiles[0] * L.ntiles[1] * L.ntiles[2] * L.ntiles[3];
  // ---- cout blocks per item: one per MMA warpgroup, as many as shared memory (>= 2 stages) allows ----
  const int cout_blocks = ceil_div(P.Cout, 64);
  L.stacked = (P.npass > 1 && P.Cout <= 64) ? 1 : 0;
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
  L.m_groups = L.stacked ? 1 : ceil_div(cout_blocks, L.mb);
  int st = (int)(budget / L.stage_bytes);
  L.stages = st > kWgMaxStages ? kWgMaxStages : st;
  L.off_bars = (uint32_t)L.stages * L.stage_bytes;
  L.total = L.off_bars + 256u + 1024u;
  // ---- pixel splits: one wave of CTAs; 4 tiles per CTA are enough to amortise the prologue ----
  const int items = L.n_types * L.n_cgroups * L.m_groups;
  int splits = wg_num_sms() / items;
  const int max_splits = L.total_tiles / 4 > 0 ? L.total_tiles / 4 : 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  L.tiles_per_split = ceil_div(L.total_tiles, splits);
  L.splits = ceil_div(L.total_tiles, L.tiles_per_split);
  return true;
}

static bool g_wgrad_tma = true;

int wgrad_tma_try(const coclr_wgrad_t& P, cudaStream_t stream) {
  if (!g_wgrad_tma || P.ws == nullptr || ((uintptr_t)P.ws & 15)) return 1;
  WgArgs args;
  MapSpec DY, X;
  if (!wgrad_tma_plan(P, args.plan, DY, X) || wg_ws_floats(args.plan) > P.ws_floats) return 1;
  args.ws = P.ws;
  CUtensorMap m_dy_hi, m_dy_lo, m_x_hi, m_x_lo;
  if (!encode_maps(&m_dy_hi, &m_dy_lo, DY, P.npass) || !encode_maps(&m_x_hi, &m_x_lo, X, P.npass)) return 1;
  const WgPlan& L = args.plan;
  args.dw = P.dw;
  args.out_scale = P.out_scale;
  args.dy_bf16 = P.dy_bf16;
  args.src_bf16 = P.src_bf16;
  const int grid = L.n_types * L.n_cgroups * L.m_groups * L.splits;
  // one kernel instance per (columns, products per K step, 16-bit format): the wgmma shapes and type are compile-time
  // constants
  int rc = COCLR_E_ARG;
  with_int<64, 128, 192, 256>(L.N, [&](auto n) {
    with_int<1, 2, 3>(L.planes == 1 ? 1 : (L.stacked ? 2 : 3), [&](auto nprod) {
      with_int<0, 1>(args.dy_bf16 != 0, [&](auto bf) {
        rc = launch_with_smem(wgrad_tma_kernel<n, nprod, bf != 0>, grid, kWgThreads, L.total, stream, m_dy_hi, m_dy_lo,
                              m_x_hi, m_x_lo, args);
      });
    });
  });
  if (rc != COCLR_OK) return rc;
  const int rows = L.stacked ? 64 : L.mb * 64;
  const dim3 rgrid((L.N * rows + 255) / 256, L.n_types * L.n_cgroups * L.m_groups);
  wgrad_reduce_kernel<<<rgrid, 256, 0, stream>>>(args);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

}  // namespace coclr

extern "C" void coclr_set_wgrad_tma(int enabled) { coclr::g_wgrad_tma = enabled != 0; }

// 1 when the TMA-staged kernel's planner accepts this shape (coclr_conv_wgrad then runs it there, given a workspace of
// coclr_wgrad_ws_floats floats); info[8] = {tile pixels dim 0, dim 1, dim 2, columns per MMA, cout blocks per item,
// pipeline stages, pixel splits, work items}
extern "C" int coclr_wgrad_tma_plan(const coclr_wgrad_t* p, int* info) {
  if (!p) return 0;
  coclr::WgPlan L;
  coclr::MapSpec DY, X;
  if (!coclr::wgrad_tma_plan(*p, L, DY, X)) return 0;
  if (info) {
    info[0] = L.box[0]; info[1] = L.box[1]; info[2] = L.box[2]; info[3] = L.N; info[4] = L.mb; info[5] = L.stages;
    info[6] = L.splits; info[7] = L.n_types * L.n_cgroups * L.m_groups * L.splits;
  }
  return 1;
}

// workspace (in floats) this shape needs to run on the TMA-staged kernel; 0 when the shape does not run there
extern "C" long coclr_wgrad_ws_floats(const coclr_wgrad_t* p) {
  if (!p) return 0;
  coclr::WgPlan L;
  coclr::MapSpec DY, X;
  if (!coclr::wgrad_tma_plan(*p, L, DY, X)) return 0;
  return coclr::wg_ws_floats(L);
}
