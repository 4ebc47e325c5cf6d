// TMA-staged implicit-GEMM convolution on wgmma tensor cores (sm_90a): forward and data-gradient of the
// stride-1 (1,k,k) / (k,1,1) / 1x1x1 convolutions and of the temporally strided (k,1,1) stem conv of the
// reference's backbones (backbone/s3dg.py:11-13 BasicConv3d, :39-42 STConv3d conv1 / conv2; cuDNN dgrad behind
// loss.backward(), main_nce.py:330).  Same C ABI as conv_igemm.cu (coclr_conv_igemm dispatches here first); what
// changes is how the operands travel:
//
//  * the A operand (channels-last 16-bit hi / lo activation planes) is described by a 5-D CUtensorMap
//    [channels, W, H, T, B] (or [channels, H*W, parity, T/2, B] for the temporal kernels).  One elected thread
//    issues cp.async.bulk.tensor loads of a HALO SLAB -- the 128-pixel output tile plus the rows the other taps
//    of the reuse dimension need -- into 128B-swizzled shared memory; convolution padding and ragged tile edges
//    are the TMA unit's out-of-bounds zero fill.  No thread computes an address.
//  * the taps along the reuse dimension (dy of a (1,3,3) conv, dt of a (k,1,1) conv) are served from the SAME
//    slab: their A descriptors differ by a whole number of 8-row swizzle atoms (tile rows are a multiple of 8
//    pixels wide), so every slab byte fetched from L2 feeds up to kh (kt) x 12 K-steps of tensor-core instructions;
//  * weights: the pre-swizzled hi / lo tile images of coclr_pack_weights, either streamed through a ring of
//    bulk copies or -- for narrow layers whose whole image fits -- loaded ONCE per CTA and kept resident;
//  * two consumer warpgroups (64 tile rows each) accumulate in registers with wgmma: one m64 x BN x k16 instruction
//    per product and K step, BN fixed at compile time.  Each 64-deep K chunk (a pipeline stage) is summed in a fresh
//    register block and added to the accumulator in fp32; the next stage's instructions are issued before that add,
//    so the tensor cores are not idle while a stage is folded and its shared-memory slots are released.
//  * epilogue: each consumer thread scales its accumulator fragment in registers and writes it, 32 columns at a time,
//    into a 128B-swizzled staging block of 32 tile rows (two warps per block, which take alternate chunks for the
//    rest).  A chunk's warp accumulates the BatchNorm statistics from it and writes it with ONE cp.async.bulk.tensor
//    store (or add-reduction, for gradient accumulation) per 32 rows x 32 channels: edge clipping, channel slices of
//    concat buffers and the strided frame order of the transposed stem conv are properties of the output tensor map,
//    not code.  The two warpgroups share no barrier, so one's epilogue runs while the other's MMAs keep the tensor
//    cores busy.
//
// Warp roles (384 threads, three warpgroups): 0 A loader, 1 weight loader, 2-3 idle (warpgroup 0 gives its registers to
// the consumers), 4-11 MMA and epilogue (warpgroups 1 and 2).
#include <cuda.h>
#include <string.h>

#include "common.cuh"
#include "coclr_b200.h"
#include "conv_tma.h"

namespace coclr {

static constexpr int kTmaThreads = 12 * 32;
static constexpr int kTmaMmaWarps = 8;
static constexpr int kTmaFirstMmaWarp = 4;     // warpgroup 0 loads, warpgroups 1-2 compute
static constexpr int kTmaMaxBN = 128;          // 64 fp32 accumulator registers per thread
static constexpr uint32_t kTmaLoaderRegs = 40, kTmaMmaRegs = 232;   // 128 x 40 + 256 x 232 <= 64 Ki registers
static constexpr int kTmaMaxASlots = 4;
static constexpr int kTmaMaxBSlots = 4;
// Shared memory the planner leaves unused: what the earlier epilogue's transpose tile and scale table took.  Handing it to
// the rings would move the temporally strided stem conv to another tile shape, and with it the summation order of its
// BatchNorm statistics; kept so that every launch runs on the tile plan it had.
static constexpr int kPlanKeepBytes = 1024 + 128 * 33 * 4;

struct TmaTile {
  int idx[4];
  int n_tile;
};
// Work item -> tile.  Items enumerate (pixel tile, N tile) with the N tile fastest.
COCLR_DEVINL TmaTile tma_decode(const TmaPlan& L, int item) {
  TmaTile t;
  t.n_tile = item % L.out.n_tiles_n;
  int m = item / L.out.n_tiles_n;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    t.idx[d] = m % L.ntiles[d];
    m /= L.ntiles[d];
  }
  t.idx[3] = m;
  return t;
}

// The tile's first slab type: t.idx[sel_dim] when the tile index selects it, else 0.  Selected without indexing t.idx at
// run time, which would put t in local memory.
COCLR_DEVINL int tma_first_type(const TmaPlan& L, const TmaTile& t) {
  int ty = 0;
#pragma unroll
  for (int d = 0; d < 4; ++d)
    if (L.sel_dim == d) ty = t.idx[d];
  return ty;
}

template <int kNPass, int kBN, bool kBf16>
__global__ void __launch_bounds__(kTmaThreads, 1)
    conv_tma_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                    const __grid_constant__ CUtensorMap map_out, const __grid_constant__ TmaArgs P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr bool kLo = kNPass > 1;
  constexpr uint32_t kPlanes = kLo ? 2u : 1u;
  constexpr uint32_t kBTileBytes = kPlanes * kBN * 128u;  // one K chunk of weights (hi, lo) in shared memory
  const TmaPlan& L = P.plan;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t a_base = smem_base;
  const uint32_t b_base = smem_base + L.off_b;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + L.off_bars);
  uint64_t* a_empty = a_full + kTmaMaxASlots;
  uint64_t* b_full = a_empty + kTmaMaxASlots;
  uint64_t* b_empty = b_full + kTmaMaxBSlots;

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);   // provably warp-uniform role branches for ptxas
  const int first_item = (int)blockIdx.x;
  const int item_stride = (int)gridDim.x;
  const int n_items = L.total_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kTmaMaxASlots; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], kTmaMmaWarps * 32);   // one arrival per consumer thread
    }
    for (int s = 0; s < kTmaMaxBSlots; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], kTmaMmaWarps * 32);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < kTmaFirstMmaWarp) {
    setmaxnreg_dec<kTmaLoaderRegs>();   // warpgroup 0: the loader warps 0-1, and warps 2-3 idle
    if (warp == 0) {
      // ===================== A loader: one TMA box (hi) + one (lo) per slab =====================
      if (elect_one()) {
        tma_prefetch_desc(&map_hi);
        if (kLo) tma_prefetch_desc(&map_lo);
        uint32_t slot = 0, phase = 0;
        for (int item = first_item; item < n_items; item += item_stride) {
          const TmaTile t = tma_decode(L, item);
          const int ty0 = tma_first_type(L, t);
          const int ty1 = L.sel_dim >= 0 ? ty0 + 1 : L.n_types;
          for (int cc = 0; cc < L.nc; ++cc) {
            for (int ty = ty0; ty < ty1; ++ty) {
              const TmaSlabType& S = L.type[ty];
              mbar_wait(&a_empty[slot], phase ^ 1u);
              const int c0 = cc * L.a_c0_step;
              const int c1 = t.idx[0] * L.a_mul[0] + S.d[0];
              const int c2 = t.idx[1] * L.a_mul[1] + S.d[1];
              const int c3 = t.idx[2] * L.a_mul[2] + S.d[2];
              const int c4 = t.idx[3] * L.a_mul[3] + S.d[3];
              const uint32_t dst = a_base + slot * (uint32_t)L.a_slot_bytes;
              mbar_arrive_expect_tx(&a_full[slot], kPlanes * (uint32_t)L.slab_bytes);
              tma_load_5d(dst, &map_hi, &a_full[slot], c0, c1, c2, c3, c4);
              if (kLo) tma_load_5d(dst + (uint32_t)L.plane_stride, &map_lo, &a_full[slot], c0, c1, c2, c3, c4);
              if (++slot == (uint32_t)L.a_slots) { slot = 0; phase ^= 1u; }
            }
          }
        }
      }
    } else if (warp == 1) {
      // ===================== weight loader: bulk copies of pre-swizzled tile images =====================
      if (elect_one()) {
        const uint32_t tile_bytes = kBTileBytes;                               // what one K chunk needs in smem
        const size_t img_stride = (size_t)2u * (size_t)kBN * 128u;             // packed image: hi and lo of every chunk
        const uint8_t* wbase = reinterpret_cast<const uint8_t*>(P.wpk);
        if (L.b_resident) {
          // the whole [nkc] image of the (single) N tile, once
          mbar_arrive_expect_tx(&b_full[0], (uint32_t)L.nkc * tile_bytes);
          for (int kc = 0; kc < L.nkc; ++kc)
            bulk_g2s(smem + L.off_b + (size_t)kc * tile_bytes, wbase + (size_t)kc * img_stride, tile_bytes, &b_full[0]);
        } else {
          uint32_t slot = 0, phase = 0;
          for (int item = first_item; item < n_items; item += item_stride) {
            const TmaTile t = tma_decode(L, item);
            const int ty0 = tma_first_type(L, t);
            const int ty1 = L.sel_dim >= 0 ? ty0 + 1 : L.n_types;
            for (int cc = 0; cc < L.nc; ++cc) {
              for (int ty = ty0; ty < ty1; ++ty) {
                const TmaSlabType& S = L.type[ty];
                for (int j = 0; j < S.nshift; ++j) {
                  const int kc = S.tap[j] * L.nc + cc;
                  mbar_wait(&b_empty[slot], phase ^ 1u);
                  mbar_arrive_expect_tx(&b_full[slot], tile_bytes);
                  bulk_g2s(smem + L.off_b + (size_t)slot * tile_bytes,
                           wbase + ((size_t)t.n_tile * L.nkc + kc) * img_stride, tile_bytes, &b_full[slot]);
                  if (++slot == (uint32_t)L.b_slots) { slot = 0; phase ^= 1u; }
                }
              }
            }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<kTmaMmaRegs>();
    // ===================== consumers (warps 4-11: two warpgroups of 64 rows): MMA and epilogue =====================
    const int cwarp = warp - kTmaFirstMmaWarp;               // warp index among the consumers
    const int wg = cwarp >> 2;
    const uint32_t a_row_off = (uint32_t)wg * 64u * 128u;   // this warpgroup's 64 rows of the slab window
    float acc[kBN / 2];
    uint32_t aslot = 0, aphase = 0, bslot = 0, bphase = 0;
    if (L.b_resident) mbar_wait_spin(&b_full[0], 0);
    ConvEpilogue<kBN> epi;
    for (int item = first_item; item < n_items; item += item_stride) {
      const TmaTile t = tma_decode(L, item);
      const int ty0 = tma_first_type(L, t);
      const int ty1 = L.sel_dim >= 0 ? ty0 + 1 : L.n_types;
      // ---- MMA ----
      // Stages (64-deep K chunks) in order cc, slab type, shift, one in flight while a warpgroup folds, releases and
      // waits on the next barrier (run_stages).
#pragma unroll
      for (int i = 0; i < kBN / 2; ++i) acc[i] = 0.f;
      int cc = 0, ty = ty0, j = 0;   // the next stage to issue
      // The A and weight slots a stage releases once it has completed (-1: none; an A slab is released after its last
      // shift, resident weights never).
      struct Rel {
        int a, b;
      };
      auto issue = [&](float (&t)[kBN / 2], Rel& rel) -> bool {
        if (cc == L.nc) return false;
        const TmaSlabType& S = L.type[ty];
        if (j == 0) mbar_wait_spin(&a_full[aslot], aphase);
        uint32_t sb;
        if (L.b_resident) {
          sb = b_base + (uint32_t)(S.tap[j] * L.nc + cc) * kBTileBytes;
          rel.b = -1;
        } else {
          mbar_wait_spin(&b_full[bslot], bphase);
          sb = b_base + bslot * kBTileBytes;
          rel.b = (int)bslot;
          if (++bslot == (uint32_t)L.b_slots) { bslot = 0; bphase ^= 1u; }
        }
        const uint32_t sa = a_base + aslot * (uint32_t)L.a_slot_bytes + (uint32_t)j * (uint32_t)L.shift_bytes + a_row_off;
        const uint64_t a_hi = make_smem_desc(sa, 16, 1024);
        const uint64_t b_hi = make_smem_desc(sb, 16, 1024);
        if constexpr (kLo) {
          const uint64_t a_lo = make_smem_desc(sa + (uint32_t)L.plane_stride, 16, 1024);
          const uint64_t b_lo = make_smem_desc(sb + (uint32_t)kBN * 128u, 16, 1024);
          const uint64_t ad[3] = {a_hi, a_lo, a_hi}, bd[3] = {b_lo, b_hi, b_hi};   // small products first
          wgmma_stage_issue<kBN, kBf16, 3>(t, ad, bd, 2u, 2u);
        } else {
          const uint64_t ad[3] = {a_hi, a_hi, a_hi}, bd[3] = {b_hi, b_hi, b_hi};
          wgmma_stage_issue<kBN, kBf16, 1>(t, ad, bd, 2u, 2u);
        }
        rel.a = -1;
        if (++j == S.nshift) {
          j = 0;
          rel.a = (int)aslot;
          if (++aslot == (uint32_t)L.a_slots) { aslot = 0; aphase ^= 1u; }
          if (++ty == ty1) { ty = ty0; ++cc; }
        }
        return true;
      };
      auto retire = [&](float (&t)[kBN / 2], const Rel& rel) {
        acc_fence(t);
#pragma unroll
        for (int i = 0; i < kBN / 2; ++i) acc[i] += t[i];
        // every consumer thread arrives: an arrival under `lane == 0` would be a thread-dependent branch inside the
        // wgmma pipeline, which ptxas answers by serialising every wgmma of the kernel
        if (rel.b >= 0) mbar_arrive(&b_empty[rel.b]);
        if (rel.a >= 0) mbar_arrive(&a_empty[rel.a]);   // the slab may be overwritten once every thread has read it
      };
      run_stages<kBN, Rel>(issue, retire);
      epi.tile(P, L.out, &map_out, smem_base + L.off_stage, acc, t.idx, t.n_tile);
    }
    epi.finish(P, L.out, smem + L.off_stage);
  }
}

// ------------------------------------------------------------------------------------------------
// host side: applicability, tile plan, tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

bool encode_map(CUtensorMap* m, const MapSpec& s, int which, int rank, bool swizzle) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[5], strides[4];
  cuuint32_t box[5], estr[5];
  for (int i = 0; i < 5; ++i) {
    dims[i] = s.dims[i];
    box[i] = s.box[i];
    estr[i] = 1;
  }
  for (int i = 0; i < 4; ++i) strides[i] = s.strides[i];
  const CUtensorMapDataType dt = s.elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16;
  return fn(m, dt, rank, s.base[which], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int ceil_div(int a, int b) { return (a + b - 1) / b; }
static int pymod(int a, int b) { return ((a % b) + b) % b; }

// Fills the plan and the two map specs; returns false when this launch shape stays on the cp.async kernel.
static bool conv_tma_plan_variant(const coclr_conv_t& P, int variant, TmaPlan& L, MapSpec& A, MapSpec& O) {
  const coclr_geom_t& g = P.g;
  const coclr_src_t& S = P.src;
  memset(&L, 0, sizeof(L));
  if (P.npass != 1 && P.npass != 3) return false;
  const int taps = g.kt * g.kh * g.kw;
  // K = tap * C + channel is cut into 64-wide chunks: chunks must not straddle taps (single-tap convs may end with a
  // partial chunk: the TMA unit zero-fills channels past C and the packed weights are zero past Kreal)
  // window kind (space-to-depth stem): the kw taps of one kernel row are kw CONSECUTIVE pixels of 64/kw channels each,
  // i.e. one contiguous 128-byte run -- a tensor map whose pixel stride is smaller than its 64-element inner extent
  // (overlapping rows) turns that run into one K chunk.  Needs the horizontal zero padding materialised in memory
  // (source rows are W + kw - 1 .. pixels wide, pw == 0) because a window straddles the row edge.
  const bool window = g.kt == 1 && g.kw > 1 && S.C * g.kw == 64 && S.ld == S.C && S.coff == 0 && g.pw == 0 &&
                      !g.transposed && g.st == 1 && S.W >= P.Wd + g.kw - 1 && S.H == P.Hd && S.T == P.Td;
  if (S.C % 8 != 0 || (taps > 1 && S.C % 64 != 0 && !window)) return false;
  if (P.BN % 32 != 0 || P.BN < 32 || P.BN > kTmaMaxBN || P.n_tiles < 1) return false;
  if (P.Kreal != g.kt * g.kh * g.kw * S.C) return false;
  if (g.sh != 1 || g.sw != 1) return false;
  const int planes = P.npass > 1 ? 2 : 1;
  const long ld2 = (long)S.ld * 2;
  L.out.BN = P.BN;
  L.out.N = P.N;
  L.out.n_tiles_n = P.n_tiles;
  L.nc = window ? 1 : (S.C + 63) / 64;
  L.nkc = window ? g.kh : taps * L.nc;
  L.sel_dim = -1;
  L.a_c0_step = 64;
  A.elem_bytes = 2;
  A.base[0] = (void*)((const uint16_t*)S.hi + S.coff);
  A.base[1] = S.lo ? (void*)((const uint16_t*)S.lo + S.coff) : nullptr;
  O.elem_bytes = 4;
  O.base[0] = (void*)(P.dst + P.dst_coff);
  O.base[1] = nullptr;
  const long old4 = (long)P.dst_ld * 4;
  int box[4] = {1, 1, 1, 1};     // tile extent per logical dim
  for (int d = 0; d < 4; ++d) L.ntiles[d] = 1;
  const bool tr = g.transposed != 0;

  if (g.kt == 1 && g.kh == 1 && g.kw == 1) {
    // ---- 1x1x1: a plain GEMM over the flattened pixels ----
    if (g.st != 1 || variant > 0) return false;
    if (S.T != P.Td || S.H != P.Hd || S.W != P.Wd) return false;
    const long M = (long)P.B * P.Td * P.Hd * P.Wd;
    if (M >= (1l << 31)) return false;
    box[0] = 128;
    L.ntiles[0] = ceil_div((int)M, 128);
    A.dims[0] = S.C; A.dims[1] = M; A.dims[2] = A.dims[3] = A.dims[4] = 1;
    A.strides[0] = ld2; A.strides[1] = A.strides[2] = A.strides[3] = (uint64_t)ld2 * M;
    A.box[0] = 64; A.box[1] = 128; A.box[2] = A.box[3] = A.box[4] = 1;
    O.dims[0] = P.N; O.dims[1] = M; O.dims[2] = O.dims[3] = O.dims[4] = 1;
    O.strides[0] = old4; O.strides[1] = O.strides[2] = O.strides[3] = (uint64_t)old4 * M;
    L.out.oext[0] = (int)M; L.out.oext[1] = L.out.oext[2] = L.out.oext[3] = 1;
    L.n_types = 1;
    L.type[0].nshift = 1;
    L.type[0].tap[0] = 0;
    L.slab_bytes = 128 * 128;
    L.shift_bytes = 0;
  } else if (window) {
    // ---- space-to-depth stem: (1, kh, kw) over 64/kw-channel pixels, one slab serves all kh*kw taps ----
    static const int kNw[2] = {16, 8}, kNh[2] = {8, 16};
    if (variant > 1 || g.kh > 8) return false;
    const int nw = kNw[variant], nh = kNh[variant];
    if (P.Wd % nw != 0 || P.Hd < nh) return false;
    box[0] = nw; box[1] = nh;
    L.ntiles[0] = ceil_div(P.Wd, nw); L.ntiles[1] = ceil_div(P.Hd, nh); L.ntiles[2] = S.T; L.ntiles[3] = P.B;
    A.dims[0] = 64; A.dims[1] = P.Wd; A.dims[2] = S.H; A.dims[3] = S.T; A.dims[4] = P.B;
    A.strides[0] = ld2; A.strides[1] = ld2 * S.W; A.strides[2] = ld2 * S.W * S.H; A.strides[3] = ld2 * S.W * S.H * S.T;
    A.box[0] = 64; A.box[1] = nw; A.box[2] = nh + g.kh - 1; A.box[3] = 1; A.box[4] = 1;
    O.dims[0] = P.N; O.dims[1] = P.Wd; O.dims[2] = P.Hd; O.dims[3] = P.Td; O.dims[4] = P.B;
    O.strides[0] = old4; O.strides[1] = old4 * P.Wd; O.strides[2] = old4 * P.Wd * P.Hd;
    O.strides[3] = old4 * P.Wd * P.Hd * P.Td;
    L.out.oext[0] = P.Wd; L.out.oext[1] = P.Hd; L.out.oext[2] = P.Td; L.out.oext[3] = P.B;
    L.n_types = 1;
    L.a_c0_step = 0;
    L.type[0].d[1] = -g.ph;
    L.type[0].nshift = g.kh;
    for (int j = 0; j < g.kh; ++j) L.type[0].tap[j] = j;     // K chunk ya = the kw taps of kernel row ya
    L.slab_bytes = nw * (nh + g.kh - 1) * 128;
    L.shift_bytes = nw * 128;
  } else if (g.kt == 1) {
    // ---- (1, kh, kw), stride 1: dy taps share one slab, one slab type per dx ----
    if (g.st != 1 || g.kw > 4 || g.kh > 8) return false;
    if (S.T != P.Td || S.H != P.Hd || S.W != P.Wd) return false;
    static const int kNw[3] = {16, 8, 32}, kNh[3] = {8, 16, 4};
    if (variant > 2) return false;
    const int nw = kNw[variant], nh = kNh[variant];
    if (S.W % nw != 0 || S.H < nh) return false;
    box[0] = nw; box[1] = nh;
    L.ntiles[0] = ceil_div(S.W, nw); L.ntiles[1] = ceil_div(S.H, nh); L.ntiles[2] = S.T; L.ntiles[3] = P.B;
    A.dims[0] = S.C; A.dims[1] = S.W; A.dims[2] = S.H; A.dims[3] = S.T; A.dims[4] = P.B;
    A.strides[0] = ld2; A.strides[1] = ld2 * S.W; A.strides[2] = ld2 * S.W * S.H; A.strides[3] = ld2 * S.W * S.H * S.T;
    A.box[0] = 64; A.box[1] = nw; A.box[2] = nh + g.kh - 1; A.box[3] = 1; A.box[4] = 1;
    O.dims[0] = P.N; O.dims[1] = P.Wd; O.dims[2] = P.Hd; O.dims[3] = P.Td; O.dims[4] = P.B;
    O.strides[0] = old4; O.strides[1] = old4 * P.Wd; O.strides[2] = old4 * P.Wd * P.Hd;
    O.strides[3] = old4 * P.Wd * P.Hd * P.Td;
    L.out.oext[0] = P.Wd; L.out.oext[1] = P.Hd; L.out.oext[2] = P.Td; L.out.oext[3] = P.B;
    L.n_types = g.kw;
    for (int xa = 0; xa < g.kw; ++xa) {
      TmaSlabType& t = L.type[xa];
      t.d[0] = tr ? g.pw - xa : xa - g.pw;
      t.d[1] = tr ? g.ph - (g.kh - 1) : -g.ph;
      t.nshift = g.kh;
      for (int j = 0; j < g.kh; ++j) {
        const int ya = tr ? g.kh - 1 - j : j;
        t.tap[j] = ya * g.kw + xa;
      }
    }
    L.slab_bytes = nw * (nh + g.kh - 1) * 128;
    L.shift_bytes = nw * 128;
  } else if (g.kh == 1 && g.kw == 1) {
    // ---- (kt, 1, 1): pixels of a frame are one flat dimension, dt taps share one slab ----
    if (g.kt > 8) return false;
    if (S.H != P.Hd || S.W != P.Wd) return false;
    const int HW = S.H * S.W;
    static const int kNpx[3] = {16, 8, 32}, kNt[3] = {8, 16, 4};
    if (variant > 2) return false;
    const int npx = kNpx[variant], nt = kNt[variant];
    const int t_tiles_over = (g.st == 1) ? P.Td : (tr ? P.Td / 2 : P.Td);
    if (HW % npx != 0 || 2 * t_tiles_over < nt + 1) return false;   // at most half a tile of temporal overhang
    box[0] = npx; box[2] = nt;
    const long oHW = (long)P.Hd * P.Wd;
    if (g.st == 1) {
      if (S.T != P.Td) return false;
      L.ntiles[0] = ceil_div(HW, npx); L.ntiles[2] = ceil_div(P.Td, nt); L.ntiles[3] = P.B;
      A.dims[0] = S.C; A.dims[1] = HW; A.dims[2] = 1; A.dims[3] = S.T; A.dims[4] = P.B;
      A.strides[0] = ld2; A.strides[1] = ld2 * HW; A.strides[2] = ld2 * HW; A.strides[3] = ld2 * HW * S.T;
      A.box[0] = 64; A.box[1] = npx; A.box[2] = 1; A.box[3] = nt + g.kt - 1; A.box[4] = 1;
      O.dims[0] = P.N; O.dims[1] = oHW; O.dims[2] = 1; O.dims[3] = P.Td; O.dims[4] = P.B;
      O.strides[0] = old4; O.strides[1] = old4 * oHW; O.strides[2] = old4 * oHW; O.strides[3] = old4 * oHW * P.Td;
      L.out.oext[0] = (int)oHW; L.out.oext[1] = 1; L.out.oext[2] = P.Td; L.out.oext[3] = P.B;
      L.n_types = 1;
      TmaSlabType& t = L.type[0];
      t.d[2] = tr ? g.pt - (g.kt - 1) : -g.pt;
      t.nshift = g.kt;
      for (int j = 0; j < g.kt; ++j) t.tap[j] = tr ? g.kt - 1 - j : j;
      L.slab_bytes = npx * (nt + g.kt - 1) * 128;
    } else if (g.st == 2 && !tr) {
      // forward, temporal stride 2: input frame 2*t' - pt + dt = 2*(t' + sh) + par; one slab type per frame parity
      if (S.T % 2 != 0 || (S.T + 2 * g.pt - g.kt) / 2 + 1 != P.Td) return false;
      L.ntiles[0] = ceil_div(HW, npx); L.ntiles[2] = ceil_div(P.Td, nt); L.ntiles[3] = P.B;
      int maxshift = 0;
      L.n_types = 2;
      for (int par = 0; par < 2; ++par) {
        TmaSlabType& t = L.type[par];
        t.nshift = 0;
        int sh_min = 0;
        for (int dt = 0; dt < g.kt; ++dt) {
          if (pymod(dt - g.pt, 2) != par) continue;
          const int sh = (dt - g.pt - par) / 2;   // exact
          if (t.nshift == 0) sh_min = sh;
          t.tap[t.nshift++] = dt;
        }
        if (t.nshift == 0) return false;
        t.d[1] = par;
        t.d[2] = sh_min;
        maxshift = t.nshift > maxshift ? t.nshift : maxshift;
      }
      A.dims[0] = S.C; A.dims[1] = HW; A.dims[2] = 2; A.dims[3] = S.T / 2; A.dims[4] = P.B;
      A.strides[0] = ld2; A.strides[1] = ld2 * HW; A.strides[2] = ld2 * HW * 2; A.strides[3] = ld2 * HW * S.T;
      A.box[0] = 64; A.box[1] = npx; A.box[2] = 1; A.box[3] = nt + maxshift - 1; A.box[4] = 1;
      O.dims[0] = P.N; O.dims[1] = oHW; O.dims[2] = 1; O.dims[3] = P.Td; O.dims[4] = P.B;
      O.strides[0] = old4; O.strides[1] = old4 * oHW; O.strides[2] = old4 * oHW; O.strides[3] = old4 * oHW * P.Td;
      L.out.oext[0] = (int)oHW; L.out.oext[1] = 1; L.out.oext[2] = P.Td; L.out.oext[3] = P.B;
      L.slab_bytes = npx * (nt + maxshift - 1) * 128;
    } else if (g.st == 2 && tr) {
      // data gradient of the temporally strided conv: output frame t = 2*th + par receives dY[th + sh] * W[dt] with
      // dt = par + pt - 2*sh; the frame parity of a tile selects its slab type
      if (P.Td % 2 != 0 || (P.Td + 2 * g.pt - g.kt) / 2 + 1 != S.T) return false;
      const int TH = P.Td / 2;
      L.ntiles[0] = ceil_div(HW, npx); L.ntiles[1] = 2; L.ntiles[2] = ceil_div(TH, nt); L.ntiles[3] = P.B;
      L.sel_dim = 1;
      L.n_types = 2;
      int maxshift = 0;
      for (int par = 0; par < 2; ++par) {
        TmaSlabType& t = L.type[par];
        t.nshift = 0;
        int sh_min = 0;
        for (int dt = g.kt - 1; dt >= 0; --dt) {    // descending dt = ascending sh
          if (pymod(par + g.pt - dt, 2) != 0) continue;
          const int sh = (par + g.pt - dt) / 2;     // may be negative: C division of an even number is exact
          if (t.nshift == 0) sh_min = sh;
          t.tap[t.nshift++] = dt;
        }
        if (t.nshift == 0) return false;
        t.d[2] = sh_min;
        maxshift = t.nshift > maxshift ? t.nshift : maxshift;
      }
      A.dims[0] = S.C; A.dims[1] = HW; A.dims[2] = 1; A.dims[3] = S.T; A.dims[4] = P.B;
      A.strides[0] = ld2; A.strides[1] = ld2 * HW; A.strides[2] = ld2 * HW; A.strides[3] = ld2 * HW * S.T;
      A.box[0] = 64; A.box[1] = npx; A.box[2] = 1; A.box[3] = nt + maxshift - 1; A.box[4] = 1;
      O.dims[0] = P.N; O.dims[1] = oHW; O.dims[2] = 2; O.dims[3] = TH; O.dims[4] = P.B;
      O.strides[0] = old4; O.strides[1] = old4 * oHW; O.strides[2] = old4 * oHW * 2; O.strides[3] = old4 * oHW * P.Td;
      L.out.oext[0] = (int)oHW; L.out.oext[1] = 2; L.out.oext[2] = TH; L.out.oext[3] = P.B;
      L.slab_bytes = npx * (nt + maxshift - 1) * 128;
    } else {
      return false;
    }
    L.shift_bytes = npx * 128;
  } else {
    return false;
  }
  if (L.slab_bytes / 128 > 256 * 4) return false;
  for (int d = 0; d < 4; ++d) {
    L.out.obox[d] = box[d];
    L.a_mul[d] = box[d];
    L.out.o_mul[d] = box[d];
  }
  if (L.sel_dim >= 0) {          // parity dimension: tile index = output parity coordinate, no A coordinate
    L.a_mul[L.sel_dim] = 0;
    L.out.o_mul[L.sel_dim] = 1;
  }
  if (g.st == 2 && !tr && g.kt > 1) L.a_mul[1] = 0, L.out.o_mul[1] = 0;   // A parity coordinate comes from the slab type
  long mt = 1;
  for (int d = 0; d < 4; ++d) mt *= L.ntiles[d];
  if (mt * L.out.n_tiles_n >= (1l << 31)) return false;
  L.m_tiles = (int)mt;
  L.total_tiles = (int)(mt * L.out.n_tiles_n);
  // epilogue sub-boxes: 32 consecutive tile rows form a rectangular box (all extents are powers of two)
  int sb[4], rem = 32;
  for (int d = 0; d < 4; ++d) {
    sb[d] = box[d] < rem ? box[d] : rem;
    rem /= sb[d];
  }
  if (rem != 1) return false;
  O.box[0] = 32;
  for (int d = 0; d < 4; ++d) O.box[1 + d] = sb[d];
  for (int w = 0; w < 4; ++w) {
    int r = 32 * w;
    for (int d = 0; d < 4; ++d) {
      L.out.sub[w][d] = r % box[d];
      r /= box[d];
    }
  }
  // alignment / limits of the tensor maps
  for (int i = 0; i < 2; ++i)
    if (A.base[i] && ((uintptr_t)A.base[i] & 15)) return false;
  if (planes == 2 && !A.base[1]) return false;
  if (((uintptr_t)O.base[0] & 15) || (old4 % 16) != 0 || (ld2 % 16) != 0) return false;
  for (int d = 0; d < 5; ++d)
    if (A.box[d] > 256 || O.box[d] > 256 || A.dims[d] == 0 || O.dims[d] == 0) return false;
  // ---- shared memory ----
  L.plane_stride = (L.slab_bytes + 1023) & ~1023;
  L.a_slot_bytes = planes * L.plane_stride;
  L.b_tile_bytes = planes * L.out.BN * 128;
  const int budget = 227 * 1024 - 1024 /*alignment slack*/ - kPlanKeepBytes - 256 /*barriers*/;
  const int stage1 = 4 * (int)kConvStageBytes, stage2 = 8 * (int)kConvStageBytes;
  const long tiles_per_cta = ((long)L.total_tiles + 131) / 132;   // one wave over the 132 SMs of an H100 SXM
  L.b_resident = 0;
  const long resident_bytes = (long)L.nkc * L.b_tile_bytes;
  if (L.out.n_tiles_n == 1 && tiles_per_cta >= 2 && resident_bytes + 2l * L.a_slot_bytes + stage1 <= budget) {
    L.b_resident = 1;
    L.b_slots = 0;
    long left = budget - resident_bytes;
    L.out.stage_bufs = (left - stage2 >= 2l * L.a_slot_bytes) ? 2 : 1;
    left -= L.out.stage_bufs == 2 ? stage2 : stage1;
    L.a_slots = (int)(left / L.a_slot_bytes);
    if (L.a_slots > kTmaMaxASlots) L.a_slots = kTmaMaxASlots;
    L.off_b = (uint32_t)(L.a_slots * L.a_slot_bytes);
    L.off_stage = L.off_b + (uint32_t)resident_bytes;
  } else {
    L.out.stage_bufs = 2;
    long left = budget - stage2;
    if (left < 2l * L.a_slot_bytes + 2l * L.b_tile_bytes) {
      L.out.stage_bufs = 1;
      left = budget - stage1;
      if (left < 2l * L.a_slot_bytes + 2l * L.b_tile_bytes) return false;
    }
    L.a_slots = 2;
    L.b_slots = 2;
    left -= 2l * L.a_slot_bytes + 2l * L.b_tile_bytes;
    // spend what is left on the ring whose entries are consumed faster first (weights: one per 64-deep K step)
    while (true) {
      if (L.b_slots < kTmaMaxBSlots && L.b_slots <= L.a_slots * 2 && left >= L.b_tile_bytes) {
        ++L.b_slots; left -= L.b_tile_bytes;
      } else if (L.a_slots < kTmaMaxASlots && left >= L.a_slot_bytes) {
        ++L.a_slots; left -= L.a_slot_bytes;
      } else if (L.b_slots < kTmaMaxBSlots && left >= L.b_tile_bytes) {
        ++L.b_slots; left -= L.b_tile_bytes;
      } else break;
    }
    L.off_b = (uint32_t)(L.a_slots * L.a_slot_bytes);
    L.off_stage = L.off_b + (uint32_t)(L.b_slots * L.b_tile_bytes);
  }
  L.off_stage = (L.off_stage + 1023u) & ~1023u;
  L.off_bars = L.off_stage + (uint32_t)(L.out.stage_bufs == 2 ? stage2 : stage1);
  L.total = L.off_bars + 256u + 1024u;
  if (L.total > 227u * 1024u) return false;
  if (L.out.stage_bufs == 1 && P.stats_sum != nullptr) {
    // the end-of-kernel statistics table (4 warps x 2 x 256 floats = 8 KB) lives in the staging area
    if (4 * (int)kConvStageBytes < 8192) return false;
  }
  return true;
}

// Tries the tile-shape variants of the launch's kind and keeps the best: double-buffered epilogue staging first, then
// the deeper A ring, then the smaller slab.
bool conv_tma_plan(const coclr_conv_t& P, TmaPlan& L, MapSpec& A, MapSpec& O) {
  bool have = false;
  long best = -1;
  for (int v = 0; v < 3; ++v) {
    TmaPlan l;
    MapSpec a, o;
    if (!conv_tma_plan_variant(P, v, l, a, o)) continue;
    const int slots = l.a_slots < 3 ? l.a_slots : 3;
    const long score = (long)(l.out.stage_bufs == 2) * (1l << 40) + (long)slots * (1l << 32) + ((1l << 31) - l.slab_bytes);
    if (!have || score > best) {
      have = true;
      best = score;
      L = l; A = a; O = o;
    }
  }
  return have;
}

}  // namespace coclr

using namespace coclr;

static bool g_tma_enabled = true;

extern "C" void coclr_set_conv_tma(int enabled) { g_tma_enabled = enabled != 0; }

// Debug / test entry: the tile plan this launch shape would get (no GPU needed). Returns 1 when the TMA kernel
// applies and fills info[] = {a_slots, b_slots, b_resident, stage_bufs, total smem, total tiles, slab bytes, n_types}.
extern "C" int coclr_conv_tma_plan(const coclr_conv_t* p, int* info) {
  if (!p) return 0;
  TmaPlan L;
  MapSpec A, O;
  if (!conv_tma_plan(*p, L, A, O)) return 0;
  if (info) {
    info[0] = L.a_slots; info[1] = L.b_slots; info[2] = L.b_resident; info[3] = L.out.stage_bufs;
    info[4] = (int)L.total; info[5] = L.total_tiles; info[6] = L.slab_bytes; info[7] = L.n_types;
  }
  return 1;
}

// Returns COCLR_OK when the launch was issued, 1 when this shape is not handled here (caller falls through to the
// cp.async kernel), a negative COCLR_E_* on a launch error.
int coclr::conv_tma_try(const coclr_conv_t& P, int num_sms, cudaStream_t stream) {
  if (!g_tma_enabled) return 1;
  TmaArgs args;
  MapSpec A, O;
  if (!conv_tma_plan(P, args.plan, A, O)) return 1;
  CUtensorMap m_hi, m_lo, m_out;
  if (!encode_map(&m_hi, A, 0)) return 1;
  if (P.npass > 1) {
    if (!encode_map(&m_lo, A, 1)) return 1;
  } else {
    m_lo = m_hi;
  }
  if (!encode_map(&m_out, O, 0)) return 1;
  const TmaPlan& L = args.plan;
  args.wpk = P.wpk;
  args.wunscale = P.wunscale;
  args.out_scale = P.out_scale;
  args.stats_sum = P.stats_sum;
  args.stats_sq = P.stats_sq;
  args.accumulate = P.accumulate;
  args.a_bf16 = P.a_bf16;
  args.b_bf16 = P.b_bf16;
  const int grid = L.total_tiles < num_sms ? L.total_tiles : num_sms;
  // one kernel instance per (pass count, tile width, 16-bit format): the wgmma shape and type are compile-time constants
  int rc = COCLR_E_ARG;
  with_int<1, 3>(P.npass > 1 ? 3 : 1, [&](auto np) {
    with_int<32, 64, 96, 128>(L.out.BN, [&](auto bn) {
      with_int<0, 1>(P.a_bf16 != 0, [&](auto bf) {
        rc = launch_with_smem(conv_tma_kernel<np, bn, bf != 0>, grid, kTmaThreads, L.total, stream, m_hi, m_lo, m_out,
                              args);
      });
    });
  });
  if (rc != COCLR_OK) return rc;
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}
