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

bool encode_maps(CUtensorMap* hi, CUtensorMap* lo, const MapSpec& s, int npass) {
  if (!encode_map(hi, s, 0)) return false;
  if (npass > 1) return encode_map(lo, s, 1);
  *lo = *hi;
  return true;
}

MapSpec plane_map(const void* hi, const void* lo, int coff, int elem_bytes, int ld, int c, const int (&ext)[4],
                  const int (&box)[5], int pitch) {
  MapSpec m;
  m.base[0] = (void*)((const char*)hi + (long)coff * elem_bytes);
  m.base[1] = lo ? (void*)((const char*)lo + (long)coff * elem_bytes) : nullptr;
  m.elem_bytes = elem_bytes;
  m.dims[0] = (uint64_t)c;
  uint64_t stride = (uint64_t)ld * (uint64_t)elem_bytes;
  for (int d = 0; d < 4; ++d) {
    m.dims[1 + d] = (uint64_t)ext[d];
    m.strides[d] = stride;
    stride *= (uint64_t)(d == 0 && pitch > 0 ? pitch : ext[d]);
  }
  for (int d = 0; d < 5; ++d) m.box[d] = (uint32_t)box[d];
  return m;
}

SlabKind slab_kind(const coclr_geom_t& g, const coclr_src_t& S, int Td, int Hd, int Wd) {
  if (g.sh != 1 || g.sw != 1) return kSlabNone;
  if (g.kt == 1 && g.kh == 1 && g.kw == 1) return g.st == 1 ? kSlabFlat : kSlabNone;
  // The space-to-depth stem: the kw taps of one kernel row are kw CONSECUTIVE pixels of 64/kw channels each, i.e. one
  // contiguous 128-byte run -- a tensor map whose pixel stride is smaller than its 64-element inner extent (overlapping
  // rows) turns that run into one K chunk.  Needs the horizontal zero padding materialised in memory (source rows are
  // W + kw - 1 .. pixels wide, pw == 0) because a window straddles the row edge.
  if (g.kt == 1 && g.kw > 1 && S.C * g.kw == 64 && S.ld == S.C && S.coff == 0 && g.pw == 0 && !g.transposed &&
      g.st == 1 && S.W >= Wd + g.kw - 1 && S.H == Hd && S.T == Td)
    return kSlabWindow;
  if (g.kt == 1) return g.st == 1 ? kSlabRows : kSlabNone;
  if (g.kh == 1 && g.kw == 1) return g.st == 1 ? kSlabFrames : (g.st == 2 ? kSlabParity : kSlabNone);
  return kSlabNone;
}

int slab_types(SlabKind kind, const coclr_geom_t& g, TmaSlabType (&type)[4]) {
  memset(type, 0, sizeof(type));
  int n = 1;
  if (kind == kSlabFlat) {
    type[0].nshift = 1;
  } else if (kind == kSlabWindow || kind == kSlabRows) {
    // the window's K chunk ya is the kw taps of kernel row ya; else one type per dx, shifts dy
    n = kind == kSlabRows ? g.kw : 1;
    for (int xa = 0; xa < n; ++xa) {
      TmaSlabType& t = type[xa];
      t.d[0] = xa - g.pw;
      t.d[1] = -g.ph;
      t.nshift = g.kh;
      for (int j = 0; j < g.kh; ++j) t.tap[j] = kind == kSlabRows ? j * g.kw + xa : j;
    }
  } else if (kind == kSlabFrames) {
    type[0].d[2] = -g.pt;
    type[0].nshift = g.kt;
    for (int j = 0; j < g.kt; ++j) type[0].tap[j] = j;
  } else if (kind == kSlabParity) {
    // input frame 2 t' - pt + dt = 2 (t' + sh) + par: the taps of one parity are consecutive shifts of its frame plane
    n = 2;
    for (int par = 0; par < 2; ++par) {
      TmaSlabType& t = type[par];
      for (int dt = 0; dt < g.kt; ++dt) {
        if (pymod(dt - g.pt, 2) != par) continue;
        if (t.nshift == 0) t.d[2] = (dt - g.pt - par) / 2;   // exact
        t.tap[t.nshift++] = dt;
      }
      t.d[1] = par;
      if (t.nshift == 0) return 0;
    }
  } else {
    return 0;
  }
  if (g.transposed) {
    // data gradient: the destination pixel reads the source at -offset, so a slab starts at the mirror of the forward
    // slab's last shift and its taps come in reverse order; the frame parity is the tile's (an output coordinate)
    const int reuse_dim = kind == kSlabRows ? 1 : 2;
    for (int i = 0; i < n; ++i) {
      TmaSlabType& t = type[i];
      for (int d = 0; d < 4; ++d) t.d[d] = -t.d[d];
      t.d[reuse_dim] -= t.nshift - 1;
      if (kind == kSlabParity) t.d[1] = 0;
      for (int j = 0; j < t.nshift / 2; ++j) {
        const int tap = t.tap[j];
        t.tap[j] = t.tap[t.nshift - 1 - j];
        t.tap[t.nshift - 1 - j] = tap;
      }
    }
  }
  return n;
}

MapSpec slab_map(SlabKind kind, const coclr_geom_t& g, const coclr_src_t& S, int B, int Wd, const int (&tile)[4],
                 int reuse) {
  int box[5] = {64, tile[0], tile[1], tile[2], tile[3]};
  box[kind == kSlabWindow || kind == kSlabRows ? 2 : 3] += reuse - 1;
  const int HW = S.H * S.W;
  if (kind == kSlabFlat) return plane_map(S.hi, S.lo, S.coff, 2, S.ld, S.C, {(int)((long)B * S.T * HW), 1, 1, 1}, box);
  if (kind == kSlabWindow) return plane_map(S.hi, S.lo, S.coff, 2, S.ld, 64, {Wd, S.H, S.T, B}, box, S.W);
  if (kind == kSlabRows) return plane_map(S.hi, S.lo, S.coff, 2, S.ld, S.C, {S.W, S.H, S.T, B}, box);
  if (kind == kSlabParity && !g.transposed) return plane_map(S.hi, S.lo, S.coff, 2, S.ld, S.C, {HW, 2, S.T / 2, B}, box);
  return plane_map(S.hi, S.lo, S.coff, 2, S.ld, S.C, {HW, 1, S.T, B}, box);
}

// Fills the plan and the two map specs; returns false when this launch shape stays on the cp.async kernel.
static bool conv_tma_plan_variant(const coclr_conv_t& P, int variant, TmaPlan& L, MapSpec& A, MapSpec& O) {
  const coclr_geom_t& g = P.g;
  const coclr_src_t& S = P.src;
  memset(&L, 0, sizeof(L));
  if (P.npass != 1 && P.npass != 3) return false;
  const SlabKind kind = slab_kind(g, S, P.Td, P.Hd, P.Wd);
  const bool window = kind == kSlabWindow;
  const int taps = g.kt * g.kh * g.kw;
  // K = tap * C + channel is cut into 64-wide chunks: chunks must not straddle taps (single-tap convs may end with a
  // partial chunk: the TMA unit zero-fills channels past C and the packed weights are zero past Kreal); a window
  // chunk is the kw taps of one kernel row
  if (S.C % 8 != 0 || (taps > 1 && S.C % 64 != 0 && !window)) return false;
  if (P.BN % 32 != 0 || P.BN < 32 || P.BN > kTmaMaxBN || P.n_tiles < 1) return false;
  if (P.Kreal != taps * S.C) return false;
  const int planes = P.npass > 1 ? 2 : 1;
  L.out.BN = P.BN;
  L.out.N = P.N;
  L.out.n_tiles_n = P.n_tiles;
  L.nc = window ? 1 : (S.C + 63) / 64;
  L.nkc = window ? g.kh : taps * L.nc;
  L.sel_dim = -1;
  L.a_c0_step = window ? 0 : 64;
  int box[4] = {1, 1, 1, 1};     // tile extent per logical dim
  for (int d = 0; d < 4; ++d) L.ntiles[d] = 1;
  int* oext = L.out.oext;
  const bool tr = g.transposed != 0;
  const bool same = S.T == P.Td && S.H == P.Hd && S.W == P.Wd;

  if (kind == kSlabFlat) {
    // a plain GEMM over the flattened pixels
    if (variant > 0 || !same) return false;
    const long M = (long)P.B * P.Td * P.Hd * P.Wd;
    if (M >= (1l << 31)) return false;
    box[0] = 128;
    L.ntiles[0] = ceil_div((int)M, 128);
    oext[0] = (int)M; oext[1] = oext[2] = oext[3] = 1;
  } else if (kind == kSlabWindow || kind == kSlabRows) {
    static const int kNw[3] = {16, 8, 32}, kNh[3] = {8, 16, 4};
    if (variant > (window ? 1 : 2) || g.kh > 8 || (!window && (g.kw > 4 || !same))) return false;
    const int nw = kNw[variant], nh = kNh[variant];
    if (P.Wd % nw != 0 || P.Hd < nh) return false;
    box[0] = nw; box[1] = nh;
    L.ntiles[0] = ceil_div(P.Wd, nw); L.ntiles[1] = ceil_div(P.Hd, nh); L.ntiles[2] = P.Td; L.ntiles[3] = P.B;
    oext[0] = P.Wd; oext[1] = P.Hd; oext[2] = P.Td; oext[3] = P.B;
  } else if (kind == kSlabFrames || kind == kSlabParity) {
    static const int kNpx[3] = {16, 8, 32}, kNt[3] = {8, 16, 4};
    if (variant > 2 || g.kt > 8 || S.H != P.Hd || S.W != P.Wd) return false;
    const int HW = P.Hd * P.Wd;
    const int npx = kNpx[variant], nt = kNt[variant];
    // the data gradient of the strided conv tiles the output frames of one parity: Td / 2 of them
    const int TH = kind == kSlabParity && tr ? P.Td / 2 : P.Td;
    if (HW % npx != 0 || 2 * TH < nt + 1) return false;   // at most half a tile of temporal overhang
    if (kind == kSlabFrames && S.T != P.Td) return false;
    if (kind == kSlabParity && !tr && (S.T % 2 != 0 || (S.T + 2 * g.pt - g.kt) / 2 + 1 != P.Td)) return false;
    if (kind == kSlabParity && tr) {
      // output frame t = 2 th + par receives dY[th + sh] * W[dt] with dt = par + pt - 2 sh; the frame parity of a tile
      // selects its slab type
      if (P.Td % 2 != 0 || (P.Td + 2 * g.pt - g.kt) / 2 + 1 != S.T) return false;
      L.ntiles[1] = 2;
      L.sel_dim = 1;
    }
    box[0] = npx; box[2] = nt;
    L.ntiles[0] = ceil_div(HW, npx); L.ntiles[2] = ceil_div(TH, nt); L.ntiles[3] = P.B;
    oext[0] = HW; oext[1] = L.ntiles[1]; oext[2] = TH; oext[3] = P.B;
  } else {
    return false;
  }
  L.n_types = slab_types(kind, g, L.type);
  if (L.n_types == 0) return false;
  int reuse = 0;
  for (int i = 0; i < L.n_types; ++i) reuse = L.type[i].nshift > reuse ? L.type[i].nshift : reuse;
  A = slab_map(kind, g, S, P.B, P.Wd, box, reuse);
  L.slab_bytes = 128 * (int)(A.box[1] * A.box[2] * A.box[3] * A.box[4]);
  L.shift_bytes = kind == kSlabFlat ? 0 : 128 * box[0];   // one row of the reuse dimension (box[1] = 1 for frames)
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
  if (kind == kSlabParity && !tr) L.a_mul[1] = 0, L.out.o_mul[1] = 0;   // A parity coordinate comes from the slab type
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
  O = plane_map(P.dst, nullptr, P.dst_coff, 4, P.dst_ld, P.N, L.out.oext, {32, sb[0], sb[1], sb[2], sb[3]});
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
  if (((uintptr_t)O.base[0] & 15) || O.strides[0] % 16 != 0 || A.strides[0] % 16 != 0) return false;
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
  if (!encode_maps(&m_hi, &m_lo, A, P.npass) || !encode_map(&m_out, O, 0)) return 1;
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
