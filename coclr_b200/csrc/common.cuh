// Shared device helpers for the sm_90a kernels: mbarrier, bulk copy (TMA engine, 1-D),
// wgmma (fences / mma / commit / wait), shared-memory matrix descriptors and the
// 128-byte swizzle used by every operand tile in this library.
//
// Everything here is inline PTX for sm_90a; there is no fallback path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define COCLR_DEVINL __device__ __forceinline__

namespace coclr {

// ---------------------------------------------------------------------------------------------
// shared-memory addressing
// ---------------------------------------------------------------------------------------------
COCLR_DEVINL uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// Operand tiles are stored as rows of 128 bytes (64 16-bit elements of one pixel / one weight row),
// eight rows per 1024-byte swizzle atom; the 16-byte chunk index inside a row is XOR-ed with (row & 7).
// This is the canonical SWIZZLE_128B layout of wgmma shared-memory descriptors, and the same bytes
// can be read K-major (row = M/N index, 64 elements = K) or MN-major (row = K index, 64 elements = M/N).
COCLR_DEVINL uint32_t swz128_offset(uint32_t row, uint32_t chunk16) {
  return row * 128u + (((chunk16 ^ row) & 7u) << 4);
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
COCLR_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
COCLR_DEVINL void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
COCLR_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar))
               : "memory");
}
COCLR_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(
                   smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// Upper bound (ns) the hardware may keep a waiting thread suspended before try_wait returns false: waiters then do not
// spin through the issue slots that the address-generating producer warps of the same SM sub-partition need.
static constexpr uint32_t kMbarSuspendHintNs = 2000;

COCLR_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(kMbarSuspendHintNs)
      : "memory");
  return ok != 0;
}
COCLR_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// latency-critical waiter (the MMA-issuing warpgroups): default (short) suspend time
COCLR_DEVINL void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}

// generic-proxy writes (st.shared, cp.async) -> async-proxy readers (wgmma / bulk copy)
COCLR_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// 1-D bulk copy global -> shared on the TMA engine, completion on an mbarrier
// ---------------------------------------------------------------------------------------------
COCLR_DEVINL void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// 16-byte asynchronous copy global -> shared (LDGSTS); src_bytes = 0 zero-fills the destination
// (convolution padding / ragged edges) without touching global memory.
COCLR_DEVINL void cp_async16(uint32_t smem_dst, const void* gmem_src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gmem_src), "r"(src_bytes)
               : "memory");
}
// The mbarrier receives one arrival from this thread once all cp.async it has issued so far have landed
// (.noinc: the arrival is part of the barrier's expected count) -- no waiting in the producer thread.
COCLR_DEVINL void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
COCLR_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int kPending>
COCLR_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a): D[registers of one warpgroup] (+)= A[smem] * B[smem], M = 64 rows per warpgroup
// ---------------------------------------------------------------------------------------------
COCLR_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
COCLR_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
COCLR_DEVINL void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int kN>
COCLR_DEVINL void acc_fence(float (&d)[kN]) {
#pragma unroll
  for (int i = 0; i < kN; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, SWIZZLE_128B (sm_90 layout type 1).
//   K-major operand : rows = M/N index (128 B = 64 K-elements), SBO = byte stride between 8-row groups
//   MN-major operand: rows = K index   (128 B = 64 M/N elements), SBO = stride between 8-row (K) groups,
//                     LBO = stride between consecutive 64-element M/N blocks
COCLR_DEVINL uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}

// m64 x n{32,64} x k16, fp32 accumulate; kTA / kTB = 1: the operand is MN-major.  Both operands have one 16-bit
// format (fp16 or bf16).  scale_d = 0 overwrites the accumulator.
template <bool kBf16, int kTA, int kTB>
COCLR_DEVINL void wgmma_n64(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (kBf16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(kTA), "n"(kTB));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(kTA), "n"(kTB));
  }
}
template <bool kBf16, int kTA, int kTB>
COCLR_DEVINL void wgmma_n32(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (kBf16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(kTA), "n"(kTB));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(kTA), "n"(kTB));
  }
}

// One 64- (n64) or 32-column block of a warpgroup's product: t holds 32 (16) accumulator registers.
template <int kTA, int kTB>
COCLR_DEVINL void wgmma_blk(float (&t)[32], uint64_t a, uint64_t b, bool n64, bool bf16, uint32_t scale_d) {
  if (n64) {
    if (bf16) wgmma_n64<true, kTA, kTB>(t, a, b, scale_d);
    else wgmma_n64<false, kTA, kTB>(t, a, b, scale_d);
  } else {
    if (bf16) wgmma_n32<true, kTA, kTB>(t, a, b, scale_d);
    else wgmma_n32<false, kTA, kTB>(t, a, b, scale_d);
  }
}

// One pipeline stage: acc += sum over the nprod (<= 3) operand pairs (ad[p], bd[p]) of 4 K = 16 steps (descriptor
// increments a_inc / b_inc), ncols (multiple of 32) columns, b_step64 = descriptor step per 64 B columns.  Each
// 64-column block is summed by the tensor core in a fresh accumulator and added to acc with fp32 adds: long
// reductions keep fp32 accuracy.  acc[16 c + r] = row 16 (warp % 4) + lane / 4 + 8 ((r >> 1) & 1), column
// 32 c + 8 (r >> 2) + 2 (lane % 4) + (r & 1) of the warpgroup's 64 rows.
template <int kChunks, int kTA, int kTB>
COCLR_DEVINL void wgmma_stage(float (&acc)[16 * kChunks], const uint64_t (&ad)[3], const uint64_t (&bd)[3], int nprod,
                              uint32_t a_inc, uint32_t b_inc, uint32_t b_step64, int ncols, bool bf16) {
#pragma unroll
  for (int j = 0; j < kChunks / 2; ++j) {
    if (64 * j < ncols) {
      const bool n64 = 64 * j + 64 <= ncols;
      float t[32];
      wgmma_fence();
#pragma unroll
      for (int p = 0; p < 3; ++p) {
        if (p < nprod) {
#pragma unroll
          for (uint32_t k = 0; k < 4; ++k)
            wgmma_blk<kTA, kTB>(t, ad[p] + k * a_inc, bd[p] + k * b_inc + (uint64_t)j * b_step64, n64, bf16,
                                (p | (int)k) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(t);
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (n64 || i < 16) acc[32 * j + i] += t[i];
    }
  }
}

// Writes 32-column chunk c of a warpgroup's accumulator into rows [64 wg, 64 wg + 64) of a [128][pitch] fp32 tile, so
// that lane i of warp w can afterwards read row 32 w + i (the row-per-lane view the epilogues work on).
template <int kChunks>
COCLR_DEVINL void acc_chunk_to_smem(const float (&acc)[16 * kChunks], int c, float* tile, int pitch, int wg,
                                    int tid_in_wg) {
  const int row0 = 64 * wg + 16 * (tid_in_wg >> 5) + ((tid_in_wg & 31) >> 2);
  const int col0 = 2 * (tid_in_wg & 3);
#pragma unroll
  for (int cc = 0; cc < kChunks; ++cc) {
    if (cc == c) {
#pragma unroll
      for (int r = 0; r < 16; ++r)
        tile[(row0 + 8 * ((r >> 1) & 1)) * pitch + col0 + 8 * (r >> 2) + (r & 1)] = acc[16 * cc + r];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------------------------
COCLR_DEVINL float4 ldg_nc_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// One lane of a converged warp.  Unlike `lane == 0`, ptxas knows that code under an elect.sync predicate is executed by
// exactly one thread, so operands of uniform-datapath instructions issued there (cp.async.bulk.*) are moved to uniform
// registers once instead of being wrapped in a per-instruction "waterfall" loop.
COCLR_DEVINL bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

COCLR_DEVINL void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// split an fp32 value into a 16-bit (hi, lo) pair with hi + lo ~= v to ~2x the 16-bit mantissa
template <bool kBf16>
COCLR_DEVINL void split2(float v, uint16_t& hi, uint16_t& lo) {
  if constexpr (kBf16) {
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(l);
  } else {
    __half h = __float2half_rn(v);
    __half l = __float2half_rn(v - __half2float(h));
    hi = __half_as_ushort(h);
    lo = __half_as_ushort(l);
  }
}

}  // namespace coclr

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor): tiled 5-D loads / stores / add-reductions through a CUtensorMap that lives in the
// kernel's parameter space (const __grid_constant__); out-of-bounds box elements are zero-filled on load and
// clipped on store, which is what implements convolution padding and ragged tile edges here.
// ---------------------------------------------------------------------------------------------
namespace coclr {
COCLR_DEVINL void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
COCLR_DEVINL void tma_load_5d(uint32_t smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3,
                              int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, "
      "%6}], [%7];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
      : "memory");
}
COCLR_DEVINL void tma_store_5d(const void* tmap, uint32_t smem_src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
COCLR_DEVINL void tma_reduce_add_5d(const void* tmap, uint32_t smem_src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.5d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(tmap)),
      "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
COCLR_DEVINL void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory source of all but the newest kPending committed bulk groups may be overwritten
template <int kPending>
COCLR_DEVINL void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kPending) : "memory");
}
template <int kPending>
COCLR_DEVINL void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(kPending) : "memory");
}
COCLR_DEVINL void st_shared_v4(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
COCLR_DEVINL float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
COCLR_DEVINL float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
}  // namespace coclr
