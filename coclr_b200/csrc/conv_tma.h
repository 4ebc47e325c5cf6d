// Tile plan of the TMA-staged convolution kernel (conv_tma.cu), shared between the host planner and the kernel.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "coclr_b200.h"

namespace coclr {

// One TMA slab load: coordinate offsets (logical dims 1..4 of the tensor map) relative to the tile origin, and the
// taps it serves -- shift j reads the slab at row offset j * shift_rows and multiplies with packed K chunk
// tap[j] * nc + channel_chunk.
struct TmaSlabType {
  int d[4];
  int nshift;
  int tap[8];
};

struct TmaPlan {
  int ntiles[4];       // tiles per logical dim (dim 0 fastest)
  int a_mul[4];        // tile index -> A-map coordinate
  int o_mul[4];        // tile index -> output-map coordinate
  int obox[4];         // tile extent per dim (rows are in this box order)
  int oext[4];         // output extent per dim (edge rows are excluded from the statistics)
  int n_tiles_n, m_tiles, total_tiles;
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
  int stage_bufs;
  int dbg;             // tuning experiments only (COCLR_TMA_DBG bit mask; 0 in production)
  int sub[4][4];       // output coordinate offsets of each epilogue warp's 32-row sub-box
  int BN, N;
  uint32_t off_b, off_stage, off_misc, off_bars, total;
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

// TMA-staged weight gradient (wgrad_tma.cu): 0 = launched, < 0 = error, 1 = shape not covered (caller falls back)
int wgrad_tma_try(const coclr_wgrad_t& P, cudaStream_t stream);

}  // namespace coclr
