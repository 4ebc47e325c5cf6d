// Fine-tuning and test augmentation (reference eval/main_classifier.py with utils/augmentation.py under PIL):
// get_transform('train' / 'val') -- RandomSizedCrop(224, consistent) -> Scale(img_dim) [-> ColorJitter] -> ToTensor,
// the train batch's horizontal flip -- and the test views of test_10crop / test_retrieval -- flip -> FiveCrop(224) or
// CenterCrop(224) -> Scale((D, D)) -> ColorJitter -> ToTensor, bit-identical to Pillow / torchvision.
//
// One CTA per output frame; a per-frame record names the sample (its decisions and resize tables) and the source frame,
// so one launch covers a train batch, test videos of different lengths, and sources of different sizes.
//
// Stage 1 resizes the crop window (or the Scale(224) + CenterCrop(224) fallback window, or a flipped frame's window)
// to M x M with the sample's tables: a horizontal pass over a band of source rows into `band`, then the vertical pass.
// With one resize (M == D) the vertical pass writes the frame planes directly, as coclr_augment does.  With two
// (M = 224 != D, the train / val recipe) Pillow clamps to uint8 between the resizes, so the stages stay separate but
// are streamed: each band's stage-1 output rows go to `rows` and straight through stage 2's horizontal pass into
// `mid` [3][M][D]; stage 2's vertical pass then writes the frame.  Only the M x D x 3 half-resized image is held.
//
// Shared memory, two resizes:  mid [3][M][D] | max(frame [3][D][D], band [3][R][M] + rows [3][Y][M])
//                one resize:   frame [3][D][D] | band [3][R][D]
#include <cuda_runtime.h>
#include <stdint.h>

#include "augment_common.cuh"
#include "coclr_b200.h"

namespace coclr {

namespace {

using namespace aug;

__global__ void __launch_bounds__(kThreads, 2) augment_clf_kernel(coclr_augment_clf_t p) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ int red;
  const coclr_augment_clf_frame_t fm = p.frames[blockIdx.x];
  const coclr_augment_clf_sample_t& sp = p.samples[fm.sample];   // read in place: op[] and factor[] are indexed
  const int D = p.D, M = p.M, K1 = p.K1, R = p.band_rows, DD = D * D;
  const bool two = M != D;
  const int Y = two ? p.rows : M;
  uint8_t* fr = two ? smem + 3 * M * D : smem;   // [3][D][D]
  uint8_t* band = two ? fr : smem + 3 * DD;       // [3][R][M]
  uint8_t* rows = band + 3 * R * M;               // [3][Y][M], two resizes only
  uint8_t* mid = smem;                            // [3][M][D], two resizes only

  // ---- stage 1: window -> M x M (horizontal pass per band of source rows, then vertical) ----
  const int* cx = p.coef1 + (size_t)fm.sample * 2 * K1 * M;
  const int* cy = cx + (size_t)K1 * M;
  const int* x0 = p.bounds1 + (size_t)fm.sample * 4 * M;
  const int* y0 = x0 + 2 * M;
  const size_t row_bytes = (size_t)p.Wmax * 3;
  const uint8_t* src = p.src + (size_t)fm.src_frame * p.Hmax * row_bytes;
  const int step = sp.src_flip ? -3 : 3;          // a flipped frame's column c is source column src_w - 1 - c
  for (int ya = 0; ya < M;) {
    const int r0 = __ldg(y0 + ya);
    int yb = ya + 1;
    while (yb < M && yb - ya < Y && __ldg(y0 + yb) + __ldg(y0 + M + yb) - r0 <= R) ++yb;
    const int nrows = __ldg(y0 + yb - 1) + __ldg(y0 + M + yb - 1) - r0;
    for (int i = threadIdx.x; i < nrows * M; i += kThreads) {
      const int r = i / M, x = i % M;
      const int xs = __ldg(x0 + x), n = __ldg(x0 + M + x);
      const uint8_t* s = src + (size_t)(r0 + r) * row_bytes + (size_t)(sp.src_flip ? sp.src_w - 1 - xs : xs) * 3;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int k = 0; k < n; ++k) {
        const int c = __ldg(cx + k * M + x);
        a0 += (int)__ldg(s + step * k) * c;
        a1 += (int)__ldg(s + step * k + 1) * c;
        a2 += (int)__ldg(s + step * k + 2) * c;
      }
      band[r * M + x] = (uint8_t)clamp255(a0 >> kPrecisionBits);
      band[(R + r) * M + x] = (uint8_t)clamp255(a1 >> kPrecisionBits);
      band[(2 * R + r) * M + x] = (uint8_t)clamp255(a2 >> kPrecisionBits);
    }
    __syncthreads();
    uint8_t* dst = two ? rows : fr;                  // row y of the vertical pass lands at dst row (y - ya) or y
    const int dst_plane = two ? Y * M : DD, dst_row0 = two ? ya : 0;
    for (int i = threadIdx.x; i < (yb - ya) * M; i += kThreads) {
      const int y = ya + i / M, x = i % M;
      const int ys = __ldg(y0 + y) - r0, n = __ldg(y0 + M + y);
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int k = 0; k < n; ++k) {
        const int c = __ldg(cy + k * M + y);
        const int o = (ys + k) * M + x;
        a0 += (int)band[o] * c;
        a1 += (int)band[R * M + o] * c;
        a2 += (int)band[2 * R * M + o] * c;
      }
      const int o = (y - dst_row0) * M + x;
      dst[o] = (uint8_t)clamp255(a0 >> kPrecisionBits);
      dst[dst_plane + o] = (uint8_t)clamp255(a1 >> kPrecisionBits);
      dst[2 * dst_plane + o] = (uint8_t)clamp255(a2 >> kPrecisionBits);
    }
    __syncthreads();
    if (two) {   // ---- stage 2, horizontal pass of the rows just made: M -> D wide, into mid ----
      const int* bx = p.bounds2;
      for (int i = threadIdx.x; i < (yb - ya) * D; i += kThreads) {
        const int r = i / D, x = i % D;
        const int xs = __ldg(bx + x), n = __ldg(bx + D + x);
        const uint8_t* s = rows + r * M + xs;
        int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
        for (int k = 0; k < n; ++k) {
          const int c = __ldg(p.coef2 + k * D + x);
          a0 += (int)s[k] * c;
          a1 += (int)s[Y * M + k] * c;
          a2 += (int)s[2 * Y * M + k] * c;
        }
        const int o = (ya + r) * D + x;
        mid[o] = (uint8_t)clamp255(a0 >> kPrecisionBits);
        mid[M * D + o] = (uint8_t)clamp255(a1 >> kPrecisionBits);
        mid[2 * M * D + o] = (uint8_t)clamp255(a2 >> kPrecisionBits);
      }
      __syncthreads();
    }
    ya = yb;
  }

  // ---- stage 2, vertical pass: mid (M rows) -> frame (D rows); the frame overwrites band and rows ----
  if (two) {
    const int* by = p.bounds2;
    for (int i = threadIdx.x; i < DD; i += kThreads) {
      const int y = i / D, x = i % D;
      const int ys = __ldg(by + y), n = __ldg(by + D + y);
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int k = 0; k < n; ++k) {
        const int c = __ldg(p.coef2 + k * D + y);
        const int o = (ys + k) * D + x;
        a0 += (int)mid[o] * c;
        a1 += (int)mid[M * D + o] * c;
        a2 += (int)mid[2 * M * D + o] * c;
      }
      fr[i] = (uint8_t)clamp255(a0 >> kPrecisionBits);
      fr[DD + i] = (uint8_t)clamp255(a1 >> kPrecisionBits);
      fr[2 * DD + i] = (uint8_t)clamp255(a2 >> kPrecisionBits);
    }
    __syncthreads();
  }

  // ---- ColorJitter in the sample's order, then the flip and ToTensor ----
  jitter_frame(fr, DD, sp.n_ops, sp.op, sp.factor, sp.hue_shift, &red);
  store_frame(fr, p.out + fm.out, fm.chan_stride, D, sp.flip);
}

inline bool args_ok(const coclr_augment_clf_t* p) {
  if (!p || !p->src || !p->frames || !p->samples || !p->coef1 || !p->bounds1 || !p->out) return false;
  if (p->n_frames < 1 || p->NF < 1 || p->Hmax < 1 || p->Wmax < 1 || p->D < 1 || p->M < 1 || p->K1 < 1) return false;
  if (p->band_rows < p->K1) return false;
  if (p->M != p->D && (!p->coef2 || !p->bounds2 || p->K2 < 1 || p->rows < 1 || p->M < p->K2)) return false;
  return (long)coclr_augment_clf_smem_bytes(p) <= 227 * 1024;
}

}  // namespace

}  // namespace coclr

extern "C" size_t coclr_augment_clf_smem_bytes(const coclr_augment_clf_t* p) {
  const size_t D = p->D, M = p->M, R = p->band_rows;
  if (M == D) return 3 * D * D + 3 * R * D;
  const size_t staging = 3 * R * M + 3 * (size_t)p->rows * M;
  return 3 * M * D + (staging > 3 * D * D ? staging : 3 * D * D);
}

extern "C" int coclr_augment_clf(const coclr_augment_clf_t* p, coclr_stream_t stream) {
  using namespace coclr;
  if (!args_ok(p)) return COCLR_E_ARG;
  const size_t smem = coclr_augment_clf_smem_bytes(p);
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(augment_clf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return COCLR_E_LAUNCH;
  augment_clf_kernel<<<p->n_frames, aug::kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(*p);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}
