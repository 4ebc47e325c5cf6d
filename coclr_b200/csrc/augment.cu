// Pre-training augmentation (reference utils/augmentation.py under PIL, get_transform('train') of main_nce.py and
// main_coclr.py): crop + bicubic resize, ColorJitter (brightness, contrast, saturation, hue in a per-clip order),
// RandomGray, GaussianBlur, horizontal flip and ToTensor, bit-identical to Pillow / torchvision.
//
// One CTA per output frame.  The frame lives in shared memory as three uint8 planes [3][D][D]; a second region of
// band_rows x D x 3 bytes holds the horizontal resize pass of a band of source rows (as many as the vertical taps of
// consecutive output rows need, so sources of any height work) and later the ping-pong plane of the blur.
//
// Every value that Pillow computes in double for a whole image (bicubic coefficients, box-blur radius and weights) comes
// precomputed from the host (coclr_b200/augment.py).  What remains per pixel is integer arithmetic (resize, luma,
// contrast mean, box blur) and Pillow's float / double expressions (blend, RGB <-> HSV), written with explicitly
// rounded intrinsics so that nvcc cannot contract them into FMAs.
#include <cuda_runtime.h>
#include <stdint.h>

#include "augment_common.cuh"
#include "coclr_b200.h"

namespace coclr {

namespace {

using namespace aug;

// One BoxBlur.c line pass (clamped edges) from `in` to `out`, planes [3][D][D]; along x (step 1) or y (step D).
__device__ __forceinline__ void box_pass(const uint8_t* in, uint8_t* out, int D, int r, unsigned ww, unsigned fw,
                                         bool vertical) {
  const int n = 3 * D * D;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const int x = i % D, y = (i / D) % D;
    const int pos = vertical ? y : x;
    const int step = vertical ? D : 1;
    const uint8_t* line = in + i - pos * step;
    unsigned s = 0;
    for (int o = -r; o <= r; ++o) s += line[min(max(pos + o, 0), D - 1) * step];
    const unsigned far = (unsigned)line[max(pos - r - 1, 0) * step] + line[min(pos + r + 1, D - 1) * step];
    out[i] = (uint8_t)((ww * s + fw * far + (1u << 23)) >> 24);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 2) augment_kernel(coclr_augment_t p) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ int red;
  const int D = p.D, S = p.S, K = p.K, R = p.band_rows, DD = D * D;
  const int b = blockIdx.y, fo = blockIdx.x, clip = fo / S, j = fo % S;
  const int ci = b * 2 + clip;
  const coclr_augment_clip_t& cp = p.clips[ci];   // read in place: op[] and factor[] are indexed at run time
  uint8_t* fr = smem;                 // [3][D][D]
  uint8_t* band = smem + 3 * DD;      // [3][R][D], later [3][D][D]

  // ---- crop + bicubic resize: horizontal pass into the band, vertical pass into the frame ----
  const int* cx = p.coef + (size_t)(ci * 2 + 0) * K * D;
  const int* cy = p.coef + (size_t)(ci * 2 + 1) * K * D;
  const int* x0 = p.bounds + (size_t)(ci * 2 + 0) * 2 * D;
  const int* y0 = p.bounds + (size_t)(ci * 2 + 1) * 2 * D;
  const size_t row_bytes = (size_t)p.Wmax * 3;
  const uint8_t* src = p.src + ((size_t)b * p.F + cp.src_frame + j) * p.Hmax * row_bytes;
  for (int ya = 0; ya < D;) {
    const int r0 = __ldg(y0 + ya);
    int yb = ya + 1;
    while (yb < D && __ldg(y0 + yb) + __ldg(y0 + D + yb) - r0 <= R) ++yb;
    const int rows = __ldg(y0 + yb - 1) + __ldg(y0 + D + yb - 1) - r0;
    for (int i = threadIdx.x; i < rows * D; i += kThreads) {
      const int r = i / D, x = i % D;
      const int xs = __ldg(x0 + x), n = __ldg(x0 + D + x);
      const uint8_t* s = src + (size_t)(r0 + r) * row_bytes + (size_t)xs * 3;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int k = 0; k < n; ++k) {
        const int c = __ldg(cx + k * D + x);
        a0 += (int)__ldg(s + 3 * k) * c;
        a1 += (int)__ldg(s + 3 * k + 1) * c;
        a2 += (int)__ldg(s + 3 * k + 2) * c;
      }
      band[r * D + x] = (uint8_t)clamp255(a0 >> kPrecisionBits);
      band[(R + r) * D + x] = (uint8_t)clamp255(a1 >> kPrecisionBits);
      band[(2 * R + r) * D + x] = (uint8_t)clamp255(a2 >> kPrecisionBits);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (yb - ya) * D; i += kThreads) {
      const int y = ya + i / D, x = i % D;
      const int ys = __ldg(y0 + y) - r0, n = __ldg(y0 + D + y);
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int k = 0; k < n; ++k) {
        const int c = __ldg(cy + k * D + y);
        const int o = (ys + k) * D + x;
        a0 += (int)band[o] * c;
        a1 += (int)band[R * D + o] * c;
        a2 += (int)band[2 * R * D + o] * c;
      }
      fr[y * D + x] = (uint8_t)clamp255(a0 >> kPrecisionBits);
      fr[DD + y * D + x] = (uint8_t)clamp255(a1 >> kPrecisionBits);
      fr[2 * DD + y * D + x] = (uint8_t)clamp255(a2 >> kPrecisionBits);
    }
    __syncthreads();
    ya = yb;
  }

  // ---- ColorJitter: ImageEnhance blends and adjust_hue, in the clip's order ----
  jitter_frame(fr, DD, cp.n_ops, cp.op, cp.factor, cp.hue_shift, &red);

  // ---- RandomGray: one channel per frame replicated ----
  const int gch = p.gray[(size_t)ci * S + j];
  if (gch >= 0) {
    for (int i = threadIdx.x; i < DD; i += kThreads) {
      const uint8_t v = fr[gch * DD + i];
      fr[i] = v; fr[DD + i] = v; fr[2 * DD + i] = v;
    }
    __syncthreads();
  }

  // ---- GaussianBlur: three horizontal, then three vertical extended-box passes ----
  if (cp.blur_radius >= 0) {
    const int r = cp.blur_radius;
    box_pass(fr, band, D, r, cp.blur_ww, cp.blur_fw, false);
    box_pass(band, fr, D, r, cp.blur_ww, cp.blur_fw, false);
    box_pass(fr, band, D, r, cp.blur_ww, cp.blur_fw, false);
    box_pass(band, fr, D, r, cp.blur_ww, cp.blur_fw, true);
    box_pass(fr, band, D, r, cp.blur_ww, cp.blur_fw, true);
    box_pass(band, fr, D, r, cp.blur_ww, cp.blur_fw, true);
  }

  // ---- flip + ToTensor (x / 255 in float32, rounded as torch's div) ----
  store_frame(fr, p.out + (size_t)b * p.out_batch_stride + (size_t)clip * p.out_clip_stride + (size_t)j * DD,
              p.out_chan_stride, D, cp.flip);
}

inline bool args_ok(const coclr_augment_t* p) {
  if (!p || !p->src || !p->clips || !p->coef || !p->bounds || !p->gray || !p->out) return false;
  if (p->B < 1 || p->S < 1 || p->F < 2 * p->S || p->D < 1 || p->K < 1 || p->Hmax < 1 || p->Wmax < 1) return false;
  if (p->band_rows < p->D || p->band_rows < p->K) return false;
  return (long)coclr_augment_smem_bytes(p) <= 227 * 1024;
}

}  // namespace

}  // namespace coclr

extern "C" size_t coclr_augment_smem_bytes(const coclr_augment_t* p) {
  return (size_t)3 * p->D * p->D + (size_t)3 * p->D * p->band_rows;
}

extern "C" int coclr_augment(const coclr_augment_t* p, coclr_stream_t stream) {
  using namespace coclr;
  if (!args_ok(p)) return COCLR_E_ARG;
  const size_t smem = coclr_augment_smem_bytes(p);
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(augment_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return COCLR_E_LAUNCH;
  augment_kernel<<<dim3(2 * p->S, p->B), kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(*p);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}
