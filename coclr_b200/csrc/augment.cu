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

#include "coclr_b200.h"

namespace coclr {

namespace {

constexpr int kThreads = 512;
constexpr int kPrecisionBits = 22;   // Resample.c

enum { kBrightness = 0, kContrast = 1, kSaturation = 2, kHue = 3 };

__device__ __forceinline__ int clamp255(int v) { return min(max(v, 0), 255); }

__device__ __forceinline__ int luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// Blend.c: float(d + alpha * (x - d)), truncated, clamped
__device__ __forceinline__ int blend(int d, int x, float alpha) {
  const float t = __fadd_rn((float)d, __fmul_rn(alpha, (float)(x - d)));
  return t <= 0.f ? 0 : (t >= 255.f ? 255 : __float2int_rz(t));
}

// Convert.c rgb2hsv_row: H and S bytes (V = max)
__device__ __forceinline__ void rgb_to_hs(int r, int g, int b, int& uh, int& us) {
  const int mx = max(r, max(g, b)), mn = min(r, min(g, b));
  if (mx == mn) {
    uh = us = 0;
    return;
  }
  const float cr = (float)(mx - mn);
  const float s = __fdiv_rn(cr, (float)mx);
  const float rc = __fdiv_rn((float)(mx - r), cr), gc = __fdiv_rn((float)(mx - g), cr),
              bc = __fdiv_rn((float)(mx - b), cr);
  float h;
  if (r == mx)
    h = __fsub_rn(bc, gc);
  else if (g == mx)
    h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc));
  else
    h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc));
  h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn((double)h, 6.0), 1.0), 1.0));
  uh = clamp255(__double2int_rz(__dmul_rn((double)h, 255.0)));
  us = clamp255(__double2int_rz(__dmul_rn((double)s, 255.0)));
}

// Convert.c hsv2rgb
__device__ __forceinline__ void hsv_to_rgb(int h, int s, int v, int& r, int& g, int& b) {
  if (s == 0) {
    r = g = b = v;
    return;
  }
  const double hh = __ddiv_rn(__dmul_rn((double)h, 6.0), 255.0);
  const int i = (int)floor(hh);
  const float f = __double2float_rn(__dsub_rn(hh, (double)(float)i));
  const float fs = __double2float_rn(__ddiv_rn((double)s, 255.0));
  const double vf = (double)v;
  const int p = clamp255((int)round(__dmul_rn(vf, __dsub_rn(1.0, (double)fs))));
  const int q = clamp255((int)round(__dmul_rn(vf, __dsub_rn(1.0, (double)__fmul_rn(fs, f)))));
  const int t = clamp255((int)round(__dmul_rn(vf, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f))))));
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// Sum over the CTA of one int per thread (exact; integer atomics on shared memory are order-independent).
__device__ __forceinline__ int block_sum(int v, int* acc) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (threadIdx.x == 0) *acc = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicAdd(acc, v);
  __syncthreads();
  const int total = *acc;
  __syncthreads();
  return total;
}

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
  for (int o = 0; o < cp.n_ops; ++o) {
    const int op = __ldg(cp.op + o);
    int mean = 0;
    if (op == kContrast) {
      int s = 0;
      for (int i = threadIdx.x; i < DD; i += kThreads) s += luma(fr[i], fr[DD + i], fr[2 * DD + i]);
      const int total = block_sum(s, &red);
      mean = (2 * total + DD) / (2 * DD);   // int(mean(L) + 0.5)
    }
    const float f = op == kHue ? 0.f : __ldg(cp.factor + op);
    for (int i = threadIdx.x; i < DD; i += kThreads) {
      int r = fr[i], g = fr[DD + i], bl = fr[2 * DD + i];
      if (op == kBrightness) {
        r = blend(0, r, f); g = blend(0, g, f); bl = blend(0, bl, f);
      } else if (op == kContrast) {
        r = blend(mean, r, f); g = blend(mean, g, f); bl = blend(mean, bl, f);
      } else if (op == kSaturation) {
        const int l = luma(r, g, bl);
        r = blend(l, r, f); g = blend(l, g, f); bl = blend(l, bl, f);
      } else {
        int h, s;
        rgb_to_hs(r, g, bl, h, s);
        hsv_to_rgb((h + cp.hue_shift) & 255, s, max(r, max(g, bl)), r, g, bl);
      }
      fr[i] = (uint8_t)r; fr[DD + i] = (uint8_t)g; fr[2 * DD + i] = (uint8_t)bl;
    }
    __syncthreads();
  }

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
  float* out = p.out + (size_t)b * p.out_batch_stride + (size_t)clip * p.out_clip_stride + (size_t)j * DD;
  for (int i = threadIdx.x; i < 3 * DD; i += kThreads) {
    const int c = i / DD, y = (i / D) % D, x = i % D;
    const int xs = cp.flip ? D - 1 - x : x;
    out[(size_t)c * p.out_chan_stride + y * D + x] = __fdiv_rn((float)fr[c * DD + y * D + xs], 255.f);
  }
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
