// Device code shared by the augmentation kernels (augment.cu: pre-training, augment_clf.cu: fine-tuning and test):
// Pillow's ImageEnhance blends and Convert.c RGB <-> HSV as explicitly rounded intrinsics (so nvcc cannot contract
// them into FMAs), the ColorJitter chain on a frame of three uint8 planes in shared memory, and the flipped ToTensor
// store.  Every function assumes a CTA of kThreads threads.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace coclr {
namespace aug {

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

// ColorJitter: the ImageEnhance blends and adjust_hue of `n_ops` ops (op[], global memory) in order, in place on the
// planes fr [3][DD].  factor[] holds the float32 blend factors of brightness, contrast, saturation by op code.
__device__ __forceinline__ void jitter_frame(uint8_t* fr, int DD, int n_ops, const int* op_list, const float* factor,
                                             int hue_shift, int* red) {
  for (int o = 0; o < n_ops; ++o) {
    const int op = __ldg(op_list + o);
    int mean = 0;
    if (op == kContrast) {
      int s = 0;
      for (int i = threadIdx.x; i < DD; i += kThreads) s += luma(fr[i], fr[DD + i], fr[2 * DD + i]);
      const int total = block_sum(s, red);
      mean = (2 * total + DD) / (2 * DD);   // int(mean(L) + 0.5)
    }
    const float f = op == kHue ? 0.f : __ldg(factor + op);
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
        hsv_to_rgb((h + hue_shift) & 255, s, max(r, max(g, bl)), r, g, bl);
      }
      fr[i] = (uint8_t)r; fr[DD + i] = (uint8_t)g; fr[2 * DD + i] = (uint8_t)bl;
    }
    __syncthreads();
  }
}

// Horizontal flip + ToTensor (x / 255 in float32, rounded as torch's div): planes fr [3][D][D] to out, channel c at
// out + c * chan_stride, rows of D floats.
__device__ __forceinline__ void store_frame(const uint8_t* fr, float* out, long chan_stride, int D, bool flip) {
  const int DD = D * D;
  for (int i = threadIdx.x; i < 3 * DD; i += kThreads) {
    const int c = i / DD, y = (i / D) % D, x = i % D;
    const int xs = flip ? D - 1 - x : x;
    out[(size_t)c * chan_stride + y * D + x] = __fdiv_rn((float)fr[c * DD + y * D + xs], 255.f);
  }
}

}  // namespace aug
}  // namespace coclr
