// S3D-G feature gating (reference backbone/s3dg.py:68-78, applied to the four branch outputs of a SepInception,
// :125-129): out[b, c, :] = sigmoid(fc(mean_thw(a[b, :, :])))[c] * a[b, c, :].  The four branches of a block write
// slices of one channels-last concat buffer, so every kernel here works on that buffer as a whole; the four
// nn.Linear layers are the diagonal blocks (coff, n) of the fc step.  All of it is HBM-bound row streaming:
//   forward   gate_mean   planes -> mean[B, C]                       (reads 4 B / element)
//             gate_fc     mean -> gate[B, C]                          (one block per member Linear)
//             gate_apply  planes <- split(gate * (hi + lo))           (reads 4 B, writes 4 B / element, in place)
//   backward  gate_bwd_reduce  dgate[b, c] = sum_thw dout * a         (a recomputed from the raw conv output: 8 B)
//             gate_fc_bwd      dW += , dbias += , dmean =             (tiny)
//             gate_bwd_apply   dout <- gate * dout + dmean / THW      (in place; BatchNorm backward follows unchanged)
#include "common.cuh"
#include "coclr_b200.h"

namespace coclr {

namespace {

constexpr int kGateCols = 16;    // threads across channels (4 channels each: 64 channels = 128-byte plane rows)
constexpr int kGateRows = 16;    // row lanes per CTA

__device__ __forceinline__ float gh2f(uint16_t h, int bf16) {
  return bf16 ? __uint_as_float((uint32_t)h << 16) : __half2float(__ushort_as_half(h));
}

__device__ __forceinline__ float4 ld_planes4(const uint16_t* hi, const uint16_t* lo, size_t off, int bf16) {
  const uint2 h = *reinterpret_cast<const uint2*>(hi + off);
  float4 v = make_float4(gh2f((uint16_t)(h.x & 0xffff), bf16), gh2f((uint16_t)(h.x >> 16), bf16),
                         gh2f((uint16_t)(h.y & 0xffff), bf16), gh2f((uint16_t)(h.y >> 16), bf16));
  if (lo != nullptr) {
    const uint2 l = *reinterpret_cast<const uint2*>(lo + off);
    v.x += gh2f((uint16_t)(l.x & 0xffff), bf16);
    v.y += gh2f((uint16_t)(l.x >> 16), bf16);
    v.z += gh2f((uint16_t)(l.y & 0xffff), bf16);
    v.w += gh2f((uint16_t)(l.y >> 16), bf16);
  }
  return v;
}

template <bool kBf16>
__device__ __forceinline__ void st_planes4(uint16_t* hi, uint16_t* lo, size_t off, float4 v) {
  uint16_t h0, h1, h2, h3, l0, l1, l2, l3;
  split2<kBf16>(v.x, h0, l0);
  split2<kBf16>(v.y, h1, l1);
  split2<kBf16>(v.z, h2, l2);
  split2<kBf16>(v.w, h3, l3);
  *reinterpret_cast<uint2*>(hi + off) =
      make_uint2((uint32_t)h0 | ((uint32_t)h1 << 16), (uint32_t)h2 | ((uint32_t)h3 << 16));
  if (lo != nullptr)
    *reinterpret_cast<uint2*>(lo + off) =
        make_uint2((uint32_t)l0 | ((uint32_t)l1 << 16), (uint32_t)l2 | ((uint32_t)l3 << 16));
}

// sums the per-thread float4 partials of the kGateRows row lanes; row lane 0 returns the total
__device__ __forceinline__ float4 reduce_rows(float4 s, float4 (*sm)[kGateCols]) {
  const int tc = threadIdx.x % kGateCols, tr = threadIdx.x / kGateCols;
  sm[tr][tc] = s;
  __syncthreads();
  if (tr == 0) {
    for (int r = 1; r < kGateRows; ++r) {
      const float4 o = sm[r][tc];
      s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
    }
  }
  return s;
}

// grid (ceil(C / 64), B): mean over the P rows of clip b
__global__ void __launch_bounds__(kGateCols * kGateRows)
gate_mean_kernel(const uint16_t* hi, const uint16_t* lo, int bf16, int ld, int P, int C, float* mean) {
  __shared__ float4 sm[kGateRows][kGateCols];
  const int tc = threadIdx.x % kGateCols, tr = threadIdx.x / kGateCols;
  const int c = (blockIdx.x * kGateCols + tc) * 4, b = blockIdx.y;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    for (int p = tr; p < P; p += kGateRows) {
      const float4 v = ld_planes4(hi, lo, ((size_t)b * P + p) * ld + c, bf16);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  s = reduce_rows(s, sm);
  if (tr == 0 && c < C) {
    const float inv = 1.f / (float)P;
    *reinterpret_cast<float4*>(mean + (size_t)b * C + c) = make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv);
  }
}

// grid (ceil(n / 8), B), 8 warps: warp w computes output i = blockIdx.x * 8 + w of the member Linear (row i of W)
__global__ void __launch_bounds__(256)
gate_fc_kernel(const float* mean, const float* W, const float* bias, float* gate, int C, int coff, int n) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, b = blockIdx.y;
  if (i >= n) return;
  const float* m = mean + (size_t)b * C + coff;
  float acc = 0.f;
  for (int j = lane; j < n; j += 32) acc = fmaf(W[(size_t)i * n + j], m[j], acc);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) gate[(size_t)b * C + coff + i] = 1.f / (1.f + expf(-(acc + bias[i])));
}

template <bool kBf16>
__global__ void __launch_bounds__(256)
gate_apply_kernel(uint16_t* hi, uint16_t* lo, int ld, int P, int C, long total4, const float* gate) {
  const int C4 = C >> 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long r = i / C4;
    const int b = (int)(r / P);
    const float4 g = *reinterpret_cast<const float4*>(gate + (size_t)b * C + c);
    float4 v = ld_planes4(hi, lo, (size_t)r * ld + c, kBf16);
    v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
    st_planes4<kBf16>(hi, lo, (size_t)r * ld + c, v);
  }
}

// grid (ceil(C / 64), B): dgate[b, c] = sum_p dout[b, p, c] * act(y[b, p, c] * scale[c] + shift[c])
__global__ void __launch_bounds__(kGateCols * kGateRows)
gate_bwd_reduce_kernel(const float* y, int ldy, const float* scale, const float* shift, int relu, const float* dout,
                       int ldd, int P, int C, float* dgate) {
  __shared__ float4 sm[kGateRows][kGateCols];
  const int tc = threadIdx.x % kGateCols, tr = threadIdx.x / kGateCols;
  const int c = (blockIdx.x * kGateCols + tc) * 4, b = blockIdx.y;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const float4 sc = *reinterpret_cast<const float4*>(scale + c), sh = *reinterpret_cast<const float4*>(shift + c);
    for (int p = tr; p < P; p += kGateRows) {
      const size_t r = (size_t)b * P + p;
      const float4 yv = *reinterpret_cast<const float4*>(y + r * ldy + c);
      const float4 d = *reinterpret_cast<const float4*>(dout + r * ldd + c);
      float4 a = make_float4(fmaf(yv.x, sc.x, sh.x), fmaf(yv.y, sc.y, sh.y), fmaf(yv.z, sc.z, sh.z),
                             fmaf(yv.w, sc.w, sh.w));
      if (relu) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f); }
      s.x = fmaf(d.x, a.x, s.x); s.y = fmaf(d.y, a.y, s.y); s.z = fmaf(d.z, a.z, s.z); s.w = fmaf(d.w, a.w, s.w);
    }
  }
  s = reduce_rows(s, sm);
  if (tr == 0 && c < C) *reinterpret_cast<float4*>(dgate + (size_t)b * C + c) = s;
}

__device__ __forceinline__ float gate_dz(const float* dgate, const float* gate, size_t at) {
  const float g = gate[at];
  return dgate[at] * g * (1.f - g);      // d sigmoid
}

// grid (n): row i of dW (threads over j), and dbias[i]; both accumulate (+=) like every other parameter gradient
__global__ void __launch_bounds__(128)
gate_fc_bwd_w_kernel(const float* dgate, const float* gate, const float* mean, float* dW, float* dbias, int B, int C,
                     int coff, int n) {
  const int i = blockIdx.x;
  __shared__ float dz[256];
  for (int b = threadIdx.x; b < B; b += blockDim.x) dz[b] = gate_dz(dgate, gate, (size_t)b * C + coff + i);
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc = fmaf(dz[b], mean[(size_t)b * C + coff + j], acc);
    dW[(size_t)i * n + j] += acc;
  }
  if (threadIdx.x == 0) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += dz[b];
    dbias[i] += acc;
  }
}

// grid (ceil(n / 128), B): dmean[b, coff + j] = sum_i W[i, j] * dz[b, i]
__global__ void __launch_bounds__(128)
gate_fc_bwd_x_kernel(const float* dgate, const float* gate, const float* W, float* dmean, int C, int coff, int n) {
  const int j = blockIdx.x * 128 + threadIdx.x, b = blockIdx.y;
  extern __shared__ float dzs[];
  for (int i = threadIdx.x; i < n; i += blockDim.x) dzs[i] = gate_dz(dgate, gate, (size_t)b * C + coff + i);
  __syncthreads();
  if (j >= n) return;
  float acc = 0.f;
  for (int i = 0; i < n; ++i) acc = fmaf(W[(size_t)i * n + j], dzs[i], acc);
  dmean[(size_t)b * C + coff + j] = acc;
}

__global__ void __launch_bounds__(256)
gate_bwd_apply_kernel(float* dout, int ldd, const float* gate, const float* dmean, int P, int C, long total4) {
  const int C4 = C >> 2;
  const float inv = 1.f / (float)P;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long r = i / C4;
    const int b = (int)(r / P);
    const float4 g = *reinterpret_cast<const float4*>(gate + (size_t)b * C + c);
    const float4 m = *reinterpret_cast<const float4*>(dmean + (size_t)b * C + c);
    float4 d = *reinterpret_cast<float4*>(dout + (size_t)r * ldd + c);
    d.x = fmaf(g.x, d.x, m.x * inv); d.y = fmaf(g.y, d.y, m.y * inv);
    d.z = fmaf(g.z, d.z, m.z * inv); d.w = fmaf(g.w, d.w, m.w * inv);
    *reinterpret_cast<float4*>(dout + (size_t)r * ldd + c) = d;
  }
}

inline int stream_grid(long total, int threads) {
  long g = (total + threads - 1) / threads;
  const long cap = 148L * 8;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

}  // namespace coclr

using namespace coclr;

#define LAUNCH_OK() (cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH)

extern "C" int coclr_gate_mean(const void* x_hi, const void* x_lo, int bf16, int ld, int B, int P, int C, float* mean,
                               coclr_stream_t stream) {
  if (!x_hi || !mean || B <= 0 || P <= 0 || C <= 0 || C % 4 || ld % 4) return COCLR_E_ARG;
  dim3 grid((C + 4 * kGateCols - 1) / (4 * kGateCols), B);
  gate_mean_kernel<<<grid, kGateCols * kGateRows, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint16_t*>(x_hi), reinterpret_cast<const uint16_t*>(x_lo), bf16, ld, P, C, mean);
  return LAUNCH_OK();
}

extern "C" int coclr_gate_fc(const float* mean, const float* W, const float* bias, float* gate, int B, int C, int coff,
                             int n, coclr_stream_t stream) {
  if (!mean || !W || !bias || !gate || B <= 0 || n <= 0 || coff < 0 || coff + n > C) return COCLR_E_ARG;
  gate_fc_kernel<<<dim3((n + 7) / 8, B), 256, 0, (cudaStream_t)stream>>>(mean, W, bias, gate, C, coff, n);
  return LAUNCH_OK();
}

extern "C" int coclr_gate_apply(void* x_hi, void* x_lo, int bf16, int ld, int B, int P, int C, const float* gate,
                                coclr_stream_t stream) {
  if (!x_hi || !gate || B <= 0 || P <= 0 || C <= 0 || C % 4 || ld % 4) return COCLR_E_ARG;
  const long total4 = (long)B * P * (C / 4);
  uint16_t* hi = reinterpret_cast<uint16_t*>(x_hi);
  uint16_t* lo = reinterpret_cast<uint16_t*>(x_lo);
  if (bf16)
    gate_apply_kernel<true><<<stream_grid(total4, 256), 256, 0, (cudaStream_t)stream>>>(hi, lo, ld, P, C, total4, gate);
  else
    gate_apply_kernel<false><<<stream_grid(total4, 256), 256, 0, (cudaStream_t)stream>>>(hi, lo, ld, P, C, total4, gate);
  return LAUNCH_OK();
}

extern "C" int coclr_gate_bwd_reduce(const float* y, int ldy, const float* scale, const float* shift, int relu,
                                     const float* dout, int ldd, int B, int P, int C, float* dgate,
                                     coclr_stream_t stream) {
  if (!y || !scale || !shift || !dout || !dgate || B <= 0 || P <= 0 || C <= 0 || C % 4 || ldy % 4 || ldd % 4)
    return COCLR_E_ARG;
  dim3 grid((C + 4 * kGateCols - 1) / (4 * kGateCols), B);
  gate_bwd_reduce_kernel<<<grid, kGateCols * kGateRows, 0, (cudaStream_t)stream>>>(y, ldy, scale, shift, relu, dout,
                                                                                     ldd, P, C, dgate);
  return LAUNCH_OK();
}

extern "C" int coclr_gate_fc_bwd(const float* dgate, const float* gate, const float* mean, const float* W, float* dW,
                                 float* dbias, float* dmean, int B, int C, int coff, int n, coclr_stream_t stream) {
  if (!dgate || !gate || !mean || !W || !dW || !dbias || !dmean || B <= 0 || B > 256 || n <= 0 || coff < 0 ||
      coff + n > C)
    return COCLR_E_ARG;
  gate_fc_bwd_w_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(dgate, gate, mean, dW, dbias, B, C, coff, n);
  gate_fc_bwd_x_kernel<<<dim3((n + 127) / 128, B), 128, (size_t)n * sizeof(float), (cudaStream_t)stream>>>(
      dgate, gate, W, dmean, C, coff, n);
  return LAUNCH_OK();
}

extern "C" int coclr_gate_bwd_apply(float* dout, int ldd, const float* gate, const float* dmean, int B, int P, int C,
                                    coclr_stream_t stream) {
  if (!dout || !gate || !dmean || B <= 0 || P <= 0 || C <= 0 || C % 4 || ldd % 4) return COCLR_E_ARG;
  const long total4 = (long)B * P * (C / 4);
  gate_bwd_apply_kernel<<<stream_grid(total4, 256), 256, 0, (cudaStream_t)stream>>>(dout, ldd, gate, dmean, P, C,
                                                                                     total4);
  return LAUNCH_OK();
}
