// Classifier head of LinearClassifier (reference model/classifier.py:47-61): F.normalize -> BatchNorm1d -> Dropout ->
// Linear, forward and backward, each stage optional.  The work is tiny next to the backbone (the fc is 2 * B * fs * ncls
// FLOP, ~13 MFLOP at B = 32 and 400 classes), so every kernel is plain fp32 FFMA.  Every sum runs in a fixed order
// (per-thread strided sums, then a fixed shared-memory tree, or one thread looping over the batch): no float atomics,
// so results are bit-identical from run to run.
//   forward   l2norm_fwd   one CTA per row                 xn, inv_norm
//             bn_fwd       one thread per feature column   xb, mean, rstd (+ running statistics in train mode)
//             dropout_fwd  four elements per thread        mask, xd
//             fc_fwd       one CTA per (class, row)        logits
//   backward  fc_bwd_w     one thread per weight           dW, dbias (+=)
//             fc_bwd_x     one thread per (row, feature)   dx (through the dropout mask)
//             bn_bwd       one thread per feature column   dx in place, dgamma, dbeta (+=)
//             l2norm_bwd   one CTA per row                 dfeat
#include <cuda_runtime.h>
#include <curand_kernel.h>

#include "coclr_b200.h"

namespace coclr {

namespace {

constexpr int kRowThreads = 256;
constexpr int kColThreads = 128;
constexpr float kNormEps = 1e-12f;   // F.normalize's eps

// sum of one value per thread over the CTA, in a fixed order; every thread returns the total
template <typename T, int kThreads>
__device__ __forceinline__ T block_sum(T v, T* sm) {
  sm[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  const T total = sm[0];
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(kRowThreads)
l2norm_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ inv_norm, int fs) {
  __shared__ double sm[kRowThreads];
  const float* xr = x + (size_t)blockIdx.x * fs;
  double s = 0.0;
  for (int k = threadIdx.x; k < fs; k += kRowThreads) s += (double)xr[k] * xr[k];
  s = block_sum<double, kRowThreads>(s, sm);
  const float inv = 1.f / fmaxf((float)sqrt(s), kNormEps);
  if (threadIdx.x == 0) inv_norm[blockIdx.x] = inv;
  float* yr = y + (size_t)blockIdx.x * fs;
  for (int k = threadIdx.x; k < fs; k += kRowThreads) yr[k] = xr[k] * inv;
}

__global__ void __launch_bounds__(kColThreads)
bn_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd,
              const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ rmean,
              float* __restrict__ rvar, int B, int fs, int training, float momentum, float eps) {
  const int c = blockIdx.x * kColThreads + threadIdx.x;
  if (c >= fs) return;
  float mu, rs;
  if (training) {
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += x[(size_t)b * fs + c];
    const double m = s / B;
    double q = 0.0;
    for (int b = 0; b < B; ++b) {
      const double d = x[(size_t)b * fs + c] - m;
      q += d * d;
    }
    mu = (float)m;
    rs = (float)(1.0 / sqrt(q / B + (double)eps));
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * mu;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)(q / (B - 1));
  } else {
    mu = rmean[c];
    rs = (float)(1.0 / sqrt((double)rvar[c] + (double)eps));
  }
  mean[c] = mu;
  rstd[c] = rs;
  const float g = gamma[c] * rs, sh = beta[c] - mu * g;
  for (int b = 0; b < B; ++b) y[(size_t)b * fs + c] = fmaf(x[(size_t)b * fs + c], g, sh);
}

__global__ void dropout_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ mask,
                                   long n, float keep, float scale, unsigned long long seed, unsigned long long offset) {
  const long i4 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 * 4 >= n) return;
  curandStatePhilox4_32_10_t st;
  curand_init(seed, (unsigned long long)i4, offset, &st);
  const float4 u = curand_uniform4(&st);
  const float uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long i = i4 * 4 + j;
    const bool k = uu[j] < keep;
    mask[i] = k ? 1 : 0;
    y[i] = k ? x[i] * scale : 0.f;
  }
}

// grid (ncls, B)
__global__ void __launch_bounds__(kColThreads)
fc_fwd_kernel(const float* __restrict__ h, const float* __restrict__ W, const float* __restrict__ bias,
              float* __restrict__ logits, int fs, int ncls) {
  __shared__ float sm[kColThreads];
  const int n = blockIdx.x, b = blockIdx.y;
  const float* hr = h + (size_t)b * fs;
  const float* wr = W + (size_t)n * fs;
  float s = 0.f;
  for (int k = threadIdx.x; k < fs; k += kColThreads) s = fmaf(hr[k], wr[k], s);
  s = block_sum<float, kColThreads>(s, sm);
  if (threadIdx.x == 0) logits[(size_t)b * ncls + n] = s + bias[n];
}

__global__ void fc_bwd_w_kernel(const float* __restrict__ dl, const float* __restrict__ h, float* __restrict__ dW,
                                float* __restrict__ dbias, int B, int fs, int ncls) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)ncls * fs) return;
  const int n = (int)(i / fs), k = (int)(i % fs);
  float s = 0.f;
  for (int b = 0; b < B; ++b) s = fmaf(dl[(size_t)b * ncls + n], h[(size_t)b * fs + k], s);
  dW[i] += s;
  if (k == 0) {
    float sb = 0.f;
    for (int b = 0; b < B; ++b) sb += dl[(size_t)b * ncls + n];
    dbias[n] += sb;
  }
}

__global__ void fc_bwd_x_kernel(const float* __restrict__ dl, const float* __restrict__ W,
                                const unsigned char* __restrict__ mask, float scale, float* __restrict__ dx, int B,
                                int fs, int ncls) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * fs) return;
  const int b = (int)(i / fs), k = (int)(i % fs);
  float s = 0.f;
  for (int n = 0; n < ncls; ++n) s = fmaf(dl[(size_t)b * ncls + n], W[(size_t)n * fs + k], s);
  if (mask != nullptr) s = mask[i] ? s * scale : 0.f;
  dx[i] = s;
}

__global__ void __launch_bounds__(kColThreads)
bn_bwd_kernel(const float* __restrict__ x, float* __restrict__ dx, const float* __restrict__ mean,
              const float* __restrict__ rstd, const float* __restrict__ gamma, float* __restrict__ dgamma,
              float* __restrict__ dbeta, int B, int fs, int training) {
  const int c = blockIdx.x * kColThreads + threadIdx.x;
  if (c >= fs) return;
  const float mu = mean[c], rs = rstd[c];
  float sdy = 0.f, sdyx = 0.f;
  for (int b = 0; b < B; ++b) {
    const float dy = dx[(size_t)b * fs + c];
    sdy += dy;
    sdyx = fmaf(dy, (x[(size_t)b * fs + c] - mu) * rs, sdyx);
  }
  dgamma[c] += sdyx;
  dbeta[c] += sdy;
  const float g = gamma[c] * rs;
  if (training) {
    const float a = sdy / B, q = sdyx / B;
    for (int b = 0; b < B; ++b) {
      const size_t o = (size_t)b * fs + c;
      dx[o] = g * (dx[o] - a - (x[o] - mu) * rs * q);
    }
  } else {
    for (int b = 0; b < B; ++b) dx[(size_t)b * fs + c] *= g;
  }
}

// dfeat = (dy - y (y . dy)) * inv_norm, or dy * inv_norm where the norm was clamped to eps (l2norm off: a copy)
__global__ void __launch_bounds__(kRowThreads)
l2norm_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, const float* __restrict__ inv_norm,
                  float* __restrict__ dfeat, int fs, int l2norm) {
  __shared__ double sm[kRowThreads];
  const size_t r = (size_t)blockIdx.x * fs;
  if (!l2norm) {
    for (int k = threadIdx.x; k < fs; k += kRowThreads) dfeat[r + k] = dy[r + k];
    return;
  }
  double s = 0.0;
  for (int k = threadIdx.x; k < fs; k += kRowThreads) s += (double)y[r + k] * dy[r + k];
  const float dot = (float)block_sum<double, kRowThreads>(s, sm);
  const float inv = inv_norm[blockIdx.x];
  const bool clamped = inv >= 1.f / kNormEps;
  for (int k = threadIdx.x; k < fs; k += kRowThreads)
    dfeat[r + k] = clamped ? dy[r + k] * inv : (dy[r + k] - y[r + k] * dot) * inv;
}

inline cudaStream_t S(coclr_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline int LAUNCH_OK() { return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH; }

bool head_args_ok(const coclr_cls_head_t* h) {
  if (!h || h->B <= 0 || h->fs <= 0 || h->fs % 4 || h->ncls <= 0 || !h->feat || !h->W || !h->bias) return false;
  if (h->l2norm && (!h->xn || !h->inv_norm)) return false;
  if (h->bn && (!h->xb || !h->mean || !h->rstd || !h->gamma || !h->beta || !h->running_mean || !h->running_var))
    return false;
  if (h->bn && h->bn_training && h->B < 2) return false;   // BatchNorm1d: more than one value per channel in training
  if (h->dropout && (!h->mask || !h->xd || !(h->p > 0.f) || h->p > 1.f)) return false;
  return true;
}

const float* bn_in(const coclr_cls_head_t* h) { return h->l2norm ? h->xn : h->feat; }
const float* fc_in(const coclr_cls_head_t* h) { return h->dropout ? h->xd : h->bn ? h->xb : bn_in(h); }
float keep_scale(const coclr_cls_head_t* h) { return h->p < 1.f ? 1.f / (1.f - h->p) : 0.f; }

}  // namespace

}  // namespace coclr

using namespace coclr;

extern "C" int coclr_cls_head_fwd(const coclr_cls_head_t* h, coclr_stream_t stream) {
  if (!head_args_ok(h) || !h->logits) return COCLR_E_ARG;
  const int B = h->B, fs = h->fs;
  if (h->l2norm) l2norm_fwd_kernel<<<B, kRowThreads, 0, S(stream)>>>(h->feat, h->xn, h->inv_norm, fs);
  if (h->bn)
    bn_fwd_kernel<<<(fs + kColThreads - 1) / kColThreads, kColThreads, 0, S(stream)>>>(
        bn_in(h), h->xb, h->mean, h->rstd, h->gamma, h->beta, h->running_mean, h->running_var, B, fs, h->bn_training,
        h->momentum, h->eps);
  if (h->dropout) {
    const long n4 = (long)B * fs / 4;
    dropout_fwd_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, S(stream)>>>(
        h->bn ? h->xb : bn_in(h), h->xd, h->mask, (long)B * fs, 1.f - h->p, keep_scale(h), h->seed, h->offset);
  }
  fc_fwd_kernel<<<dim3(h->ncls, B), kColThreads, 0, S(stream)>>>(fc_in(h), h->W, h->bias, h->logits, fs, h->ncls);
  return LAUNCH_OK();
}

extern "C" int coclr_cls_head_bwd(const coclr_cls_head_t* h, coclr_stream_t stream) {
  if (!head_args_ok(h) || !h->dlogits || !h->dW || !h->dbias || !h->dx) return COCLR_E_ARG;
  if (h->bn && (!h->dgamma || !h->dbeta)) return COCLR_E_ARG;
  const int B = h->B, fs = h->fs, ncls = h->ncls;
  const long nw = (long)ncls * fs, nx = (long)B * fs;
  fc_bwd_w_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, S(stream)>>>(h->dlogits, fc_in(h), h->dW, h->dbias, B, fs,
                                                                       ncls);
  const bool need_dx = h->bn || h->dfeat;
  if (need_dx)
    fc_bwd_x_kernel<<<(unsigned)((nx + 255) / 256), 256, 0, S(stream)>>>(
        h->dlogits, h->W, h->dropout ? h->mask : nullptr, keep_scale(h), h->dx, B, fs, ncls);
  if (h->bn)
    bn_bwd_kernel<<<(fs + kColThreads - 1) / kColThreads, kColThreads, 0, S(stream)>>>(
        bn_in(h), h->dx, h->mean, h->rstd, h->gamma, h->dgamma, h->dbeta, B, fs, h->bn_training);
  if (h->dfeat) l2norm_bwd_kernel<<<B, kRowThreads, 0, S(stream)>>>(h->xn, h->dx, h->inv_norm, h->dfeat, fs, h->l2norm);
  return LAUNCH_OK();
}
