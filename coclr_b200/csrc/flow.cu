// Batched TV-L1 optical flow (coclr_b200.h, coclr_flow_* / coclr_tvl1*): Pillow's grey conversion, the Gaussian +
// bicubic pyramid, bicubic warping and the duality-based primal-dual iterations of Zach, Pock and Bischof in the form
// of Sanchez Perez, Meinhardt-Llopis and Facciolo (IPOL 2013), and the 8-bit quantisation of the flow frames.
//
// Every plane is fp32 [P, H, W] (flow: [P, 2, H, W]); every kernel covers all P pairs of a solve in one launch
// (blockIdx.z is the pair).  One primal-dual iteration is two launches: the u-step (thresholding + u = v + theta div p,
// per-CTA partial sums of |u' - u|^2) and the p-step (dual update; CTA (0, 0) of each pair also sums that pair's
// partials in a fixed order and decides whether it has converged).  A converged pair is frozen: both kernels return at
// once for it, so its u and p do not depend on how often the host looks at the flags.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "coclr_b200.h"

namespace coclr {
namespace {

constexpr double kEta = 0.5;          // zoom factor between pyramid levels
constexpr int kMinSide = 16;          // the coarsest level's short side stays >= this
constexpr float kLambda = 0.15f, kTheta = 0.3f, kTau = 0.25f;
constexpr float kEpsilon = 0.01f;     // stopping threshold on the mean |u^{n+1} - u^n|^2 is kEpsilon^2
constexpr float kGradZero = 1e-10f;
constexpr int kRadius = 4;            // ceil(3 sigma) of the pyramid's Gaussian, sigma = 0.6 sqrt(eta^-2 - 1)
constexpr int kTx = 32, kTy = 8;      // CTA tile of every pixel kernel: one pixel per thread
constexpr int kThreads = kTx * kTy;

struct Taps {
  float w[2 * kRadius + 1];
};

dim3 grid_of(int H, int W, int planes) { return dim3((W + kTx - 1) / kTx, (H + kTy - 1) / kTy, planes); }

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Keys' cubic convolution kernel with a = -0.5: weights of the neighbours -1, 0, 1, 2 at fractional offset t
__device__ __forceinline__ void keys_weights(float t, float w[4]) {
  const float t2 = t * t, t3 = t2 * t;
  w[0] = -0.5f * t3 + t2 - 0.5f * t;
  w[1] = 1.5f * t3 - 2.5f * t2 + 1.0f;
  w[2] = -1.5f * t3 + 2.0f * t2 + 0.5f * t;
  w[3] = 0.5f * t3 - 0.5f * t2;
}

// Bicubic sampling stencil at (sx, sy) of an H x W plane, neighbour indices clamped to the image.  A position far
// outside the image reads its edge whatever its distance, so it is clamped first to keep floorf's result an int.
struct Stencil {
  int off[4][4];
  float wx[4], wy[4];
};

__device__ __forceinline__ void make_stencil(float sx, float sy, int H, int W, Stencil& s) {
  sx = fminf(fmaxf(sx, -2.0f), (float)W + 1.0f);
  sy = fminf(fmaxf(sy, -2.0f), (float)H + 1.0f);
  const float fx = floorf(sx), fy = floorf(sy);
  keys_weights(sx - fx, s.wx);
  keys_weights(sy - fy, s.wy);
  const int x0 = (int)fx, y0 = (int)fy;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int row = clampi(y0 - 1 + j, 0, H - 1) * W;
#pragma unroll
    for (int i = 0; i < 4; ++i) s.off[j][i] = row + clampi(x0 - 1 + i, 0, W - 1);
  }
}

__device__ __forceinline__ float sample(const float* __restrict__ plane, const Stencil& s) {
  float acc = 0.0f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float row = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i) row += s.wx[i] * plane[s.off[j][i]];
    acc += s.wy[j] * row;
  }
  return acc;
}

// Deterministic CTA sum (fixed shuffle pattern, then the warps' sums in warp order); the result is valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* smem) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  float s = 0.0f;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += smem[w];
  return s;
}

// ---------------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------------

__global__ void grey_kernel(const uint8_t* __restrict__ rgb, int H, int W, int64_t frame_stride, int64_t row_stride,
                            float* __restrict__ out) {
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x >= W || y >= H) return;
  const uint8_t* px = rgb + blockIdx.z * frame_stride + y * row_stride + 3 * x;
  const uint32_t l = (19595u * px[0] + 38470u * px[1] + 7471u * px[2] + 0x8000u) >> 16;   // Pillow's convert('L')
  out[((int64_t)blockIdx.z * H + y) * W + x] = (float)l;
}

// one pass of the separable Gaussian, clamp-to-edge: along rows (along_x = 1) or columns (0)
__global__ void blur_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, Taps taps, int along_x) {
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x >= W || y >= H) return;
  const float* src = in + (int64_t)blockIdx.z * H * W;
  float acc = 0.0f;
#pragma unroll
  for (int k = -kRadius; k <= kRadius; ++k) {
    const float v = along_x ? src[y * W + clampi(x + k, 0, W - 1)] : src[clampi(y + k, 0, H - 1) * W + x];
    acc += taps.w[k + kRadius] * v;
  }
  out[((int64_t)blockIdx.z * H + y) * W + x] = acc;
}

// out pixel (x, y) of component c of item z = scale_c * bicubic(in component c of item z, x * sx, y * sy): the pyramid's
// zoom-out (comps 1, scale 1) and the flow's zoom-in (comps 2, scales W_f / W_c and H_f / H_c).  Items are
// [comps, Hi, Wi] in and [comps, Ho, Wo] out; the components share one stencil.
__global__ void resample_kernel(const float* __restrict__ in, int Hi, int Wi, float* __restrict__ out, int Ho, int Wo,
                                float sx, float sy, int comps, float scale0, float scale1) {
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x >= Wo || y >= Ho) return;
  Stencil s;
  make_stencil((float)x * sx, (float)y * sy, Hi, Wi, s);
  for (int c = 0; c < comps; ++c) {
    const int64_t plane = (int64_t)blockIdx.z * comps + c;
    out[(plane * Ho + y) * Wo + x] = (c ? scale1 : scale0) * sample(in + plane * Hi * Wi, s);
  }
}

// centred differences with clamp-to-edge: 0.5 (I(x + 1) - I(x - 1))
__global__ void gradient_kernel(const float* __restrict__ in, float* __restrict__ gx, float* __restrict__ gy, int H,
                                int W) {
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x >= W || y >= H) return;
  const float* src = in + (int64_t)blockIdx.z * H * W;
  const int64_t o = ((int64_t)blockIdx.z * H + y) * W + x;
  gx[o] = 0.5f * (src[y * W + min(x + 1, W - 1)] - src[y * W + max(x - 1, 0)]);
  gy[o] = 0.5f * (src[min(y + 1, H - 1) * W + x] - src[max(y - 1, 0) * W + x]);
}

struct WarpArgs {
  const float *i0, *i1, *i1x, *i1y, *u;
  float *wx, *wy, *g, *rhoc;
  int H, W;
};

// I1, I1x and I1y warped at x + u; g = |grad I1w|^2, rho_c = I1w - grad I1w . u - I0
__global__ void warp_kernel(WarpArgs a) {
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x >= a.W || y >= a.H) return;
  const int64_t plane = (int64_t)a.H * a.W, base = blockIdx.z * plane, o = base + y * a.W + x;
  const float u1 = a.u[2 * base + y * a.W + x], u2 = a.u[2 * base + plane + y * a.W + x];
  Stencil s;
  make_stencil((float)x + u1, (float)y + u2, a.H, a.W, s);
  const float iw = sample(a.i1 + base, s), wx = sample(a.i1x + base, s), wy = sample(a.i1y + base, s);
  a.wx[o] = wx;
  a.wy[o] = wy;
  a.g[o] = wx * wx + wy * wy;
  a.rhoc[o] = iw - wx * u1 - wy * u2 - a.i0[o];
}

struct IterArgs {
  const float *wx, *wy, *g, *rhoc;
  float* u;            // [P, 2, H, W]
  float* p;            // [P, 4, H, W]: p11 p12 (dual of u1), p21 p22 (dual of u2)
  float* partial;      // [P, blocks]
  int* done;           // [P]: 1 once the pair has converged or run out of iterations
  int* active;         // [P]: the pair was iterated in this iteration's u-step
  int* iters;          // [P]: iterations of the current warp
  int H, W, blocks;
};

// backward-difference divergence matching the forward gradient: p(-1) = 0, the last column / row contributes -p(x-1)
__device__ __forceinline__ float divergence(const float* __restrict__ px, const float* __restrict__ py, int x, int y,
                                            int H, int W) {
  const int o = y * W + x;
  const float dx = (x == 0) ? px[o] : (x == W - 1) ? -px[o - 1] : px[o] - px[o - 1];
  const float dy = (y == 0) ? py[o] : (y == H - 1) ? -py[o - W] : py[o] - py[o - W];
  return dx + dy;
}

__global__ void __launch_bounds__(kThreads) tvl1_u_kernel(IterArgs a) {
  __shared__ float red[kThreads / 32];
  const int k = blockIdx.z;
  const bool first = blockIdx.x == 0 && blockIdx.y == 0;
  if (a.done[k]) {
    if (first && threadIdx.x == 0) a.active[k] = 0;
    return;
  }
  if (first && threadIdx.x == 0) a.active[k] = 1;
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  float err = 0.0f;
  if (x < a.W && y < a.H) {
    const int64_t plane = (int64_t)a.H * a.W, o = (int64_t)k * plane + y * a.W + x;
    float* u1p = a.u + 2 * k * plane + y * a.W + x;
    float* u2p = u1p + plane;
    const float* p = a.p + 4 * k * plane;
    const float u1 = *u1p, u2 = *u2p;
    const float wx = a.wx[o], wy = a.wy[o], g = a.g[o];
    const float rho = a.rhoc[o] + (wx * u1 + wy * u2);
    const float lt = kLambda * kTheta;
    float d1, d2;
    if (rho < -lt * g) {
      d1 = lt * wx;
      d2 = lt * wy;
    } else if (rho > lt * g) {
      d1 = -lt * wx;
      d2 = -lt * wy;
    } else if (g > kGradZero) {
      const float f = -rho / g;
      d1 = f * wx;
      d2 = f * wy;
    } else {
      d1 = d2 = 0.0f;
    }
    const float n1 = (u1 + d1) + kTheta * divergence(p, p + plane, x, y, a.H, a.W);
    const float n2 = (u2 + d2) + kTheta * divergence(p + 2 * plane, p + 3 * plane, x, y, a.H, a.W);
    *u1p = n1;
    *u2p = n2;
    err = (n1 - u1) * (n1 - u1) + (n2 - u2) * (n2 - u2);
  }
  const float s = block_sum(err, red);
  if (threadIdx.x == 0) a.partial[(int64_t)k * a.blocks + blockIdx.y * gridDim.x + blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) tvl1_p_kernel(IterArgs a) {
  __shared__ float red[kThreads / 32];
  const int k = blockIdx.z;
  if (!a.active[k]) return;
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x < a.W && y < a.H) {
    const int64_t plane = (int64_t)a.H * a.W;
    const int o = y * a.W + x;
    const float* u1 = a.u + 2 * k * plane;
    const float* u2 = u1 + plane;
    float* p = a.p + 4 * k * plane + o;
    const bool rx = x < a.W - 1, ry = y < a.H - 1;
    const float u1x = rx ? u1[o + 1] - u1[o] : 0.0f, u1y = ry ? u1[o + a.W] - u1[o] : 0.0f;
    const float u2x = rx ? u2[o + 1] - u2[o] : 0.0f, u2y = ry ? u2[o + a.W] - u2[o] : 0.0f;
    const float taut = kTau / kTheta;
    const float ng1 = 1.0f + taut * sqrtf(u1x * u1x + u1y * u1y);
    const float ng2 = 1.0f + taut * sqrtf(u2x * u2x + u2y * u2y);
    p[0] = (p[0] + taut * u1x) / ng1;
    p[plane] = (p[plane] + taut * u1y) / ng1;
    p[2 * plane] = (p[2 * plane] + taut * u2x) / ng2;
    p[3 * plane] = (p[3 * plane] + taut * u2y) / ng2;
  }
  if (blockIdx.x == 0 && blockIdx.y == 0) {      // second pass of the pair's error sum, in a fixed order
    float s = 0.0f;
    for (int i = threadIdx.x; i < a.blocks; i += kThreads) s += a.partial[(int64_t)k * a.blocks + i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
      const int n = a.iters[k] + 1;
      a.iters[k] = n;
      if (s / (float)(a.H * a.W) <= kEpsilon * kEpsilon || n >= COCLR_TVL1_MAX_ITERS) a.done[k] = 1;
    }
  }
}

__global__ void reset_kernel(int* done, int* iters, int P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < P) done[k] = iters[k] = 0;
}

__global__ void record_kernel(const int* iters, int* out, int P, int stride, int slot) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < P) out[(int64_t)k * stride + slot] = iters[k];
}

__global__ void quantise_kernel(const float* __restrict__ flow, uint8_t* __restrict__ out, int H, int W) {
  const int x = blockIdx.x * kTx + (threadIdx.x & (kTx - 1)), y = blockIdx.y * kTy + (threadIdx.x / kTx);
  if (x >= W || y >= H) return;
  const int64_t plane = (int64_t)H * W, o = y * W + x;
  uint8_t* px = out + (blockIdx.z * plane + o) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float f = c < 2 ? flow[(2 * blockIdx.z + c) * plane + o] : 0.0f;
    // no contraction: the bytes must equal numpy's float32 arithmetic
    float q = floorf(__fadd_rn(__fmul_rn(__fadd_rn(f, COCLR_FLOW_BOUND), 255.0f / (2.0f * COCLR_FLOW_BOUND)), 0.5f));
    q = fminf(fmaxf(q, 0.0f), 255.0f);
    px[c] = (uint8_t)q;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------------

Taps gaussian_taps() {
  const double sigma = 0.6 * sqrt(1.0 / (kEta * kEta) - 1.0);
  Taps t{};
  double w[2 * kRadius + 1], sum = 0.0;
  for (int k = -kRadius; k <= kRadius; ++k) sum += (w[k + kRadius] = exp(-0.5 * k * k / (sigma * sigma)));
  for (int k = 0; k <= 2 * kRadius; ++k) t.w[k] = (float)(w[k] / sum);
  return t;
}

struct Level {
  int H, W;
  size_t off;   // float offset of the level's [P, H, W] plane in a pyramid
};

std::vector<Level> levels(int H, int W, int P) {
  std::vector<Level> L;
  L.push_back({H, W, 0});
  while ((int)L.size() < COCLR_TVL1_MAX_SCALES) {
    const int h = (int)(L.back().H * kEta + 0.5), w = (int)(L.back().W * kEta + 0.5);
    if (std::min(h, w) < kMinSide) break;
    L.push_back({h, w, L.back().off + (size_t)P * L.back().H * L.back().W});
  }
  return L;
}

size_t align64(size_t n) { return (n + 63) & ~(size_t)63; }
int blocks_of(int H, int W) { return ((W + kTx - 1) / kTx) * ((H + kTy - 1) / kTy); }

struct Work {
  std::vector<Level> L;
  float *pyr0, *pyr1, *tmp, *tmp2, *i1x, *i1y, *wx, *wy, *g, *rhoc, *ub, *p, *partial;
  int *done, *active, *iters;
  size_t bytes;
};

// carves the workspace: pyramids of I0 and I1, two blur planes, the gradients, the warped planes, a second flow
// buffer, the dual variables, the per-CTA partial sums and three int [P] flags
Work carve(int P, int H, int W, char* base) {
  Work w{};
  w.L = levels(H, W, P);
  const size_t plane = (size_t)P * H * W;
  const size_t pyr = w.L.back().off + (size_t)P * w.L.back().H * w.L.back().W;
  size_t off = 0;
  auto take = [&](size_t floats) {
    float* r = base ? reinterpret_cast<float*>(base) + off : nullptr;
    off += align64(floats);
    return r;
  };
  w.pyr0 = take(pyr);
  w.pyr1 = take(pyr);
  w.tmp = take(plane);
  w.tmp2 = take(plane);
  w.i1x = take(plane);
  w.i1y = take(plane);
  w.wx = take(plane);
  w.wy = take(plane);
  w.g = take(plane);
  w.rhoc = take(plane);
  w.ub = take(2 * plane);
  w.p = take(4 * plane);
  w.partial = take((size_t)P * blocks_of(H, W));
  w.done = reinterpret_cast<int*>(take(P));
  w.active = reinterpret_cast<int*>(take(P));
  w.iters = reinterpret_cast<int*>(take(P));
  w.bytes = off * sizeof(float);
  return w;
}

// every kernel puts the batch in gridDim.z
bool shape_ok(int P, int H, int W) {
  return P > 0 && P <= COCLR_FLOW_MAX_BATCH && H > 0 && W > 0 && (int64_t)H * W < (1 << 30);
}

int zoom_out(const float* in, int P, int H, int W, float* tmp, float* tmp2, float* out, int Hc, int Wc,
             cudaStream_t st) {
  const Taps taps = gaussian_taps();
  blur_kernel<<<grid_of(H, W, P), kThreads, 0, st>>>(in, tmp, H, W, taps, 1);
  blur_kernel<<<grid_of(H, W, P), kThreads, 0, st>>>(tmp, tmp2, H, W, taps, 0);
  resample_kernel<<<grid_of(Hc, Wc, P), kThreads, 0, st>>>(tmp2, H, W, out, Hc, Wc, (float)((double)W / Wc),
                                                           (float)((double)H / Hc), 1, 1.0f, 1.0f);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

int zoom_in(const float* uc, int P, int Hc, int Wc, float* uf, int H, int W, cudaStream_t st) {
  resample_kernel<<<grid_of(H, W, P), kThreads, 0, st>>>(uc, Hc, Wc, uf, H, W, (float)((double)Wc / W),
                                                             (float)((double)Hc / H), 2, (float)((double)W / Wc),
                                                             (float)((double)H / Hc));
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

IterArgs iter_args(const Work& w, float* u, int H, int W) {
  IterArgs a;
  a.wx = w.wx;
  a.wy = w.wy;
  a.g = w.g;
  a.rhoc = w.rhoc;
  a.u = u;
  a.p = w.p;
  a.partial = w.partial;
  a.done = w.done;
  a.active = w.active;
  a.iters = w.iters;
  a.H = H;
  a.W = W;
  a.blocks = blocks_of(H, W);
  return a;
}

// runs primal-dual iterations until every pair has converged (or max_iters), reading the flags back every
// COCLR_TVL1_CHECK_EVERY iterations
int iterate(const IterArgs& a, int P, int max_iters, int* host_done, cudaStream_t st) {
  reset_kernel<<<(P + 255) / 256, 256, 0, st>>>(a.done, a.iters, P);
  for (int it = 1; it <= max_iters; ++it) {
    tvl1_u_kernel<<<grid_of(a.H, a.W, P), kThreads, 0, st>>>(a);
    tvl1_p_kernel<<<grid_of(a.H, a.W, P), kThreads, 0, st>>>(a);
    if (cudaGetLastError() != cudaSuccess) return COCLR_E_LAUNCH;
    if (host_done && it % COCLR_TVL1_CHECK_EVERY == 0 && it < max_iters) {
      if (cudaMemcpyAsync(host_done, a.done, P * sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
          cudaStreamSynchronize(st) != cudaSuccess)
        return COCLR_E_LAUNCH;
      bool all = true;
      for (int k = 0; k < P && all; ++k) all = host_done[k] != 0;
      if (all) break;
    }
  }
  return COCLR_OK;
}

}  // namespace
}  // namespace coclr

extern "C" int coclr_tvl1_scales(int H, int W) {
  if (!coclr::shape_ok(1, H, W)) return COCLR_E_ARG;
  return (int)coclr::levels(H, W, 1).size();
}

extern "C" size_t coclr_tvl1_work_bytes(int P, int H, int W) {
  if (!coclr::shape_ok(P, H, W)) return 0;
  return coclr::carve(P, H, W, nullptr).bytes;
}

extern "C" int coclr_tvl1(const coclr_tvl1_t* t, coclr_stream_t stream) {
  using namespace coclr;
  if (!t || !shape_ok(t->P, t->H, t->W) || !t->i0 || !t->i1 || !t->flow || !t->iterations || !t->work) return COCLR_E_ARG;
  const int P = t->P;
  Work w = carve(P, t->H, t->W, static_cast<char*>(t->work));
  if (t->work_bytes < w.bytes) return COCLR_E_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int S = (int)w.L.size();
  const size_t plane0 = (size_t)P * t->H * t->W;
  if (cudaMemcpyAsync(w.pyr0, t->i0, plane0 * sizeof(float), cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(w.pyr1, t->i1, plane0 * sizeof(float), cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return COCLR_E_LAUNCH;
  for (int s = 1; s < S; ++s) {
    const Level &f = w.L[s - 1], &c = w.L[s];
    for (float* pyr : {w.pyr0, w.pyr1}) {
      const int rc = zoom_out(pyr + f.off, P, f.H, f.W, w.tmp, w.tmp2, pyr + c.off, c.H, c.W, st);
      if (rc) return rc;
    }
  }
  std::vector<int> host_done(P);
  for (int s = S - 1; s >= 0; --s) {
    const Level& l = w.L[s];
    const size_t plane = (size_t)P * l.H * l.W;
    float* u = (s % 2 == 0) ? t->flow : w.ub;         // level 0 solves straight into the output
    if (s == S - 1) {
      if (cudaMemsetAsync(u, 0, 2 * plane * sizeof(float), st) != cudaSuccess) return COCLR_E_LAUNCH;
    } else {
      const Level& c = w.L[s + 1];
      const int rc = zoom_in((s % 2 == 0) ? w.ub : t->flow, P, c.H, c.W, u, l.H, l.W, st);
      if (rc) return rc;
    }
    if (cudaMemsetAsync(w.p, 0, 4 * plane * sizeof(float), st) != cudaSuccess) return COCLR_E_LAUNCH;
    gradient_kernel<<<grid_of(l.H, l.W, P), kThreads, 0, st>>>(w.pyr1 + l.off, w.i1x, w.i1y, l.H, l.W);
    const IterArgs a = iter_args(w, u, l.H, l.W);
    for (int k = 0; k < COCLR_TVL1_WARPS; ++k) {
      WarpArgs wa{w.pyr0 + l.off, w.pyr1 + l.off, w.i1x, w.i1y, u, w.wx, w.wy, w.g, w.rhoc, l.H, l.W};
      warp_kernel<<<grid_of(l.H, l.W, P), kThreads, 0, st>>>(wa);
      const int rc = iterate(a, P, COCLR_TVL1_MAX_ITERS, host_done.data(), st);
      if (rc) return rc;
      record_kernel<<<(P + 255) / 256, 256, 0, st>>>(w.iters, t->iterations, P, S * COCLR_TVL1_WARPS,
                                                     s * COCLR_TVL1_WARPS + k);
    }
    if (cudaGetLastError() != cudaSuccess) return COCLR_E_LAUNCH;
  }
  return COCLR_OK;
}

extern "C" int coclr_flow_grey(const uint8_t* rgb, int N, int H, int W, int64_t frame_stride, int64_t row_stride,
                               float* out, coclr_stream_t stream) {
  using namespace coclr;
  if (!rgb || !out || !shape_ok(N, H, W) || row_stride < 3 * (int64_t)W || frame_stride < row_stride * H)
    return COCLR_E_ARG;
  grey_kernel<<<grid_of(H, W, N), kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(rgb, H, W, frame_stride,
                                                                                          row_stride, out);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

extern "C" int coclr_flow_quantise(const float* flow, int P, int H, int W, uint8_t* out, coclr_stream_t stream) {
  using namespace coclr;
  if (!flow || !out || !shape_ok(P, H, W)) return COCLR_E_ARG;
  quantise_kernel<<<grid_of(H, W, P), kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(flow, out, H, W);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

extern "C" int coclr_flow_zoom_out(const float* in, int P, int H, int W, float* tmp, float* out, int Hc, int Wc,
                                   coclr_stream_t stream) {
  using namespace coclr;
  if (!in || !tmp || !out || !shape_ok(P, H, W) || !shape_ok(P, Hc, Wc)) return COCLR_E_ARG;
  return zoom_out(in, P, H, W, tmp, tmp + (size_t)P * H * W, out, Hc, Wc, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int coclr_flow_zoom_in(const float* flow, int P, int Hc, int Wc, float* out, int H, int W,
                                  coclr_stream_t stream) {
  using namespace coclr;
  if (!flow || !out || !shape_ok(P, H, W) || !shape_ok(P, Hc, Wc)) return COCLR_E_ARG;
  return zoom_in(flow, P, Hc, Wc, out, H, W, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int coclr_flow_warp(const float* i0, const float* i1, const float* flow, int P, int H, int W, float* out,
                               coclr_stream_t stream) {
  using namespace coclr;
  if (!i0 || !i1 || !flow || !out || !shape_ok(P, H, W)) return COCLR_E_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t plane = (size_t)P * H * W;
  float* o = out;   // [6, P, H, W]: I1x, I1y, I1w_x, I1w_y, g, rho_c
  gradient_kernel<<<grid_of(H, W, P), kThreads, 0, st>>>(i1, o, o + plane, H, W);
  WarpArgs wa{i0, i1, o, o + plane, flow, o + 2 * plane, o + 3 * plane, o + 4 * plane, o + 5 * plane, H, W};
  warp_kernel<<<grid_of(H, W, P), kThreads, 0, st>>>(wa);
  return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH;
}

extern "C" size_t coclr_flow_iterate_work_bytes(int P, int H, int W) {
  using namespace coclr;
  if (!shape_ok(P, H, W)) return 0;
  return (align64((size_t)P * blocks_of(H, W)) + 3 * align64(P)) * sizeof(float);
}

extern "C" int coclr_flow_iterate(const float* warped, float* flow, float* dual, int P, int H, int W, int n,
                                  int* iters, void* work, coclr_stream_t stream) {
  using namespace coclr;
  if (!warped || !flow || !dual || !iters || !work || !shape_ok(P, H, W) || n < 1) return COCLR_E_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t plane = (size_t)P * H * W;
  Work w{};
  w.wx = const_cast<float*>(warped) + 2 * plane;
  w.wy = w.wx + plane;
  w.g = w.wy + plane;
  w.rhoc = w.g + plane;
  w.p = dual;
  w.partial = static_cast<float*>(work);
  int* flags = reinterpret_cast<int*>(w.partial + align64((size_t)P * blocks_of(H, W)));
  w.done = flags;
  w.active = flags + align64(P);
  w.iters = iters;
  const IterArgs a = iter_args(w, flow, H, W);
  return iterate(a, P, n, nullptr, st);
}
