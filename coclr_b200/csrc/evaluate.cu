// Video-level evaluation of a pretrained or fine-tuned encoder (reference eval/main_classifier.py --test):
//   per-video accumulation of clip probabilities and features, the per-video means and top-1 / top-5 hits
//   (test_10crop / summarize_probability, :425-545), and nearest-neighbour retrieval (test_retrieval, :686-706).
// Every sum runs in a fixed order (per-thread strided sums, then a fixed shared-memory tree, or one thread walking the
// clips of a video in clip order); the only atomics are integer hit counters.  Results are bit-identical from run to run.
//   video_accumulate   one CTA per video segment of a pass     prob_sum, feat_sum, count (+=)
//   video_finalize     one CTA per video                       feat_mean, prob_mean, views_sum (+=), prob, rank, hits
//   column_mean        one CTA per 32 feature columns          mean (double sums)
//   center_normalize   one CTA per row                         y = (x - mean) / max(||x - mean||, 1e-12)
//   sim_fp32           128 x 128 output tile per CTA           sim = q . k^T or sim += q . k^T, fp32 FFMA, k asc.
//   retrieval_rank     one CTA per query                       rank of the best same-label item, hits (+=)
//   prob_merge         one CTA per video                       fused = (p1 + p2) / 2 in double, argmax hits (+=)
// (reference eval/merge_2stream_prob.py: sim2 = two sim_fp32 launches, the second accumulating; prob_merge.)
#include <cuda_runtime.h>

#include "coclr_b200.h"

namespace coclr {

namespace {

constexpr int kThreads = 256;
constexpr float kNormEps = 1e-12f;   // F.normalize's eps

// sum of one value per thread over the CTA, in a fixed order; every thread returns the total
template <typename T>
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

__device__ __forceinline__ float block_max(float v, float* sm) {
  sm[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] = fmaxf(sm[threadIdx.x], sm[threadIdx.x + s]);
    __syncthreads();
  }
  const float m = sm[0];
  __syncthreads();
  return m;
}

// grid B: the CTA of the first clip of each run of equal slots sums that run in clip order; other CTAs return
__global__ void __launch_bounds__(kThreads)
video_accumulate_kernel(const float* __restrict__ logits, const float* __restrict__ feat, const int* __restrict__ slot,
                        float* __restrict__ prob_sum, float* __restrict__ feat_sum, int* __restrict__ count, int B,
                        int C, int D) {
  __shared__ float smf[kThreads];
  __shared__ double smd[kThreads];
  const int b0 = blockIdx.x, v = slot[b0];
  if (v < 0 || (b0 > 0 && slot[b0 - 1] == v)) return;
  int b1 = b0 + 1;
  while (b1 < B && slot[b1] == v) ++b1;
  float* ps = prob_sum + (size_t)v * C;
  float* fs = feat_sum + (size_t)v * D;
  for (int b = b0; b < b1; ++b) {
    const float* l = logits + (size_t)b * C;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < C; j += kThreads) m = fmaxf(m, l[j]);
    m = block_max(m, smf);
    double s = 0.0;
    for (int j = threadIdx.x; j < C; j += kThreads) s += (double)expf(l[j] - m);
    const float sum = (float)block_sum<double>(s, smd);
    for (int j = threadIdx.x; j < C; j += kThreads) ps[j] += expf(l[j] - m) / sum;
    const float* f = feat + (size_t)b * D;
    for (int j = threadIdx.x; j < D; j += kThreads) fs[j] += f[j];
  }
  if (threadIdx.x == 0) count[v] += b1 - b0;
}

// grid Nv
__global__ void __launch_bounds__(kThreads)
video_finalize_kernel(coclr_video_finalize_t a) {
  __shared__ int smi[kThreads];
  const int v = blockIdx.x;
  const float n = (float)a.count[v];
  if (a.feat_mean)
    for (int j = threadIdx.x; j < a.D; j += kThreads)
      a.feat_mean[(size_t)v * a.D + j] = a.feat_sum[(size_t)v * a.D + j] / n;
  const size_t r = (size_t)v * a.C;
  for (int j = threadIdx.x; j < a.C; j += kThreads) {
    const float pm = a.prob_sum[r + j] / n;
    a.prob_mean[r + j] = pm;
    const float vs = a.views_sum[r + j] + pm;
    a.views_sum[r + j] = vs;
    a.prob[r + j] = vs / (float)a.n_views;
  }
  if (!a.target) return;
  const long tl = a.target[v];
  if (tl < 0 || tl >= a.C) {   // a label the head has no class for: ranked behind every class, never a hit
    if (threadIdx.x == 0) a.rank[v] = a.C;
    return;
  }
  __syncthreads();   // prob[r + t] written by another thread of this CTA
  const int t = (int)tl;
  const float pt = a.prob[r + t];
  int above = 0;
  for (int j = threadIdx.x; j < a.C; j += kThreads) {
    const float p = a.prob[r + j];
    above += (p > pt || (p == pt && j < t)) ? 1 : 0;
  }
  above = block_sum<int>(above, smi);
  if (threadIdx.x == 0) {
    a.rank[v] = above;
    if (above < 1) atomicAdd(&a.hits[0], 1);
    if (above < 5) atomicAdd(&a.hits[1], 1);
  }
}

// grid ceil(D / 32), block (32, 8): column sums over row groups, then a fixed tree over the groups
constexpr int kMeanCols = 32, kMeanGroups = 8;
__global__ void __launch_bounds__(kMeanCols * kMeanGroups)
column_mean_kernel(const float* __restrict__ x, float* __restrict__ mean, int N, int D) {
  __shared__ double sm[kMeanGroups][kMeanCols];
  const int c = blockIdx.x * kMeanCols + threadIdx.x;
  double s = 0.0;
  if (c < D)
    for (int i = threadIdx.y; i < N; i += kMeanGroups) s += x[(size_t)i * D + c];
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
#pragma unroll
  for (int h = kMeanGroups / 2; h > 0; h >>= 1) {
    if (threadIdx.y < h) sm[threadIdx.y][threadIdx.x] += sm[threadIdx.y + h][threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.y == 0 && c < D) mean[c] = (float)(sm[0][threadIdx.x] / N);
}

// grid N
__global__ void __launch_bounds__(kThreads)
center_normalize_kernel(const float* __restrict__ x, const float* __restrict__ mean, float* __restrict__ y, int D) {
  __shared__ double sm[kThreads];
  const size_t r = (size_t)blockIdx.x * D;
  double s = 0.0;
  for (int j = threadIdx.x; j < D; j += kThreads) {
    const float c = x[r + j] - mean[j];
    s += (double)c * c;
  }
  const float den = fmaxf((float)sqrt(block_sum<double>(s, sm)), kNormEps);
  for (int j = threadIdx.x; j < D; j += kThreads) y[r + j] = (x[r + j] - mean[j]) / den;
}

// sim[i, j] = sum_k q[i, k] * k[j, k]: one fma chain per output, k ascending.  Both operands are row-major with the
// reduction dim contiguous; a 128 x 16 slab of each is read as float4 and stored transposed ([k][row]) in shared
// memory, two slabs in flight.  Each of the 256 threads owns an 8 x 8 block of outputs split 4 + 4 rows and columns at
// offset 64, so its shared-memory reads are float4 and conflict-free.  kAccumulate: sim[i, j] = sim[i, j] + dot, one
// rounded fp32 add of the finished chain to what sim holds (the two-stream sim1 + sim2 of the reference).
constexpr int kTM = 128, kTK = 16, kPad = 4;
template <bool kAccumulate>
__global__ void __launch_bounds__(kThreads, 2)
sim_fp32_kernel(const float* __restrict__ q, const float* __restrict__ kf, float* __restrict__ sim, int Nq, int Nk,
                int D) {
  __shared__ __align__(16) float As[2][kTK][kTM + kPad];
  __shared__ __align__(16) float Bs[2][kTK][kTM + kPad];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int row0 = blockIdx.y * kTM, col0 = blockIdx.x * kTM;
  const int lr = tid / 4, lk = (tid % 4) * 4;   // this thread loads rows lr and lr + 64, k lk..lk+3
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ra[2], rb[2];
  auto load = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = row0 + lr + 64 * h, j = col0 + lr + 64 * h, k = k0 + lk;
      ra[h] = (i < Nq && k < D) ? __ldg(reinterpret_cast<const float4*>(q + (size_t)i * D + k)) : zero;
      rb[h] = (j < Nk && k < D) ? __ldg(reinterpret_cast<const float4*>(kf + (size_t)j * D + k)) : zero;
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = lr + 64 * h;
      As[buf][lk + 0][m] = ra[h].x; As[buf][lk + 1][m] = ra[h].y;
      As[buf][lk + 2][m] = ra[h].z; As[buf][lk + 3][m] = ra[h].w;
      Bs[buf][lk + 0][m] = rb[h].x; Bs[buf][lk + 1][m] = rb[h].y;
      Bs[buf][lk + 2][m] = rb[h].z; Bs[buf][lk + 3][m] = rb[h].w;
    }
  };
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const int nt = (D + kTK - 1) / kTK;
  load(0);
  store(0);
  __syncthreads();
  for (int t = 0; t < nt; ++t) {
    const int buf = t & 1;
    if (t + 1 < nt) load((t + 1) * kTK);
#pragma unroll
    for (int k = 0; k < kTK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (t + 1 < nt) store(buf ^ 1);
    __syncthreads();
  }
  const bool vec = (Nk % 4) == 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gi = row0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
    if (gi >= Nq) continue;
    float* out = sim + (size_t)gi * Nk;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gj = col0 + 64 * h + tx * 4;
      if (vec && gj + 3 < Nk) {
        float4 v = make_float4(acc[i][4 * h], acc[i][4 * h + 1], acc[i][4 * h + 2], acc[i][4 * h + 3]);
        if constexpr (kAccumulate) {
          const float4 o = *reinterpret_cast<const float4*>(out + gj);
          v = make_float4(__fadd_rn(o.x, v.x), __fadd_rn(o.y, v.y), __fadd_rn(o.z, v.z), __fadd_rn(o.w, v.w));
        }
        *reinterpret_cast<float4*>(out + gj) = v;
      } else {
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (gj + c < Nk) {
            if constexpr (kAccumulate) out[gj + c] = __fadd_rn(out[gj + c], acc[i][4 * h + c]);
            else out[gj + c] = acc[i][4 * h + c];
          }
      }
    }
  }
}

struct RankKs {
  int k[COCLR_MAX_KS];
  int n;
};

// grid Nq.  Order: sim descending, index ascending.  Pass 1 finds the first same-label item in that order, pass 2
// counts the items before it; with no same-label item the rank is Nk and no k counts it as a hit, not even k > Nk.
__global__ void __launch_bounds__(kThreads)
retrieval_rank_kernel(const float* __restrict__ sim, const long* __restrict__ qlabel, const long* __restrict__ klabel,
                      int Nk, RankKs ks, int* __restrict__ rank, int* __restrict__ hits) {
  __shared__ float sv[kThreads];
  __shared__ int si[kThreads];
  const float* row = sim + (size_t)blockIdx.x * Nk;
  const long lab = qlabel[blockIdx.x];
  float bv = -INFINITY;
  int bi = Nk;   // j ascending per thread: only a strictly larger value replaces the best
  for (int j = threadIdx.x; j < Nk; j += kThreads) {
    const float s = row[j];
    if (klabel[j] == lab && (bi == Nk || s > bv)) {
      bv = s;
      bi = j;
    }
  }
  sv[threadIdx.x] = bv;
  si[threadIdx.x] = bi;
  __syncthreads();
#pragma unroll
  for (int h = kThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      const float ov = sv[threadIdx.x + h];
      const int oi = si[threadIdx.x + h];
      const int mi = si[threadIdx.x];
      if (oi < Nk && (mi == Nk || ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && oi < mi))) {
        sv[threadIdx.x] = ov;
        si[threadIdx.x] = oi;
      }
    }
    __syncthreads();
  }
  bv = sv[0];
  bi = si[0];
  __syncthreads();
  int r = Nk;
  if (bi < Nk) {
    int above = 0;
    for (int j = threadIdx.x; j < Nk; j += kThreads) {
      const float s = row[j];
      above += (s > bv || (s == bv && j < bi)) ? 1 : 0;
    }
    r = block_sum<int>(above, si);
  }
  if (threadIdx.x == 0) {
    rank[blockIdx.x] = r;
    for (int i = 0; i < ks.n; ++i)
      if (r < ks.k[i] && r < Nk) atomicAdd(&hits[i], 1);   // r == Nk: no same-label item, never a hit
  }
}

// running argmax: ties go to the lower index, and a NaN ranks above every number (np.argmax)
struct ArgMax {
  double v;
  int i;   // -1: nothing seen yet
  __device__ __forceinline__ void offer(double ov, int oi) {
    if (oi < 0) return;
    const bool on = isnan(ov), mn = isnan(v);
    const bool better = i < 0 || ((on || mn) ? (on && (!mn || oi < i)) : (ov > v || (ov == v && oi < i)));
    if (better) {
      v = ov;
      i = oi;
    }
  }
};

__device__ __forceinline__ int block_argmax(ArgMax m, double* sv, int* si) {
  sv[threadIdx.x] = m.v;
  si[threadIdx.x] = m.i;
  __syncthreads();
#pragma unroll
  for (int h = kThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      ArgMax a{sv[threadIdx.x], si[threadIdx.x]};
      a.offer(sv[threadIdx.x + h], si[threadIdx.x + h]);
      sv[threadIdx.x] = a.v;
      si[threadIdx.x] = a.i;
    }
    __syncthreads();
  }
  const int best = si[0];
  __syncthreads();
  return best;
}

// grid Nv.  fused = (p1 + p2) / 2; the argmax of p1, p2 and fused each scores a hit when it equals the target.
__global__ void __launch_bounds__(kThreads)
prob_merge_kernel(const double* __restrict__ p1, const double* __restrict__ p2, const long* __restrict__ target,
                  int C, double* __restrict__ fused, int* __restrict__ hits) {
  __shared__ double sv[kThreads];
  __shared__ int si[kThreads];
  const size_t r = (size_t)blockIdx.x * C;
  ArgMax m1{0.0, -1}, m2{0.0, -1}, mf{0.0, -1};
  for (int j = threadIdx.x; j < C; j += kThreads) {
    const double a = p1[r + j], b = p2[r + j], f = (a + b) * 0.5;   // == / 2: both round the same exact value
    fused[r + j] = f;
    m1.offer(a, j);
    m2.offer(b, j);
    mf.offer(f, j);
  }
  const int i1 = block_argmax(m1, sv, si), i2 = block_argmax(m2, sv, si), iff = block_argmax(mf, sv, si);
  if (threadIdx.x == 0) {
    const long t = target[blockIdx.x];   // outside [0, C): equals no argmax, a miss
    if (i1 == t) atomicAdd(&hits[0], 1);
    if (i2 == t) atomicAdd(&hits[1], 1);
    if (iff == t) atomicAdd(&hits[2], 1);
  }
}

inline cudaStream_t S(coclr_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline int LAUNCH_OK() { return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH; }

}  // namespace

}  // namespace coclr

using namespace coclr;

extern "C" int coclr_video_accumulate(const float* logits, const float* feat, const int* slot, float* prob_sum,
                                      float* feat_sum, int* count, int B, int C, int D, coclr_stream_t stream) {
  if (!logits || !feat || !slot || !prob_sum || !feat_sum || !count || B <= 0 || C <= 0 || D <= 0) return COCLR_E_ARG;
  video_accumulate_kernel<<<B, kThreads, 0, S(stream)>>>(logits, feat, slot, prob_sum, feat_sum, count, B, C, D);
  return LAUNCH_OK();
}

extern "C" int coclr_video_finalize(const coclr_video_finalize_t* a, coclr_stream_t stream) {
  if (!a || a->Nv <= 0 || a->C <= 0 || !a->prob_sum || !a->count || !a->prob_mean || !a->views_sum || !a->prob ||
      a->n_views < 1)
    return COCLR_E_ARG;
  if (a->feat_mean && (a->D <= 0 || !a->feat_sum)) return COCLR_E_ARG;
  if (a->target && (!a->rank || !a->hits)) return COCLR_E_ARG;
  video_finalize_kernel<<<a->Nv, kThreads, 0, S(stream)>>>(*a);
  return LAUNCH_OK();
}

extern "C" int coclr_center_normalize(const float* x, float* y, float* mean, int N, int D, coclr_stream_t stream) {
  if (!x || !y || !mean || N <= 0 || D <= 0) return COCLR_E_ARG;
  column_mean_kernel<<<(D + kMeanCols - 1) / kMeanCols, dim3(kMeanCols, kMeanGroups), 0, S(stream)>>>(x, mean, N, D);
  center_normalize_kernel<<<N, kThreads, 0, S(stream)>>>(x, mean, y, D);
  return LAUNCH_OK();
}

extern "C" int coclr_sim_fp32(const float* q, const float* k, float* sim, int Nq, int Nk, int D,
                              coclr_stream_t stream) {
  if (!q || !k || !sim || Nq <= 0 || Nk <= 0 || D <= 0 || D % 4) return COCLR_E_ARG;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(sim)) % 16)
    return COCLR_E_ARG;
  sim_fp32_kernel<false>
      <<<dim3((Nk + kTM - 1) / kTM, (Nq + kTM - 1) / kTM), kThreads, 0, S(stream)>>>(q, k, sim, Nq, Nk, D);
  return LAUNCH_OK();
}

extern "C" int coclr_sim2_fp32(const float* q1, const float* k1, int D1, const float* q2, const float* k2, int D2,
                               float* sim, int Nq, int Nk, coclr_stream_t stream) {
  if (!q1 || !k1 || !q2 || !k2 || !sim || Nq <= 0 || Nk <= 0 || D1 <= 0 || D2 <= 0 || D1 % 4 || D2 % 4)
    return COCLR_E_ARG;
  if ((reinterpret_cast<uintptr_t>(q1) | reinterpret_cast<uintptr_t>(k1) | reinterpret_cast<uintptr_t>(q2) |
       reinterpret_cast<uintptr_t>(k2) | reinterpret_cast<uintptr_t>(sim)) % 16)
    return COCLR_E_ARG;
  const dim3 grid((Nk + kTM - 1) / kTM, (Nq + kTM - 1) / kTM);
  sim_fp32_kernel<false><<<grid, kThreads, 0, S(stream)>>>(q1, k1, sim, Nq, Nk, D1);
  sim_fp32_kernel<true><<<grid, kThreads, 0, S(stream)>>>(q2, k2, sim, Nq, Nk, D2);
  return LAUNCH_OK();
}

extern "C" int coclr_prob_merge(const double* p1, const double* p2, const long* target, int Nv, int C, double* fused,
                                int* hits, coclr_stream_t stream) {
  if (!p1 || !p2 || !target || !fused || !hits || Nv <= 0 || C <= 0) return COCLR_E_ARG;
  prob_merge_kernel<<<Nv, kThreads, 0, S(stream)>>>(p1, p2, target, C, fused, hits);
  return LAUNCH_OK();
}

extern "C" int coclr_retrieval_rank(const float* sim, const long* qlabel, const long* klabel, int Nq, int Nk,
                                    const int* ks, int nks, int* rank, int* hits, coclr_stream_t stream) {
  if (!sim || !qlabel || !klabel || Nq <= 0 || Nk <= 0 || !rank || nks < 0 || nks > COCLR_MAX_KS) return COCLR_E_ARG;
  if (nks > 0 && (!ks || !hits)) return COCLR_E_ARG;
  RankKs kk{};
  kk.n = nks;
  for (int i = 0; i < nks; ++i) kk.k[i] = ks[i];
  retrieval_rank_kernel<<<Nq, kThreads, 0, S(stream)>>>(sim, qlabel, klabel, Nk, kk, rank, hits);
  return LAUNCH_OK();
}
