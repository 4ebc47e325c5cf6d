// Linear probe on extracted features (reference eval/feature_linear_probe.py): optional BatchNorm1d + Linear trained by
// SGD (momentum 0.9, coupled weight decay) with cross-entropy, for S (lr, wd) configs at once over the same batches.
// The batch statistics and x_hat are shared by every config; each config folds its BN affine into its fc, so one GEMM
// gives the logits of all S configs (x_hat [B, D] . [W'_1 .. W'_S]^T) and one GEMM gives every weight gradient
// (G = dl^T . x_hat, [S*C, D]).  Both GEMMs are coclr_sim_fp32 (csrc/evaluate.cu): one fma chain per output, k
// ascending, so no output depends on S or on its column position.  Every other sum runs in a fixed order (per-thread
// strided sums, then a fixed shared-memory tree or a warp butterfly); there are no float atomics, and the results of a
// config are bit-identical from run to run and to a run of that config alone.
//   gather_bn   one CTA per 32 columns        gathers the batch rows; batch mean / variance (double), running stats,
//                                             x_hat [B, D] and x_hat^T [D, Bp] (rows past B zero)
//   fold        one CTA per (config, class)   W' = W * gamma (per column), b' = W . beta + b
//   ce          one warp per (row, config)    loss, top-1 hit (ties to the lower class), dl^T = (softmax - onehot) / B
//                                             (zero for padding rows), or the softmax probabilities
//   reduce      one CTA per (chunk, config)   loss (double) and hit sums over a chunk of rows
//   db_sgd      one warp per (config, class)  db = sum_b dl, then the SGD step of the fc bias
//   bn_grad     one thread per (config, col)  dgamma = sum_n W * G, dbeta = sum_n W * db (before W changes)
//   fc_sgd      one thread per weight         dW = gamma * G + db * beta, SGD step of W
//   bn_sgd      one thread per (config, col)  SGD steps of gamma and beta
//   eval_norm   one thread per element        x_hat = (x - running_mean) / sqrt(running_var + eps)
#include <cuda_runtime.h>

#include "coclr_b200.h"

namespace coclr {

namespace {

constexpr int kThreads = 256;
constexpr int kColThreads = 128;
constexpr int kCols = 32, kRowGroups = 8;   // gather_bn: 32 columns x 8 row groups
constexpr float kSgdMomentum = 0.9f;        // the reference's optim.SGD(momentum=0.9), no dampening, no Nesterov

template <typename T, int N>
__device__ __forceinline__ T block_sum(T v, T* sm) {
  sm[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = N / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  const T total = sm[0];
  __syncthreads();
  return total;
}

// xor butterfly: every lane ends with the same bits (each pairwise sum is formed from the same two operands)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// torch.optim.SGD: d = g + wd * p; buf = momentum * buf + d (buf starts at zero, so the first step gives buf = d);
// p -= lr * buf
__device__ __forceinline__ void sgd(float& p, float& buf, float g, float lr, float wd) {
  const float d = fmaf(wd, p, g);
  buf = fmaf(kSgdMomentum, buf, d);
  p = fmaf(-lr, buf, p);
}

// grid ceil(D / 32), block (32, 8)
__global__ void __launch_bounds__(kCols * kRowGroups)
gather_bn_kernel(const float* __restrict__ x, const int* __restrict__ rows, int Bc, int Bp, int D, int bn,
                 float momentum, float eps, float* __restrict__ rmean, float* __restrict__ rvar, float* __restrict__ xh,
                 float* __restrict__ xhT) {
  __shared__ double smd[kRowGroups][kCols];
  __shared__ float tile[kCols][kCols + 1];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c0 = blockIdx.x * kCols, c = c0 + tx;
  float mu = 0.f, rs = 1.f;
  if (bn) {
    // sum over the row groups (rows ty, ty + 8, ...), then a fixed tree over the groups
    auto column_total = [&](double s) {
      smd[ty][tx] = s;
      __syncthreads();
#pragma unroll
      for (int h = kRowGroups / 2; h > 0; h >>= 1) {
        if (ty < h) smd[ty][tx] += smd[ty + h][tx];
        __syncthreads();
      }
      const double t = smd[0][tx];
      __syncthreads();
      return t;
    };
    double s = 0.0;
    if (c < D)
      for (int b = ty; b < Bc; b += kRowGroups) s += x[(size_t)rows[b] * D + c];
    const double m = column_total(s) / Bc;
    double q = 0.0;
    if (c < D)
      for (int b = ty; b < Bc; b += kRowGroups) {
        const double d = x[(size_t)rows[b] * D + c] - m;
        q += d * d;
      }
    q = column_total(q);
    mu = (float)m;
    rs = (float)(1.0 / sqrt(q / Bc + (double)eps));
    if (ty == 0 && c < D) {
      rmean[c] = (1.f - momentum) * rmean[c] + momentum * mu;
      rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)(q / (Bc - 1));
    }
  }
  for (int r0 = 0; r0 < Bp; r0 += kCols) {
    for (int i = ty; i < kCols; i += kRowGroups) {
      const int b = r0 + i;
      float v = 0.f;
      if (b < Bc && c < D) {
        const float xv = x[(size_t)rows[b] * D + c];
        v = bn ? (xv - mu) * rs : xv;
        xh[(size_t)b * D + c] = v;
      }
      tile[i][tx] = v;
    }
    __syncthreads();
    for (int i = ty; i < kCols; i += kRowGroups) {
      const int cc = c0 + i, b = r0 + tx;
      if (cc < D && b < Bp) xhT[(size_t)cc * Bp + b] = tile[tx][i];
    }
    __syncthreads();
  }
}

// grid S * C
__global__ void __launch_bounds__(kColThreads)
fold_kernel(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ gamma,
            const float* __restrict__ beta, float* __restrict__ Wf, float* __restrict__ bf, int C, int D) {
  __shared__ float sm[kColThreads];
  const int j = blockIdx.x, s = j / C;
  const float* w = W + (size_t)j * D;
  const float* g = gamma + (size_t)s * D;
  const float* be = beta + (size_t)s * D;
  float acc = 0.f;
  for (int k = threadIdx.x; k < D; k += kColThreads) {
    Wf[(size_t)j * D + k] = w[k] * g[k];
    acc = fmaf(w[k], be[k], acc);
  }
  acc = block_sum<float, kColThreads>(acc, sm);
  if (threadIdx.x == 0) bf[j] = acc + bias[j];
}

// grid (ceil(Bp / 8), S), 8 warps.  Row b of config s: z = logits[b, s*C .. s*C+C) + bias.  rows (train) maps the
// batch row to its feature row for the label; NULL means identity (eval).  Rows in [B, Bp) only zero their dl^T column.
__global__ void __launch_bounds__(kThreads)
ce_kernel(const float* __restrict__ logits, int ldl, const float* __restrict__ bias, const long* __restrict__ label,
          const int* __restrict__ rows, int B, int Bp, int C, float inv_b, float* __restrict__ dlT,
          float* __restrict__ prob, float* __restrict__ row_loss, float* __restrict__ row_hit, int ldr) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5), s = blockIdx.y;
  if (b >= Bp) return;
  const size_t col0 = (size_t)s * C;
  if (b >= B) {
    for (int n = lane; n < C; n += 32) dlT[(col0 + n) * Bp + b] = 0.f;
    return;
  }
  const int y = (int)label[rows ? rows[b] : b];
  const float* z = logits + (size_t)b * ldl + col0;
  const float* bb = bias + col0;
  float m = -INFINITY;
  int arg = C;
  for (int n = lane; n < C; n += 32) {   // n ascending per lane: only a strictly larger value replaces the best
    const float v = z[n] + bb[n];
    if (arg == C || v > m) {
      m = v;
      arg = n;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (oa < C && (arg == C || om > m || (om == m && oa < arg))) {
      m = om;
      arg = oa;
    }
  }
  float se = 0.f;
  for (int n = lane; n < C; n += 32) se += expf(z[n] + bb[n] - m);
  se = warp_sum(se);
  if (lane == 0) {
    row_loss[(size_t)s * ldr + b] = m + logf(se) - (z[y] + bb[y]);
    row_hit[(size_t)s * ldr + b] = arg == y ? 1.f : 0.f;
  }
  for (int n = lane; n < C; n += 32) {
    const float p = expf(z[n] + bb[n] - m) / se;
    if (dlT) dlT[(col0 + n) * Bp + b] = (p - (n == y ? 1.f : 0.f)) * inv_b;
    if (prob) prob[((size_t)s * B + b) * C + n] = p;
  }
}

// grid (chunks, S): rows [chunk * per, min(+per, n)) of config s -> out[(slot0 + chunk) * S + s]
__global__ void __launch_bounds__(kThreads)
reduce_kernel(const float* __restrict__ row_loss, const float* __restrict__ row_hit, int ldr, int n, int per,
              double* __restrict__ out_loss, int* __restrict__ out_hits, int slot0) {
  __shared__ double smd[kThreads];
  __shared__ int smi[kThreads];
  const int chunk = blockIdx.x, s = blockIdx.y, S = gridDim.y;
  const int r0 = chunk * per, r1 = min(r0 + per, n);
  double l = 0.0;
  int h = 0;
  for (int r = r0 + threadIdx.x; r < r1; r += kThreads) {
    l += row_loss[(size_t)s * ldr + r];
    h += (int)row_hit[(size_t)s * ldr + r];
  }
  l = block_sum<double, kThreads>(l, smd);
  h = block_sum<int, kThreads>(h, smi);
  if (threadIdx.x == 0) {
    out_loss[(size_t)(slot0 + chunk) * S + s] = l;
    out_hits[(size_t)(slot0 + chunk) * S + s] = h;
  }
}

// grid ceil(S*C / 8), 8 warps
__global__ void __launch_bounds__(kThreads)
db_sgd_kernel(const float* __restrict__ dlT, int Bp, float* __restrict__ db, float* __restrict__ bias,
              float* __restrict__ bias_buf, const float* __restrict__ lr, const float* __restrict__ wd, int C, int SC) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  if (j >= SC) return;
  float acc = 0.f;
  for (int b = lane; b < Bp; b += 32) acc += dlT[(size_t)j * Bp + b];
  acc = warp_sum(acc);
  if (lane == 0) {
    const int s = j / C;
    db[j] = acc;
    sgd(bias[j], bias_buf[j], acc, lr[s], wd[s]);
  }
}

// grid (ceil(D / 128), S)
__global__ void __launch_bounds__(kColThreads)
bn_grad_kernel(const float* __restrict__ W, const float* __restrict__ G, const float* __restrict__ db,
               float* __restrict__ dgamma, float* __restrict__ dbeta, int C, int D) {
  const int k = blockIdx.x * kColThreads + threadIdx.x, s = blockIdx.y;
  if (k >= D) return;
  float dg = 0.f, dbt = 0.f;
  for (int n = 0; n < C; ++n) {
    const size_t j = (size_t)s * C + n;
    const float w = W[j * D + k];
    dg = fmaf(w, G[j * D + k], dg);
    dbt = fmaf(w, db[j], dbt);
  }
  dgamma[(size_t)s * D + k] = dg;
  dbeta[(size_t)s * D + k] = dbt;
}

__global__ void __launch_bounds__(kThreads)
fc_sgd_kernel(float* __restrict__ W, float* __restrict__ W_buf, const float* __restrict__ G,
              const float* __restrict__ db, const float* __restrict__ gamma, const float* __restrict__ beta, int bn,
              const float* __restrict__ lr, const float* __restrict__ wd, int C, int D, long n) {
  const long i = (long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const long j = i / D;
  const int k = (int)(i - j * D), s = (int)(j / C);
  float g = G[i];
  if (bn) g = fmaf(gamma[(size_t)s * D + k], g, db[j] * beta[(size_t)s * D + k]);
  sgd(W[i], W_buf[i], g, lr[s], wd[s]);
}

// grid (ceil(D / 128), S)
__global__ void __launch_bounds__(kColThreads)
bn_sgd_kernel(float* __restrict__ gamma, float* __restrict__ gamma_buf, const float* __restrict__ dgamma,
              float* __restrict__ beta, float* __restrict__ beta_buf, const float* __restrict__ dbeta,
              const float* __restrict__ lr, const float* __restrict__ wd, int D) {
  const int k = blockIdx.x * kColThreads + threadIdx.x, s = blockIdx.y;
  if (k >= D) return;
  const size_t i = (size_t)s * D + k;
  sgd(gamma[i], gamma_buf[i], dgamma[i], lr[s], wd[s]);
  sgd(beta[i], beta_buf[i], dbeta[i], lr[s], wd[s]);
}

__global__ void __launch_bounds__(kThreads)
eval_norm_kernel(const float* __restrict__ x, const float* __restrict__ rmean, const float* __restrict__ rvar,
                 float eps, float* __restrict__ y, int D, long n) {
  const long i = (long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const int k = (int)(i % D);
  y[i] = (x[i] - rmean[k]) * (float)(1.0 / sqrt((double)rvar[k] + (double)eps));
}

inline cudaStream_t ST(coclr_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline int LAUNCH_OK() { return cudaGetLastError() == cudaSuccess ? COCLR_OK : COCLR_E_LAUNCH; }
inline long round4(long n) { return (n + 3) / 4 * 4; }
inline unsigned cdiv(long a, long b) { return (unsigned)((a + b - 1) / b); }

// The workspace, carved in this order; every region starts 16-byte aligned.
struct Work {
  float *xh, *xhT, *xq, *Wf, *bf, *logits, *dlT, *G, *db, *dgamma, *dbeta, *row_loss, *row_hit;
  long ldr, floats;
};

Work carve(const coclr_probe_t* p, float* base) {
  const long Bmax = p->batch < p->N ? p->batch : p->N, Bp = round4(Bmax), SC = (long)p->S * p->C, D = p->D;
  const long rmax = Bp > p->Nq ? Bp : p->Nq;
  Work w{};
  long off = 0;
  auto take = [&](long n) {
    float* r = base ? base + off : nullptr;
    off += round4(n);
    return r;
  };
  w.xh = take(Bp * D);
  w.xhT = take(D * Bp);
  w.xq = p->final_bn ? take((long)p->Nq * D) : nullptr;
  w.Wf = p->final_bn ? take(SC * D) : nullptr;
  w.bf = p->final_bn ? take(SC) : nullptr;
  w.logits = take(rmax * SC);
  w.dlT = take(SC * Bp);
  w.G = take(SC * D);
  w.db = take(SC);
  w.dgamma = take((long)p->S * D);
  w.dbeta = take((long)p->S * D);
  w.ldr = rmax;
  w.row_loss = take((long)p->S * rmax);
  w.row_hit = take((long)p->S * rmax);
  w.floats = off;
  return w;
}

bool args_ok(const coclr_probe_t* p) {
  if (!p || p->N <= 0 || p->Nq <= 0 || p->D <= 0 || p->D % 4 || p->C <= 0 || p->S <= 0) return false;
  if (p->epochs <= 0 || p->batch <= 0 || p->eval_freq <= 0) return false;
  if (!p->train || !p->train_label || !p->test || !p->test_label || !p->order || !p->lr || !p->wd) return false;
  if (!p->W || !p->bias || !p->W_buf || !p->bias_buf || !p->work) return false;
  if (!p->train_loss || !p->train_hits || !p->val_loss || !p->val_hits || !p->prob) return false;
  if (p->final_bn) {
    if (!p->gamma || !p->beta || !p->gamma_buf || !p->beta_buf || !p->running_mean || !p->running_var) return false;
    if (p->N % p->batch == 1) return false;   // BatchNorm1d needs more than one value per channel in training
  }
  const uintptr_t a = reinterpret_cast<uintptr_t>(p->train) | reinterpret_cast<uintptr_t>(p->test) |
                      reinterpret_cast<uintptr_t>(p->W) | reinterpret_cast<uintptr_t>(p->work);
  return a % 16 == 0;
}

// eval mode over the whole test set (rows are independent); hits / loss per chunk of `batch` rows into slot `slot`
int run_eval(const coclr_probe_t* p, const Work& w, int slot, bool final, cudaStream_t st) {
  const int S = p->S, C = p->C, D = p->D, Nq = p->Nq, SC = S * C;
  const float* x = p->test;
  const float* Wsrc = p->W;
  const float* bsrc = p->bias;
  if (p->final_bn) {
    const long n = (long)Nq * D;
    eval_norm_kernel<<<cdiv(n, kThreads), kThreads, 0, st>>>(p->test, p->running_mean, p->running_var, p->eps, w.xq, D,
                                                             n);
    fold_kernel<<<SC, kColThreads, 0, st>>>(p->W, p->bias, p->gamma, p->beta, w.Wf, w.bf, C, D);
    x = w.xq;
    Wsrc = w.Wf;
    bsrc = w.bf;
  }
  int rc = coclr_sim_fp32(x, Wsrc, w.logits, Nq, SC, D, st);
  if (rc != COCLR_OK) return rc;
  ce_kernel<<<dim3(cdiv(Nq, kThreads / 32), S), kThreads, 0, st>>>(w.logits, SC, bsrc, p->test_label, nullptr, Nq, Nq,
                                                                   C, 0.f, nullptr, final ? p->prob : nullptr,
                                                                   w.row_loss, w.row_hit, (int)w.ldr);
  const int chunks = cdiv(Nq, p->batch);
  reduce_kernel<<<dim3(chunks, S), kThreads, 0, st>>>(w.row_loss, w.row_hit, (int)w.ldr, Nq, p->batch, p->val_loss,
                                                      p->val_hits, slot * chunks);
  return LAUNCH_OK();
}

}  // namespace

}  // namespace coclr

using namespace coclr;

extern "C" long coclr_probe_work_floats(const coclr_probe_t* p) {
  if (!p || p->N <= 0 || p->Nq <= 0 || p->D <= 0 || p->C <= 0 || p->S <= 0 || p->batch <= 0) return -1;
  return carve(p, nullptr).floats;
}

extern "C" int coclr_probe_run(const coclr_probe_t* p, coclr_stream_t stream) {
  if (!args_ok(p)) return COCLR_E_ARG;
  const cudaStream_t st = ST(stream);
  const Work w = carve(p, p->work);
  const int S = p->S, C = p->C, D = p->D, N = p->N, SC = S * C;
  const int steps = (N + p->batch - 1) / p->batch;
  const long nW = (long)SC * D;
  int ev = 0;
  for (int e = 0; e < p->epochs; ++e) {
    const float* lr = p->lr + (size_t)e * S;
    for (int t = 0; t < steps; ++t) {
      const int Bc = min(p->batch, N - t * p->batch), Bp = (int)round4(Bc);
      const int* rows = p->order + (size_t)e * N + (size_t)t * p->batch;
      gather_bn_kernel<<<cdiv(D, kCols), dim3(kCols, kRowGroups), 0, st>>>(
          p->train, rows, Bc, Bp, D, p->final_bn, p->momentum, p->eps, p->running_mean, p->running_var, w.xh, w.xhT);
      const float* Wsrc = p->W;
      const float* bsrc = p->bias;
      if (p->final_bn) {
        fold_kernel<<<SC, kColThreads, 0, st>>>(p->W, p->bias, p->gamma, p->beta, w.Wf, w.bf, C, D);
        Wsrc = w.Wf;
        bsrc = w.bf;
      }
      int rc = coclr_sim_fp32(w.xh, Wsrc, w.logits, Bc, SC, D, st);
      if (rc != COCLR_OK) return rc;
      ce_kernel<<<dim3(cdiv(Bp, kThreads / 32), S), kThreads, 0, st>>>(w.logits, SC, bsrc, p->train_label, rows, Bc,
                                                                       Bp, C, 1.f / (float)Bc, w.dlT, nullptr,
                                                                       w.row_loss, w.row_hit, (int)w.ldr);
      reduce_kernel<<<dim3(1, S), kThreads, 0, st>>>(w.row_loss, w.row_hit, (int)w.ldr, Bc, Bc, p->train_loss,
                                                     p->train_hits, e * steps + t);
      rc = coclr_sim_fp32(w.dlT, w.xhT, w.G, SC, D, Bp, st);
      if (rc != COCLR_OK) return rc;
      db_sgd_kernel<<<cdiv(SC, kThreads / 32), kThreads, 0, st>>>(w.dlT, Bp, w.db, p->bias, p->bias_buf, lr, p->wd, C,
                                                                  SC);
      if (p->final_bn)
        bn_grad_kernel<<<dim3(cdiv(D, kColThreads), S), kColThreads, 0, st>>>(p->W, w.G, w.db, w.dgamma, w.dbeta, C,
                                                                              D);
      fc_sgd_kernel<<<cdiv(nW, kThreads), kThreads, 0, st>>>(p->W, p->W_buf, w.G, w.db, p->gamma, p->beta,
                                                             p->final_bn, lr, p->wd, C, D, nW);
      if (p->final_bn)
        bn_sgd_kernel<<<dim3(cdiv(D, kColThreads), S), kColThreads, 0, st>>>(p->gamma, p->gamma_buf, w.dgamma, p->beta,
                                                                             p->beta_buf, w.dbeta, lr, p->wd, D);
      rc = LAUNCH_OK();
      if (rc != COCLR_OK) return rc;
    }
    if (e % p->eval_freq == 0) {
      const int rc = run_eval(p, w, ev++, false, st);
      if (rc != COCLR_OK) return rc;
    }
  }
  return run_eval(p, w, ev, true, st);
}
