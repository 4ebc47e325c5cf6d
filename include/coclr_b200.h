/*
 * coclr_b200 -- C ABI of the H100 (sm_90a) kernels behind the CoCLR data-parallel hot path.
 *
 * The reference (TengdaHan/CoCLR) has no FFI layer: its hot path is Python calling nn.Conv3d /
 * nn.BatchNorm3d / nn.MaxPool3d / torch.einsum (SURVEY.md section 8b).  Each entry point below
 * replaces the vendor-library call(s) named in its comment (reference file:line), takes raw device
 * pointers + sizes + a cudaStream_t, never allocates, never synchronises, and returns 0 on success
 * or a negative error code (COCLR_E_*).
 *
 * Data layout: activations are channels-last rows [B, T, H, W, ld].  A convolution OUTPUT is written as
 * fp32 (pre-BatchNorm, needed for the statistics and the backward pass); every convolution INPUT is a
 * pair of 16-bit planes (hi, lo) of the same shape with hi + lo ~= the fp32 value (fp16 pair: ~22 bits,
 * bf16 pair: ~16 bits), produced by coclr_affine_split / coclr_maxpool_fwd / coclr_pack_input /
 * coclr_bn_bwd.  Three tensor-core passes (hi*lo, lo*hi, hi*hi) then give an fp32-grade product.
 *
 * The Python host side (coclr_b200/lib.py) binds these with ctypes; INTEGRATION.md shows the stub.
 */
#ifndef COCLR_B200_H_
#define COCLR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COCLR_OK 0
#define COCLR_E_ARG (-1)    /* bad argument (shape / alignment / null) */
#define COCLR_E_LAUNCH (-2) /* CUDA launch error (cudaGetLastError != success) */
#define COCLR_E_DEVICE (-3) /* not an sm_90 device */

typedef void* coclr_stream_t; /* cudaStream_t */

/* A channels-last split-precision activation as an implicit-GEMM operand source. */
typedef struct {
  const void* hi; /* 16-bit plane [B, T, H, W, ld] (fp16 or bf16), 16-byte aligned */
  const void* lo; /* residual plane, same layout; may be NULL for single-pass kernels */
  int ld;         /* channels per pixel in memory (multiple of 8) */
  int coff;       /* first channel used (multiple of 8) */
  int C;          /* channels used (multiple of 8) */
  int T, H, W;
} coclr_src_t;

typedef struct {
  int kt, kh, kw;
  int st, sh, sw; /* each 1 or 2 */
  int pt, ph, pw;
  int transposed; /* 0: src = dst*s + k - p (forward conv / wgrad gather); 1: src = (dst + p - k)/s (dgrad) */
} coclr_geom_t;

/* ---- implicit-GEMM convolution, forward and data-gradient -----------------------------------
 * replaces nn.Conv3d forward (backbone/s3dg.py:11-13,39-42; model/pretrain.py:52,54) and the cuDNN
 * dgrad reached through loss.backward() (main_nce.py:330).  Y[m, n] (+)= sum_k A[m, k] * Wp[n, k],
 * m over the B*Td*Hd*Wd destination pixels, k = tap * C + channel.  Optionally accumulates the
 * per-channel sum / sum of squares of Y (train-mode BatchNorm3d statistics, s3dg.py:16,46-47). */
typedef struct {
  coclr_src_t src;
  coclr_geom_t g;
  int B, Td, Hd, Wd; /* destination pixel grid */
  int Kreal;         /* taps * src.C */
  const void* wpk;   /* packed weights from coclr_pack_weights */
  const float* wunscale; /* [n_tiles*BN] per-column 1/scale, or NULL */
  int N, BN, n_tiles;    /* real output channels, tile width (multiple of 32, <= 128), tiles */
  float* dst;            /* fp32 [B,Td,Hd,Wd,dst_ld] */
  int dst_ld, dst_coff;
  int accumulate;    /* dst += result */
  double* stats_sum; /* [N] per-output-channel sum of Y, accumulated (zero it first); NULL to skip */
  double* stats_sq;  /* [N] per-output-channel sum of Y*Y */
  int npass;         /* 1 = single 16-bit pass, 3 = hi/lo split (fp32-grade) */
  int a_bf16;        /* format of the src planes: 0 = fp16, 1 = bf16 */
  int b_bf16;        /* format of the packed weights */
  const float* out_scale; /* device scalar multiplied into the result (e.g. 1/s of gradient planes stored scaled by s, see
                           * coclr_bn_bwd_t.dy_scale), or NULL */
} coclr_conv_t;
int coclr_conv_igemm(const coclr_conv_t* p, int num_sms, coclr_stream_t stream);
size_t coclr_conv_packed_bytes(int N, int Kreal, int* BN_out, int* n_tiles_out);
/* coclr_conv_igemm runs stride-1 (1,k,k) / (k,1,1) / 1x1x1 shapes (and the temporally strided (k,1,1) stem conv) whose
 * K chunks do not straddle taps on the TMA-staged kernel (csrc/conv_tma.cu: cp.async.bulk.tensor halo slabs shared by
 * the taps of one dimension, resident or streamed weight tiles, bulk-tensor store / add-reduce epilogue) and everything
 * else on the cp.async gather kernel.  coclr_conv_tma_plan reports (without a GPU) whether a launch takes the TMA
 * kernel: returns 1 and fills info[8] = {A slots, B slots, weights resident, staging buffers, shared-memory bytes,
 * tiles, slab bytes per plane, slab types}, else 0.  coclr_set_conv_tma(0) forces the gather kernel (tests compare
 * the two kernels with it). */
int coclr_conv_tma_plan(const coclr_conv_t* p, int* info);
void coclr_set_conv_tma(int enabled);

/* ---- weight-gradient -----------------------------------------------------------------------
 * replaces cuDNN wgrad.  dW[n, c, tap] += sum_m dY[m, n] * A[m, (tap, c)] into the PyTorch weight
 * layout [Cout, Cin_real, kt, kh, kw] (zero dW first).  With a large enough workspace the TMA-staged kernel writes
 * partial sums there and adds them to dW in one reduction launch; the gather kernel adds with fp32 atomics. */
typedef struct {
  coclr_src_t src;   /* conv input planes (as the forward pass consumed them) */
  coclr_geom_t g;    /* forward geometry (transposed = 0) */
  coclr_src_t dy;    /* output-gradient planes [B,Td,Hd,Wd,ld], C = Cout rounded up to 8 */
  int B, Td, Hd, Wd;
  int Cout, Cin_real; /* real sizes of dW (src.C may be padded, e.g. 8 for the RGB stem) */
  float* dw;
  int npass;
  int dy_bf16, src_bf16;
  int splits;        /* pixel-range splits (>= 1) */
  const float* out_scale; /* device scalar multiplied into the result before it is added to dw, or NULL */
  float* ws;         /* workspace (16-byte aligned) of ws_floats floats, see coclr_wgrad_ws_floats; NULL: gather kernel */
  long ws_floats;
} coclr_wgrad_t;
int coclr_conv_wgrad(const coclr_wgrad_t* p, coclr_stream_t stream);
/* coclr_conv_wgrad runs stride-1 "same" (1,k,k) / (k,1,1) / 1x1x1 shapes on the TMA-staged kernel (csrc/wgrad_tma.cu:
 * dY tiles and X halo slabs by cp.async.bulk.tensor, the taps of the reuse dimension as the N blocks of one MMA) when
 * ws is 16-byte aligned and holds at least coclr_wgrad_ws_floats(p) floats.  Every other call (strided convs, no or a
 * too small workspace) runs on the cp.async gather kernel.  coclr_set_wgrad_tma(0) forces the gather kernel (tests
 * compare the two kernels with it); `splits` only steers the gather kernel. */
void coclr_set_wgrad_tma(int enabled);
/* 1 when the TMA-staged kernel's planner accepts the shape (whatever ws is); info[8] (may be NULL) = {tile extent
 * dims 0..2, columns per MMA, 64-cout blocks per work item, pipeline stages, pixel splits, work items} */
int coclr_wgrad_tma_plan(const coclr_wgrad_t* p, int* info);
/* floats of workspace the TMA-staged kernel needs for this shape: it writes its per-CTA partial sums there with plain
 * stores and adds them to dw in one reduction launch (no fp32 atomics: deterministic); 0 for shapes on the gather
 * kernel.  The workspace may be shared by launches on the same stream. */
long coclr_wgrad_ws_floats(const coclr_wgrad_t* p);

/* ---- weight packing -------------------------------------------------------------------------
 * PyTorch conv weight [Cout, Cin, kt, kh, kw] -> swizzled 16-bit hi/lo tile images.
 * mode 0 (forward): rows n = cout, k = tap*Cpad + cin.   mode 1 (dgrad): rows n = cin, k = tap*Cout_pad + cout.
 * Each row is scaled by a power of two (max |w| -> [0.5,1)) before the split; 1/scale goes to unscale. */
typedef struct {
  const float* w;
  int Cout, Cin, taps;
  int Cpad;      /* padded channel count of the K index (>= Cin for mode 0, >= Cout for mode 1) */
  int mode;
  int bf16;
  void* wpk;
  float* unscale; /* [n_tiles*BN] */
} coclr_pack_t;
int coclr_pack_weights(const coclr_pack_t* p, coclr_stream_t stream);
/* every weight of an encoder in one launch: table_dev = device array of n coclr_pack_t, row_start_dev = device int
 * [n + 1], first packed row (of the n_tiles*BN rows coclr_conv_packed_bytes implies) of each entry, ascending */
int coclr_pack_weights_batch(const coclr_pack_t* table_dev, const int* row_start_dev, int n, int total_rows,
                             coclr_stream_t stream);

/* ---- BatchNorm3d statistics -> affine (train mode; backbone/s3dg.py:16,46-47) ------------------
 * per-channel sums written by coclr_conv_igemm -> (scale, shift), saved (mean, rstd) for backward, running-stat
 * momentum update (unbiased variance).  training == 0: scale/shift from the running statistics (eval-mode BN,
 * main_coclr.py:363).  Stand-alone launch (coclr_bn_finalize) or fused into coclr_affine_split. */
typedef struct {
  const double* sum;
  const double* sumsq;
  long count; /* B*T*H*W */
  const float* gamma;
  const float* beta;
  float* running_mean;
  float* running_var;
  float momentum, eps;
  int training;
  float* scale;
  float* shift;
  float* save_mean; /* may be NULL */
  float* save_rstd;
  int C;
} coclr_bn_finalize_t;
int coclr_bn_finalize(const coclr_bn_finalize_t* p, coclr_stream_t stream);

/* ---- BatchNorm-apply + ReLU + precision split --------------------------------------------------
 * hi/lo[m, out_coff + c] = split( relu?( scale[c] * x[m, coff + c] + shift[c] ) ); scale == NULL: identity.
 * The elementwise half of nn.BatchNorm3d + nn.ReLU (backbone/s3dg.py:16-17,24-27), one pass, producing the
 * operand planes every consumer (conv / pool / avg-pool) reads. */
typedef struct {
  const float* x;
  int ld, coff, C; /* C multiple of 4 */
  long M;
  const float* scale;
  const float* shift;
  int relu;
  void* hi;
  void* lo; /* may be NULL */
  int out_ld, out_coff;
  int bf16;
  void* hi2; /* optional bf16 twin of the planes (same out_ld / out_coff) for the weight-gradient GEMM, whose */
  void* lo2; /* two operands must share one 16-bit format (wgmma); NULL to skip */
  /* optional fused BatchNorm finalize (bn.scale != NULL): scale/shift are derived in-kernel from the statistics
   * (bn.training) or the running stats, written to bn.scale/bn.shift/bn.save_* and the running stats are updated
   * by one block -- saves the separate coclr_bn_finalize launch; `scale`/`shift` above are then ignored.
   * hi == NULL with the fused finalize: no planes are written, the call is the finalize alone -- the same kernel over
   * zero rows, so scale / shift / running stats carry the same bits -- for a tensor whose only consumer, a max-pool,
   * reads the conv output itself (coclr_pool_t.y) */
  coclr_bn_finalize_t bn;
  /* optional residual branch of a ResNet bottleneck (`out += residual` then ReLU, backbone/resnet_2d3d.py:75-80,
   * 118-123): operand planes of the same 16-bit format as hi/lo, added after the affine and before the ReLU */
  const void* res_hi; /* NULL: no residual */
  const void* res_lo; /* may be NULL */
  int res_ld, res_coff;
} coclr_split_t;
int coclr_affine_split(const coclr_split_t* p, int num_sms, coclr_stream_t stream);


/* backward of BatchNorm+ReLU: dA (grad w.r.t. relu(bn(y)), fp32) -> dY (grad w.r.t. y) written as bf16
 * hi/lo planes for the dgrad / wgrad kernels; also dgamma / dbeta (accumulated).  Replaces
 * NativeBatchNormBackward0 + ReluBackward0 (SURVEY.md 3.2). */
typedef struct {
  const float* y;  /* raw conv output [M, ld] */
  const float* dA; /* same layout */
  int ld, coff, C;
  long M;
  const float* scale; /* [C] gamma*rstd (as written by finalize) */
  const float* shift;
  const float* mean;
  const float* rstd;
  int relu;
  double* sums;   /* workspace [2*C] */
  float* dgamma;  /* [C] or NULL, += */
  float* dbeta;
  void* dy_hi;    /* bf16 planes [M, ld] (same ld / coff as y) */
  void* dy_lo;    /* may be NULL */
  /* residual block output (relu(bn(y) + r), backbone/resnet_2d3d.py:75-80): r's forward planes enter the ReLU mask,
   * and dz = dA*[bn(y)+r > 0] is also the gradient of the residual branch, written (=) or added (+=) to dres */
  const void* res_hi; /* NULL: plain BN(+ReLU) */
  const void* res_lo;
  int res_ld, res_coff, res_bf16;
  float* dres; /* fp32 [M, dres_ld] at dres_coff, or NULL */
  int dres_ld, dres_coff, dres_accumulate;
  /* dy_fp16 != 0: the planes are written as fp16 hi/lo of dY * s, s a power of two chosen per call so that the largest
   * |dY| the data allows (a per-channel bound from max |dz|, max |xhat| and the two means, reduced over the channels)
   * lands at 2^14: ~22 significant bits near the top of the range instead of bf16 hi/lo's 16, and the weight-gradient
   * GEMM can pair them with the forward pass's fp16 activation planes (wgmma needs one format for both
   * operands) -- no bf16 twin of every activation.  dy_scale[0] = s, dy_scale[1] = 1/s (device, written by the call;
   * consumers pass &dy_scale[1] as out_scale).  amax: workspace [2*C] floats. */
  int dy_fp16;
  float* amax;
  float* dy_scale;
} coclr_bn_bwd_t;
int coclr_bn_bwd(const coclr_bn_bwd_t* p, int num_sms, coclr_stream_t stream);

/* bias+ReLU backward of the projection head (model/pretrain.py:52-53): dA <- dA*[h+b>0] in place, dbias += */
int coclr_bias_relu_bwd(const float* h, const float* bias, float* dA, float* dbias, int M, int C,
                        coclr_stream_t stream);

/* ---- nn.MaxPool3d (backbone/s3dg.py:105,151,162,173,190) ---------------------------------------- */
typedef struct {
  const void* x_hi; /* input planes [B,Ti,Hi,Wi,ldx] fp16 */
  const void* x_lo;
  int ldx, x_coff;
  void* y_hi;       /* output planes [B,To,Ho,Wo,ldy] fp16 */
  void* y_lo;
  int ldy, y_coff;
  void* y2_hi;      /* optional bf16 twin of the output planes (see coclr_split_t), or NULL */
  void* y2_lo;
  unsigned char* idx; /* [B*To*Ho*Wo, C] arg-max tap, may be NULL in forward-only use */
  int B, C, Ti, Hi, Wi, To, Ho, Wo;
  coclr_geom_t g;
  /* backward only: fp32 gradient buffers */
  const float* dy; /* [B,To,Ho,Wo,C] */
  float* dx;       /* [B,Ti,Hi,Wi,ldx] at x_coff */
  int accumulate;
  /* forward from the conv output (y != NULL; x_hi / x_lo unused): the input is relu?(scale[c] * y + shift[c]) of the
   * fp32 conv output y [B,Ti,Hi,Wi,ldx] at x_coff, split into the fp16 (hi, lo) pairs coclr_affine_split would store
   * and pooled as those planes would be -- the same output planes and idx bit for bit, without writing or reading the
   * input planes (for a BatchNorm+ReLU output whose only consumer is the pool; scale / shift as published by the
   * BatchNorm finalize).  Windows (1,3,3)/(1,2,2), (3,3,3)/2 and (2,2,2)/2 only (any padding). */
  const float* y;
  const float* scale;
  const float* shift;
  int relu;
} coclr_pool_t;
int coclr_maxpool_fwd(const coclr_pool_t* p, coclr_stream_t stream);
int coclr_maxpool_bwd(const coclr_pool_t* p, coclr_stream_t stream);

/* ---- nn.AdaptiveAvgPool3d((1,1,1)) (model/pretrain.py:51) ---------------------------------------- */
int coclr_avgpool_fwd(const void* x_hi, const void* x_lo, int bf16 /* plane format */, int ld, int coff, float* out, int B, int Pn, int C,
                      coclr_stream_t stream);
int coclr_avgpool_bwd(const float* dfeat, float* dA, int ld, int coff, int B, int Pn, int C, coclr_stream_t stream);

/* ---- block[:, i].contiguous() + NCDHW -> channels-last fp16 hi/lo planes with C padded to 8
 * (model/pretrain.py:149-150); batch_index (device int64[B], or NULL) gathers source clips
 * out[b] = x[batch_index[b]] = the shuffle-BN pick x_gather[idx_this] (pretrain.py:124).
 * peer_x != NULL (device array of one clip-buffer base per rank, NVLink peer-mapped, clips_per_peer clips each; x is
 * then ignored): clip g = batch_index[b] is read from peer_x[g / clips_per_peer] + (g % clips_per_peer) * batch_stride,
 * i.e. the all-gather of every rank's clips (pretrain.py:105-106) is replaced by P2P loads of only the B clips this
 * rank encodes.
 * norm_mean / norm_std != NULL: the per-channel (x - mean) / std of the reference's GPU-side input transform `tr`
 * (T.Normalize, main_nce.py:207-209,299-302) is applied on the fly; together with the free batch / channel strides
 * (the loader's [B, C, num_seq*seq_len, H, W] tensor is addressed in place) this folds `tr` -- normalise, view,
 * transpose(1,2), contiguous -- into the packing pass ------------------------------------------------------- */
int coclr_pack_input(const float* x, long batch_stride, long chan_stride, int Cin, void* out_hi, void* out_lo,
                     void* out2_hi, void* out2_lo /* optional bf16 twin */, int B, long thw, const long* batch_index,
                     const void* const* peer_x, int clips_per_peer,
                     const float* norm_mean, const float* norm_std /* device [Cin] or both NULL */,
                     coclr_stream_t stream);

/* space-to-depth variant for the stride-2 7x7 RGB stem (backbone/s3dg.py:145): planes [B, T, H/2, W/2 + 2*pad_x, 16]
 * with channel (dy*2+dx)*Cin + c = x[b, c, t, 2Y+dy, 2X+dx] (4*Cin real channels, rest zero) at pixel X + pad_x of a
 * row; H, W even.  The pad_x pixels on either side of a row are NOT written: the caller zeroes the planes once, which
 * materialises the conv's horizontal zero padding (pad_x = 2 for the 4x4 stem) so that the four taps of a kernel row
 * are one contiguous 128-byte run for every output pixel (the TMA window operand of csrc/conv_tma.cu). */
int coclr_pack_input_s2d(const float* x, long batch_stride, long chan_stride, int Cin, void* out_hi, void* out_lo,
                         void* out2_hi, void* out2_lo, int B, int T, int H, int W, int pad_x, const long* batch_index,
                         const void* const* peer_x, int clips_per_peer, const float* norm_mean, const float* norm_std,
                         coclr_stream_t stream);

/* ---- F.normalize(z + bias, dim=1) (model/pretrain.py:154,167) ------------------------------------- */
int coclr_l2norm_fwd(const float* z, const float* bias, float* q, float* inv_norm, int B, int D, coclr_stream_t stream);
int coclr_l2norm_bwd(const float* q, const float* dq, const float* inv_norm, float* dz, float* dbias, int B, int D,
                     coclr_stream_t stream);

/* ---- _momentum_update_key_encoder (model/pretrain.py:76-80), one launch over the flat parameters -- */
int coclr_ema_update(float* k, const float* q, float m, float one_minus_m, long n, int num_sms, coclr_stream_t stream);

/* ---- _dequeue_and_enqueue column write (model/pretrain.py:93): queue[:, ptr:ptr+n] = keys^T -------- */
int coclr_queue_enqueue(float* queue, const float* keys, int dim, int K, int ptr, int n, coclr_stream_t stream);

/* ---- torch.optim.Adam, coupled L2 (main_nce.py:190-200), flat buffers ----------------------------- */
typedef struct {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  long n;
  float grad_scale; /* e.g. 1/world_size after a sum all-reduce */
  float beta1, beta2, eps, weight_decay;
  float step_size; /* lr / (1 - beta1^t) */
  float bc2_sqrt;  /* sqrt(1 - beta2^t) */
} coclr_adam_t;
int coclr_adam_step(const coclr_adam_t* p, int num_sms, coclr_stream_t stream);

/* ---- torch.optim.SGD(lr, momentum, weight_decay), dampening 0, no Nesterov (eval/main_classifier.py:156-161),
 * flat buffers, bit-identical to torch's default CUDA path (_multi_tensor_sgd) in fp32:
 *   d = fma(wd, p, g) (skipped when wd == 0); buf = d on the first step, else buf = buf * m (rounded), then
 *   buf = buf + d; p = fma(-lr, buf, p)  (ATen's foreach `a + alpha * b` is one fused multiply-add).
 * first != 0: momentum_buf is write-only (the buffer is created from d). */
typedef struct {
  float* param;
  const float* grad;
  float* momentum_buf;
  long n;
  float lr, weight_decay, momentum;
  int first;
} coclr_sgd_t;
int coclr_sgd_step(const coclr_sgd_t* p, int num_sms, coclr_stream_t stream);

/* ---- InfoNCE logits + temperature + cross-entropy (model/pretrain.py:175-182; main_nce.py:201,314) ----
 * logits[b, 0] = q_b.k_b / T, logits[b, 1+j] = q_b.queue[:, j] / T; loss_rows[b] = logsumexp - logits[b,0];
 * dlogits = d(mean_b loss_rows)/d(logits).  loss_rows / dlogits may be NULL.
 * ws: optional scratch of 2 * B * ceil(K / 1024) floats; with it, queues longer than 2048 are cut into 1024-column
 * slices on separate CTAs (config 3: K = 16384 would otherwise run on B of the 132 SMs). */
int coclr_nce_logits_ce(const float* q, const float* k, const float* queue, float T, int B, int D, int K,
                        float* logits, float* loss_rows, float* dlogits, float* ws, coclr_stream_t stream);
/* dq = d(logits)^T contraction with [k | queue] / T (no gradient to k or the queue, pretrain.py:160,176) */
int coclr_nce_logits_bwd(const float* dlogits, const float* k, const float* queue, float T, int B, int D, int K,
                         float* dq, coclr_stream_t stream);

/* ---- CoCLR positive mining (model/pretrain.py:392-413): same-source mask OR top-k of the second view's similarity ----
 * mask[b, 0] = 1; mask[b, 1+j] = (k_vsource[b] == queue_vname[j]) OR j in top-`topk` of kf[b] . queue_second[:, j] taken
 * over the columns that are not same-source (the reference fills those with -inf before torch.topk, :406-407).
 * topk == 0 (or a queue that is not full yet, :404): same-source mask only; kf / queue_second may then be NULL.
 * mask: [B, 1+K] bytes (torch.bool storage). */
int coclr_mask_topk(const float* kf, const float* queue_second, const long* k_vsource, const long* queue_vname, int B, int D,
                    int K, int topk, unsigned char* mask, coclr_stream_t stream);

/* ---- S3D-G feature gating, SelfGating (backbone/s3dg.py:68-78) applied to the branch outputs of a SepInception
 * (:125-129): out[b, c, thw] = sigmoid(fc(mean_thw(a[b])))[c] * a[b, c, thw].  The four branches write channel slices
 * of ONE channels-last concat buffer [B, P = T*H*W, C] (16-bit hi/lo planes, row stride ld); the four nn.Linear layers
 * are the diagonal blocks (coff, n) of the fc step: call coclr_gate_fc / coclr_gate_fc_bwd once per member.
 *   forward : coclr_gate_mean -> coclr_gate_fc (x members) -> coclr_gate_apply (planes scaled in place)
 *   backward: coclr_gate_bwd_reduce (dgate[b, c] = sum_thw dout * a, a = act(y * scale + shift) recomputed from the raw
 *             conv output y and the BatchNorm affine) -> coclr_gate_fc_bwd (x members; ACCUMULATES into dW [n, n]
 *             row-major like nn.Linear.weight and dbias [n], as every parameter-gradient kernel does; writes dmean)
 *             -> coclr_gate_bwd_apply (dout <- gate * dout + dmean / P, in place:
 *             the gradient w.r.t. the un-gated activation, which coclr_bn_bwd then consumes unchanged).
 * mean / gate / dgate / dmean: fp32 [B, C]. */
int coclr_gate_mean(const void* x_hi, const void* x_lo, int bf16 /* plane format */, int ld, int B, int P, int C, float* mean,
                    coclr_stream_t stream);
int coclr_gate_fc(const float* mean, const float* W, const float* bias, float* gate, int B, int C, int coff, int n,
                  coclr_stream_t stream);
int coclr_gate_apply(void* x_hi, void* x_lo, int bf16, int ld, int B, int P, int C, const float* gate, coclr_stream_t stream);
int coclr_gate_bwd_reduce(const float* y, int ldy, const float* scale, const float* shift, int relu, const float* dout, int ldd,
                          int B, int P, int C, float* dgate, coclr_stream_t stream);
int coclr_gate_fc_bwd(const float* dgate, const float* gate, const float* mean, const float* W, float* dW, float* dbias,
                      float* dmean, int B /* <= 256 */, int C, int coff, int n, coclr_stream_t stream);
int coclr_gate_bwd_apply(float* dout, int ldd, const float* gate, const float* dmean, int B, int P, int C, coclr_stream_t stream);

/* ---- Classifier head of LinearClassifier (model/classifier.py:47-61 of the reference):
 *   feat [B, fs] -> F.normalize (l2norm) -> BatchNorm1d (bn) -> Dropout (dropout) -> Linear -> logits [B, ncls]
 * Each stage is optional; a stage that is off passes its input through, and its buffers may be NULL.  fp32
 * throughout, every sum in a fixed order (no float atomics): results are bit-identical from run to run.
 *   forward : xn = feat / max(||feat||, 1e-12) (inv_norm[b] = 1 / that denominator);
 *             bn_training: batch mean / biased variance, running stats updated with momentum and the unbiased
 *             variance (needs B >= 2); else the running stats.  mean / rstd receive the statistics used;
 *             dropout: keep element i when a Philox4x32-10 uniform (seed, subsequence i / 4, offset) is < 1 - p,
 *             mask[i] = keep, xd = keep * x / (1 - p);
 *             logits = fc_in . W^T + bias with fc_in the output of the last stage that is on.
 *   backward: from dlogits: dW / dbias / dgamma / dbeta accumulate (+=); dx is a [B, fs] scratch buffer;
 *             dfeat (may be NULL: no gradient to the backbone) receives d/dfeat. */
typedef struct {
  int B, fs, ncls;
  int l2norm, bn, bn_training, dropout;
  float p, momentum, eps;
  unsigned long long seed, offset;
  const float* feat;                                    /* [B, fs] */
  float* xn; float* inv_norm;                           /* [B, fs], [B] */
  float* xb; float* mean; float* rstd;                  /* [B, fs], [fs], [fs] */
  const float* gamma; const float* beta; float* running_mean; float* running_var;   /* [fs] */
  unsigned char* mask; float* xd;                       /* [B, fs] */
  const float* W; const float* bias; float* logits;     /* [ncls, fs] (nn.Linear.weight), [ncls], [B, ncls] */
  const float* dlogits;                                 /* [B, ncls] */
  float* dW; float* dbias; float* dgamma; float* dbeta; /* accumulated */
  float* dx; float* dfeat;                              /* [B, fs] */
} coclr_cls_head_t;
int coclr_cls_head_fwd(const coclr_cls_head_t* h, coclr_stream_t stream);
int coclr_cls_head_bwd(const coclr_cls_head_t* h, coclr_stream_t stream);

/* ---- Video-level evaluation (eval/main_classifier.py --test of the reference: test_10crop :425-545 and
 * test_retrieval :548-718).  fp32 throughout, every sum in a fixed order; the only atomics are integer hit counters,
 * so results are bit-identical from run to run.
 *   coclr_video_accumulate: one pass of B clips.  slot[b] (int32) is the video slot of clip b, -1 for a padding clip;
 *     the clips of one video are consecutive.  In clip order: prob_sum[v] += softmax(logits[b]) (max subtracted),
 *     feat_sum[v] += feat[b], count[v] += 1.  Sums carry over from pass to pass.
 *   coclr_video_finalize: per video v, feat_mean = feat_sum / count (skipped when feat_mean is NULL),
 *     prob_mean = prob_sum / count (this view's softmax(logit).mean(0)), views_sum += prob_mean, and
 *     prob = views_sum / n_views (the mean over the views so far).  With target: rank[v] = the number of classes
 *     ranked above the target in prob (higher probability, ties to the lower index); hits[0] += rank < 1,
 *     hits[1] += rank < 5.  A target outside [0, C) gets rank C and no hit (the reference scores it as a miss).
 *   coclr_center_normalize: y = F.normalize(x - x.mean(0), dim=1, eps=1e-12); mean [D] receives the column mean.
 *   coclr_sim_fp32: sim [Nq, Nk] = q [Nq, D] . k [Nk, D]^T on fp32 FFMA (D % 4 == 0, 16-byte aligned pointers).
 *   coclr_retrieval_rank: rank[i] = position of query i's best same-label item in the order (sim descending, index
 *     ascending), Nk when there is none; hits[m] += rank < ks[m] for the nks (<= COCLR_MAX_KS) values of ks, never for
 *     a query with no same-label item (so a k above Nk counts the queries that have one).
 * Two-stream merge (eval/merge_2stream_prob.py of the reference):
 *   coclr_sim2_fp32: sim [Nq, Nk] = q1 [Nq, D1] . k1 [Nk, D1]^T + q2 [Nq, D2] . k2 [Nk, D2]^T.  Each product is
 *     coclr_sim_fp32's FFMA chain (k ascending) and the two are joined by one rounded fp32 add, so the result equals
 *     coclr_sim_fp32(q1, k1) + coclr_sim_fp32(q2, k2) bit for bit without an [Nq, Nk] intermediate (two launches on
 *     `stream`, the second adding into sim).  D1, D2 % 4 == 0, 16-byte aligned pointers.
 *   coclr_prob_merge: per video v, fused[v] = (p1[v] + p2[v]) / 2 in double; hits[0] += argmax p1[v] == target[v],
 *     hits[1] += argmax p2[v] == target[v], hits[2] += argmax fused[v] == target[v] (np.argmax: ties to the lowest
 *     index, a NaN above every number).  A target outside [0, C) is a miss. */
#define COCLR_MAX_KS 8
typedef struct {
  const float* prob_sum; const float* feat_sum; const int* count;   /* [Nv, C], [Nv, D], [Nv] */
  int Nv, C, D, n_views;
  float* feat_mean; float* prob_mean;                               /* [Nv, D], [Nv, C] */
  float* views_sum; float* prob;                                    /* [Nv, C] */
  const long* target; int* rank; int* hits;                         /* [Nv] int64, [Nv], [2] (+=) */
} coclr_video_finalize_t;
int coclr_video_accumulate(const float* logits, const float* feat, const int* slot, float* prob_sum, float* feat_sum,
                           int* count, int B, int C, int D, coclr_stream_t stream);
int coclr_video_finalize(const coclr_video_finalize_t* a, coclr_stream_t stream);
int coclr_center_normalize(const float* x, float* y, float* mean, int N, int D, coclr_stream_t stream);
int coclr_sim_fp32(const float* q, const float* k, float* sim, int Nq, int Nk, int D, coclr_stream_t stream);
int coclr_retrieval_rank(const float* sim, const long* qlabel, const long* klabel, int Nq, int Nk, const int* ks,
                         int nks, int* rank, int* hits, coclr_stream_t stream);
int coclr_sim2_fp32(const float* q1, const float* k1, int D1, const float* q2, const float* k2, int D2, float* sim,
                    int Nq, int Nk, coclr_stream_t stream);
int coclr_prob_merge(const double* p1, const double* p2, const long* target, int Nv, int C, double* fused, int* hits,
                     coclr_stream_t stream);   /* [Nv, C] float64 x2, [Nv] int64, [Nv, C] float64, [3] (+=) */

/* ---- Linear probe on extracted features (eval/feature_linear_probe.py of the reference): optional BatchNorm1d
 * (final_bn) + Linear, cross-entropy, SGD (momentum 0.9, coupled weight decay on every parameter), trained for S
 * (lr, wd) configs at once over the same batches.  One call enqueues the whole run -- every epoch, every evaluation --
 * with no host synchronisation and no allocation.  fp32, every sum in a fixed order, no float atomics: config s gives
 * the same bits from run to run and as a run of that config alone (S = 1).
 *   Training step t of epoch e: the B = min(batch, N - t * batch) train rows order[e, t * batch ..]; with final_bn the
 *   batch mean / biased variance normalise the rows and update running_mean / running_var (momentum, unbiased
 *   variance, shared by all configs); logits = x_hat . (W * gamma)^T + W . beta + bias; loss and top-1 hit per row
 *   (ties to the lower class); the gradients of the batch-mean loss; then per config p -= lr[e, s] * buf with
 *   buf = 0.9 buf + grad + wd[s] p.
 *   After epoch e with e % eval_freq == 0, and once after the last epoch: eval mode (running statistics) over the test
 *   set.  The final pass also writes softmax probabilities to prob.
 * Per-chunk outputs (layout [slot, S]): train_loss / train_hits get the sum of the per-row losses and the hit count of
 * each training step (slot e * steps + t, steps = ceil(N / batch)); val_loss / val_hits those of each chunk of `batch`
 * test rows (slot v * ceil(Nq / batch) + chunk for the v-th evaluation, the final pass last).
 * Requirements (COCLR_E_ARG otherwise): D % 4 == 0, 16-byte aligned train / test / W / work; with final_bn no
 * training batch of one row (N % batch != 1).  Indices and labels are not range-checked on the device: order holds
 * rows in [0, N), train labels and test labels lie in [0, C).  work: coclr_probe_work_floats(p) floats. */
typedef struct {
  int N, Nq, D, C, S;                         /* train rows, test rows, feature width, classes, configs */
  int epochs, batch, eval_freq, final_bn;
  float momentum, eps;                        /* BatchNorm1d: 0.1, 1e-5 */
  const float* train; const long* train_label;   /* [N, D], [N] int64 */
  const float* test; const long* test_label;     /* [Nq, D], [Nq] int64 */
  const int* order;                           /* [epochs, N] int32: each epoch's train rows in batch order */
  const float* lr; const float* wd;           /* [epochs, S], [S] */
  float* W; float* bias; float* gamma; float* beta;               /* [S, C, D], [S, C], [S, D], [S, D] (updated) */
  float* W_buf; float* bias_buf; float* gamma_buf; float* beta_buf;   /* momentum buffers, zero on entry */
  float* running_mean; float* running_var;    /* [D] */
  float* work;
  double* train_loss; int* train_hits;        /* [epochs * steps, S] */
  double* val_loss; int* val_hits;            /* [(evaluations + 1) * ceil(Nq / batch), S] */
  float* prob;                                /* [S, Nq, C] */
} coclr_probe_t;
long coclr_probe_work_floats(const coclr_probe_t* p);
int coclr_probe_run(const coclr_probe_t* p, coclr_stream_t stream);

/* Pre-training augmentation (reference utils/augmentation.py, get_transform('train') of main_nce.py / main_coclr.py):
 * for every sample b and clip c in {0, 1} (the q and k clips), S frames starting at source frame clips[b, c].src_frame
 * are cropped and bicubic-resized to D x D, colour-jittered, gray-split, blurred and flipped as PIL does, then written
 * as float32 x / 255.  Output bits equal the reference's ToTensor output for the same decisions.
 * One CTA per output frame; dynamic shared memory coclr_augment_smem_bytes(p) (at most 227 KB).
 *
 * src     uint8 [B, F, Hmax, Wmax, 3] (channels last); every coordinate the tables name lies inside the sample's frames
 * clips   [B, 2] records (below); coclr_b200/augment.py builds them and the tables from a host plan
 * coef    int32 [B, 2, 2, K, D]: per clip, axis (0 = x, 1 = y), tap k and output pixel o, Pillow's 22-bit bicubic
 *         coefficient of source pixel start + k (zero past count)
 * bounds  int32 [B, 2, 2, 2, D]: per clip and axis, start[D] (absolute source coordinate, crop offset included) then
 *         count[D]; both nondecreasing in o, as Pillow's are
 * gray    int8 [B, 2, S]: channel replicated into all three for that frame, -1 for none
 * out     frame f of clip c of sample b, channel ch at out + b * out_batch_stride + c * out_clip_stride +
 *         ch * out_chan_stride + f * D * D, rows of D floats: [B, 3, 2S, D, D] or [B, 2, 3, S, D, D]
 * Requirements (COCLR_E_ARG otherwise): band_rows >= max(D, K) (the horizontal resize pass is done in bands of at most
 * band_rows source rows), F >= 2S, shared memory within 227 KB.  Table contents are not range-checked on the device. */
typedef struct {
  int src_frame;                  /* first source frame of the clip */
  int n_ops;                      /* ColorJitter ops applied (0: no jitter) */
  int op[4];                      /* in application order: 0 brightness, 1 contrast, 2 saturation, 3 hue */
  float factor[3];                /* float32 blend factor of brightness, contrast, saturation */
  int hue_shift;                  /* byte added to PIL's H plane, mod 256 */
  int blur_radius;                /* integer box radius of GaussianBlur, -1: no blur */
  unsigned blur_ww, blur_fw;      /* BoxBlur.c 24-bit window and edge weights */
  int flip;
  int pad[2];
} coclr_augment_clip_t;
typedef struct {
  const uint8_t* src;
  int B, F, Hmax, Wmax;
  int S, D, K, band_rows;         /* frames per clip, output side, taps per output pixel, rows per resize band */
  const coclr_augment_clip_t* clips;
  const int* coef;
  const int* bounds;
  const int8_t* gray;
  float* out;
  long out_batch_stride, out_clip_stride, out_chan_stride;
} coclr_augment_t;
size_t coclr_augment_smem_bytes(const coclr_augment_t* p);
int coclr_augment(const coclr_augment_t* p, coclr_stream_t stream);

/* Fine-tuning and test augmentation (reference eval/main_classifier.py with utils/augmentation.py): the train / val
 * recipe RandomSizedCrop(224, consistent) -> Scale(D) [-> ColorJitter] -> ToTensor (+ the train batch's flip), and the
 * test views flip -> FiveCrop(224) / CenterCrop(224) -> Scale((D, D)) -> ColorJitter -> ToTensor.  Every output frame
 * is a stage-1 bicubic resize of a window of its source frame to M x M (the sample's tables), then, when M != D, a
 * second bicubic resize M -> D with a uint8 image in between (Pillow's two resizes), the sample's jitter chain and
 * flip, written as float32 x / 255.  Output bits equal the reference's ToTensor output for the same decisions.
 * One CTA per output frame; dynamic shared memory coclr_augment_clf_smem_bytes(p) (at most 227 KB).
 *
 * src      uint8 [NF, Hmax, Wmax, 3] (channels last); a sample's source occupies the top-left h x w of its frames
 * frames   [n_frames] records (below): sample index, source frame, output offset and channel stride; output frame
 *          channel c, row y, column x is out[out + c * chan_stride + y * D + x]
 * samples  per-sample records (below); coclr_b200/clf_augment.py builds them and the tables from a host plan
 * coef1    int32 [NS, 2, K1, M]: per sample and axis (0 = x, 1 = y), Pillow's 22-bit bicubic coefficient of tap k of
 *          stage-1 output pixel o (zero past count); bounds1 int32 [NS, 2, 2, M]: start[M] (absolute coordinate in
 *          the sample's frame, or in its mirror image when src_flip is set) then count[M], nondecreasing in o
 * coef2    int32 [K2, D], bounds2 int32 [2, D]: the M -> D resize, the same on both axes (unused when M == D)
 * Requirements (COCLR_E_ARG otherwise): band_rows >= K1 (stage 1's horizontal pass runs in bands of at most band_rows
 * source rows), rows >= 1 and K2 <= M when M != D (stage 1's output is staged `rows` rows at a time), shared memory
 * within 227 KB.  Table contents are not range-checked on the device. */
typedef struct {
  int n_ops;                      /* ColorJitter ops applied (0: no jitter) */
  int op[4];                      /* in application order: 0 brightness, 1 contrast, 2 saturation, 3 hue */
  float factor[3];                /* float32 blend factor of brightness, contrast, saturation */
  int hue_shift;                  /* byte added to PIL's H plane, mod 256 */
  int flip;                       /* mirror the output frame (the train recipe's batch flip) */
  int src_flip;                   /* read the mirror image of the source (the test views' flip before the crop) */
  int src_w;                      /* source width, for src_flip */
  int pad[4];
} coclr_augment_clf_sample_t;
typedef struct {
  int64_t sample;                 /* index into samples */
  int64_t src_frame;              /* frame of src */
  int64_t out;                    /* float offset of the frame's channel 0 in out */
  int64_t chan_stride;            /* floats between its channels */
} coclr_augment_clf_frame_t;
typedef struct {
  const uint8_t* src;
  int NF, Hmax, Wmax;
  int n_frames;
  const coclr_augment_clf_frame_t* frames;
  const coclr_augment_clf_sample_t* samples;
  int M, D, K1, K2, band_rows, rows; /* stage-1 side, output side, taps per pixel, band and staged-row heights */
  const int* coef1;
  const int* bounds1;
  const int* coef2;
  const int* bounds2;
  float* out;
} coclr_augment_clf_t;
size_t coclr_augment_clf_smem_bytes(const coclr_augment_clf_t* p);
int coclr_augment_clf(const coclr_augment_clf_t* p, coclr_stream_t stream);

/* JPEG decoding (the reference datasets' `Image.open(BytesIO(raw)).convert('RGB')`), bit-identical to Pillow's
 * libjpeg-turbo for baseline / extended sequential Huffman JPEGs with 8-bit samples: grayscale (replicated into R, G
 * and B) or YCbCr with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1, decoded with the ISLOW IDCT, fancy upsampling
 * and libjpeg's fixed-point colour conversion.
 *
 * coclr_jpeg_parse (host only, no CUDA call) reads the headers of n frames, frame i being data[offsets[i],
 * offsets[i + 1]).  It fills frames[i] and stores every distinct quant and Huffman table once: up to max_quant /
 * max_huff of them, *n_quant / *n_huff being the number the batch needs.  It returns 0, or 1 when a table array was
 * too small (call again with the reported sizes), or COCLR_E_ARG.  A frame it cannot decode gets a non-zero reason
 * (COCLR_JPEG_*) and no blocks.  Where the scan names a Huffman table no DHT defined, tables 0 and 1 are the
 * standard ones of ITU T.81 Annex K.3, as libjpeg does. */
#define COCLR_JPEG_OK 0
#define COCLR_JPEG_NO_SOI 1
#define COCLR_JPEG_TRUNCATED 2      /* a segment runs past the end of the frame */
#define COCLR_JPEG_PROGRESSIVE 3
#define COCLR_JPEG_ARITHMETIC 4
#define COCLR_JPEG_SOF_KIND 5       /* lossless or hierarchical */
#define COCLR_JPEG_PRECISION 6      /* not 8-bit samples */
#define COCLR_JPEG_COMPONENTS 7     /* not 1 or 3 components (CMYK, YCCK, ...) */
#define COCLR_JPEG_RGB 8            /* 3 components coded as RGB (Adobe transform 0, or component ids R, G, B) */
#define COCLR_JPEG_SAMPLING 9
#define COCLR_JPEG_NO_SOF 10
#define COCLR_JPEG_NO_SOS 11
#define COCLR_JPEG_NO_EOI 12
#define COCLR_JPEG_MULTI_SCAN 13    /* more than one scan, or a scan without every component */
#define COCLR_JPEG_BAD_TABLE 14     /* a missing quant / Huffman table, or an invalid Huffman table */
#define COCLR_JPEG_BAD_SEGMENT 15   /* a malformed segment */
typedef struct {
  int reason;                     /* COCLR_JPEG_*; the other fields are valid only when it is 0 */
  int h, w;
  int ncomp;                      /* 1 (grayscale) or 3 (YCbCr) */
  int hs, vs;                     /* luma sampling (1 1, 2 1 or 2 2; chroma is 1 1); 1 1 for grayscale */
  int restart;                    /* restart interval in MCUs, 0: none */
  int mcus_x, mcus_y;             /* MCU grid; a grayscale MCU is one block */
  int qt[3];                      /* per component: index into the quant tables */
  int dc[3], ac[3];               /* per component: index into the Huffman tables */
  int pad[2];
  int64_t ecs_begin, ecs_end;     /* the entropy-coded segment: bytes [begin, end) of data, markers RSTn included */
  int64_t blocks;                 /* 8 x 8 blocks of all components */
  int64_t block0;                 /* blocks of the batch's frames before this one */
} coclr_jpeg_frame_t;
typedef struct {
  uint16_t q[64];                 /* quantiser of each coefficient, natural (row-major) order */
} coclr_jpeg_quant_t;
typedef struct {
  uint16_t look[512];             /* next 9 bits -> (code length << 8) | symbol; 0: the code is longer */
  int maxcode[18];                /* largest code of length l = 1..16, -1: none */
  int valoff[18];                 /* symbol of code c of length l: val[c + valoff[l]] */
  uint8_t val[256];
  uint8_t bits[16];               /* codes of each length 1..16 (the DHT counts) */
  int nval;
  int pad[3];
} coclr_jpeg_huff_t;
int coclr_jpeg_parse(const uint8_t* data, const int64_t* offsets, int n, coclr_jpeg_frame_t* frames,
                     coclr_jpeg_quant_t* quant, int max_quant, int* n_quant,
                     coclr_jpeg_huff_t* huff, int max_huff, int* n_huff);

/* coclr_jpeg_decode decodes n parsed frames (every reason 0) into out: frame i, row y, column x, channel c is
 * out[i * frame_stride + y * row_stride + 3 * x + c], and only the frame's h x w x 3 bytes are written.  It runs in
 * passes of consecutive frames whose blocks fit the workspace (at most 65535 frames each), three kernels per pass:
 *   entropy  one warp per frame: lane 0 decodes (9-bit lookahead tables in shared memory), the warp stores each
 *            block; raw int16 coefficients, natural order, 128 bytes per block
 *   idct     dequantise and ISLOW IDCT (13-bit constants, 2 pass-1 bits), +128 and clamp; block b's 8 x 8 uint8
 *            samples overwrite the first 64 bytes of its own 128
 *   colour   fancy upsampling of the chroma and YCbCr -> RGB (or gray replicated), fused into the store
 * Workspace: frame i's blocks start at byte 128 * (block0 of i - block0 of the pass's first frame); its component c
 * holds blocks_h(c) x blocks_w(c) blocks, row-major, after the blocks of components < c.  work_bytes must hold at
 * least the largest frame; coclr_jpeg_work_bytes gives what the whole batch needs (one pass).  status [n] int32 gets
 * 0, or COCLR_JPEG_ST_* for a frame whose entropy-coded data is invalid (its pixels are then undefined, the other
 * frames are unaffected).  Every device read of a frame stays inside its [ecs_begin, ecs_end).  No allocation, no
 * synchronisation; frames_host is read on the host to plan the passes. */
#define COCLR_JPEG_ST_BAD_CODE 1      /* a bit pattern that is no code of the Huffman table */
#define COCLR_JPEG_ST_EARLY_END 2     /* the segment (or a restart interval) ends before its last block */
#define COCLR_JPEG_ST_BAD_RESTART 3   /* a restart interval not followed by the expected RSTn marker */
typedef struct {
  int n;
  const uint8_t* data;                    /* device: the batch's bytes (offsets as given to coclr_jpeg_parse) */
  const coclr_jpeg_frame_t* frames;       /* device [n] */
  const coclr_jpeg_frame_t* frames_host;  /* host [n], the same records */
  const coclr_jpeg_quant_t* quant;        /* device */
  const coclr_jpeg_huff_t* huff;          /* device */
  uint8_t* out;
  int64_t frame_stride, row_stride;       /* bytes */
  int* status;                            /* device [n] */
  void* work;                             /* device, 16-byte aligned */
  size_t work_bytes;
} coclr_jpeg_t;
size_t coclr_jpeg_work_bytes(const coclr_jpeg_t* p);
int coclr_jpeg_decode(const coclr_jpeg_t* p, coclr_stream_t stream);
/* Repeated frames: coclr_jpeg_decode_slots writes parsed frame i to output frames slots[slot_begin[i] ..
 * slot_begin[i + 1]) -- each pixel computed once and stored once per slot -- so a frame sampled several times is
 * decoded once.  The host copies are validated before any launch: every output frame in [0, n_out) is written exactly
 * once.  slot_begin == NULL (or s == NULL) is coclr_jpeg_decode: frame i goes to output frame i. */
typedef struct {
  const int* slot_begin;                  /* device [n + 1], or NULL */
  const int* slots;                       /* device [slot_begin[n]] */
  const int* slot_begin_host;             /* host copies of the two */
  const int* slots_host;
  int n_out;
} coclr_jpeg_slots_t;
int coclr_jpeg_decode_slots(const coclr_jpeg_t* p, const coclr_jpeg_slots_t* s, coclr_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* COCLR_B200_H_ */
