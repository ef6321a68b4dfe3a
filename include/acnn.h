/*
 * acnn.h -- C ABI of libacnn.so: the H100 (sm_90a) kernels behind the assembled-ResNet hot path.
 *
 * The reference (clovaai/assembled-cnn) has no FFI layer: every op below is a TensorFlow-1.14 graph
 * op emitted by the reference's Python.  Each entry point cites the reference call site it replaces
 * (paths relative to the reference checkout).  INTEGRATION.md shows the ctypes binding.
 *
 * Conventions
 *   - plain C: pointers + sizes only; device pointers are caller-owned (the Python host passes
 *     torch tensors' data_ptr()); the library never allocates device memory.
 *   - every call returns 0 on success, non-zero on failure; acnn_last_error() gives the message.
 *   - every call only ENQUEUES work on `stream` (a cudaStream_t passed as void*): no hidden
 *     synchronisation, CUDA-graph capturable.
 *   - activations are NHWC, bf16 unless stated; "raw" = conv output before batch-norm.
 *   - conv weights are OHWI: [Cout][kh][kw][Cin] (TF's HWIO permuted; see INTEGRATION.md).
 *   - per-channel float vectors (scale/shift/sum/...) are fp32, length C.
 */
#ifndef ACNN_H_
#define ACNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACNN_OK 0
#define ACNN_ERR_INVALID 1
#define ACNN_ERR_CUDA 2
#define ACNN_ERR_UNSUPPORTED 3

/* Storage type of the activation tensors of a call (`dtype` arguments): bf16 is the production
 * path; fp32 is the parity mode (the reference's own default dtype, nets/resnet_model.py:30-33):
 * fp32 activations, every elementwise / reduction kernel instantiated on float, and the conv GEMMs
 * run on operands split into three bf16 planes (`precision` = 1 below).  fp16 is the reference's
 * --dtype=fp16 (nets/resnet_model.py:251-303): fp16 activations and gradients (round to nearest
 * even, overflow to inf), fp32 accumulation wherever the bf16 path accumulates in fp32, and the conv
 * GEMMs on fp16 operands (`precision` = ACNN_F16 below, wgmma .f16.f16, the bf16 path's tiles).
 * 2 is not a storage type. */
#define ACNN_BF16 0
#define ACNN_F32 1
#define ACNN_F16 3

/* Library / environment ------------------------------------------------------------------- */
const char* acnn_last_error(void);
int acnn_version(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
int64_t acnn_launch_count(void);
/* Programmatic dependent launch (no effect on results): 0 (default) = plain stream order, 1 = every
 * kernel, 2 = only light dependents (<= 320 CTAs, <= 48 KiB
 * shared memory).  Returns the previous setting. */
int acnn_set_pdl(int on);
/* 1: the N = 128 conv tiles with 64-channel chunks, K >= 512 and at least one 256-row tile per SM
 * pair run on CTA pairs (a cluster of two CTAs computes one 256 x 128 tile; each CTA loads half of
 * every weight stage and multicasts it to both); 0 (default): single-CTA tiles (measured faster on
 * the c3 step: 61.3 against 80.3 ms on an H100 SXM at 700 W).  Results are bit-identical; changes
 * acnn_conv_stats_parts().  Returns the previous setting. */
int acnn_set_conv_cta_pairs(int on);
/* 3x3 / stride 1 / pad 1 convolutions (fprop and dgrad) on the im2col-free "halo" kernel: a CTA tile
 * is a 16 x 8 patch of output pixels, one 18 x 10 halo tile per 64-channel chunk is loaded once and
 * the nine filter taps read shifted windows of it through the wgmma shared-memory descriptors.
 * 0 = off (im2col TMA kernel everywhere); 1 (default) = where the weight slab of an N tile fits
 * shared memory next to the halo ring, Cin a multiple of 64 and >= 56 rows (c3 step on an H100 SXM
 * at 700 W: 59.8 against 61.3 ms with 0); 2 = wherever it applies.
 * Same results up to fp32 summation order; changes acnn_conv_stats_parts().  Returns the previous
 * setting. */
int acnn_set_conv_halo(int mode);
/* Conv tuning knobs of earlier kernel generations, kept for ABI compatibility: M tiles per CTA
 * tile, the split epilogues (conv GEMM and halo kernel) and the number of output staging buffers.
 * The sm_90a kernels have one organisation (one 128-pixel M tile per CTA, two wgmma consumer
 * warpgroups that run the epilogue from their registers, one output staging buffer): each setter
 * stores its value, returns the previous one and changes nothing else. */
int acnn_set_conv_mtiles(int mode);
int acnn_set_conv_halo_split(int on);
int acnn_set_conv_split_epilogue(int mode);
int acnn_set_conv_split_mt2(int mode);
int acnn_set_conv_out_bufs(int mode);
/* Tuning knob of the wgrad launcher (no effect on results beyond fp32 summation order): pixels
 * (GEMM K) per pipeline stage, 64 or 128 (N tile <= 128 only); 0 = choose per problem (default).
 * Returns the previous setting. */
int acnn_set_wgrad_pixels(int pix);
/* Tuning knob of the wgrad launcher's split-K choice (no effect on results beyond fp32 summation
 * order): the fixed cost of one CTA (pipeline fill + epilogue) in pipeline stages used by the
 * cost model that picks the number of pixel splits (default 16); 0 = the "two waves of CTAs"
 * rule.  Returns the previous setting. */
int acnn_set_wgrad_overhead_stages(int stages);
/* Tuning knob of the wgrad launcher: n > 0 asks for n pixel splits, clamped to the capacity of the
 * partial-tile scratch (64 MiB) and to the number of pipeline stages;
 * 0 (default) = the cost model above.  deterministic != 0 still runs one split.  Returns the previous
 * setting. */
int acnn_set_wgrad_splits(int n);
/* Tuning knob: the largest grid (CTAs) of the grid-stride elementwise kernels (bn_act, bn_bwd_apply,
 * ...); no effect on results.  Values below 132 restore the default (16 x 132).  Returns the previous setting. */
int acnn_set_stream_grid_cap(int blocks);
/* SK attention chains (acnn_sk_fc_fwd / acnn_sk_fc_bwd): 1 = ONE cooperative launch per direction
 * (the whole grid walks GEMM / batch-norm / gate phases separated by grid barriers; K-split partials
 * summed in split order: deterministic, no atomics, nothing to zero); 0 = the multi-launch path (4 + 6
 * kernels and 4 memsets per SK block; unless deterministic, split-K GEMMs whose per-split partials
 * a reduction kernel adds in split order: bit-reproducible, one more launch per GEMM); -1 (default) = fused
 * when the call asks for deterministic results, multi-launch otherwise.
 * Same results up to fp32 summation order.  Returns the previous setting. */
int acnn_set_sk_fc_fused(int on);
/* The K splits of the SK / SE attention GEMMs in the EVAL model handles bound (acnn_bind) while this is
 * set: rows > 0 chooses them as for a batch of max(rows, B) rows, so that each image's outputs are
 * bit for bit those of a handle of `rows` rows (the splits depend on the batch's 64-row tiles, and
 * a different split count sums a row in a different fp32 order).  Needs no more scratch: a larger
 * batch never has more splits.  0 (default): the handle's own batch.  Training handles and the
 * direct entry points acnn_sk_fc_fwd / acnn_se_fc_fwd ignore it.  Returns the previous setting. */
int acnn_set_fc_split_rows(int rows);
/* floats of the `scratch` argument of acnn_sk_fc_fwd / acnn_sk_fc_bwd (da [B,2f] + dz [B,d] + the
 * K-split partial tiles of the widest phase, sized for 132 CTAs; callable without a GPU) */
int64_t acnn_sk_fc_scratch_floats(int B, int f, int d);

/* Convolution geometry (correlation, no bias) -- nets/model_helper.py:67-78 conv2d_fixed_padding
 * + fixed_padding :40-64.  Ho = (H + pad_h_lo + pad_h_hi - kh) / stride + 1, same for W. */
typedef struct acnn_conv_geom {
  int32_t B, H, W, Cin;
  int32_t Cout, kh, kw, stride;
  int32_t pad_h_lo, pad_h_hi, pad_w_lo, pad_w_hi;
  /* Optional element pitches of x (0 = dense NHWC): between W-adjacent pixels, between rows and
   * between images.  x_pix_stride < Cin makes neighbouring "pixels" overlap: the stem conv reads
   * its space-to-depth input [B][H][W+3][16] as W pixels of 64 channels (4 horizontal taps). */
  int32_t x_pix_stride, x_row_pitch, x_img_pitch, reserved_;
} acnn_conv_geom;

/* y[B,Ho,Wo,Cout] = conv(x[B,H,W,Cin], w[Cout,kh,kw,Cin])  as a wgmma implicit GEMM
 * (tf.layers.conv2d: nets/model_helper.py:74-78; tf.layers.dense: nets/resnet_model.py:595-597
 * when kh=kw=H=W=1).  Optional fused epilogue, applied in this order:
 *   + bias[Cout] (fp32)            -> dense bias
 *   + add_src[B,Ho,Wo,Cout] (bf16) -> gradient accumulation across consumers
 *   * (mask_src > 0)               -> ReLU backward of the tensor this gradient belongs to
 *   ch_part[parts][2][Cout]        -> batch-norm statistics (nets/model_helper.py:34-37): every CTA
 *                                     row of the persistent grid STORES its partial column sums and
 *                                     sums of squares of the bf16-rounded output (no atomics, nothing
 *                                     to zero); parts = acnn_conv_stats_parts(g); acnn_bn_finalize
 *                                     adds the rows in a fixed order (bit-reproducible).  A call
 *                                     whose add / mask / bias makes the launch write another row
 *                                     count fails with ACNN_ERR_INVALID (see acnn_conv_stats_parts)
 * out_f32 != 0 stores y as fp32 (logits), else bf16.  Requires Cin % 16 == 0, Cout % 32 == 0.
 * precision ACNN_F16 (3): x, w, add_src, mask_src and a 16-bit y are fp16 instead of bf16 (the
 * statistics are of the fp16-rounded output); everything else as precision 0.
 * precision 0: x, w bf16.  precision 1 (fp32 parity mode): x and w are each three consecutive bf16
 * planes hi / mid / lo of an fp32 tensor (acnn_split3, acnn_prep_weights(planes = 3)); plane p of x
 * starts at x + p * numel(x), plane p of w at w + p * w_plane_stride elements; the six significant
 * cross products accumulate in fp32 register accumulators; requires out_f32 and no add / mask /
 * statistics epilogue. */
int acnn_conv_fprop(const acnn_conv_geom* g, const void* x, const void* w, void* y,
                    float* ch_part, const void* add_src, const void* mask_src,
                    const float* bias, int out_f32, int precision, int64_t w_plane_stride,
                    void* stream);
/* Rows of the partial statistics buffer acnn_conv_fprop(g, ..., ch_part, ...) writes without a fused
 * add / mask / bias (a pure function of the geometry, the conv knobs and the device's SM count;
 * <= 132; 0 for an empty output or a Cout that is not a positive multiple of 32).  A fused add, mask or
 * bias can move the launch to another kernel and grid (the 3x3 halo kernel runs no bias, and by
 * default only where the add / mask staging leaves its weight slab room): acnn_conv_fprop refuses
 * ch_part with ACNN_ERR_INVALID where that changes the row count, e.g. B = 1, 56 x 56, 64 -> 128
 * 3x3 with an add (25 rows against 28). */
int acnn_conv_stats_parts(const acnn_conv_geom* g);
/* *ctas = how many CTAs of the conv GEMM kernel acnn_conv_fprop(g, ..., precision) launches fit one
 * SM together (cudaOccupancyMaxActiveBlocksPerMultiprocessor at that launch's shared memory, with the
 * add / mask epilogue staging when has_add / has_mask); nothing is launched.  The bf16 and fp16
 * kernels are laid out for 2.  ACNN_ERR_INVALID for geometries on the 3x3 halo kernel. */
int acnn_conv_ctas_per_sm(const acnn_conv_geom* g, int precision, int has_add, int has_mask,
                          int* ctas);

/* dx[B,H,W,Cin] = conv_transpose(dy[B,Ho,Wo,Cout]) for a stride-1 conv of geometry g (the backward
 * of tf.layers.conv2d the reference gets from tf.gradients, nets/optimizer_setting.py:30).
 * w_dgrad is [Cin][kh][kw][Cout] with taps already flipped (acnn_prep_weights writes it).
 * Same optional add_src / mask_src epilogue as acnn_conv_fprop (shapes of dx).  precision 1: dy and
 * w_dgrad are 3-plane operands, dx is fp32 and no epilogue may be fused.  precision ACNN_F16: dy,
 * w_dgrad, dx, add_src and mask_src are fp16. */
int acnn_conv_dgrad(const acnn_conv_geom* g, const void* dy, const void* w_dgrad, void* dx,
                    const void* add_src, const void* mask_src, int precision,
                    int64_t w_plane_stride, void* stream);

/* dw[Cout,kh,kw,Cin] (fp32) += sum_pixels x (*) dy  -- weight gradient, split-K over pixels: the
 * splits store their partials in a stream-ordered scratch of the launch (cudaMallocAsync on `stream`)
 * and a second kernel on `stream` adds them to dw in split order (bit-reproducible).  dw must be zeroed
 * (or hold the running sum) by the caller.  deterministic != 0: no split (one add per element).
 * precision 1: x and dy are 3-plane operands.  precision ACNN_F16: x and dy are fp16. */
int acnn_conv_wgrad(const acnn_conv_geom* g, const void* x, const void* dy, float* dw,
                    int precision, int deterministic, void* stream);
/* The split layout acnn_conv_wgrad(g, ..., precision, deterministic, ...) would launch with the
 * current tuning knobs: *pix pixels per pipeline stage (128 only for bf16 with Cout < 256, i.e. an
 * N tile <= 128, and P = B*Ho*Wo >= 4096, unless acnn_set_wgrad_pixels(64); else 64), the P pixels
 * in ceil(P / pix) stages, *splits CTAs along them, every
 * split but the last running *stages_per_split stages (splits = ceil(stages / stages_per_split)).
 * Host only, callable without a GPU: without a device the SM count is taken as 132 (the H100's). */
int acnn_conv_wgrad_plan(const acnn_conv_geom* g, int precision, int deterministic, int* pix,
                         int* splits, int* stages_per_split);
/* planes bf16 [3][n] = (hi, mid, lo) of x fp32 [n], x = hi + mid + lo to 24 bits (n % 8 == 0). */
int acnn_split3(const float* x, void* planes, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batch normalisation (tf.layers.batch_normalization fused=True, nets/model_helper.py:26-37)
 * ------------------------------------------------------------------------------------------- */
/* Training: mean = sum/count, var = sumsq/count - mean^2 (biased), rstd = rsqrt(var + eps);
 * moving_mean <- m*moving_mean + (1-m)*mean, moving_var likewise with the UNBIASED variance.
 * stats_mode 0: stats = [nparts][2][C] partial (sum, sumsq) rows from acnn_conv_fprop, added here
 *               in a fixed order in double precision (so E[x^2] - E[x]^2 does not cancel in fp32);
 * stats_mode 1: stats = [mean | biased variance] from acnn_bn_stats (two-pass; nparts ignored).
 * Inference (training == 0): statistics are the moving ones, nothing is updated.
 * Outputs: scale = gamma*rstd, shift = beta - mean*scale, and mean / rstd for the backward. */
int acnn_bn_finalize(const float* stats, int nparts, int stats_mode, int64_t count,
                     const float* gamma, const float* beta, float* moving_mean, float* moving_var,
                     float momentum, float eps, int training, float* scale, float* shift,
                     float* mean, float* rstd, int C, void* stream);
/* Two-pass batch statistics of x [M][C] (fp32 parity mode): mean_var = [mean | biased variance],
 * fixed-order reductions (bit-reproducible). */
int acnn_bn_stats(const void* x, float* mean_var, int64_t M, int C, int dtype, void* stream);

/* out = bf16( relu?( (a*scale_a + shift_a) [* gate[b,c]] + R ) ), all NHWC [B,H,W,C]:
 *   b_mode 0: R = 0            1: R = b*scale_b + shift_b (projection shortcut BN)
 *          2: R = b (identity) 3: R = nearest-2x upsample of b[B,H/2,W/2,C] (Big-Little merge,
 *                                   nets/resnet_model.py:499-501)
 * Replaces BN-apply + tf.nn.relu + residual add (nets/resnet_model.py:55,72,92-95,414,501) and
 * the SE multiply (nets/blocks.py:183) when gate != NULL. */
int acnn_bn_act(const void* a, const float* scale_a, const float* shift_a, const void* b,
                const float* scale_b, const float* shift_b, int b_mode, const float* gate, int relu,
                void* out, int B, int H, int W, int C, int dtype, void* stream);

/* Backward of y -> bn -> (gate) given the gradient g w.r.t. the block output (already
 * ReLU-masked).  Effective gradient of the BN output: ge = g [* gate[b,c]] [+ addbc[b,c]] (the SE
 * gate and the SE pooled-descriptor term; both NULL for a plain BN).
 * parts[p][0:C] = partial sum_m ge, parts[p][C:2C] = partial sum_m ge*xhat, xhat = (y-mean)*rstd,
 * one row per CTA, p < acnn_bn_bwd_reduce_parts(B, HW, C) (plain stores: no atomics, no zeroing). */
int acnn_bn_bwd_reduce(const void* g, const void* y, const float* mean, const float* rstd,
                       const float* gate, const float* addbc, float* parts, int B, int HW, int C,
                       int dtype, void* stream);
int acnn_bn_bwd_reduce_parts(int B, int HW, int C);
/* sums = rows of `parts` added in index order (deterministic); dgamma = sums[C:2C], dbeta =
 * sums[0:C]; coef[0:C],[C:2C],[2C:3C] = k1,k2,k3 such that
 * dy = k1*ge + k2*y + k3  (= gamma*rstd*(ge - mean(ge) - xhat*mean(ge*xhat))). */
int acnn_bn_bwd_finalize(const float* parts, int nparts, const float* gamma, const float* mean,
                         const float* rstd, int64_t count, float* coef, float* dgamma, float* dbeta,
                         int C, void* stream);
int acnn_bn_bwd_apply(const void* g, const void* y, const float* coef, const float* gate,
                      const float* addbc, void* dy, int B, int HW, int C, int dtype, void* stream);
/* The same for TWO batch norms fed by one gradient g -- the block-final BN and the projection-
 * shortcut BN of a residual block's first unit, out = relu(bn_a(y_a) + bn_b(y_b))
 * (nets/resnet_model.py:42-45,81-97): g is read once per pass instead of twice.  parts_a / parts_b as
 * acnn_bn_bwd_reduce (acnn_bn_bwd_reduce_parts(B, HW, C) rows each); results bit-identical to the
 * single-BN entry points (no gate / addbc: not used with the SE gate). */
int acnn_bn_bwd_reduce2(const void* g, const void* ya, const void* yb, const float* mean_a,
                        const float* rstd_a, const float* mean_b, const float* rstd_b, float* parts_a,
                        float* parts_b, int B, int HW, int C, int dtype, void* stream);
int acnn_bn_bwd_apply2(const void* g, const void* ya, const void* yb, const float* coef_a,
                       const float* coef_b, void* dya, void* dyb, int B, int HW, int C, int dtype,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * Selective-kernel block after its 3x3 conv (nets/blocks.py:128-152).  y = raw conv output
 * [B,H,W,2f]; u = relu(y*scale+shift) is never materialised.
 * ------------------------------------------------------------------------------------------- */
/* s[B,f] (fp32) = mean_HW(u[..., :f] + u[..., f:])                         (blocks.py:128-132) */
int acnn_sk_gap(const void* y, const float* scale, const float* shift, float* s, int B, int HW,
                int f, int dtype, void* stream);
/* zpre = s*W1^T ; z = relu(BN_batch(zpre)) ; a = z*W2^T ; att = sigmoid(a[:, :f] - a[:, f:])
 * (2-way softmax over the halves, blocks.py:136-151).  w1 [d][f], w2 [2f][d] fp32 (OHWI 1x1).
 * bnstat[0:d] = mean, [d:2d] = rstd (batch statistics over B; moving stats when !training).
 * deterministic != 0 (here and in the three functions below): the small fp32 GEMMs run without
 * split-K, so every output receives one add (bit-reproducible). */
int acnn_sk_fc_fwd(const float* s, const float* w1, const float* gamma, const float* beta,
                   float* moving_mean, float* moving_var, float momentum, float eps, int training,
                   const float* w2, float* zpre, float* bnstat, float* z, float* att,
                   float* scratch /* acnn_sk_fc_scratch_floats(B, f, d) floats */, int B, int f, int d, int deterministic,
                   void* stream);
/* v[B,HW,f] = att*u0 + (1-att)*u1                                           (blocks.py:152) */
int acnn_sk_combine(const void* y, const float* scale, const float* shift, const float* att,
                    void* v, int B, int HW, int f, int dtype, void* stream);
/* dA[B,f] = sum_HW dv*(u0-u1) */
int acnn_sk_bwd_gate(const void* dv, const void* y, const float* scale, const float* shift,
                     float* dA, int B, int HW, int f, int dtype, void* stream);
/* Backward of the two fc layers + batch BN: consumes dA, produces ds[B,f] (gradient w.r.t. the
 * pooled descriptor) and ACCUMULATES dw1[d][f], dw2[2f][d], dgamma[d], dbeta[d]. */
int acnn_sk_fc_bwd(const float* dA, const float* att, const float* z, const float* zpre,
                   const float* bnstat, const float* gamma, const float* s, const float* w1,
                   const float* w2, float* dw1, float* dw2, float* dgamma, float* dbeta, float* ds,
                   float* scratch /* acnn_sk_fc_scratch_floats(B, f, d) floats */, int B, int f, int d, int deterministic,
                   void* stream);
/* g_h = (att_h*dv + ds/HW) * [u_h > 0] for both halves; partial rows as acnn_bn_bwd_reduce over 2f
 * channels, acnn_sk_bn_bwd_reduce_parts(B, HW, f) rows. */
int acnn_sk_bn_bwd_reduce(const void* dv, const void* y, const float* scale, const float* shift,
                          const float* mean, const float* rstd, const float* att, const float* ds,
                          float* parts, int B, int HW, int f, int dtype, void* stream);
int acnn_sk_bn_bwd_reduce_parts(int B, int HW, int f);
int acnn_sk_bn_bwd_apply(const void* dv, const void* y, const float* scale, const float* shift,
                         const float* att, const float* ds, const float* coef, void* dy, int B,
                         int HW, int f, int dtype, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Squeeze-excitation gate (nets/blocks.py:156-184), applied to t = bn(y) before the residual add
 * ------------------------------------------------------------------------------------------- */
/* q[B,C] (fp32) = mean_HW(y*scale + shift) */
int acnn_se_gap(const void* y, const float* scale, const float* shift, float* q, int B, int HW,
                int C, int dtype, void* stream);
/* h = relu(q*W1^T) [B,r]; e = sigmoid(h*W2^T) [B,C];  w1 [r][C], w2 [C][r] fp32. */
int acnn_se_fc_fwd(const float* q, const float* w1, const float* w2, float* h, float* e, int B,
                   int C, int r, int deterministic, void* stream);
/* de[B,C] = sum_HW g*t (t = y*scale+shift, g = masked grad of the block output) */
int acnn_se_bwd_gate(const void* g, const void* y, const float* scale, const float* shift,
                     float* de, int B, int HW, int C, int dtype, void* stream);
/* consumes de; ACCUMULATES dw1, dw2; dq[B,C] = gradient w.r.t. q, pre-divided by HW. */
int acnn_se_fc_bwd(const float* de, const float* e, const float* h, const float* q,
                   const float* w1, const float* w2, float* dw1, float* dw2, float* dq,
                   float* scratch /* >= B*(C+r) floats */, int B, int C, int r, int HW,
                   int deterministic, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pooling / resampling (all NHWC, element type `dtype`).  Backward kernels take the same optional
 * epilogue as the convs: (+ add_src) then (* (mask_src > 0)).
 * ------------------------------------------------------------------------------------------- */
/* Anti-alias blur-pool: REFLECT pad (filt-1)/2, binomial filt x filt / sum, stride, VALID
 * (nets/blocks.py:45-107).  filt in [1,7]. */
int acnn_blurpool_fwd(const void* x, void* out, int B, int H, int W, int C, int filt, int stride,
                      int dtype, void* stream);
int acnn_blurpool_bwd(const void* dout, void* dx, const void* add_src, const void* mask_src, int B,
                      int H, int W, int C, int filt, int stride, int dtype, void* stream);
/* Average pool k x k, zero padding pad_lo before (pad after implied by Ho).  count_pad != 0:
 * divide by k*k (bl shortcut, resnet_model.py:133-138); else by the number of in-bounds cells
 * (TF SAME, resnet-d stride-1 shortcut :126). */
int acnn_avgpool_fwd(const void* x, void* out, int B, int H, int W, int C, int k, int stride,
                     int pad_lo, int Ho, int Wo, int count_pad, int dtype, void* stream);
int acnn_avgpool_bwd(const void* dout, void* dx, const void* add_src, const void* mask_src, int B,
                     int H, int W, int C, int k, int stride, int pad_lo, int Ho, int Wo,
                     int count_pad, int dtype, void* stream);
/* Max pool k x k, -inf padding, pad_lo before (TF SAME puts the odd cell after: pad_lo = 0 for
 * 3x3/s2 on even sizes, resnet_model.py:421-424).  Backward routes to the FIRST maximum. */
int acnn_maxpool_fwd(const void* x, void* out, int B, int H, int W, int C, int k, int stride,
                     int pad_lo, int Ho, int Wo, int dtype, void* stream);
int acnn_maxpool_bwd(const void* dout, const void* x, void* dx, const void* add_src,
                     const void* mask_src, int B, int H, int W, int C, int k, int stride,
                     int pad_lo, int Ho, int Wo, int dtype, void* stream);
/* dx[B,H,W,C] = 2x2 block sums of dout[B,2H,2W,C] (backward of UpSampling2D) */
int acnn_upsample2x_bwd(const void* dout, void* dx, const void* add_src, const void* mask_src,
                        int B, int H, int W, int C, int dtype, void* stream);
/* out[B,H,W,C]: out[2p,2q] = dy[p,q], zeros elsewhere (stride-2 dgrad = zero-insert + stride-1) */
int acnn_zero_insert2x(const void* dy, void* out, int B, int Ho, int Wo, int H, int W, int C,
                       int dtype, void* stream);
/* out = (a [+ add_src]) [* (mask_src > 0)] over n bf16 elements: gradient merge when no consumer
 * kernel can fuse it (identity shortcut as last contribution). */
int acnn_grad_combine(const void* a, const void* add_src, const void* mask_src, void* out,
                      int64_t n, int dtype, void* stream);
/* pooled[B,C] = mean_HW(x)                                     (nets/resnet_model.py:560-561) */
int acnn_gap_fwd(const void* x, void* pooled, int B, int HW, int C, int dtype, void* stream);
/* dx = dpooled[b,c]/HW * (mask_src > 0) */
int acnn_gap_bwd(const void* dpooled, const void* mask_src, void* dx, int B, int HW, int C,
                 int dtype, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Input packing / mixup (utils/data_util.py:97-158) and the loss (losses/cls_losses.py:28-33)
 * ------------------------------------------------------------------------------------------- */
/* images fp32 NHWC [Bin,H,W,3] -> bf16 space-to-depth(2) [B,H/2,wpad_lo + W/2 + wpad_hi,16]
 *   (channel = (dy*2+dx)*4 + c, c==3 is zero) so that the stride-2 stem conv becomes a stride-1
 *   conv with 16 input channels; the W axis is physically zero-padded so that the stem can read
 *   k2 horizontally adjacent pixels as one k2*16-channel pixel (acnn_conv_geom.x_pix_stride).  mode 0: B = Bin (copy); 1: mixup type 1, B = Bin/2,
 *   out = lam1*x[:B] + (1-lam1)*x[B:]; 2: mixup type 2, B = Bin, second half uses lam2 and the
 *   reversed second half. */
int acnn_pack_input(const float* images, const float* lam1, const float* lam2, int mode, void* out,
                    int Bin, int H, int W, int wpad_lo, int wpad_hi, int dtype, void* stream);
/* y[B,NC] (fp32) = (mixed) one-hot labels, same modes. */
int acnn_mix_labels(const int32_t* labels, const float* lam1, const float* lam2, int mode, float* y,
                    int Bin, int NC, void* stream);
/* Softmax cross-entropy with label smoothing, mean over B: loss_acc[0] += loss (caller zeroes).
 * dlogits (`dtype` [B,ld], columns >= NC zeroed) = (softmax - y')/B * grad_scale;
 * dbias[NC] (fp32) += column sums of the fp32 dlogits.  logits fp32 [B,ld].  Two launches: per-row
 * losses / gradients, then a fixed-order sum (no atomics: bit-reproducible).
 * teacher != NULL adds the knowledge-distillation term (nets/run_loop_classification.py:156-162):
 * loss_acc[2] += kd_temp^2 * mean_b CE(logits / kd_temp, teacher[b]) and its gradient to dlogits /
 * dbias; teacher [B,NC] = (mixed) softmax(teacher_logits / kd_temp) from acnn_kd_teacher_labels.
 * work: >= 2*roundup(B, 32) + B*ld floats of scratch. */
int acnn_softmax_ce(const float* logits, const float* y, const float* teacher, float kd_temp, int B,
                    int NC, int ld, float label_smoothing, float grad_scale, float* loss_acc,
                    void* dlogits, float* dbias, float* work, int dtype, void* stream);
/* acnn_softmax_ce with grad_scale read from DEVICE memory when the kernel runs (the scale of a dynamic
 * loss-scale state, acnn_loss_scale_state.scale), so a captured graph follows its changes. */
int acnn_softmax_ce_scaled(const float* logits, const float* y, const float* teacher, float kd_temp, int B,
                           int NC, int ld, float label_smoothing, const float* grad_scale_dev,
                           float* loss_acc, void* dlogits, float* dbias, float* work, int dtype,
                           void* stream);
/* Teacher labels of knowledge distillation: softmax(teacher_logits[Bin,NC] / kd_temp) mixed with the
 * images' mixup pairing (utils/data_util.py:128-156, modes as acnn_pack_input; the second half of a
 * type-2 batch mixes the supervised one-hot of `labels`, as the reference does at :154). */
int acnn_kd_teacher_labels(const float* teacher_logits, const int32_t* labels, const float* lam1,
                           const float* lam2, int mode, float kd_temp, float* yt, int Bin, int NC,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * DropBlock (nets/blocks.py:187-251; call sites nets/resnet_model.py:35-97,432-453) and GeM pooling
 * (nets/blocks.py:22-42)
 * ------------------------------------------------------------------------------------------- */
/* keep[H,W,C] (fp32, ONE mask for the whole batch, as the reference samples it) = 1 - dilation by a
 * block_size window of bernoulli(gamma) drawn on the [H-bs+1, W-bs+1, C] interior and zero-padded;
 * gamma = gamma_scale * (1 - keep_prob) * H*W / bs^2 / ((H-bs+1)(W-bs+1)); *scale = H*W*C /
 * (sum(keep) + 1e-8).  keep_prob is read from DEVICE memory (it follows a schedule,
 * functions/model_fns.py:26-33,221-228).  u != NULL supplies the uniform draws [hs,ws,C] (parity
 * tests); otherwise Philox4x32-10 keyed by `seed` with counter (element, *step).
 * scratch: acnn_dropblock_scratch_floats(H, W, C, block_size) floats. */
int acnn_dropblock_mask(const float* u, const float* keep_prob, const uint32_t* step, uint64_t seed,
                        float gamma_scale, int block_size, float* keep, float* scale,
                        float* scratch, int H, int W, int C, void* stream);
int acnn_dropblock_scratch_floats(int H, int W, int C, int block_size);
/* out[B,HW,C] = relu?(x * keep[HW,C] * *scale); with relu = 0 also the backward on gradients. */
int acnn_dropblock_apply(const void* x, const float* keep, const float* scale, int relu, void* out,
                         int B, int HW, int C, int dtype, void* stream);
/* pooled[B,C] = HW^(-1/3) * cbrt(max(S, 1e-6)), S[B,C] (fp32, kept for the backward) =
 * sum_hw clip(x, 1e-6, 1e12)^3;  dx = dpooled * HW^(-1/3) * S^(-2/3) * x^2 inside the clip range. */
int acnn_gem_fwd(const void* x, void* pooled, float* ssum, int B, int HW, int C, int dtype,
                 void* stream);
int acnn_gem_bwd(const void* dpooled, const float* ssum, const void* x, void* dx, int B, int HW,
                 int C, int dtype, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Parameters and optimizer (nets/optimizer_setting.py:23-38, run_loop_classification.py:166-179)
 * ------------------------------------------------------------------------------------------- */
/* One conv weight tensor of the flat fp32 master buffer. */
typedef struct acnn_weight_desc {
  int64_t master_off; /* elements, into the fp32 master buffer ([Cout][taps][Cin]) */
  int64_t fprop_off;  /* elements, into the bf16 fprop buffer  ([Cout][taps][Cin]) */
  int64_t dgrad_off;  /* elements, into the bf16 dgrad buffer  ([Cin][taps flipped][Cout]); <0: none */
  int32_t Cout, taps, Cin;
  int32_t pad_;
} acnn_weight_desc;
/* bf16 operand copies of every conv weight (fprop layout + flipped/transposed dgrad layout).
 * `descs` is a DEVICE array of n descriptors.  planes = 1: one bf16 copy; planes = 3 (fp32 parity
 * mode): hi / mid / lo planes, plane p at element offset p * {fprop,dgrad}_plane_stride. */
int acnn_prep_weights(const float* master, const acnn_weight_desc* descs, int n, void* w_fprop,
                      void* w_dgrad, int planes, int64_t fprop_plane_stride,
                      int64_t dgrad_plane_stride, void* stream);
/* The same with ONE fp16 copy of each layout (ACNN_F16: the fp32 master read as fp16, rounded to
 * nearest even; a weight beyond the fp16 range becomes +-inf). */
int acnn_prep_weights_f16(const float* master, const acnn_weight_desc* descs, int n, void* w_fprop,
                          void* w_dgrad, void* stream);
/* Stem: master [Cout][k][k][3] fp32 -> bf16 [Cout][k2][k2][16] for the space-to-depth input
 * (k2 taps, see acnn_pack_input); and the inverse gather-add for its gradient. */
int acnn_s2d_weight_pack(const float* w, void* w2, int Cout, int k, int pad, int k2, int pad2,
                         int dtype, void* stream);
int acnn_s2d_wgrad_unpack(const float* dw2, float* dw, int Cout, int k, int pad, int k2, int pad2,
                          void* stream);
/* Fused weight decay + momentum SGD over a flat buffer:
 *   g = grad*hp[3] + (decay ? hp[2]*w : 0);  acc = hp[1]*acc + g;  w -= hp[0]*acc
 * hp = device float[4] {lr, momentum, weight_decay, grad_scale}; decay_flag: one byte per 256
 * elements.  l2_acc[0] += sum over decayed elements of w^2/2 (pre-update), times weight_decay;
 * the per-CTA partial sums are added in index order by the last CTA to finish (bit-reproducible).
 * scratch: acnn_sgd_scratch_floats() floats, ZERO before the first call (self-resetting after). */
int acnn_sgd_momentum(float* w, const float* grad, float* acc, int64_t n,
                      const uint8_t* decay_flag, const float* hp, float* l2_acc, float* scratch,
                      void* stream);
int acnn_sgd_scratch_floats(void);
int acnn_fill_zero(void* p, int64_t bytes, void* stream);

/* Dynamic loss scaling, decided and applied on the device (the rules of TF 2 Keras' LossScaleOptimizer).
 * A step's loss seed is scale / B (acnn_softmax_ce_scaled); after the backward (and any gradient sum or
 * all-reduce) acnn_grads_nonfinite tests the gradient buffer, acnn_sgd_momentum_loss_scaled applies or skips
 * the update and acnn_loss_scale_update moves the scale:
 *   finite step:      update with grad_scale 1 / (grad_divisor * scale); good_steps += 1; when good_steps
 *                     reaches growth_interval, scale *= 2 (kept only if finite) and good_steps = 0
 *   non-finite step:  w and acc untouched; scale = max(scale / 2, 1); good_steps = 0; skipped_steps += 1
 * Nothing reaches the host: the sequence replays in a CUDA graph.  32 bytes of DEVICE memory: */
typedef struct acnn_loss_scale_state {
  float scale;            /* the loss scale of the next step */
  int32_t good_steps;     /* finite steps since the scale last changed */
  int32_t skipped_steps;  /* non-finite steps so far */
  uint32_t nonfinite;     /* != 0: the gradients of the step in flight are not all finite; 0 between steps */
  float last_scale;       /* the scale the last updated step ran with */
  int32_t reserved_[3];
} acnn_loss_scale_state;
/* *flag = 1 when any of the fp32 x[0, n) is +-inf or NaN (isfinite per element); nothing is written
 * otherwise, so the caller clears it (acnn_loss_scale_update does).  One pass in float4 vectors (scalar head
 * and tail); an OR of per-element tests, independent of the grid and of the order of the CTAs.  x: 4-byte
 * aligned. */
int acnn_grads_nonfinite(const float* x, int64_t n, uint32_t* flag, void* stream);
/* acnn_sgd_momentum with the gradient scale taken from `ls`: grad_scale = (float)(1 / (grad_divisor *
 * ls->scale)) computed in double and rounded once (grad_divisor: the data-parallel replicas the gradient
 * sums, world * replicas per device); hp[3] is not read.  ls->nonfinite != 0 leaves w and acc bit for bit as
 * they were and still adds the L2 sum to l2_acc. */
int acnn_sgd_momentum_loss_scaled(float* w, const float* grad, float* acc, int64_t n,
                                  const uint8_t* decay_flag, const float* hp,
                                  const acnn_loss_scale_state* ls, int grad_divisor, float* l2_acc,
                                  float* scratch, void* stream);
/* The scale update of the rules above from state->nonfinite, then state->last_scale = the scale the step
 * used and state->nonfinite = 0.  One thread. */
int acnn_loss_scale_update(acnn_loss_scale_state* state, int growth_interval, void* stream);

/* Several data-parallel replicas run one after another on one device (micro-steps r = 0 .. R-1 of one
 * global step, each a full forward + backward from the same moving statistics).  One fused pass per
 * micro-step over the gradient range [lo, hi) (grads and acc_grads at the same offsets) and the first
 * n_state floats of the state buffers, in fp32, element by element:
 *   SAVE   (before micro-step 0)        state_base = state; the gradients are not touched
 *   FIRST  (after micro-step 0)         acc = g;        acc_state = state;        state = state_base
 *   MIDDLE (after micro-steps 1 .. R-2) acc = acc + g;  acc_state = acc_state + state;  state = state_base
 *   LAST   (after micro-step R-1)       g = acc + g;    state = (acc_state + state) * state_scale
 * so the gradient ends as ((g0 + g1) + g2) + ... and, with state_scale = 1/R, the state as the mean of the
 * R updated copies summed in replica order.  state_base may be NULL outside SAVE: the state is then left
 * as it is (a buffer the next micro-step clears itself, such as the loss).  No atomics; any alignment
 * (16-byte vectors where the pointers of a part share their alignment).  Capturable. */
#define ACNN_REPLICA_SAVE 0
#define ACNN_REPLICA_FIRST 1
#define ACNN_REPLICA_MIDDLE 2
#define ACNN_REPLICA_LAST 3
int acnn_replica_accumulate(int phase, float* acc_grads, float* grads, float* state_base, float* acc_state,
                            float* state, int64_t lo, int64_t hi, int64_t n_state, float state_scale,
                            void* stream);

/* ---------------------------------------------------------------------------------------------
 * Zero-shot retrieval (metric/recall_metric.py:98-123: l2_normalize / tf_simple_pairwise_distance,
 * MatMul and tf.nn.top_k over the query x index similarity matrix, which is never materialised)
 * ------------------------------------------------------------------------------------------- */
/* For every query row q of Q[nq][d] (fp32): the k rows of X[nx][d] (fp32) with the largest similarity,
 * sorted by (similarity descending, index ascending) -- tf.nn.top_k's order, lower index first on ties.
 * metric 0 = cosine: rows l2-normalised first (tf.nn.l2_normalize: x * rsqrt(max(sum x^2, 1e-12)));
 * metric 1 = euclidean: -((|q|^2 + |x|^2) - 2 q.x) on the raw rows (tf_simple_pairwise_distance,
 * negated), the squared norms taken over the rounded operands.
 * dtype ACNN_BF16: bf16 operands, fp32 accumulation; ACNN_F32: three bf16 planes per operand (as the
 * conv GEMMs), whose six significant cross products are accumulated in fp32; ACNN_F16: fp16 operands
 * (round to nearest even; a row with an entry beyond +-65504 after the normalisation gets an infinite
 * operand and is not ranked), fp32 accumulation -- the reference's fp16 search
 * (metric/recall_metric.py:68-73).
 * out_idx int32 [nq][k], out_sim fp32 [nq][k].  Any d >= 1 (<= 2^24); 1 <= k <= 128 (k > 128:
 * ACNN_ERR_UNSUPPORTED); k > nx, non-positive sizes, an unknown metric or dtype: ACNN_ERR_INVALID.
 * All of these are checked before any CUDA call.  The result is the same bit for bit for every
 * column-split count, grid and stream.  Only similarities above -inf are ranked: a row with fewer
 * than k of them (a NaN or infinite input, or a squared distance that overflows fp32) is padded with
 * (similarity -inf, index 2147483647) entries -- callers that index with out_idx must check for it.
 * work: acnn_knn_work_bytes(...) bytes, caller-owned; every section starts at a 256-byte boundary:
 *   Q' bf16 [nq][K'], X' bf16 [nx][K']  (fp16 for ACNN_F16; K' = P * roundup(d, 64), zero-padded; P = 1 for bf16 / fp16, 6 for
 *        fp32: K' holds six d-segments so that one bf16 GEMM forms the six plane products, smallest
 *        first -- Q' = (hi, mid, lo, hi, mid, hi), X' = (lo, mid, hi, mid, hi, hi))
 *   |q|^2 fp32 [nq], |x|^2 fp32 [nx]   (of the rounded operands: bf16 / fp16, or (hi + mid) + lo)
 *   partial lists: similarity fp32 [8][nq][k], index int32 [8][nq][k]  (one per column split) */
int acnn_knn_topk(const float* q, const float* x, int nq, int nx, int d, int k, int metric, int dtype,
                  int32_t* out_idx, float* out_sim, void* work, int64_t work_bytes, void* stream);
/* Bytes of the `work` argument (host only, callable without a GPU); -1 for invalid sizes. */
int64_t acnn_knn_work_bytes(int nq, int nx, int d, int k, int dtype);
/* Tuning knob of acnn_knn_topk (no effect on results): n > 0 forces n column splits, clamped to
 * [1, min(8, ceil(nx / 128))]; 0 (default) = the cost model that fills the SMs.  Returns the previous
 * setting. */
int acnn_set_knn_splits(int n);
/* Search of a prepared index, for serving: the prep of X is run once (acnn_knn_prepare_index) and
 * each query batch prepares only its own rows (acnn_knn_search).
 * acnn_knn_prepare_index: X[nx][d] (fp32) -> `index`, caller-owned, 256-byte aligned, of
 * acnn_knn_index_bytes(nx, d, dtype) bytes: X' [nx][K'] then, at the next 256-byte boundary, |x|^2 fp32
 * [nx], the formats of acnn_knn_topk's work sections (metric as there: 0 cosine, 1 euclidean).
 * acnn_knn_search: for every row of Q[nq][d] (fp32) the k best rows of a prepared index, which must
 * have been prepared with the same nx, d, metric and dtype.  Results, padding and argument rules are
 * acnn_knn_topk's, and equal to acnn_knn_topk(Q, X) bit for bit.  The index is read only, so one index
 * may serve concurrent searches with separate work buffers.  The column splits come from acnn_knn_topk's
 * cost model (acnn_set_knn_splits applies too) with up to one split per SM: at most min(SMs, 132,
 * ceil(nx / 128)).  work: acnn_knn_search_work_bytes(...) bytes, caller-owned, 256-byte aligned:
 *   Q' [nq][K'], |q|^2 fp32 [nq], partial lists: similarity fp32 [S][nq][k], index int32 [S][nq][k]
 *   (S = min(132, ceil(nx / 128))), then, when S > 16, the lists of the first 16-way merge pass
 *   (similarity fp32 [ceil(S / 16)][nq][k], index int32 [ceil(S / 16)][nq][k]).
 * Both byte counts are host only (callable without a GPU); -1 for invalid sizes. */
int64_t acnn_knn_index_bytes(int nx, int d, int dtype);
int acnn_knn_prepare_index(const float* x, int nx, int d, int metric, int dtype, void* index,
                           int64_t index_bytes, void* stream);
int64_t acnn_knn_search_work_bytes(int nq, int nx, int d, int k, int dtype);
int acnn_knn_search(const float* q, int nq, const void* index, int nx, int d, int k, int metric, int dtype,
                    int32_t* out_idx, float* out_sim, void* work, int64_t work_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Robustness evaluation (mce/eval_robustness.py: ImageNet-C corruption error)
 * ------------------------------------------------------------------------------------------- */
/* out fp32 NHWC [B,H,W,3] = (float)images[b,h,w,c] - mean[c], images uint8 NHWC [B,H,W,3] (DEVICE):
 * the tf.cast + mean_image_subtraction of input_fn_imagenet_c (mce/eval_robustness.py:123-148), the same
 * fp32 subtraction.  mean: float[3], a host or a device array (a device one is read by the kernel, a
 * host one when the call enqueues).  images and out must be 16-byte aligned. */
int acnn_images_from_u8(const uint8_t* images, const float* mean, float* out, int B, int H, int W,
                        void* stream);
/* tf.nn.top_k(tf.nn.softmax(logits), 1) and the top-1 count of mce/eval_robustness.py:186-187,214-229.
 * logits fp32 [B][ld] (columns < NC are the classes), labels int32 [B].  For every row r < n_valid:
 * p_j = expf(x_j - max) / sum (the sum in a fixed order), pred[r] = the SMALLEST j with the largest p_j
 * (tf.nn.top_k's rule applied to the fp32 probabilities: two distinct logits whose probabilities round
 * to the same float tie, and the lower index wins), and *correct += 1 when pred[r] == labels[r].
 * A row with a NaN or infinite logit gets pred[r] = -1 and is never counted as correct.
 * Rows >= n_valid are padding: neither pred nor the count is touched for them.  The count uses integer
 * atomics, so the result is the same under CUDA-graph replay and on concurrent streams.
 * Null pointers, B < 1, NC < 1, ld < NC, n_valid outside [0, B]: ACNN_ERR_INVALID before any CUDA call;
 * n_valid = 0 launches nothing. */
int acnn_softmax_top1_count(const float* logits, int B, int ld, int NC, const int32_t* labels, int n_valid,
                            int32_t* pred, uint64_t* correct, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Classification evaluation (classifier.evaluate(input_fn_eval), nets/run_loop_classification.py)
 * ------------------------------------------------------------------------------------------- */
/* One decoded image of a batch: uint8 RGB [src_h][src_w][3] at `src` (DEVICE), resized to
 * [rsz_h][rsz_w] and cropped to the S x S window at (crop_y, crop_x).  32 bytes, the layout of
 * imagenet_eval.DESC_DTYPE. */
typedef struct acnn_resize_desc {
  const uint8_t* src;
  int32_t src_h, src_w;
  int32_t rsz_h, rsz_w;
  int32_t crop_y, crop_x;
} acnn_resize_desc;
/* out fp32 NHWC [B,S,S,3], row b < n_valid = central_crop(resize_bilinear(img_b, rsz_h, rsz_w), S, S)
 * - mean[c]: the eval preprocessing of preprocessing/imagenet_preprocessing.py:295-313.  The resize is
 * TF 1.14's legacy bilinear (align_corners = false, half_pixel_centers = false), bit for bit:
 * scale = (float)src / rsz, in = i * scale, lower = max(floor(in), 0), upper = min(ceil(in), src - 1),
 * lerp = in - floor(in), top = tl + (tr - tl) * x_lerp, bottom likewise, out = top + (bottom - top) *
 * y_lerp, then - mean[c]; every step a separately rounded fp32 operation (no FMA).  Only the S x S
 * pixels the crop keeps are computed, at resized coordinates (y + crop_y, x + crop_x).
 * desc: a DEVICE array of B descriptors (a captured CUDA graph holds only its address, so the image
 * buffers it points to may move between replays).  The descriptors are not checked here: the caller
 * guarantees src_h, src_w >= 1, 0 <= crop_y <= rsz_h - S, 0 <= crop_x <= rsz_w - S.  mean: float[3],
 * host or device.  Rows >= n_valid are not written.  Null pointers, B < 1, S < 1, n_valid outside
 * [0, B], out not 4-byte or desc not 8-byte aligned: ACNN_ERR_INVALID before any CUDA call. */
int acnn_resize_crop_u8(const acnn_resize_desc* desc, int B, int n_valid, int S, const float* mean, float* out,
                        void* stream);
/* One training crop window of a batch: uint8 RGB [h][w][3] at `src` (DEVICE), the window the host cut out
 * of the decoded image (sample_distorted_bounding_box + decode_and_crop_jpeg), mirrored when flip != 0.
 * 32 bytes, the layout of imagenet_train.CROP_DESC_DTYPE. */
typedef struct acnn_crop_desc {
  const uint8_t* src;
  int32_t h, w;
  int32_t flip;
  int32_t reserved_[3];
} acnn_crop_desc;
/* out fp32 NHWC [B,S,S,3], row b < n_valid = resize_bilinear(flip_b ? mirror(window_b) : window_b, S, S)
 * - mean[c]: the training preprocessing of preprocessing/imagenet_preprocessing.py:57-97,269-313 after the
 * crop (random_flip_left_right, _resize_image, mean_image_subtraction).  The resize is TF 1.14's legacy
 * bilinear with the independent scales (float)h / S and (float)w / S, every step a separately rounded fp32
 * operation, as in acnn_resize_crop_u8; the result stays fp32.  The flip comes before the resize, whose
 * sample grid is anchored at the left edge, so a mirrored window reads source columns w - 1 - lower and
 * w - 1 - upper.  A 1 x 1 window (scale < 1, upsampling) is valid.
 * desc: a DEVICE array of B descriptors (a captured CUDA graph holds only its address).  The descriptors
 * are not checked here: the caller guarantees src != 0 and h, w >= 1.  mean: float[3], host or device.
 * Rows >= n_valid are not written.  Null pointers, B < 1, S < 1, n_valid outside [0, B], out not 4-byte
 * or desc not 8-byte aligned: ACNN_ERR_INVALID before any CUDA call. */
int acnn_crop_resize_u8(const acnn_crop_desc* desc, int B, int n_valid, int S, const float* mean, float* out,
                        void* stream);
/* AutoAugment (preprocessing/autoaugment.py distort_image_with_autoaugment) of one training image: the two
 * operations of the sub-policy drawn for it, resolved on the host (assembled_cnn_b200/autoaugment.py).
 * An operation that does not apply has op = ACNN_AA_IDENTITY.  Arguments per op:
 *   POSTERIZE     i[0] = shift in [0, 7] (8 - bits, clamped as TF's shift ops do): (x >> i0) << i0
 *   SOLARIZE      i[0] = threshold in [0, 255] (the uint8 constant):  x < i0 ? x : 255 - x
 *   SOLARIZE_ADD  i[0] = addition >= 0:  x < 128 ? min(x + i0, 255) : x
 *   COLOR, BRIGHTNESS, SHARPNESS, CONTRAST  f[0] = blend factor >= 0; CONTRAST i[0] = its grey in [0, 255]
 *   ROTATE, SHEAR_X, SHEAR_Y, TRANSLATE_X, TRANSLATE_Y  f[0..5] = the projective transform t0..t5
 *   CUTOUT        i[0] = centre row, i[1] = centre column, i[2] = pad size
 * 88 bytes, the layout of autoaugment.AUTOAUG_DESC_DTYPE. */
enum {
  ACNN_AA_IDENTITY = 0, ACNN_AA_AUTOCONTRAST, ACNN_AA_EQUALIZE, ACNN_AA_INVERT, ACNN_AA_ROTATE, ACNN_AA_POSTERIZE,
  ACNN_AA_SOLARIZE, ACNN_AA_SOLARIZE_ADD, ACNN_AA_COLOR, ACNN_AA_CONTRAST, ACNN_AA_BRIGHTNESS, ACNN_AA_SHARPNESS,
  ACNN_AA_SHEAR_X, ACNN_AA_SHEAR_Y, ACNN_AA_TRANSLATE_X, ACNN_AA_TRANSLATE_Y, ACNN_AA_CUTOUT, ACNN_AA_NUM_OPS
};
typedef struct acnn_autoaugment_op {
  int32_t op;
  int32_t i[3];
  float f[6];
} acnn_autoaugment_op;
typedef struct acnn_autoaugment_desc {
  int32_t subpolicy;                 /* the drawn sub-policy (informational; the kernel does not read it) */
  int32_t reserved_;
  acnn_autoaugment_op slot[2];
} acnn_autoaugment_desc;
/* Bytes of the `work` buffer acnn_crop_resize_autoaugment_u8 needs for B images of S x S: two uint8 planes
 * per image, each S*S*3 bytes rounded up to 16.  -1 for B < 1, S < 1 or a size that overflows. */
int64_t acnn_autoaugment_work_bytes(int B, int S);
/* out fp32 NHWC [B,S,S,3], row b < n_valid = (float)autoaugment(trunc(clip(resize(window_b), 0, 255)))
 * - mean[c]: the training preprocessing of preprocessing/imagenet_preprocessing.py:269-313 with
 * autoaugment_type set.  The resize is acnn_crop_resize_u8's, bit for bit; then clip_by_value(0, 255) and a
 * truncating cast to uint8 (for every image, also when no operation applies), aug_b's two operations in
 * order on the uint8 image, each float step a separately rounded fp32 operation, then the cast to fp32 and
 * the mean.  One CTA per image; the image lives in two planes of `work` (DEVICE, acnn_autoaugment_work_bytes
 * (B, S) bytes, 16-byte aligned); histograms and minima / maxima are integer shared-memory atomics, so the
 * result does not depend on the order of execution.  desc, aug: DEVICE arrays of B descriptors, checked by
 * the caller (acnn_crop_resize_u8; autoaugment.check_autoaugment_descriptors).  mean: float[3], host or
 * device.  Rows >= n_valid are not written.  Null pointers, B < 1, S < 1, n_valid outside [0, B], out not
 * 4-byte, desc or aug not 8-byte, work not 16-byte aligned: ACNN_ERR_INVALID before any CUDA call. */
int acnn_crop_resize_autoaugment_u8(const acnn_crop_desc* desc, const acnn_autoaugment_desc* aug, int B,
                                    int n_valid, int S, const float* mean, uint8_t* work, float* out,
                                    void* stream);
/* Per-row results of the classification metrics for logits fp32 [B][ld] (columns < NC are the
 * classes) and labels int32 [B], for every row r < n_valid (rows >= n_valid are not written):
 *   pred[r]  = tf.argmax(logits): the smallest index of the largest logit;
 *   conf[r]  = the largest softmax probability, 1 / sum_j expf(x_j - max) (the sum in a fixed order);
 *   hit_k[r] = tf.nn.in_top_k(logits, label, k): 1 when fewer than k logits are strictly greater than
 *              the label's (ties count as in), 0 when the label is outside [0, NC);
 *   ce[r]    = -((1 - ls) log p[label] + ls / NC sum_j log p_j), tf.losses.softmax_cross_entropy with
 *              label_smoothing = ls; NaN when the label is outside [0, NC).
 * A row with a NaN or infinite logit gets pred = -1, conf = NaN, hit_k = 0, ce = NaN.  No atomics:
 * the results are the same under CUDA-graph replay and on concurrent streams.  Null pointers, B < 1,
 * NC < 1, ld < NC, n_valid outside [0, B], k < 1, a non-finite ls: ACNN_ERR_INVALID before any CUDA
 * call; n_valid = 0 launches nothing. */
int acnn_classify_rows(const float* logits, int B, int ld, int NC, const int32_t* labels, int n_valid, int k,
                       float label_smoothing, int32_t* pred, float* conf, int32_t* hit_k, float* ce,
                       void* stream);
/* The PREDICT-mode `predictions` dict of nets/run_loop_classification.py:126-130 for logits fp32 [B][ld]
 * (columns < NC are the classes), for every row r < n_valid (rows >= n_valid are not written):
 *   classes[r]                   = tf.argmax(logits, 1): the smallest index of the largest logit.  An
 *                                  infinite logit is an ordinary value (a row of -inf only gets 0); a row
 *                                  holding a NaN gets -1.  (acnn_softmax_top1_count gives -1 for any
 *                                  non-finite logit: its rule is about the probabilities, not the logits.)
 *   probabilities[r][j]          = expf(x_j - max) / sum_j expf(x_j - max), the sum in a fixed order;
 *                                  a row with +inf, or only -inf, gives NaN as tf.nn.softmax does;
 *   probabilities_sigmoid[r][j]  = 1 / (1 + expf(-x_j)).
 * probabilities and probabilities_sigmoid are dense [B][NC].  One CTA per row, no atomics: the results are
 * the same under CUDA-graph replay and on concurrent streams.  Null pointers, B < 1, NC < 1, ld < NC,
 * n_valid outside [0, B]: ACNN_ERR_INVALID before any CUDA call; n_valid = 0 launches nothing. */
int acnn_predict_rows(const float* logits, int B, int ld, int NC, int n_valid, int32_t* classes, float* probabilities,
                      float* probabilities_sigmoid, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training-batch metrics (the training summaries of nets/run_loop_classification.py:146-227)
 * ------------------------------------------------------------------------------------------- */
/* Device accumulator of the training metrics (280 bytes, the layout of metrics.TRAIN_METRICS_DTYPE);
 * zeroed by the caller.  Streaming fields, kept until the caller zeroes them again: */
#define ACNN_ECE_BINS 10
typedef struct acnn_train_metrics {
  int64_t rows;                            /* rows accumulated */
  int64_t top1;                            /* rows with pred == label (pred = -1 is wrong) */
  int64_t top5;                            /* rows with hit_k != 0 */
  int64_t bin_count[ACNN_ECE_BINS];        /* rows whose confidence falls in bin b */
  int64_t bin_correct[ACNN_ECE_BINS];      /*   ... and whose pred == label */
  double bin_conf[ACNN_ECE_BINS];          /*   the sum of their confidences */
  /* per-step fields, cleared by the call with step_begin != 0: */
  int64_t step_rows;
  double step_conf;                        /* the sum of conf over the step's rows (NaN rows included) */
} acnn_train_metrics;
/* Adds the rows r < n of one micro-step to *m, from acnn_classify_rows' pred, conf and hit_k (k = 5) and the
 * labels int32 [n].  Bins are (lo, hi] over the float32 thresholds [-1e-7, 0.1, ..., 0.9, 1 + 1e-7], as
 * metrics.classification_result; a NaN confidence falls in no bin.  Counts are int64.  Every fp64 sum has one
 * order: row r goes to lane r % 256, each lane adds its rows in ascending order to 0.0, lane partials are
 * combined by the tree  p[i] = p[i] + p[i + s]  for s = 128, 64, ..., 1 (i < s), and the field then becomes
 * field + p[0] (step_conf: p[0] when step_begin != 0).  One CTA, no atomics: the same bits on every replay
 * and stream.  Capturable.  Null pointers, n < 1, m not 8-byte aligned: ACNN_ERR_INVALID before any CUDA
 * call. */
int acnn_train_metrics_accumulate(const int32_t* pred, const float* conf, const int32_t* hit_k, const int32_t* labels,
                                  int n, int step_begin, acnn_train_metrics* m, void* stream);

/* ---------------------------------------------------------------------------------------------
 * JPEG decoding (the tf.image.decode_jpeg / PIL decode of every input pipeline), bit for bit equal to
 * libjpeg's ISLOW IDCT, fancy upsampling and YCbCr->RGB, i.e. to PIL's Image.open(b).convert("RGB").
 * Baseline and extended (SOF0 / SOF1) 8-bit Huffman JPEGs with one scan: grayscale, or 3-component
 * YCbCr with luma sampling 1x1, 2x1, 1x2 or 2x2 and chroma 1x1, any restart interval.  Everything
 * else is reported unsupported by acnn_jpeg_parse and is left to the caller (PIL).
 * ------------------------------------------------------------------------------------------- */
/* A Huffman table in decoding form: `look` maps the next 9 bits to (length << 8) | symbol (0: the
 * code is longer than 9 bits); for longer codes, maxcode[l] is the largest code of length l (-1: none)
 * and vals[valoff[l] + code] its symbol. */
typedef struct acnn_jpeg_huff {
  uint16_t look[512];
  int32_t maxcode[18];
  int32_t valoff[18];
  uint8_t vals[256];
} acnn_jpeg_huff;
typedef struct acnn_jpeg_comp {
  int32_t h, v;     /* sampling factors (1 x 1 for a grayscale image) */
  int32_t tq;       /* quantisation table */
  int32_t td, ta;   /* DC / AC Huffman tables */
  int32_t blk0;     /* index of the component's first block inside an MCU */
  int32_t dw, dh;   /* sample columns / rows: ceil(width * h / hmax), ceil(height * v / vmax) */
} acnn_jpeg_comp;
/* One parsed image (6368 bytes, the layout of jpeg.DESC_DTYPE), filled on the host by acnn_jpeg_parse and
 * read by the device as it is. */
typedef struct acnn_jpeg_desc {
  int32_t supported;         /* 1: acnn_jpeg_decode handles the image; 0: see reason */
  int32_t reason;            /* ACNN_JPEG_* code (acnn_jpeg_reason gives its text) */
  int32_t height, width;     /* from the frame header, whenever one was read (0 otherwise) */
  int32_t ncomp, hmax, vmax; /* 1 or 3 components; the largest sampling factors */
  int32_t bpm;               /* blocks per MCU */
  int32_t mcus_x, mcus_y;
  int32_t restart_interval;  /* MCUs per restart interval; 0: none */
  int32_t n_intervals;       /* restart markers in the scan + 1 */
  int64_t ecs_offset;        /* the entropy-coded segment: bytes [ecs_offset, ecs_offset + ecs_length) */
  int64_t ecs_length;        /*   of the image's buffer, restart markers included, stuffing not removed */
  acnn_jpeg_comp comp[3];
  int16_t quant[4][64];      /* natural order, as libjpeg's 16-bit multiplier table holds them */
  acnn_jpeg_huff dc[2], ac[2];
} acnn_jpeg_desc;
#define ACNN_JPEG_OK 0
#define ACNN_JPEG_NOT_JPEG 1        /* no SOI marker (PNG, ...) */
#define ACNN_JPEG_TRUNCATED 2       /* the buffer ends inside the header */
#define ACNN_JPEG_MALFORMED 3       /* a marker segment contradicts T.81 */
#define ACNN_JPEG_PROCESS 4         /* progressive, lossless, hierarchical or arithmetic coding */
#define ACNN_JPEG_PRECISION 5       /* not 8-bit samples */
#define ACNN_JPEG_COLOR 6           /* not 1 component or 3 YCbCr components (CMYK, Adobe RGB, ...) */
#define ACNN_JPEG_SAMPLING 7        /* sampling factors other than those above */
#define ACNN_JPEG_LAYOUT 8          /* several scans, a scan order other than the frame's, tables >= 2,
                                       DNL, fill bytes or misnumbered restart markers inside the scan, ... */
#define ACNN_JPEG_SIZE 9            /* more than 89478485 pixels or a scan of 2^27 bytes or more */
/* Text of an ACNN_JPEG_* code (host). */
const char* acnn_jpeg_reason(int code);
/* Parse the headers of n encoded images, image i at data + offsets[i], lengths[i] bytes (HOST memory):
 * SOI ... SOS (DQT, DHT, SOF, DRI, APP0 JFIF, APP14 Adobe), then a scan of the entropy-coded segment for
 * its restart markers and its end.  Every length and index is checked against the buffer; a malformed or
 * unsupported image gets supported = 0 and a reason, and never makes the call fail.  Null pointers or
 * n < 0: ACNN_ERR_INVALID. */
int acnn_jpeg_parse(const uint8_t* data, const int64_t* offsets, const int64_t* lengths, int n,
                    acnn_jpeg_desc* desc);
/* Decode plan of one image of a batch (host, filled by acnn_jpeg_plan). */
typedef struct acnn_jpeg_job {
  int64_t src;           /* offset of the image's encoded bytes in `data` */
  int64_t out;           /* offset of its uint8 [win_h][win_w][3] output in `out` (16-byte aligned) */
  int32_t win_y, win_x, win_h, win_w;
  int32_t active;        /* 0: unsupported, nothing runs for it and its status is ACNN_JPEG_ST_UNSUPPORTED */
  int32_t max_sub;       /* capacity of the subsequence tables */
  int32_t mcu_r0, mcu_r1, mcu_c0, mcu_c1;   /* MCU rows / columns the window and its upsampling context need */
  int32_t stored_blocks; /* coefficient blocks kept: MCU rows 0 .. mcu_r1 */
  int32_t idct_blocks;   /* blocks of MCU rows mcu_r0 .. mcu_r1, columns mcu_c0 .. mcu_c1 */
  int64_t o_bits, o_intervals, o_subs, o_state, o_dirty, o_prefix, o_coef, o_plane[3];  /* into `work` */
} acnn_jpeg_job;
typedef struct acnn_jpeg_batch {
  int64_t work_bytes;    /* size of `work` */
  int64_t out_bytes;     /* size of `out` */
  int64_t coef_begin, coef_end;   /* the coefficient span of `work` (zeroed by acnn_jpeg_decode) */
  int32_t n, max_sub, max_idct_blocks, max_pixels;
} acnn_jpeg_batch;
/* Plan the decode of n parsed images (host): image i's encoded bytes at offsets[i] of the device buffer
 * `data`, its crop window windows[i] = (y, x, h, w) (int32 [n][4], HOST; NULL: whole images).  Windows
 * outside the image or empty: ACNN_ERR_INVALID.  Fills jobs[n] and *batch. */
int acnn_jpeg_plan(const acnn_jpeg_desc* desc, const int64_t* offsets, const int32_t* windows, int n,
                   acnn_jpeg_job* jobs, acnn_jpeg_batch* batch);
/* Decode the batch planned by acnn_jpeg_plan into `out` (DEVICE, batch->out_bytes): the window of every
 * active image as packed uint8 RGB, the same bytes as PIL's Image.open(b).convert("RGB") sliced to it.
 * desc and jobs: DEVICE copies of the host arrays; batch: HOST.  work: DEVICE, batch->work_bytes bytes.
 * status: DEVICE int32 [n], written with ACNN_JPEG_ST_* bits: an image with a non-zero status has
 * undefined pixels in its window (and nothing outside it is written).  The entropy decode is the
 * self-synchronising parallel Huffman decode of Weissenberger & Schmidt (one thread per 1024-bit
 * subsequence of the unstuffed scan); restart markers are exact synchronisation points.  The kernels
 * read no byte outside an image's entropy-coded segment. */
#define ACNN_JPEG_ST_UNSUPPORTED 1
#define ACNN_JPEG_ST_BAD_CODE 2       /* a bit pattern that is no code of its Huffman table */
#define ACNN_JPEG_ST_OUT_OF_BITS 4    /* a restart interval or the scan ends inside an MCU */
#define ACNN_JPEG_ST_MCU_COUNT 8      /* a restart interval or the scan holds the wrong number of MCUs */
int acnn_jpeg_decode(const acnn_jpeg_desc* desc, const acnn_jpeg_job* jobs, const acnn_jpeg_batch* batch,
                     const uint8_t* data, uint8_t* out, void* work, int64_t work_bytes, int32_t* status,
                     void* stream);

/* ---------------------------------------------------------------------------------------------
 * TFRecord checksums (the writer of knowledge-distillation shards, model_fns.extract_teacher_logits)
 * ------------------------------------------------------------------------------------------- */
/* CRC-32C (Castagnoli, reflected polynomial 0x82F63B78) of n bytes of HOST memory at data, continued
 * from crc, a CRC this function returned (0 starts a new one): acnn_crc32c(b, nb, acnn_crc32c(a, na, 0))
 * is the CRC of a followed by b.  data may be NULL when n = 0.  On x86-64 it runs SSE4.2's crc32
 * instruction.  No CUDA call; never fails. */
uint32_t acnn_crc32c(const void* data, size_t n, uint32_t crc);

#ifdef __cplusplus
}
#endif
#endif /* ACNN_H_ */
