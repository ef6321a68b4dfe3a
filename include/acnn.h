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
 * run on operands split into three bf16 planes (`precision` = 1 below). */
#define ACNN_BF16 0
#define ACNN_F32 1

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
 * order): the fixed cost of one CTA (pipeline fill + atomic epilogue) in pipeline stages used by the
 * cost model that picks the number of pixel splits (default 16); 0 = the "two waves of CTAs"
 * rule.  Returns the previous setting. */
int acnn_set_wgrad_overhead_stages(int stages);
/* Tuning knob of the wgrad launcher: n > 0 asks for n pixel splits, clamped to the capacity of the
 * partial-tile scratch (64 MiB, one arrival counter per tile) and to the number of pipeline stages;
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
 *                                     adds the rows in a fixed order (bit-reproducible)
 * out_f32 != 0 stores y as fp32 (logits), else bf16.  Requires Cin % 16 == 0, Cout % 32 == 0.
 * precision 0: x, w bf16.  precision 1 (fp32 parity mode): x and w are each three consecutive bf16
 * planes hi / mid / lo of an fp32 tensor (acnn_split3, acnn_prep_weights(planes = 3)); plane p of x
 * starts at x + p * numel(x), plane p of w at w + p * w_plane_stride elements; the six significant
 * cross products accumulate in fp32 register accumulators; requires out_f32 and no add / mask /
 * statistics epilogue. */
int acnn_conv_fprop(const acnn_conv_geom* g, const void* x, const void* w, void* y,
                    float* ch_part, const void* add_src, const void* mask_src,
                    const float* bias, int out_f32, int precision, int64_t w_plane_stride,
                    void* stream);
/* Rows of the partial statistics buffer acnn_conv_fprop(g, ..., ch_part, ...) writes (a pure
 * function of the geometry and the device's SM count; <= 132). */
int acnn_conv_stats_parts(const acnn_conv_geom* g);

/* dx[B,H,W,Cin] = conv_transpose(dy[B,Ho,Wo,Cout]) for a stride-1 conv of geometry g (the backward
 * of tf.layers.conv2d the reference gets from tf.gradients, nets/optimizer_setting.py:30).
 * w_dgrad is [Cin][kh][kw][Cout] with taps already flipped (acnn_prep_weights writes it).
 * Same optional add_src / mask_src epilogue as acnn_conv_fprop (shapes of dx).  precision 1: dy and
 * w_dgrad are 3-plane operands, dx is fp32 and no epilogue may be fused. */
int acnn_conv_dgrad(const acnn_conv_geom* g, const void* dy, const void* w_dgrad, void* dx,
                    const void* add_src, const void* mask_src, int precision,
                    int64_t w_plane_stride, void* stream);

/* dw[Cout,kh,kw,Cin] (fp32) += sum_pixels x (*) dy  -- weight gradient, split-K over pixels: the
 * splits store partial tiles in a stream-ordered scratch of the launch (cudaMallocAsync on `stream`)
 * and the last split of a tile adds them to dw in split order (bit-reproducible).  dw must be zeroed
 * (or hold the running sum) by the caller.  deterministic != 0: no split (one add per element).
 * precision 1: x and dy are 3-plane operands. */
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
 * conv GEMMs), whose six significant cross products are accumulated in fp32.
 * out_idx int32 [nq][k], out_sim fp32 [nq][k].  Any d >= 1 (<= 2^24); 1 <= k <= 128 (k > 128:
 * ACNN_ERR_UNSUPPORTED); k > nx, non-positive sizes, an unknown metric or dtype: ACNN_ERR_INVALID.
 * All of these are checked before any CUDA call.  The result is the same bit for bit for every
 * column-split count, grid and stream.  Only similarities above -inf are ranked: a row with fewer
 * than k of them (a NaN or infinite input, or a squared distance that overflows fp32) is padded with
 * (similarity -inf, index 2147483647) entries -- callers that index with out_idx must check for it.
 * work: acnn_knn_work_bytes(...) bytes, caller-owned; every section starts at a 256-byte boundary:
 *   Q' bf16 [nq][K'], X' bf16 [nx][K']  (K' = P * roundup(d, 64), zero-padded; P = 1 for bf16, 6 for
 *        fp32: K' holds six d-segments so that one bf16 GEMM forms the six plane products, smallest
 *        first -- Q' = (hi, mid, lo, hi, mid, hi), X' = (lo, mid, hi, mid, hi, hi))
 *   |q|^2 fp32 [nq], |x|^2 fp32 [nx]   (of the rounded operands: bf16, or (hi + mid) + lo)
 *   partial lists: similarity fp32 [8][nq][k], index int32 [8][nq][k]  (one per column split) */
int acnn_knn_topk(const float* q, const float* x, int nq, int nx, int d, int k, int metric, int dtype,
                  int32_t* out_idx, float* out_sim, void* work, int64_t work_bytes, void* stream);
/* Bytes of the `work` argument (host only, callable without a GPU); -1 for invalid sizes. */
int64_t acnn_knn_work_bytes(int nq, int nx, int d, int k, int dtype);
/* Tuning knob of acnn_knn_topk (no effect on results): n > 0 forces n column splits, clamped to
 * [1, min(8, ceil(nx / 128))]; 0 (default) = the cost model that fills the SMs.  Returns the previous
 * setting. */
int acnn_set_knn_splits(int n);

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

#ifdef __cplusplus
}
#endif
#endif /* ACNN_H_ */
