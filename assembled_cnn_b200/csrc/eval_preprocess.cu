// ImageNet classification evaluation (classifier.evaluate(input_fn_eval), nets/run_loop_classification.py):
// the eval preprocessing of decoded images and the per-row metrics of the logits.
//
//  * resize_crop_u8_kernel: aspect-preserving resize (TF 1.14's legacy bilinear, half_pixel_centers =
//    false), central crop and mean subtraction of preprocessing/imagenet_preprocessing.py:158-226,295-313
//    in one pass over a batch of images of different sizes.  Only the S x S pixels the crop keeps are
//    computed: a resized pixel depends on its own coordinates only.
//  * classify_rows_kernel: tf.argmax(logits), the largest softmax probability, tf.nn.in_top_k and the
//    label-smoothed softmax cross-entropy of every row (nets/run_loop_classification.py:141-234), one warp
//    per row, no atomics.
#include <math.h>

#include "common.h"
#include "legacy_bilinear.cuh"
#include "vec.cuh"

namespace acnn {

// grid (ceil(S*S / 256), n_valid): one thread per output pixel of one image.
__global__ void __launch_bounds__(256)
resize_crop_u8_kernel(const acnn_resize_desc* __restrict__ desc, int S, const float* __restrict__ mean_dev,
                      float m0, float m1, float m2, float* __restrict__ out) {
  pdl_entry();
  if (mean_dev) {
    m0 = mean_dev[0];
    m1 = mean_dev[1];
    m2 = mean_dev[2];
  }
  const int b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= S * S) return;
  const acnn_resize_desc d = desc[b];
  const int y = p / S, x = p - (p / S) * S;
  // scale = (float)in_size / out_size (CalculateResizeScale, align_corners = false)
  const Interp iy = legacy_interp(y + d.crop_y, __fdiv_rn((float)d.src_h, (float)d.rsz_h), d.src_h);
  const Interp ix = legacy_interp(x + d.crop_x, __fdiv_rn((float)d.src_w, (float)d.rsz_w), d.src_w);
  const uint8_t* top = d.src + (int64_t)iy.lo * d.src_w * 3;
  const uint8_t* bot = d.src + (int64_t)iy.hi * d.src_w * 3;
  const int xl = ix.lo * 3, xh = ix.hi * 3;
  const float mean[3] = {m0, m1, m2};
  float* o = out + ((int64_t)b * S * S + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t = lerp_rn((float)top[xl + c], (float)top[xh + c], ix.lerp);
    const float u = lerp_rn((float)bot[xl + c], (float)bot[xh + c], ix.lerp);
    o[c] = __fsub_rn(lerp_rn(t, u, iy.lerp), mean[c]);
  }
}

// One warp per row of logits [B][ld] (columns < NC are the classes).  Per-lane strided partial results,
// then an xor butterfly: every reduction has the same order on every launch, and a + b == b + a keeps
// all lanes equal.
constexpr int kClassifyRows = 8;   // rows (warps) per CTA

__global__ void __launch_bounds__(32 * kClassifyRows)
classify_rows_kernel(const float* __restrict__ logits, int ld, int NC, const int32_t* __restrict__ labels,
                     int n_valid, int k, float ls, int32_t* __restrict__ pred, float* __restrict__ conf,
                     int32_t* __restrict__ hit_k, float* __restrict__ ce) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kClassifyRows + (threadIdx.x >> 5);
  if (row >= n_valid) return;    // padding rows: not written
  const float* x = logits + (size_t)row * ld;
  // tf.argmax: the smallest index of the largest logit
  float mx = -INFINITY;
  int mj = NC;
  bool finite = true;
  for (int j = lane; j < NC; j += 32) {
    const float v = x[j];
    finite = finite && isfinite(v);
    if (v > mx) {                // ascending j: the first of equal logits stays
      mx = v;
      mj = j;
    }
  }
  if (!__all_sync(0xffffffffu, finite)) {
    if (lane == 0) {
      pred[row] = -1;
      conf[row] = NAN;
      hit_k[row] = 0;
      ce[row] = NAN;
    }
    return;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oj = __shfl_xor_sync(0xffffffffu, mj, o);
    if (om > mx || (om == mx && oj < mj)) {
      mx = om;
      mj = oj;
    }
  }
  const int label = labels[row];
  const bool in_range = label >= 0 && label < NC;
  const float xt = in_range ? x[label] : 0.f;
  float s = 0.f, sd = 0.f;
  int greater = 0;
  for (int j = lane; j < NC; j += 32) {
    const float v = x[j];
    const float dv = v - mx;
    s += expf(dv);
    sd += dv;
    greater += v > xt;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    sd += __shfl_xor_sync(0xffffffffu, sd, o);
    greater += __shfl_xor_sync(0xffffffffu, greater, o);
  }
  if (lane == 0) {
    pred[row] = mj;
    conf[row] = 1.f / s;          // expf(mx - mx) / s
    // tf.nn.in_top_k: fewer than k logits strictly above the target's
    hit_k[row] = in_range && greater < k;
    // -sum_j t_j log p_j with t = onehot * (1 - ls) + ls / NC, log p_j = (x_j - mx) - log(s)
    const float lse = logf(s);
    const float logp_t = (xt - mx) - lse;
    const float sum_logp = sd - (float)NC * lse;
    ce[row] = in_range ? -((1.f - ls) * logp_t + (ls / (float)NC) * sum_logp) : NAN;
  }
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_resize_crop_u8(const acnn_resize_desc* desc, int B, int n_valid, int S, const float* mean, float* out,
                        void* stream) {
  ACNN_REQUIRE(desc && mean && out, "acnn_resize_crop_u8: null pointer");
  ACNN_REQUIRE(B > 0 && S > 0, "acnn_resize_crop_u8: bad shape B=%d S=%d", B, S);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "acnn_resize_crop_u8: n_valid=%d outside [0, B=%d]", n_valid, B);
  ACNN_REQUIRE(((uintptr_t)out & 3) == 0, "acnn_resize_crop_u8: out must be 4-byte aligned");
  ACNN_REQUIRE(((uintptr_t)desc & 7) == 0, "acnn_resize_crop_u8: desc must be 8-byte aligned");
  ACNN_REQUIRE((int64_t)S * S <= INT32_MAX, "acnn_resize_crop_u8: S=%d too large", S);
  cudaPointerAttributes at{};
  cudaError_t e = cudaPointerGetAttributes(&at, mean);
  if (e != cudaSuccess) {
    set_error("acnn_resize_crop_u8: mean: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  const bool mean_on_device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
  const float m0 = mean_on_device ? 0.f : mean[0], m1 = mean_on_device ? 0.f : mean[1],
              m2 = mean_on_device ? 0.f : mean[2];
  if (n_valid == 0) return ACNN_OK;
  launch_k(resize_crop_u8_kernel, dim3(ceil_div(S * S, 256), n_valid), dim3(256), 0, (cudaStream_t)stream, desc,
           S, mean_on_device ? mean : (const float*)nullptr, m0, m1, m2, out);
  count_launch();
  return check_launch("resize_crop_u8");
}

int acnn_classify_rows(const float* logits, int B, int ld, int NC, const int32_t* labels, int n_valid, int k,
                       float label_smoothing, int32_t* pred, float* conf, int32_t* hit_k, float* ce,
                       void* stream) {
  ACNN_REQUIRE(logits && labels && pred && conf && hit_k && ce, "acnn_classify_rows: null pointer");
  ACNN_REQUIRE(B > 0 && NC > 0 && ld >= NC, "acnn_classify_rows: bad shape B=%d ld=%d NC=%d", B, ld, NC);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "acnn_classify_rows: n_valid=%d outside [0, B=%d]", n_valid, B);
  ACNN_REQUIRE(k >= 1, "acnn_classify_rows: k=%d < 1", k);
  ACNN_REQUIRE(isfinite(label_smoothing), "acnn_classify_rows: label_smoothing is not finite");
  if (n_valid == 0) return ACNN_OK;
  launch_k(classify_rows_kernel, dim3(ceil_div(n_valid, kClassifyRows)), dim3(32 * kClassifyRows), 0,
           (cudaStream_t)stream, logits, ld, NC, labels, n_valid, k, label_smoothing, pred, conf, hit_k, ce);
  count_launch();
  return check_launch("classify_rows");
}

}  // extern "C"
