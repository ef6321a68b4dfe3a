// The input preprocessing of decoded uint8 images, for the evaluation and for training, and the per-row
// metrics of the classification evaluation (classifier.evaluate(input_fn_eval),
// nets/run_loop_classification.py).
//
//  * resample_u8: one pass over a batch of images of different sizes, resized with TF 1.14's legacy bilinear
//    (half_pixel_centers = false), cropped to S x S, minus the channel means; one thread per output pixel.
//    Only the S x S pixels the crop keeps are computed: a resized pixel depends on its own coordinates only.
//    - resize_crop_u8_kernel: the eval preprocessing (aspect-preserving resize, central crop) of
//      preprocessing/imagenet_preprocessing.py:158-226,295-313.
//    - crop_resize_u8_kernel: the training preprocessing of a crop window (imagenet_preprocessing.py:57-97,
//      269-313, is_training=True): random_flip_left_right, _resize_image to S x S with the independent
//      scales (float)h / S and (float)w / S, mean_image_subtraction.  The crop itself
//      (sample_distorted_bounding_box + decode_and_crop_jpeg) happens on the host: each descriptor points at
//      the window's packed pixels.
//  * classify_rows_kernel: tf.argmax(logits), the largest softmax probability, tf.nn.in_top_k and the
//    label-smoothed softmax cross-entropy of every row (nets/run_loop_classification.py:141-234), one warp
//    per row, no atomics.
#include <math.h>

#include "common.h"
#include "legacy_bilinear.cuh"
#include "vec.cuh"

namespace acnn {

// What the resampling reads of a descriptor: the source image, the resized size and the offset of the S x S
// crop in it, and the flip.  A training window is resized to S x S and not cropped; an eval image is never
// flipped.
struct ResampleView {
  const uint8_t* src;
  int h, w, rsz_h, rsz_w, crop_y, crop_x;
  bool flip;
};

__device__ __forceinline__ ResampleView view(const acnn_resize_desc& d, int) {
  return {d.src, d.src_h, d.src_w, d.rsz_h, d.rsz_w, d.crop_y, d.crop_x, false};
}

__device__ __forceinline__ ResampleView view(const acnn_crop_desc& d, int S) {
  return {d.src, d.h, d.w, S, S, 0, 0, d.flip != 0};
}

// grid (ceil(S*S / 256), n_valid): one thread per output pixel of one image.
template <class Desc>
__device__ __forceinline__ void resample_u8(const Desc* __restrict__ desc, int S, const float* __restrict__ mean_dev,
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
  const Desc dd = desc[b];
  const ResampleView d = view(dd, S);
  const int y = p / S, x = p - (p / S) * S;
  // scale = (float)in_size / out_size (CalculateResizeScale, align_corners = false)
  float v[3];
  legacy_bilinear_rgb(d.src, d.h, d.w, __fdiv_rn((float)d.h, (float)d.rsz_h), __fdiv_rn((float)d.w, (float)d.rsz_w),
                      y + d.crop_y, x + d.crop_x, d.flip, v);
  const float mean[3] = {m0, m1, m2};
  float* o = out + ((int64_t)b * S * S + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = __fsub_rn(v[c], mean[c]);
}

__global__ void __launch_bounds__(256)
resize_crop_u8_kernel(const acnn_resize_desc* __restrict__ desc, int S, const float* __restrict__ mean_dev,
                      float m0, float m1, float m2, float* __restrict__ out) {
  resample_u8(desc, S, mean_dev, m0, m1, m2, out);
}

__global__ void __launch_bounds__(256)
crop_resize_u8_kernel(const acnn_crop_desc* __restrict__ desc, int S, const float* __restrict__ mean_dev,
                      float m0, float m1, float m2, float* __restrict__ out) {
  resample_u8(desc, S, mean_dev, m0, m1, m2, out);
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

// The argument checks and the launch of the entry point `fn` ("acnn_" + the launch's name).
template <class Desc>
static int launch_resample(void (*kernel)(const Desc*, int, const float*, float, float, float, float*), const char* fn,
                           const Desc* desc, int B, int n_valid, int S, const float* mean, float* out, void* stream) {
  ACNN_REQUIRE(desc && mean && out, "%s: null pointer", fn);
  ACNN_REQUIRE(B > 0 && S > 0, "%s: bad shape B=%d S=%d", fn, B, S);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "%s: n_valid=%d outside [0, B=%d]", fn, n_valid, B);
  ACNN_REQUIRE(((uintptr_t)out & 3) == 0, "%s: out must be 4-byte aligned", fn);
  ACNN_REQUIRE(((uintptr_t)desc & 7) == 0, "%s: desc must be 8-byte aligned", fn);
  ACNN_REQUIRE((int64_t)S * S <= INT32_MAX, "%s: S=%d too large", fn, S);
  const float* mean_dev;
  float m[3];
  const int rc = resolve_mean(fn, mean, &mean_dev, m);
  if (rc != ACNN_OK) return rc;
  if (n_valid == 0) return ACNN_OK;
  launch_k(kernel, dim3(ceil_div(S * S, 256), n_valid), dim3(256), 0, (cudaStream_t)stream, desc, S, mean_dev, m[0],
           m[1], m[2], out);
  count_launch();
  return check_launch(fn + 5);
}

extern "C" {

int acnn_resize_crop_u8(const acnn_resize_desc* desc, int B, int n_valid, int S, const float* mean, float* out,
                        void* stream) {
  return launch_resample(resize_crop_u8_kernel, "acnn_resize_crop_u8", desc, B, n_valid, S, mean, out, stream);
}

int acnn_crop_resize_u8(const acnn_crop_desc* desc, int B, int n_valid, int S, const float* mean, float* out,
                        void* stream) {
  return launch_resample(crop_resize_u8_kernel, "acnn_crop_resize_u8", desc, B, n_valid, S, mean, out, stream);
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
