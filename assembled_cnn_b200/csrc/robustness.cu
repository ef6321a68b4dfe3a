// Robustness evaluation (ImageNet-C corruption error, mce/eval_robustness.py): the uint8 input path and
// the on-device top-1 counter.
//
//  * images_from_u8_kernel: decoded uint8 NHWC pixels -> fp32 `(float)x - mean[c]`, the cast and
//    mean_image_subtraction of input_fn_imagenet_c (mce/eval_robustness.py:123-148,
//    preprocessing/imagenet_preprocessing.py:122-149): one pass, 16 bytes per load, four float4 stores.
//  * softmax_top1_count_kernel: tf.nn.top_k(tf.nn.softmax(logits), 1) and the per-image
//    `pred == gt` count of show_corruption_error_by_distortion (mce/eval_robustness.py:186-187,
//    214-229), one warp per row, the correct count accumulated with integer atomics.
#include <math.h>

#include "common.h"
#include "vec.cuh"

namespace acnn {

__device__ __forceinline__ float select3(int r, float a, float b, float c) {
  return r == 0 ? a : (r == 1 ? b : c);
}

// n = B*H*W*3 bytes; the first n16 = n / 16 sixteen-byte groups are vectorised, the rest (< 16) is
// written by the first threads of block 0.  Element e is channel e % 3.
__global__ void __launch_bounds__(256)
images_from_u8_kernel(const uint8_t* __restrict__ in, const float* __restrict__ mean_dev, float m0, float m1,
                      float m2, float* __restrict__ out, int64_t n16, int64_t n) {
  pdl_entry();
  if (mean_dev) {
    m0 = mean_dev[0];
    m1 = mean_dev[1];
    m2 = mean_dev[2];
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(in) + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const int r = (int)(i % 3);   // channel of the group's first byte: 16 i mod 3 = i mod 3
    const float mr[3] = {select3(r, m0, m1, m2), select3(r, m1, m2, m0), select3(r, m2, m0, m1)};
    float f[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) f[k] = (float)((w[k >> 2] >> (8 * (k & 3))) & 0xffu) - mr[k % 3];
    float4* o = reinterpret_cast<float4*>(out) + 4 * i;
#pragma unroll
    for (int q = 0; q < 4; ++q) o[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
  }
  const int64_t e = 16 * n16 + threadIdx.x;
  if (blockIdx.x == 0 && e < n) {
    const int c = (int)(e % 3);
    out[e] = (float)in[e] - select3(c, m0, m1, m2);
  }
}

// One warp per row of logits [B][ld]: max, sum_j expf(x_j - max) (per-lane strided partial sums, then a
// butterfly: the same order on every launch), p_j = expf(x_j - max) / sum, pred = the smallest j with
// the largest p_j (tf.nn.top_k's rule on the fp32 probabilities).  A non-finite logit: pred = -1.
constexpr int kTop1Rows = 8;   // rows (warps) per CTA

__global__ void __launch_bounds__(32 * kTop1Rows)
softmax_top1_count_kernel(const float* __restrict__ logits, int ld, int NC, const int32_t* __restrict__ labels,
                          int n_valid, int32_t* __restrict__ pred, unsigned long long* __restrict__ correct) {
  pdl_entry();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kTop1Rows + (threadIdx.x >> 5);
  if (row >= n_valid) return;    // padding rows: neither written nor counted
  const float* x = logits + (size_t)row * ld;
  float mx = -INFINITY;
  bool finite = true;
  for (int j = lane; j < NC; j += 32) {
    const float v = x[j];
    finite = finite && isfinite(v);
    mx = fmaxf(mx, v);
  }
  if (!__all_sync(0xffffffffu, finite)) {
    if (lane == 0) pred[row] = -1;
    return;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float s = 0.f;
  for (int j = lane; j < NC; j += 32) s += expf(x[j] - mx);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);   // a + b == b + a: every lane agrees
  float bp = -1.f;
  int bj = NC;
  for (int j = lane; j < NC; j += 32) {
    const float p = expf(x[j] - mx) / s;
    if (p > bp) {                // ascending j: the first of equal probabilities stays
      bp = p;
      bj = j;
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float op = __shfl_xor_sync(0xffffffffu, bp, o);
    const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
    if (op > bp || (op == bp && oj < bj)) {
      bp = op;
      bj = oj;
    }
  }
  if (lane == 0) {
    pred[row] = bj;
    if (labels[row] == bj) atomicAdd(correct, 1ull);
  }
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_images_from_u8(const uint8_t* images, const float* mean, float* out, int B, int H, int W,
                        void* stream) {
  ACNN_REQUIRE(images && mean && out, "acnn_images_from_u8: null pointer");
  ACNN_REQUIRE(B > 0 && H > 0 && W > 0, "acnn_images_from_u8: bad shape [%d,%d,%d,3]", B, H, W);
  ACNN_REQUIRE(((uintptr_t)images & 15) == 0 && ((uintptr_t)out & 15) == 0,
               "acnn_images_from_u8: images and out must be 16-byte aligned");
  cudaPointerAttributes at{};
  cudaError_t e = cudaPointerGetAttributes(&at, mean);
  if (e != cudaSuccess) {
    set_error("acnn_images_from_u8: mean: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  const bool mean_on_device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
  const float m0 = mean_on_device ? 0.f : mean[0], m1 = mean_on_device ? 0.f : mean[1],
              m2 = mean_on_device ? 0.f : mean[2];
  const int64_t n = (int64_t)B * H * W * 3, n16 = n / 16;
  launch_k(images_from_u8_kernel, dim3(grid_for(n16 > 0 ? n16 : 1)), dim3(256), 0, (cudaStream_t)stream, images,
           mean_on_device ? mean : (const float*)nullptr, m0, m1, m2, out, n16, n);
  count_launch();
  return check_launch("images_from_u8");
}

int acnn_softmax_top1_count(const float* logits, int B, int ld, int NC, const int32_t* labels, int n_valid,
                            int32_t* pred, uint64_t* correct, void* stream) {
  ACNN_REQUIRE(logits && labels && pred && correct, "acnn_softmax_top1_count: null pointer");
  ACNN_REQUIRE(B > 0 && NC > 0 && ld >= NC, "acnn_softmax_top1_count: bad shape B=%d ld=%d NC=%d", B, ld, NC);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "acnn_softmax_top1_count: n_valid=%d outside [0, B=%d]", n_valid, B);
  if (n_valid == 0) return ACNN_OK;
  launch_k(softmax_top1_count_kernel, dim3(ceil_div(n_valid, kTop1Rows)), dim3(32 * kTop1Rows), 0,
           (cudaStream_t)stream, logits, ld, NC, labels, n_valid, pred, (unsigned long long*)correct);
  count_launch();
  return check_launch("softmax_top1_count");
}

}  // extern "C"
