// The PREDICT-mode `predictions` dict of resnet_model_fn (nets/run_loop_classification.py:126-130) on the
// device, for the exported servables (model_fns.Servable):
//
//  * predict_rows_kernel: classes = tf.argmax(logits, 1), probabilities = tf.nn.softmax(logits) and
//    probabilities_sigmoid = tf.nn.sigmoid(logits) of every row.  One CTA of kPredictThreads per row: a
//    1001-column row is 8 columns per thread, and a batch of 256 rows is 256 CTAs, about two per SM, where a
//    warp per row would leave most SMs idle.  Per-thread strided partial results in ascending column order,
//    an xor butterfly in each warp, then warp 0 combines the warps' results in warp order: every reduction has
//    the same order on every launch, and there are no atomics.
#include <math.h>

#include "common.h"
#include "vec.cuh"

namespace acnn {

constexpr int kPredictThreads = 128;
constexpr int kPredictWarps = kPredictThreads / 32;

// (mx, mj) <- the larger of (mx, mj) and (om, oj); equal values keep the lower index (mj == NC: no column yet)
__device__ __forceinline__ void first_max(float& mx, int& mj, float om, int oj) {
  if (om > mx || (om == mx && oj < mj)) {
    mx = om;
    mj = oj;
  }
}

__global__ void __launch_bounds__(kPredictThreads)
predict_rows_kernel(const float* __restrict__ logits, int ld, int NC, int32_t* __restrict__ classes,
                    float* __restrict__ prob, float* __restrict__ prob_sigmoid) {
  pdl_entry();
  __shared__ float s_max[kPredictWarps];
  __shared__ int s_arg[kPredictWarps];
  __shared__ float s_sum[kPredictWarps];
  __shared__ float s_row[2];         // the row's max, its sum
  __shared__ int s_nan;
  const int row = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* x = logits + (size_t)row * ld;
  float* p = prob + (size_t)row * NC;
  float* sg = prob_sigmoid + (size_t)row * NC;

  // tf.argmax: the smallest index of the largest logit (+-inf are ordinary values; a NaN row gets -1)
  float mx = -INFINITY;
  int mj = NC;
  bool nan = false;
  for (int j = tid; j < NC; j += kPredictThreads) {
    const float v = x[j];
    nan = nan || isnan(v);
    if (mj == NC || v > mx) {        // ascending j: the first of equal logits stays
      mx = v;
      mj = j;
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) first_max(mx, mj, __shfl_xor_sync(0xffffffffu, mx, o), __shfl_xor_sync(0xffffffffu, mj, o));
  const bool warp_nan = __any_sync(0xffffffffu, nan);
  if (lane == 0) {
    s_max[warp] = mx;
    s_arg[warp] = mj;
  }
  if (tid == 0) s_nan = 0;
  __syncthreads();
  if (lane == 0 && warp_nan) s_nan = 1;   // every writer stores the same value
  if (tid == 0) {
    float m = s_max[0];
    int a = s_arg[0];
    for (int w = 1; w < kPredictWarps; ++w) first_max(m, a, s_max[w], s_arg[w]);
    s_row[0] = m;
    s_arg[0] = a;
  }
  __syncthreads();
  const float rmax = s_row[0];
  if (tid == 0) classes[row] = s_nan ? -1 : s_arg[0];

  // softmax: expf(x_j - max) / sum, the sum in a fixed order
  float s = 0.f;
  for (int j = tid; j < NC; j += kPredictThreads) s += expf(x[j] - rmax);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) s_sum[warp] = s;
  __syncthreads();
  if (tid == 0) {
    float t = s_sum[0];
    for (int w = 1; w < kPredictWarps; ++w) t += s_sum[w];
    s_row[1] = t;
  }
  __syncthreads();
  const float rsum = s_row[1];
  for (int j = tid; j < NC; j += kPredictThreads) {
    const float v = x[j];
    p[j] = expf(v - rmax) / rsum;
    sg[j] = 1.f / (1.f + expf(-v));
  }
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_predict_rows(const float* logits, int B, int ld, int NC, int n_valid, int32_t* classes, float* probabilities,
                      float* probabilities_sigmoid, void* stream) {
  ACNN_REQUIRE(logits && classes && probabilities && probabilities_sigmoid, "acnn_predict_rows: null pointer");
  ACNN_REQUIRE(B > 0 && NC > 0 && ld >= NC, "acnn_predict_rows: bad shape B=%d ld=%d NC=%d", B, ld, NC);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "acnn_predict_rows: n_valid=%d outside [0, B=%d]", n_valid, B);
  if (n_valid == 0) return ACNN_OK;
  launch_k(predict_rows_kernel, dim3(n_valid), dim3(kPredictThreads), 0, (cudaStream_t)stream, logits, ld, NC,
           classes, probabilities, probabilities_sigmoid);
  count_launch();
  return check_launch("predict_rows");
}

}  // extern "C"
