// The training-batch metrics of resnet_model_fn's TRAIN branch (nets/run_loop_classification.py:146-227) on the
// device, accumulated over the micro-steps of a run without a host read (acnn_train_metrics_accumulate,
// include/acnn.h).  The per-row argmax / softmax / in_top_k come from acnn_classify_rows; this kernel only bins
// and sums them.
//
// One CTA of kTrainMetricsThreads.  Row r belongs to thread r % 256, which walks its rows in ascending order:
// integer counts go through warp reductions (any order gives the same integers), fp64 sums through a fixed
// shared-memory tree, so every launch adds in the order acnn.h states.
#include <math.h>

#include "common.h"
#include "vec.cuh"

namespace acnn {

constexpr int kTrainMetricsThreads = 256;
constexpr int kSums = ACNN_ECE_BINS + 1;    // the bins' confidence sums, then the step's

// The float32 bin thresholds of metrics.classification_result: [-1e-7, 0.1, ..., 0.9, 1 + 1e-7], each the
// double value rounded to float.
__constant__ float kEceThresholds[ACNN_ECE_BINS + 1] = {
    (float)(0.0 - 1e-7), (float)(1 / 10.0), (float)(2 / 10.0), (float)(3 / 10.0), (float)(4 / 10.0),
    (float)(5 / 10.0), (float)(6 / 10.0), (float)(7 / 10.0), (float)(8 / 10.0), (float)(9 / 10.0),
    (float)(1.0 + 1e-7)};

__device__ __forceinline__ int64_t block_count(int v, int64_t* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();                 // s_warp is reused by the previous count
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  int64_t t = 0;
  for (int w = 0; w < kTrainMetricsThreads / 32; ++w) t += s_warp[w];
  return t;
}

__global__ void __launch_bounds__(kTrainMetricsThreads)
train_metrics_kernel(const int32_t* __restrict__ pred, const float* __restrict__ conf,
                     const int32_t* __restrict__ hit_k, const int32_t* __restrict__ labels, int n, int step_begin,
                     acnn_train_metrics* __restrict__ m) {
  pdl_entry();
  __shared__ double s_sum[kSums][kTrainMetricsThreads];
  __shared__ int64_t s_warp[kTrainMetricsThreads / 32];
  const int tid = threadIdx.x;
  int top1 = 0, top5 = 0;
  int cnt[ACNN_ECE_BINS], cor[ACNN_ECE_BINS];
  double csum[ACNN_ECE_BINS];
  double step = 0.0;
#pragma unroll
  for (int b = 0; b < ACNN_ECE_BINS; ++b) {
    cnt[b] = cor[b] = 0;
    csum[b] = 0.0;
  }
  for (int r = tid; r < n; r += kTrainMetricsThreads) {
    const float c = conf[r];
    const int p = pred[r];
    const bool ok = p >= 0 && p == labels[r];
    top1 += ok;
    top5 += hit_k[r] != 0;
    step = __dadd_rn(step, (double)c);
#pragma unroll
    for (int b = 0; b < ACNN_ECE_BINS; ++b) {
      if (c > kEceThresholds[b] && c <= kEceThresholds[b + 1]) {   // false for NaN
        cnt[b] += 1;
        cor[b] += ok;
        csum[b] = __dadd_rn(csum[b], (double)c);
      }
    }
  }
#pragma unroll
  for (int b = 0; b < ACNN_ECE_BINS; ++b) s_sum[b][tid] = csum[b];
  s_sum[ACNN_ECE_BINS][tid] = step;
  for (int s = kTrainMetricsThreads / 2; s > 0; s >>= 1) {
    __syncthreads();
    if (tid < s) {
#pragma unroll
      for (int k = 0; k < kSums; ++k) s_sum[k][tid] = __dadd_rn(s_sum[k][tid], s_sum[k][tid + s]);
    }
  }
  // the counts (block_count's barriers also order the tree's last step before the reads below)
  const int64_t t1 = block_count(top1, s_warp);
  const int64_t t5 = block_count(top5, s_warp);
  int64_t bc[ACNN_ECE_BINS], bk[ACNN_ECE_BINS];
#pragma unroll
  for (int b = 0; b < ACNN_ECE_BINS; ++b) {
    bc[b] = block_count(cnt[b], s_warp);
    bk[b] = block_count(cor[b], s_warp);
  }
  if (tid == 0) {
    m->rows += n;
    m->top1 += t1;
    m->top5 += t5;
#pragma unroll
    for (int b = 0; b < ACNN_ECE_BINS; ++b) {
      m->bin_count[b] += bc[b];
      m->bin_correct[b] += bk[b];
      m->bin_conf[b] = __dadd_rn(m->bin_conf[b], s_sum[b][0]);
    }
    m->step_rows = step_begin ? n : m->step_rows + n;
    m->step_conf = step_begin ? s_sum[ACNN_ECE_BINS][0] : __dadd_rn(m->step_conf, s_sum[ACNN_ECE_BINS][0]);
  }
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_train_metrics_accumulate(const int32_t* pred, const float* conf, const int32_t* hit_k, const int32_t* labels,
                                  int n, int step_begin, acnn_train_metrics* m, void* stream) {
  ACNN_REQUIRE(pred && conf && hit_k && labels && m, "acnn_train_metrics_accumulate: null pointer");
  ACNN_REQUIRE(n >= 1, "acnn_train_metrics_accumulate: n=%d < 1", n);
  ACNN_REQUIRE(((uintptr_t)m & 7) == 0, "acnn_train_metrics_accumulate: m must be 8-byte aligned");
  launch_k(train_metrics_kernel, dim3(1), dim3(kTrainMetricsThreads), 0, (cudaStream_t)stream, pred, conf, hit_k,
           labels, n, step_begin ? 1 : 0, m);
  count_launch();
  return check_launch("train_metrics_accumulate");
}

}  // extern "C"
