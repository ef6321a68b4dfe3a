// TF 1.14's legacy bilinear resize (resize_bilinear_op.cc, align_corners = half_pixel_centers = false),
// the per-coordinate pieces shared by the eval (eval_preprocess.cu) and training (train_preprocess.cu)
// preprocessing kernels.  Every step is a separately rounded fp32 operation.
#pragma once

namespace acnn {

// TF's compute_interpolation_weights with the LegacyScaler (resize_bilinear_op.cc): in = i * scale,
// lower = max(floor(in), 0), upper = min(ceil(in), n - 1), lerp = in - floor(in), all in fp32.
// `lower` is also clamped to n - 1: the fp32 product never reaches n for i < out_size, so this only
// guards the read.
struct Interp {
  int lo, hi;
  float lerp;
};

__device__ __forceinline__ Interp legacy_interp(int i, float scale, int n) {
  const float in = __fmul_rn((float)i, scale);
  const float in_f = floorf(in);
  Interp r;
  r.lo = min(max((int)in_f, 0), n - 1);
  r.hi = min((int)ceilf(in), n - 1);
  r.lerp = __fsub_rn(in, in_f);
  return r;
}

// a + (b - a) * t without contraction: TF 1.14's CPU kernels were built without FMA.
__device__ __forceinline__ float lerp_rn(float a, float b, float t) {
  return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), t));
}

}  // namespace acnn
