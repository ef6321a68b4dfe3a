// TF 1.14's legacy bilinear resize (resize_bilinear_op.cc, align_corners = half_pixel_centers = false),
// shared by the resampling kernels (eval_preprocess.cu) and AutoAugment's resize (autoaugment.cu).  Every
// step is a separately rounded fp32 operation.
#pragma once

#include <stdint.h>

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

// The resized RGB pixel (y, x) of the uint8 [h][w][3] image at src, with the scales (sy, sx), into v[3]
// (fp32, not rounded to an integer).  With flip the image is mirrored before the resize, whose sample grid
// is anchored at the left edge: column j of the mirrored image is column w - 1 - j.
__device__ __forceinline__ void legacy_bilinear_rgb(const uint8_t* src, int h, int w, float sy, float sx, int y,
                                                    int x, bool flip, float (&v)[3]) {
  const Interp iy = legacy_interp(y, sy, h);
  const Interp ix = legacy_interp(x, sx, w);
  const int cl = flip ? w - 1 - ix.lo : ix.lo;
  const int ch = flip ? w - 1 - ix.hi : ix.hi;
  const uint8_t* top = src + (int64_t)iy.lo * w * 3;
  const uint8_t* bot = src + (int64_t)iy.hi * w * 3;
  const int xl = cl * 3, xh = ch * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t = lerp_rn((float)top[xl + c], (float)top[xh + c], ix.lerp);
    const float u = lerp_rn((float)bot[xl + c], (float)bot[xh + c], ix.lerp);
    v[c] = lerp_rn(t, u, iy.lerp);
  }
}

}  // namespace acnn
