// The training preprocessing of decoded crop windows (preprocessing/imagenet_preprocessing.py:57-97,
// 269-313, is_training=True): random_flip_left_right of the window, _resize_image to S x S (TF 1.14's
// legacy bilinear, independent scales (float)h / S and (float)w / S), mean_image_subtraction, in one pass
// over a batch of windows of different sizes.  The crop itself (sample_distorted_bounding_box +
// decode_and_crop_jpeg) happens on the host: each descriptor points at the window's packed pixels.
#include <math.h>

#include "common.h"
#include "legacy_bilinear.cuh"
#include "vec.cuh"

namespace acnn {

// grid (ceil(S*S / 256), n_valid): one thread per output pixel of one window.
__global__ void __launch_bounds__(256)
crop_resize_u8_kernel(const acnn_crop_desc* __restrict__ desc, int S, const float* __restrict__ mean_dev,
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
  const acnn_crop_desc d = desc[b];
  const int y = p / S, x = p - (p / S) * S;
  const Interp iy = legacy_interp(y, __fdiv_rn((float)d.h, (float)S), d.h);
  const Interp ix = legacy_interp(x, __fdiv_rn((float)d.w, (float)S), d.w);
  // the flip comes before the resize: column j of the mirrored window is column w - 1 - j of the window
  const int cl = d.flip ? d.w - 1 - ix.lo : ix.lo;
  const int ch = d.flip ? d.w - 1 - ix.hi : ix.hi;
  const uint8_t* top = d.src + (int64_t)iy.lo * d.w * 3;
  const uint8_t* bot = d.src + (int64_t)iy.hi * d.w * 3;
  const int xl = cl * 3, xh = ch * 3;
  const float mean[3] = {m0, m1, m2};
  float* o = out + ((int64_t)b * S * S + p) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t = lerp_rn((float)top[xl + c], (float)top[xh + c], ix.lerp);
    const float u = lerp_rn((float)bot[xl + c], (float)bot[xh + c], ix.lerp);
    o[c] = __fsub_rn(lerp_rn(t, u, iy.lerp), mean[c]);
  }
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_crop_resize_u8(const acnn_crop_desc* desc, int B, int n_valid, int S, const float* mean, float* out,
                        void* stream) {
  ACNN_REQUIRE(desc && mean && out, "acnn_crop_resize_u8: null pointer");
  ACNN_REQUIRE(B > 0 && S > 0, "acnn_crop_resize_u8: bad shape B=%d S=%d", B, S);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "acnn_crop_resize_u8: n_valid=%d outside [0, B=%d]", n_valid, B);
  ACNN_REQUIRE(((uintptr_t)out & 3) == 0, "acnn_crop_resize_u8: out must be 4-byte aligned");
  ACNN_REQUIRE(((uintptr_t)desc & 7) == 0, "acnn_crop_resize_u8: desc must be 8-byte aligned");
  ACNN_REQUIRE((int64_t)S * S <= INT32_MAX, "acnn_crop_resize_u8: S=%d too large", S);
  cudaPointerAttributes at{};
  cudaError_t e = cudaPointerGetAttributes(&at, mean);
  if (e != cudaSuccess) {
    set_error("acnn_crop_resize_u8: mean: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  const bool mean_on_device = at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
  const float m0 = mean_on_device ? 0.f : mean[0], m1 = mean_on_device ? 0.f : mean[1],
              m2 = mean_on_device ? 0.f : mean[2];
  if (n_valid == 0) return ACNN_OK;
  launch_k(crop_resize_u8_kernel, dim3(ceil_div(S * S, 256), n_valid), dim3(256), 0, (cudaStream_t)stream, desc,
           S, mean_on_device ? mean : (const float*)nullptr, m0, m1, m2, out);
  count_launch();
  return check_launch("crop_resize_u8");
}

}  // extern "C"
