// AutoAugment on the device (preprocessing/imagenet_preprocessing.py:280-289 and preprocessing/autoaugment.py):
// the training crop window resized to S x S exactly as acnn_crop_resize_u8 does, clip_by_value(0, 255) and a
// truncating cast to uint8, the two operations of the image's sub-policy (resolved on the host, see
// assembled_cnn_b200/autoaugment.py), then the cast back to fp32 and the mean.  Every float step is a
// separately rounded fp32 operation: TF 1.14's CPU kernels were built without FMA.
#include <math.h>

#include "common.h"
#include "legacy_bilinear.cuh"
#include "vec.cuh"

namespace acnn {

namespace {

constexpr int kThreads = 512;

__device__ __forceinline__ uint8_t trunc_u8(float v) {   // clip_by_value(0, 255), then a truncating cast
  return (uint8_t)(int)fminf(fmaxf(v, 0.f), 255.f);
}

// autoaugment.blend(img1, img2, f): f == 0 -> img1, f == 1 -> img2, else img1 + f * (img2 - img1), clipped and
// truncated.  The reference skips the clip for 0 < f < 1, where the value already lies in [0, 255].
__device__ __forceinline__ uint8_t blend(uint8_t a, uint8_t b, float f) {
  if (f == 0.f) return a;
  if (f == 1.f) return b;
  const float fa = (float)a;
  return trunc_u8(__fadd_rn(fa, __fmul_rn(f, __fsub_rn((float)b, fa))));
}

// TF 1.14 rgb_to_grayscale of uint8: convert_image_dtype to float (x * (1/255)), tensordot with the weights
// (left to right), convert_image_dtype back (trunc(g * 255.5)).
__device__ __forceinline__ uint8_t grey(const uint8_t* px) {
  const float inv = 1.f / 255.f;
  float g = __fmul_rn(__fmul_rn((float)px[0], inv), 0.2989f);
  g = __fadd_rn(g, __fmul_rn(__fmul_rn((float)px[1], inv), 0.5870f));
  g = __fadd_rn(g, __fmul_rn(__fmul_rn((float)px[2], inv), 0.1140f));
  return (uint8_t)(int)__fmul_rn(g, 255.5f);
}

struct Shared {
  int hist[3][256];      // Equalize: histogram, then the LUT
  int lo[3], hi[3];      // AutoContrast: per-channel minimum / maximum
};

// AutoContrast: per channel, x * (255 / (hi - lo)) + (-lo * scale), clipped and truncated; hi <= lo: as is.
__device__ void autocontrast(const uint8_t* src, uint8_t* dst, int n, Shared& sh) {
  const int t = threadIdx.x;
  if (t < 3) {
    sh.lo[t] = 255;
    sh.hi[t] = 0;
  }
  __syncthreads();
  int lo[3] = {255, 255, 255}, hi[3] = {0, 0, 0};
  for (int p = t; p < n; p += kThreads) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int v = src[p * 3 + c];
      lo[c] = min(lo[c], v);
      hi[c] = max(hi[c], v);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    atomicMin(&sh.lo[c], lo[c]);
    atomicMax(&sh.hi[c], hi[c]);
  }
  __syncthreads();
  float scale[3], offset[3];
  bool on[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float l = (float)sh.lo[c], h = (float)sh.hi[c];
    on[c] = h > l;
    scale[c] = __fdiv_rn(255.f, __fsub_rn(h, l));
    offset[c] = __fmul_rn(-l, scale[c]);
  }
  for (int p = t; p < n; p += kThreads) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint8_t v = src[p * 3 + c];
      dst[p * 3 + c] = on[c] ? trunc_u8(__fadd_rn(__fmul_rn((float)v, scale[c]), offset[c])) : v;
    }
  }
}

// Equalize (PIL's ImageOps.equalize, per channel, in integers): step = (n - count of the last nonzero bin)
// / 255; step == 0: as is; else lut[v] = (sum of the bins below v + step / 2) / step, clipped to 255.
__device__ void equalize(const uint8_t* src, uint8_t* dst, int n, Shared& sh) {
  const int t = threadIdx.x;
  for (int i = t; i < 3 * 256; i += kThreads) (&sh.hist[0][0])[i] = 0;
  __syncthreads();
  for (int p = t; p < n; p += kThreads) {
#pragma unroll
    for (int c = 0; c < 3; ++c) atomicAdd(&sh.hist[c][src[p * 3 + c]], 1);
  }
  __syncthreads();
  // warp c < 3 turns channel c's histogram into its LUT: each lane owns 8 consecutive bins
  const int warp = t >> 5, lane = t & 31;
  if (warp < 3) {
    int* h = sh.hist[warp];
    int v[8], own = 0, last = -1;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      v[k] = h[lane * 8 + k];
      own += v[k];
      if (v[k]) last = lane * 8 + k;
    }
    int incl = own;   // inclusive prefix over lanes
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    int top = last;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) top = max(top, __shfl_xor_sync(0xffffffffu, top, d));
    const int step = (total - (top >= 0 ? h[top] : 0)) / 255;
    __syncwarp();   // every lane has read h[top] before the LUT overwrites it
    int below = incl - own;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      h[lane * 8 + k] = step == 0 ? lane * 8 + k : min((below + step / 2) / step, 255);
      below += v[k];
    }
  }
  __syncthreads();
  for (int p = t; p < n; p += kThreads) {
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[p * 3 + c] = (uint8_t)sh.hist[c][src[p * 3 + c]];
  }
}

// Sharpness: blend(smooth, x, f), smooth = the 3x3 VALID depthwise convolution with [[1,1,1],[1,5,1],[1,1,1]]
// / 13 (fp32, taps left to right from 0), clipped and truncated; the one-pixel border keeps x.
__device__ void sharpness(const uint8_t* src, uint8_t* dst, int S, float f) {
  const float w1 = 1.f / 13.f, w5 = 5.f / 13.f;
  for (int p = threadIdx.x; p < S * S; p += kThreads) {
    const int y = p / S, x = p - y * S;
    const bool inner = y >= 1 && y <= S - 2 && x >= 1 && x <= S - 2;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint8_t v = src[p * 3 + c];
      uint8_t d = v;
      if (inner) {
        float acc = 0.f;
#pragma unroll
        for (int ky = -1; ky <= 1; ++ky) {
#pragma unroll
          for (int kx = -1; kx <= 1; ++kx) {
            const float w = (ky == 0 && kx == 0) ? w5 : w1;
            acc = __fadd_rn(acc, __fmul_rn((float)src[((y + ky) * S + x + kx) * 3 + c], w));
          }
        }
        d = trunc_u8(acc);
      }
      dst[p * 3 + c] = blend(d, v, f);
    }
  }
}

// Rotate / shear / translate: tf.contrib.image.transform with NEAREST of the wrapped image, then unwrap.
// Output (x, y) reads source (round(t3 x + t4 y + t5), round(t0 x + t1 y + t2)), std::round (half away from
// zero); a source outside the image leaves the wrap channel 0 and so becomes (128, 128, 128).
__device__ void transform(const uint8_t* src, uint8_t* dst, int S, const float* t) {
  for (int p = threadIdx.x; p < S * S; p += kThreads) {
    const int y = p / S, x = p - y * S;
    const float fx = (float)x, fy = (float)y;
    const float in_x = roundf(__fadd_rn(__fadd_rn(__fmul_rn(t[0], fx), __fmul_rn(t[1], fy)), t[2]));
    const float in_y = roundf(__fadd_rn(__fadd_rn(__fmul_rn(t[3], fx), __fmul_rn(t[4], fy)), t[5]));
    const bool inside = in_x >= 0.f && in_x < (float)S && in_y >= 0.f && in_y < (float)S;
    const uint8_t* s = inside ? src + ((int)in_y * S + (int)in_x) * 3 : nullptr;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[p * 3 + c] = inside ? s[c] : (uint8_t)128;
  }
}

// One operation from src to dst (never the same plane).  `op` is uniform across the block.
__device__ void apply_op(const acnn_autoaugment_op& o, const uint8_t* src, uint8_t* dst, int S, Shared& sh) {
  const int n = S * S;
  const int t = threadIdx.x;
  switch (o.op) {
    case ACNN_AA_AUTOCONTRAST:
      autocontrast(src, dst, n, sh);
      return;
    case ACNN_AA_EQUALIZE:
      equalize(src, dst, n, sh);
      return;
    case ACNN_AA_SHARPNESS:
      sharpness(src, dst, S, o.f[0]);
      return;
    case ACNN_AA_ROTATE:
    case ACNN_AA_SHEAR_X:
    case ACNN_AA_SHEAR_Y:
    case ACNN_AA_TRANSLATE_X:
    case ACNN_AA_TRANSLATE_Y:
      transform(src, dst, S, o.f);
      return;
    case ACNN_AA_CUTOUT: {
      const int cy = o.i[0], cx = o.i[1], pad = o.i[2];
      const int y0 = max(0, cy - pad), y1 = min(S, cy + pad), x0 = max(0, cx - pad), x1 = min(S, cx + pad);
      for (int p = t; p < n; p += kThreads) {
        const int y = p / S, x = p - y * S;
        const bool cut = y >= y0 && y < y1 && x >= x0 && x < x1;
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[p * 3 + c] = cut ? (uint8_t)128 : src[p * 3 + c];
      }
      return;
    }
    case ACNN_AA_COLOR:
      for (int p = t; p < n; p += kThreads) {
        const uint8_t g = grey(src + p * 3);
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[p * 3 + c] = blend(g, src[p * 3 + c], o.f[0]);
      }
      return;
    default:
      break;
  }
  // per-byte operations
  const int shift = o.i[0] & 7;
  for (int i = t; i < 3 * n; i += kThreads) {
    const int v = src[i];
    int r = v;
    switch (o.op) {
      case ACNN_AA_INVERT: r = 255 - v; break;
      case ACNN_AA_POSTERIZE: r = ((v >> shift) << shift) & 255; break;
      case ACNN_AA_SOLARIZE: r = v < o.i[0] ? v : 255 - v; break;
      case ACNN_AA_SOLARIZE_ADD: r = v < 128 ? min(max(v + o.i[0], 0), 255) : v; break;
      case ACNN_AA_CONTRAST: r = blend((uint8_t)o.i[0], (uint8_t)v, o.f[0]); break;
      case ACNN_AA_BRIGHTNESS: r = blend(0, (uint8_t)v, o.f[0]); break;
      default: break;
    }
    dst[i] = (uint8_t)r;
  }
}

}  // namespace

// grid n_valid: one CTA per image.  Plane A = work + b * 2 * plane, plane B = A + plane.
__global__ void __launch_bounds__(kThreads)
crop_resize_autoaugment_kernel(const acnn_crop_desc* __restrict__ desc, const acnn_autoaugment_desc* __restrict__ aug,
                               int S, int64_t plane, const float* __restrict__ mean_dev, float m0, float m1, float m2,
                               uint8_t* __restrict__ work, float* __restrict__ out) {
  pdl_entry();
  __shared__ Shared sh;
  if (mean_dev) {
    m0 = mean_dev[0];
    m1 = mean_dev[1];
    m2 = mean_dev[2];
  }
  const int b = blockIdx.x;
  const int n = S * S;
  const acnn_crop_desc d = desc[b];
  uint8_t* pa = work + (int64_t)b * 2 * plane;
  uint8_t* pb = pa + plane;
  // step 1: acnn_crop_resize_u8's flip + resize, then clip and truncate
  const float sy = __fdiv_rn((float)d.h, (float)S), sx = __fdiv_rn((float)d.w, (float)S);
  for (int p = threadIdx.x; p < n; p += kThreads) {
    const int y = p / S, x = p - y * S;
    float v[3];
    legacy_bilinear_rgb(d.src, d.h, d.w, sy, sx, y, x, d.flip != 0, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) pa[p * 3 + c] = trunc_u8(v[c]);
  }
  __syncthreads();
  // step 2: the two operations, ping-ponging between the planes; an identity slot costs nothing
  const uint8_t* cur = pa;
#pragma unroll 1
  for (int s = 0; s < 2; ++s) {
    const acnn_autoaugment_op o = aug[b].slot[s];
    if (o.op <= ACNN_AA_IDENTITY || o.op >= ACNN_AA_NUM_OPS) continue;
    uint8_t* dst = cur == pa ? pb : pa;
    apply_op(o, cur, dst, S, sh);
    __syncthreads();
    cur = dst;
  }
  // step 3: cast to fp32, - mean
  float* o = out + (int64_t)b * n * 3;
  for (int i = threadIdx.x; i < 3 * n; i += kThreads) {
    const int c = i % 3;
    o[i] = __fsub_rn((float)cur[i], c == 0 ? m0 : (c == 1 ? m1 : m2));
  }
}

}  // namespace acnn

using namespace acnn;

static int64_t aa_plane_bytes(int S) { return ((int64_t)S * S * 3 + 15) / 16 * 16; }

extern "C" {

int64_t acnn_autoaugment_work_bytes(int B, int S) {
  if (B < 1 || S < 1 || (int64_t)S * S > INT32_MAX / 3) return -1;
  return (int64_t)B * 2 * aa_plane_bytes(S);
}

int acnn_crop_resize_autoaugment_u8(const acnn_crop_desc* desc, const acnn_autoaugment_desc* aug, int B,
                                    int n_valid, int S, const float* mean, uint8_t* work, float* out,
                                    void* stream) {
  static_assert(sizeof(acnn_autoaugment_desc) == 88, "acnn_autoaugment_desc is 88 bytes");
  ACNN_REQUIRE(desc && aug && mean && work && out, "acnn_crop_resize_autoaugment_u8: null pointer");
  ACNN_REQUIRE(B > 0 && S > 0, "acnn_crop_resize_autoaugment_u8: bad shape B=%d S=%d", B, S);
  ACNN_REQUIRE(n_valid >= 0 && n_valid <= B, "acnn_crop_resize_autoaugment_u8: n_valid=%d outside [0, B=%d]",
               n_valid, B);
  ACNN_REQUIRE(((uintptr_t)out & 3) == 0, "acnn_crop_resize_autoaugment_u8: out must be 4-byte aligned");
  ACNN_REQUIRE(((uintptr_t)desc & 7) == 0, "acnn_crop_resize_autoaugment_u8: desc must be 8-byte aligned");
  ACNN_REQUIRE(((uintptr_t)aug & 7) == 0, "acnn_crop_resize_autoaugment_u8: aug must be 8-byte aligned");
  ACNN_REQUIRE(((uintptr_t)work & 15) == 0, "acnn_crop_resize_autoaugment_u8: work must be 16-byte aligned");
  ACNN_REQUIRE((int64_t)S * S <= INT32_MAX / 3, "acnn_crop_resize_autoaugment_u8: S=%d too large", S);
  const float* mean_dev;
  float m[3];
  const int rc = resolve_mean("acnn_crop_resize_autoaugment_u8", mean, &mean_dev, m);
  if (rc != ACNN_OK) return rc;
  if (n_valid == 0) return ACNN_OK;
  launch_k(crop_resize_autoaugment_kernel, dim3(n_valid), dim3(kThreads), 0, (cudaStream_t)stream, desc, aug, S,
           aa_plane_bytes(S), mean_dev, m[0], m[1], m[2], work, out);
  count_launch();
  return check_launch("crop_resize_autoaugment_u8");
}

}  // extern "C"
