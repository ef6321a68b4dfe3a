// Head / regularisation kernels outside the conv -> BN -> ReLU stack: DropBlock (mask generation with
// a counter-based Philox RNG, 7x7 dilation, global renormalisation, apply), generalized-mean (GeM)
// pooling backward, and the knowledge-distillation teacher labels.
// Reference: nets/blocks.py:22-42 (GeM), :187-251 (dropblock), nets/resnet_model.py:432-453,
// nets/run_loop_classification.py:86-96,156-162 (KD), utils/data_util.py:128-156 (teacher mixup).
#include "common.h"
#include "vec.cuh"

namespace acnn {

// ------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011): counter-based, so a mask is a pure function of
// (seed, layer, step, element) -- reproducible under CUDA-graph replay and across ranks.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// bern[s][t][c] = 1 if uniform < gamma (tf: relu(sign(gamma - u))), gamma from the DEVICE keep_prob.
__global__ void dropblock_bern_kernel(const float* __restrict__ u, const float* __restrict__ keep_prob,
                                      const uint32_t* __restrict__ step, uint32_t seed_lo,
                                      uint32_t seed_hi, float gamma_scale, int bs, int H, int W,
                                      int n, float* __restrict__ bern) {
  pdl_entry();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float kp = *keep_prob;
  const float gamma = (1.f - kp) * (float)(W * H) / (float)(bs * bs) /
                      (float)((W - bs + 1) * (H - bs + 1)) * gamma_scale;
  float r;
  if (u) {
    r = u[i];
  } else {
    const uint4 x = philox4x32_10(make_uint4((uint32_t)i, step ? *step : 0u, 0u, 0u),
                                  make_uint2(seed_lo, seed_hi));
    r = (float)(x.x >> 8) * (1.f / 16777216.f);      // [0, 1)
  }
  bern[i] = r < gamma ? 1.f : 0.f;
}

// keep[i][j][c] = 1 - max over the bs x bs window (TF SAME, stride 1) of the zero-padded sampling
// mask (tl cells before, br after); one partial sum of `keep` per CTA for the ordered total.
__global__ void __launch_bounds__(256)
dropblock_keep_kernel(const float* __restrict__ bern, float* __restrict__ keep,
                      float* __restrict__ parts, int H, int W, int C, int bs) {
  pdl_entry();
  __shared__ float red[256];
  const int n = H * W * C;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  float k = 0.f;
  if (idx < n) {
    const int c = idx % C;
    const int j = (idx / C) % W;
    const int i = idx / (C * W);
    const int br = (bs - 1) / 2, tl = (bs - 1) - br;
    const int hs = H - bs + 1, ws = W - bs + 1;
    const int lo = bs / 2;                       // SAME padding of the max-pool, odd bs
    float m = 0.f;
    for (int a = -lo; a < bs - lo; ++a) {
      const int s = i + a - tl;
      if (s < 0 || s >= hs) continue;
      for (int b = -lo; b < bs - lo; ++b) {
        const int t = j + b - tl;
        if (t < 0 || t >= ws) continue;
        m = fmaxf(m, bern[((size_t)s * ws + t) * C + c]);
      }
    }
    k = 1.f - m;
    keep[idx] = k;
  }
  red[threadIdx.x] = k;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) parts[blockIdx.x] = red[0];
}

// scale = size / (sum(keep) + 1e-8): fixed-order sum of the per-CTA partials (one CTA).
__global__ void __launch_bounds__(256)
dropblock_scale_kernel(const float* __restrict__ parts, int nparts, float size, float* scale) {
  pdl_entry();
  __shared__ float red[256];
  float t = 0.f;
  for (int p = threadIdx.x; p < nparts; p += 256) t += parts[p];
  red[threadIdx.x] = t;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *scale = size / (red[0] + 1e-8f);
}

// out = relu?(x * keep[hw, c] * scale): the forward, and (relu = 0) its backward on gradients.
template <class T>
__global__ void __launch_bounds__(256)
dropblock_apply_kernel(const T* __restrict__ x, const float* __restrict__ keep,
                       const float* __restrict__ scale, int relu, T* __restrict__ out,
                       int64_t hwc8, int64_t nvec) {
  pdl_wait();
  const float sc = *scale;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v[8], k[8];
    load8(x + i * 8, v);
    loadf8(keep + (i % hwc8) * 8, k);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[e] = v[e] * k[e] * sc;
      if (relu) v[e] = fmaxf(v[e], 0.f);
    }
    store8(out + i * 8, v);
  }
}

// ------------------------------------------------------------------------------------------
// GeM pooling, p = 3:  pooled = N^(-1/3) * cbrt(max(S, 1e-6)), S = sum_hw clip(x, 1e-6, 1e12)^3
// ------------------------------------------------------------------------------------------
// one CTA per image; thread = 8-channel group x row lane (same layout as image_reduce_kernel)
template <class T>
__global__ void __launch_bounds__(256)
gem_fwd_kernel(const T* __restrict__ x, T* __restrict__ pooled, float* __restrict__ ssum, int HW,
               int C) {
  pdl_entry();
  __shared__ float red[256][9];
  const int CG = C >> 3;
  const int cgs = CG < 256 ? CG : 256;
  const int RPB = 256 / cgs;
  const int rsub = threadIdx.x / cgs;
  const int64_t b = blockIdx.x;
  for (int cg = threadIdx.x % cgs; cg < CG; cg += cgs) {
    const int c0 = cg << 3;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int r = rsub; r < HW; r += RPB) {
      float v[8];
      load8(x + (b * HW + r) * C + c0, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float t = fminf(fmaxf(v[i], 1e-6f), 1e12f);
        acc[i] += t * t * t;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.x][i] = acc[i];
    __syncthreads();
    if (rsub == 0) {
      for (int r = 1; r < RPB; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += red[r * cgs + (threadIdx.x % cgs)][i];
      float o[8];
      const float nn = powf((float)HW, -1.f / 3.f);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = nn * cbrtf(fmaxf(acc[i], 1e-6f));
      storef8(ssum + b * C + c0, acc);
      store8(pooled + b * C + c0, o);
    }
    __syncthreads();
  }
}

// dx = dpooled * N^(-1/3) * S^(-2/3) * x^2 inside the clip range (0 where x was clipped or S was
// floored at 1e-6); x <= 0 (ReLU output) is always clipped, so no separate ReLU mask is needed.
template <class T>
__global__ void __launch_bounds__(256)
gem_bwd_kernel(const T* __restrict__ dpooled, const float* __restrict__ ssum,
               const T* __restrict__ x, T* __restrict__ dx, int HW, int C, int64_t nvec) {
  pdl_wait();
  const int CG = C >> 3;
  const float nn = powf((float)HW, -1.f / 3.f);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    const int64_t b = (i / CG) / HW;
    float dp[8], s[8], v[8], o[8];
    load8(dpooled + b * C + cg * 8, dp);
    loadf8(ssum + b * C + cg * 8, s);
    load8(x + i * 8, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const bool in = v[e] >= 1e-6f && v[e] <= 1e12f && s[e] > 1e-6f;
      const float c3 = cbrtf(s[e]);
      o[e] = in ? dp[e] * nn * v[e] * v[e] / (c3 * c3) : 0.f;
    }
    store8(dx + i * 8, o);
  }
}

// ------------------------------------------------------------------------------------------
// KD teacher labels: yt[b] = mix of softmax(teacher_logits / T) rows, same pairing as the images.
// mode 0: yt[b] = p[b]; 1: lam1*p[b] + (1-lam1)*p[half+b]; 2: first half as 1, second half
// lam2*onehot(labels[b-half]) + (1-lam2)*p[half + (half-1-(b-half))]  (sic: the reference mixes the
// SUPERVISED one-hot there, utils/data_util.py:154).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce_256(float v, bool is_max, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = sh[0];
  for (int w = 1; w < 8; ++w) v = is_max ? fmaxf(v, sh[w]) : v + sh[w];
  return v;
}

__global__ void __launch_bounds__(256)
kd_teacher_labels_kernel(const float* __restrict__ tl, const int32_t* __restrict__ labels,
                         const float* __restrict__ lam1, const float* __restrict__ lam2, int mode,
                         float inv_t, float* __restrict__ yt, int Bin, int NC) {
  pdl_entry();
  __shared__ float sh[8];
  const int b = blockIdx.x;
  const int half = Bin >> 1;
  int r1 = b, r2 = -1, onehot = -1;
  float lam = 1.f;
  if (mode == 1) {
    r2 = half + b;
    lam = lam1[b];
  } else if (mode == 2) {
    if (b < half) {
      r2 = half + b;
      lam = lam1[b];
    } else {
      r1 = -1;
      onehot = labels[b - half];
      r2 = half + (half - 1 - (b - half));
      lam = lam2[b - half];
    }
  }
  float mx[2] = {0.f, 0.f}, se[2] = {1.f, 1.f};
  const int rows[2] = {r1, r2};
  for (int k = 0; k < 2; ++k) {
    if (rows[k] < 0) continue;                               // block-uniform
    const float* p = tl + (size_t)rows[k] * NC;
    float m = -INFINITY;
    for (int c = threadIdx.x; c < NC; c += 256) m = fmaxf(m, p[c] * inv_t);
    m = block_reduce_256(m, true, sh);
    float s = 0.f;
    for (int c = threadIdx.x; c < NC; c += 256) s += expf(p[c] * inv_t - m);
    s = block_reduce_256(s, false, sh);
    mx[k] = m;
    se[k] = s;
  }
  for (int c = threadIdx.x; c < NC; c += 256) {
    const float a = r1 >= 0 ? expf(tl[(size_t)r1 * NC + c] * inv_t - mx[0]) / se[0]
                            : (onehot == c ? 1.f : 0.f);
    float v = a;
    if (r2 >= 0) v = lam * a + (1.f - lam) * expf(tl[(size_t)r2 * NC + c] * inv_t - mx[1]) / se[1];
    yt[(size_t)b * NC + c] = v;
  }
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_dropblock_scratch_floats(int H, int W, int C, int block_size) {
  if (H < block_size || W < block_size || C <= 0) return 0;
  const int n = H * W * C;
  // [bern: hs*ws*C | partial sums: ceil(n / 256)]
  return (H - block_size + 1) * (W - block_size + 1) * C + (n + 255) / 256;
}

int acnn_dropblock_mask(const float* u, const float* keep_prob, const uint32_t* step, uint64_t seed,
                        float gamma_scale, int block_size, float* keep, float* scale,
                        float* scratch, int H, int W, int C, void* stream) {
  ACNN_REQUIRE(keep_prob && keep && scale && scratch && block_size >= 1 && (block_size & 1),
               "dropblock_mask: bad arguments (odd block_size)");
  ACNN_REQUIRE(H >= block_size && W >= block_size && C > 0,
               "dropblock_mask: feature map %dx%d smaller than block_size %d", H, W, block_size);
  cudaStream_t st = (cudaStream_t)stream;
  const int hs = H - block_size + 1, ws = W - block_size + 1;
  const int nb = hs * ws * C, n = H * W * C;
  float* bern = scratch;
  float* parts = scratch + nb;
  launch_k(dropblock_bern_kernel, dim3(ceil_div(nb, 256)), dim3(256), 0, st, u, keep_prob, step,
           (uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32), gamma_scale, block_size, H, W, nb,
           bern);
  count_launch();
  int rc = check_launch("dropblock_bern");
  if (rc) return rc;
  const int nparts = ceil_div(n, 256);
  launch_k(dropblock_keep_kernel, dim3(nparts), dim3(256), 0, st, (const float*)bern, keep, parts, H,
           W, C, block_size);
  count_launch();
  if ((rc = check_launch("dropblock_keep"))) return rc;
  launch_k(dropblock_scale_kernel, dim3(1), dim3(256), 0, st, (const float*)parts, nparts, (float)n,
           scale);
  count_launch();
  return check_launch("dropblock_scale");
}

int acnn_dropblock_apply(const void* x, const float* keep, const float* scale, int relu, void* out,
                         int B, int HW, int C, int dtype, void* stream) {
  ACNN_REQUIRE(x && keep && scale && out && C % 8 == 0 && ACNN_DTYPE_OK(dtype),
               "dropblock_apply: bad arguments");
  const int64_t hwc8 = (int64_t)HW * C / 8, nvec = (int64_t)B * hwc8;
  ACNN_BY_DTYPE(dtype, launch_k(dropblock_apply_kernel<T>, dim3(grid_for(nvec)), dim3(256), 0,
                                (cudaStream_t)stream, (const T*)x, keep, scale, relu, (T*)out, hwc8,
                                nvec));
  count_launch();
  return check_launch("dropblock_apply");
}

int acnn_gem_fwd(const void* x, void* pooled, float* ssum, int B, int HW, int C, int dtype,
                 void* stream) {
  ACNN_REQUIRE(x && pooled && ssum && C % 8 == 0 && ACNN_DTYPE_OK(dtype), "gem_fwd: bad arguments");
  const int cg = C >> 3;
  ACNN_REQUIRE(cg >= 256 ? cg % 256 == 0 : 256 % cg == 0, "gem_fwd: C=%d unsupported", C);
  ACNN_BY_DTYPE(dtype, launch_k(gem_fwd_kernel<T>, dim3(B), dim3(256), 0, (cudaStream_t)stream,
                                (const T*)x, (T*)pooled, ssum, HW, C));
  count_launch();
  return check_launch("gem_fwd");
}

int acnn_gem_bwd(const void* dpooled, const float* ssum, const void* x, void* dx, int B, int HW,
                 int C, int dtype, void* stream) {
  ACNN_REQUIRE(dpooled && ssum && x && dx && C % 8 == 0 && ACNN_DTYPE_OK(dtype),
               "gem_bwd: bad arguments");
  const int64_t nvec = (int64_t)B * HW * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(gem_bwd_kernel<T>, dim3(grid_for(nvec)), dim3(256), 0,
                                (cudaStream_t)stream, (const T*)dpooled, ssum, (const T*)x, (T*)dx,
                                HW, C, nvec));
  count_launch();
  return check_launch("gem_bwd");
}

int acnn_kd_teacher_labels(const float* teacher_logits, const int32_t* labels, const float* lam1,
                           const float* lam2, int mode, float kd_temp, float* yt, int Bin, int NC,
                           void* stream) {
  ACNN_REQUIRE(teacher_logits && yt && kd_temp > 0.f && mode >= 0 && mode <= 2,
               "kd_teacher_labels: bad arguments");
  ACNN_REQUIRE(mode == 0 || (lam1 && Bin % 2 == 0), "kd_teacher_labels: mixup needs lam1, even batch");
  ACNN_REQUIRE(mode != 2 || (lam2 && labels), "kd_teacher_labels: mixup type 2 needs lam2 and labels");
  const int B = mode == 1 ? Bin / 2 : Bin;
  launch_k(kd_teacher_labels_kernel, dim3(B), dim3(256), 0, (cudaStream_t)stream, teacher_logits,
           labels, lam1, lam2, mode, 1.f / kd_temp, yt, Bin, NC);
  count_launch();
  return check_launch("kd_teacher_labels");
}

}  // extern "C"
