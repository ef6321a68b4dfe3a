// Parameter handling: bf16 / fp16 operand copies of the fp32 master weights (fprop + dgrad layouts), the
// space-to-depth stem weight transform, and the fused weight-decay + momentum SGD step over the
// flat parameter buffer.  nets/optimizer_setting.py:23-38, nets/run_loop_classification.py:166-179.
#include <algorithm>

#include "common.h"
#include "vec.cuh"

namespace acnn {

// blockIdx.y = tensor; 32x32 tiles of the [Cout][Cin] matrix of every tap, transposed through
// shared memory so both the read (along Cin) and the dgrad write (along Cout) are coalesced.
// x = hi + mid + lo with three bf16 values (24 mantissa bits): the operand planes of the fp32
// parity mode of the conv GEMMs.
__device__ __forceinline__ void split3(float v, bf16& h, bf16& m, bf16& l) {
  h = __float2bfloat16_rn(v);
  const float r1 = v - __bfloat162float(h);      // exact
  m = __float2bfloat16_rn(r1);
  l = __float2bfloat16_rn(r1 - __bfloat162float(m));
}
// fp16 weight copies (ACNN_F16): one plane, round to nearest even
__device__ __forceinline__ void store_planes(f16* base, int64_t idx, float v, int, int64_t) {
  base[idx] = __float2half_rn(v);
}
__device__ __forceinline__ void store_planes(bf16* base, int64_t idx, float v, int planes,
                                             int64_t plane_stride) {
  if (planes == 1) {
    base[idx] = __float2bfloat16_rn(v);
  } else {
    bf16 h, m, l;
    split3(v, h, m, l);
    base[idx] = h;
    base[idx + plane_stride] = m;
    base[idx + 2 * plane_stride] = l;
  }
}

// x fp32 [n] -> planes bf16 [3][n]
__global__ void __launch_bounds__(256)
split3_kernel(const float* __restrict__ x, bf16* __restrict__ planes, int64_t nvec) {
  pdl_wait();
  const int64_t n = nvec * 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v[8], h[8], m[8], l[8];
    loadf8(x + i * 8, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      h[k] = __bfloat162float(__float2bfloat16_rn(v[k]));
      const float r1 = v[k] - h[k];
      m[k] = __bfloat162float(__float2bfloat16_rn(r1));
      l[k] = r1 - m[k];
    }
    store8(planes + i * 8, h);
    store8(planes + n + i * 8, m);
    store8(planes + 2 * n + i * 8, l);
  }
}

template <class E>
__global__ void __launch_bounds__(256)
prep_weights_kernel(const float* __restrict__ master, const acnn_weight_desc* __restrict__ descs,
                    E* __restrict__ w_fprop, E* __restrict__ w_dgrad, int planes,
                    int64_t fprop_plane_stride, int64_t dgrad_plane_stride) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  __shared__ float tile[32][33];
  const acnn_weight_desc d = descs[blockIdx.y];
  const int tco = (d.Cout + 31) / 32, tci = (d.Cin + 31) / 32;
  const int ntiles = tco * tci * d.taps;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int tile_id = blockIdx.x; tile_id < ntiles; tile_id += gridDim.x) {
    const int t = tile_id % d.taps;
    const int rest = tile_id / d.taps;
    const int ci0 = (rest % tci) * 32, co0 = (rest / tci) * 32;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int co = co0 + ty + k * 8, ci = ci0 + tx;
      float v = 0.f;
      if (co < d.Cout && ci < d.Cin) {
        const int64_t idx = ((int64_t)co * d.taps + t) * d.Cin + ci;
        v = master[d.master_off + idx];
        store_planes(w_fprop, d.fprop_off + idx, v, planes, fprop_plane_stride);
      }
      tile[ty + k * 8][tx] = v;
    }
    __syncthreads();
    if (d.dgrad_off >= 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int ci = ci0 + ty + k * 8, co = co0 + tx;
        if (co < d.Cout && ci < d.Cin) {
          const int64_t idx = ((int64_t)ci * d.taps + (d.taps - 1 - t)) * d.Cout + co;
          store_planes(w_dgrad, d.dgrad_off + idx, tile[tx][ty + k * 8], planes,
                       dgrad_plane_stride);
        }
      }
    }
  }
}

// w [Cout][k][k][3] -> w2 [Cout][k2][k2][16]; input pixel offset u - pad = 2*r + a with
// r = tap2 - pad2, a in {0,1};  channel = (a*2 + b)*4 + c.
template <class T>
__global__ void s2d_weight_pack_kernel(const float* __restrict__ w, T* __restrict__ w2, int Cout,
                                       int k, int pad, int k2, int pad2) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)Cout * k2 * k2 * 16;
  if (i >= n) return;
  const int ch = (int)(i % 16);
  int64_t t = i / 16;
  const int s2 = (int)(t % k2);
  t /= k2;
  const int r2 = (int)(t % k2);
  const int co = (int)(t / k2);
  const int c = ch & 3, b = (ch >> 2) & 1, a = ch >> 3;
  const int u = 2 * (r2 - pad2) + a + pad, v = 2 * (s2 - pad2) + b + pad;
  float val = 0.f;
  if (c < 3 && u >= 0 && u < k && v >= 0 && v < k) val = w[(((int64_t)co * k + u) * k + v) * 3 + c];
  store1(w2 + i, val);
}

__global__ void s2d_wgrad_unpack_kernel(const float* __restrict__ dw2, float* __restrict__ dw,
                                        int Cout, int k, int pad, int k2, int pad2) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t n = (int64_t)Cout * k * k * 3;
  if (i >= n) return;
  const int c = (int)(i % 3);
  int64_t t = i / 3;
  const int v = (int)(t % k);
  t /= k;
  const int u = (int)(t % k);
  const int co = (int)(t / k);
  // u - pad = 2*r + a  (floor division)
  const int du = u - pad, dv = v - pad;
  const int r = (du >= 0) ? du / 2 : -((-du + 1) / 2);
  const int s = (dv >= 0) ? dv / 2 : -((-dv + 1) / 2);
  const int a = du - 2 * r, b = dv - 2 * s;
  const int r2 = r + pad2, s2 = s + pad2;
  dw[i] = dw2[(((int64_t)co * k2 + r2) * k2 + s2) * 16 + (a * 2 + b) * 4 + c];
}

// l2_part: acnn_sgd_scratch_floats() floats of scratch: one partial per CTA, and the arrival counter
// (self-resetting) in the LAST slot, whatever the grid: at slot gridDim.x a call with a smaller grid
// than the previous one would read that call's partial sum as its counter and never finish the sum
constexpr int kSgdMaxBlocks = kMaxSms * 8;

// kScaled: the gradient scale comes from the dynamic loss-scale state, 1 / (grad_divisor * scale) rounded
// once from double (what the host computes for a static scale), and a step whose gradients are not finite
// writes neither w nor acc; its L2 sum is still taken
template <bool kScaled>
__global__ void __launch_bounds__(256)
sgd_momentum_kernel(float* __restrict__ w, const float* __restrict__ grad, float* __restrict__ acc,
                    int64_t n, const uint8_t* __restrict__ decay_flag, const float* __restrict__ hp,
                    const acnn_loss_scale_state* __restrict__ ls, int grad_divisor, float* l2_acc,
                    float* l2_part) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  __shared__ float sh[8];
  const float lr = hp[0], mom = hp[1], wd = hp[2];
  float gs = 0.f;
  bool skip = false;
  if constexpr (kScaled) {
    gs = (float)(1.0 / ((double)grad_divisor * (double)ls->scale));
    skip = ls->nonfinite != 0u;
  } else {
    gs = hp[3];
  }
  float l2 = 0.f;
  const int64_t nvec = n >> 2;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const bool dec = decay_flag[(i * 4) >> 8] != 0;
    float4 wv = reinterpret_cast<float4*>(w)[i];
    const float4 gv = reinterpret_cast<const float4*>(grad)[i];
    float4 av = reinterpret_cast<float4*>(acc)[i];
    float ww[4] = {wv.x, wv.y, wv.z, wv.w};
    const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
    float aa[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float g = gg[k] * gs;
      if (dec) {
        l2 += ww[k] * ww[k];
        g = fmaf(wd, ww[k], g);
      }
      aa[k] = fmaf(mom, aa[k], g);
      ww[k] = fmaf(-lr, aa[k], ww[k]);
    }
    if (skip) continue;
    reinterpret_cast<float4*>(w)[i] = make_float4(ww[0], ww[1], ww[2], ww[3]);
    reinterpret_cast<float4*>(acc)[i] = make_float4(aa[0], aa[1], aa[2], aa[3]);
  }
  if (l2_acc) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l2 += __shfl_xor_sync(0xffffffffu, l2, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = l2;
    __syncthreads();
    // per-CTA partial, then the LAST CTA to arrive adds all partials in a fixed pattern (thread t
    // takes partials t, t+256, ...; the 256 thread sums are added in index order): deterministic,
    // the arrival order does not enter the sum
    __shared__ bool is_last;
    __shared__ float tsum[256];
    unsigned int* counter = reinterpret_cast<unsigned int*>(l2_part + kSgdMaxBlocks);
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int k = 0; k < 8; ++k) s += sh[k];
      l2_part[blockIdx.x] = s;
      __threadfence();
      const unsigned int prev = atomicAdd(counter, 1u);
      is_last = prev == gridDim.x - 1;
    }
    __syncthreads();
    if (is_last) {
      __threadfence();
      float t = 0.f;
      for (unsigned int b = threadIdx.x; b < gridDim.x; b += 256) t += __ldcg(l2_part + b);
      tsum[threadIdx.x] = t;
      __syncthreads();
      if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int k = 0; k < 256; ++k) tot += tsum[k];
        l2_acc[0] += 0.5f * wd * tot;
        *counter = 0u;
      }
    }
  }
}

// exponent bits all ones: +-inf or NaN (the complement of isfinite)
__device__ __forceinline__ bool nonfinite(float v) { return (__float_as_uint(v) & 0x7f800000u) == 0x7f800000u; }
__device__ __forceinline__ bool nonfinite4(float4 v) {
  return nonfinite(v.x) | nonfinite(v.y) | nonfinite(v.z) | nonfinite(v.w);
}

// *flag = 1 when any of x[0, n) is not finite; nothing is written otherwise.  An OR of per-element tests:
// neither the grid nor the order of the CTAs changes the result.  The `head` elements before the first
// 16-byte boundary and the tail after the last whole float4 are tested one by one.
__global__ void __launch_bounds__(256)
grads_nonfinite_kernel(const float* __restrict__ x, int64_t head, int64_t nvec, int64_t tail,
                       uint32_t* __restrict__ flag) {
  pdl_wait();
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float4* v = reinterpret_cast<const float4*>(x + head);
  bool bad = false;
  int64_t i = tid;
  // four independent 16-byte loads in flight per thread and iteration
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    const float4 a = __ldcs(v + i), b = __ldcs(v + i + stride), c = __ldcs(v + i + 2 * stride),
                 d = __ldcs(v + i + 3 * stride);
    bad |= nonfinite4(a) | nonfinite4(b) | nonfinite4(c) | nonfinite4(d);
  }
  for (; i < nvec; i += stride) bad |= nonfinite4(__ldcs(v + i));
  if (tid < head) bad |= nonfinite(x[tid]);
  if (tid < tail) bad |= nonfinite(x[head + 4 * nvec + tid]);
  if (__syncthreads_or(bad) && threadIdx.x == 0) *flag = 1u;
}

// TF 2 Keras LossScaleOptimizer's update of the dynamic loss scale, after the SGD step of the flagged
// gradients; clears the flag for the next step.  One thread: the whole state is 32 bytes.
__global__ void loss_scale_update_kernel(acnn_loss_scale_state* __restrict__ s, int growth_interval) {
  pdl_wait();
  const float scale = s->scale;
  s->last_scale = scale;
  if (s->nonfinite != 0u) {
    s->scale = fmaxf(scale * 0.5f, 1.f);
    s->good_steps = 0;
    s->skipped_steps += 1;
  } else {
    int good = s->good_steps + 1;
    if (good >= growth_interval) {
      const float up = scale * 2.f;
      if (!nonfinite(up)) s->scale = up;
      good = 0;
    }
    s->good_steps = good;
  }
  s->nonfinite = 0u;
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_prep_weights(const float* master, const acnn_weight_desc* descs, int n, void* w_fprop,
                      void* w_dgrad, int planes, int64_t fprop_plane_stride,
                      int64_t dgrad_plane_stride, void* stream) {
  ACNN_REQUIRE(master && descs && w_fprop && n > 0 && n < 65536 && (planes == 1 || planes == 3),
               "prep_weights: bad arguments");
  dim3 grid(96, n, 1);
  launch_k(prep_weights_kernel<bf16>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, master, descs,
           (bf16*)w_fprop, (bf16*)w_dgrad, planes, fprop_plane_stride, dgrad_plane_stride);
  count_launch();
  return check_launch("prep_weights");
}

int acnn_prep_weights_f16(const float* master, const acnn_weight_desc* descs, int n, void* w_fprop,
                          void* w_dgrad, void* stream) {
  ACNN_REQUIRE(master && descs && w_fprop && n > 0 && n < 65536, "prep_weights_f16: bad arguments");
  dim3 grid(96, n, 1);
  launch_k(prep_weights_kernel<f16>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, master, descs,
           (f16*)w_fprop, (f16*)w_dgrad, 1, (int64_t)0, (int64_t)0);
  count_launch();
  return check_launch("prep_weights_f16");
}

int acnn_split3(const float* x, void* planes, int64_t n, void* stream) {
  ACNN_REQUIRE(x && planes && n > 0 && n % 8 == 0, "split3: bad arguments (n %% 8)");
  launch_k(split3_kernel, dim3(grid_for(n / 8)), dim3(256), 0, (cudaStream_t)stream, x,
           (bf16*)planes, n / 8);
  count_launch();
  return check_launch("split3");
}

int acnn_s2d_weight_pack(const float* w, void* w2, int Cout, int k, int pad, int k2, int pad2,
                         int dtype, void* stream) {
  ACNN_REQUIRE(w && w2 && ACNN_DTYPE_OK(dtype), "s2d_weight_pack: bad argument");
  const int64_t n = (int64_t)Cout * k2 * k2 * 16;
  if (dtype == ACNN_F32) {
    launch_k(s2d_weight_pack_kernel<float>, dim3((int)ceil_div64(n, 256)), dim3(256), 0,
             (cudaStream_t)stream, w, (float*)w2, Cout, k, pad, k2, pad2);
  } else if (dtype == ACNN_F16) {
    launch_k(s2d_weight_pack_kernel<f16>, dim3((int)ceil_div64(n, 256)), dim3(256), 0,
             (cudaStream_t)stream, w, (f16*)w2, Cout, k, pad, k2, pad2);
  } else {
    launch_k(s2d_weight_pack_kernel<bf16>, dim3((int)ceil_div64(n, 256)), dim3(256), 0,
             (cudaStream_t)stream, w, (bf16*)w2, Cout, k, pad, k2, pad2);
  }
  count_launch();
  return check_launch("s2d_weight_pack");
}

int acnn_s2d_wgrad_unpack(const float* dw2, float* dw, int Cout, int k, int pad, int k2, int pad2,
                          void* stream) {
  ACNN_REQUIRE(dw2 && dw, "s2d_wgrad_unpack: null argument");
  const int64_t n = (int64_t)Cout * k * k * 3;
  launch_k(s2d_wgrad_unpack_kernel, dim3((int)ceil_div64(n, 256)), dim3(256), 0, (cudaStream_t)stream, dw2, dw, Cout, k, pad, k2, pad2);
  count_launch();
  return check_launch("s2d_wgrad_unpack");
}

int acnn_sgd_scratch_floats(void) { return acnn::kSgdMaxBlocks + 1; }

int acnn_sgd_momentum(float* w, const float* grad, float* acc, int64_t n,
                      const uint8_t* decay_flag, const float* hp, float* l2_acc, float* scratch,
                      void* stream) {
  ACNN_REQUIRE(w && grad && acc && decay_flag && hp && n % 256 == 0 && (!l2_acc || scratch),
               "sgd_momentum: bad arguments (n must be a multiple of 256; l2_acc needs scratch)");
  launch_k(sgd_momentum_kernel<false>, dim3(grid_for(n / 4, 256, acnn::kSgdMaxBlocks)), dim3(256), 0,
           (cudaStream_t)stream, w, grad, acc, n, decay_flag, hp, (const acnn_loss_scale_state*)nullptr, 1,
           l2_acc, scratch);
  count_launch();
  return check_launch("sgd_momentum");
}

int acnn_sgd_momentum_loss_scaled(float* w, const float* grad, float* acc, int64_t n, const uint8_t* decay_flag,
                                  const float* hp, const acnn_loss_scale_state* ls, int grad_divisor,
                                  float* l2_acc, float* scratch, void* stream) {
  ACNN_REQUIRE(w && grad && acc && decay_flag && hp && ls && grad_divisor >= 1 && n % 256 == 0 &&
                   (!l2_acc || scratch),
               "sgd_momentum_loss_scaled: bad arguments (n must be a multiple of 256; grad_divisor >= 1; l2_acc "
               "needs scratch)");
  launch_k(sgd_momentum_kernel<true>, dim3(grid_for(n / 4, 256, acnn::kSgdMaxBlocks)), dim3(256), 0,
           (cudaStream_t)stream, w, grad, acc, n, decay_flag, hp, ls, grad_divisor, l2_acc, scratch);
  count_launch();
  return check_launch("sgd_momentum_loss_scaled");
}

int acnn_grads_nonfinite(const float* x, int64_t n, uint32_t* flag, void* stream) {
  ACNN_REQUIRE(x && flag && n > 0 && ((uintptr_t)x & 3) == 0,
               "grads_nonfinite: bad arguments (n > 0, x 4-byte aligned)");
  const int64_t head = std::min<int64_t>(n, (int64_t)((16 - ((uintptr_t)x & 15)) & 15) / 4);
  const int64_t nvec = (n - head) / 4, tail = n - head - 4 * nvec;
  launch_k(grads_nonfinite_kernel, dim3(grid_for(std::max<int64_t>(nvec, 1), 256, acnn::kMaxSms * 8)), dim3(256), 0,
           (cudaStream_t)stream, x, head, nvec, tail, flag);
  count_launch();
  return check_launch("grads_nonfinite");
}

int acnn_loss_scale_update(acnn_loss_scale_state* state, int growth_interval, void* stream) {
  ACNN_REQUIRE(state && growth_interval >= 1, "loss_scale_update: bad arguments (growth_interval >= 1)");
  launch_k(loss_scale_update_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, state, growth_interval);
  count_launch();
  return check_launch("loss_scale_update");
}

int acnn_fill_zero(void* p, int64_t bytes, void* stream) {
  ACNN_REQUIRE(p && bytes >= 0, "fill_zero: bad arguments");
  cudaError_t e = cudaMemsetAsync(p, 0, (size_t)bytes, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    set_error("fill_zero: %s", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

}  // extern "C"
