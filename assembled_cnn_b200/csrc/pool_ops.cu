// Pooling / resampling, input packing + mixup, and the softmax cross-entropy loss.
// All activations NHWC bf16, one thread per (pixel, 8-channel group), 16-byte accesses.
// Reference: nets/blocks.py:45-107 (blur-pool), nets/resnet_model.py:123-141,421-424,499,560-561,
// utils/data_util.py:97-158 (mixup), losses/cls_losses.py:28-33.
#include "common.h"
#include "vec.cuh"

namespace acnn {

constexpr int kPT = 256;

struct Binomial {
  float w[7];
};

static Binomial binomial(int filt) {
  static const float rows[7][7] = {{1}, {1, 1}, {1, 2, 1}, {1, 3, 3, 1}, {1, 4, 6, 4, 1},
                                   {1, 5, 10, 10, 5, 1}, {1, 6, 15, 20, 15, 6, 1}};
  Binomial b;
  float s = 0;
  for (int i = 0; i < filt; ++i) s += rows[filt - 1][i];
  for (int i = 0; i < 7; ++i) b.w[i] = i < filt ? rows[filt - 1][i] / s : 0.f;
  return b;
}

__device__ __forceinline__ int reflect(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// ---------------------------------------------------------------------------- blur-pool
// Every thread handles kBlurRows consecutive output rows of one (column, channel-group): the loads
// of all its windows are independent and issued back to back (with one row per thread a short-lived
// CTA keeps too little in flight to fill HBM).
constexpr int kBlurRows = 4;

// FS = filt * 8 + stride as a compile-time constant (0: runtime values): the reference's sconv / 3
// configuration (filt 3, stride 2) gets shifts and fully unrolled windows instead of runtime
// divisions and data-dependent loop bounds (the generic backward is integer-instruction bound)
template <class T, int FS>
__global__ void __launch_bounds__(kPT)
blurpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ out, Binomial bw, int H, int W,
                    int C, int filt_rt, int stride_rt, int pad_rt, int Ho, int Wo) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int filt = FS ? FS / 8 : filt_rt, stride = FS ? FS % 8 : stride_rt;
  const int pad = FS ? (FS / 8 - 1) / 2 : pad_rt;
  // grid = (ceil(Wo * C/8 / threads), ceil(Ho / kBlurRows), B): no 64-bit index decomposition
  const int CG = C >> 3;
  const int idx = blockIdx.x * kPT + threadIdx.x;
  if (idx >= Wo * CG) return;
  const int q = idx / CG;
  const int cg = idx - q * CG;
  const int p0 = blockIdx.y * kBlurRows;
  const int64_t b = blockIdx.z;
  float acc[kBlurRows][8];
#pragma unroll
  for (int r = 0; r < kBlurRows; ++r)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[r][k] = 0.f;
  for (int s = 0; s < filt; ++s) {
    const int iw = reflect(q * stride + s - pad, W);
    for (int t = 0; t < filt; ++t) {
      V8<T> v[kBlurRows];
#pragma unroll
      for (int r = 0; r < kBlurRows; ++r) {
        const int p = p0 + r < Ho ? p0 + r : Ho - 1;          // clamped: loads stay unconditional
        const int ih = reflect(p * stride + t - pad, H);
        v[r].ld(x + ((b * H + ih) * W + iw) * C + cg * 8);
      }
      const float wt = bw.w[t] * bw.w[s];
#pragma unroll
      for (int r = 0; r < kBlurRows; ++r) {
        float f[8];
        v[r].unpack(f);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[r][k] = fmaf(wt, f[k], acc[r][k]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kBlurRows; ++r) {
    if (p0 + r < Ho) store8(out + (((b * Ho + p0 + r) * Wo + q) * CG + cg) * 8, acc[r]);
  }
}

// 1-D adjoint weight: sum over padded positions ip that reflect onto i, and over output positions p
// whose window covers ip.  Calls f(p, weight).
template <class F>
__device__ __forceinline__ void blur_adjoint_1d(int i, int n, int no, const Binomial& bw, int filt,
                                                int stride, int pad, F f) {
  int cand[3];
  int nc = 0;
  cand[nc++] = i;
  if (i > 0 && i <= pad) cand[nc++] = -i;
  if (i < n - 1 && (n - 1 - i) <= pad) cand[nc++] = 2 * (n - 1) - i;
  for (int k = 0; k < nc; ++k) {
    const int ip = cand[k] + pad;   // coordinate in the padded frame
    // p*stride <= ip < p*stride + filt
    int p_hi = ip / stride;
    if (p_hi > no - 1) p_hi = no - 1;
    for (int p = p_hi; p >= 0 && ip - p * stride < filt; --p) f(p, bw.w[ip - p * stride]);
  }
}

template <class T, int FS>
__global__ void __launch_bounds__(kPT)
blurpool_bwd_kernel(const T* __restrict__ dout, T* __restrict__ dx,
                    const T* __restrict__ add_src, const T* __restrict__ mask_src,
                    Binomial bw, int H, int W, int C, int filt_rt, int stride_rt, int pad_rt, int Ho,
                    int Wo) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int filt = FS ? FS / 8 : filt_rt, stride = FS ? FS % 8 : stride_rt;
  const int pad = FS ? (FS / 8 - 1) / 2 : pad_rt;
  // grid = (ceil(W * C/8 / threads), ceil(H / kBlurRows), B)
  const int CG = C >> 3;
  const int idx = blockIdx.x * kPT + threadIdx.x;
  if (idx >= W * CG) return;
  const int iw = idx / CG;
  const int cg = idx - iw * CG;
  const int ih0 = blockIdx.y * kBlurRows;
  const int64_t b = blockIdx.z;
  // the two full-size streams of all rows first (2 * kBlurRows loads in flight), then the gathers
  V8<T> addv[kBlurRows], maskv[kBlurRows];
#pragma unroll
  for (int r = 0; r < kBlurRows; ++r) {
    const int ih = ih0 + r < H ? ih0 + r : H - 1;
    const size_t off = (((size_t)b * H + ih) * W + iw) * C + cg * 8;
    addv[r].zero();
    maskv[r].zero();
    if (add_src) addv[r].ld(add_src + off);
    if (mask_src) maskv[r].ld(mask_src + off);
  }
#pragma unroll
  for (int r = 0; r < kBlurRows; ++r) {
    const int ih = ih0 + r;
    if (ih >= H) break;
    const size_t off = (((size_t)b * H + ih) * W + iw) * C + cg * 8;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    blur_adjoint_1d(ih, H, Ho, bw, filt, stride, pad, [&](int p, float wr) {
      blur_adjoint_1d(iw, W, Wo, bw, filt, stride, pad, [&](int q, float ws) {
        float v[8];
        load8(dout + ((b * Ho + p) * Wo + q) * C + cg * 8, v);
        const float wt = wr * ws;
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(wt, v[k], acc[k]);
      });
    });
    if (add_src) {
      float a[8];
      addv[r].unpack(a);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += a[k];
    }
    if (mask_src) {
      float m[8];
      maskv[r].unpack(m);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (!(m[k] > 0.f)) acc[k] = 0.f;
    }
    store8(dx + off, acc);
  }
}

// ---------------------------------------------------------------------------- avg / max pool
template <class T>
__global__ void __launch_bounds__(kPT)
avgpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ out, int H, int W, int C, int k,
                   int stride, int pad, int Ho, int Wo, int count_pad) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  // grid = (ceil(Wo * C/8 / threads), Ho, B)
  const int CG = C >> 3;
  const int idx = blockIdx.x * kPT + threadIdx.x;
  if (idx >= Wo * CG) return;
  const int q = idx / CG;
  const int cg = idx - q * CG;
  const int p = blockIdx.y;
  const int64_t b = blockIdx.z;
  {
    const int64_t i = ((b * Ho + p) * Wo + q) * CG + cg;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    int cnt = 0;
    for (int r = 0; r < k; ++r) {
      const int ih = p * stride + r - pad;
      if (ih < 0 || ih >= H) continue;
      for (int s = 0; s < k; ++s) {
        const int iw = q * stride + s - pad;
        if (iw < 0 || iw >= W) continue;
        float v[8];
        load8(x + ((b * H + ih) * W + iw) * C + cg * 8, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += v[e];
        ++cnt;
      }
    }
    const float inv = 1.f / (count_pad ? k * k : cnt);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] *= inv;
    store8(out + i * 8, acc);
  }
}

__device__ __forceinline__ int window_count(int p, int stride, int pad, int k, int n) {
  int lo = p * stride - pad, hi = lo + k;
  if (lo < 0) lo = 0;
  if (hi > n) hi = n;
  return hi - lo;
}

// grid = (ceil(W*C/8 / 256), ceil(H / kRows), B): no 64-bit index divisions on the hot path.
// STRIDE > 0 makes the stride a compile-time constant (shifts instead of divisions).  Every thread
// handles kRows consecutive rows of one (column, channel-group): the two full-size streams (add /
// mask tiles) of all its rows are requested first (2 * kRows 16-byte loads in flight per thread),
// the small dout gather (L2 hits) overlaps them.  (With one vector per thread the CTAs are too
// short-lived to keep the memory system full.)
constexpr int kPoolRows = 4;

template <class T, int STRIDE>
__global__ void __launch_bounds__(kPT)
avgpool_bwd_kernel(const T* __restrict__ dout, T* __restrict__ dx,
                   const T* __restrict__ add_src, const T* __restrict__ mask_src, int H, int W,
                   int C, int k, int stride_rt, int pad, int Ho, int Wo, int count_pad) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int stride = STRIDE > 0 ? STRIDE : stride_rt;
  const int CG = C >> 3;
  const int idx = blockIdx.x * kPT + threadIdx.x;
  if (idx >= W * CG) return;
  const int iw = idx / CG;
  const int cg = idx - iw * CG;
  const int ih0 = blockIdx.y * kPoolRows;
  const int64_t b = blockIdx.z;
  V8<T> addv[kPoolRows], maskv[kPoolRows];
#pragma unroll
  for (int r = 0; r < kPoolRows; ++r) {
    const int ih = ih0 + r < H ? ih0 + r : H - 1;          // clamped: loads stay unconditional
    const size_t off = (((size_t)b * H + ih) * W + iw) * C + cg * 8;
    addv[r].zero();
    maskv[r].zero();
    if (add_src) addv[r].ld(add_src + off);
    if (mask_src) maskv[r].ld(mask_src + off);
  }
  int q_hi = (iw + pad) / stride;
  if (q_hi > Wo - 1) q_hi = Wo - 1;
  const float inv_full = 1.f / (k * k);
#pragma unroll
  for (int r = 0; r < kPoolRows; ++r) {
    const int ih = ih0 + r;
    if (ih >= H) break;
    const size_t off = (((size_t)b * H + ih) * W + iw) * C + cg * 8;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    int p_hi = (ih + pad) / stride;
    if (p_hi > Ho - 1) p_hi = Ho - 1;
    for (int p = p_hi; p >= 0 && ih + pad - p * stride < k; --p) {
      const float inv_p = count_pad ? inv_full : 1.f / window_count(p, stride, pad, k, H);
      for (int q = q_hi; q >= 0 && iw + pad - q * stride < k; --q) {
        float v[8];
        load8(dout + ((b * Ho + p) * Wo + q) * C + cg * 8, v);
        const float inv = count_pad ? inv_full : inv_p / window_count(q, stride, pad, k, W);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(inv, v[e], acc[e]);
      }
    }
    if (add_src) {
      float a[8];
      addv[r].unpack(a);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += a[e];
    }
    if (mask_src) {
      float m[8];
      maskv[r].unpack(m);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (!(m[e] > 0.f)) acc[e] = 0.f;
    }
    store8(dx + off, acc);
  }
}

template <class T>
__global__ void __launch_bounds__(kPT)
maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ out, int H, int W, int C, int k,
                   int stride, int pad, int Ho, int Wo, int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    int64_t t = i / CG;
    const int q = (int)(t % Wo);
    t /= Wo;
    const int p = (int)(t % Ho);
    const int64_t b = t / Ho;
    float m[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = -INFINITY;
    for (int r = 0; r < k; ++r) {
      const int ih = p * stride + r - pad;
      if (ih < 0 || ih >= H) continue;
      for (int s = 0; s < k; ++s) {
        const int iw = q * stride + s - pad;
        if (iw < 0 || iw >= W) continue;
        float v[8];
        load8(x + ((b * H + ih) * W + iw) * C + cg * 8, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) m[e] = fmaxf(m[e], v[e]);
      }
    }
    store8(out + i * 8, m);
  }
}

template <class T>
__global__ void __launch_bounds__(kPT)
maxpool_bwd_kernel(const T* __restrict__ dout, const T* __restrict__ x,
                   T* __restrict__ dx, const T* __restrict__ add_src,
                   const T* __restrict__ mask_src, int H, int W, int C, int k, int stride,
                   int pad, int Ho, int Wo, int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    int64_t t = i / CG;
    const int iw = (int)(t % W);
    t /= W;
    const int ih = (int)(t % H);
    const int64_t b = t / H;
    float acc[8], me[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    load8(x + i * 8, me);
    int p_hi = (ih + pad) / stride;
    if (p_hi > Ho - 1) p_hi = Ho - 1;
    int q_hi = (iw + pad) / stride;
    if (q_hi > Wo - 1) q_hi = Wo - 1;
    for (int p = p_hi; p >= 0 && ih + pad - p * stride < k; --p) {
      for (int q = q_hi; q >= 0 && iw + pad - q * stride < k; --q) {
        // (ih, iw) receives the gradient iff it is the FIRST maximum of window (p, q)
        bool win[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) win[e] = true;
        for (int r = 0; r < k; ++r) {
          const int jh = p * stride + r - pad;
          if (jh < 0 || jh >= H) continue;
          for (int s = 0; s < k; ++s) {
            const int jw = q * stride + s - pad;
            if (jw < 0 || jw >= W) continue;
            if (jh == ih && jw == iw) continue;
            float v[8];
            load8(x + ((b * H + jh) * W + jw) * C + cg * 8, v);
            const bool before = (jh < ih) || (jh == ih && jw < iw);
#pragma unroll
            for (int e = 0; e < 8; ++e)
              if (v[e] > me[e] || (before && v[e] == me[e])) win[e] = false;
          }
        }
        float g[8];
        load8(dout + ((b * Ho + p) * Wo + q) * C + cg * 8, g);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (win[e]) acc[e] += g[e];
      }
    }
    grad_epilogue(acc, add_src, mask_src, (size_t)i * 8);
    store8(dx + i * 8, acc);
  }
}

// ---------------------------------------------------------------------------- resampling
template <class T>
__global__ void __launch_bounds__(kPT)
upsample2x_bwd_kernel(const T* __restrict__ dout, T* __restrict__ dx,
                      const T* __restrict__ add_src, const T* __restrict__ mask_src, int H,
                      int W, int C, int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    int64_t t = i / CG;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const int64_t b = t / H;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        float v[8];
        load8(dout + ((b * 2 * H + 2 * h + a) * (2 * W) + 2 * w + c) * C + cg * 8, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += v[e];
      }
    grad_epilogue(acc, add_src, mask_src, (size_t)i * 8);
    store8(dx + i * 8, acc);
  }
}

template <class T>
__global__ void __launch_bounds__(kPT)
zero_insert2x_kernel(const T* __restrict__ dy, T* __restrict__ out, int Ho, int Wo, int H,
                     int W, int C, int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    int64_t t = i / CG;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const int64_t b = t / H;
    V8<T> v;
    v.zero();
    if (!(h & 1) && !(w & 1) && (h >> 1) < Ho && (w >> 1) < Wo)
      v.ld(dy + ((b * Ho + (h >> 1)) * Wo + (w >> 1)) * C + cg * 8);
    v.st(out + i * 8);
  }
}

template <class T>
__global__ void __launch_bounds__(kPT)
gap_bwd_kernel(const T* __restrict__ dpooled, const T* __restrict__ mask_src,
               T* __restrict__ dx, int HW, int C, int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  const float inv = 1.f / HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % CG);
    const int64_t b = (i / CG) / HW;
    float v[8];
    load8(dpooled + b * C + cg * 8, v);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] *= inv;
    grad_epilogue(v, (const T*)nullptr, mask_src, (size_t)i * 8);
    store8(dx + i * 8, v);
  }
}

template <class T>
__global__ void __launch_bounds__(kPT)
grad_combine_kernel(const T* __restrict__ a, const T* __restrict__ add_src,
                    const T* __restrict__ mask_src, T* __restrict__ out, int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v[8];
    load8(a + i * 8, v);
    grad_epilogue(v, add_src, mask_src, (size_t)i * 8);
    store8(out + i * 8, v);
  }
}

// ---------------------------------------------------------------------------- input packing
// One thread per output pixel (b, i, j): 2x2 input pixels x 3 channels -> 16 bf16.
template <class T>
__global__ void __launch_bounds__(kPT)
pack_input_kernel(const float* __restrict__ img, const float* __restrict__ lam1,
                  const float* __restrict__ lam2, int mode, T* __restrict__ out, int Bin, int B,
                  int H, int W, int wpad_lo, int wpad_hi, int64_t npix) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int H2 = H >> 1, W2 = W >> 1;
  const int Wp = W2 + wpad_lo + wpad_hi;
  const int half = Bin >> 1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npix;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % Wp) - wpad_lo;
    int64_t t = i / Wp;
    const int ii = (int)(t % H2);
    const int b = (int)(t / H2);
    if (j < 0 || j >= W2) {              // physical zero padding of the W axis
      V8<T> z;
      z.zero();
      z.st(out + i * 16);
      z.st(out + i * 16 + 8);
      continue;
    }
    int b1 = b, b2 = b;
    float lam = 1.f;
    if (mode == 1) {
      b1 = b;
      b2 = half + b;
      lam = lam1[b];
    } else if (mode == 2) {
      if (b < half) {
        b1 = b;
        b2 = half + b;
        lam = lam1[b];
      } else {
        b1 = b - half;
        b2 = half + (half - 1 - (b - half));
        lam = lam2[b - half];
      }
    }
    float o[16];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const size_t off = ((size_t)(2 * ii + dy) * W + (2 * j + dx)) * 3;
        const float* p1 = img + (size_t)b1 * H * W * 3 + off;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float v = __ldg(p1 + c);
          if (mode != 0) {
            const float v2 = __ldg(img + (size_t)b2 * H * W * 3 + off + c);
            v = lam * v + (1.f - lam) * v2;
          }
          o[(dy * 2 + dx) * 4 + c] = v;
        }
        o[(dy * 2 + dx) * 4 + 3] = 0.f;
      }
    float lo[8], hi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      lo[e] = o[e];
      hi[e] = o[8 + e];
    }
    store8(out + i * 16, lo);
    store8(out + i * 16 + 8, hi);
  }
}

__global__ void mix_labels_kernel(const int32_t* __restrict__ labels,
                                  const float* __restrict__ lam1, const float* __restrict__ lam2,
                                  int mode, float* __restrict__ y, int Bin, int B, int NC) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * NC) return;
  const int b = (int)(i / NC), c = (int)(i - (int64_t)b * NC);
  const int half = Bin >> 1;
  int b1 = b, b2 = b;
  float lam = 1.f;
  if (mode == 1) {
    b2 = half + b;
    lam = lam1[b];
  } else if (mode == 2) {
    if (b < half) {
      b2 = half + b;
      lam = lam1[b];
    } else {
      b1 = b - half;
      b2 = half + (half - 1 - (b - half));
      lam = lam2[b - half];
    }
  }
  const float v1 = labels[b1] == c ? 1.f : 0.f;
  const float v2 = labels[b2] == c ? 1.f : 0.f;
  y[i] = mode == 0 ? v1 : lam * v1 + (1.f - lam) * v2;
}

// ---------------------------------------------------------------------------- loss
__device__ __forceinline__ float block_reduce(float v, bool is_max, float* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  const int nw = blockDim.x >> 5;
  v = sh[0];
  for (int w = 1; w < nw; ++w) v = is_max ? fmaxf(v, sh[w]) : v + sh[w];
  return v;
}

template <class T>
__global__ void __launch_bounds__(kPT)
softmax_ce_kernel(const float* __restrict__ logits, const float* __restrict__ y,
                  const float* __restrict__ yt, float kd_temp, int B, int NC, int ld, float ls,
                  float grad_scale, const float* __restrict__ grad_scale_dev, float* __restrict__ loss_rows, float* __restrict__ kd_rows,
                  float* __restrict__ g32, T* __restrict__ dlogits) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  __shared__ float sh[kPT / 32];
  const int b = blockIdx.x;
  const float* lg = logits + (size_t)b * ld;
  const float* yy = y + (size_t)b * NC;
  const float unif = ls / NC;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < NC; c += kPT) mx = fmaxf(mx, lg[c]);
  mx = block_reduce(mx, true, sh);
  float se = 0.f, sy = 0.f, syl = 0.f;
  for (int c = threadIdx.x; c < NC; c += kPT) {
    const float l = lg[c];
    const float yp = yy[c] * (1.f - ls) + unif;
    se += expf(l - mx);
    sy += yp;
    syl += yp * l;
  }
  se = block_reduce(se, false, sh);
  sy = block_reduce(sy, false, sh);
  syl = block_reduce(syl, false, sh);
  const float lse = mx + logf(se);
  // per-example loss (already / B); summed in a fixed order by ce_finalize_kernel
  if (threadIdx.x == 0) loss_rows[b] = (lse * sy - syl) / B;
  // knowledge distillation (run_loop_classification.py:156-162): T^2 * CE(logits / T, teacher),
  // no label smoothing; d/dlogits = T * (softmax(logits / T) * sum(t) - t) / B
  const float* tt = yt ? yt + (size_t)b * NC : nullptr;
  float lse_t = 0.f, st = 0.f, inv_t = 0.f;
  if (tt) {
    inv_t = 1.f / kd_temp;
    float se_t = 0.f, stl = 0.f;
    for (int c = threadIdx.x; c < NC; c += kPT) {
      se_t += expf((lg[c] - mx) * inv_t);
      st += tt[c];
      stl += tt[c] * lg[c] * inv_t;
    }
    se_t = block_reduce(se_t, false, sh);
    st = block_reduce(st, false, sh);
    stl = block_reduce(stl, false, sh);
    lse_t = mx * inv_t + logf(se_t);
    if (threadIdx.x == 0) kd_rows[b] = kd_temp * kd_temp * (lse_t * st - stl) / B;
  }
  const float gs = (grad_scale_dev ? *grad_scale_dev : grad_scale) / B;
  for (int c = threadIdx.x; c < ld; c += kPT) {
    float g = 0.f;
    if (c < NC) {
      const float yp = yy[c] * (1.f - ls) + unif;
      g = (expf(lg[c] - lse) * sy - yp) * gs;
      if (tt) g += kd_temp * (expf(lg[c] * inv_t - lse_t) * st - tt[c]) * gs;
    }
    g32[(size_t)b * ld + c] = g;
    store1(dlogits + (size_t)b * ld + c, g);
  }
}

// loss_acc[0] += sum_b loss_rows[b]; dbias[c] += sum_b g32[b][c] -- one thread per column, rows in
// order: deterministic (no atomics).  One CTA.
__global__ void __launch_bounds__(1024)
ce_finalize_kernel(const float* __restrict__ loss_rows, const float* __restrict__ kd_rows,
                   const float* __restrict__ g32, int B, int NC, int ld, float* loss_acc,
                   float* dbias) {
  pdl_entry();
  for (int c = threadIdx.x; c <= NC + 1; c += blockDim.x) {
    if (c == NC + 1) {
      if (kd_rows) {
        float s = 0.f;
#pragma unroll 8
        for (int b = 0; b < B; ++b) s += __ldg(kd_rows + b);
        loss_acc[2] += s;
      }
    } else if (c == NC) {
      float s = 0.f;
#pragma unroll 8
      for (int b = 0; b < B; ++b) s += __ldg(loss_rows + b);
      loss_acc[0] += s;
    } else if (dbias) {
      float s = 0.f;
#pragma unroll 8
      for (int b = 0; b < B; ++b) s += __ldg(g32 + (size_t)b * ld + c);
      dbias[c] += s;
    }
  }
}

}  // namespace acnn

using namespace acnn;

template <class T>
static void launch_avgpool_bwd(dim3 grid, cudaStream_t st, const void* dout, void* dx,
                               const void* add_src, const void* mask_src, int H, int W, int C, int k,
                               int stride, int pad_lo, int Ho, int Wo, int count_pad) {
  if (stride == 2) {
    launch_k(avgpool_bwd_kernel<T, 2>, grid, dim3(kPT), 0, st, (const T*)dout, (T*)dx,
             (const T*)add_src, (const T*)mask_src, H, W, C, k, stride, pad_lo, Ho, Wo, count_pad);
  } else if (stride == 1) {
    launch_k(avgpool_bwd_kernel<T, 1>, grid, dim3(kPT), 0, st, (const T*)dout, (T*)dx,
             (const T*)add_src, (const T*)mask_src, H, W, C, k, stride, pad_lo, Ho, Wo, count_pad);
  } else {
    launch_k(avgpool_bwd_kernel<T, 0>, grid, dim3(kPT), 0, st, (const T*)dout, (T*)dx,
             (const T*)add_src, (const T*)mask_src, H, W, C, k, stride, pad_lo, Ho, Wo, count_pad);
  }
}

extern "C" {

int acnn_blurpool_fwd(const void* x, void* out, int B, int H, int W, int C, int filt, int stride,
                      int dtype, void* stream) {
  ACNN_REQUIRE(x && out && C % 8 == 0 && filt >= 1 && filt <= 7 && stride >= 1 &&
                   ACNN_DTYPE_OK(dtype), "blurpool_fwd: bad arguments");
  const int pad = (filt - 1) / 2;
  ACNN_REQUIRE(pad < H && pad < W, "blurpool_fwd: reflect pad %d >= size", pad);
  const int Ho = (H + 2 * pad - filt) / stride + 1, Wo = (W + 2 * pad - filt) / stride + 1;
  ACNN_REQUIRE(Ho <= 65535 && B <= 65535, "blurpool_fwd: Ho / B exceed the grid limits");
  dim3 grid(ceil_div(Wo * (C / 8), kPT), ceil_div(Ho, kBlurRows), B);
  if (filt == 3 && stride == 2) {
    ACNN_BY_DTYPE(dtype, (launch_k(blurpool_fwd_kernel<T, 3 * 8 + 2>, grid, dim3(kPT), 0,
                                   (cudaStream_t)stream, (const T*)x, (T*)out, binomial(filt), H, W,
                                   C, filt, stride, pad, Ho, Wo)));
  } else {
    ACNN_BY_DTYPE(dtype, (launch_k(blurpool_fwd_kernel<T, 0>, grid, dim3(kPT), 0,
                                   (cudaStream_t)stream, (const T*)x, (T*)out, binomial(filt), H, W,
                                   C, filt, stride, pad, Ho, Wo)));
  }
  count_launch();
  return check_launch("blurpool_fwd");
}

int acnn_blurpool_bwd(const void* dout, void* dx, const void* add_src, const void* mask_src, int B,
                      int H, int W, int C, int filt, int stride, int dtype, void* stream) {
  ACNN_REQUIRE(dout && dx && C % 8 == 0 && filt >= 1 && filt <= 7 && stride >= 1 &&
                   ACNN_DTYPE_OK(dtype), "blurpool_bwd: bad arguments");
  const int pad = (filt - 1) / 2;
  const int Ho = (H + 2 * pad - filt) / stride + 1, Wo = (W + 2 * pad - filt) / stride + 1;
  ACNN_REQUIRE(H <= 65535 && B <= 65535, "blurpool_bwd: H / B exceed the grid limits");
  dim3 grid(ceil_div(W * (C / 8), kPT), ceil_div(H, kBlurRows), B);
  if (filt == 3 && stride == 2) {
    ACNN_BY_DTYPE(dtype, (launch_k(blurpool_bwd_kernel<T, 3 * 8 + 2>, grid, dim3(kPT), 0,
                                   (cudaStream_t)stream, (const T*)dout, (T*)dx, (const T*)add_src,
                                   (const T*)mask_src, binomial(filt), H, W, C, filt, stride, pad,
                                   Ho, Wo)));
  } else {
    ACNN_BY_DTYPE(dtype, (launch_k(blurpool_bwd_kernel<T, 0>, grid, dim3(kPT), 0,
                                   (cudaStream_t)stream, (const T*)dout, (T*)dx, (const T*)add_src,
                                   (const T*)mask_src, binomial(filt), H, W, C, filt, stride, pad,
                                   Ho, Wo)));
  }
  count_launch();
  return check_launch("blurpool_bwd");
}

int acnn_avgpool_fwd(const void* x, void* out, int B, int H, int W, int C, int k, int stride,
                     int pad_lo, int Ho, int Wo, int count_pad, int dtype, void* stream) {
  ACNN_REQUIRE(x && out && C % 8 == 0 && k >= 1 && stride >= 1 && ACNN_DTYPE_OK(dtype),
               "avgpool_fwd: bad arguments");
  ACNN_REQUIRE(Ho <= 65535 && B <= 65535, "avgpool_fwd: Ho / B exceed the grid limits");
  dim3 grid(ceil_div(Wo * (C / 8), kPT), Ho, B);
  ACNN_BY_DTYPE(dtype, launch_k(avgpool_fwd_kernel<T>, grid, dim3(kPT), 0, (cudaStream_t)stream,
                                (const T*)x, (T*)out, H, W, C, k, stride, pad_lo, Ho, Wo,
                                count_pad));
  count_launch();
  return check_launch("avgpool_fwd");
}

int acnn_avgpool_bwd(const void* dout, void* dx, const void* add_src, const void* mask_src, int B,
                     int H, int W, int C, int k, int stride, int pad_lo, int Ho, int Wo,
                     int count_pad, int dtype, void* stream) {
  ACNN_REQUIRE(dout && dx && C % 8 == 0 && k >= 1 && stride >= 1 && ACNN_DTYPE_OK(dtype),
               "avgpool_bwd: bad arguments");
  ACNN_REQUIRE(H <= 65535 && B <= 65535, "avgpool_bwd: H / B exceed the grid limits");
  dim3 grid(ceil_div(W * (C / 8), kPT), ceil_div(H, kPoolRows), B);
  ACNN_BY_DTYPE(dtype, launch_avgpool_bwd<T>(grid, (cudaStream_t)stream, dout, dx, add_src, mask_src,
                                             H, W, C, k, stride, pad_lo, Ho, Wo, count_pad));
  count_launch();
  return check_launch("avgpool_bwd");
}

int acnn_maxpool_fwd(const void* x, void* out, int B, int H, int W, int C, int k, int stride,
                     int pad_lo, int Ho, int Wo, int dtype, void* stream) {
  ACNN_REQUIRE(x && out && C % 8 == 0 && k >= 1 && stride >= 1 && ACNN_DTYPE_OK(dtype),
               "maxpool_fwd: bad arguments");
  const int64_t nvec = (int64_t)B * Ho * Wo * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(maxpool_fwd_kernel<T>, dim3(grid_for(nvec)), dim3(kPT), 0,
                                (cudaStream_t)stream, (const T*)x, (T*)out, H, W, C, k, stride,
                                pad_lo, Ho, Wo, nvec));
  count_launch();
  return check_launch("maxpool_fwd");
}

int acnn_maxpool_bwd(const void* dout, const void* x, void* dx, const void* add_src,
                     const void* mask_src, int B, int H, int W, int C, int k, int stride,
                     int pad_lo, int Ho, int Wo, int dtype, void* stream) {
  ACNN_REQUIRE(dout && x && dx && C % 8 == 0 && ACNN_DTYPE_OK(dtype), "maxpool_bwd: bad arguments");
  const int64_t nvec = (int64_t)B * H * W * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(maxpool_bwd_kernel<T>, dim3(grid_for(nvec)), dim3(kPT), 0,
                                (cudaStream_t)stream, (const T*)dout, (const T*)x, (T*)dx,
                                (const T*)add_src, (const T*)mask_src, H, W, C, k, stride, pad_lo,
                                Ho, Wo, nvec));
  count_launch();
  return check_launch("maxpool_bwd");
}

int acnn_upsample2x_bwd(const void* dout, void* dx, const void* add_src, const void* mask_src,
                        int B, int H, int W, int C, int dtype, void* stream) {
  ACNN_REQUIRE(dout && dx && C % 8 == 0 && ACNN_DTYPE_OK(dtype), "upsample2x_bwd: bad arguments");
  const int64_t nvec = (int64_t)B * H * W * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(upsample2x_bwd_kernel<T>, dim3(grid_for(nvec)), dim3(kPT), 0,
                                (cudaStream_t)stream, (const T*)dout, (T*)dx, (const T*)add_src,
                                (const T*)mask_src, H, W, C, nvec));
  count_launch();
  return check_launch("upsample2x_bwd");
}

int acnn_zero_insert2x(const void* dy, void* out, int B, int Ho, int Wo, int H, int W, int C,
                       int dtype, void* stream) {
  ACNN_REQUIRE(dy && out && C % 8 == 0 && ACNN_DTYPE_OK(dtype), "zero_insert2x: bad arguments");
  const int64_t nvec = (int64_t)B * H * W * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(zero_insert2x_kernel<T>, dim3(grid_for(nvec)), dim3(kPT), 0,
                                (cudaStream_t)stream, (const T*)dy, (T*)out, Ho, Wo, H, W, C, nvec));
  count_launch();
  return check_launch("zero_insert2x");
}

int acnn_gap_bwd(const void* dpooled, const void* mask_src, void* dx, int B, int HW, int C,
                 int dtype, void* stream) {
  ACNN_REQUIRE(dpooled && dx && C % 8 == 0 && ACNN_DTYPE_OK(dtype), "gap_bwd: bad arguments");
  const int64_t nvec = (int64_t)B * HW * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(gap_bwd_kernel<T>, dim3(grid_for(nvec)), dim3(kPT), 0,
                                (cudaStream_t)stream, (const T*)dpooled, (const T*)mask_src, (T*)dx,
                                HW, C, nvec));
  count_launch();
  return check_launch("gap_bwd");
}

int acnn_grad_combine(const void* a, const void* add_src, const void* mask_src, void* out,
                      int64_t n, int dtype, void* stream) {
  ACNN_REQUIRE(a && out && n % 8 == 0 && ACNN_DTYPE_OK(dtype), "grad_combine: bad arguments");
  ACNN_BY_DTYPE(dtype, launch_k(grad_combine_kernel<T>, dim3(grid_for(n / 8)), dim3(kPT), 0,
                                (cudaStream_t)stream, (const T*)a, (const T*)add_src,
                                (const T*)mask_src, (T*)out, n / 8));
  count_launch();
  return check_launch("grad_combine");
}

int acnn_pack_input(const float* images, const float* lam1, const float* lam2, int mode, void* out,
                    int Bin, int H, int W, int wpad_lo, int wpad_hi, int dtype, void* stream) {
  ACNN_REQUIRE(images && out && H % 2 == 0 && W % 2 == 0 && mode >= 0 && mode <= 2 &&
                   ACNN_DTYPE_OK(dtype), "pack_input: bad arguments");
  ACNN_REQUIRE(mode == 0 || (lam1 && Bin % 2 == 0), "pack_input: mixup needs lam1 and even batch");
  ACNN_REQUIRE(mode != 2 || lam2, "pack_input: mixup type 2 needs lam2");
  const int B = mode == 1 ? Bin / 2 : Bin;
  ACNN_REQUIRE(wpad_lo >= 0 && wpad_hi >= 0, "pack_input: negative padding");
  const int64_t npix = (int64_t)B * (H / 2) * (W / 2 + wpad_lo + wpad_hi);
  ACNN_BY_DTYPE(dtype, launch_k(pack_input_kernel<T>, dim3(grid_for(npix)), dim3(kPT), 0,
                                (cudaStream_t)stream, images, lam1, lam2, mode, (T*)out, Bin, B, H,
                                W, wpad_lo, wpad_hi, npix));
  count_launch();
  return check_launch("pack_input");
}

int acnn_mix_labels(const int32_t* labels, const float* lam1, const float* lam2, int mode, float* y,
                    int Bin, int NC, void* stream) {
  ACNN_REQUIRE(labels && y && mode >= 0 && mode <= 2, "mix_labels: bad arguments");
  ACNN_REQUIRE(mode == 0 || (lam1 && Bin % 2 == 0), "mix_labels: mixup needs lam1, even batch");
  ACNN_REQUIRE(mode != 2 || lam2, "mix_labels: mixup type 2 needs lam2");
  const int B = mode == 1 ? Bin / 2 : Bin;
  const int64_t n = (int64_t)B * NC;
  launch_k(mix_labels_kernel, dim3((int)ceil_div64(n, 256)), dim3(256), 0, (cudaStream_t)stream, labels, lam1, lam2, mode, y, Bin, B, NC);
  count_launch();
  return check_launch("mix_labels");
}

static int softmax_ce(const float* logits, const float* y, const float* teacher, float kd_temp, int B, int NC,
                      int ld, float label_smoothing, float grad_scale, const float* grad_scale_dev,
                      float* loss_acc, void* dlogits, float* dbias, float* work, int dtype, void* stream) {
  ACNN_REQUIRE(logits && y && loss_acc && dlogits && work && NC <= ld && B > 0 &&
                   ACNN_DTYPE_OK(dtype) && (!teacher || kd_temp > 0.f), "softmax_ce: bad arguments");
  const int Bp = ((B + 31) / 32) * 32;
  float* loss_rows = work;                     // [Bp]
  float* kd_rows = work + Bp;                  // [Bp]
  float* g32 = work + 2 * Bp;                  // [B][ld]
  ACNN_BY_DTYPE(dtype, launch_k(softmax_ce_kernel<T>, dim3(B), dim3(kPT), 0, (cudaStream_t)stream,
                                logits, y, teacher, kd_temp, B, NC, ld, label_smoothing, grad_scale,
                                grad_scale_dev, loss_rows, kd_rows, g32, (T*)dlogits));
  count_launch();
  int rc = check_launch("softmax_ce");
  if (rc) return rc;
  launch_k(ce_finalize_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream,
           (const float*)loss_rows, teacher ? (const float*)kd_rows : (const float*)nullptr,
           (const float*)g32, B, NC, ld, loss_acc, dbias);
  count_launch();
  return check_launch("ce_finalize");
}

int acnn_softmax_ce(const float* logits, const float* y, const float* teacher, float kd_temp, int B,
                    int NC, int ld, float label_smoothing, float grad_scale, float* loss_acc,
                    void* dlogits, float* dbias, float* work, int dtype, void* stream) {
  return softmax_ce(logits, y, teacher, kd_temp, B, NC, ld, label_smoothing, grad_scale, nullptr, loss_acc, dlogits,
                    dbias, work, dtype, stream);
}

int acnn_softmax_ce_scaled(const float* logits, const float* y, const float* teacher, float kd_temp, int B,
                           int NC, int ld, float label_smoothing, const float* grad_scale_dev,
                           float* loss_acc, void* dlogits, float* dbias, float* work, int dtype,
                           void* stream) {
  ACNN_REQUIRE(grad_scale_dev, "softmax_ce_scaled: null grad_scale_dev");
  return softmax_ce(logits, y, teacher, kd_temp, B, NC, ld, label_smoothing, 0.f, grad_scale_dev, loss_acc, dlogits,
                    dbias, work, dtype, stream);
}

}  // extern "C"
