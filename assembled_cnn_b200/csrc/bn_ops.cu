// Batch-norm, SK and SE elementwise / reduction kernels (HBM-bound; 16-byte vector accesses along
// the NHWC channel dimension, per-channel reductions through shared memory + one atomic per
// channel per CTA).  Reference: nets/model_helper.py:26-37, nets/blocks.py:110-184 and the
// explicit backward formulas of batch normalisation.
#include "common.h"
#include "stream_pipe.cuh"
#include "vec.cuh"

namespace acnn {

constexpr int kT = 256;

// ------------------------------------------------------------------------------------------
// bn_finalize
// ------------------------------------------------------------------------------------------
// stats_mode 0: `stats` = [nparts][2][C] partial (sum x, sum x^2) rows written by the conv epilogue,
//               summed here in a FIXED order (deterministic, no atomics) in double precision so
//               that E[x^2] - E[x]^2 does not cancel in fp32;
// stats_mode 1: `stats` = [mean | biased variance] from the two-pass bn_stats_kernel (fp32 mode).
__global__ void bn_finalize_kernel(const float* __restrict__ stats, int nparts, int stats_mode,
                                   float count, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* moving_mean,
                                   float* moving_var, float momentum, float eps, int training,
                                   float* scale, float* shift, float* mean_out, float* rstd_out,
                                   int C) {
  pdl_entry();
  // 8 channels per CTA x 32 lanes over the partial rows: lane l adds rows l, l+32, ... (<= 5 loads,
  // all in flight at once), then the 32 lane sums are added in lane order -- a fixed tree:
  // deterministic.  (A single thread walking all rows would be a chain of L2 latencies.)
  __shared__ double red[2][32][9];
  const int cc = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + cc;
  double s = 0.0, q = 0.0;
  if (training && stats_mode == 0 && c < C) {
#pragma unroll 5
    for (int p = pl; p < nparts; p += 32) {
      s += (double)__ldg(stats + (size_t)p * 2 * C + c);
      q += (double)__ldg(stats + (size_t)p * 2 * C + C + c);
    }
  }
  red[0][pl][cc] = s;
  red[1][pl][cc] = q;
  __syncthreads();
  if (pl != 0 || c >= C) return;
  float mean, var;
  if (training) {
    if (stats_mode == 0) {
      s = q = 0.0;
#pragma unroll
      for (int l = 0; l < 32; ++l) {
        s += red[0][l][cc];
        q += red[1][l][cc];
      }
      const double m = s / (double)count;
      double v = q / (double)count - m * m;
      mean = (float)m;
      var = (float)(v > 0.0 ? v : 0.0);
    } else {
      mean = stats[c];
      var = stats[C + c];
    }
    const float unbiased = var * (count / fmaxf(count - 1.f, 1.f));
    moving_mean[c] = moving_mean[c] * momentum + mean * (1.f - momentum);
    moving_var[c] = moving_var[c] * momentum + unbiased * (1.f - momentum);
  } else {
    mean = moving_mean[c];
    var = moving_var[c];
  }
  const float rstd = rsqrtf(var + eps);
  const float sc = gamma[c] * rstd;
  scale[c] = sc;
  shift[c] = beta[c] - mean * sc;
  mean_out[c] = mean;
  rstd_out[c] = rstd;
}

// Two-pass batch statistics of an [M][C] tensor (fp32 parity mode): one CTA per 8-channel group,
// fixed-order tree reductions -> bit-reproducible; out = [mean | biased variance].
template <class T>
__global__ void __launch_bounds__(256)
bn_stats_kernel(const T* __restrict__ x, float* __restrict__ out, int64_t M, int C) {
  pdl_entry();
  __shared__ float red[256][9];
  __shared__ float mean_s[8];
  const int c0 = blockIdx.x * 8;
  float acc[8];
  for (int pass = 0; pass < 2; ++pass) {
    float mu[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      acc[i] = 0.f;
      mu[i] = pass ? mean_s[i] : 0.f;
    }
    for (int64_t r = threadIdx.x; r < M; r += 256) {
      float v[8];
      load8(x + r * C + c0, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = v[i] - mu[i];
        acc[i] += pass ? d * d : d;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) red[threadIdx.x][i] = acc[i];
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if (threadIdx.x < s) {
#pragma unroll
        for (int i = 0; i < 8; ++i) red[threadIdx.x][i] += red[threadIdx.x + s][i];
      }
      __syncthreads();
    }
    if (threadIdx.x < 8) {
      const float v = red[0][threadIdx.x] / (float)M;
      if (pass == 0) {
        mean_s[threadIdx.x] = v;
        out[c0 + threadIdx.x] = v;
      } else {
        out[C + c0 + threadIdx.x] = v;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// bn_act : out = relu?( (a*sa + ha) [*gate] + R )
// ------------------------------------------------------------------------------------------
// U vectors per thread per trip: the loads of a trip are issued back to back, so U (x2 with a
// second operand) x 16 B x resident threads is what is in flight per SM; ~64 KiB is needed to
// cover the HBM latency at full bandwidth.
template <class T, int U, bool HAS_B>
__global__ void __launch_bounds__(kT, 2)
bn_act_kernel(const T* __restrict__ a, const float* __restrict__ sa,
              const float* __restrict__ ha, const T* __restrict__ b,
              const float* __restrict__ sb, const float* __restrict__ hb, int b_mode,
              const float* __restrict__ gate, int relu, T* __restrict__ out, int H, int W, int C,
              int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  const int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  // CG divides the grid stride (a power of two <= 256 dividing 256*gridDim): the 8-channel group
  // of a thread never changes, so its coefficients are loaded once
  const int cg = (int)(i0 % CG);
  const int c0 = cg << 3;
  float s[8], h[8], s2[8], h2[8];
  loadf8(sa + c0, s);
  loadf8(ha + c0, h);
  if (b_mode == 1) {
    loadf8(sb + c0, s2);
    loadf8(hb + c0, h2);
  }
  // U vectors per trip, loads batched ahead of the math (index clamped, store predicated)
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t ib = i0; ib < nvec; ib += U * stride) {
    V8<T> av[U], bv[HAS_B ? U : 1];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      int64_t i = ib + u * stride;
      i = i < nvec ? i : nvec - 1;
      av[u].ld(a + i * 8);
      if (HAS_B && (b_mode == 1 || b_mode == 2)) {
        bv[u].ld(b + i * 8);
      } else if (HAS_B && b_mode == 3) {
        const int64_t pix = i / CG;
        const int w = (int)(pix % W);
        const int64_t t = pix / W;
        const int hh = (int)(t % H);
        const int64_t bimg = t / H;
        const int64_t src = ((bimg * (H >> 1) + (hh >> 1)) * (W >> 1) + (w >> 1)) * C + c0;
        bv[u].ld(b + src);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = ib + u * stride;
      if (i >= nvec) break;
      float v[8];
      av[u].unpack(v);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = fmaf(v[k], s[k], h[k]);
      if (gate) {
        const int64_t bimg = (i / CG) / ((int64_t)H * W);
        float g[8];
        loadf8(gate + bimg * C + c0, g);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] *= g[k];
      }
      if (HAS_B && b_mode == 1) {
        float r[8];
        bv[u].unpack(r);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] += fmaf(r[k], s2[k], h2[k]);
      } else if (HAS_B && b_mode >= 2) {
        float r[8];
        bv[u].unpack(r);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] += r[k];
      }
      if (relu) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.f);
      }
      store8(out + i * 8, v);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Column (per-channel) reductions over [M][C]
// ------------------------------------------------------------------------------------------
// Every thread owns one 8-channel group `cg` and walks rows; NACC accumulator vectors per thread.
// dest(a, i) gives the index into the partial row of accumulator a, lane-channel i.
// The per-CTA result goes to row `part_row` of a [parts][ncols] partial buffer with PLAIN stores:
// the finalize kernel sums the rows in a fixed order (deterministic; nothing to zero beforehand).
template <int NACC, class Dest>
__device__ __forceinline__ void block_reduce_store(float (&acc)[NACC][8], int CG, float* part_row,
                                                   Dest dest) {
  __shared__ float red[kT][NACC * 8 + 1];
  const int tid = threadIdx.x;
#pragma unroll
  for (int a = 0; a < NACC; ++a)
#pragma unroll
    for (int i = 0; i < 8; ++i) red[tid][a * 8 + i] = acc[a][i];
  __syncthreads();
  const int RPB = kT / CG;
  // spread the final sums over all threads: thread t reduces value (t % (NACC*8)) of group t / ..
  for (int item = tid; item < CG * NACC * 8; item += kT) {
    const int cg = item / (NACC * 8);
    const int k = item % (NACC * 8);
    float s = 0.f;
    for (int r = 0; r < RPB; ++r) s += red[r * CG + cg][k];
    part_row[dest(k >> 3, cg * 8 + (k & 7))] = s;
  }
}

template <class T>
__global__ void __launch_bounds__(kT, 2)
bn_bwd_reduce_kernel(const T* __restrict__ g, const T* __restrict__ y,
                     const float* __restrict__ mean, const float* __restrict__ rstd,
                     const float* __restrict__ gate, const float* __restrict__ addbc,
                     float* sums, int64_t M, int HW, int C) {
  pdl_entry();
  const int CG = C >> 3;
  const int RPB = kT / CG;
  const int cg = threadIdx.x % CG;
  const int rsub = threadIdx.x / CG;
  const int c0 = cg << 3;
  float mu[8], rs[8];
  loadf8(mean + c0, mu);
  loadf8(rstd + c0, rs);
  float acc[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[0][i] = acc[1][i] = 0.f;
  // 4 rows per trip.  The loads are unconditional (row index clamped, contribution zeroed) so
  // that all 8 of them are issued back to back: 8 x 16 B in flight per thread.
  const int64_t step = (int64_t)gridDim.x * RPB;
  for (int64_t r0 = (int64_t)blockIdx.x * RPB + rsub; r0 < M; r0 += 4 * step) {
    V8<T> gq[4], yq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      int64_t r = r0 + u * step;
      r = r < M ? r : M - 1;
      gq[u].ld(g + r * C + c0);
      yq[u].ld(y + r * C + c0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t r = r0 + u * step;
      const float valid = r < M ? 1.f : 0.f;
      float gv[8], yv[8];
      gq[u].unpack(gv);
      yq[u].unpack(yv);
      if (gate || addbc) {
        const int64_t bimg = (r < M ? r : M - 1) / HW;
        if (gate) {
          float t[8];
          loadf8(gate + bimg * C + c0, t);
#pragma unroll
          for (int i = 0; i < 8; ++i) gv[i] *= t[i];
        }
        if (addbc) {
          float t[8];
          loadf8(addbc + bimg * C + c0, t);
#pragma unroll
          for (int i = 0; i < 8; ++i) gv[i] += t[i];
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float gg = gv[i] * valid;
        acc[0][i] += gg;
        acc[1][i] += gg * ((yv[i] - mu[i]) * rs[i]);
      }
    }
  }
  block_reduce_store<2>(acc, CG, sums + (size_t)blockIdx.x * 2 * C,
                        [C](int a, int c) { return a * C + c; });
}

// Two batch norms fed by the SAME gradient g (the block-final BN and the projection-shortcut BN of a
// residual block's first unit: out = relu(bn_a(y_a) + bn_b(y_b))): one pass reads g once and writes
// one partial row per BN (sum g is shared).  Same per-thread summation order as two calls of
// bn_bwd_reduce_kernel, so the results are bit-identical to the separate kernels.
template <class T>
__global__ void __launch_bounds__(kT, 2)
bn_bwd_reduce2_kernel(const T* __restrict__ g, const T* __restrict__ ya, const T* __restrict__ yb,
                      const float* __restrict__ mean_a, const float* __restrict__ rstd_a,
                      const float* __restrict__ mean_b, const float* __restrict__ rstd_b,
                      float* sums_a, float* sums_b, int64_t M, int C) {
  pdl_entry();
  const int CG = C >> 3;
  const int RPB = kT / CG;
  const int cg = threadIdx.x % CG;
  const int rsub = threadIdx.x / CG;
  const int c0 = cg << 3;
  float mua[8], rsa[8], mub[8], rsb[8];
  loadf8(mean_a + c0, mua);
  loadf8(rstd_a + c0, rsa);
  loadf8(mean_b + c0, mub);
  loadf8(rstd_b + c0, rsb);
  float acc_a[2][8], acc_b[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc_a[0][i] = acc_a[1][i] = acc_b[0][i] = acc_b[1][i] = 0.f;
  const int64_t step = (int64_t)gridDim.x * RPB;
  for (int64_t r0 = (int64_t)blockIdx.x * RPB + rsub; r0 < M; r0 += 4 * step) {
    V8<T> gq[4], aq[4], bq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {          // 12 x 16 B in flight per thread (row index clamped)
      int64_t r = r0 + u * step;
      r = r < M ? r : M - 1;
      gq[u].ld(g + r * C + c0);
      aq[u].ld(ya + r * C + c0);
      bq[u].ld(yb + r * C + c0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t r = r0 + u * step;
      const float valid = r < M ? 1.f : 0.f;
      float gv[8], av[8], bv[8];
      gq[u].unpack(gv);
      aq[u].unpack(av);
      bq[u].unpack(bv);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float gg = gv[i] * valid;
        acc_a[0][i] += gg;
        acc_a[1][i] += gg * ((av[i] - mua[i]) * rsa[i]);
        acc_b[1][i] += gg * ((bv[i] - mub[i]) * rsb[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) acc_b[0][i] = acc_a[0][i];
  block_reduce_store<2>(acc_a, CG, sums_a + (size_t)blockIdx.x * 2 * C,
                        [C](int a, int c) { return a * C + c; });
  __syncthreads();                          // the reduction scratch is reused
  block_reduce_store<2>(acc_b, CG, sums_b + (size_t)blockIdx.x * 2 * C,
                        [C](int a, int c) { return a * C + c; });
}

__global__ void bn_bwd_finalize_kernel(const float* __restrict__ sums, int nparts,
                                       const float* __restrict__ gamma,
                                       const float* __restrict__ mean,
                                       const float* __restrict__ rstd, float count, float* coef,
                                       float* dgamma, float* dbeta, int C) {
  pdl_entry();
  // same fixed 32-lane tree over the partial rows as bn_finalize_kernel: deterministic
  __shared__ float red[2][32][9];
  const int cc = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + cc;
  float s1 = 0.f, s2 = 0.f;
  if (c < C) {
#pragma unroll 6
    for (int p = pl; p < nparts; p += 32) {
      s1 += __ldg(sums + (size_t)p * 2 * C + c);
      s2 += __ldg(sums + (size_t)p * 2 * C + C + c);
    }
  }
  red[0][pl][cc] = s1;
  red[1][pl][cc] = s2;
  __syncthreads();
  if (pl != 0 || c >= C) return;
  s1 = s2 = 0.f;
#pragma unroll
  for (int l = 0; l < 32; ++l) {
    s1 += red[0][l][cc];
    s2 += red[1][l][cc];
  }
  const float k1 = gamma[c] * rstd[c];
  const float k2 = -k1 * rstd[c] * s2 / count;
  const float k3 = -k1 * s1 / count - k2 * mean[c];
  coef[c] = k1;
  coef[C + c] = k2;
  coef[2 * C + c] = k3;
  dgamma[c] = s2;
  dbeta[c] = s1;
}

template <class T>
__global__ void __launch_bounds__(kT)
bn_bwd_apply_kernel(const T* __restrict__ g, const T* __restrict__ y,
                    const float* __restrict__ coef, const float* __restrict__ gate,
                    const float* __restrict__ addbc, T* __restrict__ dy, int HW, int C,
                    int64_t nvec) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int CG = C >> 3;
  const int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int cg = (int)(i0 % CG);           // loop-invariant (see bn_act_kernel)
  const int c0 = cg << 3;
  float k1[8], k2[8], k3[8];
  loadf8(coef + c0, k1);
  loadf8(coef + C + c0, k2);
  loadf8(coef + 2 * C + c0, k3);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t ib = i0; ib < nvec; ib += 4 * stride) {
    V8<T> gq[4], yq[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {          // batched loads (index clamped)
      int64_t i = ib + u * stride;
      i = i < nvec ? i : nvec - 1;
      gq[u].ld(g + i * 8);
      yq[u].ld(y + i * 8);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t i = ib + u * stride;
      if (i >= nvec) break;
      float gv[8], yv[8];
      gq[u].unpack(gv);
      yq[u].unpack(yv);
      if (gate || addbc) {
        const int64_t bimg = (i / CG) / HW;
        if (gate) {
          float t[8];
          loadf8(gate + bimg * C + c0, t);
#pragma unroll
          for (int k = 0; k < 8; ++k) gv[k] *= t[k];
        }
        if (addbc) {
          float t[8];
          loadf8(addbc + bimg * C + c0, t);
#pragma unroll
          for (int k = 0; k < 8; ++k) gv[k] += t[k];
        }
      }
      float o[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = fmaf(k1[k], gv[k], fmaf(k2[k], yv[k], k3[k]));
      store8(dy + i * 8, o);
    }
  }
}

// dy_a = k1a*g + k2a*ya + k3a and dy_b = k1b*g + k2b*yb + k3b in one pass (g read once): the two
// batch norms of bn_bwd_reduce2_kernel.
template <class T>
__global__ void __launch_bounds__(kT)
bn_bwd_apply2_kernel(const T* __restrict__ g, const T* __restrict__ ya, const T* __restrict__ yb,
                     const float* __restrict__ coef_a, const float* __restrict__ coef_b,
                     T* __restrict__ dya, T* __restrict__ dyb, int C, int64_t nvec) {
  pdl_wait();   // multi-wave grid (see bn_bwd_apply_kernel)
  const int CG = C >> 3;
  const int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int cg = (int)(i0 % CG);           // loop-invariant (see bn_act_kernel)
  const int c0 = cg << 3;
  float k1a[8], k2a[8], k3a[8], k1b[8], k2b[8], k3b[8];
  loadf8(coef_a + c0, k1a);
  loadf8(coef_a + C + c0, k2a);
  loadf8(coef_a + 2 * C + c0, k3a);
  loadf8(coef_b + c0, k1b);
  loadf8(coef_b + C + c0, k2b);
  loadf8(coef_b + 2 * C + c0, k3b);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t ib = i0; ib < nvec; ib += 2 * stride) {
    V8<T> gq[2], aq[2], bq[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {          // batched loads (index clamped)
      int64_t i = ib + u * stride;
      i = i < nvec ? i : nvec - 1;
      gq[u].ld(g + i * 8);
      aq[u].ld(ya + i * 8);
      bq[u].ld(yb + i * 8);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int64_t i = ib + u * stride;
      if (i >= nvec) break;
      float gv[8], av[8], bv[8], oa[8], ob[8];
      gq[u].unpack(gv);
      aq[u].unpack(av);
      bq[u].unpack(bv);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        oa[k] = fmaf(k1a[k], gv[k], fmaf(k2a[k], av[k], k3a[k]));
        ob[k] = fmaf(k1b[k], gv[k], fmaf(k2b[k], bv[k], k3b[k]));
      }
      store8(dya + i * 8, oa);
      store8(dyb + i * 8, ob);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Per-image spatial reductions  out[b, c] = (1/HW or 1) * sum_hw f(...)
// MODE 0: sk_gap      relu(y0*s+h) + relu(y1*s+h)        (y has 2f channels)       * 1/HW
// MODE 1: sk_bwd_gate dv * (u0 - u1)                                                * 1
// MODE 2: se_gap      y*s+h                                                          * 1/HW
// MODE 3: se_bwd_gate g * (y*s+h)                                                    * 1
// MODE 4: gap         x                                 (bf16 output)                * 1/HW
// ------------------------------------------------------------------------------------------
template <class T, int MODE>
__global__ void __launch_bounds__(kT)
image_reduce_kernel(const T* __restrict__ p0, const T* __restrict__ p1,
                    const float* __restrict__ scale, const float* __restrict__ shift, void* out,
                    int HW, int f) {
  pdl_entry();
  // f = number of OUTPUT channels; MODE 0/1 read y with 2f channels.
  __shared__ float red[kT][9];
  // gridDim.y > 1 splits the channels of an image over several CTAs (each then owns f / gridDim.y of
  // them and its threads share the rows: more loads in flight when f alone would fill the block)
  const int fl = f / (int)gridDim.y;
  const int CG = fl >> 3;
  const int cgs_per_block = CG < kT ? CG : kT;   // CG <= 256 by construction
  const int RPB = kT / cgs_per_block;
  const int cg = threadIdx.x % cgs_per_block;
  const int rsub = threadIdx.x / cgs_per_block;
  const int b = blockIdx.x;
  const int c0 = (int)blockIdx.y * fl + (cg << 3);
  const int ldy = (MODE <= 1) ? 2 * f : f;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  float s0[8], h0[8], s1[8], h1[8];
  if (MODE <= 3) {
    loadf8(scale + c0, s0);
    loadf8(shift + c0, h0);
    if (MODE <= 1) {
      loadf8(scale + f + c0, s1);
      loadf8(shift + f + c0, h1);
    }
  }
  // U rows per trip: all loads of a trip are issued before any math (row clamped, contribution
  // zeroed), since only ~1.7 CTAs of 256 threads are resident per SM (grid = images)
  constexpr int U = (MODE == 1 || MODE == 3) ? 4 : 1;   // measured: batching only pays with 3 loads/row
  for (int rb = rsub; rb < HW; rb += U * RPB) {
    V8<T> qa[U], qb[U], qc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      int r = rb + u * RPB;
      r = r < HW ? r : HW - 1;
      const int64_t row = (int64_t)b * HW + r;
      qa[u].ld(p0 + row * ldy + c0);
      if (MODE <= 1) qb[u].ld(p0 + row * ldy + f + c0);
      if (MODE == 1 || MODE == 3) qc[u].ld(p1 + row * f + c0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float valid = (rb + u * RPB) < HW ? 1.f : 0.f;
      if (MODE == 0 || MODE == 1) {
        float y0[8], y1[8], dv[8];
        qa[u].unpack(y0);
        qb[u].unpack(y1);
        if (MODE == 1) qc[u].unpack(dv);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float u0 = fmaxf(fmaf(y0[i], s0[i], h0[i]), 0.f);
          const float u1 = fmaxf(fmaf(y1[i], s1[i], h1[i]), 0.f);
          acc[i] += valid * ((MODE == 0) ? (u0 + u1) : dv[i] * (u0 - u1));
        }
      } else if (MODE == 2 || MODE == 3) {
        float yv[8], gv[8];
        qa[u].unpack(yv);
        if (MODE == 3) qc[u].unpack(gv);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float t = fmaf(yv[i], s0[i], h0[i]);
          acc[i] += valid * ((MODE == 2) ? t : gv[i] * t);
        }
      } else {
        float xv[8];
        qa[u].unpack(xv);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += valid * xv[i];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[threadIdx.x][i] = acc[i];
  __syncthreads();
  if (rsub == 0) {
    for (int r = 1; r < RPB; ++r)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += red[r * cgs_per_block + cg][i];
    const float norm = (MODE == 0 || MODE == 2 || MODE == 4) ? 1.f / HW : 1.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= norm;
    if (MODE == 4)
      store8(reinterpret_cast<T*>(out) + (int64_t)b * f + c0, acc);
    else
      storef8(reinterpret_cast<float*>(out) + (int64_t)b * f + c0, acc);
  }
}

// ------------------------------------------------------------------------------------------
// SK elementwise
// ------------------------------------------------------------------------------------------
constexpr int kSkStages = 3;
// stage = the rows of y (2f wide) and of dv (f wide) of one trip; sized for bf16 (16 + 8 KiB) and
// doubled for fp32 storage (the parity mode runs one CTA per SM there)
template <class T>
struct SkCfg {
  static constexpr int kYBytes = 8 * 1024 * (int)sizeof(T);
  static constexpr int kDvBytes = 4 * 1024 * (int)sizeof(T);
  static constexpr int kStageBytes = kYBytes + kDvBytes;
  static constexpr int kSmemBytes = kSkStages * kStageBytes + 128;
};

// v = att * relu(bn(y0)) + (1 - att) * relu(bn(y1)).  grid = (row slabs, images): the image and the
// channel group of a thread are fixed, so the BN coefficients and the attention weights live in
// registers; the rows of y are streamed through shared memory (stream_pipe.cuh), 2 rows per thread
// per trip = 16 KiB of y.
template <class T>
__global__ void __launch_bounds__(kT, 2)
sk_combine_kernel(const T* __restrict__ y, const float* __restrict__ scale,
                  const float* __restrict__ shift, const float* __restrict__ att,
                  T* __restrict__ v, int HW, int f) {
  constexpr int kSkStageBytes = SkCfg<T>::kStageBytes;
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  extern __shared__ uint8_t sk_smem_raw[];
  __shared__ uint64_t bars[kSkStages];
  const int CG = f >> 3;
  const int RPB = kT / CG;
  const int RT = 2 * RPB;
  const int cg = threadIdx.x % CG;
  const int rsub = threadIdx.x / CG;
  const int c0 = cg << 3;
  const int64_t b = blockIdx.y;
  const int rows_per = (HW + gridDim.x - 1) / gridDim.x;
  const int r_begin = blockIdx.x * rows_per;
  const int r_end = (r_begin + rows_per < HW) ? r_begin + rows_per : HW;
  const int trips = r_end > r_begin ? (r_end - r_begin + RT - 1) / RT : 0;
  const uint32_t sbase = (smem_u32(sk_smem_raw) + 127u) & ~127u;
  const uint8_t* sgen = sk_smem_raw + (sbase - smem_u32(sk_smem_raw));
  RowPipe<kSkStages> pipe(bars);
  pipe.init(bars);
  auto issue = [&](int t, int stage, uint32_t bar) {
    const int r0 = r_begin + t * RT;
    const int rows = (r_end - r0 < RT) ? r_end - r0 : RT;
    mbar_expect_tx_a(bar, rows * 2 * f * (int)sizeof(T));
    bulk_load(sbase + stage * kSkStageBytes, y + (b * HW + r0) * 2 * f, rows * 2 * f * (int)sizeof(T), bar);
  };
  pipe.prologue(trips, issue);
  float s0[8], h0[8], s1[8], h1[8], a[8];
  loadf8(scale + c0, s0);
  loadf8(shift + c0, h0);
  loadf8(scale + f + c0, s1);
  loadf8(shift + f + c0, h1);
  loadf8(att + b * f + c0, a);
  for (int t = 0; t < trips; ++t) {
    pipe.acquire(t, trips, issue);
    const uint8_t* sy = sgen + pipe.stage(t) * kSkStageBytes;
    const int r0 = r_begin + t * RT;
    const int rows = r_end - r0;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int rl = rsub + u * RPB;
      if (rl < rows) {
        float y0[8], y1[8], o[8];
        lds8<T>(sy, rl * 2 * f + c0, y0);
        lds8<T>(sy, rl * 2 * f + f + c0, y1);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float u0 = fmaxf(fmaf(y0[k], s0[k], h0[k]), 0.f);
          const float u1 = fmaxf(fmaf(y1[k], s1[k], h1[k]), 0.f);
          o[k] = a[k] * u0 + (1.f - a[k]) * u1;
        }
        store8(v + (b * HW + r0 + rl) * f + c0, o);
      }
    }
    pipe.release();
  }
}

// The 2f channels of the SK conv output are handled as one 2f-wide tensor whose gradient is
// computed on the fly: g = (a_h * dv + ds/HW) * [u > 0], a_0 = att, a_1 = 1 - att.  One thread =
// 8 channels of ONE half.  grid = (row slabs, images): everything that depends only on (image,
// channel) stays in registers, and the rows of y / dv are streamed through shared memory
// (stream_pipe.cuh): a trip is 4 rows per thread = 16 KiB of y + 8 KiB of dv for every f.
struct SkSlab {
  int C2, CG2, RPB, RT, cg2, rsub, cb, c0, r_begin, r_end, trips;
  bool second;
  int64_t b;
};
__device__ __forceinline__ SkSlab sk_slab(int HW, int f) {
  SkSlab q;
  q.C2 = 2 * f;
  q.CG2 = q.C2 >> 3;
  q.RPB = kT / q.CG2;
  q.RT = 4 * q.RPB;                              // rows per trip
  q.cg2 = threadIdx.x % q.CG2;
  q.rsub = threadIdx.x / q.CG2;
  q.second = q.cg2 >= (q.CG2 >> 1);
  q.cb = (q.cg2 % (q.CG2 >> 1)) << 3;            // channel inside the half
  q.c0 = q.cg2 << 3;                             // channel inside the 2f-wide tensor
  q.b = blockIdx.y;
  const int rows_per = (HW + gridDim.x - 1) / gridDim.x;
  q.r_begin = blockIdx.x * rows_per;
  q.r_end = (q.r_begin + rows_per < HW) ? q.r_begin + rows_per : HW;
  const int n = q.r_end - q.r_begin;
  q.trips = n > 0 ? (n + q.RT - 1) / q.RT : 0;
  return q;
}

template <class T>
__global__ void __launch_bounds__(kT, 2)
sk_bn_bwd_reduce_kernel(const T* __restrict__ dv, const T* __restrict__ y,
                        const float* __restrict__ scale, const float* __restrict__ shift,
                        const float* __restrict__ mean, const float* __restrict__ rstd,
                        const float* __restrict__ att, const float* __restrict__ ds, float* sums,
                        int HW, int f) {
  pdl_entry();
  constexpr int kSkStageBytes = SkCfg<T>::kStageBytes, kSkYBytes = SkCfg<T>::kYBytes;
  extern __shared__ uint8_t sk_smem_raw[];
  __shared__ uint64_t bars[kSkStages];
  const SkSlab q = sk_slab(HW, f);
  const uint32_t sbase = (smem_u32(sk_smem_raw) + 127u) & ~127u;
  const uint8_t* sgen = sk_smem_raw + (sbase - smem_u32(sk_smem_raw));
  RowPipe<kSkStages> pipe(bars);
  pipe.init(bars);
  auto issue = [&](int t, int stage, uint32_t bar) {
    const int r0 = q.r_begin + t * q.RT;
    const int rows = (q.r_end - r0 < q.RT) ? q.r_end - r0 : q.RT;
    const int64_t row = q.b * HW + r0;
    mbar_expect_tx_a(bar, rows * (q.C2 + f) * (int)sizeof(T));
    bulk_load(sbase + stage * kSkStageBytes, y + row * q.C2, rows * q.C2 * (int)sizeof(T), bar);
    bulk_load(sbase + stage * kSkStageBytes + kSkYBytes, dv + row * f, rows * f * (int)sizeof(T), bar);
  };
  pipe.prologue(q.trips, issue);
  float sc[8], sh[8], mu[8], rs[8], ah[8], sg[8];
  loadf8(scale + q.c0, sc);
  loadf8(shift + q.c0, sh);
  loadf8(mean + q.c0, mu);
  loadf8(rstd + q.c0, rs);
  loadf8(att + q.b * f + q.cb, ah);
  loadf8(ds + q.b * f + q.cb, sg);
  const float inv_hw = 1.f / HW;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (q.second) ah[i] = 1.f - ah[i];
    sg[i] *= inv_hw;
  }
  float acc[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[0][i] = acc[1][i] = 0.f;
  for (int t = 0; t < q.trips; ++t) {
    pipe.acquire(t, q.trips, issue);
    const uint8_t* sy = sgen + pipe.stage(t) * kSkStageBytes;
    const uint8_t* sd = sy + kSkYBytes;
    const int rows = q.r_end - (q.r_begin + t * q.RT);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int rl = q.rsub + u * q.RPB;
      if (rl < rows) {
        float yv[8], d[8];
        lds8<T>(sy, rl * q.C2 + q.c0, yv);
        lds8<T>(sd, rl * f + q.cb, d);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float tt = fmaf(yv[i], sc[i], sh[i]);
          const float gg = tt > 0.f ? fmaf(ah[i], d[i], sg[i]) : 0.f;
          acc[0][i] += gg;
          acc[1][i] += gg * ((yv[i] - mu[i]) * rs[i]);
        }
      }
    }
    pipe.release();
  }
  const int C2 = q.C2;
  block_reduce_store<2>(acc, q.CG2, sums + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 * C2,
                        [C2](int a, int c) { return a * C2 + c; });
}

template <class T>
__global__ void __launch_bounds__(kT, 2)
sk_bn_bwd_apply_kernel(const T* __restrict__ dv, const T* __restrict__ y,
                       const float* __restrict__ scale, const float* __restrict__ shift,
                       const float* __restrict__ att, const float* __restrict__ ds,
                       const float* __restrict__ coef, T* __restrict__ dy, int HW, int f) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  constexpr int kSkStageBytes = SkCfg<T>::kStageBytes, kSkYBytes = SkCfg<T>::kYBytes;
  extern __shared__ uint8_t sk_smem_raw[];
  __shared__ uint64_t bars[kSkStages];
  const SkSlab q = sk_slab(HW, f);
  const uint32_t sbase = (smem_u32(sk_smem_raw) + 127u) & ~127u;
  const uint8_t* sgen = sk_smem_raw + (sbase - smem_u32(sk_smem_raw));
  RowPipe<kSkStages> pipe(bars);
  pipe.init(bars);
  auto issue = [&](int t, int stage, uint32_t bar) {
    const int r0 = q.r_begin + t * q.RT;
    const int rows = (q.r_end - r0 < q.RT) ? q.r_end - r0 : q.RT;
    const int64_t row = q.b * HW + r0;
    mbar_expect_tx_a(bar, rows * (q.C2 + f) * (int)sizeof(T));
    bulk_load(sbase + stage * kSkStageBytes, y + row * q.C2, rows * q.C2 * (int)sizeof(T), bar);
    bulk_load(sbase + stage * kSkStageBytes + kSkYBytes, dv + row * f, rows * f * (int)sizeof(T), bar);
  };
  pipe.prologue(q.trips, issue);
  // o = k1 * g + k2 * y + k3 with g = [sc*y+sh > 0] (ah*dv + sg): folded into
  // o = [..] (ka * dv + kb) + k2 * y + k3
  float sc[8], sh[8], ka[8], kb[8], k2[8], k3[8];
  {
    float k1[8], ah[8], sg[8];
    loadf8(coef + q.c0, k1);
    loadf8(att + q.b * f + q.cb, ah);
    loadf8(ds + q.b * f + q.cb, sg);
    const float inv_hw = 1.f / HW;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a = q.second ? 1.f - ah[i] : ah[i];
      ka[i] = k1[i] * a;
      kb[i] = k1[i] * (sg[i] * inv_hw);
    }
  }
  loadf8(scale + q.c0, sc);
  loadf8(shift + q.c0, sh);
  loadf8(coef + q.C2 + q.c0, k2);
  loadf8(coef + 2 * q.C2 + q.c0, k3);
  for (int t = 0; t < q.trips; ++t) {
    pipe.acquire(t, q.trips, issue);
    const uint8_t* sy = sgen + pipe.stage(t) * kSkStageBytes;
    const uint8_t* sd = sy + kSkYBytes;
    const int r0 = q.r_begin + t * q.RT;
    const int rows = q.r_end - r0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int rl = q.rsub + u * q.RPB;
      if (rl < rows) {
        float yv[8], d[8], o[8];
        lds8<T>(sy, rl * q.C2 + q.c0, yv);
        lds8<T>(sd, rl * f + q.cb, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float tt = fmaf(yv[k], sc[k], sh[k]);
          const float base = fmaf(k2[k], yv[k], k3[k]);
          o[k] = tt > 0.f ? base + fmaf(ka[k], d[k], kb[k]) : base;
        }
        store8(dy + (q.b * HW + r0 + rl) * q.C2 + q.c0, o);
      }
    }
    pipe.release();
  }
}

// Per-image reductions over the SK conv output, one CTA per image, rows streamed through shared
// memory.  MODE 0 (sk_gap): s[b, c] = mean_hw relu(bn(y0)) + relu(bn(y1)); MODE 1 (sk_bwd_gate):
// dA[b, c] = sum_hw dv * (u0 - u1).  One thread = 8 output channels (both halves of y); a trip is
// 2 rows per thread = 16 KiB of y (+ 8 KiB of dv), the same stage layout as the kernels above.
template <class T, int MODE>
__global__ void __launch_bounds__(kT, 2)
sk_image_reduce_kernel(const T* __restrict__ y, const T* __restrict__ dv,
                       const float* __restrict__ scale, const float* __restrict__ shift,
                       float* __restrict__ out, int HW, int f) {
  pdl_entry();
  constexpr int kSkStageBytes = SkCfg<T>::kStageBytes, kSkYBytes = SkCfg<T>::kYBytes;
  extern __shared__ uint8_t sk_smem_raw[];
  __shared__ uint64_t bars[kSkStages];
  __shared__ float red[kT][9];
  const int CG = f >> 3;
  const int RPB = kT / CG;
  const int RT = 2 * RPB;
  const int cg = threadIdx.x % CG;
  const int rsub = threadIdx.x / CG;
  const int c0 = cg << 3;
  const int64_t b = blockIdx.x;
  const int trips = (HW + RT - 1) / RT;
  const uint32_t sbase = (smem_u32(sk_smem_raw) + 127u) & ~127u;
  const uint8_t* sgen = sk_smem_raw + (sbase - smem_u32(sk_smem_raw));
  RowPipe<kSkStages> pipe(bars);
  pipe.init(bars);
  auto issue = [&](int t, int stage, uint32_t bar) {
    const int r0 = t * RT;
    const int rows = (HW - r0 < RT) ? HW - r0 : RT;
    const int64_t row = b * HW + r0;
    mbar_expect_tx_a(bar, rows * (MODE == 1 ? 3 : 2) * f * (int)sizeof(T));
    bulk_load(sbase + stage * kSkStageBytes, y + row * 2 * f, rows * 2 * f * (int)sizeof(T), bar);
    if (MODE == 1)
      bulk_load(sbase + stage * kSkStageBytes + kSkYBytes, dv + row * f, rows * f * (int)sizeof(T), bar);
  };
  pipe.prologue(trips, issue);
  float s0[8], h0[8], s1[8], h1[8], acc[8];
  loadf8(scale + c0, s0);
  loadf8(shift + c0, h0);
  loadf8(scale + f + c0, s1);
  loadf8(shift + f + c0, h1);
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int t = 0; t < trips; ++t) {
    pipe.acquire(t, trips, issue);
    const uint8_t* sy = sgen + pipe.stage(t) * kSkStageBytes;
    const uint8_t* sd = sy + kSkYBytes;
    const int rows = HW - t * RT;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int rl = rsub + u * RPB;
      if (rl < rows) {
        float y0[8], y1[8], d[8];
        lds8<T>(sy, rl * 2 * f + c0, y0);
        lds8<T>(sy, rl * 2 * f + f + c0, y1);
        if (MODE == 1) lds8<T>(sd, rl * f + c0, d);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float u0 = fmaxf(fmaf(y0[i], s0[i], h0[i]), 0.f);
          const float u1 = fmaxf(fmaf(y1[i], s1[i], h1[i]), 0.f);
          acc[i] += (MODE == 0) ? (u0 + u1) : d[i] * (u0 - u1);
        }
      }
    }
    pipe.release();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[threadIdx.x][i] = acc[i];
  __syncthreads();
  if (rsub == 0) {
    for (int r = 1; r < RPB; ++r)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += red[r * CG + cg][i];
    const float norm = (MODE == 0) ? 1.f / HW : 1.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= norm;
    storef8(out + b * f + c0, acc);
  }
}

template <class T, int MODE>
static void launch_sk_image_reduce(const void* y, const void* dv, const float* scale,
                                   const float* shift, float* out, int B, int HW, int f,
                                   cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(sk_image_reduce_kernel<T, MODE>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, SkCfg<T>::kSmemBytes);
    attr = true;
  }
  launch_k(sk_image_reduce_kernel<T, MODE>, dim3(B), dim3(kT), SkCfg<T>::kSmemBytes, st,
           (const T*)y, (const T*)dv, scale, shift, out, HW, f);
}

// Row slabs per image for the image-aligned SK kernels: ~`ctas_per_sm` CTAs per SM overall, at
// least one trip of the unrolled row loop (4 * rpb rows) per CTA.
static int row_slabs(int B, int HW, int rpb, int ctas_per_sm = 8) {
  int s = (kMaxSms * ctas_per_sm + B - 1) / B;
  const int max_s = (HW + 4 * rpb - 1) / (4 * rpb);
  if (s > max_s) s = max_s;
  return s < 1 ? 1 : s;
}

static bool cg_ok(int C) {
  const int cg = C >> 3;
  return C % 8 == 0 && cg >= 1 && cg <= kT && (kT % cg) == 0;
}

static int bn_bwd_reduce_grid(int64_t M, int C) {
  const int rpb = kT / (C >> 3);
  return grid_for(ceil_div64(M, 4 * rpb), 1, kMaxSms * 2);
}

template <class T>
static void set_sk_attr(const void* kern) {
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SkCfg<T>::kSmemBytes);
}

}  // namespace acnn

using namespace acnn;

#define ACNN_DTYPE_OK(dt) ((dt) == ACNN_BF16 || (dt) == ACNN_F32)
#define ACNN_BY_DTYPE(dt, ...)      \
  do {                              \
    if ((dt) == ACNN_F32) {         \
      using T = float;              \
      __VA_ARGS__;                  \
    } else {                        \
      using T = bf16;               \
      __VA_ARGS__;                  \
    }                               \
  } while (0)

template <class T>
static void launch_bn_act(cudaStream_t st, const void* a, const float* scale_a, const float* shift_a,
                          const void* b, const float* scale_b, const float* shift_b, int b_mode,
                          const float* gate, int relu, void* out, int H, int W, int C,
                          int64_t nvec) {
  if (b_mode == 0) {
    launch_k(bn_act_kernel<T, 8, false>, dim3(grid_for(nvec)), dim3(kT), 0, st, (const T*)a, scale_a,
             shift_a, (const T*)b, scale_b, shift_b, b_mode, gate, relu, (T*)out, H, W, C, nvec);
  } else {
    launch_k(bn_act_kernel<T, 4, true>, dim3(grid_for(nvec)), dim3(kT), 0, st, (const T*)a, scale_a,
             shift_a, (const T*)b, scale_b, shift_b, b_mode, gate, relu, (T*)out, H, W, C, nvec);
  }
}

extern "C" {

int acnn_bn_stats(const void* x, float* mean_var, int64_t M, int C, int dtype, void* stream) {
  ACNN_REQUIRE(x && mean_var && M > 0 && C % 8 == 0 && ACNN_DTYPE_OK(dtype),
               "bn_stats: bad arguments");
  ACNN_BY_DTYPE(dtype, launch_k(bn_stats_kernel<T>, dim3(C / 8), dim3(256), 0,
                                (cudaStream_t)stream, (const T*)x, mean_var, M, C));
  count_launch();
  return check_launch("bn_stats");
}

int acnn_bn_finalize(const float* stats, int nparts, int stats_mode, int64_t count,
                     const float* gamma, const float* beta, float* moving_mean, float* moving_var,
                     float momentum, float eps, int training, float* scale, float* shift,
                     float* mean, float* rstd, int C, void* stream) {
  ACNN_REQUIRE(C > 0 && gamma && beta && moving_mean && moving_var && scale && shift && mean &&
                   rstd, "bn_finalize: null argument");
  ACNN_REQUIRE(!training || (stats && count > 0 && (stats_mode == 1 || nparts >= 1)),
               "bn_finalize: training needs statistics");
  launch_k(bn_finalize_kernel, dim3(ceil_div(C, 8)), dim3(256), 0, (cudaStream_t)stream, stats,
           nparts, stats_mode, (float)count, gamma, beta, moving_mean, moving_var, momentum, eps,
           training, scale, shift, mean, rstd, C);
  count_launch();
  return check_launch("bn_finalize");
}

int acnn_bn_act(const void* a, const float* scale_a, const float* shift_a, const void* b,
                const float* scale_b, const float* shift_b, int b_mode, const float* gate, int relu,
                void* out, int B, int H, int W, int C, int dtype, void* stream) {
  ACNN_REQUIRE(a && scale_a && shift_a && out && C % 8 == 0 && ACNN_DTYPE_OK(dtype),
               "bn_act: bad arguments (C=%d)", C);
  ACNN_REQUIRE(b_mode >= 0 && b_mode <= 3 && (b_mode == 0 || b), "bn_act: bad b_mode %d", b_mode);
  ACNN_REQUIRE(b_mode != 1 || (scale_b && shift_b), "bn_act: b_mode 1 needs scale_b/shift_b");
  ACNN_REQUIRE(b_mode != 3 || (H % 2 == 0 && W % 2 == 0), "bn_act: upsample needs even H, W");
  // the channel group of a thread must be loop-invariant: C/8 divides the grid stride
  ACNN_REQUIRE(cg_ok(C), "bn_act: C=%d (C/8 must divide 256)", C);
  const int64_t nvec = (int64_t)B * H * W * C / 8;
  ACNN_BY_DTYPE(dtype, launch_bn_act<T>((cudaStream_t)stream, a, scale_a, shift_a, b, scale_b,
                                        shift_b, b_mode, gate, relu, out, H, W, C, nvec));
  count_launch();
  return check_launch("bn_act");
}

int acnn_bn_bwd_reduce_parts(int B, int HW, int C) {
  if (!cg_ok(C) || B <= 0 || HW <= 0) return 0;
  return bn_bwd_reduce_grid((int64_t)B * HW, C);
}

int acnn_bn_bwd_reduce(const void* g, const void* y, const float* mean, const float* rstd,
                       const float* gate, const float* addbc, float* parts, int B, int HW, int C,
                       int dtype, void* stream) {
  ACNN_REQUIRE(g && y && mean && rstd && parts && cg_ok(C) && ACNN_DTYPE_OK(dtype),
               "bn_bwd_reduce: bad arguments C=%d", C);
  const int64_t M = (int64_t)B * HW;
  ACNN_BY_DTYPE(dtype, launch_k(bn_bwd_reduce_kernel<T>, dim3(bn_bwd_reduce_grid(M, C)), dim3(kT), 0,
                                (cudaStream_t)stream, (const T*)g, (const T*)y, mean, rstd, gate,
                                addbc, parts, M, HW, C));
  count_launch();
  return check_launch("bn_bwd_reduce");
}

int acnn_bn_bwd_reduce2(const void* g, const void* ya, const void* yb, const float* mean_a,
                        const float* rstd_a, const float* mean_b, const float* rstd_b, float* parts_a,
                        float* parts_b, int B, int HW, int C, int dtype, void* stream) {
  ACNN_REQUIRE(g && ya && yb && mean_a && rstd_a && mean_b && rstd_b && parts_a && parts_b &&
                   cg_ok(C) && ACNN_DTYPE_OK(dtype), "bn_bwd_reduce2: bad arguments C=%d", C);
  const int64_t M = (int64_t)B * HW;
  ACNN_BY_DTYPE(dtype, launch_k(bn_bwd_reduce2_kernel<T>, dim3(bn_bwd_reduce_grid(M, C)), dim3(kT), 0,
                                (cudaStream_t)stream, (const T*)g, (const T*)ya, (const T*)yb, mean_a,
                                rstd_a, mean_b, rstd_b, parts_a, parts_b, M, C));
  count_launch();
  return check_launch("bn_bwd_reduce2");
}

int acnn_bn_bwd_apply2(const void* g, const void* ya, const void* yb, const float* coef_a,
                       const float* coef_b, void* dya, void* dyb, int B, int HW, int C, int dtype,
                       void* stream) {
  ACNN_REQUIRE(g && ya && yb && coef_a && coef_b && dya && dyb && cg_ok(C) && ACNN_DTYPE_OK(dtype),
               "bn_bwd_apply2: bad arguments");
  const int64_t nvec = (int64_t)B * HW * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(bn_bwd_apply2_kernel<T>, dim3(grid_for(nvec)), dim3(kT), 0,
                                (cudaStream_t)stream, (const T*)g, (const T*)ya, (const T*)yb, coef_a,
                                coef_b, (T*)dya, (T*)dyb, C, nvec));
  count_launch();
  return check_launch("bn_bwd_apply2");
}

int acnn_bn_bwd_finalize(const float* parts, int nparts, const float* gamma, const float* mean,
                         const float* rstd, int64_t count, float* coef, float* dgamma, float* dbeta,
                         int C, void* stream) {
  ACNN_REQUIRE(parts && nparts >= 1 && gamma && mean && rstd && coef && dgamma && dbeta && count > 0,
               "bn_bwd_finalize: bad argument");
  launch_k(bn_bwd_finalize_kernel, dim3(ceil_div(C, 8)), dim3(256), 0, (cudaStream_t)stream, parts,
           nparts, gamma, mean, rstd, (float)count, coef, dgamma, dbeta, C);
  count_launch();
  return check_launch("bn_bwd_finalize");
}

int acnn_bn_bwd_apply(const void* g, const void* y, const float* coef, const float* gate,
                      const float* addbc, void* dy, int B, int HW, int C, int dtype, void* stream) {
  ACNN_REQUIRE(g && y && coef && dy && cg_ok(C) && ACNN_DTYPE_OK(dtype),
               "bn_bwd_apply: bad arguments");
  const int64_t nvec = (int64_t)B * HW * C / 8;
  ACNN_BY_DTYPE(dtype, launch_k(bn_bwd_apply_kernel<T>, dim3(grid_for(nvec)), dim3(kT), 0,
                                (cudaStream_t)stream, (const T*)g, (const T*)y, coef, gate, addbc,
                                (T*)dy, HW, C, nvec));
  count_launch();
  return check_launch("bn_bwd_apply");
}

int acnn_sk_gap(const void* y, const float* scale, const float* shift, float* s, int B, int HW,
                int f, int dtype, void* stream) {
  ACNN_REQUIRE(y && scale && shift && s && cg_ok(f) && ACNN_DTYPE_OK(dtype),
               "sk_gap: bad arguments f=%d", f);
  ACNN_BY_DTYPE(dtype, (launch_sk_image_reduce<T, 0>(y, nullptr, scale, shift, s, B, HW, f,
                                                     (cudaStream_t)stream)));
  count_launch();
  return check_launch("sk_gap");
}

int acnn_sk_bwd_gate(const void* dv, const void* y, const float* scale, const float* shift,
                     float* dA, int B, int HW, int f, int dtype, void* stream) {
  ACNN_REQUIRE(dv && y && scale && shift && dA && cg_ok(f) && ACNN_DTYPE_OK(dtype),
               "sk_bwd_gate: bad arguments");
  ACNN_BY_DTYPE(dtype, (launch_sk_image_reduce<T, 1>(y, dv, scale, shift, dA, B, HW, f,
                                                     (cudaStream_t)stream)));
  count_launch();
  return check_launch("sk_bwd_gate");
}

int acnn_se_gap(const void* y, const float* scale, const float* shift, float* q, int B, int HW,
                int C, int dtype, void* stream) {
  ACNN_REQUIRE(y && scale && shift && q && cg_ok(C) && ACNN_DTYPE_OK(dtype), "se_gap: bad arguments");
  ACNN_BY_DTYPE(dtype, (launch_k(image_reduce_kernel<T, 2>, dim3(B), dim3(kT), 0,
                                 (cudaStream_t)stream, (const T*)y, (const T*)nullptr, scale, shift,
                                 (void*)q, HW, C)));
  count_launch();
  return check_launch("se_gap");
}

int acnn_se_bwd_gate(const void* g, const void* y, const float* scale, const float* shift,
                     float* de, int B, int HW, int C, int dtype, void* stream) {
  ACNN_REQUIRE(g && y && scale && shift && de && cg_ok(C) && ACNN_DTYPE_OK(dtype),
               "se_bwd_gate: bad arguments");
  ACNN_BY_DTYPE(dtype, (launch_k(image_reduce_kernel<T, 3>, dim3(B), dim3(kT), 0,
                                 (cudaStream_t)stream, (const T*)y, (const T*)g, scale, shift,
                                 (void*)de, HW, C)));
  count_launch();
  return check_launch("se_bwd_gate");
}

int acnn_gap_fwd(const void* x, void* pooled, int B, int HW, int C, int dtype, void* stream) {
  ACNN_REQUIRE(x && pooled && cg_ok(C) && ACNN_DTYPE_OK(dtype), "gap_fwd: bad arguments C=%d", C);
  // C = 2048 would give every thread its own channel group and all HW rows (one 16-byte load in flight
  // per thread: too few bytes in flight to fill HBM); 512 channels per CTA let four threads share the
  // rows of a group
  const int csplit = (C >= 1024 && C % 512 == 0) ? C / 512 : 1;
  ACNN_BY_DTYPE(dtype, (launch_k(image_reduce_kernel<T, 4>, dim3(B, csplit), dim3(kT), 0,
                                 (cudaStream_t)stream, (const T*)x, (const T*)nullptr,
                                 (const float*)nullptr, (const float*)nullptr, pooled, HW, C)));
  count_launch();
  return check_launch("gap_fwd");
}

int acnn_sk_combine(const void* y, const float* scale, const float* shift, const float* att,
                    void* v, int B, int HW, int f, int dtype, void* stream) {
  ACNN_REQUIRE(y && scale && shift && att && v && cg_ok(f) && B <= 65535 && ACNN_DTYPE_OK(dtype),
               "sk_combine: bad arguments");
  dim3 grid(row_slabs(B, HW, kT / (f >> 3)), B);
  ACNN_BY_DTYPE(dtype, {
    static bool attr = false;
    if (!attr) {
      set_sk_attr<T>((const void*)sk_combine_kernel<T>);
      attr = true;
    }
    launch_k(sk_combine_kernel<T>, grid, dim3(kT), SkCfg<T>::kSmemBytes, (cudaStream_t)stream,
             (const T*)y, scale, shift, att, (T*)v, HW, f);
  });
  count_launch();
  return check_launch("sk_combine");
}

int acnn_sk_bn_bwd_reduce_parts(int B, int HW, int f) {
  if (!cg_ok(2 * f) || B <= 0 || HW <= 0) return 0;
  return row_slabs(B, HW, kT / (f >> 2), 2) * B;
}

int acnn_sk_bn_bwd_reduce(const void* dv, const void* y, const float* scale, const float* shift,
                          const float* mean, const float* rstd, const float* att, const float* ds,
                          float* parts, int B, int HW, int f, int dtype, void* stream) {
  ACNN_REQUIRE(dv && y && scale && shift && mean && rstd && att && ds && parts && cg_ok(2 * f) &&
                   B <= 65535 && ACNN_DTYPE_OK(dtype), "sk_bn_bwd_reduce: bad arguments");
  // one resident wave of long-lived CTAs; every CTA writes one partial row (2 x 2f floats)
  dim3 grid(row_slabs(B, HW, kT / (f >> 2), 2), B);
  ACNN_BY_DTYPE(dtype, {
    static bool attr = false;
    if (!attr) {
      set_sk_attr<T>((const void*)sk_bn_bwd_reduce_kernel<T>);
      attr = true;
    }
    launch_k(sk_bn_bwd_reduce_kernel<T>, grid, dim3(kT), SkCfg<T>::kSmemBytes, (cudaStream_t)stream,
             (const T*)dv, (const T*)y, scale, shift, mean, rstd, att, ds, parts, HW, f);
  });
  count_launch();
  return check_launch("sk_bn_bwd_reduce");
}

int acnn_sk_bn_bwd_apply(const void* dv, const void* y, const float* scale, const float* shift,
                         const float* att, const float* ds, const float* coef, void* dy, int B,
                         int HW, int f, int dtype, void* stream) {
  ACNN_REQUIRE(dv && y && scale && shift && att && ds && coef && dy && cg_ok(2 * f) && B <= 65535 &&
                   ACNN_DTYPE_OK(dtype), "sk_bn_bwd_apply: bad arguments");
  dim3 grid(row_slabs(B, HW, kT / (f >> 2)), B);
  ACNN_BY_DTYPE(dtype, {
    static bool attr = false;
    if (!attr) {
      set_sk_attr<T>((const void*)sk_bn_bwd_apply_kernel<T>);
      attr = true;
    }
    launch_k(sk_bn_bwd_apply_kernel<T>, grid, dim3(kT), SkCfg<T>::kSmemBytes, (cudaStream_t)stream,
             (const T*)dv, (const T*)y, scale, shift, att, ds, coef, (T*)dy, HW, f);
  });
  count_launch();
  return check_launch("sk_bn_bwd_apply");
}

}  // extern "C"
