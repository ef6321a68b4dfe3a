// The tiny fully-connected layers of the SK / SE attention paths (<= 0.3 MMAC per image):
// fp32 CUDA-core GEMMs on [B, <=2048] descriptors.  nets/blocks.py:136-151 (SK), :171-182 (SE).
//
// One shared-memory-tiled SGEMM (64x64x16 tile, 4x4 micro-tile per thread, split-K with partials
// summed in split order) serves all of them through generic element strides; the batch-norm-over-batch, gate and
// activation glue are separate one-warp-per-channel / elementwise kernels.
#include "common.h"
#include "vec.cuh"

#include <cooperative_groups.h>

namespace acnn {

static int num_sms_small() {
  static int n = 0;
  if (n == 0) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) {
      (void)cudaGetLastError();
      return 132;        // no device (host-only sizing queries): the H100 SXM's SM count
    }
    n = v;
  }
  return n;
}

constexpr int kFT = 256;
constexpr int kTM = 64, kTN = 64, kTK = 16;

// C[M][N] (row-major, ldc = N) += sum_k A(m,k) * B(k,n)
//   A(m,k) = A[m*sAm + k*sAk],  B(k,n) = B[k*sBk + n*sBn]
// gridDim = (ceil(N/64), ceil(M/64), splits).  part == nullptr (one split): the CTA adds its tile
// to C; else split z stores its partial tile at part + z*M*N and sgemm_reduce_kernel adds them.
__global__ void __launch_bounds__(kFT)
sgemm_acc_kernel(const float* __restrict__ A, const float* __restrict__ B, float* C, int M, int N,
                 int K, int sAm, int sAk, int sBk, int sBn, int k_per_split, float* part) {
  pdl_entry();
  __shared__ float As[kTK][kTM + 4];
  __shared__ float Bs[kTK][kTN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;          // 16 x 16 threads, 4x4 outputs each
  const int m0 = blockIdx.y * kTM, n0 = blockIdx.x * kTN;
  const int k_begin = blockIdx.z * k_per_split;
  int k_end = k_begin + k_per_split;
  if (k_end > K) k_end = K;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = k_begin; k0 < k_end; k0 += kTK) {
    // coalesce along whichever index is unit-stride in global memory
#pragma unroll
    for (int e = 0; e < (kTM * kTK) / kFT; ++e) {
      const int idx = tid + e * kFT;
      int mm, kk;
      if (sAm == 1) { mm = idx % kTM; kk = idx / kTM; } else { kk = idx % kTK; mm = idx / kTK; }
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < M && k < k_end) ? __ldg(A + (size_t)m * sAm + (size_t)k * sAk) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < (kTN * kTK) / kFT; ++e) {
      const int idx = tid + e * kFT;
      int nn, kk;
      if (sBn == 1) { nn = idx % kTN; kk = idx / kTN; } else { kk = idx % kTK; nn = idx / kTK; }
      const int n = n0 + nn, k = k0 + kk;
      Bs[kk][nn] = (n < N && k < k_end) ? __ldg(B + (size_t)k * sBk + (size_t)n * sBn) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kTK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      if (part) part[((size_t)blockIdx.z * M + m) * N + n] = acc[i][j];
      else C[(size_t)m * N + n] += acc[i][j];
    }
  }
}

// C[i] += sum over splits s (in order) of part[s][i]
__global__ void __launch_bounds__(kFT)
sgemm_reduce_kernel(const float* __restrict__ part, float* C, int64_t n, int splits) {
  pdl_entry();
  for (int64_t i = blockIdx.x * (int64_t)kFT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kFT) {
    float t = 0.f;
    for (int s = 0; s < splits; ++s) t += part[s * n + i];
    C[i] += t;
  }
}

// C (+)= A*B with split-K sized so that ~2 CTAs per SM are in flight; the partials of a split-K
// product are summed in split order (bit-reproducible).  det: no split-K -- every element of C
// receives exactly one add.
static int sgemm(const float* A, const float* B, float* C, int M, int N, int K, int sAm, int sAk,
                 int sBk, int sBn, bool zero_c, int det, cudaStream_t s) {
  if (zero_c) {
    cudaError_t e = cudaMemsetAsync(C, 0, (size_t)M * N * sizeof(float), s);
    if (e != cudaSuccess) {
      set_error("sgemm memset: %s", cudaGetErrorString(e));
      return ACNN_ERR_CUDA;
    }
  }
  const int tiles = ceil_div(M, kTM) * ceil_div(N, kTN);
  int splits = ceil_div(2 * num_sms_small(), tiles);
  const int max_splits = ceil_div(K, 2 * kTK);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1 || det) splits = 1;
  int kps = ceil_div(ceil_div(K, splits), kTK) * kTK;
  splits = ceil_div(K, kps);
  dim3 grid(ceil_div(N, kTN), ceil_div(M, kTM), splits);
  if (splits == 1) {
    launch_k(sgemm_acc_kernel, dim3(grid), dim3(kFT), 0, s, A, B, C, M, N, K, sAm, sAk, sBk, sBn, kps,
             (float*)nullptr);
    count_launch();
    return check_launch("sgemm_acc");
  }
  // split-K partials in a stream-ordered scratch, then one ordered reduction into C
  void* part = nullptr;
  const int64_t n = (int64_t)M * N;
  int rc = scratch_alloc(&part, (size_t)splits * n * sizeof(float), s, "sgemm");
  if (rc) return rc;
  launch_k(sgemm_acc_kernel, dim3(grid), dim3(kFT), 0, s, A, B, C, M, N, K, sAm, sAk, sBk, sBn, kps,
           static_cast<float*>(part));
  count_launch();
  rc = check_launch("sgemm_acc");
  if (rc == ACNN_OK) {
    launch_k(sgemm_reduce_kernel, dim3(grid_for(n, kFT, 2 * num_sms_small())), dim3(kFT), 0, s,
             static_cast<const float*>(part), C, n, splits);
    count_launch();
    rc = check_launch("sgemm_reduce");
  }
  const int rc2 = scratch_free(part, s, "sgemm");
  return rc ? rc : rc2;
}

// One warp per channel j: batch-norm over the batch dimension, then ReLU.
__global__ void __launch_bounds__(kFT)
bn_batch_relu_fwd_kernel(const float* __restrict__ zpre, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float* moving_mean, float* moving_var,
                         float momentum, float eps, int training, float* __restrict__ z,
                         float* __restrict__ bnstat, int B, int d) {
  pdl_entry();
  const int j = blockIdx.x * (kFT / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= d) return;
  float mean, var;
  if (training) {
    // two-pass (mean, then centred squares): with only B samples per channel and eps = 1e-5,
    // E[x^2] - E[x]^2 in fp32 loses the variance of nearly constant channels
    float s = 0.f, q = 0.f;
    for (int b = lane; b < B; b += 32) s += zpre[(size_t)b * d + j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    mean = s / B;
    for (int b = lane; b < B; b += 32) {
      const float c = zpre[(size_t)b * d + j] - mean;
      q += c * c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    var = q / B;
    if (lane == 0) {
      const float unbiased = var * ((float)B / fmaxf((float)B - 1.f, 1.f));
      moving_mean[j] = moving_mean[j] * momentum + mean * (1.f - momentum);
      moving_var[j] = moving_var[j] * momentum + unbiased * (1.f - momentum);
    }
  } else {
    mean = moving_mean[j];
    var = moving_var[j];
  }
  const float rstd = rsqrtf(var + eps);
  if (lane == 0) {
    bnstat[j] = mean;
    bnstat[d + j] = rstd;
  }
  const float sc = gamma[j] * rstd, sh = beta[j] - mean * sc;
  for (int b = lane; b < B; b += 32)
    z[(size_t)b * d + j] = fmaxf(fmaf(zpre[(size_t)b * d + j], sc, sh), 0.f);
}

// dz (in: grad wrt z; out: grad wrt zpre), one warp per channel.
__global__ void __launch_bounds__(kFT)
bn_batch_relu_bwd_kernel(float* dz, const float* __restrict__ z, const float* __restrict__ zpre,
                         const float* __restrict__ bnstat, const float* __restrict__ gamma,
                         float* dgamma, float* dbeta, int B, int d) {
  pdl_entry();
  const int j = blockIdx.x * (kFT / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= d) return;
  const float mean = bnstat[j], rstd = bnstat[d + j];
  float s1 = 0.f, s2 = 0.f;
  for (int b = lane; b < B; b += 32) {
    const size_t i = (size_t)b * d + j;
    const float g = z[i] > 0.f ? dz[i] : 0.f;
    s1 += g;
    s2 += g * ((zpre[i] - mean) * rstd);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  const float k1 = gamma[j] * rstd;
  for (int b = lane; b < B; b += 32) {
    const size_t i = (size_t)b * d + j;
    const float g = z[i] > 0.f ? dz[i] : 0.f;
    const float xh = (zpre[i] - mean) * rstd;
    dz[i] = k1 * (g - s1 / B - xh * s2 / B);
  }
  if (lane == 0) {
    dgamma[j] += s2;
    dbeta[j] += s1;
  }
}

__global__ void sk_gate_fwd_kernel(const float* __restrict__ a, float* __restrict__ att, int B,
                                   int f) {
  pdl_entry();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * f) return;
  const int b = (int)(i / f), c = (int)(i - (int64_t)b * f);
  const float d = a[(size_t)b * 2 * f + c] - a[(size_t)b * 2 * f + f + c];
  att[i] = 1.f / (1.f + expf(-d));
}

__global__ void sk_gate_bwd_kernel(const float* __restrict__ dA, const float* __restrict__ att,
                                   float* __restrict__ da, int B, int f) {
  pdl_entry();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * f) return;
  const int b = (int)(i / f), c = (int)(i - (int64_t)b * f);
  const float t = att[i] * (1.f - att[i]) * dA[i];
  da[(size_t)b * 2 * f + c] = t;
  da[(size_t)b * 2 * f + f + c] = -t;
}

// mode 1: out = relu(in) ; 2: out = sigmoid(in) ; 3: out = in*(act>0) ; 4: out = in*act*(1-act) ;
// 5: out = in*scale
__global__ void ew_kernel(const float* in, const float* act, float* out, int64_t n, int mode,
                          float scale) {
  pdl_entry();
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = in[i];
  float o;
  if (mode == 1) o = fmaxf(v, 0.f);
  else if (mode == 2) o = 1.f / (1.f + expf(-v));
  else if (mode == 3) o = act[i] > 0.f ? v : 0.f;
  else if (mode == 4) o = v * act[i] * (1.f - act[i]);
  else o = v * scale;
  out[i] = o;
}

static int ew(const float* in, const float* act, float* out, int64_t n, int mode, float scale,
              cudaStream_t s) {
  launch_k(ew_kernel, dim3((int)ceil_div64(n, 256)), dim3(256), 0, s, in, act, out, n, mode, scale);
  count_launch();
  return check_launch("ew");
}

// ------------------------------------------------------------------------------------------
// Fused SK attention chains: ONE cooperative launch per direction instead of 4 kernels + 2 memsets
// (forward) / 6 kernels + 2 memsets (backward) per SK block -- 19 blocks per Assemble-ResNet-50
// step, i.e. 266 of the step's ~1000 graph nodes, every one of them a few microseconds of launch
// latency around almost no work.  The whole grid (<= kMaxSms CTAs, all resident: cooperative launch)
// walks the phases of the chain separated by grid barriers:
//   * a GEMM phase deals (64x64 output tile, K split) units round-robin to the CTAs; every unit
//     writes its partial tile to scratch (plain stores, one owner per element),
//   * the consumer phase sums the partials in split order -- deterministic, nothing to zero, no
//     atomics -- fused with whatever follows (batch-norm over the batch + ReLU, the 2-way softmax
//     gate, the += into the gradient buffer).
// (One 8-CTA cluster without K splits would be too small: the phases need the whole GPU.)
// ------------------------------------------------------------------------------------------
constexpr int kGridMax = kMaxSms;  // scratch is sized for this many CTAs (plan.py mirrors it)
constexpr int kMaxSplits = 8;

struct GJob {
  const float* A;
  const float* B;
  float* P;                 // partials [splits][M][N]
  int M, N, K, sAm, sAk, sBk, sBn;
  int splits, kper, tn, units;
};

// K splits of one GEMM job when `share` CTAs are available to it: enough units to occupy them, at
// least 32 k-elements (two k-steps) per unit
static int job_splits(int M, int N, int K, int share) {
  const int tiles = ceil_div(M, kTM) * ceil_div(N, kTN);
  int s = share / tiles;
  if (s > K / 32) s = K / 32;
  if (s > kMaxSplits) s = kMaxSplits;
  return s < 1 ? 1 : s;
}

static GJob make_job(const float* A, const float* B, float* P, int M, int N, int K, int sAm, int sAk,
                     int sBk, int sBn, int share) {
  GJob j{A, B, P, M, N, K, sAm, sAk, sBk, sBn, 0, 0, 0, 0};
  j.splits = job_splits(M, N, K, share);
  j.kper = ceil_div(ceil_div(K, j.splits), kTK) * kTK;
  j.splits = ceil_div(K, j.kper);
  j.tn = ceil_div(N, kTN);
  j.units = ceil_div(M, kTM) * j.tn * j.splits;
  return j;
}
static int64_t job_floats(const GJob& j) { return (int64_t)j.splits * j.M * j.N; }

// one (tile, split) unit: P[split][m0.., n0..] = A[m0.., k range] * B[k range, n0..]; the operands of
// the next k-step are fetched into registers while the current one is multiplied.  Intermediates
// written by other CTAs in an earlier phase are read with ld.global.cg (L2: the L1 is not coherent).
__device__ __forceinline__ void gemm_unit(const GJob& j, int u, float (*As)[kTM + 4],
                                          float (*Bs)[kTN + 4]) {
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int split = u % j.splits, t = u / j.splits;
  const int m0 = (t / j.tn) * kTM, n0 = (t % j.tn) * kTN;
  const int kb = split * j.kper;
  const int ke = kb + j.kper < j.K ? kb + j.kper : j.K;
  constexpr int kEA = (kTM * kTK) / kFT, kEB = (kTN * kTK) / kFT;
  int amm[kEA], akk[kEA], bnn[kEB], bkk[kEB];
#pragma unroll
  for (int e = 0; e < kEA; ++e) {
    const int idx = tid + e * kFT;
    if (j.sAm == 1) { amm[e] = idx % kTM; akk[e] = idx / kTM; } else { akk[e] = idx % kTK; amm[e] = idx / kTK; }
  }
#pragma unroll
  for (int e = 0; e < kEB; ++e) {
    const int idx = tid + e * kFT;
    if (j.sBn == 1) { bnn[e] = idx % kTN; bkk[e] = idx / kTN; } else { bkk[e] = idx % kTK; bnn[e] = idx / kTK; }
  }
  float ra[kEA], rb[kEB];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < kEA; ++e) {
      const int m = m0 + amm[e], k = k0 + akk[e];
      ra[e] = (m < j.M && k < ke) ? __ldcg(j.A + (size_t)m * j.sAm + (size_t)k * j.sAk) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < kEB; ++e) {
      const int n = n0 + bnn[e], k = k0 + bkk[e];
      rb[e] = (n < j.N && k < ke) ? __ldcg(j.B + (size_t)k * j.sBk + (size_t)n * j.sBn) : 0.f;
    }
  };
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[i][q] = 0.f;
  fetch(kb);
  for (int k0 = kb; k0 < ke; k0 += kTK) {
#pragma unroll
    for (int e = 0; e < kEA; ++e) As[akk[e]][amm[e]] = ra[e];
#pragma unroll
    for (int e = 0; e < kEB; ++e) Bs[bkk[e]][bnn[e]] = rb[e];
    __syncthreads();
    if (k0 + kTK < ke) fetch(k0 + kTK);
#pragma unroll
    for (int kk = 0; kk < kTK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int q = 0; q < 4; ++q) b[q] = Bs[kk][tx * 4 + q];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][q] = fmaf(a[i], b[q], acc[i][q]);
    }
    __syncthreads();
  }
  float* C = j.P + (size_t)split * j.M * j.N;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= j.M) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = n0 + tx * 4 + q;
      if (n < j.N) C[(size_t)m * j.N + n] = acc[i][q];
    }
  }
}

// the units of up to two jobs, dealt round-robin over the grid (job 1's units follow job 0's)
__device__ __forceinline__ void run_jobs(const GJob& j0, const GJob* j1, float (*As)[kTM + 4],
                                         float (*Bs)[kTN + 4]) {
  const int total = j0.units + (j1 ? j1->units : 0);
  for (int u = blockIdx.x; u < total; u += gridDim.x) {
    if (u < j0.units) gemm_unit(j0, u, As, Bs);
    else gemm_unit(*j1, u - j0.units, As, Bs);
  }
}

// sum over the splits of element i of a job's partials, in split order
__device__ __forceinline__ float partial_sum(const GJob& j, size_t i) {
  const size_t mn = (size_t)j.M * j.N;
  float v = __ldcg(j.P + i);
  for (int s = 1; s < j.splits; ++s) v += __ldcg(j.P + s * mn + i);
  return v;
}

__device__ __forceinline__ void grid_barrier() {
  asm volatile("" ::: "memory");
  cooperative_groups::this_grid().sync();
}

struct SkFcFwdArgs {
  GJob fc1, fc2;
  const float *gamma, *beta;
  float *moving_mean, *moving_var, *zpre, *bnstat, *z, *att;
  float momentum, eps;
  int training, B, f, d;
};

__global__ void __launch_bounds__(kFT)
sk_fc_fwd_fused_kernel(const SkFcFwdArgs p) {
  __shared__ float As[kTK][kTM + 4];
  __shared__ float Bs[kTK][kTN + 4];
  const int B = p.B, f = p.f, d = p.d;
  const int lane = threadIdx.x & 31;
  // zpre[B,d] = s[B,f] * W1[d,f]^T  (partials)
  run_jobs(p.fc1, nullptr, As, Bs);
  grid_barrier();
  // batch-norm over the batch (two-pass variance) + ReLU, one warp per channel
  for (int j = blockIdx.x * (kFT / 32) + (threadIdx.x >> 5); j < d; j += gridDim.x * (kFT / 32)) {
    float sm = 0.f;
    for (int b = lane; b < B; b += 32) {
      const float v = partial_sum(p.fc1, (size_t)b * d + j);
      p.zpre[(size_t)b * d + j] = v;
      sm += v;
    }
    float mean, var;
    if (p.training) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
      mean = sm / B;
      float q = 0.f;
      for (int b = lane; b < B; b += 32) {
        const float c = p.zpre[(size_t)b * d + j] - mean;      // this lane's own stores
        q += c * c;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      var = q / B;
      if (lane == 0) {
        const float unbiased = var * ((float)B / fmaxf((float)B - 1.f, 1.f));
        p.moving_mean[j] = p.moving_mean[j] * p.momentum + mean * (1.f - p.momentum);
        p.moving_var[j] = p.moving_var[j] * p.momentum + unbiased * (1.f - p.momentum);
      }
    } else {
      mean = p.moving_mean[j];
      var = p.moving_var[j];
    }
    const float rstd = rsqrtf(var + p.eps);
    if (lane == 0) {
      p.bnstat[j] = mean;
      p.bnstat[d + j] = rstd;
    }
    const float sc = p.gamma[j] * rstd, sh = p.beta[j] - mean * sc;
    for (int b = lane; b < B; b += 32)
      p.z[(size_t)b * d + j] = fmaxf(fmaf(p.zpre[(size_t)b * d + j], sc, sh), 0.f);
  }
  grid_barrier();
  // a[B,2f] = z[B,d] * W2[2f,d]^T  (partials)
  run_jobs(p.fc2, nullptr, As, Bs);
  grid_barrier();
  // 2-way softmax over the halves: att = sigmoid(a0 - a1)
  for (int i = blockIdx.x * kFT + threadIdx.x; i < B * f; i += gridDim.x * kFT) {
    const int b = i / f, c = i - b * f;
    const float dd = partial_sum(p.fc2, (size_t)b * 2 * f + c) -
                     partial_sum(p.fc2, (size_t)b * 2 * f + f + c);
    p.att[i] = 1.f / (1.f + expf(-dd));
  }
}

struct SkFcBwdArgs {
  GJob dw2, dz, dw1, ds;
  const float *dA, *att, *z, *zpre, *bnstat, *gamma;
  float *g_w1, *g_w2, *dgamma, *dbeta, *ds_out, *da, *dzpre;
  int B, f, d;
};

__global__ void __launch_bounds__(kFT)
sk_fc_bwd_fused_kernel(const SkFcBwdArgs p) {
  __shared__ float As[kTK][kTM + 4];
  __shared__ float Bs[kTK][kTN + 4];
  const int B = p.B, f = p.f, d = p.d;
  const int lane = threadIdx.x & 31;
  const int gtid = blockIdx.x * kFT + threadIdx.x, gthreads = gridDim.x * kFT;
  // softmax-2 backward: da0 = att (1 - att) dA = -da1
  for (int i = gtid; i < B * f; i += gthreads) {
    const int b = i / f, c = i - b * f;
    const float a = p.att[i];
    const float t = a * (1.f - a) * p.dA[i];
    p.da[(size_t)b * 2 * f + c] = t;
    p.da[(size_t)b * 2 * f + f + c] = -t;
  }
  grid_barrier();
  // dW2[2f,d] = da^T[2f,B] * z[B,d] ;  dz[B,d] = da[B,2f] * W2[2f,d]   (partials)
  run_jobs(p.dw2, &p.dz, As, Bs);
  grid_barrier();
  // dW2 += its partials; ReLU + batch-norm (over the batch) backward, one warp per channel
  for (int i = gtid; i < 2 * f * d; i += gthreads) p.g_w2[i] += partial_sum(p.dw2, i);
  for (int j = blockIdx.x * (kFT / 32) + (threadIdx.x >> 5); j < d; j += gridDim.x * (kFT / 32)) {
    const float mean = p.bnstat[j], rstd = p.bnstat[d + j];
    float s1 = 0.f, s2 = 0.f;
    for (int b = lane; b < B; b += 32) {
      const size_t i = (size_t)b * d + j;
      const float g = p.z[i] > 0.f ? partial_sum(p.dz, i) : 0.f;
      p.dzpre[i] = g;
      s1 += g;
      s2 += g * ((p.zpre[i] - mean) * rstd);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float k1 = p.gamma[j] * rstd;
    for (int b = lane; b < B; b += 32) {
      const size_t i = (size_t)b * d + j;
      const float xh = (p.zpre[i] - mean) * rstd;
      p.dzpre[i] = k1 * (p.dzpre[i] - s1 / B - xh * s2 / B);    // this lane's own stores
    }
    if (lane == 0) {
      p.dgamma[j] += s2;
      p.dbeta[j] += s1;
    }
  }
  grid_barrier();
  // dW1[d,f] = dzpre^T[d,B] * s[B,f] ;  ds[B,f] = dzpre[B,d] * W1[d,f]   (partials)
  run_jobs(p.dw1, &p.ds, As, Bs);
  grid_barrier();
  for (int i = gtid; i < d * f; i += gthreads) p.g_w1[i] += partial_sum(p.dw1, i);
  for (int i = gtid; i < B * f; i += gthreads) p.ds_out[i] = partial_sum(p.ds, i);
}

// grid of the fused chains: enough CTAs for the widest phase, all of them resident
static int fused_grid(int max_units) {
  int g = num_sms_small();
  if (g > kGridMax) g = kGridMax;
  if (max_units < g) g = max_units < 8 ? 8 : max_units;
  return g;
}

template <class Args>
static int launch_coop(void (*kern)(const Args), const Args& a, int grid, cudaStream_t st,
                       const char* what) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kFT);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kern, a);
  count_launch();
  return check_launch(what);
}

// -1 (default): the fused cooperative kernels when the caller asks for deterministic results (they
// are bit-reproducible and need no zeroing; the multi-launch path then runs WITHOUT split-K),
// otherwise the multi-launch split-K path; 0 / 1 force one of them.  A grid barrier costs about
// what a kernel boundary inside a CUDA graph costs, so fusing the 10 launches of a block into 2 only
// trades 8 boundaries for 7 barriers; the chain needs fewer PHASES, not fewer launches, to get
// faster.
static int g_sk_fc_fused = -1;
static bool use_fused(int deterministic) {
  return g_sk_fc_fused == 1 || (g_sk_fc_fused == -1 && deterministic);
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int64_t acnn_sk_fc_scratch_floats(int B, int f, int d) {
  if (B <= 0 || f <= 0 || d <= 0) return 0;
  const int G = kGridMax;
  const GJob fc1 = make_job(nullptr, nullptr, nullptr, B, d, f, f, 1, 1, f, G);
  const GJob fc2 = make_job(nullptr, nullptr, nullptr, B, 2 * f, d, d, 1, 1, d, G);
  const GJob dw2 = make_job(nullptr, nullptr, nullptr, 2 * f, d, B, 1, 2 * f, d, 1, G / 2);
  const GJob dz = make_job(nullptr, nullptr, nullptr, B, d, 2 * f, 2 * f, 1, d, 1, G / 2);
  const GJob dw1 = make_job(nullptr, nullptr, nullptr, d, f, B, 1, d, f, 1, G / 2);
  const GJob ds = make_job(nullptr, nullptr, nullptr, B, f, d, d, 1, f, 1, G / 2);
  int64_t m = job_floats(fc1);
  if (job_floats(fc2) > m) m = job_floats(fc2);
  if (job_floats(dw2) + job_floats(dz) > m) m = job_floats(dw2) + job_floats(dz);
  if (job_floats(dw1) + job_floats(ds) > m) m = job_floats(dw1) + job_floats(ds);
  return (int64_t)B * (2 * f + d) + m;
}

int acnn_set_sk_fc_fused(int on) {
  const int prev = g_sk_fc_fused;
  g_sk_fc_fused = on < 0 ? -1 : (on ? 1 : 0);
  return prev;
}

int acnn_sk_fc_fwd(const float* s, const float* w1, const float* gamma, const float* beta,
                   float* moving_mean, float* moving_var, float momentum, float eps, int training,
                   const float* w2, float* zpre, float* bnstat, float* z, float* att,
                   float* scratch, int B, int f, int d, int deterministic, void* stream) {
  ACNN_REQUIRE(s && w1 && gamma && beta && moving_mean && moving_var && w2 && zpre && bnstat && z &&
                   att && scratch, "sk_fc_fwd: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (use_fused(deterministic)) {
    const int G = num_sms_small() < kGridMax ? num_sms_small() : kGridMax;
    float* part = scratch + (size_t)B * (2 * f + d);
    SkFcFwdArgs a{};
    a.fc1 = make_job(s, w1, part, B, d, f, f, 1, 1, f, G);
    a.fc2 = make_job(z, w2, part, B, 2 * f, d, d, 1, 1, d, G);
    a.gamma = gamma; a.beta = beta; a.moving_mean = moving_mean; a.moving_var = moving_var;
    a.zpre = zpre; a.bnstat = bnstat; a.z = z; a.att = att;
    a.momentum = momentum; a.eps = eps; a.training = training; a.B = B; a.f = f; a.d = d;
    const int units = a.fc1.units > a.fc2.units ? a.fc1.units : a.fc2.units;
    return launch_coop(sk_fc_fwd_fused_kernel, a, fused_grid(units), st, "sk_fc_fwd_fused");
  }
  // zpre[B,d] = s[B,f] * W1[d,f]^T
  int rc = sgemm(s, w1, zpre, B, d, f, f, 1, 1, f, true, deterministic, st);
  if (rc) return rc;
  launch_k(bn_batch_relu_fwd_kernel, dim3(ceil_div(d, kFT / 32)), dim3(kFT), 0, st, zpre, gamma, beta, moving_mean, moving_var, momentum, eps, training, z, bnstat, B, d);
  count_launch();
  if ((rc = check_launch("sk bn_batch_relu_fwd"))) return rc;
  // a[B,2f] = z[B,d] * W2[2f,d]^T
  if ((rc = sgemm(z, w2, scratch, B, 2 * f, d, d, 1, 1, d, true, deterministic, st))) return rc;
  launch_k(sk_gate_fwd_kernel, dim3((int)ceil_div64((int64_t)B * f, 256)), dim3(256), 0, st, scratch, att, B, f);
  count_launch();
  return check_launch("sk_gate_fwd");
}

int acnn_sk_fc_bwd(const float* dA, const float* att, const float* z, const float* zpre,
                   const float* bnstat, const float* gamma, const float* s, const float* w1,
                   const float* w2, float* dw1, float* dw2, float* dgamma, float* dbeta, float* ds,
                   float* scratch, int B, int f, int d, int deterministic, void* stream) {
  ACNN_REQUIRE(dA && att && z && zpre && bnstat && gamma && s && w1 && w2 && dw1 && dw2 && dgamma &&
                   dbeta && ds && scratch, "sk_fc_bwd: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (use_fused(deterministic)) {
    const int G = num_sms_small() < kGridMax ? num_sms_small() : kGridMax;
    float* da = scratch;                       // [B][2f]
    float* dzp = scratch + (size_t)B * 2 * f;  // [B][d]
    float* part = scratch + (size_t)B * (2 * f + d);
    SkFcBwdArgs a{};
    a.dw2 = make_job(da, z, part, 2 * f, d, B, 1, 2 * f, d, 1, G / 2);
    a.dz = make_job(da, w2, part + job_floats(a.dw2), B, d, 2 * f, 2 * f, 1, d, 1, G / 2);
    a.dw1 = make_job(dzp, s, part, d, f, B, 1, d, f, 1, G / 2);
    a.ds = make_job(dzp, w1, part + job_floats(a.dw1), B, f, d, d, 1, f, 1, G / 2);
    a.dA = dA; a.att = att; a.z = z; a.zpre = zpre; a.bnstat = bnstat; a.gamma = gamma;
    a.g_w1 = dw1; a.g_w2 = dw2; a.dgamma = dgamma; a.dbeta = dbeta; a.ds_out = ds;
    a.da = da; a.dzpre = dzp; a.B = B; a.f = f; a.d = d;
    const int u2 = a.dw2.units + a.dz.units, u4 = a.dw1.units + a.ds.units;
    return launch_coop(sk_fc_bwd_fused_kernel, a, fused_grid(u2 > u4 ? u2 : u4), st,
                       "sk_fc_bwd_fused");
  }
  float* da = scratch;                       // [B][2f]
  float* dz = scratch + (size_t)B * 2 * f;   // [B][d]
  launch_k(sk_gate_bwd_kernel, dim3((int)ceil_div64((int64_t)B * f, 256)), dim3(256), 0, st, dA, att, da, B, f);
  count_launch();
  int rc = check_launch("sk_gate_bwd");
  if (rc) return rc;
  // dW2[2f,d] += da^T[2f,B] * z[B,d]
  if ((rc = sgemm(da, z, dw2, 2 * f, d, B, 1, 2 * f, d, 1, false, deterministic, st))) return rc;
  // dz[B,d] = da[B,2f] * W2[2f,d]
  if ((rc = sgemm(da, w2, dz, B, d, 2 * f, 2 * f, 1, d, 1, true, deterministic, st))) return rc;
  launch_k(bn_batch_relu_bwd_kernel, dim3(ceil_div(d, kFT / 32)), dim3(kFT), 0, st, dz, z, zpre, bnstat, gamma,
                                                                  dgamma, dbeta, B, d);
  count_launch();
  if ((rc = check_launch("sk bn_batch_relu_bwd"))) return rc;
  // dW1[d,f] += dzpre^T[d,B] * s[B,f]
  if ((rc = sgemm(dz, s, dw1, d, f, B, 1, d, f, 1, false, deterministic, st))) return rc;
  // ds[B,f] = dzpre[B,d] * W1[d,f]
  return sgemm(dz, w1, ds, B, f, d, d, 1, f, 1, true, deterministic, st);
}

int acnn_se_fc_fwd(const float* q, const float* w1, const float* w2, float* h, float* e, int B,
                   int C, int r, int deterministic, void* stream) {
  ACNN_REQUIRE(q && w1 && w2 && h && e, "se_fc_fwd: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  // h = relu(q[B,C] * W1[r,C]^T) ; e = sigmoid(h[B,r] * W2[C,r]^T)
  int rc = sgemm(q, w1, h, B, r, C, C, 1, 1, C, true, deterministic, st);
  if (rc) return rc;
  if ((rc = ew(h, nullptr, h, (int64_t)B * r, 1, 0.f, st))) return rc;
  if ((rc = sgemm(h, w2, e, B, C, r, r, 1, 1, r, true, deterministic, st))) return rc;
  return ew(e, nullptr, e, (int64_t)B * C, 2, 0.f, st);
}

int acnn_se_fc_bwd(const float* de, const float* e, const float* h, const float* q,
                   const float* w1, const float* w2, float* dw1, float* dw2, float* dq,
                   float* scratch, int B, int C, int r, int HW, int deterministic,
                   void* stream) {
  ACNN_REQUIRE(de && e && h && q && w1 && w2 && dw1 && dw2 && dq && scratch,
               "se_fc_bwd: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  float* da2 = scratch;                     // [B][C]
  float* dh = scratch + (size_t)B * C;      // [B][r]
  int rc = ew(de, e, da2, (int64_t)B * C, 4, 0.f, st);
  if (rc) return rc;
  if ((rc = sgemm(da2, h, dw2, C, r, B, 1, C, r, 1, false, deterministic, st))) return rc;    // dW2[C,r]
  if ((rc = sgemm(da2, w2, dh, B, r, C, C, 1, r, 1, true, deterministic, st))) return rc;     // dh = da2 * W2
  if ((rc = ew(dh, h, dh, (int64_t)B * r, 3, 0.f, st))) return rc;
  if ((rc = sgemm(dh, q, dw1, r, C, B, 1, r, C, 1, false, deterministic, st))) return rc;     // dW1[r,C]
  if ((rc = sgemm(dh, w1, dq, B, C, r, r, 1, C, 1, true, deterministic, st))) return rc;      // dq = da1 * W1
  return ew(dq, nullptr, dq, (int64_t)B * C, 5, 1.f / HW, st);
}

}  // extern "C"
