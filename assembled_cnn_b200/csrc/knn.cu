// Zero-shot retrieval top-k (metric/recall_metric.py:98-123) for sm_90a: the query x index
// similarity matrix is computed tile by tile with wgmma and reduced to a running top-k in the GEMM
// epilogue, so it never reaches HBM.
//
//   knn_prep_kernel : l2-normalised (cosine) or raw rows -> bf16 operands (or six plane segments in
//                     the fp32 mode, or fp16 operands in the fp16 mode), zero-padded to a multiple of
//                     64 in d, and their squared norms.
//   knn_topk_kernel : a CTA owns 128 query rows and walks a range of 128-column index tiles.  Warp 0
//                     is the TMA producer of an mbarrier ring (the organisation of conv_gemm_kernel);
//                     two consumer warpgroups accumulate 64 rows x 128 columns each in registers.
//                     Epilogue: a per-row threshold (the k-th best so far) filters the tile in
//                     registers; survivors go to a per-row candidate buffer in shared memory, which
//                     is merged into the row's sorted list when it could overflow.  The list lives in
//                     the (row, split) partial output.  A row is owned by one quad of one warp, so
//                     the warp maintains its 16 rows without any CTA-wide synchronisation.
//   knn_merge_kernel: the final k of every row from its per-split sorted lists, W lists per pass.
//
// acnn_knn_topk runs all three on Q and X.  For serving, acnn_knn_prepare_index runs the prep of X
// once into a caller-owned index, and acnn_knn_search prepares Q only and searches that index in up
// to one column split per SM (a small query batch is one row block), merged 16 lists per pass.
//
// Every selection uses the total order (similarity desc, index asc) and every similarity is the same
// fp32 value whatever the tile schedule, so the result does not depend on the split count.
#include <float.h>
#include <limits.h>
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "common.h"
#include "ptx.cuh"

namespace acnn {
namespace {

typedef __nv_bfloat16 bf16;

constexpr int kRows = 128;         // query rows per CTA (two consumer warpgroups x 64)
constexpr int kCols = 128;         // index columns per tile
constexpr int kStageK = 64;        // K elements per pipeline stage (one 128-byte swizzle row)
constexpr int kStages = 4;
constexpr int kThreads = 384;
constexpr int kConsumerWarps = 8;
constexpr int kBufCap = 64;        // candidates per row between merges: one half tile
constexpr int kBufStride = kBufCap + 1;
constexpr int kMaxK = 128;
constexpr int kMaxSplits = 8;
constexpr int kABytes = kRows * kStageK * 2;
constexpr int kBBytes = kCols * kStageK * 2;
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + 2 * kRows * kBufStride * 4 +
                           2 * kConsumerWarps * kMaxK * 4;
static_assert(kSmemBytes <= 227 * 1024, "shared memory");

struct KnnParams {
  int nq, nx, kp, k, euclid;
  int col_tiles, tiles_per_split;
  const float* qn;
  const float* xn;
  float* part_sim;   // [splits][nq][k]
  int* part_idx;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// (s1, i1) comes before (s2, i2): similarity descending, index ascending
__device__ __forceinline__ bool beats(float s1, int i1, float s2, int i2) {
  return s1 > s2 || (s1 == s2 && i1 < i2);
}

// One warp per row of Q and X.  E = bf16 (one plane, or six plane segments) or __half (one plane).
template <class E>
__global__ void __launch_bounds__(256)
knn_prep_kernel(const float* __restrict__ q, const float* __restrict__ x, int nq, int nx, int d,
                int dp, int planes, int cosine, E* __restrict__ qp, E* __restrict__ xp,
                float* __restrict__ qn, float* __restrict__ xn) {
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= nq + nx) return;
  const bool is_q = r < nq;
  const int row = is_q ? r : r - nq;
  const float* src = (is_q ? q : x) + (int64_t)row * d;
  E* dst = (is_q ? qp : xp) + (int64_t)row * dp * planes;
  float scale = 1.f;
  if (cosine) {
    float ss = 0.f;
    for (int i = lane; i < d; i += 32) ss = fmaf(src[i], src[i], ss);
    scale = rsqrtf(fmaxf(warp_sum(ss), 1e-12f));
  }
  float nrm = 0.f;
  for (int i = lane; i < dp; i += 32) {
    const float v = i < d ? src[i] * scale : 0.f;
    if constexpr (std::is_same<E, __half>::value) {
      // fp16 operands: round to nearest even (beyond +-65504: inf, then an unranked row)
      const __half h = __float2half_rn(v);
      dst[i] = h;
      const float r0 = __half2float(h);
      nrm = fmaf(r0, r0, nrm);
    } else {
      const bf16 h = __float2bfloat16_rn(v);
      if (planes == 1) {
        dst[i] = h;
        const float r0 = __bfloat162float(h);
        nrm = fmaf(r0, r0, nrm);
      } else {
        // v = hi + mid + lo (24 mantissa bits), the split of acnn_split3
        const float r1 = v - __bfloat162float(h);
        const bf16 m = __float2bfloat16_rn(r1);
        const bf16 l = __float2bfloat16_rn(r1 - __bfloat162float(m));
        const float rv = (__bfloat162float(h) + __bfloat162float(m)) + __bfloat162float(l);
        nrm = fmaf(rv, rv, nrm);
        // segments of the six plane products, smallest first: lo*hi, mid*mid, hi*lo, mid*hi,
        // hi*mid, hi*hi (Q' = hi mid lo hi mid hi, X' = lo mid hi mid hi hi)
        const bf16 seg_q[6] = {h, m, l, h, m, h};
        const bf16 seg_x[6] = {l, m, h, m, h, h};
#pragma unroll
        for (int s = 0; s < 6; ++s) dst[i + (int64_t)s * dp] = is_q ? seg_q[s] : seg_x[s];
      }
    }
  }
  nrm = warp_sum(nrm);
  if (lane == 0) (is_q ? qn : xn)[row] = nrm;
}

// Merges the candidate buffer of one row (nb entries, unsorted, shared memory) into its sorted list
// (nl entries, global memory): every entry's new position is the number of entries that beat it.
// Called by the whole warp.  Returns the new list length; *thr = its k-th similarity (or -inf).
__device__ int merge_row(int lane, const float* bs, const int* bi, int nb, float* ls, int* li, int nl,
                         int k, float* ws, int* wi, float* thr) {
  for (int i = lane; i < nl; i += 32) {
    ws[i] = ls[i];
    wi[i] = li[i];
  }
  __syncwarp();
  float cs[2 + kMaxK / 32];
  int ci[2 + kMaxK / 32], cr[2 + kMaxK / 32];
#pragma unroll
  for (int t = 0; t < 2 + kMaxK / 32; ++t) {
    const bool from_buf = t < 2;
    const int e = lane + 32 * (from_buf ? t : t - 2);
    cr[t] = INT_MAX;
    cs[t] = 0.f;
    ci[t] = 0;
    if (e < (from_buf ? nb : nl)) {
      const float s = from_buf ? bs[e] : ws[e];
      const int id = from_buf ? bi[e] : wi[e];
      int r = 0;
      if (from_buf) {          // list entries that beat it: binary search of the sorted list
        int lo = 0, hi = nl;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (beats(ws[mid], wi[mid], s, id)) lo = mid + 1;
          else hi = mid;
        }
        r = lo;
      } else {
        r = e;
      }
      for (int b = 0; b < nb; ++b) r += beats(bs[b], bi[b], s, id);
      cs[t] = s;
      ci[t] = id;
      cr[t] = r;
    }
  }
  __syncwarp();
  bool last = false;
  float last_s = -INFINITY;
#pragma unroll
  for (int t = 0; t < 2 + kMaxK / 32; ++t) {
    if (cr[t] < k) {
      ls[cr[t]] = cs[t];
      li[cr[t]] = ci[t];
    }
    if (cr[t] == k - 1) {
      last = true;
      last_s = cs[t];
    }
  }
  const int n = min(k, nl + nb);
  const unsigned who = __ballot_sync(0xffffffffu, last);
  *thr = n == k ? __shfl_sync(0xffffffffu, last_s, __ffs(who) - 1) : -INFINITY;
  __syncwarp();
  return n;
}

template <bool F16>
__global__ void __launch_bounds__(kThreads, 1)
knn_topk_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmX,
                const KnnParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  float* bsim = reinterpret_cast<float*>(smem + kStages * kStageBytes);
  int* bidx = reinterpret_cast<int*>(bsim + kRows * kBufStride);
  float* wsim = reinterpret_cast<float*>(bidx + kRows * kBufStride);
  int* widx = reinterpret_cast<int*>(wsim + kConsumerWarps * kMaxK);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kRows;
  const int split = blockIdx.y;
  const int t0 = split * p.tiles_per_split;
  const int t1 = min(p.col_tiles, t0 + p.tiles_per_split);
  const int num_kb = p.kp / kStageK;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmX);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_entry();

  const uint32_t smem_a0 = smem_u32(smem);
  const uint32_t full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    uint32_t stage = 0, phase = 0;
    for (int t = t0; t < t1; ++t) {
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_a(empty0 + stage * 8, phase ^ 1);
        if (elect_one()) {
          const uint32_t fb = full0 + stage * 8;
          const uint32_t sa = smem_a0 + stage * kStageBytes;
          mbar_expect_tx_a(fb, kStageBytes);
          tma_load_2d_a(sa, &tmQ, fb, kb * kStageK, m0);
          tma_load_2d_a(sa + kABytes, &tmX, fb, kb * kStageK, t * kCols);
        }
        __syncwarp();
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ wgmma consumers
    const int cg = (warp >> 2) - 1;                 // rows cg*64 ..
    const int row_base = cg * 64 + (warp & 3) * 16; // this warp's 16 rows (CTA-local)
    const int quad = lane >> 2;                     // fragment rows row_base + quad (+ 8)
    const int cq = (lane & 3) * 2;                  // fragment column offset
    float* ws = wsim + (warp - 4) * kMaxK;
    int* wi = widx + (warp - 4) * kMaxK;
    const uint64_t a_desc0 = make_smem_desc(smem_a0 + cg * 64 * kStageK * 2, 16, 8 * kStageK * 2,
                                            swizzle_layout_type(kStageK * 2));
    const uint64_t b_desc0 = make_smem_desc(smem_a0 + kABytes, 16, 8 * kStageK * 2,
                                            swizzle_layout_type(kStageK * 2));
    float acc[kCols / 2];
    // state of rows row_base + quad + 8h, identical in the four lanes of the quad
    int nl[2] = {0, 0}, nb[2] = {0, 0};
    float thr[2] = {-INFINITY, -INFINITY}, qnr[2] = {0.f, 0.f};
    bool rvalid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = m0 + row_base + quad + 8 * h;
      rvalid[h] = grow < p.nq;
      if (p.euclid && rvalid[h]) qnr[h] = p.qn[grow];
    }
    // merges row R (0..15) of this warp into its partial list; called by the whole warp
    auto flush = [&](int R) {
      const int src = 4 * (R & 7);
      const bool hi = R >= 8;
      const int rb = __shfl_sync(0xffffffffu, hi ? nb[1] : nb[0], src);
      const int rl = __shfl_sync(0xffffffffu, hi ? nl[1] : nl[0], src);
      const int row = row_base + R;
      const size_t off = ((size_t)split * p.nq + (m0 + row)) * p.k;
      float t;
      const int n = merge_row(lane, bsim + row * kBufStride, bidx + row * kBufStride, rb,
                              p.part_sim + off, p.part_idx + off, rl, p.k, ws, wi, &t);
      if (quad == (R & 7)) {
        if (hi) { nl[1] = n; nb[1] = 0; thr[1] = t; }
        else { nl[0] = n; nb[0] = 0; thr[0] = t; }
      }
    };
    // rows (bit R) of this warp whose buffer fails the predicate of their quad's leader
    auto rows_where = [&](bool c0, bool c1) {
      const unsigned b0 = __ballot_sync(0xffffffffu, (lane & 3) == 0 && c0);
      const unsigned b1 = __ballot_sync(0xffffffffu, (lane & 3) == 0 && c1);
      unsigned m = 0;
#pragma unroll
      for (int r = 0; r < 8; ++r) m |= (((b0 >> (4 * r)) & 1u) << r) | (((b1 >> (4 * r)) & 1u) << (r + 8));
      return m;
    };

    uint32_t stage = 0, phase = 0;
    for (int t = t0; t < t1; ++t) {
      const int n0 = t * kCols;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_a(full0 + stage * 8, phase);
        wgmma_fence_operand(acc);
        wgmma_fence();
        const uint64_t da0 = a_desc0 + ((stage * kStageBytes) >> 4);
        const uint64_t db0 = b_desc0 + ((stage * kStageBytes) >> 4);
#pragma unroll
        for (int ks = 0; ks < kStageK / 16; ++ks)
          WgmmaOp<kCols, F16>::type::template mma<0, 0>(acc, da0 + ((ks * 32) >> 4), db0 + ((ks * 32) >> 4),
                                           (ks | kb) ? 1u : 0u);
        wgmma_commit();
        wgmma_fence_operand(acc);
        wgmma_wait<1>();
        __syncwarp();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = static_cast<int>(stage);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue, per half tile (64 columns = the buffer capacity)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        float xc[16];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = n0 + (hf * 8 + jj) * 8 + cq + e;
            xc[jj * 2 + e] = (p.euclid && col < p.nx) ? __ldg(p.xn + col) : 0.f;
          }
        // similarity of fragment value (jj, e) of row h; -inf for padding rows / columns
        auto sim = [&](int h, int jj, int e) {
          const int col = n0 + (hf * 8 + jj) * 8 + cq + e;
          const float a = acc[(hf * 8 + jj) * 4 + h * 2 + e];
          const float v = p.euclid ? -__fsub_rn(__fadd_rn(qnr[h], xc[jj * 2 + e]), 2.f * a) : a;
          return (rvalid[h] && col < p.nx) ? v : -INFINITY;
        };
        // a column beyond every listed index passes only above the threshold (ties go to the
        // lower index); the counts use the threshold from before this half's flushes
        const float tc[2] = {thr[0], thr[1]};
        int cnt[2] = {0, 0};
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int e = 0; e < 2; ++e) cnt[h] += sim(h, jj, e) > tc[h];
        // positions in the quad's part of the row buffer: exclusive scan over the quad
        int excl[2], tot[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          int incl = cnt[h];
          int y = __shfl_up_sync(0xffffffffu, incl, 1, 4);
          if ((lane & 3) >= 1) incl += y;
          y = __shfl_up_sync(0xffffffffu, incl, 2, 4);
          if ((lane & 3) >= 2) incl += y;
          tot[h] = __shfl_sync(0xffffffffu, incl, 3, 4);
          excl[h] = incl - cnt[h];
        }
        unsigned need = rows_where(nb[0] + tot[0] > kBufCap, nb[1] + tot[1] > kBufCap);
        while (need) {
          const int R = __ffs(need) - 1;
          need &= need - 1;
          flush(R);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (cnt[h]) {
            const int row = row_base + quad + 8 * h;
            int pos = row * kBufStride + nb[h] + excl[h];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float v = sim(h, jj, e);
                if (v > tc[h]) {
                  bsim[pos] = v;
                  bidx[pos] = n0 + (hf * 8 + jj) * 8 + cq + e;
                  ++pos;
                }
              }
          }
          nb[h] += tot[h];
        }
        __syncwarp();
      }
    }
    // ---- final merges, then the unfilled tail of every list (fewer than k columns in the range)
    unsigned need = rows_where(nb[0] > 0, nb[1] > 0);
    while (need) {
      const int R = __ffs(need) - 1;
      need &= need - 1;
      flush(R);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!rvalid[h]) continue;
      const size_t off = ((size_t)split * p.nq + (m0 + row_base + quad + 8 * h)) * p.k;
      for (int s = nl[h] + (lane & 3); s < p.k; s += 4) {
        p.part_sim[off + s] = -INFINITY;
        p.part_idx[off + s] = INT_MAX;
      }
    }
  }
}

// One thread per row: W-way merge of the row's sorted lists.  blockIdx.y = g merges lists
// [g * W, min((g + 1) * W, splits)) into output list g (out + g * nq * k), so passes of W-way merges
// reduce any number of lists.
template <int W>
__global__ void __launch_bounds__(128)
knn_merge_kernel(const float* __restrict__ ps, const int* __restrict__ pi, int nq, int k, int splits,
                 int32_t* __restrict__ out_idx, float* __restrict__ out_sim) {
  pdl_wait();
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= nq) return;
  const size_t stride = (size_t)nq * k;
  const size_t base = (size_t)row * k;
  ps += blockIdx.y * W * stride;
  pi += blockIdx.y * W * stride;
  out_idx += blockIdx.y * stride;
  out_sim += blockIdx.y * stride;
  splits = min(splits - (int)blockIdx.y * W, W);
  int head[W];
  float hs[W];
  int hi[W];
#pragma unroll
  for (int s = 0; s < W; ++s) {
    head[s] = 0;
    hs[s] = -INFINITY;
    hi[s] = INT_MAX;
    if (s < splits) {
      hs[s] = ps[s * stride + base];
      hi[s] = pi[s * stride + base];
    }
  }
  for (int o = 0; o < k; ++o) {
    // the best head, carried in scalars: the arrays are indexed by unrolled constants only, so they
    // stay in registers
    int best = 0;
    float bs = hs[0];
    int bi = hi[0];
#pragma unroll
    for (int s = 1; s < W; ++s)
      if (s < splits && beats(hs[s], hi[s], bs, bi)) { best = s; bs = hs[s]; bi = hi[s]; }
    out_sim[base + o] = bs;
    out_idx[base + o] = bi;
#pragma unroll
    for (int s = 0; s < W; ++s) {
      if (s == best) {
        ++head[s];
        hs[s] = head[s] < k ? ps[s * stride + base + head[s]] : -INFINITY;
        hi[s] = head[s] < k ? pi[s * stride + base + head[s]] : INT_MAX;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
int g_knn_splits = 0;

inline int64_t align256(int64_t b) { return (b + 255) & ~int64_t(255); }

struct KnnLayout {
  int dp, planes;
  int64_t kp, q, x, qn, xn, ps, pi, total;   // element counts / byte offsets
};

KnnLayout knn_layout(int nq, int nx, int d, int k, int dtype) {
  KnnLayout l;
  l.dp = (d + kStageK - 1) / kStageK * kStageK;
  l.planes = dtype == ACNN_F32 ? 6 : 1;
  l.kp = (int64_t)l.planes * l.dp;
  l.q = 0;
  l.x = align256(l.q + (int64_t)nq * l.kp * 2);
  l.qn = align256(l.x + (int64_t)nx * l.kp * 2);
  l.xn = align256(l.qn + (int64_t)nq * 4);
  l.ps = align256(l.xn + (int64_t)nx * 4);
  l.pi = align256(l.ps + (int64_t)kMaxSplits * nq * k * 4);
  l.total = align256(l.pi + (int64_t)kMaxSplits * nq * k * 4);
  return l;
}

// acnn_knn_search: up to one column split per SM, reduced by passes of kMergeFanIn-way merges
constexpr int kMaxSearchSplits = kMaxSms;
constexpr int kMergeFanIn = 16;

int search_max_splits(int nx) { return std::min(ceil_div(nx, kCols), kMaxSearchSplits); }

// The prepared index (X' [nx][K'], then |x|^2 [nx]) and the search work (Q' [nq][K'], |q|^2 [nq],
// the per-split lists, the lists of the first merge pass when there is more than one pass)
struct SearchLayout {
  int dp, planes;
  int64_t kp, xn, index_total;                    // index
  int64_t qn, ps, pi, ms, mi, total;              // work
};

SearchLayout search_layout(int nq, int nx, int d, int k, int dtype) {
  SearchLayout l;
  l.dp = (d + kStageK - 1) / kStageK * kStageK;
  l.planes = dtype == ACNN_F32 ? 6 : 1;
  l.kp = (int64_t)l.planes * l.dp;
  l.xn = align256((int64_t)nx * l.kp * 2);
  l.index_total = align256(l.xn + (int64_t)nx * 4);
  const int64_t lists = (int64_t)search_max_splits(nx);
  const int64_t mlists = lists > kMergeFanIn ? ceil_div64(lists, kMergeFanIn) : 0;
  l.qn = align256((int64_t)nq * l.kp * 2);
  l.ps = align256(l.qn + (int64_t)nq * 4);
  l.pi = align256(l.ps + lists * nq * k * 4);
  l.ms = align256(l.pi + lists * nq * k * 4);
  l.mi = align256(l.ms + mlists * nq * k * 4);
  l.total = align256(l.mi + mlists * nq * k * 4);
  return l;
}

// Column splits: forced by acnn_set_knn_splits, else the count that minimises
// waves x (tiles per split + 1 tile of pipeline fill and list writes) with one CTA per SM;
// at most max_splits (kMaxSplits for acnn_knn_topk)
int knn_splits(int q_blocks, int col_tiles, int max_splits = kMaxSplits) {
  const int cap = std::min(col_tiles, max_splits);
  int s = g_knn_splits;
  if (s <= 0) {
    int64_t best = INT64_MAX;
    for (int c = 1; c <= cap; ++c) {
      const int64_t waves = ceil_div64((int64_t)q_blocks * c, num_sms());
      const int64_t cost = waves * (ceil_div(col_tiles, c) + 1);
      if (cost < best) { best = cost; s = c; }
    }
  }
  return std::max(1, std::min(s, cap));
}

int knn_check(int nq, int nx, int d, int k, int metric, int dtype) {
  ACNN_REQUIRE(nq > 0 && nx > 0 && d > 0 && d <= (1 << 24) && k >= 1,
               "knn_topk: bad sizes nq=%d nx=%d d=%d k=%d", nq, nx, d, k);
  ACNN_REQUIRE(metric == 0 || metric == 1, "knn_topk: unknown metric %d", metric);
  ACNN_REQUIRE(dtype == ACNN_BF16 || dtype == ACNN_F32 || dtype == ACNN_F16, "knn_topk: unknown dtype %d",
               dtype);
  if (k > kMaxK) {
    set_error("knn_topk: k=%d > %d is not supported", k, kMaxK);
    return ACNN_ERR_UNSUPPORTED;
  }
  ACNN_REQUIRE(k <= nx, "knn_topk: k=%d exceeds the %d index rows", k, nx);
  return ACNN_OK;
}


// knn_prep_kernel over nq query rows and nx index rows (either may be 0)
int knn_prep(const float* q, const float* x, int nq, int nx, int d, int dp, int planes, int metric, bool f16,
             void* qp, void* xp, float* qn, float* xn, cudaStream_t st) {
  const int cosine = metric == 0 ? 1 : 0;
  if (f16) {
    launch_k(knn_prep_kernel<__half>, dim3(ceil_div(nq + nx, 8)), dim3(256), 0, st, q, x, nq, nx, d, dp, planes,
             cosine, static_cast<__half*>(qp), static_cast<__half*>(xp), qn, xn);
  } else {
    launch_k(knn_prep_kernel<bf16>, dim3(ceil_div(nq + nx, 8)), dim3(256), 0, st, q, x, nq, nx, d, dp, planes,
             cosine, static_cast<bf16*>(qp), static_cast<bf16*>(xp), qn, xn);
  }
  return check_launch("knn_prep_kernel");
}

// knn_topk_kernel over prepared operands (Q' [nq][kp], X' [nx][kp] and their squared norms) in up to
// max_splits column splits, then the merges of the per-split lists (ps / pi, [splits][nq][k]) into
// out: one pass of kMaxSplits-way merges when max_splits <= kMaxSplits, else passes of
// kMergeFanIn-way merges through ms / mi ([ceil(splits / kMergeFanIn)][nq][k]) and back.
// `launches` counts the launches before this one (the prep).
int knn_run(const void* qp, const void* xp, const float* qn, const float* xn, int nq, int nx, int kp, int k,
            int metric, bool f16, int max_splits, float* ps, int* pi, float* ms, int* mi, int32_t* out_idx,
            float* out_sim, cudaStream_t st, int launches) {
  int rc;
  auto* topk = f16 ? knn_topk_kernel<true> : knn_topk_kernel<false>;
  static bool attr_set[2] = {false, false};
  if (!attr_set[f16]) {
    cudaError_t e = cudaFuncSetAttribute(topk, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(knn_topk): %s", cudaGetErrorString(e));
      return ACNN_ERR_CUDA;
    }
    attr_set[f16] = true;
  }
  CUtensorMap tmQ, tmX;
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if ((rc = make_map_2d(&tmQ, qp, nq, kp, kp, kRows, kStageK, dt))) return rc;
  if ((rc = make_map_2d(&tmX, xp, nx, kp, kp, kCols, kStageK, dt))) return rc;

  KnnParams p;
  p.nq = nq;
  p.nx = nx;
  p.kp = kp;
  p.k = k;
  p.euclid = metric == 1;
  p.col_tiles = ceil_div(nx, kCols);
  const int q_blocks = ceil_div(nq, kRows);
  const int splits_req = knn_splits(q_blocks, p.col_tiles, max_splits);
  p.tiles_per_split = ceil_div(p.col_tiles, splits_req);
  const int splits = ceil_div(p.col_tiles, p.tiles_per_split);   // no empty split
  p.qn = qn;
  p.xn = xn;
  p.part_sim = ps;
  p.part_idx = pi;
  launch_k(topk, dim3(q_blocks, splits), dim3(kThreads), kSmemBytes, st, tmQ, tmX, p);
  if ((rc = check_launch("knn_topk_kernel"))) return rc;

  const int fan_in = max_splits <= kMaxSplits ? kMaxSplits : kMergeFanIn;
  auto* merge = fan_in == kMaxSplits ? knn_merge_kernel<kMaxSplits> : knn_merge_kernel<kMergeFanIn>;
  const float* ls = ps;
  const int* li = pi;
  int lists = splits;
  launches += 2;
  for (bool to_m = true; lists > fan_in; to_m = !to_m, ++launches) {
    const int groups = ceil_div(lists, fan_in);
    float* os = to_m ? ms : ps;
    int* oi = to_m ? mi : pi;
    launch_k(merge, dim3(ceil_div(nq, 128), groups), dim3(128), 0, st, ls, li, nq, k, lists, oi, os);
    if ((rc = check_launch("knn_merge_kernel"))) return rc;
    ls = os;
    li = oi;
    lists = groups;
  }
  launch_k(merge, dim3(ceil_div(nq, 128)), dim3(128), 0, st, ls, li, nq, k, lists, out_idx, out_sim);
  count_launch(launches);
  return check_launch("knn_merge_kernel");
}

}  // namespace
}  // namespace acnn

extern "C" {

int64_t acnn_knn_work_bytes(int nq, int nx, int d, int k, int dtype) {
  if (acnn::knn_check(nq, nx, d, k, 0, dtype) != ACNN_OK) return -1;
  return acnn::knn_layout(nq, nx, d, k, dtype).total;
}

int acnn_set_knn_splits(int n) {
  const int prev = acnn::g_knn_splits;
  acnn::g_knn_splits = n > 0 ? n : 0;
  return prev;
}

int acnn_knn_topk(const float* q, const float* x, int nq, int nx, int d, int k, int metric, int dtype,
                  int32_t* out_idx, float* out_sim, void* work, int64_t work_bytes, void* stream) {
  using namespace acnn;
  int rc = knn_check(nq, nx, d, k, metric, dtype);
  if (rc) return rc;
  ACNN_REQUIRE(q && x && out_idx && out_sim && work, "knn_topk: null pointer");
  const KnnLayout l = knn_layout(nq, nx, d, k, dtype);
  ACNN_REQUIRE(work_bytes >= l.total, "knn_topk: work of %lld bytes, %lld needed",
               (long long)work_bytes, (long long)l.total);
  ACNN_REQUIRE(reinterpret_cast<uintptr_t>(work) % 256 == 0, "knn_topk: work must be 256-byte aligned");
  if ((rc = load_driver_fns())) return rc;
  // fp16 mode (ACNN_F16): fp16 operands, wgmma .f16.f16, fp32 accumulation; the rest is shared
  const bool f16 = dtype == ACNN_F16;
  uint8_t* w = static_cast<uint8_t*>(work);
  float* qn = reinterpret_cast<float*>(w + l.qn);
  float* xn = reinterpret_cast<float*>(w + l.xn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = knn_prep(q, x, nq, nx, d, l.dp, l.planes, metric, f16, w + l.q, w + l.x, qn, xn, st))) return rc;
  float* ps = reinterpret_cast<float*>(w + l.ps);
  int* pi = reinterpret_cast<int*>(w + l.pi);
  return knn_run(w + l.q, w + l.x, qn, xn, nq, nx, (int)l.kp, k, metric, f16, kMaxSplits, ps, pi, ps, pi,
                 out_idx, out_sim, st, 1);
}

int64_t acnn_knn_index_bytes(int nx, int d, int dtype) {
  if (acnn::knn_check(1, nx, d, 1, 0, dtype) != ACNN_OK) return -1;
  return acnn::search_layout(1, nx, d, 1, dtype).index_total;
}

int acnn_knn_prepare_index(const float* x, int nx, int d, int metric, int dtype, void* index,
                           int64_t index_bytes, void* stream) {
  using namespace acnn;
  int rc = knn_check(1, nx, d, 1, metric, dtype);
  if (rc) return rc;
  ACNN_REQUIRE(x && index, "knn_prepare_index: null pointer");
  const SearchLayout l = search_layout(1, nx, d, 1, dtype);
  ACNN_REQUIRE(index_bytes >= l.index_total, "knn_prepare_index: index of %lld bytes, %lld needed",
               (long long)index_bytes, (long long)l.index_total);
  ACNN_REQUIRE(reinterpret_cast<uintptr_t>(index) % 256 == 0,
               "knn_prepare_index: index must be 256-byte aligned");
  uint8_t* ix = static_cast<uint8_t*>(index);
  count_launch(1);
  return knn_prep(nullptr, x, 0, nx, d, l.dp, l.planes, metric, dtype == ACNN_F16, nullptr, ix,
                  nullptr, reinterpret_cast<float*>(ix + l.xn), static_cast<cudaStream_t>(stream));
}

int64_t acnn_knn_search_work_bytes(int nq, int nx, int d, int k, int dtype) {
  if (acnn::knn_check(nq, nx, d, k, 0, dtype) != ACNN_OK) return -1;
  return acnn::search_layout(nq, nx, d, k, dtype).total;
}

int acnn_knn_search(const float* q, int nq, const void* index, int nx, int d, int k, int metric, int dtype,
                    int32_t* out_idx, float* out_sim, void* work, int64_t work_bytes, void* stream) {
  using namespace acnn;
  int rc = knn_check(nq, nx, d, k, metric, dtype);
  if (rc) return rc;
  ACNN_REQUIRE(q && index && out_idx && out_sim && work, "knn_search: null pointer");
  const SearchLayout l = search_layout(nq, nx, d, k, dtype);
  ACNN_REQUIRE(work_bytes >= l.total, "knn_search: work of %lld bytes, %lld needed",
               (long long)work_bytes, (long long)l.total);
  ACNN_REQUIRE(reinterpret_cast<uintptr_t>(work) % 256 == 0 && reinterpret_cast<uintptr_t>(index) % 256 == 0,
               "knn_search: work and index must be 256-byte aligned");
  if ((rc = load_driver_fns())) return rc;
  const bool f16 = dtype == ACNN_F16;
  uint8_t* w = static_cast<uint8_t*>(work);
  const uint8_t* ix = static_cast<const uint8_t*>(index);
  float* qn = reinterpret_cast<float*>(w + l.qn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = knn_prep(q, nullptr, nq, 0, d, l.dp, l.planes, metric, f16, w, nullptr, qn, nullptr, st))) return rc;
  return knn_run(w, ix, qn, reinterpret_cast<const float*>(ix + l.xn), nq, nx, (int)l.kp, k, metric, f16,
                 std::min(search_max_splits(nx), num_sms()), reinterpret_cast<float*>(w + l.ps),
                 reinterpret_cast<int*>(w + l.pi), reinterpret_cast<float*>(w + l.ms),
                 reinterpret_cast<int*>(w + l.mi), out_idx, out_sim, st, 1);
}

}  // extern "C"
