// wgmma implicit-GEMM convolutions for sm_90a.
//
//   conv_gemm_kernel : y[M, Cout] = im2col(x)[M, K] * w[Cout, K]^T          (fprop, dgrad, dense)
//                      A tiles arrive by TMA (tiled 2-D for 1x1/s1, im2col 4-D otherwise) in the
//                      128B/64B/32B-swizzled K-major layout wgmma reads directly; the fp32
//                      accumulator lives in the registers of two consumer warpgroups, which then
//                      fuse bias / gradient-accumulate / ReLU-mask / batch-norm column sums.
//   wgrad_gemm_kernel: dw[Cout, K] += dy[P, Cout]^T * im2col(x)[P, K]       (split-K over pixels)
//                      both operands are MN-major (the pixel index is the GEMM K dimension).
//
// Warp roles (384 threads): warp 0 = TMA producer (warps 1..3 idle), warpgroups 1 and 2 = wgmma
// consumers + epilogue, 64 accumulator rows each.  The bf16 / fp16 fprop and dgrad GEMMs with
// K <= 512 run conv_gemm_kernel two CTAs per SM instead (160 threads: one consumer warpgroup for all
// 128 rows, warp 4 = TMA producer), so one CTA's epilogue overlaps the other's MMAs.
//
// Reference semantics: nets/model_helper.py:67-78 (conv2d_fixed_padding), tf.gradients backward.
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "common.h"
#include "ptx.cuh"

namespace acnn {

// Element pitches of the input tensor: dense NHWC unless the geometry overrides them (used by the
// space-to-depth stem, whose "pixels" are overlapping 4-pixel windows of a W-padded image).
static void input_pitches(const acnn_conv_geom& g, int64_t* pix, int64_t* row, int64_t* img) {
  *pix = g.x_pix_stride > 0 ? g.x_pix_stride : g.Cin;
  *row = g.x_row_pitch > 0 ? g.x_row_pitch : (int64_t)g.W * *pix;
  *img = g.x_img_pitch > 0 ? g.x_img_pitch : (int64_t)g.H * *row;
}

static bool is_plain(const acnn_conv_geom& g) {
  return g.kh == 1 && g.kw == 1 && g.stride == 1 && g.pad_h_lo == 0 && g.pad_w_lo == 0 &&
         g.pad_h_hi == 0 && g.pad_w_hi == 0 && g.x_pix_stride <= 0 && g.x_row_pitch <= 0 &&
         g.x_img_pitch <= 0;
}

// bf16 NHWC tensor [B][H][W][C]; one load = `pixels` consecutive output pixels x `cw` channels of
// one filter tap.  The bounding box of base pixels is [-pad_lo, dim + pad_hi - (k-1)).
static int make_map_im2col(CUtensorMap* m, const void* base, const acnn_conv_geom& g, int cw,
                           int pixels, CUtensorMapDataType dt) {
  int64_t pix, row, img;
  input_pitches(g, &pix, &row, &img);
  cuuint64_t dims[4] = {(cuuint64_t)g.Cin, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.B};
  cuuint64_t strides[3] = {(cuuint64_t)pix * 2, (cuuint64_t)row * 2, (cuuint64_t)img * 2};
  int lower[2] = {-g.pad_w_lo, -g.pad_h_lo};
  int upper[2] = {g.pad_w_hi - (g.kw - 1), g.pad_h_hi - (g.kh - 1)};
  cuuint32_t estr[4] = {1, (cuuint32_t)g.stride, (cuuint32_t)g.stride, 1};
  CUresult r = g_encode_im2col(m, dt, 4, const_cast<void*>(base),
                               dims, strides, lower, upper, (cuuint32_t)cw, (cuuint32_t)pixels,
                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_enum(cw * 2),
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed (%d): B=%d H=%d W=%d C=%d k=%dx%d s=%d cw=%d px=%d "
              "pitches=%lld/%lld/%lld", (int)r, g.B, g.H, g.W, g.Cin, g.kh, g.kw, g.stride, cw,
              pixels, (long long)pix, (long long)row, (long long)img);
    return ACNN_ERR_CUDA;
  }
  // Driver <= 13.1 mis-encodes im2col maps of tensors smaller than 128 KiB (same fix-up the
  // CUTLASS im2col descriptor builder applies): clear bit 21 of the second descriptor word.
  if (g_driver_version <= 13010 && (int64_t)g.B * img * 2 < 131072) {
    reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
  }
  return ACNN_OK;
}

// ------------------------------------------------------------------------------------------
// fprop / dgrad / dense kernel (persistent, warp-specialised)
// ------------------------------------------------------------------------------------------
struct ConvGemmParams {
  int M;          // output pixels B*Ho*Wo
  int Cout;       // GEMM N
  int Cin;        // channels per filter tap
  int Ktot;       // kh*kw*Cin
  int kw;         // taps per filter row
  int HoWo, Wo;   // to decompose a row index into (n, p, q)
  int stride, pad_h_lo, pad_w_lo;
  int b_sw_bytes; // swizzle span of the weight tile (128 unless Ktot < 64)
  int stages;     // smem pipeline depth
  int m_tiles, n_tiles;
  void* y;
  float* ch_part;   // [gridDim.x / n_tiles][2][Cout] per-CTA partial (sum, sum of squares) rows
  const float* bias;
  int has_add, has_mask;
  int out_f32;
};

constexpr int kBM = 128;        // output pixels per CTA tile (two consumer warpgroups x 64 rows)
constexpr int kStageK = 64;     // K elements per pipeline stage
// 3 warpgroups: warpgroup 0 = TMA producer (warp 0 issues), warpgroups 1 and 2 = wgmma consumers,
// rows 0..63 and 64..127 of every tile, which then run the epilogue from their accumulator registers
constexpr int kThreads = 384;
constexpr int kConsumerThreads = 256;
constexpr int kConsumerWarps = 8;
constexpr int kMaxStages = 8;
constexpr int kSmemBudget = 224 * 1024;   // dynamic smem (227 KiB max per CTA on sm_90)
// Two co-resident CTAs per SM (WG = 1 below): one consumer warpgroup (warps 0..3, both 64-row halves
// of the 128-row tile) + one TMA producer warp (warp 4), so one CTA's epilogue runs while the other's
// MMAs do.  Dynamic smem per CTA: 2 x (dynamic + static barriers + 1 KiB reserved) <= 228 KiB.
constexpr int kSmemBudget2 = 112 * 1024 + 512;
__host__ __device__ constexpr int conv_threads(int wg) { return wg == 2 ? kThreads : 160; }

// (a-plane, b-plane) of the t-th cross product of two 3-plane operands, smallest magnitude first:
// (2,0) (1,1) (0,2) [2^-16]  (1,0) (0,1) [2^-8]  (0,0)
__host__ __device__ constexpr int plane_term_a(int t) { return t == 0 ? 2 : ((t == 1 || t == 3) ? 1 : 0); }
__host__ __device__ constexpr int plane_term_b(int t) { return t == 2 ? 2 : ((t == 1 || t == 4) ? 1 : 0); }

// NP = operand planes: 1 = bf16 operands; 3 = fp32 operands split into three bf16 planes
// (x = hi + mid + lo, 24 mantissa bits) whose six significant cross products are accumulated in
// fp32 -- the fp32 parity mode (acnn.h ACNN_F32) on the same TMA / im2col / descriptor / epilogue
// code as the bf16 path.
static inline int fprop_stage_bytes(int bn, int np) { return np * (kBM * kStageK * 2 + bn * kStageK * 2); }
// column width of one epilogue step (one staged tile): 128 with two consumer warpgroups; with one
// (two CTAs per SM) the kSubW = 64-column TMA sub-tile, so that the staging leaves room for stages
__host__ __device__ constexpr int fprop_epi_cols(int bn, int wg) {
  return wg == 2 ? (bn > 128 ? 128 : bn) : (bn > 64 ? 64 : bn);
}
// dynamic shared memory of one conv_gemm_kernel launch, and its pipeline depth in *stages:
// [stages x (A|B)] [out staging] [add staging] [mask staging]
static inline int fprop_smem(int bn, int np, int wg, bool has_add, bool has_mask, bool out_f32,
                             int* stages) {
  const int tile = kBM * fprop_epi_cols(bn, wg) * 2;
  const int fixed = 1024 + (out_f32 ? 0 : tile) + (has_add ? tile : 0) + (has_mask ? tile : 0);
  int st = ((wg == 2 ? kSmemBudget : kSmemBudget2) - fixed) / fprop_stage_bytes(bn, np);
  if (st > kMaxStages) st = kMaxStages;
  if (st < 2) st = 2;
  *stages = st;
  return fixed + st * fprop_stage_bytes(bn, np);
}

template <int BN, int NP = 1, int WG = 2>
struct FpropCfg {
  static constexpr int kABytes = kBM * kStageK * 2;       // one plane, 16 KiB
  static constexpr int kBBytes = BN * kStageK * 2;        // one plane
  static constexpr int kStageBytes = NP * (kABytes + kBBytes);
  static_assert(2 * kStageBytes + 1024 <= (WG == 2 ? kSmemBudget : kSmemBudget2),
                "two pipeline stages must fit");
  static_assert(WG == 2 || NP == 1, "two CTAs per SM: bf16 / fp16 operands only");
  // the epilogue stages the tile in column groups of fprop_epi_cols (one staging buffer each for
  // the output, add and mask tiles), so a 128 x 256 tile needs no more staging than 128 x 128
  static constexpr int kHalfN = fprop_epi_cols(BN, WG);
  static constexpr int kNHalf = BN / kHalfN;
  static constexpr int kSubW = BN < 64 ? BN : 64;         // staging sub-tile width (TMA box)
  static constexpr int kTileBytes = kBM * kHalfN * 2;      // one staged half tile (bf16)
  // NP == 3 keeps TWO accumulators -- the hi*hi products and the five small cross terms
  // separately (added in the epilogue) -- because the tensor core truncates an addend below the
  // accumulator's ulp: small terms summed into the big accumulator lose ~6 bits each
  static_assert(NP == 1 || BN <= 128, "fp32 mode: N tile <= 128 (registers)");
  // (NP == 3 at BN = 128: acc + acc2 are 128 fp32 registers per thread under the 168-register cap of
  // a 384-thread CTA, so the epilogue spills a few hundred bytes; the fp32 parity mode is a
  // correctness mode, the bf16 path does not spill)
  // smem layout: fprop_smem
};

// byte offset of the bf16 pair (row r, column c, c even) of a staged half tile: sub-tiles of kSubW
// columns, rows of kSubW * 2 bytes in the TMA swizzle layout (16-byte piece j of row r at j ^ swz)
template <int kSubW>
__device__ __forceinline__ int staged_offset(int r, int c) {
  constexpr int kRowBytes = kSubW * 2;
  const int sub = c / kSubW, cb = (c % kSubW) * 2;
  const int swz = (kRowBytes == 128) ? (r & 7) : ((r >> 1) & 3);
  return sub * (kBM * kRowBytes) + r * kRowBytes + ((((cb >> 4) ^ swz)) << 4) + (cb & 15);
}

// One CTA per SM walks output tiles (fixed N tile, M tiles strided by the grid).  CG2: a cluster of
// two CTAs walks 256-row tiles (rank r computes rows r*128 ..) of one N tile; each CTA loads half of
// every weight stage and multicasts it to both, halving the weight traffic per tile.  The TMA producer
// runs ahead across tiles through the smem ring (it keeps loading the next tile's stages while the
// consumers run the epilogue); each consumer warpgroup accumulates 64 rows x BN in registers with
// wgmma, keeping one k-block of MMAs in flight, and releases a stage as soon as the MMAs that read
// it have completed.
// WG = consumer warpgroups: 2 = one 384-thread CTA per SM (warp 0 produces, warpgroup g computes rows
// 64g ..); 1 = two 160-thread CTAs per SM (warps 0..3 compute all 128 rows as two 64-row blocks,
// warp 4 produces), which lets the SM run one CTA's epilogue under the other's MMAs.
template <int BN, int CW, bool IM2COL, int NP, bool CG2, bool F16, int WG>
__global__ void __launch_bounds__(conv_threads(WG), WG == 2 ? 1 : 2)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAdd,
                 const __grid_constant__ CUtensorMap tmMask, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB1,
                 const __grid_constant__ CUtensorMap tmB2, const ConvGemmParams p) {
  using Cfg = FpropCfg<BN, NP, WG>;
  static_assert(WG == 2 || !CG2, "CTA pairs: two consumer warpgroups");
  constexpr int kChunks = kStageK / CW;        // A chunks (one filter tap each when Cin < 64)
  constexpr int kChunkBytes = kBM * CW * 2;
  constexpr int kKSteps = CW / 16;             // wgmma K = 16 bf16
  constexpr int kHalfN = Cfg::kHalfN;
  constexpr int kNHalf = Cfg::kNHalf;
  constexpr int kSubW = Cfg::kSubW;
  constexpr int kSubBytes = kBM * kSubW * 2;
  constexpr int kNSub = kHalfN / kSubW;
  constexpr int kConsThreads = 128 * WG;
  constexpr int kRB = 2 / WG;                  // 64-row accumulator blocks per consumer warpgroup
  constexpr int kProducerWarp = WG == 2 ? 0 : 4;

  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kMaxStages];
  __shared__ uint64_t empty_bar[kMaxStages];
  __shared__ uint64_t aux_bar;

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int kStages = p.stages;
  uint8_t* s_out = smem + kStages * Cfg::kStageBytes;
  uint8_t* s_add = s_out + (p.out_f32 ? 0 : Cfg::kTileBytes);
  uint8_t* s_mask = s_add + (p.has_add ? Cfg::kTileBytes : 0);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = (p.Ktot + kStageK - 1) / kStageK;
  // static tile schedule: this CTA (CG2: this CTA pair) owns N tile n_tile and M tiles m_first,
  // m_first + m_step, ...; with CG2 the CTA of rank r computes rows r*128 .. of each 256-row tile
  constexpr int kTileM = (CG2 ? 2 : 1) * kBM;
  const uint32_t cta_rank = CG2 ? cluster_ctarank() : 0u;
  const int unit = CG2 ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int units = CG2 ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
  const int n_tile = unit % p.n_tiles;
  const int m_first = unit / p.n_tiles;
  const int m_step = units / p.n_tiles;
  const int n0 = n_tile * BN;
  const int my_tiles = m_first < p.m_tiles ? (p.m_tiles - m_first + m_step - 1) / m_step : 0;
  const int m_rank_off = static_cast<int>(cta_rank) * kBM;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (NP == 3) {
      tma_prefetch_desc(&tmA1);
      tma_prefetch_desc(&tmA2);
      tma_prefetch_desc(&tmB1);
      tma_prefetch_desc(&tmB2);
    }
    if (!p.out_f32) tma_prefetch_desc(&tmC);
    if (p.has_add) tma_prefetch_desc(&tmAdd);
    if (p.has_mask) tma_prefetch_desc(&tmMask);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      // one arrival per consumer warp (CG2: of both CTAs -- the stage receives the peer's multicast)
      mbar_init(&empty_bar[s], 4 * WG * (CG2 ? 2 : 1));
    }
    mbar_init(&aux_bar, 1);
    fence_barrier_init();
  }
  if (CG2) cluster_sync();      // the peer's barriers are initialised before any multicast / arrive
  else __syncthreads();
  // everything above (barrier init, descriptor prefetch) overlapped the tail of the preceding
  // kernel; its outputs are read only after this point
  pdl_entry();

  const uint32_t smem_a0 = smem_u32(smem);
  const uint32_t full0 = smem_u32(full_bar), empty0 = smem_u32(empty_bar);
  // chunks of the last k-block (a partial stage exists only when a filter tap is narrower than
  // a stage, i.e. Cin < 64 with an odd tap count)
  const int tail_chunks = kChunks == 1 ? 1 : ((p.Ktot - (num_kb - 1) * kStageK + CW - 1) / CW);

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer
    // The whole warp stays converged and every lane tracks the same loop state; one elected lane
    // issues.
    uint32_t stage = 0, phase = 0;
    const uint32_t b_bytes = BN * (p.b_sw_bytes < 128 ? p.b_sw_bytes : 128);
    const uint32_t full_bytes = NP * (kChunks * kChunkBytes + b_bytes);
    const uint32_t tail_bytes = NP * (tail_chunks * kChunkBytes + b_bytes);
    const int Cin = p.Cin, fkw = p.kw;
    for (int it = 0; it < my_tiles; ++it) {
      const int m0 = (m_first + it * m_step) * kTileM + m_rank_off;
      int img = 0, h0 = 0, w0 = 0;
      if (IM2COL) {
        img = m0 / p.HoWo;
        const int rem = m0 - img * p.HoWo;
        const int po = rem / p.Wo;
        const int qo = rem - po * p.Wo;
        h0 = po * p.stride - p.pad_h_lo;
        w0 = qo * p.stride - p.pad_w_lo;
      }
      // filter tap (tr, ts) and channel offset tc of the next chunk, advanced incrementally
      int tr = 0, ts = 0, tc = 0, k0 = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        const bool last = kb == num_kb - 1;
        const int nch = (kChunks > 1 && last) ? tail_chunks : kChunks;
        mbar_wait_a(empty0 + stage * 8, phase ^ 1);
        const bool leader = elect_one();
        const uint32_t fb = full0 + stage * 8;
        const uint32_t sa = smem_a0 + stage * Cfg::kStageBytes;
        if (leader) {
          mbar_expect_tx_a(fb, (kChunks > 1 && last) ? tail_bytes : full_bytes);
          if (CG2) {      // this CTA's half of the weight rows, into both CTAs of the pair
            const int half = BN / 2;
            tma_load_2d_multicast(sa + NP * Cfg::kABytes + cta_rank * half * (b_bytes / BN), &tmB,
                                  fb, k0, n0 + static_cast<int>(cta_rank) * half, (uint16_t)3);
          } else {
#pragma unroll
            for (int pl = 0; pl < NP; ++pl)
              tma_load_2d_a(sa + NP * Cfg::kABytes + pl * Cfg::kBBytes,
                            pl == 0 ? &tmB : (pl == 1 ? &tmB1 : &tmB2), fb, k0, n0);
          }
        }
#pragma unroll
        for (int j = 0; j < kChunks; ++j) {
          if (j < nch) {
            if (leader) {
#pragma unroll
              for (int pl = 0; pl < NP; ++pl) {
                const CUtensorMap* mA = pl == 0 ? &tmA : (pl == 1 ? &tmA1 : &tmA2);
                const uint32_t dst = sa + pl * Cfg::kABytes + j * kChunkBytes;
                if (IM2COL)
                  tma_load_im2col_4d_a(dst, mA, fb, tc, w0, h0, img, (uint16_t)ts, (uint16_t)tr);
                else
                  tma_load_2d_a(dst, mA, fb, k0 + j * CW, m0);
              }
            }
            tc += CW;
            if (tc >= Cin) {
              tc = 0;
              if (++ts == fkw) { ts = 0; ++tr; }
            }
          }
        }
        __syncwarp();
        k0 += kStageK;
        if (++stage == static_cast<uint32_t>(kStages)) { stage = 0; phase ^= 1; }
      }
    }
  } else if (WG == 2 ? warp >= 4 : warp < 4) {
    // ------------------------------------------------------------------ wgmma consumers
    const int cg = WG == 2 ? (warp >> 2) - 1 : 0;      // consumer warpgroup: rows cg*64*kRB ..
    const int ct = static_cast<int>(threadIdx.x) - (WG == 2 ? 128 : 0);   // 0 .. kConsThreads-1
    const bool leader = ct == 0;
    const bool stats = p.ch_part != nullptr;
    const bool has_aux = p.has_add || p.has_mask;
    // fragment rows rb*64 + r0 and rb*64 + r0 + 8 of accumulator block rb
    const int r0 = cg * kRB * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = (lane & 3) * 2;                              // fragment column offset
    // descriptors of stage 0 / chunk 0 (K-major, 8-row groups SBO apart); this group's first 64
    // rows start cg*kRB*64 rows into every A chunk
    const uint64_t a_desc0 = make_smem_desc(smem_a0 + cg * kRB * 64 * CW * 2, 16, 8 * CW * 2,
                                            swizzle_layout_type(CW * 2));
    const uint64_t b_desc0 = make_smem_desc(smem_a0 + NP * Cfg::kABytes, 16, 8 * p.b_sw_bytes,
                                            swizzle_layout_type(p.b_sw_bytes));
    float acc[kRB][BN / 2];
    float acc2[NP == 3 ? BN / 2 : 1];
    // batch-norm statistics: thread t owns the 8 columns of 16-byte chunk `st_chunk` (of every
    // staged column group) over the rows st_rg, st_rg + kNRg, ... of every tile, read back from the
    // staged bf16 tile
    constexpr int kNChunk = kHalfN / 8;
    constexpr int kStatThreads = (BN == 32) ? 128 : kConsThreads;
    constexpr int kNRg = kStatThreads / kNChunk;       // row groups; kBM / kNRg rows per thread
    const bool st_on = ct < kStatThreads;
    const int st_chunk = ct % kNChunk, st_rg = ct / kNChunk;
    float acc_s[kNHalf][8], acc_q[kNHalf][8];
#pragma unroll
    for (int hf = 0; hf < kNHalf; ++hf)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc_s[hf][e] = acc_q[hf][e] = 0.f;
    uint32_t aux_n = 0;                                // completed aux-barrier phases
    // add / mask column groups are fetched ONE GROUP AHEAD: the loads of the next group are issued
    // as soon as every thread has consumed the current one (they overlap this group's TMA store,
    // the statistics pass and the next tile's k-loop)
    auto issue_aux = [&](int am0, int anh) {
      mbar_expect_tx(&aux_bar, (p.has_add ? Cfg::kTileBytes : 0) +
                                   (p.has_mask ? Cfg::kTileBytes : 0));
#pragma unroll
      for (int sub = 0; sub < kNSub; ++sub) {
        if (p.has_add)
          tma_load_2d(s_add + sub * kSubBytes, &tmAdd, &aux_bar, anh + sub * kSubW, am0);
        if (p.has_mask)
          tma_load_2d(s_mask + sub * kSubBytes, &tmMask, &aux_bar, anh + sub * kSubW, am0);
      }
    };
    if (leader && has_aux && my_tiles > 0) issue_aux(m_first * kTileM + m_rank_off, n0);
    // a stage is released to this CTA's producer and (CG2) to the peer's, whose multicast fills it too
    const uint32_t empty_peer = CG2 ? mapa_shared(empty0, cta_rank ^ 1u) : 0u;
    auto release = [&](int st) {
      if (CG2) {
        mbar_arrive_cluster(mapa_shared(empty0, cta_rank) + st * 8);
        mbar_arrive_cluster(empty_peer + st * 8);
      } else {
        mbar_arrive(&empty_bar[st]);
      }
    };
    auto fence_acc = [&]() {
#pragma unroll
      for (int rb = 0; rb < kRB; ++rb) wgmma_fence_operand(acc[rb]);
      if (NP == 3) wgmma_fence_operand(acc2);
    };
    // the MMAs of one k-block over its first N chunks as one straight-line wgmma group: a
    // data-dependent branch between the wgmmas of a group makes ptxas serialise them (C7520)
    auto mma_kblock = [&](auto n_chunks, uint32_t stage_off, uint32_t first_accum) {
      constexpr int kN = decltype(n_chunks)::value;
      fence_acc();
      wgmma_fence();
      const uint64_t da0 = a_desc0 + (stage_off >> 4);
      const uint64_t db0 = b_desc0 + (stage_off >> 4);
#pragma unroll
      for (int j = 0; j < kN; ++j) {
#pragma unroll
        for (int ks = 0; ks < kKSteps; ++ks) {
          // NP == 3: the six cross products of the (hi, mid, lo) planes that are significant
          // at fp32 precision, smallest first; t = 5 is hi*hi -> acc, t < 5 -> acc2
#pragma unroll
          for (int t = 0; t < (NP == 3 ? 6 : 1); ++t) {
            const int pa = NP == 3 ? plane_term_a(t) : 0;
            const int pb = NP == 3 ? plane_term_b(t) : 0;
            const bool small = NP == 3 && t < 5;
            const uint64_t db = db0 + ((pb * Cfg::kBBytes + (j * kKSteps + ks) * 32) >> 4);
            const uint32_t accum = (j | ks | (small ? t : 0)) ? 1u : first_accum;
#pragma unroll
            for (int rb = 0; rb < kRB; ++rb) {
              const uint64_t da =
                  da0 + ((pa * Cfg::kABytes + j * kChunkBytes + rb * 64 * CW * 2 + ks * 32) >> 4);
              if constexpr (NP == 3) {
                if (small) WgmmaOp<BN, F16>::type::template mma<0, 0>(acc2, da, db, accum);
                else WgmmaOp<BN, F16>::type::template mma<0, 0>(acc[rb], da, db, accum);
              } else {
                WgmmaOp<BN, F16>::type::template mma<0, 0>(acc[rb], da, db, accum);
              }
            }
          }
        }
      }
      wgmma_commit();
      fence_acc();
    };

    uint32_t stage = 0, phase = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int m0 = (m_first + it * m_step) * kTileM + m_rank_off;
      // ---- k-loop: one k-block of wgmma in flight; the stage before it is released
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        const bool last = kb == num_kb - 1;
        const int nch = (kChunks > 1 && last) ? tail_chunks : kChunks;
        mbar_wait_a(full0 + stage * 8, phase);
        const uint32_t stage_off = stage * Cfg::kStageBytes;
        const uint32_t first_accum = static_cast<uint32_t>(kb != 0);
        if (nch == kChunks) {
          mma_kblock(std::integral_constant<int, kChunks>{}, stage_off, first_accum);
        } else if constexpr (kChunks > 1) {     // the partial last k-block (Cin < 64, odd taps)
          if (nch == 1) {
            mma_kblock(std::integral_constant<int, 1>{}, stage_off, first_accum);
          } else if constexpr (kChunks > 2) {
            if (nch == 2) mma_kblock(std::integral_constant<int, 2>{}, stage_off, first_accum);
            else mma_kblock(std::integral_constant<int, 3>{}, stage_off, first_accum);
          }
        }
        wgmma_wait<1>();
        __syncwarp();
        if (prev >= 0 && lane == 0) release(prev);
        prev = static_cast<int>(stage);
        if (++stage == static_cast<uint32_t>(kStages)) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_acc();
      if (NP == 3) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[0][i] += acc2[i];
      }
      __syncwarp();
      if (lane == 0) release(prev);

      // ---- epilogue, per column group: (+bias) (+add) (x mask) -> bf16 -> swizzled staging ->
      // TMA store; statistics from the staged (rounded) tile
#pragma unroll
      for (int hf = 0; hf < kNHalf; ++hf) {
        const int nh = n0 + hf * kHalfN;               // first output column of this group
        // the TMA store that last used the staging buffer must have finished READING it
        if (leader && !p.out_f32) tma_store_wait_read();
        named_bar_sync(1, kConsThreads);
        if (has_aux) {
          mbar_wait(&aux_bar, aux_n & 1);
          ++aux_n;
        }
#pragma unroll
        for (int jj = 0; jj < kHalfN / 8; ++jj) {
          const int j = hf * (kHalfN / 8) + jj;
          const int c = jj * 8 + cq;                   // column inside the group
          float b0 = 0.f, b1 = 0.f;
          if (p.bias) {
            b0 = __ldg(p.bias + nh + c);
            b1 = __ldg(p.bias + nh + c + 1);
          }
#pragma unroll
          for (int rb = 0; rb < kRB; ++rb)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + rb * 64 + h * 8;
            float v0 = acc[rb][j * 4 + h * 2] + b0, v1 = acc[rb][j * 4 + h * 2 + 1] + b1;
            const int off = staged_offset<kSubW>(r, c);
            if (p.has_add) x2_add<F16>(v0, v1, *reinterpret_cast<const uint32_t*>(s_add + off));
            // ReLU mask of the destination tensor: 0xffff per bf16 half that is > 0, applied to the
            // packed bf16 output (zeroing the half == zeroing the fp32 value before rounding)
            if (p.out_f32) {
              if (p.has_mask) {
                const uint32_t k2 = x2_gt0_mask<F16>(*reinterpret_cast<const uint32_t*>(s_mask + off));
                if (!(k2 & 0xffffu)) v0 = 0.f;
                if (!(k2 >> 16)) v1 = 0.f;
              }
              if (m0 + r < p.M)
                *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.y) +
                                           static_cast<size_t>(m0 + r) * p.Cout + nh + c) =
                    make_float2(v0, v1);
            } else {
              uint32_t pk = pack_x2<F16>(v0, v1);
              if (p.has_mask) pk &= x2_gt0_mask<F16>(*reinterpret_cast<const uint32_t*>(s_mask + off));
              *reinterpret_cast<uint32_t*>(s_out + off) = pk;
            }
          }
        }
        if (!p.out_f32) fence_proxy_async();             // generic smem writes -> async proxy
        named_bar_sync(1, kConsThreads);
        if (leader) {
          if (!p.out_f32) {
#pragma unroll
            for (int sub = 0; sub < kNSub; ++sub)
              tma_store_2d(&tmC, s_out + sub * kSubBytes, nh + sub * kSubW, m0);
            tma_store_commit();
          }
          if (has_aux) {
            // the staging tiles were consumed by everyone before the barrier above: fetch the next
            // group's (same rows / next columns, else the next M tile of this CTA)
            if (hf + 1 < kNHalf) issue_aux(m0, nh + kHalfN);
            else if (it + 1 < my_tiles) issue_aux((m_first + (it + 1) * m_step) * kTileM + m_rank_off, n0);
          }
        }
        if (stats && st_on) {
          // column sums of the group as stored (bf16-rounded); rows past M were computed
          // from zero-filled operands and contribute zero.  Overlaps the TMA store (both read).
          constexpr int kRowBytes = kSubW * 2;
          const int sub = st_chunk / (kSubW / 8), jj = st_chunk % (kSubW / 8);
#pragma unroll 4
          for (int i = 0; i < kBM / kNRg; ++i) {
            const int rr = st_rg + i * kNRg;
            const int sw = (kRowBytes == 128) ? (rr & 7) : ((rr >> 1) & 3);
            const uint4 u = *reinterpret_cast<const uint4*>(s_out + sub * kSubBytes +
                                                            rr * kRowBytes + ((jj ^ sw) << 4));
            const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
              x2_sum_sq<F16>(acc_s[hf][2 * e], acc_q[hf][2 * e], acc_s[hf][2 * e + 1],
                            acc_q[hf][2 * e + 1], w4[e]);
          }
        }
      }
    }
    if (leader && !p.out_f32) tma_store_wait_all();
    if (stats && my_tiles > 0) {
      // final cross-row-group reduction in the (now idle) output staging buffer
      float* red_sum = reinterpret_cast<float*>(s_out);
      float* red_sq = red_sum + kNRg * BN;
      static_assert(2 * kNRg * BN * 4 <= Cfg::kTileBytes, "staging buffer too small for stats");
      named_bar_sync(1, kConsThreads);                 // the last TMA store has drained
      if (st_on) {
#pragma unroll
        for (int hf = 0; hf < kNHalf; ++hf)
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            red_sum[st_rg * BN + hf * kHalfN + st_chunk * 8 + e] = acc_s[hf][e];
            red_sq[st_rg * BN + hf * kHalfN + st_chunk * 8 + e] = acc_q[hf][e];
          }
      }
      named_bar_sync(1, kConsThreads);
      for (int col = ct; col < BN; col += kConsThreads) {
        float ss = 0.f, qq = 0.f;
        for (int g2 = 0; g2 < kNRg; ++g2) {
          ss += red_sum[g2 * BN + col];
          qq += red_sq[g2 * BN + col];
        }
        // one partial row per CTA of this N tile, plain stores: bn_finalize sums the rows in a
        // fixed order (deterministic; no pre-zeroed accumulator)
        float* row = p.ch_part +
                     static_cast<size_t>(CG2 ? m_first * 2 + static_cast<int>(cta_rank) : m_first) * 2 *
                         p.Cout;
        row[n0 + col] = ss;
        row[p.Cout + n0 + col] = qq;
      }
    }
  }
  // CG2: neither CTA leaves while the peer may still multicast into it or arrive on its barriers
  if (CG2) cluster_sync();
}

// ------------------------------------------------------------------------------------------
// 3x3 / stride 1 / pad 1 convolution WITHOUT im2col copies ("halo" kernel).
//
// The im2col kernel fetches every input pixel nine times (once per filter tap) from L2 into shared
// memory.  Here a CTA tile is a 16 x 8 PATCH of output pixels of one image, and ONE 18 x 10 pixel halo
// tile per channel chunk is loaded by a 4-D tiled TMA box at (h0-1, w0-1) (out-of-image pixels are
// zero-filled: the padding).  The A operand of filter tap (r, s) is the same shared-memory tile read
// through a wgmma descriptor that starts (r*10 + s) pixel rows further on, with 10 pixel rows between
// 8-row groups (group g = output row h0+g, 8 pixels): the swizzle is a function of the absolute
// shared-memory address (as for TMA), so any row may start a descriptor and the group stride need
// not be a multiple of the swizzle atom.  Consumer warpgroup g covers output rows 8g .. 8g+7.
// Weight tiles [BN x CW] per (tap, chunk) stream through their own ring; when the whole N-tile slab
// fits the ring it is loaded once and stays (weights-stationary).
// Epilogue = the im2col kernel's (add / mask one tile ahead, bf16 staging, TMA store, statistics),
// with 4-D boxes for the patch and the out-of-image rows excluded from the statistics.
// ------------------------------------------------------------------------------------------
constexpr int kHaloH = 18, kHaloW = 10, kPatchH = 16, kPatchW = 8;
constexpr int kHaloMaxB = 32;      // weight ring slots (barriers)

struct HaloParams {
  int H, W, B;            // output = input spatial size
  int Cin, Cout;
  int n_tiles, ph, pw;    // N tiles; patches per image
  int m_tiles;            // B * ph * pw
  int a_stages, b_slots, stationary;
  float* ch_part;
  int has_add, has_mask;
};

template <int BN, int CW>
struct HaloCfg {
  static constexpr int kRowB = CW * 2;
  static constexpr int kABytes = kHaloH * kHaloW * kRowB;
  static constexpr int kAStage = (kABytes + 1023) / 1024 * 1024;
  static constexpr int kBTile = BN * kRowB;
  static constexpr int kSubW = BN < 64 ? BN : 64;
  static constexpr int kTileBytes = kBM * BN * 2;
  static_assert(BN <= 128 && kBTile % 512 == 0, "halo kernel: N tile <= 128");
};

// Patch coordinates of the tiles first, first + step, ... advanced without divisions.
struct PatchIter {
  int img, row, col;          // image, patch row / column inside the image
  int d_img, d_row, d_col;
  int ph, pw;
  __device__ __forceinline__ PatchIter(int first, int step, int ph_, int pw_) : ph(ph_), pw(pw_) {
    const int tpi = ph * pw;
    img = first / tpi;
    int rem = first - img * tpi;
    row = rem / pw;
    col = rem - row * pw;
    d_img = step / tpi;
    rem = step - d_img * tpi;
    d_row = rem / pw;
    d_col = rem - d_row * pw;
  }
  __device__ __forceinline__ void next() {
    col += d_col;
    if (col >= pw) { col -= pw; ++row; }
    row += d_row;
    if (row >= ph) { row -= ph; ++img; }
    img += d_img;
  }
};

template <int BN, int CW, bool F16>
__global__ void __launch_bounds__(kThreads, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAdd,
                 const __grid_constant__ CUtensorMap tmMask, const HaloParams p) {
  using Cfg = HaloCfg<BN, CW>;
  constexpr int kRowB = Cfg::kRowB;
  constexpr int kKSteps = CW / 16;
  constexpr uint32_t kLayout = swizzle_layout_type(kRowB);
  constexpr int kSubW = Cfg::kSubW;
  constexpr int kSubBytes = kBM * kSubW * 2;
  constexpr int kNSub = BN / kSubW;

  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t a_full[4], a_empty[4];
  __shared__ uint64_t b_full[kHaloMaxB], b_empty[kHaloMaxB];
  __shared__ uint64_t aux_bar;

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int AS = p.a_stages, NB = p.b_slots;
  uint8_t* s_out = smem + AS * Cfg::kAStage + NB * Cfg::kBTile;
  uint8_t* s_add = s_out + Cfg::kTileBytes;
  uint8_t* s_mask = s_add + (p.has_add ? Cfg::kTileBytes : 0);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nchunks = p.Cin / CW;
  const int n_tile = blockIdx.x % p.n_tiles;
  const int m_first = blockIdx.x / p.n_tiles;
  const int m_step = gridDim.x / p.n_tiles;
  const int n0 = n_tile * BN;
  const int my_tiles = m_first < p.m_tiles ? (p.m_tiles - m_first + m_step - 1) / m_step : 0;
  const int tpi = p.ph * p.pw;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
    if (p.has_add) tma_prefetch_desc(&tmAdd);
    if (p.has_mask) tma_prefetch_desc(&tmMask);
    for (int s = 0; s < AS; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], kConsumerWarps);
    }
    for (int s = 0; s < NB; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], kConsumerWarps);
    }
    mbar_init(&aux_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_entry();
  const uint32_t a_base = smem_u32(smem), b_base = a_base + AS * Cfg::kAStage;
  const uint32_t afull0 = smem_u32(a_full), bfull0 = smem_u32(b_full);

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    const uint32_t aempty0 = smem_u32(a_empty), bempty0 = smem_u32(b_empty);
    uint32_t sa = 0, a_ph = 0, sb = 0, b_ph = 0;
    if (p.stationary && my_tiles > 0) {
      // the whole weight slab of this N tile: loaded once, ONE barrier, stays for the CTA's lifetime
      if (elect_one()) {
        mbar_expect_tx_a(bfull0, static_cast<uint32_t>(nchunks) * 9 * Cfg::kBTile);
        for (int kc = 0; kc < nchunks; ++kc)
          for (int t = 0; t < 9; ++t)
            tma_load_2d_a(b_base + (kc * 9 + t) * Cfg::kBTile, &tmB, bfull0, t * p.Cin + kc * CW, n0);
      }
      __syncwarp();
    }
    for (int it = 0; it < my_tiles; ++it) {
      const int tile = m_first + it * m_step;
      const int img = tile / tpi;
      const int rem = tile - img * tpi;
      const int h0 = (rem / p.pw) * kPatchH, w0 = (rem % p.pw) * kPatchW;
      for (int kc = 0; kc < nchunks; ++kc) {
        mbar_wait_a(aempty0 + sa * 8, a_ph ^ 1);
        if (elect_one()) {
          mbar_expect_tx_a(afull0 + sa * 8, Cfg::kABytes);
          tma_load_4d_tile_a(a_base + sa * Cfg::kAStage, &tmA, afull0 + sa * 8, kc * CW, w0 - 1,
                             h0 - 1, img);
        }
        __syncwarp();
        if (++sa == static_cast<uint32_t>(AS)) { sa = 0; a_ph ^= 1; }
        if (!p.stationary) {
          for (int t = 0; t < 9; ++t) {
            mbar_wait_a(bempty0 + sb * 8, b_ph ^ 1);
            if (elect_one()) {
              mbar_expect_tx_a(bfull0 + sb * 8, Cfg::kBTile);
              tma_load_2d_a(b_base + sb * Cfg::kBTile, &tmB, bfull0 + sb * 8, t * p.Cin + kc * CW,
                            n0);
            }
            __syncwarp();
            if (++sb == static_cast<uint32_t>(NB)) { sb = 0; b_ph ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ wgmma consumers
    const int cg = (warp >> 2) - 1;                    // output rows 8cg .. 8cg+7 of the patch
    const int ct = static_cast<int>(threadIdx.x) - 128;
    const bool leader = ct == 0;
    const bool stats = p.ch_part != nullptr;
    const bool has_aux = p.has_add || p.has_mask;
    const int r0 = cg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows r0, r0 + 8
    const int cq = (lane & 3) * 2;
    const uint64_t a_desc0 = make_smem_desc(a_base + cg * 8 * kHaloW * kRowB, 16, kHaloW * kRowB, kLayout);
    const uint64_t b_desc0 = make_smem_desc(b_base, 16, 8 * kRowB, kLayout);
    float acc[BN / 2];
    constexpr int kNChunk = BN / 8;
    constexpr int kStatThreads = (BN == 32) ? 128 : kConsumerThreads;
    constexpr int kNRg = kStatThreads / kNChunk;
    const bool st_on = ct < kStatThreads;
    const int st_chunk = ct % kNChunk, st_rg = ct / kNChunk;
    float acc_s[8], acc_q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc_s[e] = acc_q[e] = 0.f;
    uint32_t aux_n = 0;
    auto issue_aux = [&](int img, int h0, int w0) {
      mbar_expect_tx(&aux_bar, (p.has_add ? Cfg::kTileBytes : 0) + (p.has_mask ? Cfg::kTileBytes : 0));
#pragma unroll
      for (int sub = 0; sub < kNSub; ++sub) {
        if (p.has_add)
          tma_load_4d_tile_a(smem_u32(s_add + sub * kSubBytes), &tmAdd, smem_u32(&aux_bar),
                             n0 + sub * kSubW, w0, h0, img);
        if (p.has_mask)
          tma_load_4d_tile_a(smem_u32(s_mask + sub * kSubBytes), &tmMask, smem_u32(&aux_bar),
                             n0 + sub * kSubW, w0, h0, img);
      }
    };
    // resources read by the most recent committed wgmma group, released once it has completed
    int pend_a = -1, pend_b = -1;
    auto release_pending = [&]() {
      __syncwarp();
      if (lane == 0) {
        if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
        if (pend_b >= 0) mbar_arrive(&b_empty[pend_b]);
      }
      pend_a = pend_b = -1;
    };
    PatchIter pi(m_first, m_step, p.ph, p.pw);
    if (leader && has_aux && my_tiles > 0) issue_aux(pi.img, pi.row * kPatchH, pi.col * kPatchW);
    if (p.stationary && my_tiles > 0) mbar_wait_a(bfull0, 0);
    uint32_t sa = 0, a_ph = 0, sb = 0, b_ph = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int img = pi.img, h0 = pi.row * kPatchH, w0 = pi.col * kPatchW;
      pi.next();
      for (int kc = 0; kc < nchunks; ++kc) {
        mbar_wait_a(afull0 + sa * 8, a_ph);
        const uint64_t a_st = a_desc0 + ((sa * Cfg::kAStage) >> 4);
        if (p.stationary) {
          wgmma_fence_operand(acc);
          wgmma_fence();
          const uint64_t b_st = b_desc0 + ((static_cast<uint32_t>(kc) * 9 * Cfg::kBTile) >> 4);
#pragma unroll
          for (int t = 0; t < 9; ++t)
#pragma unroll
            for (int ks = 0; ks < kKSteps; ++ks)
              WgmmaOp<BN, F16>::type::template mma<0, 0>(
                  acc, a_st + ((((t / 3) * kHaloW + (t % 3)) * kRowB + ks * 32) >> 4),
                  b_st + ((t * Cfg::kBTile + ks * 32) >> 4), (t | ks) ? 1u : static_cast<uint32_t>(kc != 0));
          wgmma_commit();
          wgmma_fence_operand(acc);
          wgmma_wait<1>();
          release_pending();
          pend_a = static_cast<int>(sa);
        } else {
#pragma unroll 1
          for (int t = 0; t < 9; ++t) {
            mbar_wait_a(bfull0 + sb * 8, b_ph);
            wgmma_fence_operand(acc);
            wgmma_fence();
            const uint64_t a_tap = a_st + ((((t / 3) * kHaloW + (t % 3)) * kRowB) >> 4);
            const uint64_t b_tap = b_desc0 + ((sb * Cfg::kBTile) >> 4);
#pragma unroll
            for (int ks = 0; ks < kKSteps; ++ks)
              WgmmaOp<BN, F16>::type::template mma<0, 0>(acc, a_tap + ((ks * 32) >> 4), b_tap + ((ks * 32) >> 4),
                                            (kc | t | ks) ? 1u : 0u);
            wgmma_commit();
            wgmma_fence_operand(acc);
            wgmma_wait<1>();
            release_pending();
            pend_b = static_cast<int>(sb);
            if (t == 8) pend_a = static_cast<int>(sa);
            if (++sb == static_cast<uint32_t>(NB)) { sb = 0; b_ph ^= 1; }
          }
        }
        if (++sa == static_cast<uint32_t>(AS)) { sa = 0; a_ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      release_pending();

      // ---- epilogue: (+add) (x mask) -> bf16 -> swizzled staging -> 4-D TMA store; statistics
      if (leader) tma_store_wait_read();
      named_bar_sync(1, kConsumerThreads);
      if (has_aux) {
        mbar_wait(&aux_bar, aux_n & 1);
        ++aux_n;
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = j * 8 + cq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + h * 8;
          float v0 = acc[j * 4 + h * 2], v1 = acc[j * 4 + h * 2 + 1];
          const int off = staged_offset<kSubW>(r, c);
          if (p.has_add) x2_add<F16>(v0, v1, *reinterpret_cast<const uint32_t*>(s_add + off));
          uint32_t pk = pack_x2<F16>(v0, v1);
          if (p.has_mask) pk &= x2_gt0_mask<F16>(*reinterpret_cast<const uint32_t*>(s_mask + off));
          *reinterpret_cast<uint32_t*>(s_out + off) = pk;
        }
      }
      fence_proxy_async();
      named_bar_sync(1, kConsumerThreads);
      if (leader) {
#pragma unroll
        for (int sub = 0; sub < kNSub; ++sub)
          tma_store_4d(&tmC, s_out + sub * kSubBytes, n0 + sub * kSubW, w0, h0, img);
        tma_store_commit();
        if (has_aux && it + 1 < my_tiles) issue_aux(pi.img, pi.row * kPatchH, pi.col * kPatchW);
      }
      if (stats && st_on) {
        // column sums of the tile as stored (bf16-rounded); patch pixels outside the image excluded
        // (they were computed from real neighbours and are clipped by the store)
        constexpr int kRowBytes = kSubW * 2;
        const int sub = st_chunk / (kSubW / 8), jj = st_chunk % (kSubW / 8);
#pragma unroll 4
        for (int rr = st_rg; rr < kBM; rr += kNRg) {
          if (h0 + (rr >> 3) >= p.H || w0 + (rr & 7) >= p.W) continue;
          const int sw = (kRowBytes == 128) ? (rr & 7) : ((rr >> 1) & 3);
          const uint4 u = *reinterpret_cast<const uint4*>(s_out + sub * kSubBytes + rr * kRowBytes +
                                                          ((jj ^ sw) << 4));
          const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
            x2_sum_sq<F16>(acc_s[2 * e], acc_q[2 * e], acc_s[2 * e + 1], acc_q[2 * e + 1], w4[e]);
        }
      }
    }
    if (leader) tma_store_wait_all();
    if (stats && my_tiles > 0) {
      float* red_sum = reinterpret_cast<float*>(s_out);
      float* red_sq = red_sum + kNRg * BN;
      static_assert(2 * kNRg * BN * 4 <= Cfg::kTileBytes, "staging buffer too small for stats");
      named_bar_sync(1, kConsumerThreads);
      if (st_on) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          red_sum[st_rg * BN + st_chunk * 8 + e] = acc_s[e];
          red_sq[st_rg * BN + st_chunk * 8 + e] = acc_q[e];
        }
      }
      named_bar_sync(1, kConsumerThreads);
      for (int col = ct; col < BN; col += kConsumerThreads) {
        float ss = 0.f, qq = 0.f;
        for (int g2 = 0; g2 < kNRg; ++g2) {
          ss += red_sum[g2 * BN + col];
          qq += red_sq[g2 * BN + col];
        }
        float* row = p.ch_part + static_cast<size_t>(m_first) * 2 * p.Cout;
        row[n0 + col] = ss;
        row[p.Cout + n0 + col] = qq;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// wgrad kernel:  D[(tap,ci) = M 128 rows][co = N] += sum over pixels of  x_im2col^T * dy
// ------------------------------------------------------------------------------------------
struct WgradParams {
  int P;           // pixels B*Ho*Wo (GEMM K)
  int Cout;        // GEMM N
  int Cin;
  int Ktot;        // kh*kw*Cin (GEMM M)
  int kw;
  int HoWo, Wo;
  int stride, pad_h_lo, pad_w_lo;
  int pix;               // pixels per stage (64 or 128)
  int stages_total;      // ceil(P / pix)
  int stages_per_split;
  int splits;            // CTAs along the pixel range (gridDim.z)
  float* dw;
  float* part;           // splits > 1: [splits][Cout][Ktot] fp32 partials (dw order), else null
};

constexpr int kWgPix = 64;   // default pixels per pipeline stage (4 wgmma K-steps); PIX = 128: 8 steps

// PIX = pixels (GEMM K) per pipeline stage: 64, or 128 (twice the MMAs per TMA / barrier round trip)
template <int BN, int NP = 1, int PIX = kWgPix>
struct WgradCfg {
  static constexpr int kABytes = PIX * 128 * 2;   // PIX pixels x 128 (tap,ci) columns, one plane
  static constexpr int kBBytes = PIX * BN * 2;    // PIX pixels x BN output channels, one plane
  static constexpr int kStageBytes = NP * (kABytes + kBBytes);
  static constexpr int kStagesFit = (kSmemBudget - 1024) / kStageBytes;
  static constexpr int kStages =
      PIX != kWgPix ? (kStagesFit > 4 ? 4 : kStagesFit)
      : NP == 3 ? (kStagesFit > 3 ? 3 : kStagesFit)
              : ((BN >= 256) ? 4 : ((BN == 128) ? 3 : 4));
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024;
  static_assert((NP == 1 || BN <= 128) && kStages >= (NP == 3 ? 2 : 3), "wgrad tile does not fit");
};

// CW: channel width of one im2col chunk of x (16/32/64), CWB: channel width of one dy chunk.
// Both operands are MN-major in shared memory (the pixel index is the GEMM K dimension): one pixel
// row = width*2 bytes, 8-row groups SBO apart, column blocks (64/32/16 channels) LBO apart.
template <int BN, int CW, int CWB, bool IM2COL, int NP, int PIX, bool F16>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_gemm_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmDY,
                  const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                  const __grid_constant__ CUtensorMap tmDY1,
                  const __grid_constant__ CUtensorMap tmDY2, const WgradParams p) {
  using Cfg = WgradCfg<BN, NP, PIX>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kAChunks = 128 / CW;
  constexpr int kAChunkBytes = PIX * CW * 2;
  constexpr int kBChunkBytes = PIX * CWB * 2;

  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[kStages];
  __shared__ uint64_t empty_bar[kStages];

  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * 128;          // first (tap,ci) column of dw handled here
  const int co0 = blockIdx.y * BN;
  const int ks_begin = blockIdx.z * p.stages_per_split;
  int ks_end = ks_begin + p.stages_per_split;
  if (ks_end > p.stages_total) ks_end = p.stages_total;
  const int num_ks = ks_end - ks_begin;   // >= 1 by construction of the grid

  int a_chunks = 0;
#pragma unroll
  for (int j = 0; j < kAChunks; ++j) a_chunks += (m0 + j * CW < p.Ktot) ? 1 : 0;
  const int b_chunks = (p.Cout - co0 < BN ? p.Cout - co0 : BN) / CWB;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // everything above (barrier init, descriptor prefetch) overlapped the tail of the preceding
  // kernel; its outputs are read only after this point
  pdl_entry();

  if (warp == 0) {
    // whole warp converged, one elected lane issues (no election loops around TMA instructions)
    int stage = 0;
    uint32_t phase = 0;
    // (tap r, tap s, channel) of each A chunk of this CTA: fixed for the whole kernel
    int ch_r[kAChunks], ch_s[kAChunks], ch_c[kAChunks];
#pragma unroll
    for (int j = 0; j < kAChunks; ++j) {
      const int n = m0 + j * CW;
      const int tap = n / p.Cin;
      ch_c[j] = n - tap * p.Cin;
      ch_r[j] = tap / p.kw;
      ch_s[j] = tap - ch_r[j] * p.kw;
    }
    for (int it = 0; it < num_ks; ++it) {
      const int p0 = (ks_begin + it) * PIX;
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (elect_one()) {
        uint8_t* sa = smem + stage * Cfg::kStageBytes;
        uint8_t* sb = sa + NP * Cfg::kABytes;
        mbar_expect_tx(&full_bar[stage], NP * (a_chunks * kAChunkBytes + b_chunks * kBChunkBytes));
        int img = 0, h0 = 0, w0 = 0;
        if (IM2COL) {
          img = p0 / p.HoWo;
          const int rem = p0 - img * p.HoWo;
          const int po = rem / p.Wo;
          const int qo = rem - po * p.Wo;
          h0 = po * p.stride - p.pad_h_lo;
          w0 = qo * p.stride - p.pad_w_lo;
        }
#pragma unroll
        for (int pl = 0; pl < NP; ++pl) {
          const CUtensorMap* mX = pl == 0 ? &tmX : (pl == 1 ? &tmX1 : &tmX2);
          const CUtensorMap* mDY = pl == 0 ? &tmDY : (pl == 1 ? &tmDY1 : &tmDY2);
#pragma unroll
          for (int j = 0; j < kAChunks; ++j) {
            if (j < a_chunks) {
              uint8_t* dst = sa + pl * Cfg::kABytes + j * kAChunkBytes;
              if (IM2COL) {
                tma_load_im2col_4d(dst, mX, &full_bar[stage], ch_c[j], w0, h0, img,
                                   (uint16_t)ch_s[j], (uint16_t)ch_r[j]);
              } else {
                tma_load_2d(dst, mX, &full_bar[stage], ch_c[j], p0);
              }
            }
          }
          for (int i = 0; i < b_chunks; ++i)
            tma_load_2d(sb + pl * Cfg::kBBytes + i * kBChunkBytes, mDY, &full_bar[stage],
                        co0 + i * CWB, p0);
        }
      }
      __syncwarp();
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
  } else if (warp >= 4) {
    // consumer warpgroup cg: rows (tap,ci) cg*64 .. of the 128, i.e. A chunks from cg*64/CW on
    const int cg = (warp >> 2) - 1;
    const uint32_t sbase = smem_u32(smem);
    const uint64_t a_desc0 = make_smem_desc(sbase + (cg * 64 / CW) * kAChunkBytes, kAChunkBytes,
                                            8 * CW * 2, swizzle_layout_type(CW * 2));
    const uint64_t b_desc0 = make_smem_desc(sbase + NP * Cfg::kABytes, kBChunkBytes, 8 * CWB * 2,
                                            swizzle_layout_type(CWB * 2));
    float acc[BN / 2];
    float acc2[NP == 3 ? BN / 2 : 1];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int it = 0; it < num_ks; ++it) {
      mbar_wait(&full_bar[stage], phase);
      wgmma_fence_operand(acc);
      if (NP == 3) wgmma_fence_operand(acc2);
      wgmma_fence();
      const uint64_t da0 = a_desc0 + static_cast<uint64_t>(stage * (Cfg::kStageBytes >> 4));
      const uint64_t db0 = b_desc0 + static_cast<uint64_t>(stage * (Cfg::kStageBytes >> 4));
#pragma unroll
      for (int ks = 0; ks < PIX / 16; ++ks) {
#pragma unroll
        for (int t = 0; t < (NP == 3 ? 6 : 1); ++t) {
          const int pa = NP == 3 ? plane_term_a(t) : 0;
          const int pb = NP == 3 ? plane_term_b(t) : 0;
          const bool small = NP == 3 && t < 5;
          const uint64_t da = da0 + ((pa * Cfg::kABytes + ks * 16 * CW * 2) >> 4);
          const uint64_t db = db0 + ((pb * Cfg::kBBytes + ks * 16 * CWB * 2) >> 4);
          const uint32_t accum = (it | ks | (small ? t : 0)) ? 1u : 0u;
          if constexpr (NP == 3) {
            if (small) WgmmaOp<BN, F16>::type::template mma<1, 1>(acc2, da, db, accum);
            else WgmmaOp<BN, F16>::type::template mma<1, 1>(acc, da, db, accum);
          } else {
            WgmmaOp<BN, F16>::type::template mma<1, 1>(acc, da, db, accum);
          }
        }
      }
      wgmma_commit();
      wgmma_fence_operand(acc);
      if (NP == 3) wgmma_fence_operand(acc2);
      wgmma_wait<1>();
      __syncwarp();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);
    if (NP == 3) {
      wgmma_fence_operand(acc2);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] += acc2[i];
    }
    // fragment row = (tap,ci) column n of dw, fragment column = output channel
    const int rl = cg * 64 + (warp & 3) * 16 + (lane >> 2);   // row inside the 128-row tile
    const int rb = m0 + rl;
    const int cq = (lane & 3) * 2;
    // split-K: this split's partial goes to its own slice in dw order, summed in split order by
    // wgrad_reduce_kernel.  Either way a warp's store covers 8 consecutive (tap,ci) rows of 4
    // output channels: four full 32-byte sectors.
    float* part = p.part ? p.part + static_cast<size_t>(blockIdx.z) * p.Cout * p.Ktot : nullptr;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = rb + h * 8;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int co = co0 + j * 8 + cq + e;
          if (n < p.Ktot && co < p.Cout) {
            const size_t i = static_cast<size_t>(co) * p.Ktot + n;
            if (part) part[i] = acc[j * 4 + h * 2 + e];
            // one add per dw element (the whole pixel range of this tile is summed above)
            else atomicAdd(p.dw + i, acc[j * 4 + h * 2 + e]);
          }
        }
      }
    }
  }
}

// dw[i] += (((0 + part[0][i]) + part[1][i]) + ... + part[splits-1][i]): the ordered split-K sum,
// one dw element per thread over the whole GPU.  Loads are issued kWgRedDepth splits ahead of the
// (serial) adds so that each thread keeps that many L2 reads in flight.
constexpr int kWgRedThreads = 128;
constexpr int kWgRedDepth = 16;

__global__ void __launch_bounds__(kWgRedThreads)
wgrad_reduce_kernel(const float* __restrict__ part, float* dw, int64_t n, int splits) {
  pdl_entry();
  const int64_t i = blockIdx.x * static_cast<int64_t>(kWgRedThreads) + threadIdx.x;
  if (i >= n) return;
  const float* src = part + i;
  float t = 0.f;
  int s = 0;
  for (; s + kWgRedDepth <= splits; s += kWgRedDepth) {
    float v[kWgRedDepth];
#pragma unroll
    for (int u = 0; u < kWgRedDepth; ++u) v[u] = __ldcs(src + (s + u) * n);
#pragma unroll
    for (int u = 0; u < kWgRedDepth; ++u) t += v[u];
  }
  for (; s < splits; ++s) t += __ldcs(src + s * n);
  dw[i] += t;
}

// ------------------------------------------------------------------------------------------
// Host launchers
// ------------------------------------------------------------------------------------------
struct ConvMaps {
  CUtensorMap a[3], b[3], c, add, mask;
};

// Epilogue / tiling knobs of the C ABI from earlier kernel generations.  The sm_90 kernels have one
// epilogue organisation (the consumer warpgroups drain their own registers) and one 128-pixel M
// tile per CTA: these setters keep and return their value and change nothing.
static int g_conv_out_bufs = 1;
static int g_conv_split_epi = 1;
static int g_conv_split_mt2 = 1;
static int g_conv_mtiles_mode = -1;
// epilogue organisation of an earlier kernel generation: the sm_90 halo kernel has one (the
// consumer warpgroups drain their registers); acnn_set_conv_halo_split keeps and returns the value
static int g_conv_halo_split = 1;
// CTA pairs (clusters of two sharing the weight stages by TMA multicast): 1 = the N = 128 tiles with
// K >= 512 and enough tiles for every SM; 0 (default) = single CTAs (acnn_set_conv_cta_pairs).  Off
// by default: c3 step on an H100 SXM at 700 W, 80.3 ms with pairs against 61.3 ms without
static int g_conv_pairs = 0;
// Two CTAs per SM only up to this GEMM K (kh*kw*Cin): there the per-tile fixed cost (pipeline fill,
// epilogue) rivals the MMAs and overlapping it pays; on deeper K the 128 x 64 tiles' extra operand
// traffic from L2 costs more (c3 step on an H100 SXM at 700 W, fprop + dgrad launches: K <= 512
// 10.9 -> 9.5 ms; K = 576 .. 1024 unchanged; K >= 1152 6.2 -> 7.7 ms)
constexpr int kTwoCtaMaxK = 512;
// halo (im2col-free 3x3) kernel: 0: off; 1 (default): where the weight slab stays in shared memory
// and the images are large (the mode 1 rule of conv_choice; c3 step on an H100 SXM at 700 W: 59.8 ms
// against 61.3 ms with 0); 2: wherever the kernel applies (acnn_set_conv_halo)
static int g_conv_halo = 1;

static int chunk_width(int cin) { return cin % 64 == 0 ? 64 : (cin % 32 == 0 ? 32 : 16); }

static int out_hw(const acnn_conv_geom& g, int* Ho, int* Wo) {
  *Ho = (g.H + g.pad_h_lo + g.pad_h_hi - g.kh) / g.stride + 1;
  *Wo = (g.W + g.pad_w_lo + g.pad_w_hi - g.kw) / g.stride + 1;
  return (*Ho > 0 && *Wo > 0) ? 1 : 0;
}

// elements of the input tensor (one operand plane)
static int64_t input_elems(const acnn_conv_geom& g) {
  int64_t pix, row, img;
  input_pitches(g, &pix, &row, &img);
  return (int64_t)g.B * img;
}

// Shared-memory plan of the halo kernel for one problem (a pure function of the shape).
struct HaloPlan {
  int a_stages, b_slots, stationary, smem;
};

static HaloPlan halo_plan(int bn, int cw, int Cin, bool has_add, bool has_mask) {
  HaloPlan h;
  const int row_b = cw * 2;
  const int a_stage = (kHaloH * kHaloW * row_b + 1023) / 1024 * 1024;
  const int b_tile = bn * row_b;
  const int tile = kBM * bn * 2;
  const int nchunks = Cin / cw;
  const int fixed = 1024 + tile * (1 + (has_add ? 1 : 0) + (has_mask ? 1 : 0));
  h.a_stages = 3;
  h.b_slots = (kSmemBudget - fixed - h.a_stages * a_stage) / b_tile;
  if (h.b_slots < nchunks * 9) {         // one A stage fewer if that makes the slab stationary
    const int b2 = (kSmemBudget - fixed - 2 * a_stage) / b_tile;
    if (b2 >= nchunks * 9 || h.b_slots < 3) {
      h.a_stages = 2;
      h.b_slots = b2;
    }
  }
  if (h.b_slots > kHaloMaxB) h.b_slots = kHaloMaxB;
  h.stationary = (h.b_slots >= 2 && nchunks * 9 <= h.b_slots) ? 1 : 0;
  if (h.stationary) h.b_slots = nchunks * 9;
  h.smem = fixed + h.a_stages * a_stage + h.b_slots * b_tile;
  return h;
}

// What one fprop / dgrad launch runs: its kernel, tile and persistent grid.  A pure host function of
// the geometry, the precision, the fused epilogue parts present, the tuning knobs and the SM count;
// conv_gemm_host launches it, acnn_conv_stats_parts() reports its statistics rows and
// acnn_conv_ctas_per_sm() its occupancy.
struct ConvChoice {
  bool halo;     // conv_halo_kernel (im2col-free 3x3) instead of conv_gemm_kernel
  int bn;        // N tile
  int cw;        // channels per A chunk (one filter tap each when Cin < 64)
  bool im2col;   // A tiles by im2col TMA (else 2-D tiles: dense 1x1, stride 1)
  int np;        // operand planes: 1 = bf16 / fp16, 3 = the fp32 parity mode
  bool f16;      // fp16 operands and output (ACNN_F16), one plane, the bf16 path's tiles
  int wg;        // consumer warpgroups per CTA: 2 = one CTA per SM, 1 = two CTAs per SM
  int pair;      // 1: clusters of two CTAs sharing the weight stages, one 256 x bn tile per pair
  int per_n;     // CTAs (pair = 1: CTA pairs) per N tile
  int parts;     // rows of the partial statistics buffer (= CTAs per N tile)
  int stages;    // conv_gemm_kernel: smem pipeline depth
  int smem;      // dynamic shared memory per CTA
  HaloPlan hp;   // conv_halo_kernel: its shared-memory plan
};

static ConvChoice conv_choice(const acnn_conv_geom& g, int precision, bool has_add, bool has_mask,
                              bool out_f32, bool has_bias) {
  ConvChoice c{};
  c.np = precision == ACNN_F32 ? 3 : 1;
  c.f16 = precision == ACNN_F16;
  c.cw = chunk_width(g.Cin);
  c.im2col = !is_plain(g);
  // N tile <= 128: a 64 x 256 fp32 accumulator per consumer warpgroup (128 registers per thread)
  // does not fit next to the epilogue under the 168-register limit of a 384-thread CTA
  c.bn = (g.Cout % 128 == 0) ? 128 : ((g.Cout % 64 == 0) ? 64 : 32);
  c.wg = 2;
  const bool halo_applies = g_conv_halo > 0 && g.kh == 3 && g.kw == 3 && g.stride == 1 &&
                            g.pad_h_lo == 1 && g.pad_h_hi == 1 && g.pad_w_lo == 1 &&
                            g.pad_w_hi == 1 && g.x_pix_stride <= 0 && g.x_row_pitch <= 0 &&
                            g.x_img_pitch <= 0 && c.np == 1 && !out_f32 && !has_bias &&
                            (g.Cin % 64 == 0 || g.Cin == 32) && g.Cout % 32 == 0;
  if (halo_applies) {
    c.hp = halo_plan(c.bn, c.cw, g.Cin, has_add, has_mask);
    // mode 1: the weight slab of an N tile stays in shared memory (otherwise the weight stream
    // replaces the im2col re-reads as the ingest bound) and the images have >= 56 rows (16 x 8
    // patches waste <= 12.5 % of a 56 x 56 image, 27 % of 28 x 28)
    c.halo = g_conv_halo >= 2 || (c.hp.stationary && g.H >= 56);
  }
  int m_tiles;
  if (c.halo) {
    c.smem = c.hp.smem;
    m_tiles = g.B * ceil_div(g.H, kPatchH) * ceil_div(g.W, kPatchW);
    c.per_n = num_sms() / (g.Cout / c.bn);
  } else {
    int Ho, Wo;
    out_hw(g, &Ho, &Wo);
    const int M = g.B * Ho * Wo, Ktot = g.kh * g.kw * g.Cin;
    // CTA pairs: full-width (64-channel) chunks, K >= 512 (the k-loop, not the epilogue, paces the
    // tile) and at least one pair tile per SM pair
    c.pair = (g_conv_pairs && c.bn == 128 && c.np == 1 && !out_f32 && c.cw == 64 && Ktot >= 512 &&
              (int64_t)ceil_div(M, 2 * kBM) * (g.Cout / 128) >= num_sms() / 2) ? 1 : 0;
    // bf16 / fp16 operands with K <= kTwoCtaMaxK: two co-resident CTAs per SM on 128 x 64 (Cout % 64
    // != 0: 128 x 32) tiles -- a 128 x 128 fp32 accumulator does not fit one warpgroup under the 168
    // registers per thread of two 5-warp CTAs (ptxas spills) -- where that gives >= 2 N tiles (<=
    // kMaxSms CTAs, i.e. partial statistics rows, per N tile).  The fp32 parity mode's three operand
    // planes and the CTA pairs keep one CTA per SM.
    const int bn2 = (g.Cout % 64 == 0 && g.Cout >= 128) ? 64 : 32;
    c.wg = (c.np == 1 && !c.pair && g.Cout / bn2 >= 2 && Ktot <= kTwoCtaMaxK) ? 1 : 2;
    if (c.wg == 1) c.bn = bn2;
    // persistent grid: a multiple of the N tiles so that every CTA keeps one N tile (its weights
    // and its per-channel statistics), at most one CTA per SM (two with wg = 1)
    m_tiles = ceil_div(M, (c.pair ? 2 : 1) * kBM);
    c.per_n = (c.pair ? num_sms() / 2 : (c.wg == 1 ? 2 * num_sms() : num_sms())) / (g.Cout / c.bn);
    c.smem = fprop_smem(c.bn, c.np, c.wg, has_add, has_mask, out_f32, &c.stages);
  }
  if (c.per_n < 1) c.per_n = 1;
  if (c.per_n > m_tiles) c.per_n = m_tiles;
  c.parts = c.pair ? 2 * c.per_n : c.per_n;
  return c;
}

// the type of every conv_gemm_kernel instantiation
typedef void (*ConvGemmFn)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap,
                           CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, ConvGemmParams);

// one instantiation, its shared-memory attributes set on first use (nullptr if that fails)
template <int BN, int CW, bool IM2COL, int NP, bool CG2, bool F16, int WG>
static ConvGemmFn conv_gemm_instance() {
  static bool attr_set = false;
  const ConvGemmFn kern = conv_gemm_kernel<BN, CW, IM2COL, NP, CG2, F16, WG>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         WG == 2 ? kSmemBudget + 2048 : kSmemBudget2);
    // two CTAs per SM need the largest shared-memory carveout
    if (e == cudaSuccess && WG == 1)
      e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                               cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(conv_gemm): %s", cudaGetErrorString(e));
      return nullptr;
    }
    attr_set = true;
  }
  return kern;
}

template <int BN, int NP, bool F16, int WG>
static ConvGemmFn conv_gemm_instance_cw(const ConvChoice& c) {
  if (c.im2col) {
    if (c.cw == 64) return conv_gemm_instance<BN, 64, true, NP, false, F16, WG>();
    if (c.cw == 32) return conv_gemm_instance<BN, 32, true, NP, false, F16, WG>();
    return conv_gemm_instance<BN, 16, true, NP, false, F16, WG>();
  }
  if (c.cw == 64) return conv_gemm_instance<BN, 64, false, NP, false, F16, WG>();
  if (c.cw == 32) return conv_gemm_instance<BN, 32, false, NP, false, F16, WG>();
  return conv_gemm_instance<BN, 16, false, NP, false, F16, WG>();
}

template <int BN>
static ConvGemmFn conv_gemm_instance_bn(const ConvChoice& c) {
  if constexpr (BN == 128) {
    if (c.pair) {     // full-width (64-channel) chunks only: bounds the instantiation count
      if (c.f16) {
        if (c.im2col) return conv_gemm_instance<128, 64, true, 1, true, true, 2>();
        return conv_gemm_instance<128, 64, false, 1, true, true, 2>();
      }
      if (c.im2col) return conv_gemm_instance<128, 64, true, 1, true, false, 2>();
      return conv_gemm_instance<128, 64, false, 1, true, false, 2>();
    }
  }
  if (c.np == 3) return conv_gemm_instance_cw<BN, 3, false, 2>(c);
  if constexpr (BN <= 64) {
    if (c.wg == 1) {
      if (c.f16) return conv_gemm_instance_cw<BN, 1, true, 1>(c);
      return conv_gemm_instance_cw<BN, 1, false, 1>(c);
    }
  }
  if (c.f16) return conv_gemm_instance_cw<BN, 1, true, 2>(c);
  return conv_gemm_instance_cw<BN, 1, false, 2>(c);
}

// The conv_gemm_kernel instantiation of a choice: the kernel conv_gemm_host launches and whose
// occupancy acnn_conv_ctas_per_sm() reports.  nullptr (error recorded) if its attributes cannot be set.
static ConvGemmFn conv_gemm_kernel_for(const ConvChoice& c) {
  if (c.bn == 128) return conv_gemm_instance_bn<128>(c);
  if (c.bn == 64) return conv_gemm_instance_bn<64>(c);
  return conv_gemm_instance_bn<32>(c);
}

static int make_map_4d(CUtensorMap* m, const void* base, int C, int W, int H, int B, int box_c,
                       int box_w, int box_h, CUtensorMapDataType dt) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode_tiled(m, dt, 4, const_cast<void*>(base), dims,
                              strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              swizzle_enum(box_c * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (4-d) failed (%d): C=%d W=%d H=%d B=%d box=%dx%dx%d", (int)r,
              C, W, H, B, box_c, box_w, box_h);
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

template <int BN, int CW, bool F16>
static int launch_conv_halo(const acnn_conv_geom& g, const ConvChoice& c, const void* x,
                            const void* w, void* y, float* ch_part, const void* add_src,
                            const void* mask_src, cudaStream_t stream) {
  using Cfg = HaloCfg<BN, CW>;
  static bool attr_set = false;
  auto kern = conv_halo_kernel<BN, CW, F16>;
  const CUtensorMapDataType dt = F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kSmemBudget + 2048);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(conv_halo): %s", cudaGetErrorString(e));
      return ACNN_ERR_CUDA;
    }
    attr_set = true;
  }
  HaloParams p;
  p.H = g.H; p.W = g.W; p.B = g.B; p.Cin = g.Cin; p.Cout = g.Cout;
  p.n_tiles = g.Cout / BN;
  p.ph = ceil_div(g.H, kPatchH);
  p.pw = ceil_div(g.W, kPatchW);
  p.m_tiles = g.B * p.ph * p.pw;
  p.ch_part = ch_part;
  p.has_add = add_src != nullptr;
  p.has_mask = mask_src != nullptr;
  p.a_stages = c.hp.a_stages;
  p.b_slots = c.hp.b_slots;
  p.stationary = c.hp.stationary;
  ACNN_REQUIRE(p.b_slots >= 2, "conv (halo): shared memory does not fit");
  CUtensorMap tmA, tmB, tmC, tmAdd, tmMask;
  int rc = make_map_4d(&tmA, x, g.Cin, g.W, g.H, g.B, CW, kHaloW, kHaloH, dt);
  if (rc) return rc;
  if ((rc = make_map_2d(&tmB, w, g.Cout, 9 * g.Cin, 9 * g.Cin, BN, CW, dt))) return rc;
  if ((rc = make_map_4d(&tmC, y, g.Cout, g.W, g.H, g.B, Cfg::kSubW, kPatchW, kPatchH, dt))) return rc;
  tmAdd = tmMask = tmC;
  if (add_src && (rc = make_map_4d(&tmAdd, add_src, g.Cout, g.W, g.H, g.B, Cfg::kSubW, kPatchW,
                                   kPatchH, dt)))
    return rc;
  if (mask_src && (rc = make_map_4d(&tmMask, mask_src, g.Cout, g.W, g.H, g.B, Cfg::kSubW, kPatchW,
                                    kPatchH, dt)))
    return rc;
  launch_k(kern, dim3(c.per_n * p.n_tiles), dim3(kThreads), c.smem, stream, tmA, tmB, tmC, tmAdd,
           tmMask, p);
  count_launch();
  return check_launch("conv_halo_kernel");
}

template <bool F16>
static int conv_halo_host(const acnn_conv_geom& g, const ConvChoice& c, const void* x, const void* w,
                          void* y, float* ch_part, const void* add_src, const void* mask_src,
                          cudaStream_t stream) {
  const bool c64 = c.cw == 64;
  if (c.bn == 128) {
    return c64 ? launch_conv_halo<128, 64, F16>(g, c, x, w, y, ch_part, add_src, mask_src, stream)
               : launch_conv_halo<128, 32, F16>(g, c, x, w, y, ch_part, add_src, mask_src, stream);
  }
  if (c.bn == 64) {
    return c64 ? launch_conv_halo<64, 64, F16>(g, c, x, w, y, ch_part, add_src, mask_src, stream)
               : launch_conv_halo<64, 32, F16>(g, c, x, w, y, ch_part, add_src, mask_src, stream);
  }
  return c64 ? launch_conv_halo<32, 64, F16>(g, c, x, w, y, ch_part, add_src, mask_src, stream)
             : launch_conv_halo<32, 32, F16>(g, c, x, w, y, ch_part, add_src, mask_src, stream);
}

// The argument checks of one fprop / dgrad launch with these epilogue parts.
static int conv_check(const acnn_conv_geom& g, bool has_stats, bool has_add, bool has_mask,
                      int out_f32, int precision, int64_t w_plane_stride) {
  ACNN_REQUIRE(g.B > 0 && g.H > 0 && g.W > 0 && g.Cin > 0 && g.Cout > 0, "conv: empty geometry");
  ACNN_REQUIRE(g.Cin % 16 == 0, "conv: Cin=%d must be a multiple of 16", g.Cin);
  ACNN_REQUIRE(g.Cout % 32 == 0, "conv: Cout=%d must be a multiple of 32", g.Cout);
  ACNN_REQUIRE(g.stride >= 1 && g.kh >= 1 && g.kw >= 1, "conv: bad kernel/stride");
  ACNN_REQUIRE(!(has_stats && out_f32), "conv: statistics only with bf16 output");
  ACNN_REQUIRE(precision == ACNN_BF16 || precision == ACNN_F32 || precision == ACNN_F16,
               "conv: precision must be 0 (bf16), 1 (fp32) or 3 (fp16)");
  ACNN_REQUIRE(precision != ACNN_F32 || (out_f32 && !has_add && !has_mask && !has_stats &&
                                         w_plane_stride > 0),
               "conv: the fp32 (3-plane) mode needs fp32 output, a weight plane stride and no "
               "fused add / mask / statistics epilogue");
  int Ho, Wo;
  ACNN_REQUIRE(out_hw(g, &Ho, &Wo), "conv: empty output");
  ACNN_REQUIRE(g.pad_h_lo <= 128 && g.pad_w_lo <= 128 && g.kh <= 128 && g.kw <= 128,
               "conv: padding / filter exceed the TMA im2col corner range");
  // the weight tile's swizzle span: 128 bytes, or the whole 32- or 64-byte row of a smaller K
  const int Ktot = g.kh * g.kw * g.Cin;
  ACNN_REQUIRE(Ktot >= 64 || Ktot == 32 || Ktot == 16, "conv: unsupported K=%d", Ktot);
  return ACNN_OK;
}

// precision 0: x / w are bf16.  precision 1 (fp32 parity mode): x and w each are THREE consecutive
// bf16 planes (acnn_split3 / acnn_prep_weights with planes = 3), plane p of x at x + p * numel(x),
// plane p of w at w + p * w_plane_stride elements; y must be fp32 (out_f32), no fused epilogue.
// precision ACNN_F16: x / w (and y, add, mask unless out_f32) are fp16, on the bf16 path's tiles.
static int conv_gemm_host(const acnn_conv_geom& g, const void* x, const void* w, void* y,
                          float* ch_part, const void* add_src, const void* mask_src,
                          const float* bias, int out_f32, int precision, int64_t w_plane_stride,
                          cudaStream_t stream) {
  int rc = conv_check(g, ch_part != nullptr, add_src != nullptr, mask_src != nullptr, out_f32,
                      precision, w_plane_stride);
  if (rc) return rc;
  const ConvChoice c = conv_choice(g, precision, add_src != nullptr, mask_src != nullptr,
                                   out_f32 != 0, bias != nullptr);
  // ch_part holds the rows acnn_conv_stats_parts() counts, those of the launch without add / mask /
  // bias: a fused part that moves the launch to another kernel or grid would leave rows unwritten
  // or write past the buffer
  if (ch_part) {
    const int parts = acnn_conv_stats_parts(&g);
    ACNN_REQUIRE(c.parts == parts,
                 "conv: with its add / mask / bias epilogue this launch writes %d partial "
                 "statistics rows, acnn_conv_stats_parts() counts %d", c.parts, parts);
  }
  if ((rc = load_driver_fns())) return rc;
  if (c.halo) {
    return c.f16 ? conv_halo_host<true>(g, c, x, w, y, ch_part, add_src, mask_src, stream)
                 : conv_halo_host<false>(g, c, x, w, y, ch_part, add_src, mask_src, stream);
  }
  int Ho, Wo;
  out_hw(g, &Ho, &Wo);
  const CUtensorMapDataType dt = c.f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  ConvGemmParams p;
  p.M = g.B * Ho * Wo;
  p.Cout = g.Cout;
  p.Cin = g.Cin;
  p.Ktot = g.kh * g.kw * g.Cin;
  p.kw = g.kw;
  p.HoWo = Ho * Wo;
  p.Wo = Wo;
  p.stride = g.stride;
  p.pad_h_lo = g.pad_h_lo;
  p.pad_w_lo = g.pad_w_lo;
  p.b_sw_bytes = p.Ktot >= 64 ? 128 : p.Ktot * 2;
  p.stages = c.stages;
  p.m_tiles = ceil_div(p.M, (c.pair ? 2 : 1) * kBM);
  p.n_tiles = g.Cout / c.bn;
  p.y = y;
  p.ch_part = ch_part;
  p.bias = bias;
  p.has_add = add_src != nullptr;
  p.has_mask = mask_src != nullptr;
  p.out_f32 = out_f32;

  ConvMaps tm;
  const int64_t x_plane = input_elems(g);
  for (int pl = 0; pl < c.np; ++pl) {
    const __nv_bfloat16* xp = static_cast<const __nv_bfloat16*>(x) + pl * x_plane;
    const __nv_bfloat16* wp = static_cast<const __nv_bfloat16*>(w) + pl * w_plane_stride;
    if (c.im2col) {
      rc = make_map_im2col(&tm.a[pl], xp, g, c.cw, kBM, dt);
    } else {
      rc = make_map_2d(&tm.a[pl], xp, p.M, g.Cin, g.Cin, kBM, c.cw, dt);
    }
    if (rc) return rc;
    rc = make_map_2d(&tm.b[pl], wp, g.Cout, p.Ktot, p.Ktot, c.pair ? c.bn / 2 : c.bn,
                     p.Ktot >= 64 ? 64 : p.Ktot, dt);
    if (rc) return rc;
  }
  for (int pl = c.np; pl < 3; ++pl) {   // placeholders
    tm.a[pl] = tm.a[0];
    tm.b[pl] = tm.b[0];
  }
  tm.c = tm.add = tm.mask = tm.b[0];   // placeholders when unused
  const int subw = c.bn < 64 ? c.bn : 64;
  if (!out_f32 && (rc = make_map_2d(&tm.c, y, p.M, g.Cout, g.Cout, kBM, subw, dt))) return rc;
  if (add_src && (rc = make_map_2d(&tm.add, add_src, p.M, g.Cout, g.Cout, kBM, subw, dt))) return rc;
  if (mask_src && (rc = make_map_2d(&tm.mask, mask_src, p.M, g.Cout, g.Cout, kBM, subw, dt)))
    return rc;

  const ConvGemmFn kern = conv_gemm_kernel_for(c);
  if (!kern) return ACNN_ERR_CUDA;
  if (c.pair) {
    // per_n CTA PAIRS per N tile, launched as clusters of two
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(2 * c.per_n * p.n_tiles);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = c.smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    (void)cudaLaunchKernelEx(&cfg, kern, tm.a[0], tm.b[0], tm.c, tm.add, tm.mask, tm.a[1], tm.a[2],
                             tm.b[1], tm.b[2], p);
  } else {
    launch_k(kern, dim3(c.per_n * p.n_tiles), dim3(conv_threads(c.wg)), c.smem, stream, tm.a[0],
             tm.b[0], tm.c, tm.add, tm.mask, tm.a[1], tm.a[2], tm.b[1], tm.b[2], p);
  }
  count_launch();
  return check_launch("conv_gemm_kernel");
}

struct WgradMaps {
  CUtensorMap x[3], dy[3];
};

// fixed cost of one wgrad CTA (pipeline fill + epilogue) in units of pipeline stages, for the
// split-K cost model (0 = the "two waves of CTAs" rule); acnn_set_wgrad_overhead_stages.  With the
// partials summed by wgrad_reduce_kernel, a sweep of forced split counts over the 43 wgrad
// geometries of the c3 step (H100 80GB HBM3, 700 W) puts the layouts this value picks within
// 0.11 ms per step of the fastest swept layout of every geometry, so it stays.
static int g_wgrad_overhead_stages = 16;

// Split-K partials are bounded (the split count is capped so that the tile-padded partials of all
// splits would fit): 64 MiB per launch.
constexpr size_t kWgPartFloats = size_t(16) << 20;

// 0: the cost model picks the split count; n > 0: n splits, within the capacity caps
// (acnn_set_wgrad_splits)
static int g_wgrad_splits = 0;

// 0: choose per problem; 64 / 128: force the pixels per stage where the shape allows it
static int g_wgrad_pix = 0;

// Tiling and split-K layout of one wgrad launch: a pure host function of the geometry, the
// precision, `deterministic`, the tuning knobs and the SM count, shared by the launcher and
// acnn_conv_wgrad_plan.
struct WgradPlan {
  int P;                 // pixels (GEMM K)
  int bn;                // N tile
  int n_tiles, m_tiles;
  int pix;               // pixels per pipeline stage
  int stages_total;
  int splits;            // CTAs along the pixel range
  int stages_per_split;  // every split but the last runs this many stages
};

static int wgrad_plan(const acnn_conv_geom& g, int precision, int deterministic, WgradPlan* w) {
  ACNN_REQUIRE(g.Cin % 16 == 0 && g.Cout % 32 == 0, "wgrad: Cin %% 16 / Cout %% 32 required");
  ACNN_REQUIRE(precision == ACNN_BF16 || precision == ACNN_F32 || precision == ACNN_F16,
               "wgrad: precision must be 0 (bf16), 1 (fp32) or 3 (fp16)");
  int Ho, Wo;
  ACNN_REQUIRE(out_hw(g, &Ho, &Wo), "wgrad: empty output");
  const int np = precision == ACNN_F32 ? 3 : 1;
  w->P = g.B * Ho * Wo;
  int bn = g.Cout >= 256 ? 256 : (g.Cout >= 128 ? 128 : (g.Cout >= 64 ? 64 : 32));
  if (np == 3 && bn > 128) bn = 128;   // three operand planes per stage: smem
  ACNN_REQUIRE(g.Cout % bn == 0, "wgrad: Cout=%d not a multiple of its N tile %d", g.Cout, bn);
  w->bn = bn;
  w->n_tiles = g.Cout / bn;
  w->m_tiles = ceil_div(g.kh * g.kw * g.Cin, 128);
  // 128-pixel stages (twice the MMAs per barrier round trip) wherever they fit, unless 64 are
  // forced: only the bf16 path, N tile <= 128 (smem), enough pixels to split
  w->pix = kWgPix;
  if (np == 1 && bn <= 128 && w->P >= 4096 && g_wgrad_pix != 64) w->pix = 128;
  w->stages_total = ceil_div(w->P, w->pix);
  // split the pixel (K) range over CTAs; the partial tiles are summed in split order, so the result
  // does not depend on which split finishes first.  deterministic: no split -- one add per dw
  // element.  One CTA per SM (384 threads with register accumulators).
  const int tiles = w->m_tiles * w->n_tiles;
  // capacity: the partial tiles of all splits fit kWgPartFloats
  const int64_t tile_floats = (int64_t)tiles * 128 * bn;
  int cap = (int)std::min<int64_t>(w->stages_total, (int64_t)kWgPartFloats / tile_floats);
  if (cap < 1) cap = 1;
  const int max_splits = std::min(cap, w->stages_total >= 8 ? w->stages_total / 4 : 1);
  int splits;
  if (g_wgrad_splits > 0) {
    splits = std::min(g_wgrad_splits, cap);
  } else if (g_wgrad_overhead_stages <= 0) {
    // (simple rule: roughly two waves of CTAs)
    splits = std::min(ceil_div(2 * num_sms(), tiles), max_splits);
  } else {
    // cost model: an SM runs its CTAs' pipeline stages back to back and pays a fixed pipeline-fill
    // + epilogue cost, worth g_wgrad_overhead_stages stages, once per CTA; pick the split count
    // with the least modelled time
    splits = 1;
    int64_t best = -1;
    for (int s = 1; s <= max_splits; ++s) {
      const int per = ceil_div(w->stages_total, s);
      const int s_eff = ceil_div(w->stages_total, per);
      if (s_eff != s) continue;
      const int per_sm = ceil_div(tiles * s, num_sms());
      const int64_t t = (int64_t)per_sm * per + (int64_t)per_sm * g_wgrad_overhead_stages;
      if (best < 0 || t < best) { best = t; splits = s; }
    }
  }
  if (splits < 1 || deterministic) splits = 1;
  w->stages_per_split = ceil_div(w->stages_total, splits);
  w->splits = ceil_div(w->stages_total, w->stages_per_split);
  return ACNN_OK;
}

template <int BN, int CW, int CWB, bool IM2COL, int NP, int PIX = kWgPix, bool F16 = false>
static int launch_wgrad(const WgradMaps& tm, WgradParams p, int m_tiles, int n_tiles,
                        cudaStream_t stream) {
  using Cfg = WgradCfg<BN, NP, PIX>;
  static bool attr_set = false;
  auto kern = wgrad_gemm_kernel<BN, CW, CWB, IM2COL, NP, PIX, F16>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(wgrad): %s", cudaGetErrorString(e));
      return ACNN_ERR_CUDA;
    }
    attr_set = true;
  }
  const int splits = p.splits;
  const int64_t n = (int64_t)p.Cout * p.Ktot;
  p.part = nullptr;
  if (splits > 1) {
    // this launch's partials, stream-ordered (per stream, capturable)
    void* scratch = nullptr;
    int rc = scratch_alloc(&scratch, (size_t)splits * n * sizeof(float), stream, "wgrad");
    if (rc) return rc;
    p.part = static_cast<float*>(scratch);
  }
  dim3 grid(m_tiles, n_tiles, splits);
  launch_k(kern, dim3(grid), dim3(kThreads), Cfg::kSmemBytes, stream, tm.x[0], tm.dy[0], tm.x[1],
           tm.x[2], tm.dy[1], tm.dy[2], p);
  count_launch();
  int rc = check_launch("wgrad_gemm_kernel");
  if (!p.part) return rc;
  if (rc == ACNN_OK) {
    launch_k(wgrad_reduce_kernel, dim3((unsigned)ceil_div64(n, kWgRedThreads)), dim3(kWgRedThreads),
             0, stream, static_cast<const float*>(p.part), p.dw, n, splits);
    count_launch();
    rc = check_launch("wgrad_reduce_kernel");
  }
  const int rc2 = scratch_free(p.part, stream, "wgrad");
  return rc ? rc : rc2;
}

template <int BN, int CW, bool IM2COL, bool F16>
static int dispatch_wgrad_cwb(int cwb, int np, const WgradMaps& tm, const WgradParams& p, int mt,
                              int nt, cudaStream_t s) {
  if constexpr (BN <= 128 && !F16) {
    if (np == 3) {
      if constexpr (BN >= 64) {
        if (cwb == 64) return launch_wgrad<BN, CW, 64, IM2COL, 3>(tm, p, mt, nt, s);
      }
      return launch_wgrad<BN, CW, 32, IM2COL, 3>(tm, p, mt, nt, s);
    }
  }
  if constexpr (BN >= 64) {
    if (cwb == 64) {
      if constexpr (BN <= 128) {
        if (p.pix == 128) return launch_wgrad<BN, CW, 64, IM2COL, 1, 128, F16>(tm, p, mt, nt, s);
      }
      return launch_wgrad<BN, CW, 64, IM2COL, 1, kWgPix, F16>(tm, p, mt, nt, s);
    }
  }
  if constexpr (BN <= 128) {
    if (p.pix == 128) return launch_wgrad<BN, CW, 32, IM2COL, 1, 128, F16>(tm, p, mt, nt, s);
  }
  return launch_wgrad<BN, CW, 32, IM2COL, 1, kWgPix, F16>(tm, p, mt, nt, s);
}

template <int BN, bool IM2COL, bool F16>
static int dispatch_wgrad_cw(int cw, int cwb, int np, const WgradMaps& tm, const WgradParams& p,
                             int mt, int nt, cudaStream_t s) {
  if (cw == 64) return dispatch_wgrad_cwb<BN, 64, IM2COL, F16>(cwb, np, tm, p, mt, nt, s);
  if (cw == 32) return dispatch_wgrad_cwb<BN, 32, IM2COL, F16>(cwb, np, tm, p, mt, nt, s);
  return dispatch_wgrad_cwb<BN, 16, IM2COL, F16>(cwb, np, tm, p, mt, nt, s);
}

// F16: fp16 operands (ACNN_F16), one plane, the bf16 path's tiles
template <bool IM2COL, bool F16>
static int dispatch_wgrad(int bn, int cw, int cwb, int np, const WgradMaps& tm, const WgradParams& p,
                          int mt, int nt, cudaStream_t s) {
  if (bn == 256) return dispatch_wgrad_cw<256, IM2COL, F16>(cw, cwb, np, tm, p, mt, nt, s);
  if (bn == 128) return dispatch_wgrad_cw<128, IM2COL, F16>(cw, cwb, np, tm, p, mt, nt, s);
  if (bn == 64) return dispatch_wgrad_cw<64, IM2COL, F16>(cw, cwb, np, tm, p, mt, nt, s);
  return dispatch_wgrad_cw<32, IM2COL, F16>(cw, cwb, np, tm, p, mt, nt, s);
}

static int conv_wgrad_host(const acnn_conv_geom& g, const void* x, const void* dy, float* dw,
                           int precision, int deterministic, cudaStream_t stream) {
  WgradPlan w;
  int rc = wgrad_plan(g, precision, deterministic, &w);
  if (rc) return rc;
  rc = load_driver_fns();
  if (rc) return rc;
  int Ho, Wo;
  out_hw(g, &Ho, &Wo);
  const bool plain = is_plain(g);
  const int np = precision == ACNN_F32 ? 3 : 1;
  const bool f16 = precision == ACNN_F16;
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  WgradParams p;
  p.P = w.P;
  p.Cout = g.Cout;
  p.Cin = g.Cin;
  p.Ktot = g.kh * g.kw * g.Cin;
  p.kw = g.kw;
  p.HoWo = Ho * Wo;
  p.Wo = Wo;
  p.stride = g.stride;
  p.pad_h_lo = g.pad_h_lo;
  p.pad_w_lo = g.pad_w_lo;
  p.pix = w.pix;
  p.stages_total = w.stages_total;
  p.stages_per_split = w.stages_per_split;
  p.splits = w.splits;
  p.dw = dw;
  const int cw = chunk_width(g.Cin);
  const int cwb = (g.Cout % 64 == 0) ? 64 : 32;
  WgradMaps tm;
  const int64_t x_plane = input_elems(g), dy_plane = (int64_t)p.P * g.Cout;
  for (int pl = 0; pl < np; ++pl) {
    const __nv_bfloat16* xp = static_cast<const __nv_bfloat16*>(x) + pl * x_plane;
    const __nv_bfloat16* dp = static_cast<const __nv_bfloat16*>(dy) + pl * dy_plane;
    rc = make_map_2d(&tm.dy[pl], dp, p.P, g.Cout, g.Cout, p.pix, cwb, dt);
    if (rc) return rc;
    if (plain) {
      rc = make_map_2d(&tm.x[pl], xp, p.P, g.Cin, g.Cin, p.pix, cw, dt);
    } else {
      rc = make_map_im2col(&tm.x[pl], xp, g, cw, p.pix, dt);
    }
    if (rc) return rc;
  }
  for (int pl = np; pl < 3; ++pl) {
    tm.x[pl] = tm.x[0];
    tm.dy[pl] = tm.dy[0];
  }
  if (f16) {
    if (plain) return dispatch_wgrad<false, true>(w.bn, cw, cwb, np, tm, p, w.m_tiles, w.n_tiles, stream);
    return dispatch_wgrad<true, true>(w.bn, cw, cwb, np, tm, p, w.m_tiles, w.n_tiles, stream);
  }
  if (plain) return dispatch_wgrad<false, false>(w.bn, cw, cwb, np, tm, p, w.m_tiles, w.n_tiles, stream);
  return dispatch_wgrad<true, false>(w.bn, cw, cwb, np, tm, p, w.m_tiles, w.n_tiles, stream);
}

}  // namespace acnn

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

int acnn_set_conv_mtiles(int mode) {
  const int prev = acnn::g_conv_mtiles_mode;
  acnn::g_conv_mtiles_mode = (mode == 1 || mode == 2) ? mode : -1;
  return prev;
}

int acnn_set_conv_halo(int mode) {
  const int prev = acnn::g_conv_halo;
  acnn::g_conv_halo = mode < 0 ? 0 : (mode > 2 ? 2 : mode);
  return prev;
}

int acnn_set_conv_split_epilogue(int mode) {
  const int prev = acnn::g_conv_split_epi;
  acnn::g_conv_split_epi = mode < 0 ? 0 : (mode > 2 ? 2 : mode);
  return prev;
}

int acnn_set_conv_split_mt2(int mode) {
  const int prev = acnn::g_conv_split_mt2;
  acnn::g_conv_split_mt2 = mode < 0 ? 0 : (mode > 2 ? 2 : mode);
  return prev;
}

int acnn_set_conv_halo_split(int on) {
  const int prev = acnn::g_conv_halo_split;
  acnn::g_conv_halo_split = on ? 1 : 0;
  return prev;
}

int acnn_set_conv_out_bufs(int mode) {
  const int prev = acnn::g_conv_out_bufs;
  acnn::g_conv_out_bufs = mode < 0 ? 0 : (mode > 2 ? 2 : mode);
  return prev;
}

int acnn_set_wgrad_overhead_stages(int stages) {
  const int prev = acnn::g_wgrad_overhead_stages;
  acnn::g_wgrad_overhead_stages = stages < 0 ? 0 : stages;
  return prev;
}

int acnn_set_wgrad_pixels(int pix) {
  const int prev = acnn::g_wgrad_pix;
  acnn::g_wgrad_pix = (pix == 64 || pix == 128) ? pix : 0;
  return prev;
}

int acnn_set_wgrad_splits(int n) {
  const int prev = acnn::g_wgrad_splits;
  acnn::g_wgrad_splits = n < 0 ? 0 : n;
  return prev;
}

int acnn_conv_wgrad_plan(const acnn_conv_geom* g, int precision, int deterministic, int* pix,
                         int* splits, int* stages_per_split) {
  if (!g) {
    acnn::set_error("acnn_conv_wgrad_plan: null geometry");
    return ACNN_ERR_INVALID;
  }
  acnn::WgradPlan w;
  const int rc = acnn::wgrad_plan(*g, precision, deterministic, &w);
  if (rc) return rc;
  if (pix) *pix = w.pix;
  if (splits) *splits = w.splits;
  if (stages_per_split) *stages_per_split = w.stages_per_split;
  return ACNN_OK;
}

int acnn_conv_stats_parts(const acnn_conv_geom* g) {
  if (!g) return 0;
  int Ho, Wo;
  if (!acnn::out_hw(*g, &Ho, &Wo) || g->Cout <= 0 || g->Cout % 32 != 0) return 0;
  // the launch with statistics and no add / mask / bias (precision 0 and 3 choose alike)
  return acnn::conv_choice(*g, ACNN_BF16, false, false, false, false).parts;
}

int acnn_conv_ctas_per_sm(const acnn_conv_geom* g, int precision, int has_add, int has_mask,
                          int* ctas) {
  if (!g || !ctas) {
    acnn::set_error("acnn_conv_ctas_per_sm: null argument");
    return ACNN_ERR_INVALID;
  }
  *ctas = 0;
  const int out_f32 = precision == ACNN_F32 ? 1 : 0;   // the fp32 mode stores fp32
  const int rc = acnn::conv_check(*g, false, has_add != 0, has_mask != 0, out_f32, precision,
                                  out_f32);
  if (rc) return rc;
  const acnn::ConvChoice c =
      acnn::conv_choice(*g, precision, has_add != 0, has_mask != 0, out_f32 != 0, false);
  ACNN_REQUIRE(!c.halo, "conv: this geometry runs on the halo kernel");
  const acnn::ConvGemmFn kern = acnn::conv_gemm_kernel_for(c);
  if (!kern) return ACNN_ERR_CUDA;
  const cudaError_t e =
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, kern, acnn::conv_threads(c.wg), c.smem);
  if (e != cudaSuccess) {
    acnn::set_error("cudaOccupancyMaxActiveBlocksPerMultiprocessor(conv_gemm): %s",
                    cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

int acnn_set_conv_cta_pairs(int on) {
  const int prev = acnn::g_conv_pairs;
  acnn::g_conv_pairs = on ? 1 : 0;
  return prev;
}

int acnn_conv_fprop(const acnn_conv_geom* g, const void* x, const void* w, void* y,
                    float* ch_part, const void* add_src, const void* mask_src, const float* bias,
                    int out_f32, int precision, int64_t w_plane_stride, void* stream) {
  if (!g || !x || !w || !y) {
    acnn::set_error("acnn_conv_fprop: null argument");
    return ACNN_ERR_INVALID;
  }
  return acnn::conv_gemm_host(*g, x, w, y, ch_part, add_src, mask_src, bias, out_f32, precision,
                              w_plane_stride, static_cast<cudaStream_t>(stream));
}

int acnn_conv_dgrad(const acnn_conv_geom* g, const void* dy, const void* w_dgrad, void* dx,
                    const void* add_src, const void* mask_src, int precision,
                    int64_t w_plane_stride, void* stream) {
  if (!g || !dy || !w_dgrad || !dx) {
    acnn::set_error("acnn_conv_dgrad: null argument");
    return ACNN_ERR_INVALID;
  }
  if (g->stride != 1) {
    acnn::set_error("acnn_conv_dgrad: stride %d (zero-insert dy first, then call with stride 1)",
                    g->stride);
    return ACNN_ERR_UNSUPPORTED;
  }
  // dx = correlation of dy with the flipped, channel-transposed filter; padding k-1-pad.
  const int Ho = g->H + g->pad_h_lo + g->pad_h_hi - g->kh + 1;
  const int Wo = g->W + g->pad_w_lo + g->pad_w_hi - g->kw + 1;
  acnn_conv_geom t;
  t.B = g->B;
  t.H = Ho;
  t.W = Wo;
  t.Cin = g->Cout;
  t.Cout = g->Cin;
  t.kh = g->kh;
  t.kw = g->kw;
  t.stride = 1;
  t.pad_h_lo = g->kh - 1 - g->pad_h_lo;
  t.pad_h_hi = g->kh - 1 - g->pad_h_hi;
  t.pad_w_lo = g->kw - 1 - g->pad_w_lo;
  t.pad_w_hi = g->kw - 1 - g->pad_w_hi;
  t.x_pix_stride = t.x_row_pitch = t.x_img_pitch = t.reserved_ = 0;
  return acnn::conv_gemm_host(t, dy, w_dgrad, dx, nullptr, add_src, mask_src, nullptr,
                              precision == ACNN_F32 ? 1 : 0, precision, w_plane_stride,
                              static_cast<cudaStream_t>(stream));
}

int acnn_conv_wgrad(const acnn_conv_geom* g, const void* x, const void* dy, float* dw,
                    int precision, int deterministic, void* stream) {
  if (!g || !x || !dy || !dw) {
    acnn::set_error("acnn_conv_wgrad: null argument");
    return ACNN_ERR_INVALID;
  }
  return acnn::conv_wgrad_host(*g, x, dy, dw, precision, deterministic,
                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
