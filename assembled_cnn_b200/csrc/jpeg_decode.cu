// Device JPEG decode of a batch (acnn_jpeg_decode, include/acnn.h), in seven launches:
//   unstuff  one CTA per image: drop the stuffed zeros and the restart markers of the scan (a block-wide
//            prefix sum places every kept byte), record where each restart interval starts, and cut every
//            interval into subsequences of kSubBits bits
//   phase    one thread per subsequence (Weissenberger & Schmidt, "Massively Parallel Huffman Decoding on
//            GPUs", ICPP 2018; "Accelerating JPEG Decompression on GPUs", HiPC 2021): pass 0 decodes each
//            subsequence from its start, guessing the state (first block of an MCU, DC next); pass 1
//            decodes it again from the state its predecessor ended in, and marks the successor dirty when
//            that changed its exit state
//   sync     one CTA per image: re-decode dirty subsequences until no exit state changes (the decode
//            self-synchronises, so this is usually one or two subsequences), then a prefix sum of the
//            blocks each subsequence completes places its output, and the block count of every restart
//            interval is checked.  The first subsequence of an interval starts in a known state, so
//            restart markers are exact synchronisation points.
//   write    one thread per subsequence: decode from the synchronised state, writing int16 coefficients
//   dc       one CTA per image: per component, a prefix sum of the DC differences, reset at every restart
//            interval
//   idct     one thread per 8x8 block of the MCU rows and columns the window needs
//   color    one thread per window pixel: upsampling, YCbCr->RGB, packed uint8 RGB out
// The arithmetic of every stage is in jpeg_stages.cuh.
#include <algorithm>

#include <cub/block/block_scan.cuh>

#include "common.h"
#include "jpeg_stages.cuh"
#include "vec.cuh"

namespace acnn {
namespace {

using jpeg::State;
using jpeg::kSubBits;

struct Sub {
  int32_t start, end, iend;
  int32_t first;   // interval index + 1 for the first subsequence of a restart interval, else 0
};

__device__ __forceinline__ const uint8_t* wk(void* work, int64_t off) { return (const uint8_t*)work + off; }
template <class T>
__device__ __forceinline__ T* wp(void* work, int64_t off) {
  return (T*)((uint8_t*)work + off);
}

// the image's Huffman tables in shared memory
struct __align__(16) HuffSmem {
  acnn_jpeg_huff dc[2], ac[2];
};
__device__ __forceinline__ void load_tables(const acnn_jpeg_desc& d, HuffSmem& s) {
  const int4* src = reinterpret_cast<const int4*>(&d.dc[0]);
  int4* dst = reinterpret_cast<int4*>(&s);
  static_assert(sizeof(HuffSmem) % 16 == 0, "table copy in int4");
  for (int i = threadIdx.x; i < (int)(sizeof(HuffSmem) / 16); i += blockDim.x) dst[i] = src[i];
}

// ------------------------------------------------------------------------------------ unstuff
constexpr int kUnThreads = 256, kUnItems = 8;

__global__ void __launch_bounds__(kUnThreads)
jpeg_unstuff_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs,
                    const uint8_t* __restrict__ data, void* work, int32_t* __restrict__ status) {
  pdl_entry();
  const int img = blockIdx.x;
  const acnn_jpeg_job& j = jobs[img];
  if (!j.active) {
    if (threadIdx.x == 0) status[img] = ACNN_JPEG_ST_UNSUPPORTED;
    return;
  }
  if (threadIdx.x == 0) status[img] = 0;
  const acnn_jpeg_desc& d = descs[img];
  const uint8_t* e = data + j.src + d.ecs_offset;
  const int64_t n = d.ecs_length;
  uint8_t* bits = wp<uint8_t>(work, j.o_bits);
  int32_t* intervals = wp<int32_t>(work, j.o_intervals);
  typedef cub::BlockScan<int, kUnThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int64_t s_kept;
  __shared__ int s_rst;
  if (threadIdx.x == 0) {
    s_kept = 0;
    s_rst = 0;
    intervals[0] = 0;
  }
  __syncthreads();
  for (int64_t base = 0; base < n; base += kUnThreads * kUnItems) {
    const int64_t i0 = base + (int64_t)threadIdx.x * kUnItems;
    int cls[kUnItems];
    int kept = 0, rst = 0;
#pragma unroll
    for (int k = 0; k < kUnItems; ++k) {
      cls[k] = i0 + k < n ? jpeg::unstuff_class(e, i0 + k, n) : 0;
      kept += cls[k] == 1;
      rst += cls[k] == 2;
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(kept | rst << 16, excl, total);
    const int64_t kb = s_kept;
    const int rb = s_rst;
    int64_t o = kb + (excl & 0xFFFF);
    int r = rb + (excl >> 16);
#pragma unroll
    for (int k = 0; k < kUnItems; ++k) {
      if (cls[k] == 1) bits[o++] = e[i0 + k];
      else if (cls[k] == 2 && r + 1 < d.n_intervals) intervals[++r] = (int32_t)(o * 8);
      else if (cls[k] == 2) ++r;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      s_kept = kb + (total & 0xFFFF);
      s_rst = rb + (total >> 16);
    }
    __syncthreads();
  }
  const int64_t kept = s_kept;
  for (int k = threadIdx.x; k < jpeg::kBitsPad; k += kUnThreads) bits[kept + k] = 0;
  if (threadIdx.x == 0) {
    intervals[d.n_intervals] = (int32_t)(kept * 8);
    if (s_rst != d.n_intervals - 1) atomicOr(&status[img], ACNN_JPEG_ST_MCU_COUNT);   // parser guarantees not
  }
  __syncthreads();
  // subsequences: interval k holds max(1, ceil(len_k / kSubBits)) of them, the first at first[k] (in the
  // prefix region, which the sync pass overwrites later); every thread then writes every blockDim-th entry
  Sub* subs = wp<Sub>(work, j.o_subs);
  int32_t* first = wp<int32_t>(work, j.o_prefix);
  int64_t sbase = 0;
  for (int k0 = 0; k0 < d.n_intervals; k0 += kUnThreads) {
    const int k = k0 + threadIdx.x;
    int m = 0;
    if (k < d.n_intervals) {
      const int a = intervals[k], b = intervals[k + 1];
      m = b > a ? (b - a + kSubBits - 1) / kSubBits : 1;
    }
    int excl, total;
    __syncthreads();
    Scan(tmp).ExclusiveSum(m, excl, total);
    if (k < d.n_intervals) first[k] = (int32_t)(sbase + excl);
    sbase += total;
  }
  const int ns = (int)(sbase < j.max_sub ? sbase : j.max_sub);
  __syncthreads();
  for (int s = threadIdx.x; s < ns; s += kUnThreads) {
    int lo = 0, hi = d.n_intervals - 1;   // the last interval whose first subsequence is <= s
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (first[mid] <= s) lo = mid;
      else hi = mid - 1;
    }
    const int a = intervals[lo], b = intervals[lo + 1], t = s - first[lo];
    const int st = a + t * kSubBits;
    subs[s] = Sub{st, min(st + kSubBits, b), b, t == 0 ? lo + 1 : 0};
  }
  if (threadIdx.x == 0) {
    intervals[d.n_intervals + 1] = ns;
    if (sbase > j.max_sub) atomicOr(&status[img], ACNN_JPEG_ST_MCU_COUNT);   // cannot happen: capacity bound
  }
}

__device__ __forceinline__ int n_subs(const acnn_jpeg_job& j, const acnn_jpeg_desc& d, void* work) {
  return wp<int32_t>(work, j.o_intervals)[d.n_intervals + 1];
}

// entry state of subsequence s: its start (first block of an MCU, DC next) for the first of an interval
// or when the predecessor's exit is unknown; the predecessor's exit otherwise
__device__ __forceinline__ State entry_of(const Sub& s, const State* prev) {
  if (s.first || prev->p < 0) return State{s.start, 0, 0, 0};
  return *prev;
}

__device__ __forceinline__ State run_sub(const acnn_jpeg_desc& d, const HuffSmem& h, const uint8_t* bits,
                                         const Sub& s, State in) {
  State r = jpeg::decode_run<false>(d, h.dc, h.ac, bits, in, s.end, s.iend, nullptr, 0, 0);
  if (r.err) r.p = -1;
  return r;
}

// ------------------------------------------------------------------------------------ phase
constexpr int kSubThreads = 128;

__global__ void __launch_bounds__(kSubThreads)
jpeg_phase_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs, void* work,
                  int pass) {
  pdl_entry();
  const int img = blockIdx.y;
  const acnn_jpeg_job& j = jobs[img];
  if (!j.active) return;
  const acnn_jpeg_desc& d = descs[img];
  const int ns = n_subs(j, d, work);
  if ((int)(blockIdx.x * kSubThreads) >= ns) return;
  __shared__ HuffSmem h;
  load_tables(d, h);
  __syncthreads();
  const int t = blockIdx.x * kSubThreads + threadIdx.x;
  if (t >= ns) return;
  const Sub* subs = wp<Sub>(work, j.o_subs);
  State* st0 = wp<State>(work, j.o_state);
  State* st1 = st0 + j.max_sub;
  const uint8_t* bits = wk(work, j.o_bits);
  const Sub s = subs[t];
  if (pass == 0) {
    st0[t] = run_sub(d, h, bits, s, State{s.start, 0, 0, 0});
    return;
  }
  uint8_t* dirty = wp<uint8_t>(work, j.o_dirty);
  State r = st0[t];
  if (!s.first && st0[t - 1].p >= 0) r = run_sub(d, h, bits, s, st0[t - 1]);
  st1[t] = r;
  if (t + 1 < ns) dirty[t + 1] = !jpeg::same_entry(r, st0[t]) && !subs[t + 1].first;
  if (t == 0) dirty[0] = 0;
}

// ------------------------------------------------------------------------------------ sync
constexpr int kSyncThreads = 256;

__global__ void __launch_bounds__(kSyncThreads)
jpeg_sync_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs, void* work,
                 int32_t* __restrict__ status) {
  pdl_entry();
  const int img = blockIdx.x;
  const acnn_jpeg_job& j = jobs[img];
  if (!j.active) return;
  const acnn_jpeg_desc& d = descs[img];
  const int ns = n_subs(j, d, work);
  __shared__ HuffSmem h;
  __shared__ int s_any;
  load_tables(d, h);
  const Sub* subs = wp<Sub>(work, j.o_subs);
  State* st = wp<State>(work, j.o_state) + j.max_sub;
  uint8_t* dirty = wp<uint8_t>(work, j.o_dirty);
  const uint8_t* bits = wk(work, j.o_bits);
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    for (int base = 0; base < ns; base += kSyncThreads) {
      const int t = base + threadIdx.x;
      bool upd = false;
      State r{};
      Sub s{};
      if (t < ns && dirty[t]) {
        // cleared before the barrier: the predecessor may mark it again after the barrier
        dirty[t] = 0;
        s = subs[t];
        r = run_sub(d, h, bits, s, entry_of(s, &st[t - 1]));
        upd = true;
      }
      __syncthreads();
      if (upd) {
        const bool changed = !jpeg::same_entry(r, st[t]);
        st[t] = r;
        if (changed && t + 1 < ns && !subs[t + 1].first) {
          dirty[t + 1] = 1;
          s_any = 1;
        }
      }
      __syncthreads();
    }
    if (!s_any) break;
  }
  // output placement and checks: exclusive prefix of the completed blocks; every interval starts at its
  // first block, ends on an MCU boundary, and the scan holds every block of the image
  typedef cub::BlockScan<int, kSyncThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int32_t* prefix = wp<int32_t>(work, j.o_prefix);
  const int64_t per_interval = (int64_t)d.restart_interval * d.bpm;
  int carry = 0, err = 0;
  for (int base = 0; base < ns; base += kSyncThreads) {
    const int t = base + threadIdx.x;
    State r{};
    Sub s{};
    if (t < ns) {
      r = st[t];
      s = subs[t];
    }
    int excl, total;
    __syncthreads();
    Scan(tmp).ExclusiveSum(t < ns ? r.nb : 0, excl, total);
    if (t < ns) {
      const int pre = carry + excl;
      prefix[t] = pre;
      err |= r.err;
      if (s.first && (int64_t)pre != (int64_t)(s.first - 1) * per_interval) err |= ACNN_JPEG_ST_MCU_COUNT;
      const bool last_of_interval = t + 1 == ns || subs[t + 1].first;
      if (last_of_interval && (r.cz & 0xFFFF) != 0) err |= ACNN_JPEG_ST_MCU_COUNT;
      if (t + 1 == ns && (int64_t)pre + r.nb != (int64_t)d.mcus_x * d.mcus_y * d.bpm) err |= ACNN_JPEG_ST_MCU_COUNT;
    }
    carry += total;
  }
  if (err) atomicOr(&status[img], err);
}

// ------------------------------------------------------------------------------------ write
__global__ void __launch_bounds__(kSubThreads)
jpeg_write_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs, void* work,
                  const int32_t* __restrict__ status) {
  pdl_entry();
  const int img = blockIdx.y;
  const acnn_jpeg_job& j = jobs[img];
  if (!j.active || status[img]) return;
  const acnn_jpeg_desc& d = descs[img];
  const int ns = n_subs(j, d, work);
  if ((int)(blockIdx.x * kSubThreads) >= ns) return;
  __shared__ HuffSmem h;
  load_tables(d, h);
  __syncthreads();
  const int t = blockIdx.x * kSubThreads + threadIdx.x;
  if (t >= ns) return;
  const int32_t blk0 = wp<int32_t>(work, j.o_prefix)[t];
  if (blk0 >= j.stored_blocks) return;
  const Sub s = wp<Sub>(work, j.o_subs)[t];
  const State* st = wp<State>(work, j.o_state) + j.max_sub;
  const State in = entry_of(s, &st[t - 1]);
  jpeg::decode_run<true>(d, h.dc, h.ac, wk(work, j.o_bits), in, s.end, s.iend, wp<int16_t>(work, j.o_coef), blk0,
                         j.stored_blocks);
}

// ------------------------------------------------------------------------------------ dc
struct Seg {
  int32_t f;
  uint32_t v;
};
struct SegOp {
  __device__ __forceinline__ Seg operator()(const Seg& a, const Seg& b) const {
    return Seg{a.f | b.f, b.f ? b.v : a.v + b.v};
  }
};
struct SegCarry {
  Seg run;
  __device__ Seg operator()(const Seg& agg) {
    const Seg old = run;
    run = SegOp()(run, agg);
    return old;
  }
};

constexpr int kDcThreads = 256, kDcItems = 4;

__global__ void __launch_bounds__(kDcThreads)
jpeg_dc_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs, void* work,
               const int32_t* __restrict__ status) {
  pdl_entry();
  const int img = blockIdx.x, ci = blockIdx.y;
  const acnn_jpeg_job& j = jobs[img];
  if (!j.active || status[img]) return;
  const acnn_jpeg_desc& d = descs[img];
  if (ci >= d.ncomp) return;
  typedef cub::BlockScan<Seg, kDcThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int16_t* coef = wp<int16_t>(work, j.o_coef);
  const int nbc = d.comp[ci].h * d.comp[ci].v, blk0 = d.comp[ci].blk0;
  const int64_t T = (int64_t)(j.mcu_r1 + 1) * d.mcus_x * nbc;
  const int R = d.restart_interval;
  SegCarry carry{Seg{0, 0}};
  for (int64_t base = 0; base < T; base += kDcThreads * kDcItems) {
    Seg v[kDcItems];
    int64_t blk[kDcItems];
#pragma unroll
    for (int k = 0; k < kDcItems; ++k) {
      const int64_t t = base + threadIdx.x * kDcItems + k;
      const int64_t m = t / nbc, u = t - m * nbc;
      blk[k] = m * d.bpm + blk0 + u;
      const bool first = t == 0 || (R > 0 && u == 0 && m % R == 0);
      v[k] = t < T ? Seg{first ? 1 : 0, (uint32_t)(int32_t)coef[blk[k] * 64]} : Seg{0, 0};
    }
    __syncthreads();
    Scan(tmp).InclusiveScan(v, v, SegOp(), carry);
#pragma unroll
    for (int k = 0; k < kDcItems; ++k)
      if (base + threadIdx.x * kDcItems + k < T) coef[blk[k] * 64] = (int16_t)v[k].v;
  }
}

// ------------------------------------------------------------------------------------ idct
__global__ void __launch_bounds__(128)
jpeg_idct_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs, void* work,
                 const int32_t* __restrict__ status) {
  pdl_entry();
  const int img = blockIdx.y;
  const acnn_jpeg_job& j = jobs[img];
  const int idx = blockIdx.x * 128 + threadIdx.x;
  if (!j.active || idx >= j.idct_blocks || status[img]) return;
  const acnn_jpeg_desc& d = descs[img];
  const int cols = j.mcu_c1 - j.mcu_c0 + 1;
  const int mcu = idx / d.bpm, c = idx - mcu * d.bpm;
  const int mr = j.mcu_r0 + mcu / cols, mc = j.mcu_c0 + mcu % cols;
  const int ci = jpeg::block_comp(d, c);
  const acnn_jpeg_comp& cp = d.comp[ci];
  const int u = (c - cp.blk0) % cp.h, w = (c - cp.blk0) / cp.h;
  const int16_t* in = wp<int16_t>(work, j.o_coef) + ((int64_t)(mr * d.mcus_x + mc) * d.bpm + c) * 64;
  __align__(16) int16_t blk[64];
  const int4* in4 = reinterpret_cast<const int4*>(in);
#pragma unroll
  for (int k = 0; k < 8; ++k) reinterpret_cast<int4*>(blk)[k] = in4[k];
  const int64_t pitch = (int64_t)cols * 8 * cp.h;
  uint8_t* out = wp<uint8_t>(work, j.o_plane[ci]) + (int64_t)(((mr - j.mcu_r0) * cp.v + w) * 8) * pitch +
                 ((mc - j.mcu_c0) * cp.h + u) * 8;
  jpeg::idct_islow(blk, d.quant[cp.tq], out, pitch);
}

// ------------------------------------------------------------------------------------ color
__global__ void __launch_bounds__(256)
jpeg_color_kernel(const acnn_jpeg_desc* __restrict__ descs, const acnn_jpeg_job* __restrict__ jobs, void* work,
                  uint8_t* __restrict__ out, const int32_t* __restrict__ status) {
  pdl_entry();
  const int img = blockIdx.y;
  const acnn_jpeg_job& j = jobs[img];
  const int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (!j.active || idx >= (int64_t)j.win_h * j.win_w || status[img]) return;
  const acnn_jpeg_desc& d = descs[img];
  const int cols = j.mcu_c1 - j.mcu_c0 + 1;
  jpeg::Plane pl[3];
  for (int c = 0; c < d.ncomp; ++c) {
    const acnn_jpeg_comp& cp = d.comp[c];
    pl[c] = jpeg::Plane{wk(work, j.o_plane[c]), (int64_t)cols * 8 * cp.h, j.mcu_r0 * 8 * cp.v, j.mcu_c0 * 8 * cp.h,
                        cp.dw, cp.dh};
  }
  const int py = (int)(idx / j.win_w), px = (int)(idx - (int64_t)py * j.win_w);
  uint8_t rgb[3];
  jpeg::pixel_rgb(d, pl, j.win_y + py, j.win_x + px, rgb);
  uint8_t* o = out + j.out + idx * 3;
  o[0] = rgb[0];
  o[1] = rgb[1];
  o[2] = rgb[2];
}

}  // namespace
}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_jpeg_decode(const acnn_jpeg_desc* desc, const acnn_jpeg_job* jobs, const acnn_jpeg_batch* batch,
                     const uint8_t* data, uint8_t* out, void* work, int64_t work_bytes, int32_t* status,
                     void* stream) {
  ACNN_REQUIRE(desc && jobs && batch && data && out && work && status, "acnn_jpeg_decode: null pointer");
  ACNN_REQUIRE(batch->n >= 1 && batch->n <= 65535, "acnn_jpeg_decode: batch of %d images outside [1, 65535]",
               batch->n);
  ACNN_REQUIRE(work_bytes >= batch->work_bytes, "acnn_jpeg_decode: work holds %lld bytes, the plan needs %lld",
               (long long)work_bytes, (long long)batch->work_bytes);
  ACNN_REQUIRE(((uintptr_t)work & 255) == 0 && ((uintptr_t)desc & 15) == 0 && ((uintptr_t)jobs & 7) == 0,
               "acnn_jpeg_decode: work must be 256-byte, desc 16-byte and jobs 8-byte aligned");
  const cudaStream_t s = (cudaStream_t)stream;
  const int n = batch->n;
  if (batch->coef_end > batch->coef_begin) {
    cudaError_t e = cudaMemsetAsync((uint8_t*)work + batch->coef_begin, 0, batch->coef_end - batch->coef_begin, s);
    if (e != cudaSuccess) {
      set_error("acnn_jpeg_decode: memset: %s", cudaGetErrorString(e));
      return ACNN_ERR_CUDA;
    }
  }
  launch_k(jpeg_unstuff_kernel, dim3(n), dim3(kUnThreads), 0, s, desc, jobs, data, work, status);
  const dim3 gsub(ceil_div(std::max(batch->max_sub, 1), kSubThreads), n);
  launch_k(jpeg_phase_kernel, gsub, dim3(kSubThreads), 0, s, desc, jobs, work, 0);
  launch_k(jpeg_phase_kernel, gsub, dim3(kSubThreads), 0, s, desc, jobs, work, 1);
  launch_k(jpeg_sync_kernel, dim3(n), dim3(kSyncThreads), 0, s, desc, jobs, work, status);
  launch_k(jpeg_write_kernel, gsub, dim3(kSubThreads), 0, s, desc, jobs, work, (const int32_t*)status);
  launch_k(jpeg_dc_kernel, dim3(n, 3), dim3(kDcThreads), 0, s, desc, jobs, work, (const int32_t*)status);
  launch_k(jpeg_idct_kernel, dim3(ceil_div(std::max(batch->max_idct_blocks, 1), 128), n), dim3(128), 0, s, desc,
           jobs, work, (const int32_t*)status);
  launch_k(jpeg_color_kernel, dim3((unsigned)ceil_div64(std::max(batch->max_pixels, 1), 256), n), dim3(256), 0, s,
           desc, jobs, work, out, (const int32_t*)status);
  count_launch(8);
  return check_launch("jpeg_decode");
}

}  // extern "C"
