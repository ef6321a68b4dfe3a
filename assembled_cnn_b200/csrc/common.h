// Host-side helpers shared by every translation unit of libacnn.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/acnn.h"

namespace acnn {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// Returns ACNN_OK or records the CUDA error (launch-configuration errors surface here).
int check_launch(const char* what);
// The H100 SXM's SM count: grid-size heuristics and the capacities of the per-CTA partial-sum
// buffers (model_plan.h, plan.py) are sized for one wave of it, and the conv launchers use at most
// this many SMs, so those capacities hold on any device.
constexpr int kMaxSms = 132;

// Stream-ordered scratch of one launch (split-K partials): cudaMallocAsync on `stream`, released by
// scratch_free on the same stream after the kernels that use it.  Concurrent streams get distinct
// buffers; under stream capture both become graph memory nodes.
int scratch_alloc(void** p, size_t bytes, cudaStream_t stream, const char* what);
int scratch_free(void* p, cudaStream_t stream, const char* what);

#define ACNN_REQUIRE(cond, ...)        \
  do {                                 \
    if (!(cond)) {                     \
      ::acnn::set_error(__VA_ARGS__);  \
      return ACNN_ERR_INVALID;         \
    }                                  \
  } while (0)

// The float[3] `mean` argument of the entry point `fn`, host or device memory: device memory gives
// *mean_dev = mean, host memory *mean_dev = nullptr and its values in m.  A failed pointer query is
// reported as "<fn>: mean: <CUDA error>" (ACNN_ERR_CUDA).
int resolve_mean(const char* fn, const float* mean, const float** mean_dev, float m[3]);

// Programmatic dependent launch (PDL): every kernel of this library starts with
// `griddepcontrol.launch_dependents; griddepcontrol.wait;` (pdl_entry() in vec.cuh / ptx.cuh), so a
// kernel launched with the programmatic-stream-serialization attribute may be scheduled (CTAs
// resident, prologue done) while its predecessor drains, and only proceeds past the wait once the
// predecessor grid has completed and flushed.  Meant to hide the per-kernel launch / drain latency
// of the dependent launches of a step; opt-in (an early dependent takes SM resources from its
// still-running predecessor).
extern int g_use_pdl;   // 0 by default; ACNN_PDL=1|2 / acnn_set_pdl

template <class... KArgs, class... Args>
inline void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                     Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  // mode 1: every launch; mode 2: only LIGHT dependents (few CTAs, little shared memory: the
  // finalize / small-GEMM / loss kernels) -- their early-resident CTAs cost the still-running
  // predecessor nothing, while their launch latency (~400 such launches per step) is hidden
  const bool light = (size_t)grid.x * grid.y * grid.z <= 320 && smem <= 48 * 1024;
  cfg.numAttrs = (g_use_pdl == 1 || (g_use_pdl == 2 && light)) ? 1 : 0;
  (void)cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);   // errors: check_launch()
}

// SM count of the current device, at most kMaxSms (kMaxSms without a device: host-only queries).
int num_sms();

// ------------------------------------------------------------------------------------------
// Tensor-map creation (driver entry points fetched lazily: libacnn.so does not link libcuda).
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const int*, const int*,
                                   cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
extern EncodeTiledFn g_encode_tiled;
extern EncodeIm2colFn g_encode_im2col;
extern int g_driver_version;

int load_driver_fns();
CUtensorMapSwizzle swizzle_enum(int bytes);
// 16-bit (bf16 unless dt says fp16) matrix [rows][cols] (cols contiguous, row pitch ld elements);
// box = [box_rows][box_cols].
int make_map_2d(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld,
                int box_rows, int box_cols,
                CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// acnn_sk_fc_fwd / acnn_se_fc_fwd with their GEMMs' split-K chosen as for max(B, split_rows) rows
// (acnn_set_fc_split_rows): each row gets the bits of the same row in a batch of split_rows.
int sk_fc_fwd(const float* s, const float* w1, const float* gamma, const float* beta, float* moving_mean,
              float* moving_var, float momentum, float eps, int training, const float* w2, float* zpre,
              float* bnstat, float* z, float* att, float* scratch, int B, int f, int d, int deterministic,
              int split_rows, void* stream);
int se_fc_fwd(const float* q, const float* w1, const float* w2, float* h, float* e, int B, int C, int r,
              int deterministic, int split_rows, void* stream);
int fc_split_rows();   // acnn_set_fc_split_rows

}  // namespace acnn
