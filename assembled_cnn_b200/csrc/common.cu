#include "common.h"

#include <stdarg.h>
#include <stdlib.h>
#include <atomic>

namespace acnn {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int pdl_default() {
  // opt-in: an early resident dependent takes registers / SM slots from a still-running HBM-bound
  // predecessor
  const char* e = getenv("ACNN_PDL");
  return (e && (e[0] == '1' || e[0] == '2')) ? e[0] - '0' : 0;
}
int g_use_pdl = pdl_default();
int g_stream_grid_cap = kMaxSms * 16;   // vec.cuh grid_for(); acnn_set_stream_grid_cap

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

}  // namespace acnn

extern "C" {

const char* acnn_last_error(void) { return acnn::g_err; }
int acnn_version(void) { return 100; }
int acnn_set_pdl(int on) {
  const int prev = acnn::g_use_pdl;
  acnn::g_use_pdl = (on == 1 || on == 2) ? on : 0;
  return prev;
}
int acnn_set_stream_grid_cap(int blocks) {
  const int prev = acnn::g_stream_grid_cap;
  acnn::g_stream_grid_cap = blocks >= acnn::kMaxSms ? blocks : acnn::kMaxSms * 16;
  return prev;
}
int64_t acnn_launch_count(void) { return acnn::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"

namespace acnn {

int scratch_alloc(void** p, size_t bytes, cudaStream_t stream, const char* what) {
  cudaError_t e = cudaMallocAsync(p, bytes, stream);
  if (e != cudaSuccess) {
    set_error("%s: scratch of %zu bytes: %s", what, bytes, cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

int scratch_free(void* p, cudaStream_t stream, const char* what) {
  cudaError_t e = cudaFreeAsync(p, stream);
  if (e != cudaSuccess) {
    set_error("%s: releasing scratch: %s", what, cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

static int g_num_sms = 0;
int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
      (void)cudaGetLastError();   // no device (host-only queries): size for the H100's kMaxSms
      g_num_sms = 0;
    }
    // at most kMaxSms: the partial statistics rows (one per CTA of an N tile) are sized for it
    if (g_num_sms <= 0 || g_num_sms > kMaxSms) g_num_sms = kMaxSms;
  }
  return g_num_sms;
}

EncodeTiledFn g_encode_tiled = nullptr;
EncodeIm2colFn g_encode_im2col = nullptr;
int g_driver_version = 0;

int load_driver_fns() {
  if (g_encode_tiled && g_encode_im2col) return ACNN_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !fn) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  g_encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
  fn = nullptr;
  e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !fn) {
    set_error("cuTensorMapEncodeIm2col entry point unavailable (%s)", cudaGetErrorString(e));
    return ACNN_ERR_CUDA;
  }
  g_encode_im2col = reinterpret_cast<EncodeIm2colFn>(fn);
  cudaDriverGetVersion(&g_driver_version);
  return ACNN_OK;
}

CUtensorMapSwizzle swizzle_enum(int bytes) {
  return bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                      : (bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

int make_map_2d(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld,
                int box_rows, int box_cols) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base),
                              dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              swizzle_enum(box_cols * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rows=%lld cols=%lld ld=%lld box=%dx%d", (int)r,
              (long long)rows, (long long)cols, (long long)ld, box_rows, box_cols);
    return ACNN_ERR_CUDA;
  }
  return ACNN_OK;
}

}  // namespace acnn
