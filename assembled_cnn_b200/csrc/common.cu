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

}  // namespace acnn
