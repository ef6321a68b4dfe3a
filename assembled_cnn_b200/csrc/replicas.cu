// Several data-parallel replicas per device: the accumulation of the per-replica gradients, BN moving
// statistics and loss between the micro-steps of one global step (acnn_replica_accumulate, include/acnn.h).
//
// One grid-stride pass over two parts, the gradient range [lo, hi) and the state [0, n_state).  Each part is
// a scalar head up to the first 16-byte boundary, a body of float4 vectors and a scalar tail; a part whose
// pointers are not equally aligned runs as scalars only.  Every element is read and written once per phase,
// each output by one thread: no atomics, and the same bits on every launch.
#include "common.h"
#include "vec.cuh"

namespace acnn {

struct ReplicaPart {
  float* acc;         // acc_grads + lo | acc_state (state_base in SAVE)
  float* x;           // grads + lo | state
  float* base;        // nullptr | state_base
  int64_t n;          // elements
  int64_t head;       // scalars before the float4 body (n when the part runs as scalars only)
  int64_t nvec;       // float4 vectors of the body
  int state;          // 1: the state part (scaled in LAST)
};

__device__ __forceinline__ float radd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float4 radd(float4 a, float4 b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}
__device__ __forceinline__ float rmul(float a, float s) { return __fmul_rn(a, s); }
__device__ __forceinline__ float4 rmul(float4 a, float s) {
  return make_float4(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s), __fmul_rn(a.w, s));
}

// the V (float or float4) at element e of one part
template <class V>
__device__ __forceinline__ void replica_elem(int phase, const ReplicaPart& p, int64_t e, float scale) {
  V* x = reinterpret_cast<V*>(p.x + e);
  if (phase == ACNN_REPLICA_SAVE) {
    *reinterpret_cast<V*>(p.acc + e) = *x;
    return;
  }
  V* acc = reinterpret_cast<V*>(p.acc + e);
  if (phase == ACNN_REPLICA_LAST) {
    const V v = radd(*acc, *x);
    *x = p.state ? rmul(v, scale) : v;
    return;
  }
  *acc = phase == ACNN_REPLICA_FIRST ? *x : radd(*acc, *x);
  if (p.base) *x = *reinterpret_cast<const V*>(p.base + e);
}

// scalar k of a part: its head, then its tail after the body
__device__ __forceinline__ int64_t scalar_elem(const ReplicaPart& p, int64_t k) {
  return k < p.head ? k : p.head + 4 * p.nvec + (k - p.head);
}

// items: [part 0 vectors][part 1 vectors][part 0 scalars][part 1 scalars]
__global__ void __launch_bounds__(256)
replica_accumulate_kernel(int phase, ReplicaPart g, ReplicaPart s, float scale) {
  pdl_wait();   // multi-wave grid: an early trigger would let the next kernel's CTAs take SM slots from this one
  const int64_t gs = g.n - 4 * g.nvec, ss = s.n - 4 * s.nvec;
  const int64_t total = g.nvec + s.nvec + gs + ss;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t k = i;
    if (k < g.nvec) {
      replica_elem<float4>(phase, g, g.head + 4 * k, scale);
    } else if ((k -= g.nvec) < s.nvec) {
      replica_elem<float4>(phase, s, s.head + 4 * k, scale);
    } else if ((k -= s.nvec) < gs) {
      replica_elem<float>(phase, g, scalar_elem(g, k), scale);
    } else {
      replica_elem<float>(phase, s, scalar_elem(s, k - gs), scale);
    }
  }
}

// The part's split: the float4 body starts at the first 16-byte boundary of x and needs acc (and base) at
// the same alignment; otherwise the whole part runs as scalars.
ReplicaPart make_part(float* acc, float* x, float* base, int64_t n, int state) {
  ReplicaPart p{acc, x, base, n, n, 0, state};
  const uintptr_t mis = (uintptr_t)x & 15;
  if (n == 0 || mis % 4 != 0 || (uintptr_t)acc % 16 != mis || (base && (uintptr_t)base % 16 != mis)) return p;
  p.head = std::min<int64_t>(n, (int64_t)((16 - mis) & 15) / 4);
  p.nvec = (n - p.head) / 4;
  return p;
}

}  // namespace acnn

using namespace acnn;

extern "C" {

int acnn_replica_accumulate(int phase, float* acc_grads, float* grads, float* state_base, float* acc_state,
                            float* state, int64_t lo, int64_t hi, int64_t n_state, float state_scale,
                            void* stream) {
  ACNN_REQUIRE(phase >= ACNN_REPLICA_SAVE && phase <= ACNN_REPLICA_LAST, "acnn_replica_accumulate: bad phase %d",
               phase);
  ACNN_REQUIRE(lo >= 0 && hi >= lo && n_state >= 0,
               "acnn_replica_accumulate: bad range lo=%lld hi=%lld n_state=%lld", (long long)lo, (long long)hi,
               (long long)n_state);
  const bool with_grads = phase != ACNN_REPLICA_SAVE && hi > lo;
  ACNN_REQUIRE(!with_grads || (acc_grads && grads), "acnn_replica_accumulate: null gradient buffer");
  ACNN_REQUIRE(n_state == 0 || (state && (phase == ACNN_REPLICA_SAVE ? state_base != nullptr : acc_state != nullptr)),
               "acnn_replica_accumulate: null state buffer");
  const ReplicaPart none{nullptr, nullptr, nullptr, 0, 0, 0, 0};
  const ReplicaPart g = with_grads ? make_part(acc_grads + lo, grads + lo, nullptr, hi - lo, 0) : none;
  const ReplicaPart s = n_state == 0 ? none
                        : phase == ACNN_REPLICA_SAVE ? make_part(state_base, state, nullptr, n_state, 1)
                                                     : make_part(acc_state, state, state_base, n_state, 1);
  const int64_t items = g.nvec + s.nvec + (g.n - 4 * g.nvec) + (s.n - 4 * s.nvec);
  if (items == 0) return ACNN_OK;
  launch_k(replica_accumulate_kernel, dim3(grid_for(items)), dim3(256), 0, (cudaStream_t)stream, phase, g, s,
           state_scale);
  count_launch();
  return check_launch("replica_accumulate");
}

}  // extern "C"
