// 16-byte vector helpers for the HBM-bound NHWC bf16 kernels (8 channels per thread).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace acnn {

#ifndef ACNN_PDL_PRIMS
#define ACNN_PDL_PRIMS
// Programmatic dependent launch entry (see common.h): let the dependent kernel start launching, then
// wait until the preceding kernel has completed and its writes are visible.  No-ops when the kernel
// was launched without the attribute.
__device__ __forceinline__ void pdl_trigger() {
  asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_entry() {
  pdl_trigger();
  pdl_wait();
}
#endif

typedef __nv_bfloat16 bf16;
typedef __half f16;

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void load8(const bf16* p, float (&f)[8]) {
  unpack8(__ldg(reinterpret_cast<const uint4*>(p)), f);
}
__device__ __forceinline__ void store8(bf16* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) = pack8(f);
}
__device__ __forceinline__ void loadf8(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void storef8(float* p, const float (&f)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}

// fp32 activation storage (the parity mode, acnn.h ACNN_F32): the same 8-element accessors on float.
__device__ __forceinline__ void load8(const float* p, float (&f)[8]) { loadf8(p, f); }
__device__ __forceinline__ void store8(float* p, const float (&f)[8]) { storef8(p, f); }

// fp16 activation storage (acnn.h ACNN_F16): exact widening, round-to-nearest-even narrowing
// (values beyond the fp16 range become +-inf).
__device__ __forceinline__ void unpack8_f16(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8_f16(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void load8(const f16* p, float (&f)[8]) {
  unpack8_f16(__ldg(reinterpret_cast<const uint4*>(p)), f);
}
__device__ __forceinline__ void store8(f16* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) = pack8_f16(f);
}

__device__ __forceinline__ void store1(bf16* p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void store1(f16* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void store1(float* p, float v) { *p = v; }
__device__ __forceinline__ float load1(const bf16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float load1(const f16* p) { return __half2float(*p); }
__device__ __forceinline__ float load1(const float* p) { return *p; }

// Raw 8-element vector of an activation tensor: loads can be issued back to back (batched ahead
// of the math) and unpacked later.  V8<bf16> is one 16-byte register quad, V8<float> two.
template <class T>
struct V8;
template <>
struct V8<bf16> {
  uint4 r;
  __device__ __forceinline__ void ld(const bf16* p) { r = __ldg(reinterpret_cast<const uint4*>(p)); }
  __device__ __forceinline__ void lds(const uint8_t* base, int elem) {
    r = *reinterpret_cast<const uint4*>(base + (size_t)elem * 2);
  }
  __device__ __forceinline__ void zero() { r = make_uint4(0, 0, 0, 0); }
  __device__ __forceinline__ void unpack(float (&f)[8]) const { unpack8(r, f); }
  __device__ __forceinline__ void st(bf16* p) const { *reinterpret_cast<uint4*>(p) = r; }
};
template <>
struct V8<f16> {
  uint4 r;
  __device__ __forceinline__ void ld(const f16* p) { r = __ldg(reinterpret_cast<const uint4*>(p)); }
  __device__ __forceinline__ void lds(const uint8_t* base, int elem) {
    r = *reinterpret_cast<const uint4*>(base + (size_t)elem * 2);
  }
  __device__ __forceinline__ void zero() { r = make_uint4(0, 0, 0, 0); }
  __device__ __forceinline__ void unpack(float (&f)[8]) const { unpack8_f16(r, f); }
  __device__ __forceinline__ void st(f16* p) const { *reinterpret_cast<uint4*>(p) = r; }
};
template <>
struct V8<float> {
  float4 a, b;
  __device__ __forceinline__ void ld(const float* p) {
    a = __ldg(reinterpret_cast<const float4*>(p));
    b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  }
  __device__ __forceinline__ void lds(const uint8_t* base, int elem) {
    a = *reinterpret_cast<const float4*>(base + (size_t)elem * 4);
    b = *reinterpret_cast<const float4*>(base + (size_t)elem * 4 + 16);
  }
  __device__ __forceinline__ void zero() { a = b = make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ __forceinline__ void unpack(float (&f)[8]) const {
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
    f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  __device__ __forceinline__ void st(float* p) const {
    reinterpret_cast<float4*>(p)[0] = a;
    reinterpret_cast<float4*>(p)[1] = b;
  }
};

// 8 elements at element offset `elem` of a shared-memory staging area holding T.
template <class T>
__device__ __forceinline__ void lds8(const uint8_t* base, int elem, float (&f)[8]) {
  V8<T> v;
  v.lds(base, elem);
  v.unpack(f);
}

// Optional gradient epilogue shared by every backward kernel: (+ add_src) then (* (mask_src > 0)).
template <class T>
__device__ __forceinline__ void grad_epilogue(float (&v)[8], const T* add_src,
                                              const T* mask_src, size_t off) {
  if (add_src) {
    float a[8];
    load8(add_src + off, a);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] += a[i];
  }
  if (mask_src) {
    float m[8];
    load8(mask_src + off, m);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (!(m[i] > 0.f)) v[i] = 0.f;
  }
}

// Storage types of the `dtype` argument of the elementwise / reduction entry points (acnn.h), and
// the dispatch that instantiates a launch on the matching element type T.
#define ACNN_DTYPE_OK(dt) ((dt) == ACNN_BF16 || (dt) == ACNN_F32 || (dt) == ACNN_F16)
#define ACNN_BY_DTYPE(dt, ...)      \
  do {                              \
    if ((dt) == ACNN_F32) {         \
      using T = float;              \
      __VA_ARGS__;                  \
    } else if ((dt) == ACNN_F16) {  \
      using T = f16;                \
      __VA_ARGS__;                  \
    } else {                        \
      using T = bf16;               \
      __VA_ARGS__;                  \
    }                               \
  } while (0)

// cap of the grid-stride elementwise kernels' grids (acnn_set_stream_grid_cap; common.cu)
extern int g_stream_grid_cap;

inline int grid_for(int64_t work_items, int threads = 256, int max_blocks = -1) {
  if (max_blocks < 0) max_blocks = g_stream_grid_cap;
  int64_t b = (work_items + threads - 1) / threads;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

}  // namespace acnn
