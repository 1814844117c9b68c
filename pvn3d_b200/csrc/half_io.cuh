// half_io.cuh -- element access for the float32 / float16 / bfloat16 forms of the PointNet++ and PSPNet ops that
// autocast hands 16-bit tensors (pn2_ops.cu, determinism.cu).
//
// Every kernel templated on the element type T reads T, computes in float32 and rounds each output element once, to
// nearest even, when it stores a 16-bit T.  For T = float both conversions are the identity, so the float32
// instantiations are the kernels they were before the templates.  Rounding keeps inf and NaN, and a float32 value
// that rounds past float16's largest finite value (65504) becomes inf, as GradScaler expects to find it.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace pvn3d {

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ unsigned short bits16(__half v) { return __half_as_ushort(v); }
__device__ __forceinline__ unsigned short bits16(__nv_bfloat16 v) { return __bfloat16_as_ushort(v); }

// streaming (evict-first) stores of one 16-bit element and of two adjacent ones (p 4-byte aligned)
template <typename T>
__device__ __forceinline__ void stg_stream(T *p, T v) {
  asm volatile("st.global.cs.b16 [%0], %1;" ::"l"(p), "h"(bits16(v)) : "memory");
}
template <typename T>
__device__ __forceinline__ void stg_stream2(T *p, T lo, T hi) {
  const unsigned v = static_cast<unsigned>(bits16(lo)) | (static_cast<unsigned>(bits16(hi)) << 16);
  asm volatile("st.global.cs.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// a plain store of two adjacent elements (p 4-byte aligned)
template <typename T>
__device__ __forceinline__ void st_pair(T *p, T lo, T hi) {
  *reinterpret_cast<unsigned *>(p) = static_cast<unsigned>(bits16(lo)) | (static_cast<unsigned>(bits16(hi)) << 16);
}

// out[i] = round16(src[i]): the one rounding of the 16-bit atomic grads, which scatter into a float32 scratch.  Pairs
// (a float2 load, one 4-byte store) when both pointers allow it, a scalar tail.
template <typename T, int kVec>
__global__ void round_to16_kernel(const float *__restrict__ src, long long count, T *__restrict__ out) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i * kVec < count; i += stride) {
    if (kVec == 2 && 2 * i + 1 < count) {
      const float2 v = *reinterpret_cast<const float2 *>(src + 2 * i);
      st_pair(out + 2 * i, from_f32<T>(v.x), from_f32<T>(v.y));
    } else {
      out[kVec * i] = from_f32<T>(src[kVec * i]);
    }
  }
}

static inline bool aligned_to(const void *p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// f(T{}) for the 16-bit element type a PVN3D_F16 / PVN3D_BF16 code names; any other code is refused before f runs
template <typename F>
static int with_dtype16(int dtype, F &&f) {
  if (dtype == PVN3D_F16) return f(__half{});
  if (dtype == PVN3D_BF16) return f(__nv_bfloat16{});
  return PVN3D_ERR_INVALID_ARG;
}

}  // namespace pvn3d
