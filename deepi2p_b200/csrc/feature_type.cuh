// Feature element types of the differentiable ops that run under bfloat16 autocast (DESIGN.md 4.37): float and
// bfloat16.  A kernel templated on the type T converts at its loads (load_f32: exact, bf16 is a truncated float) and
// at its stores (store_as<T>: round to nearest even), and keeps its float / double arithmetic, so a bf16 call computes
// exactly what the float call computes on the widened inputs, rounded once to bf16 at each store.  The C ABI passes
// bf16 data as uint16_t bit patterns; as_bf16 reinterprets them.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace dib {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ float load_f32(float v) { return v; }
__device__ __forceinline__ float load_f32(bf16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T store_as(float v);
template <>
__device__ __forceinline__ float store_as<float>(float v) { return v; }
template <>
__device__ __forceinline__ bf16 store_as<bf16>(float v) { return __float2bfloat16_rn(v); }

inline const bf16* as_bf16(const uint16_t* p) { return reinterpret_cast<const bf16*>(p); }
inline bf16* as_bf16(uint16_t* p) { return reinterpret_cast<bf16*>(p); }

}  // namespace dib
