// Row loader shared by the fast DSA-family kernels: D contiguous elements, 16-byte loads when the row
// size allows (rows start at multiples of D elements from a 128-byte aligned base).
// Free of CUDA runtime includes (tests/hostshim/ compiles it on the CPU).
#pragma once
#include <stdint.h>

// D contiguous elements; 16-byte loads when the row size allows (rows start at multiples of D
// elements from a 128-byte aligned base)
template <typename T, int D>
__host__ __device__ __forceinline__ void fg_load_row(const T *__restrict__ p, T (&r)[D]) {
  if constexpr (sizeof(T) == 4 && D % 4 == 0) {
    const float4 *q = reinterpret_cast<const float4 *>(p);
#pragma unroll
    for (int i = 0; i < D / 4; ++i) {
      const float4 v = q[i];
      r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
    }
  } else if constexpr (sizeof(T) == 8 && D % 2 == 0) {
    const double2 *q = reinterpret_cast<const double2 *>(p);
#pragma unroll
    for (int i = 0; i < D / 2; ++i) {
      const double2 v = q[i];
      r[2 * i] = v.x; r[2 * i + 1] = v.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < D; ++i) r[i] = p[i];
  }
}

// Oriented DSA / MGM tables keep every row on its own cache-line slot: a row of D elements is stored with
// stride fg_row_stride<T, D>() = the next power of two >= D (rounded to whole 128-byte lines above 128 bytes),
// so the ONE row a slot reads per cycle costs one or two whole DRAM lines instead of the 1.5 lines an
// unaligned 80-byte row averaged.  pydcop_b200/engine.py::dsa_row_stride is the same rule.
template <typename T, int D>
__host__ __device__ constexpr int fg_row_stride() {
  int p2 = 1;
  while (p2 < D) p2 *= 2;
  const int line = 128 / (int)sizeof(T);
  return p2 * (int)sizeof(T) > 128 ? (D + line - 1) / line * line : p2;
}

// D elements of a row stored with fg_row_stride: whole 16 / 8 / 4-byte vectors (the pad is readable)
template <typename T, int D>
__host__ __device__ __forceinline__ void fg_load_row_padded(const T *__restrict__ p, T (&r)[D]) {
  constexpr int RSB = fg_row_stride<T, D>() * (int)sizeof(T);
  constexpr int VB = RSB % 16 == 0 ? 16 : (RSB % 8 == 0 ? 8 : (int)sizeof(T));
  constexpr int V = VB / (int)sizeof(T);
  constexpr int NV = (D + V - 1) / V;
  T tmp[NV * V];
  if constexpr (VB == 16 && sizeof(T) == 4) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 v = reinterpret_cast<const float4 *>(p)[i];
      tmp[4 * i] = v.x; tmp[4 * i + 1] = v.y; tmp[4 * i + 2] = v.z; tmp[4 * i + 3] = v.w;
    }
  } else if constexpr (VB == 16 && sizeof(T) == 8) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const double2 v = reinterpret_cast<const double2 *>(p)[i];
      tmp[2 * i] = v.x; tmp[2 * i + 1] = v.y;
    }
  } else if constexpr (VB == 8 && sizeof(T) == 4) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float2 v = reinterpret_cast<const float2 *>(p)[i];
      tmp[2 * i] = v.x; tmp[2 * i + 1] = v.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < NV * V; ++i) tmp[i] = p[i];
  }
#pragma unroll
  for (int i = 0; i < D; ++i) r[i] = tmp[i];
}
