// Shared device helpers for the factor-graph kernels (sm_90a).
// Arithmetic note: every floating-point expression below keeps the operand ORDER of the
// reference (pydcop/algorithms/maxsum.py) and the file is compiled with -fmad=false, so the
// f64 instantiation is bit-identical to the reference's Python floats and the f32 instantiation
// is bit-identical to the f32 build of the CPU oracle.
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include <vector>

#include "../../include/pydcop_b200.h"

#define FG_SAME_COUNT 4  // maxsum.py:106

template <typename T> struct Inf;
template <> struct Inf<float> { __device__ static float pos() { return CUDART_INF_F; } };
template <> struct Inf<double> { __device__ static double pos() { return CUDART_INF; } };

template <typename T> __device__ __forceinline__ T fg_abs(T x);
template <> __device__ __forceinline__ float fg_abs<float>(float x) { return fabsf(x); }
template <> __device__ __forceinline__ double fg_abs<double>(double x) { return fabs(x); }

// maxsum.py:688-710, one element: true when `c` matches `prev_c` within `stab`
template <typename T>
__device__ __forceinline__ bool approx_match1(T c, T prev_c, T stab) {
  if (prev_c != c) {
    T delta = fg_abs<T>(prev_c - c);
    T s = prev_c + c;
    if (s != (T)0) {
      if (!(((T)2 * delta / fg_abs<T>(s)) < stab)) return false;
    } else {
      return false;
    }
  }
  return true;
}

// optimum update with the reference's strict comparison (maxsum.py:439-443)
template <typename T>
__device__ __forceinline__ void opt_update(T &opt, T cur, bool mode_max) {
  if (mode_max ? (opt < cur) : (opt > cur)) opt = cur;
}

// Send gate shared by both sides (maxsum.py:356-377, 545-564).
// cnt byte: bit0 = sender recorded a previous message, bits 1.. = times the same message was sent.
// Returns true when the message is posted; updates cnt.
__device__ __forceinline__ bool gate_decide(bool match, uint8_t &cnt_byte) {
  int cnt = cnt_byte >> 1;
  if (!match) { cnt_byte = (uint8_t)(1u | (1u << 1)); return true; }
  if (cnt < FG_SAME_COUNT) { cnt_byte = (uint8_t)(1u | ((cnt + 1) << 1)); return true; }
  return false;
}

struct MaxSumParams {
  int mode_max, damp_vars, damp_factors;
  double damping, one_minus_damping, stability;
  // multi-GPU, fused halo (warp kernels only; null = no peer stores): per edge / per slot the address in the consumer's
  // `next` buffer of the row this cycle produces, 0 for interior rows (fg_halo_plan_t::dev_edge_dst_r / dev_slot_dst_q)
  const int64_t *edge_dst, *slot_dst;
};

// The entry of `per_dev` for the current device, added on first use.  What a kernel's launch code works out once
// (its dynamic shared-memory attribute, its occupancy, the SM count) holds for one device only: an attribute set with
// cudaFuncSetAttribute belongs to the function in the current device's context.
template <class S>
inline S &fg_per_device(std::vector<S> &per_dev) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
  if ((size_t)dev >= per_dev.size()) per_dev.resize((size_t)dev + 1);
  return per_dev[(size_t)dev];
}

#define CUDA_TRY(h, expr)                                                          \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      snprintf((h)->err, sizeof((h)->err), "%s:%d %s: %s", __FILE__, __LINE__, #expr, \
               cudaGetErrorString(_e));                                            \
      return FG_ERR_CUDA;                                                          \
    }                                                                              \
  } while (0)
