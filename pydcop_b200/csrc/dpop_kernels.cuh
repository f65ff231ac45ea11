// DPOP kernels (pydcop/algorithms/dpop.py:115-441): UTIL propagation up the pseudo-tree and VALUE
// propagation down it, on the schedule pydcop_b200/pseudotree.py computes.  Included by dpop.cu and, on
// the CPU, by tests/hostshim/dpop_host.cpp.
//
// A node u's joined table has the dims {u} + separator(u).  Its entry for own value v at separator
// digits dig[] is the left-associated f64 (or f32) sum, adds only (the build uses -fmad=false):
//     unary[u][v] + child_1 + ... + child_k + constraint_1 + ... + constraint_m
// with the children in the pseudo-tree's children order and the constraints u owns in constraint order
// (dpop.py:204-210, :332, :381-382).  Term t reads  data_t[base_t + v * own_t + sum_j dig[pos_tj] * stride_tj].
//
// Projection / argopt (find_arg_optimal, relations.py:1554-1591): the running best starts at the int32
// sentinel, 2147483647 (min) or -2147483648 (max), not at +-inf; an entry replaces it when strictly better,
// so NaN never wins; the chosen value is the first in domain order whose entry equals the final best.  When
// none does (every entry worse than the sentinel, or NaN) the reference raises IndexError (dpop.py:358,
// :422); the VALUE kernel takes value 0, writes cost NaN and counts the node instead.
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"

#ifndef __CUDACC__
#include <cmath>
#endif

#define FG_DPOP_MAX_SEP 32

struct DpopNodes {
  const int32_t *dom_size;      // [V] canonical variable order
  const int64_t *unary_off;     // [V] start of the variable's own costs in `unary`
  const int64_t *util_off;      // [V] start of the node's UTIL in the arena
  const int64_t *util_size;     // [V] entries of the node's UTIL (product of the separator's domains)
  const int32_t *sep_ptr;       // [V+1]
  const int32_t *sep_var;       // separator, root side first; UTIL entries are row-major over it
  const int32_t *term_ptr;      // [V+1]
  const int32_t *term_kind;     // 0: child UTIL in the arena, 1: constraint table
  const int64_t *term_base;
  const int64_t *term_own;      // stride along the node's own value
  const int32_t *tdim_ptr;      // [n_terms+1]
  const int32_t *tdim_pos;      // separator position of each (dim, stride) pair
  const int64_t *tdim_stride;
};

template <typename T>
struct DpopData {
  const T *unary;
  const T *tables;
  T *arena;
};

template <typename T>
__host__ __device__ __forceinline__ T dpop_sentinel(int mode_max) {
  return mode_max ? (T)-2147483648.0 : (T)2147483647.0;
}

template <typename T>
__host__ __device__ __forceinline__ bool dpop_better(T e, T best, int mode_max) {
  return mode_max ? e > best : e < best;
}

// Joined entries of node u at separator digits dig[] for own values v0, v0 + vstep, ...: the best of
// them against the sentinel and the first value reaching it (-1: none does).
template <typename T>
__host__ __device__ __forceinline__ T dpop_row(const DpopNodes &g, const DpopData<T> &a, int u,
                                               const int32_t *dig, int v0, int vstep, int mode_max,
                                               int *arg) {
  const int d = g.dom_size[u];
  const T *un = a.unary + g.unary_off[u];
  const int t0 = g.term_ptr[u], t1 = g.term_ptr[u + 1];
  T best = dpop_sentinel<T>(mode_max);
  int first = -1;
  for (int v = v0; v < d; v += vstep) {
    T e = un[v];
    for (int t = t0; t < t1; ++t) {
      int64_t off = g.term_base[t] + (int64_t)v * g.term_own[t];
      for (int j = g.tdim_ptr[t]; j < g.tdim_ptr[t + 1]; ++j) off += (int64_t)dig[g.tdim_pos[j]] * g.tdim_stride[j];
      e = e + (g.term_kind[t] ? a.tables[off] : a.arena[off]);
    }
    if (dpop_better(e, best, mode_max)) {
      best = e;
      first = v;
    } else if (e == best && first < 0) {
      first = v;
    }
  }
  *arg = first;
  return best;
}

// UTIL entry `idx` of node u: the projection of its joined table over u (relations.py:1717-1756).
template <typename T>
__host__ __device__ __forceinline__ void dpop_util_entry(const DpopNodes &g, const DpopData<T> &a, int u,
                                                         int64_t idx, int mode_max) {
  int32_t dig[FG_DPOP_MAX_SEP];
  const int s0 = g.sep_ptr[u], s1 = g.sep_ptr[u + 1];
  int64_t r = idx;
  for (int k = s1 - s0 - 1; k >= 0; --k) {
    const int dk = g.dom_size[g.sep_var[s0 + k]];
    dig[k] = (int32_t)(r % dk);
    r /= dk;
  }
  int arg;
  a.arena[g.util_off[u] + idx] = dpop_row(g, a, u, dig, 0, 1, mode_max, &arg);
}

// Separator digits of node u from the values its ancestors chose (the VALUE message, dpop.py:411-417).
__host__ __device__ __forceinline__ void dpop_value_digits(const DpopNodes &g, int u, const int32_t *value,
                                                           int32_t *dig) {
  const int s0 = g.sep_ptr[u], s1 = g.sep_ptr[u + 1];
  for (int k = 0; k < s1 - s0; ++k) dig[k] = value[g.sep_var[s0 + k]];
}

// The outcome of a VALUE node from its row's best and first arg: value index and cost, or value 0, cost
// NaN and one more unresolved node.
template <typename T>
__host__ __device__ __forceinline__ void dpop_value_store(int u, T best, int arg, int32_t *value, T *cost,
                                                          int32_t *unresolved) {
  if (arg < 0) {
    value[u] = 0;
    cost[u] = (T)NAN;
#ifdef __CUDA_ARCH__
    atomicAdd(unresolved, 1);
#else
    ++*unresolved;
#endif
  } else {
    value[u] = arg;
    cost[u] = best;
  }
}

// The whole VALUE step of node u on one thread (the host shim's reference of the warp kernel below).
template <typename T>
__host__ __device__ __forceinline__ void dpop_value_node(const DpopNodes &g, const DpopData<T> &a, int u,
                                                         int mode_max, int32_t *value, T *cost,
                                                         int32_t *unresolved) {
  int32_t dig[FG_DPOP_MAX_SEP];
  dpop_value_digits(g, u, value, dig);
  int arg;
  const T best = dpop_row(g, a, u, dig, 0, 1, mode_max, &arg);
  dpop_value_store(u, best, arg, value, cost, unresolved);
}

#ifdef __CUDACC__
// One warp per UTIL segment: the segment's nodes bottom-up, the lanes over each node's UTIL entries.
template <typename T>
__global__ void __launch_bounds__(128) k_dpop_util_walk(DpopNodes g, DpopData<T> a, const int32_t *nodes,
                                                        const int32_t *seg_ptr, int seg0, int n_seg,
                                                        int mode_max) {
  const int w = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n_seg) return;
  const int s = seg0 + w;
  for (int i = seg_ptr[s]; i < seg_ptr[s + 1]; ++i) {
    const int u = nodes[i];
    const int64_t n = g.util_size[u];
    for (int64_t idx = lane; idx < n; idx += 32) dpop_util_entry(g, a, u, idx, mode_max);
    __syncwarp();   // the parent, next in the segment, reads this UTIL from other lanes
  }
}

// A big node: its UTIL entries over the whole grid.
template <typename T>
__global__ void __launch_bounds__(256) k_dpop_util_big(DpopNodes g, DpopData<T> a, int u, int mode_max) {
  const int64_t n = g.util_size[u];
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x)
    dpop_util_entry(g, a, u, idx, mode_max);
}

template <typename T>
__device__ __forceinline__ T dpop_shfl_xor(T x, int m) {
  return __shfl_xor_sync(0xffffffffu, x, m);
}

// One warp per heavy path, top-down: the lanes split the node's own values, then a warp reduction keeps
// the best (exact: a selection) and the lowest value index reaching it.
template <typename T>
__global__ void __launch_bounds__(128) k_dpop_value_walk(DpopNodes g, DpopData<T> a, const int32_t *nodes,
                                                         const int32_t *seg_ptr, int seg0, int n_seg,
                                                         int mode_max, int32_t *value, T *cost,
                                                         int32_t *unresolved) {
  const int w = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n_seg) return;
  const int s = seg0 + w;
  int32_t dig[FG_DPOP_MAX_SEP];
  for (int i = seg_ptr[s]; i < seg_ptr[s + 1]; ++i) {
    const int u = nodes[i];
    dpop_value_digits(g, u, value, dig);
    int arg;
    T best = dpop_row(g, a, u, dig, lane, 32, mode_max, &arg);
    const T lane_best = best;
    for (int m = 16; m; m >>= 1) {
      const T o = dpop_shfl_xor(best, m);
      if (dpop_better(o, best, mode_max)) best = o;
    }
    int cand = (arg >= 0 && lane_best == best) ? arg : 0x7fffffff;
    for (int m = 16; m; m >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, m));
    // the cost is the chosen value's own entry (0.0 and -0.0 compare equal)
    best = __shfl_sync(0xffffffffu, lane_best, cand == 0x7fffffff ? 0 : cand & 31);
    if (lane == 0) dpop_value_store(u, best, cand == 0x7fffffff ? -1 : cand, value, cost, unresolved);
    __syncwarp();   // the next node down reads this value
  }
}
#endif
