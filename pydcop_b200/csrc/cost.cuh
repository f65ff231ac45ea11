// The per-factor and per-variable terms of the solution cost (dcop.py:319-367), shared by fg_solution_cost's kernels
// and the trace record (engine.cu), and the rule that keeps a trace's best row.  __host__ __device__, so
// tests/hostshim/cost_host.cpp and best_host.cpp run the same code on the CPU.  A term is (cost, violation): an entry equal to `infinity` (compared in the tables' precision) is one
// violation, any other entry is summed.
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"

template <typename T>
__host__ __device__ inline void cost_term(T t, T infinity, double &cst, double &viol) {
  if (t != infinity) cst = (double)t; else viol = 1.0;   // `r_cost != infinity`, dcop.py:355 and :363
}

// segment of item i (a class's factor first_factor + f, or a variable) or -1: seg NULL puts every item in segment 0,
// an id outside 0..n_seg-1 does not count
__host__ __device__ inline int cost_seg(int64_t i, const int32_t *seg, int32_t n_seg) {
  const int s = seg ? seg[i] : 0;
  return s < n_seg ? s : -1;
}

// factor f of class c (f >= c.n_factors: nothing): adds its term to (cst, viol) unless skipped, returns its segment
template <typename T>
__host__ __device__ inline int cost_factor_lane(const fg_class_t &c, int f, const T *tables, const int32_t *edge_var,
                                                const int32_t *value, const uint8_t *skip, T infinity,
                                                const int32_t *seg, int32_t n_seg, double &cst, double &viol) {
  if (f >= c.n_factors) return -1;
  const int s = cost_seg(c.first_factor + f, seg, n_seg);
  if (s < 0 || (skip && skip[c.first_factor + f])) return s;
  int64_t idx = 0, stride = 1;
  const int e0 = c.first_edge + f * c.arity;
  for (int i = c.arity - 1; i >= 0; --i) { idx += (int64_t)value[edge_var[e0 + i]] * stride; stride *= c.dom[i]; }
  cost_term<T>(tables[c.table_base + (int64_t)f * c.table_size + idx], infinity, cst, viol);
  return s;
}

// The anytime rule of fg_trace_set_best: a recorded (cost, violations) row replaces the best kept so far only when it
// is strictly better, so ties keep the earlier cycle.  Fewer violations win; at equal violations the cost decides
// (`<` in min mode, `>` in max mode), a NaN cost never beats a non-NaN one and any non-NaN cost beats a NaN best.
__host__ __device__ inline bool best_better(double cost, double viol, double best_cost, double best_viol,
                                            int32_t mode_max) {
  if (viol != best_viol) return viol < best_viol;
  if (cost != cost) return false;
  if (best_cost != best_cost) return true;
  return mode_max ? cost > best_cost : cost < best_cost;
}

// variable v (v >= n_vars: nothing): its own cost at its value, as cost_factor_lane
template <typename T>
__host__ __device__ inline int cost_var_lane(int v, int n_vars, const T *unary, const int64_t *unary_off,
                                             const int32_t *value, const uint8_t *skip, T infinity,
                                             const int32_t *seg, int32_t n_seg, double &cst, double &viol) {
  if (v >= n_vars) return -1;
  const int s = cost_seg(v, seg, n_seg);
  if (s < 0 || (skip && skip[v])) return s;
  cost_term<T>(unary[unary_off[v] + value[v]], infinity, cst, viol);
  return s;
}
