// Host shim of the solution-cost terms (csrc/cost.cuh) that fg_solution_cost's kernels and the trace record share:
// every factor of every non-ghost class, then every variable, summed per segment in order.  tests/test_trace_cpu.py.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/cost.cuh"

template <typename T>
static void cost_sums(const fg_class_t *classes, int32_t n_classes, const T *tables, const int32_t *edge_var,
                      const int32_t *value, const T *unary, const int64_t *unary_off, int32_t n_vars, T infinity,
                      const int32_t *factor_seg, const int32_t *var_seg, int32_t n_seg, double *out) {
  auto add = [&](int s, double c, double v) { if (s >= 0) { out[2 * s] += c; out[2 * s + 1] += v; } };
  for (int i = 0; i < n_classes; ++i) {
    const fg_class_t &c = classes[i];
    if (c.flags & FG_CLASS_GHOST) continue;
    for (int f = 0; f < c.n_factors; ++f) {
      double cst = 0.0, viol = 0.0;
      const int s = cost_factor_lane<T>(c, f, tables, edge_var, value, nullptr, infinity, factor_seg, n_seg, cst, viol);
      add(s, cst, viol);
    }
  }
  for (int v = 0; v < n_vars && unary; ++v) {
    double cst = 0.0, viol = 0.0;
    const int s = cost_var_lane<T>(v, n_vars, unary, unary_off, value, nullptr, infinity, var_seg, n_seg, cst, viol);
    add(s, cst, viol);
  }
}

extern "C" int64_t cost_host(int32_t precision, const fg_class_t *classes, int32_t n_classes, const void *tables,
                             const int32_t *edge_var, const int32_t *value, const void *unary,
                             const int64_t *unary_off, int32_t n_vars, double infinity, const int32_t *factor_seg,
                             const int32_t *var_seg, int32_t n_seg, double *out) {
  if (precision == FG_F64)
    cost_sums<double>(classes, n_classes, (const double *)tables, edge_var, value, (const double *)unary, unary_off,
                      n_vars, infinity, factor_seg, var_seg, n_seg, out);
  else
    cost_sums<float>(classes, n_classes, (const float *)tables, edge_var, value, (const float *)unary, unary_off,
                     n_vars, (float)infinity, factor_seg, var_seg, n_seg, out);
  return 0;
}
