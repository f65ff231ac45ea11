// Host shim of the rule the trace record keeps each segment's best row by (csrc/cost.cuh's best_better), applied as
// k_trace_record applies it: row r of rows[n_rows][n_seg][2] replaces segment s's best when that has none yet or
// best_better says so.  tests/test_best_cpu.py.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/cost.cuh"

extern "C" int64_t best_host_better(double cost, double viol, double best_cost, double best_viol, int32_t mode_max) {
  return best_better(cost, viol, best_cost, best_viol, mode_max) ? 1 : 0;
}

// best: [n_seg * 2] (cost, violations), best_cycle: [n_seg] (1-based row, 0 = none), both written from scratch
extern "C" int64_t best_host_rows(const double *rows, int64_t n_rows, int32_t n_seg, int32_t mode_max, double *best,
                                  int64_t *best_cycle) {
  for (int s = 0; s < n_seg; ++s) best_cycle[s] = 0, best[2 * s] = best[2 * s + 1] = 0.0;
  for (int64_t r = 0; r < n_rows; ++r)
    for (int s = 0; s < n_seg; ++s) {
      const double c = rows[(r * n_seg + s) * 2], v = rows[(r * n_seg + s) * 2 + 1];
      if (best_cycle[s] == 0 || best_better(c, v, best[2 * s], best[2 * s + 1], mode_max)) {
        best[2 * s] = c;
        best[2 * s + 1] = v;
        best_cycle[s] = r + 1;
      }
    }
  return 0;
}
