// TEST INFRASTRUCTURE: runs the SyncBB step logic of the CUDA kernel SOURCE (pydcop_b200/csrc/syncbb_kernels.cuh) on
// the CPU, so it can be compared with the oracle and the reference traces without a GPU.  The block-wide selections
// of k_syncbb become sequential scans over the candidates with the same predicates.  Nothing in the product links or
// calls this.
// The descriptor is the C-ABI's fg_syncbb_desc_t with HOST pointers.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/syncbb_kernels.cuh"

template <typename T>
static SbbSide<T> side(const fg_syncbb_desc_t *d) {
  return SbbSide<T>{d->n_vars, d->mode_max, d->dev_dom, d->dev_elt_ptr, d->dev_elt_pos, d->dev_elt_tab,
                    (const T *)d->dev_pair, (T *)d->dev_ub, d->dev_sel, d->dev_path_val, (T *)d->dev_path_cost,
                    (T *)d->dev_path_sum, (T *)d->dev_path_comp, d->dev_msg, (T *)d->dev_msg_ub, d->dev_count, d->dev_cycles};
}

template <typename T>
static void init_t(const fg_syncbb_desc_t *d) {
  gridDim = Dim3{1, 1, 1};
  blockDim = Dim3{1, 1, 1};
  blockIdx = Dim3{0, 0, 0};
  threadIdx = Dim3{0, 0, 0};
  k_syncbb_init<T>(side<T>(d));
}

// one launch of k_syncbb delivering up to n_steps messages
template <typename T>
static void steps_t(const fg_syncbb_desc_t *d, int64_t n_steps) {
  const SbbSide<T> g = side<T>(d);
  for (int64_t s = 0; s < n_steps && !g.msg[3]; ++s) {
    const int type = g.msg[0], p = g.msg[1];
    int x = -1;
    T cost = (T)0, best = (T)0;
    if (type != SBB_TERMINATE) {
      const int start = sbb_receive(g, type, p, *g.msg_ub);
      const T ub = g.ub[p];
      int stop = p;
      if (!g.mode_max)
        for (int q = 0; q < p; ++q)
          if (sbb_blocks(g, g.path_cost, p, q, ub)) { stop = q; break; }
      const bool last = type == SBB_FORWARD && p == g.n - 1;
      for (int c = start; c < g.dom[p]; ++c) {
        T my;
        if (!sbb_candidate(g, g.path_val, g.path_cost, p, c, stop, ub, &my)) continue;
        if (!last) { x = c; cost = my; break; }
        const T tot = p > 0 ? sbb_path_bound(g, p - 1) + my : my;
        if (sbb_pick(sbb_better(tot, ub, g.mode_max), tot, c, x >= 0, best, x, g.mode_max)) { x = c; best = tot; }
      }
    }
    sbb_transition(g, g.path_val, g.path_cost, type, p, x, cost, best);
  }
}

extern "C" {
void syncbb_host_init(const fg_syncbb_desc_t *d) {
  if (d->precision == FG_F64) init_t<double>(d);
  else init_t<float>(d);
}

void syncbb_host_step(const fg_syncbb_desc_t *d, int64_t n_steps) {
  if (d->precision == FG_F64) steps_t<double>(d, n_steps);
  else steps_t<float>(d, n_steps);
}
}  // extern "C"
