// MGM value phase, fast shape (opt-in, DESIGN.md §10): every constraint binary over ONE domain size D.
// Same arithmetic and results as k_mgm_gain (mgm_kernels.cuh); the table of each incidence is read
// ORIENTED (the DSA fast-path arrays, engine.py::dsa_fast_arrays: row y = value of the neighbour is
// contiguous over my values) so an incidence costs one contiguous row instead of D strided reads, and
// the slot loop handles U incidences per trip.
// Free of CUDA runtime includes (tests/hostshim/ runs it on the CPU).
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"
#include "row_load.cuh"       // fg_load_row
#include "mgm_kernels.cuh"     // MgmSide

template <typename T, int D, int U>
__global__ void __launch_bounds__(128)
k_mgm_gain_bin(MgmSide g, int n_vars, const int32_t *__restrict__ slot_nbr, const int64_t *__restrict__ slot_tab,
               const T *__restrict__ tables_or, const T *__restrict__ unary, const int32_t *__restrict__ val,
               T *__restrict__ cost, uint8_t *__restrict__ has_cost, T *__restrict__ gain,
               int32_t *__restrict__ new_val, int mode_max, uint64_t seed, uint32_t cycle) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  const int cur = val[v];
  T rel[D];
#pragma unroll
  for (int x = 0; x < D; ++x) rel[x] = (T)0;
  const int s0 = g.var_ptr[v], s1 = g.var_ptr[v + 1];
  for (int s = s0; s < s1; s += U) {
    int nb[U];
    int64_t tb[U];
    bool ok[U];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      ok[i] = s + i < s1;
      const int si = ok[i] ? s + i : s;
      nb[i] = slot_nbr[si];
      tb[i] = slot_tab[si];
    }
    int y[U];
#pragma unroll
    for (int i = 0; i < U; ++i) y[i] = val[nb[i]];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      T r[D];
      fg_load_row_padded<T, D>(tables_or + tb[i] + (int64_t)y[i] * fg_row_stride<T, D>(), r);
      const bool first = (s + i == s0);   // ((f1 + f2) + f3)...: the first constraint starts the sum (mgm.py:443)
#pragma unroll
      for (int x = 0; x < D; ++x) {
        const T nc = rel[x] + r[x];
        rel[x] = first ? r[x] : (ok[i] ? nc : rel[x]);
      }
    }
  }
  const T own = unary[g.unary_off[v] + cur];
  T cst;
  if (!has_cost[v]) {  // first round: current_cost (mgm.py:349-368); rel[cur] without a dynamic register index
    T rc = (T)0;
#pragma unroll
    for (int x = 0; x < D; ++x) rc = (x == cur) ? rel[x] : rc;
    cst = rc;
    cst += own;
    for (int i = n0; i < n1; ++i) {
      const int u = g.nbr_idx[i];
      cst += unary[g.unary_off[u] + val[u]];
    }
    cost[v] = cst;
    has_cost[v] = 1;
  } else {
    cst = cost[v];
  }
  T best = mode_max ? (T)-2147483648.0 : (T)2147483647.0;  // find_arg_optimal, relations.py:1554-1591
  int nbest = 0;
#pragma unroll
  for (int x = 0; x < D; ++x) {
    const T c = rel[x];
    if (mode_max ? (best < c) : (best > c)) { best = c; nbest = 1; }
    else if (c == best) ++nbest;
  }
  T evaluation = best + own;  // own cost at the CURRENT value (mgm.py:449)
  for (int i = n0; i < n1; ++i) {
    const int u = g.nbr_idx[i];
    evaluation += unary[g.unary_off[u] + val[u]];
  }
  const T gn = cst - evaluation;
  gain[v] = gn;
  int nv = cur;
  if (mode_max ? (gn < (T)0) : (gn > (T)0)) {  // mgm.py:382-385
    uint32_t b[4];
    philox_draw((uint32_t)g.var_id[v], cycle, 0u, fg_var_seed(g.var_seed, v, seed), b);
    int pick = philox_choice(b, nbest);
    bool done = false;
#pragma unroll
    for (int x = 0; x < D; ++x) {
      if (!done && rel[x] == best) {
        if (pick == 0) { nv = x; done = true; }
        --pick;
      }
    }
  }
  new_val[v] = nv;
}

// ---- launch sequences of fg_mgm_init / fg_mgm_step, shared with tests/hostshim/mgm_host.cpp ----------------------
// Here rather than in mgm_kernels.cuh because the value phase picks between both headers' kernels.  L is a launcher
// (fg_launcher in handle.cuh, fg_host_launcher on the CPU); `classes` is the class table the kernels read.  The entry
// points run them only when there are variables.  mgm.cu tries the active-row value phase (mgm_cached_kernels.cuh)
// before mgm_gain.

static inline MgmSide mgm_side(const fg_mgm_desc_t &d, const fg_class_t *classes) {
  return MgmSide{classes, d.dev_dom_size, d.dev_var_id, d.dev_var_rank, d.dev_edge_var, d.dev_edge_class,
                 d.dev_var_ptr, d.dev_slot_edge, d.dev_nbr_ptr, d.dev_nbr_idx, d.dev_unary_off, d.dev_var_seed};
}

// the descriptor carries the oriented tables in a shape k_mgm_gain_bin is compiled for
static inline bool mgm_fast_shape(const fg_mgm_desc_t &d) {
  if (!d.dev_tables_or || !d.dev_slot_nbr || !d.dev_slot_tab || (d.fast_chunk != 2 && d.fast_chunk != 4)) return false;
  return d.fast_dom == 4 || d.fast_dom == 8 || d.fast_dom == 10 || d.fast_dom == 16 || d.fast_dom == 20;
}

template <class L>
static void mgm_init(const fg_mgm_desc_t &d, const fg_class_t *classes, L &launch) {
  launch(d.n_vars, 128, k_mgm_init, mgm_side(d, classes), d.n_vars, d.dev_init_value, d.seed, d.dev_value,
         d.dev_has_cost);
}

template <typename T, int D, class L>
static void mgm_gain_bin(const fg_mgm_desc_t &d, const MgmSide &g, uint32_t cyc, L &launch) {
  launch(d.n_vars, 128, d.fast_chunk == 2 ? k_mgm_gain_bin<T, D, 2> : k_mgm_gain_bin<T, D, 4>, g, d.n_vars,
         d.dev_slot_nbr, d.dev_slot_tab, (const T *)d.dev_tables_or, (const T *)d.dev_unary, d.dev_value,
         (T *)d.dev_cost, d.dev_has_cost, (T *)d.dev_gain, d.dev_new_value, d.mode_max, d.seed, cyc);
}

// value phase of round done + 1: the oriented tables when mgm_fast_shape, else the generic kernel
template <typename T, class L>
static void mgm_gain(const fg_mgm_desc_t &d, const fg_class_t *classes, int64_t done, L &launch) {
  const MgmSide g = mgm_side(d, classes);
  const uint32_t cyc = (uint32_t)(done + 1);
  if (mgm_fast_shape(d)) {
    switch (d.fast_dom) {
      case 4: mgm_gain_bin<T, 4>(d, g, cyc, launch); return;
      case 8: mgm_gain_bin<T, 8>(d, g, cyc, launch); return;
      case 10: mgm_gain_bin<T, 10>(d, g, cyc, launch); return;
      case 16: mgm_gain_bin<T, 16>(d, g, cyc, launch); return;
      default: mgm_gain_bin<T, 20>(d, g, cyc, launch); return;
    }
  }
  launch(d.n_vars, 128, k_mgm_gain<T>, g, d.n_vars, (const T *)d.dev_tables, (const T *)d.dev_unary, d.dev_value,
         (T *)d.dev_cost, d.dev_has_cost, (T *)d.dev_gain, d.dev_new_value, d.mode_max, d.seed, cyc);
}

// gain phase
template <typename T, class L>
static void mgm_decide(const fg_mgm_desc_t &d, const fg_class_t *classes, L &launch) {
  launch(d.n_vars, 256, k_mgm_decide<T>, mgm_side(d, classes), d.n_vars, (const T *)d.dev_gain, d.dev_new_value,
         d.dev_value, (T *)d.dev_cost);
}
