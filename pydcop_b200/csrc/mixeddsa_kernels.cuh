// MixedDSA kernels (included by mixeddsa.cu).  One thread per variable, any arity / domain sizes.  Free of CUDA
// runtime includes like gdba_kernels.cuh: tests/hostshim/mixeddsa_host.cpp compiles this same file with g++ and runs
// every "thread" in a loop on the CPU.
//
// Floating-point operand order follows pydcop/algorithms/mixeddsa.py (_compute_dcop_cost :410-446), per candidate x
// with the neighbours at their values of the previous round:
//   C(x) = ((((0 + soft_1(x)) + soft_2(x) + ...) + vc(own, x)) + vc(n_1) + ...) + hard_1(x) + ...
//          soft and hard slots each in node.constraints order (the host puts the soft slots first, see
//          fg_mixeddsa_desc_t); a hard entry equal to +inf is not added but counted in H(x) instead.  The
//          variable costs are those of `concerned_vars`, a set the reference sums in hash order: here the own
//          variable, then the distinct neighbours in order of first appearance; a variable without any
//          constraint has no such term.
//   best   = smallest H first, then C with a strict < (> in max mode), ties in domain order (:381-402)
//   dH = H(cur) - H_best, dC = C(cur) - C_best; the decision of :300-358 (a NaN dC makes no move).
#pragma once
#include <stdint.h>

#include <limits>

#include "../../include/pydcop_b200.h"
#include "philox.cuh"

// MgmSide (the neighbourhood arrays) comes from the MGM kernels' header, included with internal linkage as in
// gdba_kernels.cuh.
namespace {
#include "mgm_kernels.cuh"
}

// Largest domain over the constraint classes: every variable with a constraint has a slot in one of them, and a
// variable without any never builds candidate arrays.  k_mixeddsa_step keeps one cost and one count per value on its
// stack, so instances whose domains are all <= 32 run the DMAX = 32 instance (384 B of stack per thread in f64
// instead of 3 KB).
static inline int mixeddsa_dmax(const fg_class_t *classes, int n_classes) {
  int m = 1;
  for (int c = 0; c < n_classes; ++c)
    for (int i = 0; i < classes[c].arity; ++i) m = classes[c].dom[i] > m ? classes[c].dom[i] : m;
  return m <= 32 ? 32 : FG_MAX_DOM;
}

// on_start (:231-255): EVERY variable takes its initial value or a draw (unlike DSA, isolated ones too); no cost yet
__global__ void k_mixeddsa_init(MgmSide g, int n_vars, const int32_t *__restrict__ init_value, uint64_t seed,
                                int32_t *__restrict__ value, uint8_t *__restrict__ has_cost) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  has_cost[v] = 0;
  if (init_value && init_value[v] >= 0) {
    value[v] = init_value[v];
    return;
  }
  uint32_t b[4];
  philox_draw((uint32_t)g.var_id[v], FG_PHILOX_INIT_CYCLE, 0u, fg_var_seed(g.var_seed, v, seed), b);
  value[v] = philox_choice(b, g.dom_size[v]);
}

// table of slot s (v at scope position j) with the other scope variables at `val`, and v's stride in it
template <typename T>
__device__ __forceinline__ const T *mixeddsa_row(const MgmSide &g, int s, const T *__restrict__ tables,
                                                 const int32_t *__restrict__ val, int64_t &sv, int &factor) {
  const int e = g.slot_edge[s];
  const fg_class_t &c = g.classes[g.edge_class[e]];
  const int le = e - c.first_edge;
  const int f = le / c.arity, j = le - f * c.arity;
  const int e0 = c.first_edge + f * c.arity;
  int64_t base = 0, stride = 1;
  sv = 0;
  for (int i = c.arity - 1; i >= 0; --i) {
    if (i == j) sv = stride;
    else base += (int64_t)val[g.edge_var[e0 + i]] * stride;
    stride *= c.dom[i];
  }
  factor = c.first_factor + f;
  return tables + c.table_base + (int64_t)f * c.table_size + base;
}

// One round (_on_neighbors_values :272-373) for every variable; every dom_size of a variable with a constraint is
// <= DMAX.  `inf` is +infinity in T (the hard test is `entry == INFINITY`, :438).  Writes the next value of every
// variable to val_out, so nothing read in this launch is written in it.
template <typename T, int DMAX>
__global__ void __launch_bounds__(128)
k_mixeddsa_step(MgmSide g, int n_vars, const T *__restrict__ tables, const T *__restrict__ unary,
                const int32_t *__restrict__ soft_end, const T *__restrict__ con_opt, const int32_t *__restrict__ val,
                int32_t *__restrict__ val_out, T *__restrict__ cost, uint8_t *__restrict__ has_cost,
                int32_t *__restrict__ h_best, uint8_t *__restrict__ branch, int mode_max, int variant,
                double proba_hard, double proba_soft, T inf, uint64_t seed, uint32_t cycle) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int cur = val[v];
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  const int s0 = g.var_ptr[v], sm = soft_end[v], s1 = g.var_ptr[v + 1];
  val_out[v] = cur;
  // without neighbours the reference evaluates once, from on_start, with cycle_count 1 (:372-373)
  if (n0 == n1 && cycle != 1u) {
    h_best[v] = -1;
    branch[v] = FG_MIXEDDSA_BRANCH_NONE;
    return;
  }
  if (s0 == s1) {  // no constraint: every candidate costs 0 with H 0, nothing is violated, no move
    h_best[v] = 0;
    branch[v] = FG_MIXEDDSA_BRANCH_IDLE;
    return;
  }
  const int d = g.dom_size[v];
  T c[DMAX];
  int32_t nh[DMAX];
  for (int x = 0; x < d; ++x) {
    c[x] = (T)0;
    nh[x] = 0;
  }
  bool soft_violated = false;  // exists_violated_soft_constraint (:464-476), function-relation meaning
  for (int s = s0; s < sm; ++s) {
    int64_t sv;
    int f;
    const T *t = mixeddsa_row(g, s, tables, val, sv, f);
    for (int x = 0; x < d; ++x) c[x] = c[x] + t[x * sv];
    soft_violated |= t[cur * sv] != con_opt[f];
  }
  const T *own = unary + g.unary_off[v];
  for (int x = 0; x < d; ++x) c[x] = c[x] + own[x];
  for (int i = n0; i < n1; ++i) {
    const int u = g.nbr_idx[i];
    const T cu = unary[g.unary_off[u] + val[u]];
    for (int x = 0; x < d; ++x) c[x] = c[x] + cu;
  }
  for (int s = sm; s < s1; ++s) {
    int64_t sv;
    int f;
    const T *t = mixeddsa_row(g, s, tables, val, sv, f);
    for (int x = 0; x < d; ++x) {
      const T e = t[x * sv];
      if (e == inf) ++nh[x];
      else c[x] = c[x] + e;
    }
  }
  // _compute_best_value: starts at H = len(hard) + 1, so the first value always sets the best
  int hb = s1 - sm + 1, first = 0, nbest = 0;
  T cb = (T)0;
  for (int x = 0; x < d; ++x) {
    if (nh[x] < hb) {
      hb = nh[x]; cb = c[x]; first = x; nbest = 1;
    } else if (nh[x] == hb) {
      if (mode_max ? (c[x] > cb) : (c[x] < cb)) { cb = c[x]; first = x; nbest = 1; }
      else if (c[x] == cb) ++nbest;
    }
  }
  const int dh = nh[cur] - hb;
  const T dc = c[cur] - cb;
  int br = FG_MIXEDDSA_BRANCH_IDLE;
  double p = 0.0;  // the probability the draw is tested against (0: no draw)
  bool drop_cur = false;
  if (dh > 0) {
    br = FG_MIXEDDSA_BRANCH_HARD;
    p = proba_hard;
  } else if (dh == 0) {
    if (mode_max ? (dc < (T)0) : (dc > (T)0)) {
      br = FG_MIXEDDSA_BRANCH_SOFT;
      p = proba_soft;
    } else if (dc == (T)0) {
      // the current value is then one of the best (its (H, C) equals the best's, C not NaN): it is removed
      if (hb > 0) {
        br = FG_MIXEDDSA_BRANCH_STUCK_HARD;
        p = nbest > 1 ? proba_hard : 0.0;
        drop_cur = true;
      } else if (soft_violated && variant != FG_DSA_A) {  // variant C takes B's branch (:342 is unreachable)
        br = FG_MIXEDDSA_BRANCH_STUCK_SOFT;
        p = nbest > 1 ? proba_soft : 0.0;
        drop_cur = true;
      }
    }
  }
  int moved = 0;
  if (p > 0.0) {
    uint32_t b[4];
    philox_draw((uint32_t)g.var_id[v], cycle, 0u, fg_var_seed(g.var_seed, v, seed), b);
    if (p > philox_u53(b)) {
      // bests: `first` (the value that set the best last) and every later value with the same (H, C)
      int pick = philox_choice(b, drop_cur ? nbest - 1 : nbest);
      int nv = cur;
      for (int x = first; x < d; ++x) {
        if ((x == first || (nh[x] == hb && c[x] == cb)) && !(drop_cur && x == cur)) {
          if (pick == 0) { nv = x; break; }
          --pick;
        }
      }
      val_out[v] = nv;
      cost[v] = hb > 0 ? inf : cb;  // value_selection(choice, eff_cost) (:448-462)
      has_cost[v] = 1;
      moved = FG_MIXEDDSA_MOVED;
    }
  }
  h_best[v] = hb;
  branch[v] = (uint8_t)(br | moved);
}

// ---- launch sequences of fg_mixeddsa_init / fg_mixeddsa_step, shared with tests/hostshim/mixeddsa_host.cpp --------
// L is a launcher (fg_launcher in handle.cuh, fg_host_launcher on the CPU); `classes` is the class table the kernels
// read; `dmax` is mixeddsa_dmax of the class table.  k_dsa_con_opt comes from dsa_generic.cuh, which the includer
// includes first.

static inline MgmSide mixeddsa_side(const fg_mixeddsa_desc_t &d, const fg_class_t *classes) {
  return MgmSide{classes, d.dev_dom_size, d.dev_var_id, nullptr, d.dev_edge_var, d.dev_edge_class,
                 d.dev_var_ptr, d.dev_slot_edge, d.dev_nbr_ptr, d.dev_nbr_idx, d.dev_unary_off, d.dev_var_seed};
}

template <typename T, class L>
static void mixeddsa_init(const fg_mixeddsa_desc_t &d, const fg_class_t *classes, L &launch) {
  for (int ci = 0; ci < d.n_classes; ++ci) {
    const fg_class_t &c = d.classes[ci];
    if (c.n_factors)
      launch(c.n_factors, 128, k_dsa_con_opt<T>, c, (const T *)d.dev_tables, (T *)d.dev_con_opt, d.mode_max);
  }
  if (d.n_vars)
    launch(d.n_vars, 128, k_mixeddsa_init, mixeddsa_side(d, classes), d.n_vars, d.dev_init_value, d.seed,
           d.dev_value[0], d.dev_has_cost);
}

// round done + 1
template <typename T, class L>
static void mixeddsa_cycle(const fg_mixeddsa_desc_t &d, const fg_class_t *classes, int dmax, int64_t done, L &launch) {
  int32_t *vin = d.dev_value[done & 1], *vout = d.dev_value[(done + 1) & 1];
  launch(d.n_vars, 128, dmax <= 32 ? k_mixeddsa_step<T, 32> : k_mixeddsa_step<T, FG_MAX_DOM>,
         mixeddsa_side(d, classes), d.n_vars, (const T *)d.dev_tables, (const T *)d.dev_unary, d.dev_soft_end,
         (const T *)d.dev_con_opt, vin, vout, (T *)d.dev_cost, d.dev_has_cost, d.dev_h_best, d.dev_branch, d.mode_max,
         d.variant, d.proba_hard, d.proba_soft, std::numeric_limits<T>::infinity(), d.seed, (uint32_t)(done + 1));
}
