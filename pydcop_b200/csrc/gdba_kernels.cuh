// GDBA kernels (included by gdba.cu).  One thread per variable, any arity / domain sizes.
// Free of CUDA runtime includes like mgm_kernels.cuh: tests/hostshim/gdba_host.cpp compiles this
// same file with g++ and runs every "thread" in a loop on the CPU (test infrastructure only).
//
// Floating-point operand order follows pydcop/algorithms/gdba.py (compute_eval_value :428-461):
//   eval(x)  = ((((0 + eff_0(x)) + vc_0) + eff_1(x)) + vc_1) + ...   constraints in node.constraints order
//   eff_k(x) = base + (T)m  (modifier A)  |  base * (T)m  (modifier M)
//   vc_k     = variable costs of the distinct variables in the scopes of constraints 0..k, the own one at
//              its CURRENT value: own cost, then the neighbours in order of first appearance (the
//              reference sums a set; its order is undefined)
//   improve  = eval(current) - best;  cost after a move = eval(current) + improve  (:522)
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"
#include "philox.cuh"

// MgmSide and k_mgm_init come from the MGM kernels' header, included with internal linkage as in
// mgm2_kernels.cuh (see the comment there: the includes above must stay above the namespace).
namespace {
#include "mgm_kernels.cuh"
}

// scope position of incidence e: the factor's first edge, v's position j and the table of factor f
struct GdbaSlot {
  const fg_class_t *c;
  int f, j, e0;
};

__device__ __forceinline__ GdbaSlot gdba_slot(const MgmSide &g, int e) {
  GdbaSlot s;
  s.c = &g.classes[g.edge_class[e]];
  const int le = e - s.c->first_edge;
  s.f = le / s.c->arity;
  s.j = le - s.f * s.c->arity;
  s.e0 = s.c->first_edge + s.f * s.c->arity;
  return s;
}

// entry index of the other scope variables at `val` (v's coordinate 0) and v's stride
__device__ __forceinline__ int64_t gdba_base_index(const MgmSide &g, const GdbaSlot &s,
                                                   const int32_t *__restrict__ val, int64_t &sv) {
  int64_t base = 0, stride = 1;
  sv = 0;
  for (int i = s.c->arity - 1; i >= 0; --i) {
    if (i == s.j) sv = stride;
    else base += (int64_t)val[g.edge_var[s.e0 + i]] * stride;
    stride *= s.c->dom[i];
  }
  return base;
}

// ok phase (gdba.py:352-387): evaluation of every value, violations at the current value, improve and
// the value an improving variable would take.  Modifier counts: increase_mode T, one per slot at
// mod[s] (mod_off == NULL); E / R / C, a table of the constraint's entries at mod + mod_off[s] for a
// slot whose constraint spans the variable's neighbourhood, none (mod_off[s] < 0) elsewhere.  PS: every variable reads
// its modifier and violation mode from its parameter set (var_pset); without, the instantiation is the one the runs
// without sets have always had.
template <typename T, bool PS>
__global__ void __launch_bounds__(128, 8)
k_gdba_eval(MgmSide g, int n_vars, const T *__restrict__ tables, const T *__restrict__ unary,
            const int64_t *__restrict__ unary_off, const T *__restrict__ viol_ref,
            const int32_t *__restrict__ mod, const int64_t *__restrict__ mod_off, int modifier_m, int violation,
            const int32_t *__restrict__ val, T *__restrict__ cost, uint8_t *__restrict__ has_cost,
            T *__restrict__ improve, int32_t *__restrict__ new_value, uint8_t *__restrict__ violated,
            int mode_max, uint64_t seed, uint32_t cycle, const uint16_t *__restrict__ var_pset,
            const fg_gdba_pset_t *__restrict__ psets) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  if (PS) {
    const fg_gdba_pset_t &p = fg_pset(var_pset, psets, v);
    modifier_m = p.modifier;
    violation = p.violation;
  }
  const int cur = val[v];
  const int d = g.dom_size[v];
  const int base_mod = modifier_m ? 1 : 0;
  T rel[FG_MAX_DOM];
  for (int x = 0; x < d; ++x) rel[x] = (T)0;
  T vc = unary[unary_off[v] + cur];
  int p = n0;  // next neighbour not yet seen (neighbours are listed in order of first appearance)
  for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) {
    const GdbaSlot sl = gdba_slot(g, g.slot_edge[s]);
    int64_t sv;
    const int64_t base = gdba_base_index(g, sl, val, sv);
    while (p < n1) {
      const int u = g.nbr_idx[p];
      bool in_scope = false;
      for (int i = 0; i < sl.c->arity; ++i) in_scope |= g.edge_var[sl.e0 + i] == u;
      if (!in_scope) break;
      vc = vc + unary[unary_off[u] + val[u]];
      ++p;
    }
    const T *t = tables + sl.c->table_base + (int64_t)sl.f * sl.c->table_size + base;
    const T bc = t[cur * sv];
    const T ref = violation == FG_GDBA_VIOLATION_NZ ? (T)0 : viol_ref[sl.c->first_factor + sl.f];
    violated[s] = violation == FG_GDBA_VIOLATION_MX ? (bc == ref) : (bc != ref);
    const int32_t *mt = nullptr;
    int32_t m0 = base_mod;
    if (!mod_off) m0 += mod[s];
    else if (mod_off[s] >= 0) mt = mod + mod_off[s] + base;
    for (int x = 0; x < d; ++x) {
      const T m = (T)(mt ? m0 + mt[x * sv] : m0);
      const T eff = modifier_m ? t[x * sv] * m : t[x * sv] + m;
      rel[x] = (rel[x] + eff) + vc;
    }
  }
  const T cst = rel[cur];
  cost[v] = cst;
  has_cost[v] = 1;
  // _compute_best_improvement (:395-417): the first value starts, strict improvement, ties in domain order
  T best = rel[0];
  int nbest = 1;
  for (int x = 1; x < d; ++x) {
    if (mode_max ? (rel[x] > best) : (rel[x] < best)) { best = rel[x]; nbest = 1; }
    else if (rel[x] == best) ++nbest;
  }
  const T gn = cst - best;
  improve[v] = gn;
  int nv = cur;
  if (mode_max ? (gn < (T)0) : (gn > (T)0)) {
    uint32_t b[4];
    philox_draw((uint32_t)g.var_id[v], cycle, 0u, fg_var_seed(g.var_seed, v, seed), b);
    int pick = philox_choice(b, nbest);
    for (int x = 0; x < d; ++x) {
      if (rel[x] == best) {
        if (pick == 0) { nv = x; break; }
        --pick;
      }
    }
  }
  new_value[v] = nv;
}

// improve phase (gdba.py:493-541): an improving variable moves when its improve is the largest of its
// neighbourhood (literal `>`, ties to the smallest name); a variable that cannot improve breaks out when
// the largest improve is 0 and raises its own modifiers on its violated constraints (:627-654).  The
// breakouts read this round's values from val_in; every variable writes its value for the next round to
// val_out, so nothing read in this launch is written in it.
template <typename T>
__global__ void __launch_bounds__(256)
k_gdba_decide(MgmSide g, int n_vars, const T *__restrict__ improve, const int32_t *__restrict__ new_value,
              const uint8_t *__restrict__ violated, int32_t *__restrict__ mod, const int64_t *__restrict__ mod_off,
              int increase_mode, int mode_max, const int32_t *__restrict__ val_in, int32_t *__restrict__ val_out,
              T *__restrict__ cost, uint8_t *__restrict__ breakout) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  const int cur = val_in[v];
  if (n0 == n1) {
    val_out[v] = cur;
    return;
  }
  const T mine = improve[v];
  T maxi = mine;
  for (int i = n0; i < n1; ++i) {
    const T gu = improve[g.nbr_idx[i]];
    if (gu > maxi) maxi = gu;
  }
  int nv = cur;
  uint8_t broke = 0;
  if (mode_max ? (mine < (T)0) : (mine > (T)0)) {
    bool move = mine == maxi;
    const int my_rank = g.var_rank[v];
    for (int i = n0; i < n1 && move; ++i) {
      const int u = g.nbr_idx[i];
      if (improve[u] == maxi && g.var_rank[u] < my_rank) move = false;
    }
    if (move) {
      nv = new_value[v];
      cost[v] = cost[v] + mine;
    }
  } else if (maxi == (T)0) {
    for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) {
      if (!violated[s]) continue;
      broke = 1;
      if (increase_mode == FG_GDBA_INCREASE_T) {
        mod[s] += 1;
        continue;
      }
      if (mod_off[s] < 0) continue;  // the write's key names the whole neighbourhood: never read here
      const GdbaSlot sl = gdba_slot(g, g.slot_edge[s]);
      int64_t sv;
      const int64_t base = gdba_base_index(g, sl, val_in, sv);
      int32_t *mt = mod + mod_off[s];
      const int d = g.dom_size[v];
      if (increase_mode == FG_GDBA_INCREASE_E) {
        mt[base + cur * sv] += 1;
      } else if (increase_mode == FG_GDBA_INCREASE_R) {
        for (int x = 0; x < d; ++x) mt[base + x * sv] += 1;
      } else {  // C: every entry with the own value at cur
        const int64_t outer = sl.c->table_size / (sv * d);
        for (int64_t hi = 0; hi < outer; ++hi)
          for (int64_t lo = 0; lo < sv; ++lo) mt[hi * sv * d + cur * sv + lo] += 1;
      }
    }
  }
  breakout[v] = broke;
  val_out[v] = nv;
}

// ---- launch sequences of fg_gdba_init / fg_gdba_step, shared with tests/hostshim/gdba_host.cpp -------------------
// L is a launcher (fg_launcher in handle.cuh, fg_host_launcher on the CPU); `classes` is the class table the kernels
// read.  fg_gdba_step runs gdba_cycle only when there are variables.

static inline MgmSide gdba_side(const fg_gdba_desc_t &d, const fg_class_t *classes) {
  return MgmSide{classes, d.dev_dom_size, d.dev_var_id, d.dev_var_rank, d.dev_edge_var, d.dev_edge_class,
                 d.dev_var_ptr, d.dev_slot_edge, d.dev_nbr_ptr, d.dev_nbr_idx, nullptr, d.dev_var_seed};
}

template <class L>
static void gdba_init(const fg_gdba_desc_t &d, const fg_class_t *classes, L &launch) {
  if (d.mod_size > 0) launch.fill(d.dev_mod, 0, sizeof(int32_t) * (size_t)d.mod_size);
  if (d.n_vars)
    launch(d.n_vars, 128, k_mgm_init, gdba_side(d, classes), d.n_vars, d.dev_init_value, d.seed, d.dev_value[0],
           d.dev_has_cost);
}

// round done + 1
template <typename T, class L>
static void gdba_cycle(const fg_gdba_desc_t &d, const fg_class_t *classes, int64_t done, L &launch) {
  const MgmSide g = gdba_side(d, classes);
  const uint32_t cyc = (uint32_t)(done + 1);
  const int n = d.n_vars;
  int32_t *vin = d.dev_value[done & 1], *vout = d.dev_value[(done + 1) & 1];
  const int64_t *mod_off = d.increase_mode == FG_GDBA_INCREASE_T ? nullptr : d.dev_mod_off;
  launch(n, 128, d.dev_var_pset ? k_gdba_eval<T, true> : k_gdba_eval<T, false>, g, n, (const T *)d.dev_tables,
         (const T *)d.dev_unary, d.dev_unary_off, (const T *)d.dev_viol_ref, d.dev_mod, mod_off, d.modifier,
         d.violation, vin, (T *)d.dev_cost, d.dev_has_cost, (T *)d.dev_improve, d.dev_new_value, d.dev_violated,
         d.mode_max, d.seed, cyc, d.dev_var_pset, d.psets);
  launch(n, 256, k_gdba_decide<T>, g, n, (const T *)d.dev_improve, d.dev_new_value, d.dev_violated, d.dev_mod,
         mod_off, d.increase_mode, d.mode_max, vin, vout, (T *)d.dev_cost, d.dev_breakout);
}
