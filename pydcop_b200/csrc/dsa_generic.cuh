// Generic DSA kernels (any arity / domain sizes): one thread per variable.
#pragma once
#include "common.cuh"
#include "philox.cuh"

struct DsaSide {
  const fg_class_t *classes;  // device copy of the class table
  const int32_t *dom_size, *var_id, *edge_var, *edge_class, *var_ptr, *slot_edge;
  const uint8_t *has_nbr;
  const double *prob;
  const uint64_t *var_seed;  // [n_vars] Philox key of each variable, NULL: the run's seed
  const uint16_t *var_pset;  // [n_vars] parameter set of each variable, NULL: the descriptor's scalars
  const fg_dsa_pset_t *psets;
};

// find_optimum (relations.py:1367-1400): optimum of the whole table of each constraint
template <typename T>
__global__ void k_dsa_con_opt(const fg_class_t c, const T *__restrict__ tables, T *__restrict__ con_opt,
                              int mode_max) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= c.n_factors) return;
  const T *t = tables + c.table_base + (int64_t)f * c.table_size;
  T o = t[0];
  for (int64_t i = 1; i < c.table_size; ++i) {
    T x = t[i];
    if (mode_max ? (x > o) : (x < o)) o = x;
  }
  con_opt[c.first_factor + f] = o;
}

// on_start (dsa.py:277-295): injected random initial value for connected variables
__global__ void k_dsa_init(DsaSide g, int n_vars, uint64_t seed, int32_t *__restrict__ value) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || g.has_nbr[v] != 1) return;
  uint32_t b[4];
  philox_draw((uint32_t)g.var_id[v], FG_PHILOX_INIT_CYCLE, 0u, fg_var_seed(g.var_seed, v, seed), b);
  value[v] = philox_choice(b, g.dom_size[v]);
}

// evaluate_cycle (dsa.py:320-357) for every variable.  PS: every variable reads its variant from its parameter set
// (g.var_pset); without, the instantiation is the one the runs without sets have always had.
template <typename T, bool PS>
__global__ void __launch_bounds__(128)
k_dsa_step_generic(DsaSide g, int n_vars, const T *__restrict__ tables,
                   const T *__restrict__ con_opt, const int32_t *__restrict__ val,
                   int32_t *__restrict__ val_next, T *__restrict__ val_cost, int mode_max,
                   int variant, uint64_t seed, uint32_t cycle, const T *__restrict__ var_cost = nullptr,
                   const int64_t *__restrict__ unary_off = nullptr) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int cur = val[v];
  const uint8_t hn = g.has_nbr[v];  // 0 isolated (value carried over), 1 active, 2 ghost of another rank's variable:
  if (hn != 1) {                    // never written here — its owner's push / the halo unpack fills `next`
    if (hn == 0) val_next[v] = cur;
    return;
  }
  if (PS) variant = fg_pset(g.var_pset, g.psets, v).variant;
  const int d = g.dom_size[v];
  T cost[FG_MAX_DOM];
  for (int x = 0; x < d; ++x) cost[x] = (T)0;
  bool violated = false;
  for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) {
    const int e = g.slot_edge[s];
    const fg_class_t &c = g.classes[g.edge_class[e]];
    const int le = e - c.first_edge;
    const int f = le / c.arity, j = le - f * c.arity;
    const int e0 = c.first_edge + f * c.arity;
    int64_t base = 0, stride = 1, stride_j = 0;
    for (int i = c.arity - 1; i >= 0; --i) {
      if (i == j) stride_j = stride;
      else base += (int64_t)val[g.edge_var[e0 + i]] * stride;
      stride *= c.dom[i];
    }
    const T *t = tables + c.table_base + (int64_t)f * c.table_size + base;
    for (int x = 0; x < d; ++x) cost[x] += t[x * stride_j];  // assignment_cost, relations.py:1479
    if (variant == FG_DSA_B && t[cur * stride_j] != con_opt[c.first_factor + f]) violated = true;
  }
  // A-DSA (adsa.py:344-377): the candidates carry the variable's own cost, the current cost (adsa.py:262) does not
  const T cur_cost = cost[cur];
  if (var_cost) {
    const T *vc = var_cost + unary_off[v];
    for (int x = 0; x < d; ++x) cost[x] += vc[x];
  }
  // find_optimal (relations.py:1594-1638): all values whose cost == best, in domain order
  T best_cost = mode_max ? -Inf<T>::pos() : Inf<T>::pos();
  int nbest = 0;
  bool cur_best = false;   // the current value is one of the best
  for (int x = 0; x < d; ++x) {
    T c = cost[x];
    if (c == best_cost) { ++nbest; cur_best |= x == cur; }
    else if (mode_max ? (c > best_cost) : (c < best_cost)) { best_cost = c; nbest = 1; cur_best = x == cur; }
  }
  const T delta = fg_abs<T>(cur_cost - best_cost);
  bool attempt = false, drop_cur = false;
  if (delta > (T)0) {
    attempt = true;
  } else if (delta == (T)0) {
    if (variant == FG_DSA_C || (variant == FG_DSA_B && violated)) {
      attempt = true;
      // best_values.remove(current_value), dsa.py:380-384.  With A-DSA's own costs delta == 0 does not make the
      // current value one of the best (cur_cost leaves its own cost out), and then nothing is removed (adsa.py:294-299)
      drop_cur = nbest > 1 && cur_best;
    }
  }
  int nv = cur;
  if (attempt) {  // probabilistic_change, dsa.py:407-417
    uint32_t b[4];
    philox_draw((uint32_t)g.var_id[v], cycle, 0u, fg_var_seed(g.var_seed, v, seed), b);
    if (g.prob[v] > philox_u53(b)) {
      int n = drop_cur ? nbest - 1 : nbest;
      int pick = philox_choice(b, n);
      for (int x = 0; x < d; ++x) {
        if (cost[x] == best_cost && !(drop_cur && x == cur)) {
          if (pick == 0) { nv = x; break; }
          --pick;
        }
      }
      val_cost[v] = best_cost;
    }
  }
  val_next[v] = nv;
}

// ---- launch sequences of fg_dsa_init / fg_dsa_cycle_compute, shared with tests/hostshim/dsa_generic_host.cpp -------
// L is a launcher (fg_launcher in handle.cuh, fg_host_launcher on the CPU); `classes` is the class table the kernels
// read.  engine.cu tries the active-row and oriented-table steps (dsa_cached.cuh, dsa_fast.cuh) before dsa_step.

static inline DsaSide dsa_side(const fg_dsa_desc_t &d, const fg_class_t *classes) {
  return DsaSide{classes, d.dev_dom_size, d.dev_var_id, d.dev_edge_var, d.dev_edge_class, d.dev_var_ptr,
                 d.dev_slot_edge, d.dev_has_nbr, d.dev_prob, d.dev_var_seed, d.dev_var_pset, d.psets};
}

// constraint optima, start values into both buffers, and the active-row array's "no row read yet"
template <typename T, class L>
static void dsa_init(const fg_dsa_desc_t &d, const fg_class_t *classes, L &launch) {
  for (int ci = 0; ci < d.n_classes; ++ci) {
    const fg_class_t &c = d.classes[ci];
    if (c.n_factors)
      launch(c.n_factors, 128, k_dsa_con_opt<T>, c, (const T *)d.dev_tables, (T *)d.dev_con_opt, d.mode_max);
  }
  if (d.n_vars) {
    launch(d.n_vars, 128, k_dsa_init, dsa_side(d, classes), d.n_vars, d.seed, d.dev_value[0]);
    launch.copy(d.dev_value[1], d.dev_value[0], sizeof(int32_t) * (size_t)d.n_vars);
  }
  if (d.dev_slot_last && d.n_edges) launch.fill(d.dev_slot_last, 0xFF, (size_t)d.n_edges);
}

// evaluate_cycle of round `cycle` from buffer cur into buffer cur ^ 1, on the generic kernel
template <typename T, class L>
static void dsa_step(const fg_dsa_desc_t &d, const fg_class_t *classes, int cur, uint32_t cycle, L &launch) {
  launch(d.n_vars, 128, d.dev_var_pset ? k_dsa_step_generic<T, true> : k_dsa_step_generic<T, false>,
         dsa_side(d, classes), d.n_vars, (const T *)d.dev_tables,
         (const T *)d.dev_con_opt, d.dev_value[cur], d.dev_value[cur ^ 1], (T *)d.dev_value_cost, d.mode_max,
         d.variant, d.seed, cycle, (const T *)d.dev_var_cost, d.dev_unary_off);
}
