// MGM kernels (included by mgm.cu).  One thread per variable, any arity / domain sizes.
// Deliberately free of CUDA runtime includes: tests/hostshim/ compiles this same file with g++ and
// runs every "thread" in a loop on the CPU, so the kernel SOURCE is checked against the oracle and
// the reference trajectories even on a box without a GPU (test infrastructure only — the product
// never runs it on the host).
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"
#include "philox.cuh"

struct MgmSide {
  const fg_class_t *classes;
  const int32_t *dom_size, *var_id, *var_rank, *edge_var, *edge_class, *var_ptr, *slot_edge;
  const int32_t *nbr_ptr, *nbr_idx;
  const int64_t *unary_off;
  const uint64_t *var_seed;  // [n_vars] Philox key of each variable, NULL: the run's seed
};

// on_start (mgm.py:296-310): connected variables take initial_value or random.choice(domain)
__global__ void k_mgm_init(MgmSide g, int n_vars, const int32_t *__restrict__ init_value, uint64_t seed,
                           int32_t *__restrict__ value, uint8_t *__restrict__ has_cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || g.nbr_ptr[v + 1] == g.nbr_ptr[v]) return;
  has_cost[v] = 0;
  if (init_value && init_value[v] >= 0) { value[v] = init_value[v]; return; }
  uint32_t b[4];
  philox_draw((uint32_t)g.var_id[v], FG_PHILOX_INIT_CYCLE, 0u, fg_var_seed(g.var_seed, v, seed), b);
  value[v] = philox_choice(b, g.dom_size[v]);
}

// value phase (mgm.py:343-397): best local gain and intended move of every connected variable
template <typename T>
__global__ void __launch_bounds__(128)
k_mgm_gain(MgmSide g, int n_vars, const T *__restrict__ tables, const T *__restrict__ unary,
           const int32_t *__restrict__ val, T *__restrict__ cost, uint8_t *__restrict__ has_cost,
           T *__restrict__ gain, int32_t *__restrict__ new_val, int mode_max, uint64_t seed, uint32_t cycle) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  const int cur = val[v];
  const int d = g.dom_size[v];
  T rel[FG_MAX_DOM];
  const int s0 = g.var_ptr[v], s1 = g.var_ptr[v + 1];
  for (int s = s0; s < s1; ++s) {
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
    if (s == s0) {
      for (int x = 0; x < d; ++x) rel[x] = t[x * stride_j];
    } else {
      for (int x = 0; x < d; ++x) rel[x] += t[x * stride_j];
    }
  }
  const T own = unary[g.unary_off[v] + cur];
  T cst;
  if (!has_cost[v]) {  // first round: current_cost (mgm.py:349-368)
    cst = rel[cur];
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
  // find_arg_optimal (relations.py:1554-1591): starts from the int32 extreme, strict improvement,
  // exact equality collects ties in domain order
  T best = mode_max ? (T)-2147483648.0 : (T)2147483647.0;
  int nbest = 0;
  for (int x = 0; x < d; ++x) {
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
    for (int x = 0; x < d; ++x) {
      if (rel[x] == best) {
        if (pick == 0) { nv = x; break; }
        --pick;
      }
    }
  }
  new_val[v] = nv;
}

// gain phase (mgm.py:497-537,574-591): the variable moves when its gain is strictly the largest of
// its neighbourhood, or ties for it and has the smallest name among the tied
template <typename T>
__global__ void __launch_bounds__(256)
k_mgm_decide(MgmSide g, int n_vars, const T *__restrict__ gain, const int32_t *__restrict__ new_val,
             int32_t *__restrict__ val, T *__restrict__ cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  const T mine = gain[v];
  const int my_rank = g.var_rank[v];
  T mx = gain[g.nbr_idx[n0]];
  for (int i = n0 + 1; i < n1; ++i) {
    const T gu = gain[g.nbr_idx[i]];
    if (gu > mx) mx = gu;
  }
  bool move = false;
  if (mine > mx) {
    move = true;
  } else if (mine == mx) {
    move = true;
    for (int i = n0; i < n1; ++i) {
      const int u = g.nbr_idx[i];
      if (gain[u] == mx && g.var_rank[u] < my_rank) move = false;
    }
  }
  if (move) {  // value_selection(new_value, current_cost - gain), mgm.py:518; nobody reads val here
    val[v] = new_val[v];
    cost[v] = cost[v] - mine;
  }
}

