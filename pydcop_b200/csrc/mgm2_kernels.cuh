// MGM-2 kernels (included by mgm2.cu).  One thread per variable, any arity / domain sizes.
// Free of CUDA runtime includes like mgm_kernels.cuh: tests/hostshim/mgm2_host.cpp compiles this
// same file with g++ and runs every "thread" in a loop on the CPU (test infrastructure only).
//
// Every cost is the reference's assignment_cost: a sum from 0 over the variable's constraints in
// node.constraints order, variable costs never counted (mgm2.py:1060-1062, relations.py:1479-1532).
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"
#include "philox.cuh"

// MgmSide comes from the MGM kernels' header, which this change leaves as it is.  mgm.cu defines those
// kernels in its own translation unit, so here they get internal linkage: no duplicate host stubs at
// link time.  Two consequences to keep in mind:
//   - the namespace only holds because <stdint.h>, pydcop_b200.h and philox.cuh are included ABOVE it
//     (include guards / #pragma once make their second inclusion inside the namespace empty); an
//     include added to mgm_kernels.cuh must be added here, before the namespace, as well;
//   - mgm2.cu carries an unused copy of the non-template k_mgm_init (the templates are not
//     instantiated).  Moving MgmSide to a header of its own removes both.
namespace {
#include "mgm_kernels.cuh"
}

enum { MGM2_PURPOSE_INIT = 0, MGM2_PURPOSE_OFFER = 1, MGM2_PURPOSE_VALUE = 2, MGM2_PURPOSE_FAVOR = 3,
       MGM2_PURPOSE_PICK = 4 };

// table row of incidence e (variable v at scope position j) at the current values of the other
// scope variables: entry of (v = x, u = y) at t[x * sv + y * su]; su = 0 when u is not in the scope
// (u = -1: nobody excluded)
template <typename T>
__device__ __forceinline__ const T *mgm2_row(const MgmSide &g, const T *__restrict__ tables,
                                             const int32_t *__restrict__ val, int e, int u, int64_t &sv,
                                             int64_t &su) {
  const fg_class_t &c = g.classes[g.edge_class[e]];
  const int le = e - c.first_edge;
  const int f = le / c.arity, j = le - f * c.arity;
  const int e0 = c.first_edge + f * c.arity;
  int64_t base = 0, stride = 1;
  sv = 0;
  su = 0;
  for (int i = c.arity - 1; i >= 0; --i) {
    if (i == j) {
      sv = stride;
    } else {
      const int w = g.edge_var[e0 + i];
      if (w == u) su += stride;
      else base += (int64_t)val[w] * stride;
    }
    stride *= c.dom[i];
  }
  return tables + c.table_base + (int64_t)f * c.table_size + base;
}

template <typename T>
__device__ __forceinline__ bool mgm2_better(T a, T b, int mode_max) {
  return mode_max ? (a > b) : (a < b);
}

// rel[x] = cost of v = x over all its constraints, the other variables at `val`
template <typename T>
__device__ __forceinline__ void mgm2_local_costs(const MgmSide &g, const T *__restrict__ tables,
                                                 const int32_t *__restrict__ val, int v, int d, T *rel) {
  for (int x = 0; x < d; ++x) rel[x] = (T)0;
  for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) {
    int64_t sv, su;
    const T *t = mgm2_row(g, tables, val, g.slot_edge[s], -1, sv, su);
    for (int x = 0; x < d; ++x) rel[x] += t[x * sv];
  }
}

// best of rel in domain order: strict improvement from the first value, ties counted
// (_compute_best_value, mgm2.py:495-519)
template <typename T>
__device__ __forceinline__ T mgm2_best(const T *rel, int d, int mode_max, int &nbest) {
  T best = rel[0];
  nbest = 1;
  for (int x = 1; x < d; ++x) {
    if (mgm2_better(rel[x], best, mode_max)) { best = rel[x]; nbest = 1; }
    else if (rel[x] == best) ++nbest;
  }
  return best;
}

template <typename T>
__device__ __forceinline__ int mgm2_nth_best(const T *rel, int d, T best, int pick) {
  for (int x = 0; x < d; ++x) {
    if (rel[x] == best) {
      if (pick == 0) return x;
      --pick;
    }
  }
  return 0;
}

// Each phase is a per-variable device function (mgm2_<phase>_at) behind its kernel, so the sharded kernels
// (csrc/mgm2_shard_kernels.cuh) run the same code on the variables a rank owns.

// on_start (mgm2.py:459-493)
template <typename T>
__device__ __forceinline__ void mgm2_init_at(int v, const MgmSide &g, const T *__restrict__ tables,
                                             const int32_t *__restrict__ init_value, int mode_max, uint64_t seed,
                                             int32_t *__restrict__ value, T *__restrict__ cost,
                                             uint8_t *__restrict__ has_cost) {
  const int d = g.dom_size[v];
  uint32_t b[4];
  philox_draw((uint32_t)g.var_id[v], FG_PHILOX_INIT_CYCLE, MGM2_PURPOSE_INIT, fg_var_seed(g.var_seed, v, seed), b);
  if (g.nbr_ptr[v + 1] != g.nbr_ptr[v]) {
    has_cost[v] = 0;
    value[v] = (init_value && init_value[v] >= 0) ? init_value[v] : philox_choice(b, d);
    return;
  }
  // no neighbour: random.choice among the best values over its (unary) constraints, then finished;
  // its constraints read no other variable's value
  T rel[FG_MAX_DOM];
  mgm2_local_costs(g, tables, value, v, d, rel);
  int nbest;
  const T best = mgm2_best(rel, d, mode_max, nbest);
  value[v] = mgm2_nth_best(rel, d, best, philox_choice(b, nbest));
  cost[v] = best;
  has_cost[v] = 1;
}

template <typename T>
__global__ void k_mgm2_init(MgmSide g, int n_vars, const T *__restrict__ tables, const int32_t *__restrict__ init_value,
                            int mode_max, uint64_t seed, int32_t *__restrict__ value, T *__restrict__ cost,
                            uint8_t *__restrict__ has_cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  mgm2_init_at<T>(v, g, tables, init_value, mode_max, seed, value, cost, has_cost);
}

// 1. value phase (mgm2.py:742-785)
template <typename T>
__device__ __forceinline__ void mgm2_value_at(int v, const MgmSide &g, const T *__restrict__ tables,
                                              const int32_t *__restrict__ val, T *__restrict__ cost,
                                              uint8_t *__restrict__ has_cost, T *__restrict__ local_cost,
                                              T *__restrict__ gain, int32_t *__restrict__ pvalue,
                                              uint8_t *__restrict__ offerer, int32_t *__restrict__ partner,
                                              uint8_t *__restrict__ committed, uint8_t *__restrict__ answer,
                                              const int64_t *__restrict__ offer_off, T *__restrict__ offer,
                                              int mode_max, double threshold, uint64_t seed, uint32_t cycle) {
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  const int cur = val[v];
  const int d = g.dom_size[v];
  const uint32_t vid = (uint32_t)g.var_id[v];
  const uint64_t key = fg_var_seed(g.var_seed, v, seed);   // every connected variable draws its offer coin
  T rel[FG_MAX_DOM];
  mgm2_local_costs(g, tables, val, v, d, rel);
  const T cst = rel[cur];  // _current_local_cost
  local_cost[v] = cst;
  cost[v] = cst;
  has_cost[v] = 1;
  // best unilateral move
  int nbest;
  const T best = mgm2_best(rel, d, mode_max, nbest);
  const T pg = cst - best;
  int pv = cur;
  if (mode_max ? (pg < (T)0) : (pg > (T)0)) {
    uint32_t b[4];
    philox_draw(vid, cycle, MGM2_PURPOSE_VALUE, key, b);
    pv = mgm2_nth_best(rel, d, best, philox_choice(b, nbest));
  }
  gain[v] = pg;
  pvalue[v] = pv;
  committed[v] = 0;
  answer[v] = 0;
  // offerer coin and partner pick (one Philox block)
  uint32_t b[4];
  philox_draw(vid, cycle, MGM2_PURPOSE_OFFER, key, b);
  if (!(philox_u53(b) < threshold)) {
    offerer[v] = 0;
    partner[v] = -1;
    return;
  }
  const int p = g.nbr_idx[n0 + philox_choice(b, n1 - n0)];
  offerer[v] = 1;
  partner[v] = p;
  // offer table (_compute_offers_to_send, mgm2.py:521-554): every (own, partner) value pair over all
  // constraints; improving pairs keep their gain, the others 0
  const int dp = g.dom_size[p];
  T *out = offer + offer_off[v];
  const int s0 = g.var_ptr[v], s1 = g.var_ptr[v + 1];
  for (int a = 0; a < d; ++a) {
    T *row = out + (int64_t)a * dp;
    for (int y = 0; y < dp; ++y) rel[y] = (T)0;
    for (int s = s0; s < s1; ++s) {
      int64_t sv, su;
      const T *t = mgm2_row(g, tables, val, g.slot_edge[s], p, sv, su);
      t += a * sv;
      for (int y = 0; y < dp; ++y) rel[y] += t[y * su];
    }
    for (int y = 0; y < dp; ++y) {
      const T c = rel[y];
      row[y] = mgm2_better(c, cst, mode_max) ? (T)(cst - c) : (T)0;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(128, 8)
k_mgm2_value(MgmSide g, int n_vars, const T *__restrict__ tables, const int32_t *__restrict__ val,
             T *__restrict__ cost, uint8_t *__restrict__ has_cost, T *__restrict__ local_cost,
             T *__restrict__ gain, int32_t *__restrict__ pvalue, uint8_t *__restrict__ offerer,
             int32_t *__restrict__ partner, uint8_t *__restrict__ committed, uint8_t *__restrict__ answer,
             const int64_t *__restrict__ offer_off, T *__restrict__ offer, int mode_max, double threshold,
             uint64_t seed, uint32_t cycle) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  mgm2_value_at<T>(v, g, tables, val, cost, has_cost, local_cost, gain, pvalue, offerer, partner, committed, answer,
                   offer_off, offer, mode_max, threshold, seed, cycle);
}

// 2. answers of the non-offerers (mgm2.py:787-856, _find_best_offer :556-603).  The offers are read
// in canonical order (offerer's neighbour position, offerer value, own value); only variable v
// writes its own state and the answer slot of the one offerer it accepts.
template <typename T>
__device__ __forceinline__ void mgm2_answer_at(int v, const MgmSide &g, const T *__restrict__ tables,
                                               const int32_t *__restrict__ val, const T *__restrict__ local_cost,
                                               T *__restrict__ gain, int32_t *__restrict__ pvalue,
                                               const uint8_t *__restrict__ offerer, int32_t *__restrict__ partner,
                                               uint8_t *__restrict__ committed, uint8_t *__restrict__ answer,
                                               int32_t *__restrict__ answer_value, T *__restrict__ answer_gain,
                                               const int64_t *__restrict__ offer_off, const T *__restrict__ offer,
                                               int mode_max, int favor, uint64_t seed, uint32_t cycle) {
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1 || offerer[v]) return;
  const int d = g.dom_size[v];
  const int s0 = g.var_ptr[v], s1 = g.var_ptr[v + 1];
  const T cst = local_cost[v];
  T cc[FG_MAX_DOM];
  T best = (T)0;
  int nb = 0, pick = -1;
  int acc_u = -1, acc_a = 0, acc_b = 0;
  // pass 0 finds the best global gain and its number of ties, pass 1 (only on commit) the drawn one
  for (int pass = 0; pass < 2; ++pass) {
    for (int i = n0; i < n1; ++i) {
      const int u = g.nbr_idx[i];
      if (!offerer[u] || partner[u] != v) continue;
      // cost over the constraints that do not contain the offerer (find_dependent_relations)
      for (int x = 0; x < d; ++x) cc[x] = (T)0;
      for (int s = s0; s < s1; ++s) {
        int64_t sv, su;
        const T *t = mgm2_row(g, tables, val, g.slot_edge[s], u, sv, su);
        if (su) continue;
        for (int x = 0; x < d; ++x) cc[x] += t[x * sv];
      }
      const T *tab = offer + offer_off[u];
      const int du = g.dom_size[u];
      for (int a = 0; a < du; ++a) {
        for (int x = 0; x < d; ++x) {
          const T og = tab[(int64_t)a * d + x];
          if (!(mode_max ? (og < (T)0) : (og > (T)0))) continue;   // not in the offer
          const T gg = (T)(cst - cc[x]) + og;
          if (pass == 0) {
            if (mode_max ? (gg < best) : (gg > best)) { best = gg; nb = 1; }
            else if (gg == best) ++nb;
          } else if (gg == best && pick-- == 0) {
            acc_u = u; acc_a = a; acc_b = x;
          }
        }
      }
    }
    if (pass == 1) break;
    // commit rule
    bool commit = false;
    const T pg = gain[v];
    if (nb == 0 || best == (T)0) commit = false;
    else if (mode_max ? (best < pg) : (best > pg)) commit = true;
    else if (best == pg) {
      if (favor == FG_MGM2_FAVOR_COORDINATED) {
        commit = true;
      } else if (favor == FG_MGM2_FAVOR_NO) {
        uint32_t b[4];
        philox_draw((uint32_t)g.var_id[v], cycle, MGM2_PURPOSE_FAVOR, fg_var_seed(g.var_seed, v, seed), b);
        commit = philox_u53(b) > 0.5;
      }
    }
    if (!commit) return;
    uint32_t b[4];
    philox_draw((uint32_t)g.var_id[v], cycle, MGM2_PURPOSE_PICK, fg_var_seed(g.var_seed, v, seed), b);
    pick = philox_choice(b, nb);
  }
  committed[v] = 1;
  gain[v] = best;
  pvalue[v] = acc_b;
  partner[v] = acc_u;
  answer[acc_u] = 1;
  answer_value[acc_u] = acc_a;
  answer_gain[acc_u] = best;
}

template <typename T>
__global__ void __launch_bounds__(128)
k_mgm2_answer(MgmSide g, int n_vars, const T *__restrict__ tables, const int32_t *__restrict__ val,
              const T *__restrict__ local_cost, T *__restrict__ gain, int32_t *__restrict__ pvalue,
              const uint8_t *__restrict__ offerer, int32_t *__restrict__ partner, uint8_t *__restrict__ committed,
              uint8_t *__restrict__ answer, int32_t *__restrict__ answer_value, T *__restrict__ answer_gain,
              const int64_t *__restrict__ offer_off, const T *__restrict__ offer, int mode_max, int favor,
              uint64_t seed, uint32_t cycle) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  mgm2_answer_at<T>(v, g, tables, val, local_cost, gain, pvalue, offerer, partner, committed, answer, answer_value,
                    answer_gain, offer_off, offer, mode_max, favor, seed, cycle);
}

// 3. an accepted offerer commits to the joint move (mgm2.py:858-890)
template <typename T>
__device__ __forceinline__ void mgm2_commit_at(int v, const uint8_t *__restrict__ offerer,
                                               const uint8_t *__restrict__ answer,
                                               const int32_t *__restrict__ answer_value,
                                               const T *__restrict__ answer_gain, T *__restrict__ gain,
                                               int32_t *__restrict__ pvalue, uint8_t *__restrict__ committed) {
  if (!offerer[v] || !answer[v]) return;
  pvalue[v] = answer_value[v];
  gain[v] = answer_gain[v];
  committed[v] = 1;
}

template <typename T>
__global__ void __launch_bounds__(256)
k_mgm2_commit(int n_vars, const uint8_t *__restrict__ offerer, const uint8_t *__restrict__ answer,
              const int32_t *__restrict__ answer_value, const T *__restrict__ answer_gain, T *__restrict__ gain,
              int32_t *__restrict__ pvalue, uint8_t *__restrict__ committed) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  mgm2_commit_at<T>(v, offerer, answer, answer_value, answer_gain, gain, pvalue, committed);
}

// 4. gain phase (mgm2.py:892-972): a committed variable sends GO when its gain beats every other
// neighbour's; the others move on MGM's rule (strict maximum, or tie and smallest name)
template <typename T>
__device__ __forceinline__ void mgm2_gain_at(int v, const MgmSide &g, const T *__restrict__ gain,
                                             const int32_t *__restrict__ pvalue, const uint8_t *__restrict__ committed,
                                             const int32_t *__restrict__ partner, uint8_t *__restrict__ go,
                                             int32_t *__restrict__ val, T *__restrict__ cost) {
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  go[v] = 0;
  const T mine = gain[v];
  if (mine == (T)0) return;
  if (committed[v]) {
    const int p = partner[v];
    bool any = false;
    T mx = (T)0;
    for (int i = n0; i < n1; ++i) {
      const int u = g.nbr_idx[i];
      if (u == p) continue;
      const T gu = gain[u];
      if (!any || gu > mx) { mx = gu; any = true; }
    }
    go[v] = (!any || mine > mx) ? 1 : 0;
    return;
  }
  T mx = gain[g.nbr_idx[n0]];
  for (int i = n0 + 1; i < n1; ++i) {
    const T gu = gain[g.nbr_idx[i]];
    if (gu > mx) mx = gu;
  }
  bool move = false;
  if (mine > mx) {
    move = true;
  } else if (mine == mx) {
    const int my_rank = g.var_rank[v];
    move = true;
    for (int i = n0; i < n1; ++i) {
      const int u = g.nbr_idx[i];
      if (gain[u] == mx && g.var_rank[u] < my_rank) move = false;
    }
  }
  if (move) {  // value_selection(potential_value, current_cost - potential_gain)
    val[v] = pvalue[v];
    cost[v] = cost[v] - mine;
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
k_mgm2_gain(MgmSide g, int n_vars, const T *__restrict__ gain, const int32_t *__restrict__ pvalue,
            const uint8_t *__restrict__ committed, const int32_t *__restrict__ partner, uint8_t *__restrict__ go,
            int32_t *__restrict__ val, T *__restrict__ cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  mgm2_gain_at<T>(v, g, gain, pvalue, committed, partner, go, val, cost);
}

// 5. coordinated moves (mgm2.py:974-1001)
template <typename T>
__device__ __forceinline__ void mgm2_go_at(int v, const uint8_t *__restrict__ committed,
                                           const int32_t *__restrict__ partner, const uint8_t *__restrict__ go,
                                           const T *__restrict__ gain, const int32_t *__restrict__ pvalue,
                                           int32_t *__restrict__ val, T *__restrict__ cost) {
  if (!committed[v] || !go[v] || !go[partner[v]]) return;
  val[v] = pvalue[v];
  cost[v] = cost[v] - gain[v];
}

template <typename T>
__global__ void __launch_bounds__(256)
k_mgm2_go(int n_vars, const uint8_t *__restrict__ committed, const int32_t *__restrict__ partner,
          const uint8_t *__restrict__ go, const T *__restrict__ gain, const int32_t *__restrict__ pvalue,
          int32_t *__restrict__ val, T *__restrict__ cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  mgm2_go_at<T>(v, committed, partner, go, gain, pvalue, val, cost);
}

// ---- launch sequences of fg_mgm2_init / fg_mgm2_step, shared with tests/hostshim/mgm2_host.cpp -------------------
// L is a launcher (fg_launcher in handle.cuh, fg_host_launcher on the CPU); `classes` is the class table the kernels
// read.  The entry points run them only when there are variables.

static inline MgmSide mgm2_side(const fg_mgm2_desc_t &d, const fg_class_t *classes) {
  return MgmSide{classes, d.dev_dom_size, d.dev_var_id, d.dev_var_rank, d.dev_edge_var, d.dev_edge_class,
                 d.dev_var_ptr, d.dev_slot_edge, d.dev_nbr_ptr, d.dev_nbr_idx, nullptr, d.dev_var_seed};
}

template <typename T, class L>
static void mgm2_init(const fg_mgm2_desc_t &d, const fg_class_t *classes, L &launch) {
  launch(d.n_vars, 128, k_mgm2_init<T>, mgm2_side(d, classes), d.n_vars, (const T *)d.dev_tables, d.dev_init_value,
         d.mode_max, d.seed, d.dev_value, (T *)d.dev_cost, d.dev_has_cost);
}

// round done + 1: five kernels, each boundary a synchronisation point of the reference's message exchange
template <typename T, class L>
static void mgm2_cycle(const fg_mgm2_desc_t &d, const fg_class_t *classes, int64_t done, L &launch) {
  const MgmSide g = mgm2_side(d, classes);
  const uint32_t cyc = (uint32_t)(done + 1);
  const int n = d.n_vars;
  T *cost = (T *)d.dev_cost, *local = (T *)d.dev_local_cost, *gain = (T *)d.dev_gain;
  launch(n, 128, k_mgm2_value<T>, g, n, (const T *)d.dev_tables, d.dev_value, cost, d.dev_has_cost, local, gain,
         d.dev_potential_value, d.dev_offerer, d.dev_partner, d.dev_committed, d.dev_answer, d.dev_offer_off,
         (T *)d.dev_offer, d.mode_max, d.threshold, d.seed, cyc);
  launch(n, 128, k_mgm2_answer<T>, g, n, (const T *)d.dev_tables, d.dev_value, local, gain, d.dev_potential_value,
         d.dev_offerer, d.dev_partner, d.dev_committed, d.dev_answer, d.dev_answer_value, (T *)d.dev_answer_gain,
         d.dev_offer_off, (const T *)d.dev_offer, d.mode_max, d.favor, d.seed, cyc);
  launch(n, 256, k_mgm2_commit<T>, n, d.dev_offerer, d.dev_answer, d.dev_answer_value, (const T *)d.dev_answer_gain,
         gain, d.dev_potential_value, d.dev_committed);
  launch(n, 256, k_mgm2_gain<T>, g, n, gain, d.dev_potential_value, d.dev_committed, d.dev_partner, d.dev_go,
         d.dev_value, cost);
  launch(n, 256, k_mgm2_go<T>, n, d.dev_committed, d.dev_partner, d.dev_go, gain, d.dev_potential_value, d.dev_value,
         cost);
}
