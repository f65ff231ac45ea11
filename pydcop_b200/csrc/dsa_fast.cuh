// DSA fast path: every constraint binary over one domain size D (BASELINE config C4).
// One thread per variable; per incident constraint it reads ONE contiguous row of D costs from the
// table oriented towards the variable (the transposed copy for scope position 0), so the table
// traffic is 4*D bytes per incidence instead of D strided sectors; rows are stored with the stride of
// row_load.cuh::fg_row_stride so that a row never straddles a line it does not have to.
#pragma once
#include <vector>

#include "common.cuh"
#include "maxsum_fast.cuh"
#include "philox.cuh"
#include "row_load.cuh"

// PS: every variable reads its variant from its parameter set (var_pset), as k_dsa_step_generic
template <typename T, int D, bool PS>
__global__ void __launch_bounds__(128)
k_dsa_step_bin(int n_vars, const int32_t *__restrict__ var_ptr, const int32_t *__restrict__ slot_nbr,
               const int64_t *__restrict__ slot_tab, const T *__restrict__ slot_opt,
               const T *__restrict__ tables_or, const uint8_t *__restrict__ has_nbr,
               const double *__restrict__ prob, const int32_t *__restrict__ var_id,
               const uint64_t *__restrict__ var_seed, const uint16_t *__restrict__ var_pset,
               const fg_dsa_pset_t *__restrict__ psets, const int32_t *__restrict__ val,
               int32_t *__restrict__ val_next, T *__restrict__ val_cost,
               int mode_max, int variant, uint64_t seed, uint32_t cycle, const T *__restrict__ var_cost,
               const int64_t *__restrict__ unary_off) {
  constexpr int RS = fg_row_stride<T, D>();   // rows on their own line slots
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const int cur = val[v];
  const uint8_t hn = has_nbr[v];  // 0 isolated (value carried over), 1 active, 2 ghost of another rank's variable:
  if (hn != 1) {                  // never written here — its owner's push / the halo unpack fills `next`
    if (hn == 0) val_next[v] = cur;
    return;
  }
  if (PS) variant = fg_pset(var_pset, psets, v).variant;
  T cost[D];
#pragma unroll
  for (int x = 0; x < D; ++x) cost[x] = (T)0;
  bool violated = false;
  const int s1 = var_ptr[v + 1];
  for (int s = var_ptr[v]; s < s1; ++s) {
    const int y = val[slot_nbr[s]];
    const T *row = tables_or + slot_tab[s] + (int64_t)y * RS;
    T r[D];
    fg_load_row_padded<T, D>(row, r);
#pragma unroll
    for (int x = 0; x < D; ++x) cost[x] += r[x];  // assignment_cost, relations.py:1479-1532
    if (variant == FG_DSA_B && row[cur] != slot_opt[s]) violated = true;  // dsa.py:419-431
  }
  // A-DSA (adsa.py:344-377): the candidates carry the variable's own cost, the current cost (adsa.py:262) does not
  T cur_cost = (T)0;
#pragma unroll
  for (int x = 0; x < D; ++x)
    if (x == cur) cur_cost = cost[x];
  if (var_cost) {
    const T *vc = var_cost + unary_off[v];
#pragma unroll
    for (int x = 0; x < D; ++x) cost[x] += vc[x];
  }
  // find_optimal (relations.py:1594-1638)
  T best_cost = mode_max ? -Inf<T>::pos() : Inf<T>::pos();
  int nbest = 0;
  bool cur_best = false;   // the current value is one of the best
#pragma unroll
  for (int x = 0; x < D; ++x) {
    const T c = cost[x];
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
      drop_cur = nbest > 1 && cur_best;
    }
  }
  int nv = cur;
  if (attempt) {  // probabilistic_change, dsa.py:407-417
    uint32_t b[4];
    philox_draw((uint32_t)var_id[v], cycle, 0u, fg_var_seed(var_seed, v, seed), b);
    if (prob[v] > philox_u53(b)) {
      int pick = philox_choice(b, drop_cur ? nbest - 1 : nbest);
      bool done = false;
#pragma unroll
      for (int x = 0; x < D; ++x) {
        if (!done && cost[x] == best_cost && !(drop_cur && x == cur)) {
          if (pick == 0) { nv = x; done = true; }
          --pick;
        }
      }
      val_cost[v] = best_cost;
    }
  }
  val_next[v] = nv;
}

template <typename T>
inline bool dsa_fast_step(const fg_dsa_desc_t &d, const std::vector<fg_class_t> &, const int32_t *val,
                          int32_t *val_next, uint32_t cycle, cudaStream_t st, int64_t &launches) {
  if (!d.dev_tables_or || !d.dev_slot_nbr || !d.dev_slot_tab || !d.dev_slot_opt || d.fast_dom <= 0) return false;
  if (fg_fast_disabled()) return false;
  const unsigned blocks = (unsigned)((d.n_vars + 127) / 128);
  switch (d.fast_dom) {
#define X(n)                                                                                               \
  case n:                                                                                                  \
    (d.dev_var_pset ? k_dsa_step_bin<T, n, true> : k_dsa_step_bin<T, n, false>)<<<blocks, 128, 0, st>>>(    \
        d.n_vars, d.dev_var_ptr, d.dev_slot_nbr, d.dev_slot_tab, (const T *)d.dev_slot_opt,                  \
        (const T *)d.dev_tables_or, d.dev_has_nbr, d.dev_prob, d.dev_var_id, d.dev_var_seed, d.dev_var_pset,   \
        d.psets, val, val_next, (T *)d.dev_value_cost, d.mode_max, d.variant, d.seed, cycle,                   \
        (const T *)d.dev_var_cost, d.dev_unary_off);                                                         \
    ++launches;                                                                                            \
    return true;
    FG_FAST_DOMS(X)
#undef X
  }
  return false;
}
