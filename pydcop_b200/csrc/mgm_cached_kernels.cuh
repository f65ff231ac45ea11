// MGM value phase with the ACTIVE-ROW array (the DSA kernel's idea, dsa_cached.cuh): binary constraints over one
// domain size D.  The relation value of x is ((f1(x) + f2(x)) + f3(x)) ... in node.constraints order (mgm.py:443);
// each f_i(x) is one row of the table oriented towards the variable — the row of the neighbour's current value —
// and a neighbour's value changes only when it wins its neighbourhood's gain contest, i.e. rarely.  The row each
// slot read last is kept in a slot-major array next to the value it belongs to; a cycle streams the CTA's rows
// (1-D bulk async copy), goes to the oriented table ONLY for the slots whose neighbour moved, and sums per
// variable in slot order — same adds, same order as k_mgm_gain_bin, bit-identical.  The decision part is
// k_mgm_gain_bin's.  slot_last = 0xFF (fg_mgm_init) marks a row as not yet read.
#pragma once
#include "common.cuh"
#include "mgm_kernels.cuh"
#include "row_load.cuh"
#include "tma.cuh"

template <typename T, int D>
struct MgmCachedCfg {
  static constexpr int THREADS = 128;
  static constexpr int NV = THREADS;
  static constexpr int SPT = (D * sizeof(T) <= 32) ? 8 : (D * sizeof(T) <= 80 ? 4 : 2);
  static constexpr int CH = THREADS * SPT;
  static constexpr bool VEC = (D * sizeof(T)) % 16 == 0;
};

template <typename T, int D>
__global__ void __launch_bounds__(MgmCachedCfg<T, D>::THREADS)
k_mgm_gain_cached(MgmSide g, int n_vars, const int32_t *__restrict__ slot_nbr, const int64_t *__restrict__ slot_tab,
                  const T *__restrict__ tables_or, const T *__restrict__ unary, const int32_t *__restrict__ val,
                  T *__restrict__ cost, uint8_t *__restrict__ has_cost, T *__restrict__ gain, int32_t *__restrict__ new_val,
                  int mode_max, uint64_t seed, uint32_t cycle, T *row_cache, uint8_t *slot_last) {
  using Cfg = MgmCachedCfg<T, D>;
  constexpr int RS = fg_row_stride<T, D>();
  constexpr int NV = Cfg::NV, CH = Cfg::CH, NT = Cfg::THREADS, SPT = Cfg::SPT;
  __shared__ __align__(16) T rows[CH * D];
  __shared__ int16_t snew[CH];
  __shared__ int sptr[NV + 1];
  __shared__ __align__(8) uint64_t bar;
  uint32_t phase = 0;
  const int tid = threadIdx.x;
  if (tid == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
  const int v0 = blockIdx.x * NV;
  const int nv = min(NV, n_vars - v0);
  for (int i = tid; i <= nv; i += NT) sptr[i] = g.var_ptr[v0 + i];
  const int v = v0 + tid;
  const bool mine = tid < nv;
  const int cur = mine ? val[v] : 0;
  __syncthreads();
  const int sb = sptr[0], se = sptr[nv];
  const int my_a = mine ? sptr[tid] : 0, my_b = mine ? sptr[tid + 1] : 0;
  T rel[D];
#pragma unroll
  for (int x = 0; x < D; ++x) rel[x] = (T)0;
  for (int c0 = sb; c0 < se; c0 += CH) {
    const int n = min(CH, se - c0);
    if constexpr (Cfg::VEC) {
      if (tid == 0) {
        fence_proxy_async_smem();
        const uint32_t bytes = (uint32_t)(n * D) * (uint32_t)sizeof(T);
        mbar_expect_tx(&bar, bytes);
        const unsigned char *src = reinterpret_cast<const unsigned char *>(row_cache + (int64_t)c0 * D);
        unsigned char *dst = reinterpret_cast<unsigned char *>(rows);
        for (uint32_t o = 0; o < bytes; o += 16384u) tma_load_1d(dst + o, src + o, min(16384u, bytes - o), &bar);
      }
    }
    int yv[SPT], lastv[SPT];
#pragma unroll
    for (int k = 0; k < SPT; ++k) {
      const int i = tid + k * NT;
      yv[k] = 0; lastv[k] = 0;
      if (i < n) { yv[k] = val[slot_nbr[c0 + i]]; lastv[k] = slot_last[c0 + i]; }
    }
    if constexpr (!Cfg::VEC) {
      const T *src = row_cache + (int64_t)c0 * D;
#pragma unroll 8
      for (int i = tid; i < n * D; i += NT) rows[i] = src[i];
    }
#pragma unroll
    for (int k = 0; k < SPT; ++k) {
      const int i = tid + k * NT;
      if (i < n) snew[i] = (int16_t)(yv[k] != lastv[k] ? yv[k] : -1);
    }
    if constexpr (Cfg::VEC) {
      mbar_wait(&bar, phase & 1u);
      ++phase;
    }
    __syncthreads();
#pragma unroll 1
    for (int i = tid; i < n; i += NT) {   // rows whose neighbour moved
      const int y = snew[i];
      if (y < 0) continue;
      T fresh[D];
      fg_load_row_padded<T, D>(tables_or + slot_tab[c0 + i] + (int64_t)y * RS, fresh);
      T *rc = row_cache + (int64_t)(c0 + i) * D;
#pragma unroll
      for (int x = 0; x < D; ++x) { rows[i * D + x] = fresh[x]; rc[x] = fresh[x]; }
      slot_last[c0 + i] = (uint8_t)y;
    }
    __syncthreads();
    {
      const int a = max(my_a, c0), b = min(my_b, c0 + n);
      for (int t = a; t < b; ++t) {
        T r[D];
        fg_load_row<T, D>(rows + (t - c0) * D, r);
        const bool first = t == my_a;   // ((f1 + f2) + f3)...: the first constraint starts the sum (mgm.py:443)
#pragma unroll
        for (int x = 0; x < D; ++x) rel[x] = first ? r[x] : rel[x] + r[x];
      }
    }
    __syncthreads();
  }
  if (!mine) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  if (n0 == n1) return;
  const T own = unary[g.unary_off[v] + cur];
  T cst;
  if (!has_cost[v]) {  // first round: current_cost (mgm.py:349-368)
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
  int nvv = cur;
  if (mode_max ? (gn < (T)0) : (gn > (T)0)) {  // mgm.py:382-385
    uint32_t b[4];
    philox_draw((uint32_t)g.var_id[v], cycle, 0u, fg_var_seed(g.var_seed, v, seed), b);
    int pick = philox_choice(b, nbest);
    bool done = false;
#pragma unroll
    for (int x = 0; x < D; ++x) {
      if (!done && rel[x] == best) {
        if (pick == 0) { nvv = x; done = true; }
        --pick;
      }
    }
  }
  new_val[v] = nvv;
}
