// DSA fast path with an ACTIVE-ROW array (binary constraints over one domain size D, BASELINE config C4).
//
// evaluate_cycle (dsa.py:320-357) needs, per incident constraint, ONE row of D costs of the table oriented
// towards the variable: the row of the neighbour's current value.  Read from the oriented tables
// (dsa_fast.cuh) that is one random 128-byte line per incidence, and random lines are all HBM delivers to
// that pattern (tools/gather_peak.py measures it alone).  But a neighbour's value changes rarely once DSA has taken its first steps, and the row is
// a function of that value alone.  So the engine keeps, per slot, the row it read last in a slot-major array
// (`row_cache`, the rows of one variable contiguous, variables in kernel order) next to the neighbour value
// it belongs to (`slot_last`); a cycle
//   1. streams the block's run of cached rows into shared memory (coalesced, every byte used),
//   2. compares each slot's neighbour value with `slot_last`; ONLY where it changed it fetches the new row
//      from the oriented table and replaces it in shared memory and in the array,
//   3. sums the rows per variable in slot order, one thread per variable with its D costs in registers —
//      the same adds in the same order as k_dsa_step_bin, so the result is bit-identical — and runs the
//      decision rule.
// The bytes that cross HBM per cycle are the algorithmic ones (one row per incidence, SURVEY §8d), now
// sequential; a cycle in which EVERY neighbour changed costs what the uncached kernel costs plus the
// write-back.  slot_last = 0xFF (fg_dsa_init) marks a row as not yet read.
#pragma once
#include "dsa_fast.cuh"
#include "tma.cuh"

template <typename T, int D>
struct DsaCachedCfg {
  static constexpr int THREADS = 128;    // one thread per variable in the summing phase
  static constexpr int NV = THREADS;     // variables per CTA
  static constexpr int SPT = (D * sizeof(T) <= 32) ? 8 : (D * sizeof(T) <= 80 ? 4 : 2);   // slots per thread and chunk
  static constexpr int CH = THREADS * SPT;   // slots per chunk (<= 40 KB of rows)
  static constexpr bool VEC = (D * sizeof(T)) % 16 == 0;
};

// PS: every variable reads its variant from its parameter set (var_pset), as k_dsa_step_generic
template <typename T, int D, bool PS>
__global__ void __launch_bounds__(DsaCachedCfg<T, D>::THREADS)
k_dsa_step_cached(int n_vars, const int32_t *__restrict__ var_ptr, const int32_t *__restrict__ slot_nbr,
                  const int64_t *__restrict__ slot_tab, const T *__restrict__ slot_opt, const T *__restrict__ tables_or,
                  const uint8_t *__restrict__ has_nbr, const double *__restrict__ prob, const int32_t *__restrict__ var_id,
                  const uint64_t *__restrict__ var_seed, const uint16_t *__restrict__ var_pset,
                  const fg_dsa_pset_t *__restrict__ psets, const int32_t *__restrict__ val,
                  int32_t *__restrict__ val_next, T *__restrict__ val_cost, int mode_max,
                  int variant, uint64_t seed, uint32_t cycle, const T *__restrict__ var_cost,
                  const int64_t *__restrict__ unary_off, T *row_cache, uint8_t *slot_last) {
  using Cfg = DsaCachedCfg<T, D>;
  constexpr int RS = fg_row_stride<T, D>();
  constexpr int NV = Cfg::NV, CH = Cfg::CH, NT = Cfg::THREADS, SPT = Cfg::SPT;
  __shared__ __align__(16) T rows[CH * D];
  __shared__ T sopt[CH];          // optimum of the slot's constraint (variant B)
  __shared__ int16_t snew[CH];    // neighbour value when it differs from the one the cached row belongs to, else -1
  __shared__ int sptr[NV + 1];
  __shared__ __align__(8) uint64_t bar;
  uint32_t phase = 0;
  const int tid = threadIdx.x;
  if (tid == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
  const int v0 = blockIdx.x * NV;
  const int nv = min(NV, n_vars - v0);
  for (int i = tid; i <= nv; i += NT) sptr[i] = var_ptr[v0 + i];
  const int v = v0 + tid;
  const bool mine = tid < nv;
  const int cur = mine ? val[v] : 0;
  if (PS && mine) variant = fg_pset(var_pset, psets, v).variant;
  __syncthreads();
  const int sb = sptr[0], se = sptr[nv];
  const int my_a = mine ? sptr[tid] : 0, my_b = mine ? sptr[tid + 1] : 0;
  T cost[D];
#pragma unroll
  for (int x = 0; x < D; ++x) cost[x] = (T)0;
  bool violated = false;
  for (int c0 = sb; c0 < se; c0 += CH) {
    const int n = min(CH, se - c0);
    // B. cached rows of the chunk: one contiguous run -> 1-D bulk async copies (TMA) on an mbarrier, issued first
    //    so that the row stream and the gathers of step A are in flight together
    if constexpr (Cfg::VEC) {
      if (tid == 0) {
        fence_proxy_async_smem();   // the previous chunk's generic-proxy writes to `rows` are ordered before the copy
        const uint32_t bytes = (uint32_t)(n * D) * (uint32_t)sizeof(T);
        mbar_expect_tx(&bar, bytes);
        const unsigned char *src = reinterpret_cast<const unsigned char *>(row_cache + (int64_t)c0 * D);
        unsigned char *dst = reinterpret_cast<unsigned char *>(rows);
        for (uint32_t o = 0; o < bytes; o += 16384u) tma_load_1d(dst + o, src + o, min(16384u, bytes - o), &bar);
      }
    }
    // A. per-slot metadata, slot-ordered (coalesced)
    int yv[SPT], lastv[SPT];
    T optv[SPT];
#pragma unroll
    for (int k = 0; k < SPT; ++k) {
      const int i = tid + k * NT;
      yv[k] = 0; lastv[k] = 0; optv[k] = (T)0;
      if (i < n) {
        yv[k] = val[slot_nbr[c0 + i]];
        lastv[k] = slot_last[c0 + i];
        optv[k] = slot_opt[c0 + i];
      }
    }
    if constexpr (!Cfg::VEC) {
      const T *src = row_cache + (int64_t)c0 * D;
#pragma unroll 8
      for (int i = tid; i < n * D; i += NT) rows[i] = src[i];
    }
#pragma unroll
    for (int k = 0; k < SPT; ++k) {
      const int i = tid + k * NT;
      if (i < n) { sopt[i] = optv[k]; snew[i] = (int16_t)(yv[k] != lastv[k] ? yv[k] : -1); }
    }
    if constexpr (Cfg::VEC) {
      mbar_wait(&bar, phase & 1u);
      ++phase;
    }
    __syncthreads();
    // C. rows whose neighbour moved: from the oriented table, into shared memory and back into the array
#pragma unroll 1
    for (int i = tid; i < n; i += NT) {
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
    // D. cost[x] += row_s[x] over the variable's slots inside the chunk, in slot order (assignment_cost,
    //    relations.py:1479-1532); exists_violated_constraint (dsa.py:419-431) for variant B
    {
      const int a = max(my_a, c0), b = min(my_b, c0 + n);
      for (int t = a; t < b; ++t) {
        T r[D];
        fg_load_row<T, D>(rows + (t - c0) * D, r);
#pragma unroll
        for (int x = 0; x < D; ++x) cost[x] += r[x];
        if (variant == FG_DSA_B && rows[(t - c0) * D + cur] != sopt[t - c0]) violated = true;
      }
    }
    __syncthreads();
  }
  if (!mine) return;
  const uint8_t hn = has_nbr[v];   // 0 isolated (value carried over), 1 active, 2 ghost (never written here)
  if (hn != 1) {
    if (hn == 0) val_next[v] = cur;
    return;
  }
  T cur_cost = (T)0;   // A-DSA (adsa.py:344-377): candidates carry the variable's own cost, the current cost does not
#pragma unroll
  for (int x = 0; x < D; ++x)
    if (x == cur) cur_cost = cost[x];
  if (var_cost) {
    const T *vc = var_cost + unary_off[v];
#pragma unroll
    for (int x = 0; x < D; ++x) cost[x] += vc[x];
  }
  T best_cost = mode_max ? -Inf<T>::pos() : Inf<T>::pos();   // find_optimal (relations.py:1594-1638)
  int nbest = 0;
  bool cur_best = false;   // the current value is one of the best
#pragma unroll
  for (int x = 0; x < D; ++x) {
    const T cx = cost[x];
    if (cx == best_cost) { ++nbest; cur_best |= x == cur; }
    else if (mode_max ? (cx > best_cost) : (cx < best_cost)) { best_cost = cx; nbest = 1; cur_best = x == cur; }
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
  int nvv = cur;
  if (attempt) {  // probabilistic_change, dsa.py:407-417
    uint32_t b[4];
    philox_draw((uint32_t)var_id[v], cycle, 0u, fg_var_seed(var_seed, v, seed), b);
    if (prob[v] > philox_u53(b)) {
      int pick = philox_choice(b, drop_cur ? nbest - 1 : nbest);
      bool done = false;
#pragma unroll
      for (int x = 0; x < D; ++x) {
        if (!done && cost[x] == best_cost && !(drop_cur && x == cur)) {
          if (pick == 0) { nvv = x; done = true; }
          --pick;
        }
      }
      val_cost[v] = best_cost;
    }
  }
  val_next[v] = nvv;
}

template <typename T>
inline bool dsa_cached_step(const fg_dsa_desc_t &d, const int32_t *val, int32_t *val_next, uint32_t cycle, cudaStream_t st,
                            int64_t &launches) {
  if (!d.dev_row_cache || !d.dev_slot_last || !d.dev_tables_or || !d.dev_slot_nbr || !d.dev_slot_tab || !d.dev_slot_opt ||
      d.fast_dom <= 0 || d.fast_dom > 254)
    return false;
  if (fg_fast_disabled() || fg_env_is("PYDCOP_B200_DSA_CACHE", '0')) return false;
  switch (d.fast_dom) {
#define X(n)                                                                                                          \
  case n: {                                                                                                           \
    using Cfg = DsaCachedCfg<T, n>;                                                                                   \
    static_assert(sizeof(T) * Cfg::CH * (n + 1) + 2 * Cfg::CH + 4 * (Cfg::NV + 1) <= 48 * 1024, "static shared memory");    \
    const unsigned blocks = (unsigned)((d.n_vars + Cfg::NV - 1) / Cfg::NV);                                           \
    (d.dev_var_pset ? k_dsa_step_cached<T, n, true>                                                                   \
                    : k_dsa_step_cached<T, n, false>)<<<blocks, Cfg::THREADS, 0, st>>>(                               \
        d.n_vars, d.dev_var_ptr, d.dev_slot_nbr, d.dev_slot_tab, (const T *)d.dev_slot_opt, (const T *)d.dev_tables_or, \
        d.dev_has_nbr, d.dev_prob, d.dev_var_id, d.dev_var_seed, d.dev_var_pset, d.psets, val, val_next,               \
        (T *)d.dev_value_cost, d.mode_max,                                                                            \
        d.variant, d.seed, cycle, (const T *)d.dev_var_cost, d.dev_unary_off, (T *)d.dev_row_cache, d.dev_slot_last);                     \
    ++launches;                                                                                                       \
    return true;                                                                                                      \
  }
    FG_FAST_DOMS(X)
#undef X
  }
  return false;
}
