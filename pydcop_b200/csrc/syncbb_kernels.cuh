// SyncBB (pydcop/algorithms/syncbb.py:176-512) for the whole chain in ONE CTA: the block loops over the messages of
// the token walk, one message per iteration, with the threads covering the receiver's candidate values.  The step
// logic (bound update on receipt, candidate test, the path elements every candidate fails at, the transition that
// posts the next message) is in __host__ __device__ functions, so tests/hostshim/syncbb_host.cpp runs this source on
// the CPU; only the block-wide selections (first accepted candidate, first strict best) are device-only.
//
// Arithmetic: every sum keeps the reference's operand order (-fmad=false): a candidate's cost is summed element by
// element in path order by one thread, and the path bound is CPython's compensated sum(), kept per path prefix.
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"

#define SBB_FORWARD 0
#define SBB_BACKWARD 1
#define SBB_TERMINATE 2
#define SBB_THREADS FG_MAX_DOM   // one thread per candidate value

template <typename T>
struct SbbSide {
  int n, mode_max;
  const int32_t *dom, *elt_ptr, *elt_pos;
  const int64_t *elt_tab;
  const T *pair;
  T *ub;
  int32_t *sel;
  int32_t *path_val;   // global path; the kernel may read a shared-memory copy
  T *path_cost, *path_sum, *path_comp;
  int32_t *msg;        // type, receiver, path length, finished
  T *msg_ub;
  int64_t *count;      // steps, messages
  int64_t *cycles;     // per variable: new_cycle count
};

template <typename T>
__host__ __device__ __forceinline__ T sbb_abs(T x) { return x < (T)0 ? -x : x; }

// a strictly better bound (syncbb.py:294-299, 362-367)
template <typename T>
__host__ __device__ __forceinline__ bool sbb_better(T a, T b, int mode_max) { return mode_max ? a > b : a < b; }

// is chain position q an earlier neighbour of p (binary search in its ascending elt_pos)
template <typename T>
__host__ __device__ inline bool sbb_is_neighbour(const SbbSide<T> &g, int p, int q) {
  int lo = g.elt_ptr[p], hi = g.elt_ptr[p + 1];
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    int v = g.elt_pos[mid];
    if (v == q) return true;
    if (v < q) lo = mid + 1;
    else hi = mid;
  }
  return false;
}

// Min mode: path element q fails for EVERY candidate of p.  A non-neighbour contributes ass = 0, so the running sum
// cc is the one the previous element passed with (cc < ub) and only `0 + elt_cost >= ub` can fail; at q = 0 cc = 0
// and elt_cost = 0 (the first variable's element), the same test.  Neighbours are tested per candidate.
template <typename T>
__host__ __device__ inline bool sbb_blocks(const SbbSide<T> &g, const T *pc, int p, int q, T ub) {
  return pc[q] >= ub && !sbb_is_neighbour(g, p, q);
}

// get_next_assignment (:448-473) for one candidate x of chain position p against the path prefix of length p.
// `stop` is the first element every candidate fails at (p if none; always p in max mode).  Returns accepted; *cost
// is the sum up to the last element that passed (the full sum when none failed).
template <typename T>
__host__ __device__ inline bool sbb_candidate(const SbbSide<T> &g, const int32_t *pv, const T *pc, int p, int x,
                                              int stop, T ub, T *cost) {
  T cc = (T)0;
  if (p == 0) { *cost = cc; return true; }   // an empty path accepts the first candidate
  const int64_t d = g.dom[p];
  for (int k = g.elt_ptr[p]; k < g.elt_ptr[p + 1]; ++k) {
    const int q = g.elt_pos[k];
    if (q >= stop) break;
    const T a = g.pair[g.elt_tab[k] + (int64_t)pv[q] * d + x];
    const T c2 = cc + a;
    if (!g.mode_max && (c2 >= ub || a + pc[q] >= ub)) { stop = q; break; }
    cc = c2;
  }
  *cost = cc;
  return g.mode_max || stop > 0;   // rejected only when the FIRST element fails
}

// Receipt: a backward message's bound replaces a worse one, and the receiver then selects its path value (:361-367).
// Returns the first candidate: after the path value for backward, 0 for forward.
template <typename T>
__host__ __device__ inline int sbb_receive(const SbbSide<T> &g, int type, int p, T msg_ub) {
  if (type != SBB_BACKWARD) return 0;
  if (sbb_better(msg_ub, g.ub[p], g.mode_max)) {
    g.ub[p] = msg_ub;
    g.sel[p] = g.path_val[p];
  }
  return g.path_val[p] + 1;
}

// CPython's sum() of the path's costs (Neumaier's compensation, added when finite and non-zero): the bound of the
// prefix ending at q (syncbb.py:290)
template <typename T>
__host__ __device__ __forceinline__ T sbb_path_bound(const SbbSide<T> &g, int q) {
  const T s = g.path_sum[q], c = g.path_comp[q];
  return (c != (T)0 && c - c == (T)0) ? s + c : s;
}

template <typename T>
__host__ __device__ inline void sbb_post(const SbbSide<T> &g, int type, int to, int plen, T ub) {
  g.msg[0] = type;
  g.msg[1] = to;
  g.msg[2] = plen;
  *g.msg_ub = ub;
  ++g.count[1];
}

// Path element p := (x, cost), and its compensated prefix sum.  `pv` / `pc`: the copy the kernel reads (may be the
// global arrays themselves).
template <typename T>
__host__ __device__ inline void sbb_write_path(const SbbSide<T> &g, int32_t *pv, T *pc, int p, int x, T cost) {
  T s = (T)0, c = (T)0;
  if (p > 0) { s = g.path_sum[p - 1]; c = g.path_comp[p - 1]; }
  const T t = s + cost;
  if (sbb_abs(s) >= sbb_abs(cost)) c = c + ((s - t) + cost);
  else c = c + ((cost - t) + s);
  g.path_val[p] = x; g.path_cost[p] = cost; g.path_sum[p] = t; g.path_comp[p] = c;
  pv[p] = x; pc[p] = cost;
}

// The rest of the step at chain position p after the candidates: x = the first accepted candidate with its cost
// (-1: none), or at the last variable the first strict best with its total `best` (-1: no improvement).
template <typename T>
__host__ __device__ inline void sbb_transition(const SbbSide<T> &g, int32_t *pv, T *pc, int type, int p, int x,
                                               T cost, T best) {
  const int n = g.n;
  const T nan = (T)0 / (T)0;
  ++g.count[0];
  ++g.cycles[p];                               // every handler ends in one new_cycle()
  if (type == SBB_TERMINATE) {                 // :213-232
    if (p + 1 < n) sbb_post(g, SBB_TERMINATE, p + 1, 0, nan);
    else g.msg[3] = 1;
    return;
  }
  if (type == SBB_FORWARD && p == n - 1) {     // :287-328: both outcomes send the bound backward
    if (x >= 0) { g.ub[p] = best; g.sel[p] = x; }
    sbb_post(g, SBB_BACKWARD, p - 1, p, g.ub[p]);
    return;
  }
  if (x >= 0) {                                 // :330-341, 378-390
    sbb_write_path(g, pv, pc, p, x, cost);
    sbb_post(g, SBB_FORWARD, p + 1, p + 1, g.ub[p]);
  } else if (type == SBB_BACKWARD && p == 0) {  // :392-401 (the first variable never receives forward)
    sbb_post(g, SBB_TERMINATE, 1, 0, nan);
  } else {                                      // :275-283, 402-412
    sbb_post(g, SBB_BACKWARD, p - 1, p, g.ub[p]);
  }
}

// (total, index) a beats b: strictly better, or as good and earlier (the first strict best of a sequential scan)
template <typename T>
__host__ __device__ __forceinline__ bool sbb_pick(bool va, T ta, int ia, bool vb, T tb, int ib, int mode_max) {
  if (!va) return false;
  if (!vb) return true;
  if (sbb_better(ta, tb, mode_max)) return true;
  if (sbb_better(tb, ta, mode_max)) return false;
  return ia < ib;
}

// fg_syncbb_init: bounds +-inf, no selection, the start message (:195-211)
template <typename T>
__global__ void k_syncbb_init(SbbSide<T> g) {
  const T inf = g.mode_max ? -(T)1 / (T)0 : (T)1 / (T)0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += gridDim.x * blockDim.x) {
    g.ub[i] = inf;
    g.sel[i] = -1;
    g.path_val[i] = 0;
    g.path_cost[i] = (T)0;
    g.path_sum[i] = (T)0;
    g.path_comp[i] = (T)0;
    g.cycles[i] = i == 0;                      // on_start's new_cycle (:211)
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    g.msg[3] = 0;
    g.count[0] = 0;
    g.count[1] = 0;
    sbb_post(g, SBB_FORWARD, 1, 1, inf);       // [(x0, domain[0], 0)]: path element 0 stays (0, 0)
  }
}

#ifdef __CUDACC__
// Up to n_steps messages.  With `smem_path` the path values and costs are read from a shared-memory copy (loaded
// here, written through), otherwise from global memory.
template <typename T>
__global__ void __launch_bounds__(SBB_THREADS, 1) k_syncbb(SbbSide<T> g, int64_t n_steps, int smem_path) {
  extern __shared__ __align__(16) unsigned char sbb_smem[];
  __shared__ T s_cost[SBB_THREADS];
  __shared__ T s_wtot[SBB_THREADS / 32];
  __shared__ int s_widx[SBB_THREADS / 32];
  __shared__ int s_type, s_p, s_start, s_stop;
  __shared__ T s_ub;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = g.n;
  int32_t *pv = g.path_val;
  T *pc = g.path_cost;
  if (smem_path) {
    pc = (T *)sbb_smem;
    pv = (int32_t *)(pc + n);
    for (int i = tid; i < n; i += blockDim.x) { pc[i] = g.path_cost[i]; pv[i] = g.path_val[i]; }
  }
  for (int64_t step = 0; step < n_steps; ++step) {
    if (tid == 0) {
      if (g.msg[3]) {
        s_type = -1;
      } else {
        s_type = g.msg[0];
        s_p = g.msg[1];
        s_start = s_type == SBB_TERMINATE ? 0 : sbb_receive(g, s_type, s_p, *g.msg_ub);
        s_ub = g.ub[s_p];
        s_stop = s_p;
      }
    }
    __syncthreads();
    const int type = s_type, p = s_p;
    if (type < 0) break;
    int x = -1;
    T cost = (T)0, best = (T)0;
    if (type != SBB_TERMINATE) {
      const T ub = s_ub;
      if (!g.mode_max) {   // the first element every candidate fails at
        for (int q = tid; q < p; q += blockDim.x)
          if (sbb_blocks(g, pc, p, q, ub)) { atomicMin(&s_stop, q); break; }
        __syncthreads();
      }
      const int stop = s_stop, c = s_start + tid;
      bool acc = false;
      T my = (T)0;
      if (c < g.dom[p]) acc = sbb_candidate(g, pv, pc, p, c, stop, ub, &my);
      s_cost[tid] = my;
      if (type == SBB_FORWARD && p == n - 1) {
        // the first strict best of bound + cost over the accepted candidates, against the variable's own bound
        const T tot = p > 0 ? sbb_path_bound(g, p - 1) + my : my;
        bool v = acc && sbb_better(tot, ub, g.mode_max);
        T t = tot;
        int i = c;
        for (int o = 16; o > 0; o >>= 1) {
          const bool v2 = __shfl_down_sync(0xffffffffu, v, o);
          const T t2 = __shfl_down_sync(0xffffffffu, t, o);
          const int i2 = __shfl_down_sync(0xffffffffu, i, o);
          if (lane + o < 32 && sbb_pick(v2, t2, i2, v, t, i, g.mode_max)) { v = v2; t = t2; i = i2; }
        }
        if (lane == 0) { s_widx[warp] = v ? i : -1; s_wtot[warp] = t; }
        __syncthreads();
        if (tid == 0) {
          for (int w = 0; w < SBB_THREADS / 32; ++w)
            if (sbb_pick(s_widx[w] >= 0, s_wtot[w], s_widx[w], x >= 0, best, x, g.mode_max)) {
              x = s_widx[w];
              best = s_wtot[w];
            }
        }
      } else {
        const unsigned m = __ballot_sync(0xffffffffu, acc);
        if (lane == 0) s_widx[warp] = m ? warp * 32 + __ffs(m) - 1 : -1;
        __syncthreads();
        if (tid == 0) {
          for (int w = 0; w < SBB_THREADS / 32; ++w)
            if (s_widx[w] >= 0) { x = s_start + s_widx[w]; cost = s_cost[s_widx[w]]; break; }
        }
      }
    }
    if (tid == 0) sbb_transition(g, pv, pc, type, p, x, cost, best);
    __syncthreads();
  }
}
#endif
