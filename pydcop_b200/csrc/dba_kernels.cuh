// DBA kernels (included by dba.cu).  One thread per variable (per bit-row word for k_dba_bits), any arity /
// domain sizes.  Free of CUDA runtime includes like gdba_kernels.cuh: tests/hostshim/dba_host.cpp compiles this
// same file with g++ and runs every "thread" in a loop on the CPU.
//
// pydcop/algorithms/dba.py reads a constraint only through `rel(val) >= infinity` (:478), so the tables are
// reduced once to violation bit rows (include/pydcop_b200.h, fg_dba_desc_t) and everything after that is integer
// arithmetic on the per-slot weights:
//   eval(x)  = sum of weight[s] over the slots whose row has bit x set          (int64)
//   best     = strict minimum starting from `infinity`, ties collected in domain order (:428-445)
//   improve  = eval(cur) - best
// End flood: a variable finishes at phase p iff a neighbour's finish phase is < p.  Stamps written in phase p
// equal p, so the one value a launch may read while another thread writes it never decides anything.
#pragma once
#include <stdint.h>

#include "../../include/pydcop_b200.h"
#include "philox.cuh"

// MgmSide (the neighbourhood arrays) comes from the MGM kernels' header, included with internal linkage as in
// gdba_kernels.cuh.
namespace {
#include "mgm_kernels.cuh"
}

#define FG_DBA_LIVE 0x7fffffff

#ifdef __CUDA_ARCH__
__device__ __forceinline__ int dba_ffs(uint32_t m) { return __ffs((int)m); }
__device__ __forceinline__ int32_t dba_dec(int32_t *p) { return atomicSub(p, 1); }
__device__ __forceinline__ void dba_inc(int32_t *p) { atomicAdd(p, 1); }
#else
static inline int dba_ffs(uint32_t m) { return __builtin_ffs((int)m); }
static inline int32_t dba_dec(int32_t *p) { return (*p)--; }
static inline void dba_inc(int32_t *p) { ++*p; }
#endif

// slot s of its variable: class, factor, scope position, first edge of the factor
struct DbaSlot {
  const fg_class_t *c;
  int f, j, e0;
};

__device__ __forceinline__ DbaSlot dba_slot(const MgmSide &g, int e) {
  DbaSlot s;
  s.c = &g.classes[g.edge_class[e]];
  const int le = e - s.c->first_edge;
  s.f = le / s.c->arity;
  s.j = le - s.f * s.c->arity;
  s.e0 = s.c->first_edge + s.f * s.c->arity;
  return s;
}

// the variable finishes at phase p; the thread that finishes the last live variable records the round
__device__ __forceinline__ void dba_finish(int v, int32_t p, int32_t round, int32_t *__restrict__ finish_phase,
                                           int32_t *__restrict__ status) {
  finish_phase[v] = p;
  if (dba_dec(&status[0]) == 1) status[1] = round;
}

// true when a neighbour of v finished before phase p (the message phase p waits for was never sent)
__device__ __forceinline__ bool dba_flooded(const MgmSide &g, int n0, int n1, const int32_t *finish_phase,
                                            int32_t p) {
  for (int i = n0; i < n1; ++i)
    if (finish_phase[g.nbr_idx[i]] < p) return true;
  return false;
}

// One thread per bit-row word: word w of row r of slot s holds, for x = 32 w + b < dom(v), bit b =
// table[f][other variables at row r, v = x] >= infinity, compared in T as fg_solution_cost compares.
template <typename T>
__global__ void __launch_bounds__(256)
k_dba_bits(MgmSide g, int n_edges, const T *__restrict__ tables, const int64_t *__restrict__ bit_off,
           int64_t n_words, T infinity, uint32_t *__restrict__ bits) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_words) return;
  int lo = 0, hi = n_edges;  // last slot s with bit_off[s] <= t
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (bit_off[mid] <= t) lo = mid;
    else hi = mid;
  }
  const int s = lo;
  const DbaSlot sl = dba_slot(g, g.slot_edge[s]);
  const int d = sl.c->dom[sl.j];
  const int W = (d + 31) >> 5;
  const uint32_t local = (uint32_t)(t - bit_off[s]);  // a slot has fewer than 2^32 words (dba_plan checks)
  uint32_t r = local / (uint32_t)W;
  const int w = (int)(local - r * (uint32_t)W);
  int64_t base = 0, stride = 1, sv = 0;
  for (int i = sl.c->arity - 1; i >= 0; --i) {
    const uint32_t di = (uint32_t)sl.c->dom[i];
    if (i == sl.j) {
      sv = stride;
    } else {
      const uint32_t q = r / di;
      base += (int64_t)(r - q * di) * stride;
      r = q;
    }
    stride *= di;
  }
  const T *tb = tables + sl.c->table_base + (int64_t)sl.f * sl.c->table_size + base;
  uint32_t word = 0;
  for (int b = 0; b < 32; ++b) {
    const int x = w * 32 + b;
    if (x < d && tb[x * sv] >= infinity) word |= 1u << b;
  }
  bits[t] = word;
}

// on_start (:341-349): every variable draws its start value, initial_value is ignored; weights 1, counters 0
__global__ void k_dba_init(MgmSide g, int n_vars, uint64_t seed, int32_t n_live, int32_t *__restrict__ value,
                           uint8_t *__restrict__ has_cost, int32_t *__restrict__ counter_own,
                           int32_t *__restrict__ finish_phase, int32_t *__restrict__ weight,
                           int32_t *__restrict__ status, int32_t *__restrict__ unresolved) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) {
    status[0] = n_live;
    status[1] = n_live ? FG_DBA_LIVE : 0;
    unresolved[0] = 0;
  }
  if (v >= n_vars) return;
  uint32_t b[4];
  philox_draw((uint32_t)g.var_id[v], FG_PHILOX_INIT_CYCLE, 0u, seed, b);
  value[v] = philox_choice(b, g.dom_size[v]);
  has_cost[v] = 0;
  counter_own[v] = 0;
  finish_phase[v] = FG_DBA_LIVE;
  for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) weight[s] = 1;
}

// Largest domain over the constraint classes: every variable that evaluates (one with a neighbour) has a slot in
// one of them.  k_dba_ok keeps one int64 eval per value on its stack, so instances whose domains are all <= 32 run
// the DMAX = 32 instance (256 B of stack per thread instead of 2 KB).
static inline int dba_eval_dmax(const fg_class_t *classes, int n_classes) {
  int m = 1;
  for (int c = 0; c < n_classes; ++c)
    for (int i = 0; i < classes[c].arity; ++i) m = classes[c].dom[i] > m ? classes[c].dom[i] : m;
  return m <= 32 ? 32 : FG_MAX_DOM;
}

// ok phase of round k (phase 2k, dba.py:366-420); every evaluating variable has dom_size <= DMAX
template <int DMAX>
__global__ void __launch_bounds__(128)
k_dba_ok(MgmSide g, int n_vars, const uint32_t *__restrict__ bits, const int64_t *__restrict__ bit_off,
         const int32_t *__restrict__ weight, const int32_t *__restrict__ val, int64_t infinity, uint64_t seed,
         int32_t round, int32_t *finish_phase, int32_t *status, const int32_t *__restrict__ counter_own,
         int64_t *__restrict__ eval, int64_t *__restrict__ improve, int32_t *__restrict__ counter,
         int32_t *__restrict__ new_value, uint8_t *__restrict__ can_move, uint8_t *__restrict__ qlm,
         uint8_t *__restrict__ consistent, uint8_t *__restrict__ violated, int64_t *__restrict__ cost,
         uint8_t *__restrict__ has_cost, int32_t *__restrict__ unresolved) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || status[1] < round) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  const int32_t p = 2 * round, fv = finish_phase[v];
  // A variable that stopped in the last improve phase goes back to waiting for ok messages (_go_to_wait_ok_mode
  // runs after _send_ok, :529), so it evaluates once more when no neighbour stopped with it; it never gets the
  // improve messages that would let it move.
  if (n0 == n1 || (fv != FG_DBA_LIVE && fv != p - 1)) return;
  if (dba_flooded(g, n0, n1, finish_phase, p)) {
    if (fv == FG_DBA_LIVE) dba_finish(v, p, round, finish_phase, status);
    return;
  }
  const int cur = val[v];
  const int d = g.dom_size[v];
  const int W = (d + 31) >> 5;
  int64_t ev[DMAX];
  for (int x = 0; x < d; ++x) ev[x] = 0;
  for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) {
    const DbaSlot sl = dba_slot(g, g.slot_edge[s]);
    int64_t row = 0, rs = 1;
    for (int i = sl.c->arity - 1; i >= 0; --i) {
      if (i == sl.j) continue;
      row += (int64_t)val[g.edge_var[sl.e0 + i]] * rs;
      rs *= sl.c->dom[i];
    }
    const uint32_t *rw = bits + bit_off[s] + row * W;
    const int64_t wt = weight[s];
    for (int w = 0; w < W; ++w) {
      uint32_t m = rw[w];
      while (m) {
        ev[w * 32 + dba_ffs(m) - 1] += wt;
        m &= m - 1;
      }
    }
    violated[s] = (rw[cur >> 5] >> (cur & 31)) & 1u;
  }
  const int64_t cur_eval = ev[cur];
  int64_t best = infinity;  // _compute_best_improvement (:428-445)
  int nbest = 0;
  for (int x = 0; x < d; ++x) {
    if (ev[x] < best) { best = ev[x]; nbest = 1; }
    else if (ev[x] == best) ++nbest;
  }
  const int64_t gn = cur_eval - best;
  const bool cons = cur_eval == 0;
  uint8_t cm = gn > 0, q = gn <= 0;
  int nv = -1;
  if (cm) {
    if (nbest == 0) {  // every value above infinity: the reference raises on random.choice([])
      dba_inc(unresolved);
      cm = 0;
    } else {
      uint32_t b[4];
      philox_draw((uint32_t)g.var_id[v], (uint32_t)(round - 1), 0u, seed, b);
      int pick = philox_choice(b, nbest);
      for (int x = 0; x < d; ++x) {
        if (ev[x] == best) {
          if (pick == 0) { nv = x; break; }
          --pick;
        }
      }
    }
  }
  eval[v] = cur_eval;
  cost[v] = cur_eval;  // the reference assigns its current_cost field directly (:385)
  has_cost[v] = 1;
  improve[v] = gn;
  counter[v] = cons ? counter_own[v] : 0;
  new_value[v] = nv;
  can_move[v] = cm;
  qlm[v] = q;
  consistent[v] = cons;
}

// improve phase of round k (phase 2k + 1, dba.py:504-562).  Every variable writes its value for the next round
// to val_out, so nothing read in this launch is written in it.
__global__ void __launch_bounds__(256)
k_dba_improve(MgmSide g, int n_vars, const int64_t *__restrict__ eval, const int64_t *__restrict__ improve,
              const int32_t *__restrict__ counter, const int32_t *__restrict__ new_value, int32_t max_distance,
              int32_t round, int32_t *finish_phase, int32_t *status, const uint8_t *__restrict__ violated,
              const int32_t *__restrict__ val_in, int32_t *__restrict__ val_out, int32_t *__restrict__ counter_own,
              uint8_t *__restrict__ can_move, uint8_t *__restrict__ qlm, uint8_t *__restrict__ consistent,
              int32_t *__restrict__ weight, int64_t *__restrict__ cost) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || status[1] < round) return;
  const int n0 = g.nbr_ptr[v], n1 = g.nbr_ptr[v + 1];
  const int cur = val_in[v];
  val_out[v] = cur;
  if (n0 == n1 || finish_phase[v] != FG_DBA_LIVE) return;
  const int32_t p = 2 * round + 1;
  if (dba_flooded(g, n0, n1, finish_phase, p)) {
    dba_finish(v, p, round, finish_phase, status);
    return;
  }
  const int64_t mine = improve[v];
  const int my_rank = g.var_rank[v];
  int32_t cnt = counter[v];
  bool cm = can_move[v], q = qlm[v], cons = consistent[v];
  for (int i = n0; i < n1; ++i) {
    const int u = g.nbr_idx[i];
    cnt = counter[u] < cnt ? counter[u] : cnt;
    const int64_t gu = improve[u];
    if (gu > mine) cm = q = false;
    else if (gu == mine && g.var_rank[u] < my_rank) cm = false;
    if (eval[u] > 0) cons = false;
  }
  bool stop = false;
  if (cons) {  // _send_ok (:537-562)
    ++cnt;
    stop = cnt == max_distance;
  }
  counter_own[v] = cnt;
  can_move[v] = cm;
  qlm[v] = q;
  consistent[v] = cons;
  if (stop) {
    dba_finish(v, p, round, finish_phase, status);
    return;
  }
  if (q)
    for (int s = g.var_ptr[v]; s < g.var_ptr[v + 1]; ++s) weight[s] += violated[s];
  if (cm) {
    val_out[v] = new_value[v];
    cost[v] = eval[v] - mine;
  }
}
