// Sharded MGM-2 kernels (included by mgm2.cu; tests/hostshim/mgm2_shard_host.cpp compiles this file with g++ as
// well, so it stays free of CUDA runtime includes).
//
// A shard is a closed local problem: the variables a rank owns with all their constraints, plus a GHOST for every
// remote variable in the scope of one of those constraints (pydcop_b200/multigpu_mgm2.py).  The phase kernels are the
// single-GPU ones (mgm2_<phase>_at) run on the owned variables only: a ghost is never computed here, so no local
// kernel writes its value, cost, gain, offer or any other per-variable state.  Ghost state arrives through five
// exchanges per cycle, each one pack (sender) -> transport -> unpack (receiver):
//   0 offers   owner -> holders, after the value phase: offerer flag, partner (translated), the offer prefix
//   1 answers  holder -> owner, after the answer phase: the receiver's accepted joint move for a ghost offerer
//   2 gains    owner -> holders, after the commit phase
//   3 go       owner -> holders, after the gain phase
//   4 values   owner -> holders, after the go phase (and after init)
// A record is a run of T elements; an integer travels as the bits of one element (mgm2x_put_i / mgm2x_get_i).  The
// only ghost entries a local kernel writes are answer / answer_value / answer_gain of a ghost offerer (the answer
// phase of the receiver that accepted it) and the clear of answer[ghost] in the value phase: that is the reverse
// channel of exchange 1, and nothing else writes those entries on this rank.
#pragma once
#include "mgm2_kernels.cuh"

enum { MGM2X_OFFERS = 0, MGM2X_ANSWERS = 1, MGM2X_GAINS = 2, MGM2X_GO = 3, MGM2X_VALUES = 4, MGM2X_N = 5 };

template <typename T>
__device__ __forceinline__ void mgm2x_put_i(T *p, int32_t v) {
  union {
    T t;
    int32_t i;
  } u;
  u.t = (T)0;
  u.i = v;
  *p = u.t;
}

template <typename T>
__device__ __forceinline__ int32_t mgm2x_get_i(const T *p) {
  union {
    T t;
    int32_t i;
  } u;
  u.t = *p;
  return u.i;
}

// the per-variable state the exchanges read and write (internal variable order)
template <typename T>
struct Mgm2State {
  int32_t *value;
  uint8_t *offerer;
  int32_t *partner;
  uint8_t *answer;
  int32_t *answer_value;
  T *answer_gain;
  T *gain;
  uint8_t *go;
  const int64_t *offer_off;
  T *offer;
};

// one direction of one exchange: entry i moves the state of local variable var[i] in record
// buf[off[i] .. off[i + 1])
template <typename T>
struct Mgm2List {
  int64_t n;
  const int32_t *var;
  const int64_t *off;
  T *buf;
};

// partner translation for exchange 0: what the receiving rank must see as the partner of offerer u is ITS id of the
// partner when it owns the partner, else -1 (matches none of its variables: none of them answers)
struct Mgm2Xlat {
  const int32_t *send_peer;    // [n] rank of the receiver of entry i
  const int32_t *owner_rank;   // [n_local] rank that owns the variable
  const int32_t *owner_local;  // [n_local] its internal id on that rank
};

template <typename T>
__device__ __forceinline__ void mgm2x_pack_at(int x, int64_t i, const Mgm2List<T> &l, const Mgm2State<T> &s,
                                              const Mgm2Xlat &xl) {
  const int u = l.var[i];
  T *r = l.buf + l.off[i];
  switch (x) {
    case MGM2X_OFFERS: {
      const int p = s.offerer[u] ? s.partner[u] : -1;
      const int tp = (p >= 0 && xl.owner_rank[p] == xl.send_peer[i]) ? xl.owner_local[p] : -1;
      mgm2x_put_i(r, tp);
      if (tp < 0) return;   // the prefix is only read when the receiver owns the partner
      const int64_t len = l.off[i + 1] - l.off[i] - 1;
      const T *src = s.offer + s.offer_off[u];
      for (int64_t k = 0; k < len; ++k) r[1 + k] = src[k];
      return;
    }
    case MGM2X_ANSWERS:
      mgm2x_put_i(r, s.answer[u] ? s.answer_value[u] : -1);
      r[1] = s.answer_gain[u];
      return;
    case MGM2X_GAINS: r[0] = s.gain[u]; return;
    case MGM2X_GO: mgm2x_put_i(r, (int32_t)s.go[u]); return;
    default: mgm2x_put_i(r, s.value[u]); return;
  }
}

// exchange 1 MERGES: an owner's offerer may be held by several ranks, at most one of which (the partner's owner)
// flags an answer; the others leave what the local answer phase wrote
template <typename T>
__device__ __forceinline__ void mgm2x_unpack_at(int x, int64_t i, const Mgm2List<T> &l, const Mgm2State<T> &s) {
  const int g = l.var[i];
  const T *r = l.buf + l.off[i];
  switch (x) {
    case MGM2X_OFFERS: {
      const int tp = mgm2x_get_i(r);
      s.offerer[g] = tp >= 0 ? 1 : 0;
      s.partner[g] = tp;
      if (tp < 0) return;
      const int64_t len = l.off[i + 1] - l.off[i] - 1;
      T *dst = s.offer + s.offer_off[g];
      for (int64_t k = 0; k < len; ++k) dst[k] = r[1 + k];
      return;
    }
    case MGM2X_ANSWERS: {
      const int a = mgm2x_get_i(r);
      if (a < 0) return;
      s.answer[g] = 1;
      s.answer_value[g] = a;
      s.answer_gain[g] = r[1];
      return;
    }
    case MGM2X_GAINS: s.gain[g] = r[0]; return;
    case MGM2X_GO: s.go[g] = (uint8_t)mgm2x_get_i(r); return;
    default: s.value[g] = mgm2x_get_i(r); return;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) k_mgm2x_pack(int x, Mgm2List<T> l, Mgm2State<T> s, Mgm2Xlat xl) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < l.n) mgm2x_pack_at<T>(x, i, l, s, xl);
}

template <typename T>
__global__ void __launch_bounds__(256) k_mgm2x_unpack(int x, Mgm2List<T> l, Mgm2State<T> s) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < l.n) mgm2x_unpack_at<T>(x, i, l, s);
}

// ---- the phase kernels on the owned variables (ghost[v] != 0: another rank's variable) ----

template <typename T>
__global__ void k_mgm2s_init(MgmSide g, int n_vars, const uint8_t *__restrict__ ghost, const T *__restrict__ tables,
                             const int32_t *__restrict__ init_value, int mode_max, uint64_t seed,
                             int32_t *__restrict__ value, T *__restrict__ cost, uint8_t *__restrict__ has_cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || ghost[v]) return;
  mgm2_init_at<T>(v, g, tables, init_value, mode_max, seed, value, cost, has_cost);
}

// a ghost's answer flag is this rank's reverse channel (exchange 1): cleared every cycle, as the owner clears its own
template <typename T>
__global__ void __launch_bounds__(128, 8)
k_mgm2s_value(MgmSide g, int n_vars, const uint8_t *__restrict__ ghost, const T *__restrict__ tables,
              const int32_t *__restrict__ val, T *__restrict__ cost, uint8_t *__restrict__ has_cost,
              T *__restrict__ local_cost, T *__restrict__ gain, int32_t *__restrict__ pvalue,
              uint8_t *__restrict__ offerer, int32_t *__restrict__ partner, uint8_t *__restrict__ committed,
              uint8_t *__restrict__ answer, const int64_t *__restrict__ offer_off, T *__restrict__ offer, int mode_max,
              double threshold, uint64_t seed, uint32_t cycle) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  if (ghost[v]) {
    answer[v] = 0;
    return;
  }
  mgm2_value_at<T>(v, g, tables, val, cost, has_cost, local_cost, gain, pvalue, offerer, partner, committed, answer,
                   offer_off, offer, mode_max, threshold, seed, cycle);
}

template <typename T>
__global__ void __launch_bounds__(128)
k_mgm2s_answer(MgmSide g, int n_vars, const uint8_t *__restrict__ ghost, const T *__restrict__ tables,
               const int32_t *__restrict__ val, const T *__restrict__ local_cost, T *__restrict__ gain,
               int32_t *__restrict__ pvalue, const uint8_t *__restrict__ offerer, int32_t *__restrict__ partner,
               uint8_t *__restrict__ committed, uint8_t *__restrict__ answer, int32_t *__restrict__ answer_value,
               T *__restrict__ answer_gain, const int64_t *__restrict__ offer_off, const T *__restrict__ offer,
               int mode_max, int favor, uint64_t seed, uint32_t cycle) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || ghost[v]) return;
  mgm2_answer_at<T>(v, g, tables, val, local_cost, gain, pvalue, offerer, partner, committed, answer, answer_value,
                    answer_gain, offer_off, offer, mode_max, favor, seed, cycle);
}

template <typename T>
__global__ void __launch_bounds__(256)
k_mgm2s_commit(int n_vars, const uint8_t *__restrict__ ghost, const uint8_t *__restrict__ offerer,
               const uint8_t *__restrict__ answer, const int32_t *__restrict__ answer_value,
               const T *__restrict__ answer_gain, T *__restrict__ gain, int32_t *__restrict__ pvalue,
               uint8_t *__restrict__ committed) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || ghost[v]) return;
  mgm2_commit_at<T>(v, offerer, answer, answer_value, answer_gain, gain, pvalue, committed);
}

template <typename T>
__global__ void __launch_bounds__(256)
k_mgm2s_gain(MgmSide g, int n_vars, const uint8_t *__restrict__ ghost, const T *__restrict__ gain,
             const int32_t *__restrict__ pvalue, const uint8_t *__restrict__ committed,
             const int32_t *__restrict__ partner, uint8_t *__restrict__ go, int32_t *__restrict__ val,
             T *__restrict__ cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || ghost[v]) return;
  mgm2_gain_at<T>(v, g, gain, pvalue, committed, partner, go, val, cost);
}

template <typename T>
__global__ void __launch_bounds__(256)
k_mgm2s_go(int n_vars, const uint8_t *__restrict__ ghost, const uint8_t *__restrict__ committed,
           const int32_t *__restrict__ partner, const uint8_t *__restrict__ go, const T *__restrict__ gain,
           const int32_t *__restrict__ pvalue, int32_t *__restrict__ val, T *__restrict__ cost) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars || ghost[v]) return;
  mgm2_go_at<T>(v, committed, partner, go, gain, pvalue, val, cost);
}
