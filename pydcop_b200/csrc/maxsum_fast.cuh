// Shape-specialised MaxSum kernels for uniform-domain graphs (compile-time arity A and domain D).
//
//  k_f2v_tile<T,A,D>  factor -> variable.  One CTA = one tile of NF same-shaped factors.
//      HBM side: the tile's cost tables, previous r rows and the produced r rows are CONTIGUOUS
//      (class-major layout) and move with 1-D bulk async copies (TMA, mbarrier completion) when no
//      padding is needed, otherwise with 16-byte cp.async into a bank-conflict-free padded layout;
//      q rows are gathered through edge_qoff with cp.async.  All global traffic is issued as whole
//      16-byte (or row-sized) async transactions; the math runs out of shared memory with one
//      thread per directed edge, lanes mapped (position j, factor f) so a warp is uniform in j.
//  k_v2f_tile<T,D>    variable -> factor (+ select_value).  One CTA = 256 consecutive slots
//      (variable-major).  r rows are gathered through slot_roff into a TRANSPOSED shared tile,
//      q_old / q_next tiles are contiguous (slot order) and move with bulk async copies.
//
// Floating-point operand order is the reference's (see common.cuh); results are bit-identical to
// the generic kernels and to the CPU oracle of the same precision.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "tma.cuh"

// ------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------
constexpr int fg_ipow(int b, int e) { return e == 0 ? 1 : b * fg_ipow(b, e - 1); }
constexpr int fg_gcd(int a, int b) { return b == 0 ? a : fg_gcd(b, a % b); }
constexpr int fg_clamp(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }

template <typename T, int N> struct VecT;
template <> struct VecT<float, 4> { using type = float4; };
template <> struct VecT<float, 2> { using type = float2; };
template <> struct VecT<float, 1> { using type = float; };
template <> struct VecT<double, 2> { using type = double2; };
template <> struct VecT<double, 1> { using type = double; };

// load N contiguous elements with vector width V (V | N), static indexing only
template <typename T, int N, int V>
__device__ __forceinline__ void ld_row(const T *__restrict__ p, T (&out)[N]) {
  using VT = typename VecT<T, V>::type;
#pragma unroll
  for (int i = 0; i < N / V; ++i) {
    VT v = reinterpret_cast<const VT *>(p)[i];
    const T *e = reinterpret_cast<const T *>(&v);
#pragma unroll
    for (int k = 0; k < V; ++k) out[i * V + k] = e[k];
  }
}
template <typename T, int N, int V>
__device__ __forceinline__ void st_row(T *__restrict__ p, const T (&in)[N]) {
  using VT = typename VecT<T, V>::type;
#pragma unroll
  for (int i = 0; i < N / V; ++i) {
    VT v;
    T *e = reinterpret_cast<T *>(&v);
#pragma unroll
    for (int k = 0; k < V; ++k) e[k] = in[i * V + k];
    reinterpret_cast<VT *>(p)[i] = v;
  }
}

// async copy of `bytes` (4, 8 or 16) global -> shared
template <int BYTES> __device__ __forceinline__ void cp_async_b(void *dst, const void *src);
template <> __device__ __forceinline__ void cp_async_b<16>(void *d, const void *s) { cp_async_16(d, s); }
template <> __device__ __forceinline__ void cp_async_b<8>(void *d, const void *s) { cp_async_8(d, s); }
template <> __device__ __forceinline__ void cp_async_b<4>(void *d, const void *s) { cp_async_4(d, s); }

// cooperative contiguous copy global -> shared (both 16-B aligned at the start)
template <typename T>
__device__ __forceinline__ void coop_copy_in(T *dst, const T *__restrict__ src, int n, int tid, int nt) {
  constexpr int E16 = 16 / (int)sizeof(T);
  const int nv = n / E16;
  for (int i = tid; i < nv; i += nt) cp_async_16(dst + i * E16, src + i * E16);
  for (int i = nv * E16 + tid; i < n; i += nt) cp_async_b<(int)sizeof(T)>(dst + i, src + i);
}
// cooperative contiguous copy shared -> global
template <typename T>
__device__ __forceinline__ void coop_copy_out(T *__restrict__ dst, const T *src, int n, int tid, int nt) {
  constexpr int E16 = 16 / (int)sizeof(T);
  using V16 = typename VecT<T, E16>::type;
  const int nv = n / E16;
  for (int i = tid; i < nv; i += nt) reinterpret_cast<V16 *>(dst)[i] = reinterpret_cast<const V16 *>(src)[i];
  for (int i = nv * E16 + tid; i < n; i += nt) dst[i] = src[i];
}

template <typename T> struct MatchEps;
template <> struct MatchEps<float> { __device__ static float lo() { return 1.0f - 9.5367431640625e-07f; } __device__ static float hi() { return 1.0f + 9.5367431640625e-07f; } __device__ static float tiny() { return 1e-30f; } };
template <> struct MatchEps<double> { __device__ static double lo() { return 1.0 - 3.552713678800501e-15; } __device__ static double hi() { return 1.0 + 3.552713678800501e-15; } __device__ static double tiny() { return 1e-290; } };

// Same predicate as approx_match1 (maxsum.py:688-710), bit-for-bit, but the IEEE division is only
// executed when 2*delta is within a few ulps of stab*|s|; otherwise the comparison of the products
// decides (the margins are wider than the worst-case rounding of the quotient).
template <typename T>
__device__ __forceinline__ bool approx_match_fast(T c, T prev_c, T stab) {
  const T s = prev_c + c;
  const T d2 = (T)2 * fg_abs<T>(prev_c - c);
  const T as = fg_abs<T>(s);
  const T rhs = stab * as;
  const bool safe = (rhs > MatchEps<T>::tiny()) && (rhs < Inf<T>::pos());
  const bool lt = d2 < rhs * MatchEps<T>::lo();
  const bool gt = d2 > rhs * MatchEps<T>::hi();
  bool res = lt;
  if (!(safe && (lt || gt))) res = (s != (T)0) && ((d2 / as) < stab);  // rare: a few ulps from the threshold
  return (prev_c == c) || res;
}

// damping + approx_match for (a part of) one message row held in registers.
// cand: fresh values in, damped values out.  Returns whether every element matches `prev`.
// The predicate is evaluated division-free for the whole row (straight-line code); only if some
// element sits within a few ulps of the threshold (or in the denormal / overflow range) the
// literal form with the IEEE division is evaluated.
template <typename T, int N>
__device__ __forceinline__ bool damp_match_row(T (&cand)[N], const T (&prev)[N], bool has_prev, bool damp_side,
                                               T lam, T oml, T stab) {
  if (!has_prev) return false;
  bool all_ok = true, unsure = false;
#pragma unroll
  for (int x = 0; x < N; ++x) {
    T c = cand[x];
    if (damp_side) c = lam * prev[x] + oml * c;
    cand[x] = c;
    const T s = prev[x] + c;
    const T d2 = (T)2 * fg_abs<T>(prev[x] - c);
    const T rhs = stab * fg_abs<T>(s);
    const bool safe = (rhs > MatchEps<T>::tiny()) && (rhs < Inf<T>::pos());
    const bool lt = d2 < rhs * MatchEps<T>::lo();
    const bool gt = d2 > rhs * MatchEps<T>::hi();
    const bool eq = prev[x] == c;
    unsure = unsure || (!eq && !(safe && (lt || gt)));
    all_ok = all_ok && (eq || lt);
  }
  if (unsure) {  // rare
    all_ok = true;
#pragma unroll
    for (int x = 0; x < N; ++x)
      if (!approx_match1<T>(cand[x], prev[x], stab)) all_ok = false;
  }
  return all_ok;
}

// whole row: damping, match, send gate.  Returns `sent`; cand holds the row to store.
template <typename T, int D>
__device__ __forceinline__ bool damp_gate_row(T (&cand)[D], const T (&prev)[D], uint8_t &cnt, bool damp_side,
                                              T lam, T oml, T stab) {
  const bool match = damp_match_row<T, D>(cand, prev, (cnt & 1) != 0, damp_side, lam, oml, stab);
  const bool sent = gate_decide(match, cnt);
  if (!sent) {
#pragma unroll
    for (int x = 0; x < D; ++x) cand[x] = prev[x];
  }
  return sent;
}

template <typename T> __device__ __forceinline__ T fg_opt(T a, T b, bool mx);
template <> __device__ __forceinline__ float fg_opt<float>(float a, float b, bool mx) { return mx ? fmaxf(a, b) : fminf(a, b); }
template <> __device__ __forceinline__ double fg_opt<double>(double a, double b, bool mx) { return mx ? fmax(a, b) : fmin(a, b); }

// ------------------------------------------------------------------------------------------------
// factor -> variable
// ------------------------------------------------------------------------------------------------
template <typename T, int A, int D>
struct F2VCfg {
  static constexpr int S = fg_ipow(D, A);
  static constexpr int R = A * D;
  static constexpr int INNER = S / D;
  static constexpr int E16 = 16 / (int)sizeof(T);
  static constexpr bool QUADS = (S * (int)sizeof(T)) % 16 == 0;
  static constexpr int Q = (S * (int)sizeof(T)) / 16;
  static constexpr int PAD = (QUADS && (Q % 2 == 0)) ? E16 : 0;  // odd 16-B stride: no bank conflicts
  static constexpr int SP = S + PAD;
  static constexpr int PER_FACTOR = (SP + 3 * R) * (int)sizeof(T);
  static constexpr int NF = fg_clamp(((20 * 1024) / PER_FACTOR) / 32 * 32, 32, 512);
  // two threads per directed edge (each owns half of the D outputs) when D is even: twice the
  // warps per tile for the same shared memory
  static constexpr int SPLIT = (A >= 2 && D % 2 == 0 && D >= 4) ? 2 : 1;
  static constexpr int HD = D / SPLIT;
  static constexpr int NT = fg_clamp(NF * A * SPLIT, 64, 256);
  static constexpr int VH_BYTES = fg_gcd(16, HD * (int)sizeof(T));
  static constexpr int VH = VH_BYTES / (int)sizeof(T);
  // vector width (elements) for table rows (D contiguous elements at multiples of D inside a
  // factor whose stride is SP) and for message rows
  static constexpr int VT_BYTES = fg_gcd(16, fg_gcd(D * (int)sizeof(T), SP * (int)sizeof(T)));
  static constexpr int VT = VT_BYTES / (int)sizeof(T);
  static constexpr int VR_BYTES = fg_gcd(16, D * (int)sizeof(T));
  static constexpr int VR = VR_BYTES / (int)sizeof(T);
  static constexpr size_t SMEM = (size_t)(NF * SP + 3 * NF * R) * sizeof(T) + 16;
};

// pairwise (tree) optimum of N values: same result as the sequential scan, more ILP
template <typename T, int N>
__device__ __forceinline__ T opt_tree(const T (&v)[N], bool mx) {
  T w[N];
#pragma unroll
  for (int i = 0; i < N; ++i) w[i] = v[i];
#pragma unroll
  for (int n = N; n > 1; n = (n + 1) / 2) {
#pragma unroll
    for (int i = 0; i < n / 2; ++i) w[i] = fg_opt<T>(w[i], w[n - 1 - i], mx);
  }
  return w[0];
}

// All edges of one staged tile: min-marginal (factor_costs_for_var, maxsum.py:382-447), damping,
// send gate; results into `ot` (same [f][j][x] layout as the class-major r array).
// Work item w -> (position j, factor f, half h): lanes of a warp share j, the two halves of an edge
// sit in adjacent lanes (h = lane & 1) and combine their match flags with one shuffle.
template <typename T, int A, int D, int WPT>
__device__ __forceinline__ void f2v_compute_tile(const T *__restrict__ tab, const T *__restrict__ qt,
                                                 const T *__restrict__ rt, T *__restrict__ ot, int nf, int e_base,
                                                 const uint8_t (&cnt_in)[WPT], uint8_t *__restrict__ r_cnt,
                                                 uint8_t *__restrict__ r_sent, const MaxSumParams &p, int tid) {
  using C = F2VCfg<T, A, D>;
  constexpr int R = C::R, SP = C::SP, NF = C::NF, NT = C::NT, INNER = C::INNER, SPLIT = C::SPLIT, HD = C::HD;
  const bool mx = p.mode_max != 0;
  const T lam = (T)p.damping, oml = (T)p.one_minus_damping, stab = (T)p.stability;
  const T init = mx ? -Inf<T>::pos() : Inf<T>::pos();
#pragma unroll
  for (int u = 0; u < WPT; ++u) {
    const int w = tid + u * NT;
    const bool in_range = w < NF * A * SPLIT;
    const int j = w / (NF * SPLIT), rem = w - j * (NF * SPLIT);  // warp-uniform j
    const int f = rem / SPLIT, h = rem - f * SPLIT;
    const bool active = in_range && f < nf;
    const int x_lo = h * HD;  // this thread's outputs are x_lo .. x_lo + HD - 1
    T cand[HD];
    bool match = false;
    uint8_t cnt = cnt_in[u];
    T prev[HD];
    T *of = ot + f * R + j * D + x_lo;
    if (active) {
      const T *tf = tab + f * SP;
      const T *qf = qt + f * R;
      if (A == 1) {
        ld_row<T, HD, C::VH>(tf + x_lo, cand);
      } else if (A == 2) {
        if (j == 0) {
          T qo[D];
          ld_row<T, D, C::VR>(qf + D, qo);
#pragma unroll
          for (int i = 0; i < HD; ++i) {
            T row[D];
            ld_row<T, D, C::VT>(tf + (x_lo + i) * D, row);
#pragma unroll
            for (int x1 = 0; x1 < D; ++x1) row[x1] = row[x1] + qo[x1];
            cand[i] = fg_opt<T>(init, opt_tree<T, D>(row, mx), mx);   // all candidates NaN: +/-inf, as the reference
          }
        } else {
#pragma unroll
          for (int i = 0; i < HD; ++i) cand[i] = init;
          T q0r[D];
          ld_row<T, D, C::VR>(qf, q0r);
#pragma unroll
          for (int x0 = 0; x0 < D; ++x0) {
            T row[HD];
            ld_row<T, HD, C::VH>(tf + x0 * D + x_lo, row);
#pragma unroll
            for (int i = 0; i < HD; ++i) cand[i] = fg_opt<T>(cand[i], row[i] + q0r[x0], mx);
          }
        }
      } else {  // A == 3, table[x0][x1][x2]; sum of the two other rows in position order
        if (j == 0) {
          T q1[D], q2[D];
          ld_row<T, D, C::VR>(qf + D, q1);
          ld_row<T, D, C::VR>(qf + 2 * D, q2);
#pragma unroll 1
          for (int i = 0; i < HD; ++i) {
            T part[D];
#pragma unroll
            for (int x1 = 0; x1 < D; ++x1) {
              T row[D];
              ld_row<T, D, C::VT>(tf + (x_lo + i) * INNER + x1 * D, row);
#pragma unroll
              for (int x2 = 0; x2 < D; ++x2) row[x2] = row[x2] + (q1[x1] + q2[x2]);
              part[x1] = opt_tree<T, D>(row, mx);
            }
            of[i] = fg_opt<T>(init, opt_tree<T, D>(part, mx), mx);
          }
          ld_row<T, HD, C::VH>(of, cand);
        } else if (j == 1) {
#pragma unroll
          for (int i = 0; i < HD; ++i) cand[i] = init;
          T q2[D];
          ld_row<T, D, C::VR>(qf + 2 * D, q2);
#pragma unroll 1
          for (int x0 = 0; x0 < D; ++x0) {
            const T q0 = qf[x0];
            T s[D];
#pragma unroll
            for (int x = 0; x < D; ++x) s[x] = q0 + q2[x];
#pragma unroll
            for (int i = 0; i < HD; ++i) {
              T row[D];
              ld_row<T, D, C::VT>(tf + x0 * INNER + (x_lo + i) * D, row);
#pragma unroll
              for (int x2 = 0; x2 < D; ++x2) row[x2] = row[x2] + s[x2];
              cand[i] = fg_opt<T>(cand[i], opt_tree<T, D>(row, mx), mx);
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < HD; ++i) cand[i] = init;
          T q1[D];
          ld_row<T, D, C::VR>(qf + D, q1);
#pragma unroll 1
          for (int x0 = 0; x0 < D; ++x0) {
            const T q0 = qf[x0];
#pragma unroll
            for (int x1 = 0; x1 < D; ++x1) {
              const T s = q0 + q1[x1];
              T row[HD];
              ld_row<T, HD, C::VH>(tf + x0 * INNER + x1 * D + x_lo, row);
#pragma unroll
              for (int i = 0; i < HD; ++i) cand[i] = fg_opt<T>(cand[i], row[i] + s, mx);
            }
          }
        }
      }
      // damping and match of this thread's part of the row
      ld_row<T, HD, C::VH>(rt + f * R + j * D + x_lo, prev);
      match = damp_match_row<T, HD>(cand, prev, (cnt & 1) != 0, p.damp_factors != 0, lam, oml, stab);
    }
    if (SPLIT == 2) {  // both halves must match; partner = adjacent lane (same warp, same activity)
      const bool other = __shfl_xor_sync(0xffffffffu, match ? 1 : 0, 1) != 0;
      match = match && other;
    }
    if (active) {
      const bool sent = gate_decide(match, cnt);
      if (!sent) {
#pragma unroll
        for (int i = 0; i < HD; ++i) cand[i] = prev[i];
      }
      st_row<T, HD, C::VH>(of, cand);
      if (h == 0) {
        const int e = e_base + f * A + j;
        r_cnt[e] = cnt;
        if (r_sent) r_sent[e] = sent ? 1 : 0;
      }
    }
  }
}

// Persistent, software-pipelined factor->variable kernel.  Each CTA walks tiles
// blockIdx.x, blockIdx.x + gridDim.x, ...; while tile k is being computed the loads of tiles
// k+1 .. k+NS-1 are in flight (bulk async copies on per-stage mbarriers, cp.async gathers in
// per-tile commit groups, gather indices prefetched one more tile ahead in registers).
#define FG_SMEM_LIMIT (220 * 1024)
#ifndef FG_F2V_NS
#define FG_F2V_NS 2
#endif
template <typename T, int A, int D>
struct F2VPipe {
  using C = F2VCfg<T, A, D>;
  static constexpr int STAGE = C::NF * C::SP + 2 * C::NF * C::R;  // tab | qt | rt (elements)
  static constexpr int EPT = (C::NF * A + C::NT - 1) / C::NT;     // gathered edges per thread per tile
  static constexpr int WPT = (C::NF * A * C::SPLIT + C::NT - 1) / C::NT;  // compute items per thread
  static constexpr size_t smem_for(int ns) { return (size_t)(ns * STAGE + 2 * C::NF * C::R) * sizeof(T) + 64; }
  static constexpr int NS = FG_F2V_NS <= 2 ? 2 : (smem_for(FG_F2V_NS) <= FG_SMEM_LIMIT ? FG_F2V_NS : 2);
  static constexpr bool FITS = smem_for(2) <= FG_SMEM_LIMIT;
  static constexpr size_t SMEM = smem_for(NS);
};

template <typename T, int A, int D, typename OffT>
__global__ void __launch_bounds__(F2VCfg<T, A, D>::NT)
k_f2v_pipe(const fg_class_t c, const T *__restrict__ tables, const T *__restrict__ q_cur,
           const T *__restrict__ r_cur, T *__restrict__ r_next, const OffT *__restrict__ edge_qoff,
           uint8_t *__restrict__ r_cnt, uint8_t *__restrict__ r_sent, MaxSumParams p) {
  using C = F2VCfg<T, A, D>;
  using P = F2VPipe<T, A, D>;
  constexpr int S = C::S, R = C::R, SP = C::SP, NF = C::NF, NT = C::NT, NS = P::NS, EPT = P::EPT, WPT = P::WPT;
  constexpr int SPLIT = C::SPLIT;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T *stage0 = reinterpret_cast<T *>(smem_raw);
  T *ot0 = stage0 + NS * P::STAGE;  // two output buffers: the bulk store of tile k-1 may still be reading
  uint64_t *bars = reinterpret_cast<uint64_t *>(ot0 + 2 * NF * R);

  const int tid = threadIdx.x;
  const int n_tiles = (c.n_factors + NF - 1) / NF;
  const int n_my = ((int)blockIdx.x < n_tiles) ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    fence_mbar_init();
  }
  __syncthreads();

  // gather indices of my k-th tile -> registers
  auto load_idx = [&](int k, OffT (&idx)[EPT]) {
    if (k < n_my) {
      const int tile = (int)blockIdx.x + k * (int)gridDim.x;
      const int f0 = tile * NF;
      const int nf = min(NF, c.n_factors - f0);
      const int e_base = c.first_edge + f0 * A;
#pragma unroll
      for (int u = 0; u < EPT; ++u) {
        const int le = tid + u * NT;
        idx[u] = (le < nf * A) ? edge_qoff[e_base + le] : (OffT)0;
      }
    }
  };
  // start every load of my k-th tile into stage k % NS
  auto issue = [&](int k, const OffT (&idx)[EPT]) {
    if (k < n_my) {
      const int tile = (int)blockIdx.x + k * (int)gridDim.x;
      const int f0 = tile * NF;
      const int nf = min(NF, c.n_factors - f0);
      T *tab = stage0 + (k % NS) * P::STAGE;
      T *qt = tab + NF * SP;
      T *rt = qt + NF * R;
      const T *gtab = tables + c.table_base + (int64_t)f0 * S;
      const int64_t rbase = c.msg_base + (int64_t)f0 * R;
      const bool full = (nf == NF);
      const bool tma_tab = full && C::PAD == 0 && ((NF * S * (int)sizeof(T)) % 16 == 0);
      const bool tma_rows = full && ((NF * R * (int)sizeof(T)) % 16 == 0);
      if (tid == 0) {
        uint32_t bytes = 0;
        if (tma_tab) bytes += NF * S * (uint32_t)sizeof(T);
        if (tma_rows) bytes += NF * R * (uint32_t)sizeof(T);
        mbar_expect_tx(&bars[k % NS], bytes);  // bytes == 0: the plain arrival completes the phase
        if (tma_tab) tma_load_1d(tab, gtab, NF * S * (uint32_t)sizeof(T), &bars[k % NS]);
        if (tma_rows) tma_load_1d(rt, r_cur + rbase, NF * R * (uint32_t)sizeof(T), &bars[k % NS]);
      }
      if (!tma_tab) {
        if constexpr (C::QUADS) {  // 16-byte units into the (possibly padded) per-factor stride
          constexpr int Q = C::Q, E16 = C::E16;
          for (int u = tid; u < nf * Q; u += NT) {
            const int f = u / Q, w = u - f * Q;
            cp_async_16(tab + f * SP + w * E16, gtab + (int64_t)f * S + w * E16);
          }
        } else {
          for (int i = tid; i < nf * S; i += NT) cp_async_b<(int)sizeof(T)>(tab + i, gtab + i);
        }
      }
      if (!tma_rows) coop_copy_in<T>(rt, r_cur + rbase, nf * R, tid, NT);
      // q rows: thread le <-> edge (f, j) = (le / A, le % A)
#pragma unroll
      for (int u = 0; u < EPT; ++u) {
        const int le = tid + u * NT;
        if (le < nf * A) {
          const T *src = q_cur + (int64_t)idx[u];
          T *dst = qt + le * D;
#pragma unroll
          for (int i = 0; i < D / C::VR; ++i) cp_async_b<C::VR_BYTES>(dst + i * C::VR, src + i * C::VR);
        }
      }
    }
    cp_async_commit();  // one group per tile slot, even when empty: uniform accounting
  };

  // send-gate counters of my k-th tile -> registers, in the compute mapping (le -> (j, f))
  auto load_cnt = [&](int k, uint8_t (&cn)[WPT]) {
    if (k < n_my) {
      const int tile = (int)blockIdx.x + k * (int)gridDim.x;
      const int f0 = tile * NF;
      const int nf = min(NF, c.n_factors - f0);
      const int e_base = c.first_edge + f0 * A;
#pragma unroll
      for (int u = 0; u < WPT; ++u) {
        const int w = tid + u * NT;
        const int j = w / (NF * SPLIT), f = (w - j * (NF * SPLIT)) / SPLIT;
        cn[u] = (w < NF * A * SPLIT && f < nf) ? r_cnt[e_base + f * A + j] : (uint8_t)0;
      }
    }
  };

  OffT idx[EPT];
  uint8_t cnt[WPT];
  // prologue: tiles 0 .. NS-2 in flight, indices of tile NS-1 on their way
#pragma unroll 1
  for (int k = 0; k < NS - 1; ++k) {
    load_idx(k, idx);
    issue(k, idx);
  }
  load_idx(NS - 1, idx);
  load_cnt(0, cnt);

#pragma unroll 1
  for (int k = 0; k < n_my; ++k) {
    OffT idx_next[EPT];
    uint8_t cnt_next[WPT];
    load_idx(k + NS, idx_next);
    load_cnt(k + 1, cnt_next);
    issue(k + NS - 1, idx);  // into the stage tile k-1 has just vacated
#pragma unroll
    for (int u = 0; u < EPT; ++u) idx[u] = idx_next[u];
    cp_async_wait_group<NS - 1>();  // my gathers / padded copies of tile k have landed
    mbar_wait(&bars[k % NS], (uint32_t)((k / NS) & 1));
    if (tid == 0) tma_store_wait_read1();  // the bulk store of tile k-2 has finished reading ot[k & 1]
    __syncthreads();

    const int tile = (int)blockIdx.x + k * (int)gridDim.x;
    const int f0 = tile * NF;
    const int nf = min(NF, c.n_factors - f0);
    const T *tab = stage0 + (k % NS) * P::STAGE;
    T *ot = ot0 + (k & 1) * NF * R;
    f2v_compute_tile<T, A, D, WPT>(tab, tab + NF * SP, tab + NF * SP + NF * R, ot, nf, c.first_edge + f0 * A, cnt,
                                   r_cnt, r_sent, p, tid);
#pragma unroll
    for (int u = 0; u < WPT; ++u) cnt[u] = cnt_next[u];
    const int64_t rbase = c.msg_base + (int64_t)f0 * R;
    if (nf == NF && ((NF * R * (int)sizeof(T)) % 16 == 0)) {
      fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
        tma_store_1d(r_next + rbase, ot, NF * R * (uint32_t)sizeof(T));
        tma_store_commit();
      }
    } else {
      __syncthreads();
      coop_copy_out<T>(r_next + rbase, ot, nf * R, tid, NT);
      __syncthreads();
    }
  }
  cp_async_wait_all();
  if (tid == 0) tma_store_wait_read();
}

// ------------------------------------------------------------------------------------------------
// variable -> factor: one thread per variable, variables grouped in (domain, degree) classes
// ------------------------------------------------------------------------------------------------
#define FG_V2F_MAX_ENTRIES 24
#define FG_V2F_NT 256
#define FG_V2F_ROUNDS 1   // a thread finishes at most this many slots per tile

struct V2FEntry {
  fg_varclass_t vc;
  int32_t tile_begin;  // first tile of this class in the launch
  int32_t nv_tile;     // variables per tile
};
struct V2FTable {
  int32_t n;
  int32_t total_tiles;
  int32_t stage_elems;  // elements of one stage buffer (max over the classes)
  int32_t out_elems;    // elements of the output buffer
  int32_t avg_elems;    // elements of the per-slot normalisation scratch
  V2FEntry e[FG_V2F_MAX_ENTRIES];
};

template <typename T, int D>
struct V2FCfg {
  static constexpr int VR_BYTES = fg_gcd(16, D * (int)sizeof(T));
  static constexpr int VR = VR_BYTES / (int)sizeof(T);
};

struct V2FTile {
  int K, VS, nv_full, nv, nslots, slot0, var0, valid;
  int64_t qoff, uoff;
};

// variable stride (elements) of the gathered rows of one variable: K*D rounded up so that
// the stride counted in row-vector units is odd -> one-thread-per-variable reads hit distinct banks
__host__ __device__ inline int v2f_vstride(int K, int D, int VR) { return (((K * D) / VR) | 1) * VR; }

// tile t of the launch; `ci` is a cursor that only moves forward (tiles are visited in order)
__device__ __forceinline__ V2FTile v2f_tile(const V2FTable &tab, int t, int D, int VR, int &ci) {
  V2FTile o;
  o.valid = t < tab.total_tiles;
  if (!o.valid) { o.K = 1; o.VS = D; o.nv_full = o.nv = o.nslots = o.slot0 = o.var0 = 0; o.qoff = o.uoff = 0; return o; }
#pragma unroll 1
  while (ci + 1 < tab.n && t >= tab.e[ci + 1].tile_begin) ++ci;
  const V2FEntry &en = tab.e[ci];
  o.K = en.vc.degree;
  o.VS = v2f_vstride(o.K, D, VR);
  o.nv_full = en.nv_tile;
  const int v0 = (t - en.tile_begin) * en.nv_tile;
  o.nv = min(en.nv_tile, en.vc.n_vars - v0);
  o.nslots = o.nv * o.K;
  o.slot0 = en.vc.first_slot + v0 * o.K;
  o.var0 = en.vc.first_var + v0;
  o.qoff = en.vc.q_base + (int64_t)v0 * o.K * D;
  o.uoff = en.vc.unary_base + (int64_t)v0 * D;
  return o;
}

// costs_for_factor (maxsum.py:623-676) for slot f of a variable whose K gathered r rows are at
// col[g*D + x]: value-major, then factor order; the own factor contributes +0 (exact).
// K > 0: compile-time degree (inner loop unrolled); K == 0: run-time degree `k_rt`.  The loop over
// the values is a run-time loop on purpose: it keeps every degree variant a few dozen
// instructions, so the whole kernel stays resident in the instruction cache.  Raw sums go to
// `out` (shared memory); returns the normalisation term sum_cost / D.
template <typename T, int D, int K>
__device__ __forceinline__ T v2f_slot_msg(const T *__restrict__ col, const T *__restrict__ ur, int f, int k_rt,
                                          T *__restrict__ out) {
  T sum_cost = (T)0;
#pragma unroll 1
  for (int x = 0; x < D; ++x) {
    T m = ur[x];
    if constexpr (K > 0) {
#pragma unroll
      for (int g = 0; g < K; ++g) {
        const T cst = (g != f) ? col[g * D + x] : (T)0;
        sum_cost += cst;
        m += cst;
      }
    } else {
      for (int g = 0; g < k_rt; ++g) {
        const T cst = (g != f) ? col[g * D + x] : (T)0;
        sum_cost += cst;
        m += cst;
      }
    }
    out[x] = m;
  }
  return sum_cost / (T)D;
}

// select_value (maxsum.py:584-620): costs summed in `links` order, first optimum wins
template <typename T, int D, int K>
__device__ __forceinline__ void v2f_select(const T *__restrict__ col, const T *__restrict__ ur, int k_rt, bool mx,
                                           int32_t *value_out, T *cost_out) {
  int best = 0;
  T best_c = (T)0;
#pragma unroll 1
  for (int x = 0; x < D; ++x) {
    T tot = ur[x];
    if constexpr (K > 0) {
#pragma unroll
      for (int g = 0; g < K; ++g) tot += col[g * D + x];
    } else {
      for (int g = 0; g < k_rt; ++g) tot += col[g * D + x];
    }
    if (x == 0 || (mx ? (tot > best_c) : (tot < best_c))) { best = x; best_c = tot; }
  }
  *value_out = best;
  *cost_out = best_c;
}

#define FG_V2F_K_SWITCH(K_, CALL)              \
  switch (K_) {                                \
    case 1: { constexpr int KK = 1; CALL; } break; \
    case 2: { constexpr int KK = 2; CALL; } break; \
    case 3: { constexpr int KK = 3; CALL; } break; \
    case 4: { constexpr int KK = 4; CALL; } break; \
    case 5: { constexpr int KK = 5; CALL; } break; \
    case 6: { constexpr int KK = 6; CALL; } break; \
    case 7: { constexpr int KK = 7; CALL; } break; \
    case 8: { constexpr int KK = 8; CALL; } break; \
    default: { constexpr int KK = 0; CALL; } break; \
  }

// Persistent, software-pipelined variable->factor kernel over the (domain D, degree K) classes of
// one launch.  A tile is nv variables of one class = nv*K consecutive slots.  While tile k is being
// computed, the r-row gather (cp.async through slot_roff), the q_old tile and the unary tile (bulk
// async copies) of tile k+1 are in flight; gather indices and gate counters are prefetched in
// registers.  Compute: one thread per slot (message, damping, send gate), one thread per variable
// (value selection).
template <typename T, int D, typename OffT>
__global__ void __launch_bounds__(FG_V2F_NT)
k_v2f_pipe(const V2FTable tab, const OffT *__restrict__ slot_roff, const T *__restrict__ unary,
           const T *__restrict__ r_cur, const T *__restrict__ q_cur, T *__restrict__ q_next,
           uint8_t *__restrict__ q_cnt, uint8_t *__restrict__ q_sent, int32_t *__restrict__ value,
           T *__restrict__ value_cost, MaxSumParams p) {
  using C = V2FCfg<T, D>;
  constexpr int NT = FG_V2F_NT, NS = 2, RND = FG_V2F_ROUNDS;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T *stage0 = reinterpret_cast<T *>(smem_raw);  // per stage: rrow | qio | un
  T *qout = stage0 + NS * tab.stage_elems;      // output rows; also the scratch of the run-time-K path
  T *avg = qout + tab.out_elems;
  uint64_t *bars = reinterpret_cast<uint64_t *>(avg + tab.avg_elems);

  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  int cursor = 0;
  auto tile_at = [&](int k) { return v2f_tile(tab, (int)blockIdx.x + k * (int)gridDim.x, D, C::VR, cursor); };
  auto load_idx = [&](const V2FTile &t, OffT (&idx)[RND]) {
#pragma unroll
    for (int u = 0; u < RND; ++u) {
      const int sl = tid + u * NT;
      idx[u] = (t.valid && sl < t.nslots) ? slot_roff[t.slot0 + sl] : (OffT)0;
    }
  };
  auto load_cnt = [&](const V2FTile &t, uint8_t (&cn)[RND]) {
#pragma unroll
    for (int u = 0; u < RND; ++u) {
      const int sl = tid + u * NT;
      cn[u] = (t.valid && sl < t.nslots) ? q_cnt[t.slot0 + sl] : (uint8_t)0;
    }
  };
  auto issue = [&](int k, const V2FTile &t, const OffT (&idx)[RND]) {
    if (t.valid) {
      T *rrow = stage0 + (k % NS) * tab.stage_elems;
      T *qio = rrow + t.nv_full * t.VS;
      T *un = qio + t.nv_full * t.K * D;
      const uint32_t qbytes = (uint32_t)(t.nslots * D) * (uint32_t)sizeof(T);
      const uint32_t ubytes = (uint32_t)(t.nv * D) * (uint32_t)sizeof(T);
      const bool al = ((((size_t)t.nv_full * t.VS * sizeof(T)) & 15) == 0) &&
                      ((((size_t)t.nv_full * t.K * D * sizeof(T)) & 15) == 0);
      const bool tma_q = al && (qbytes % 16 == 0) && (((t.qoff * (int64_t)sizeof(T)) & 15) == 0);
      const bool tma_u = al && (ubytes % 16 == 0) && (((t.uoff * (int64_t)sizeof(T)) & 15) == 0);
      if (tid == 0) {
        mbar_expect_tx(&bars[k % NS], (tma_q ? qbytes : 0u) + (tma_u ? ubytes : 0u));
        if (tma_q) tma_load_1d(qio, q_cur + t.qoff, qbytes, &bars[k % NS]);
        if (tma_u) tma_load_1d(un, unary + t.uoff, ubytes, &bars[k % NS]);
      }
      if (!tma_q)
        for (int i = tid; i < t.nslots * D; i += NT) cp_async_b<(int)sizeof(T)>(qio + i, q_cur + t.qoff + i);
      if (!tma_u)
        for (int i = tid; i < t.nv * D; i += NT) cp_async_b<(int)sizeof(T)>(un + i, unary + t.uoff + i);
#pragma unroll
      for (int u = 0; u < RND; ++u) {
        const int sl = tid + u * NT;
        if (sl < t.nslots) {
          const int i = sl / t.K, g = sl - i * t.K;
          const T *src = r_cur + (int64_t)idx[u];
          T *dst = rrow + i * t.VS + g * D;
#pragma unroll
          for (int w = 0; w < D / C::VR; ++w) cp_async_b<C::VR_BYTES>(dst + w * C::VR, src + w * C::VR);
        }
      }
    }
    cp_async_commit();
  };

  OffT idx[RND];
  uint8_t cnt[RND];
  V2FTile t_cur = tile_at(0), t_n1 = tile_at(1), t_n2 = tile_at(2);
  load_idx(t_cur, idx);
  issue(0, t_cur, idx);
  load_idx(t_n1, idx);
  load_cnt(t_cur, cnt);
  const bool mx = p.mode_max != 0;
  const T lam = (T)p.damping, oml = (T)p.one_minus_damping, stab = (T)p.stability;

#pragma unroll 1
  for (int k = 0; t_cur.valid; ++k) {
    OffT idx_next[RND];
    uint8_t cnt_next[RND];
    load_idx(t_n2, idx_next);
    load_cnt(t_n1, cnt_next);
    issue(k + 1, t_n1, idx);  // into the stage tile k-1 has vacated
#pragma unroll
    for (int u = 0; u < RND; ++u) idx[u] = idx_next[u];
    cp_async_wait_group<1>();
    mbar_wait(&bars[k % NS], (uint32_t)((k / NS) & 1));
    if (tid == 0) tma_store_wait_read();  // the previous tile's bulk store no longer reads qout
    __syncthreads();

    const V2FTile t = t_cur;
    const int K = t.K;
    T *rrow = stage0 + (k % NS) * tab.stage_elems;
    const T *qio = rrow + t.nv_full * t.VS;
    const T *un = qio + t.nv_full * K * D;
    {  // one thread per variable, packed into the first warps (a spread mapping would make every
       // warp issue the whole selection code for a handful of lanes)
      const int vi = tid;
      if (vi < t.nv) {
        int32_t val;
        T cst;
        FG_V2F_K_SWITCH(K, (v2f_select<T, D, KK>(rrow + vi * t.VS, un + vi * D, K, mx, &val, &cst)))
        value[t.var0 + vi] = val;
        value_cost[t.var0 + vi] = cst;
      }
    }
    // one thread per slot: message, damping, send gate
#pragma unroll
    for (int u = 0; u < RND; ++u) {
      const int sl = tid + u * NT;
      if (sl < t.nslots) {
        const int i = sl / K, f = sl - i * K;
        const T *col = rrow + i * t.VS;
        T cand[D], prev[D];
        T avg_c;
        FG_V2F_K_SWITCH(K, (avg_c = v2f_slot_msg<T, D, KK>(col, un + i * D, f, K, qout + sl * D)))
        ld_row<T, D, C::VR>(qout + sl * D, cand);
#pragma unroll
        for (int x = 0; x < D; ++x) cand[x] = cand[x] - avg_c;
        ld_row<T, D, C::VR>(qio + sl * D, prev);
        uint8_t c8 = cnt[u];
        const bool sent = damp_gate_row<T, D>(cand, prev, c8, p.damp_vars != 0, lam, oml, stab);
        st_row<T, D, C::VR>(qout + sl * D, cand);
        q_cnt[t.slot0 + sl] = c8;
        if (q_sent) q_sent[t.slot0 + sl] = sent ? 1 : 0;
      }
    }
#pragma unroll
    for (int u = 0; u < RND; ++u) cnt[u] = cnt_next[u];
    const uint32_t obytes = (uint32_t)(t.nslots * D) * (uint32_t)sizeof(T);
    if ((obytes % 16 == 0) && (((t.qoff * (int64_t)sizeof(T)) & 15) == 0)) {
      fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
        tma_store_1d(q_next + t.qoff, qout, obytes);
        tma_store_commit();
      }
    } else {
      __syncthreads();
      for (int i = tid; i < t.nslots * D; i += NT) q_next[t.qoff + i] = qout[i];
      __syncthreads();
    }
    t_cur = t_n1;
    t_n1 = t_n2;
    t_n2 = tile_at(k + 3);
  }
  cp_async_wait_all();
  if (tid == 0) tma_store_wait_read();
}

// ------------------------------------------------------------------------------------------------
// host-side dispatch
// ------------------------------------------------------------------------------------------------
#define FG_FAST_DOMS(X) X(2) X(3) X(4) X(5) X(6) X(8) X(10) X(16) X(20)
#define FG_FAST_DOMS_A3(X) X(2) X(3) X(4) X(5) X(8)

inline bool fg_fast_dom(int d) {
#define X(n) if (d == n) return true;
  FG_FAST_DOMS(X)
#undef X
  return false;
}
inline bool fg_fast_dom_a3(int d) {
#define X(n) if (d == n) return true;
  FG_FAST_DOMS_A3(X)
#undef X
  return false;
}

inline int fg_env_int(const char *name, int dflt) {
  const char *e = getenv(name);
  const int v = e ? atoi(e) : 0;
  return v > 0 ? v : dflt;
}

inline bool fg_env_is(const char *name, char first) {
  const char *e = getenv(name);
  return e && e[0] == first;
}

inline bool fg_fast_disabled() {
  const char *e = getenv("PYDCOP_B200_NO_FAST");
  return e && e[0] == '1';
}

template <typename T, int A, int D>
inline void launch_f2v_tile(const fg_class_t &c, const fg_maxsum_desc_t &d, const T *q_cur, const T *r_cur, T *r_next,
                            const MaxSumParams &p, cudaStream_t st) {
  using C = F2VCfg<T, A, D>;
  auto kern = k_f2v_pipe<T, A, D, uint32_t>;
  using PP = F2VPipe<T, A, D>;
  static int ctas_per_sm = 0, n_sm = 0;  // one per instantiation
  if (!ctas_per_sm) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PP::SMEM);
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, C::NT, PP::SMEM);
    if (ctas_per_sm < 1) ctas_per_sm = 1;
    // the two sides of a cycle run concurrently on two streams: leave room for the other kernel
    const int cap = fg_env_int("PYDCOP_B200_F2V_CPS", 2);
    if (ctas_per_sm > cap) ctas_per_sm = cap;
  }
  const int n_tiles = (c.n_factors + C::NF - 1) / C::NF;
  const unsigned blocks = (unsigned)min(n_tiles, n_sm * ctas_per_sm);
  kern<<<blocks, C::NT, PP::SMEM, st>>>(c, (const T *)d.dev_tables, q_cur, r_cur, r_next, d.dev_edge_qoff32, d.dev_r_cnt,
                                       d.dev_r_sent, p);
}

template <typename T, int A, int D>
inline bool try_f2v_tile(bool probe, const fg_class_t &c, const fg_maxsum_desc_t &d, const T *q_cur, const T *r_cur,
                         T *r_next, const MaxSumParams &p, cudaStream_t st) {
  if constexpr (F2VPipe<T, A, D>::FITS) {
    if (!probe) launch_f2v_tile<T, A, D>(c, d, q_cur, r_cur, r_next, p, st);
    return true;
  } else {
    return false;  // staging does not fit in shared memory: generic kernel
  }
}

// probe == true: only report whether a tiled kernel exists for the class
template <typename T>
inline bool dispatch_f2v(bool probe, const fg_class_t &c, const fg_maxsum_desc_t &d, const T *q_cur, const T *r_cur,
                         T *r_next, const MaxSumParams &p, cudaStream_t st) {
  const int D = c.dom[0];
  switch (c.arity) {
    case 1:
      switch (D) {
#define X(n) case n: return try_f2v_tile<T, 1, n>(probe, c, d, q_cur, r_cur, r_next, p, st);
        FG_FAST_DOMS(X)
#undef X
      }
      return false;
    case 2:
      switch (D) {
#define X(n) case n: return try_f2v_tile<T, 2, n>(probe, c, d, q_cur, r_cur, r_next, p, st);
        FG_FAST_DOMS(X)
#undef X
      }
      return false;
    case 3:
      switch (D) {
#define X(n) case n: return try_f2v_tile<T, 3, n>(probe, c, d, q_cur, r_cur, r_next, p, st);
        FG_FAST_DOMS_A3(X)
#undef X
      }
      return false;
  }
  return false;
}

struct V2FLaunch {
  V2FTable tab;
  size_t smem = 0;
};

// Split the regular variable classes (degree 1..16, one domain size D) into launches of at most
// FG_V2F_MAX_ENTRIES classes each, choosing the tile size of every class.
inline void v2f_build_launches(const std::vector<fg_varclass_t> &vcs, int D, size_t elem, std::vector<V2FLaunch> &out) {
  V2FLaunch cur;
  auto reset = [&]() {
    cur = V2FLaunch();
    cur.tab.n = 0;
    cur.tab.total_tiles = 0;
    cur.tab.stage_elems = 0;
    cur.tab.out_elems = 0;
    cur.tab.avg_elems = 0;
  };
  auto flush = [&]() {
    if (cur.tab.n) {
      // 16-byte aligned section sizes
      const int al = (int)(16 / elem);
      cur.tab.stage_elems = (cur.tab.stage_elems + al - 1) / al * al;
      cur.tab.out_elems = (cur.tab.out_elems + al - 1) / al * al;
      cur.tab.avg_elems = (cur.tab.avg_elems + al - 1) / al * al;
      cur.smem = (size_t)(2 * cur.tab.stage_elems + cur.tab.out_elems + cur.tab.avg_elems) * elem + 64;
      out.push_back(cur);
    }
    reset();
  };
  reset();
  std::vector<fg_varclass_t> order(vcs);
  std::stable_sort(order.begin(), order.end(),
                   [](const fg_varclass_t &a, const fg_varclass_t &b) { return a.degree > b.degree; });  // costly tiles first
  for (const fg_varclass_t &vc : order) {
    if (vc.dom != D || vc.degree < 1 || vc.n_vars == 0) continue;
    const int K = vc.degree;
    const int VR = fg_gcd(16, D * (int)elem) / (int)elem;
    const int VS = v2f_vstride(K, D, VR);
    const size_t per_var = (size_t)(VS + K * D + D) * elem;  // stage bytes per variable
    static const int stage_kb = fg_env_int("PYDCOP_B200_V2F_STAGE_KB", 14);
    int nv = (int)((size_t)(stage_kb * 1024) / per_var);
    const int cap = (FG_V2F_ROUNDS * FG_V2F_NT) / K;        // slots per tile <= ROUNDS * NT
    if (nv > cap) nv = cap;
    nv = nv / 8 * 8;
    if (nv < 8) nv = 8;
    if (nv > FG_V2F_NT) nv = FG_V2F_NT;
    V2FEntry e;
    e.vc = vc;
    e.tile_begin = cur.tab.total_tiles;
    e.nv_tile = nv;
    cur.tab.e[cur.tab.n++] = e;
    cur.tab.total_tiles += (vc.n_vars + nv - 1) / nv;
    const int st = nv * (VS + K * D + D), ot = nv * K * D;
    if (st > cur.tab.stage_elems) cur.tab.stage_elems = st;
    if (ot > cur.tab.out_elems) cur.tab.out_elems = ot;
    if (ot / D > cur.tab.avg_elems) cur.tab.avg_elems = ot / D;
    if (cur.tab.n == FG_V2F_MAX_ENTRIES) flush();
  }
  flush();
}

template <typename T, int D>
inline void launch_v2f_classes(const V2FLaunch &L, const fg_maxsum_desc_t &d, const T *r_cur, const T *q_cur, T *q_next,
                               const MaxSumParams &p, cudaStream_t st) {
  auto kern = k_v2f_pipe<T, D, uint32_t>;
  static size_t attr_smem = 0;
  static int n_sm = 0;
  if (L.smem > attr_smem) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem);
    attr_smem = L.smem;
  }
  if (!n_sm) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  }
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, FG_V2F_NT, L.smem);
  if (per_sm < 1) per_sm = 1;
  static const int cap = fg_env_int("PYDCOP_B200_V2F_CPS", 3);
  if (per_sm > cap) per_sm = cap;
  const unsigned blocks = (unsigned)std::min(L.tab.total_tiles, n_sm * per_sm);
  kern<<<blocks, FG_V2F_NT, L.smem, st>>>(L.tab, d.dev_slot_roff32, (const T *)d.dev_unary, r_cur, q_cur, q_next,
                                          d.dev_q_cnt, d.dev_q_sent, d.dev_value, (T *)d.dev_value_cost, p);
}

template <typename T>
inline bool dispatch_v2f_classes(int D, const V2FLaunch &L, const fg_maxsum_desc_t &d, const T *r_cur, const T *q_cur,
                                 T *q_next, const MaxSumParams &p, cudaStream_t st) {
  switch (D) {
#define X(n) case n: launch_v2f_classes<T, n>(L, d, r_cur, q_cur, q_next, p, st); return true;
    FG_FAST_DOMS(X)
#undef X
  }
  return false;
}

struct MaxSumFastPlan {
  bool off32 = false;                    // 32-bit gather offsets available (required by the fast kernels)
  std::vector<uint8_t> f2v;              // per factor class: tiled kernel available
  std::vector<V2FLaunch> v2f;            // fused launches over regular variable classes
  std::vector<int> v2f_dom;              // domain size of each launch
  std::vector<int> slow_varclasses;      // variable classes left to the generic kernel
};

inline void maxsum_fast_plan(const fg_maxsum_desc_t &d, const std::vector<fg_class_t> &classes,
                             const std::vector<fg_varclass_t> &vcs, MaxSumFastPlan &plan) {
  plan.f2v.assign(classes.size(), 0);
  plan.v2f.clear();
  plan.v2f_dom.clear();
  plan.slow_varclasses.clear();
  plan.off32 = d.dev_slot_roff32 != nullptr && d.dev_edge_qoff32 != nullptr;
  const bool fast = plan.off32 && !fg_fast_disabled();
  for (size_t i = 0; fast && i < classes.size(); ++i) {
    const fg_class_t &c = classes[i];
    bool uni = true;
    for (int j = 1; j < c.arity; ++j) uni = uni && c.dom[j] == c.dom[0];
    if (!uni) continue;
    MaxSumParams dummy{};
    const bool ok = d.precision == FG_F64
                        ? dispatch_f2v<double>(true, c, d, nullptr, nullptr, nullptr, dummy, nullptr)
                        : dispatch_f2v<float>(true, c, d, nullptr, nullptr, nullptr, dummy, nullptr);
    if (ok) plan.f2v[i] = 1;
  }
  const size_t elem = d.precision == FG_F64 ? 8 : 4;
  std::vector<uint8_t> taken(vcs.size(), 0);
  for (size_t i = 0; fast && i < vcs.size(); ++i) {
    if (vcs[i].flags & FG_CLASS_GHOST) { taken[i] = 1; continue; }
    if (taken[i] || vcs[i].degree < 1 || !fg_fast_dom(vcs[i].dom)) continue;
    const int D = vcs[i].dom;
    std::vector<fg_varclass_t> same;
    for (size_t j = i; j < vcs.size(); ++j)
      if (!taken[j] && !(vcs[j].flags & FG_CLASS_GHOST) && vcs[j].dom == D && vcs[j].degree >= 1) {
        same.push_back(vcs[j]);
        taken[j] = 1;
      }
    std::vector<V2FLaunch> ls;
    v2f_build_launches(same, D, elem, ls);
    for (auto &l : ls) { plan.v2f.push_back(l); plan.v2f_dom.push_back(D); }
  }
  for (size_t i = 0; i < vcs.size(); ++i)
    if (!taken[i] && vcs[i].n_slots > 0) plan.slow_varclasses.push_back((int)i);
}

template <typename T>
inline bool maxsum_fast_f2v(const MaxSumFastPlan &plan, int ci, const fg_class_t &c, const fg_maxsum_desc_t &d,
                            const T *q_cur, const T *r_cur, T *r_next, const MaxSumParams &p, cudaStream_t st,
                            int64_t &launches) {
  if (!plan.f2v[ci]) return false;
  const bool ok = dispatch_f2v<T>(false, c, d, q_cur, r_cur, r_next, p, st);
  if (ok) ++launches;
  return ok;
}
