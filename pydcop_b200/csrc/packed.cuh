// Pair arithmetic helpers for the warp-autonomous kernels (sm_90a).
//
// The kernels keep message rows as pairs of values (float2 / double2) so that loads and stores move 8 or
// 16 bytes per lane.  Hopper has no packed fp32 add / mul and no three-input min / max, so every helper is
// one correctly rounded IEEE operation per element (__fadd_rn / __fsub_rn / __fmul_rn are never contracted
// into an FMA): results are bit-identical to the scalar code and to the CPU oracle.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "maxsum_fast.cuh"   // MatchEps, approx_match1, fg_abs, Inf

template <typename T> struct Pair;
template <> struct Pair<float> { using type = float2; };
template <> struct Pair<double> { using type = double2; };

__device__ __forceinline__ float2 padd(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 psub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 pmul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ double2 padd(double2 a, double2 b) { return make_double2(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y)); }
__device__ __forceinline__ double2 psub(double2 a, double2 b) { return make_double2(__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y)); }
__device__ __forceinline__ double2 pmul(double2 a, double2 b) { return make_double2(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)); }

template <typename T> __device__ __forceinline__ typename Pair<T>::type pmake(T x, T y);
template <> __device__ __forceinline__ float2 pmake<float>(float x, float y) { return make_float2(x, y); }
template <> __device__ __forceinline__ double2 pmake<double>(double x, double y) { return make_double2(x, y); }

// optimum of two / three values; MX: max instead of min.  NaN operands are ignored like fminf / fmaxf.
template <bool MX> __device__ __forceinline__ float opt2(float a, float b) { return MX ? fmaxf(a, b) : fminf(a, b); }
template <bool MX> __device__ __forceinline__ double opt2(double a, double b) { return MX ? fmax(a, b) : fmin(a, b); }
template <bool MX> __device__ __forceinline__ float opt3(float a, float b, float c) { return opt2<MX>(opt2<MX>(a, b), c); }
template <bool MX> __device__ __forceinline__ double opt3(double a, double b, double c) { return opt2<MX>(opt2<MX>(a, b), c); }

// optimum of N values held in registers (static indices): tree of three-way optima
template <bool MX, typename T, int N>
__device__ __forceinline__ T opt_tree3(const T (&v)[N]) {
  if constexpr (N == 1) {
    return v[0];
  } else if constexpr (N == 2) {
    return opt2<MX>(v[0], v[1]);
  } else if constexpr (N == 3) {
    return opt3<MX>(v[0], v[1], v[2]);
  } else {
    constexpr int M = (N + 2) / 3;
    T w[M];
#pragma unroll
    for (int g = 0; g < N / 3; ++g) w[g] = opt3<MX>(v[3 * g], v[3 * g + 1], v[3 * g + 2]);
    if constexpr (N % 3 == 1) w[M - 1] = v[N - 1];
    if constexpr (N % 3 == 2) w[M - 1] = opt2<MX>(v[N - 2], v[N - 1]);
    return opt_tree3<MX, T, M>(w);
  }
}

// Damping + approx_match (maxsum.py:679-710) of N values (N even) held as N/2 pairs: same results as
// damp_match_row (maxsum_fast.cuh) — cand <- damped values, returns whether every element matches
// `prev` — with the arithmetic in packed form.  Division-free classification with the literal form
// (IEEE division) whenever an element sits within 2^-20 of the threshold or outside the safe range.
template <typename T, int N>
__device__ __forceinline__ bool damp_match_pairs(T (&cand)[N], const T (&prev)[N], bool has_prev, bool damp_side, T lam,
                                                 T oml, T stab) {
  static_assert(N % 2 == 0, "pairs");
  using P = typename Pair<T>::type;
  if (!has_prev) return false;
  const P lam2 = pmake<T>(lam, lam), oml2 = pmake<T>(oml, oml), stab2 = pmake<T>(stab, stab);
  const P two2 = pmake<T>((T)2, (T)2);
  const P lo2 = pmake<T>(MatchEps<T>::lo(), MatchEps<T>::lo()), hi2 = pmake<T>(MatchEps<T>::hi(), MatchEps<T>::hi());
  const bool stab_pos = stab > (T)0;   // the product form needs a positive threshold; otherwise the literal form
  bool all_ok = true, unsure = !stab_pos;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const P p = pmake<T>(prev[2 * i], prev[2 * i + 1]);
    P c = pmake<T>(cand[2 * i], cand[2 * i + 1]);
    if (damp_side) c = padd(pmul(lam2, p), pmul(oml2, c));   // lam * prev + (1 - lam) * c: three roundings
    cand[2 * i] = c.x;
    cand[2 * i + 1] = c.y;
    const P s = padd(p, c);
    const P d2 = pmul(two2, psub(p, c));      // 2 * (prev - c): |.| taken in the comparisons
    const P rhs = pmul(stab2, s);             // stab * (prev + c)
    const P rl = pmul(rhs, lo2), rh = pmul(rhs, hi2);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const T ad = fg_abs<T>(k ? d2.y : d2.x), ar = fg_abs<T>(k ? rhs.y : rhs.x);
      const T al = fg_abs<T>(k ? rl.y : rl.x), ah = fg_abs<T>(k ? rh.y : rh.x);
      const bool eq = (k ? p.y : p.x) == (k ? c.y : c.x);
      const bool safe = (ar > MatchEps<T>::tiny()) && (ar < Inf<T>::pos());
      const bool lt = ad < al, gt = ad > ah;
      unsure = unsure || (!eq && !(safe && (lt || gt)));
      all_ok = all_ok && (eq || lt);
    }
  }
  if (unsure) {  // rare
    all_ok = true;
#pragma unroll
    for (int x = 0; x < N; ++x)
      if (!approx_match1<T>(cand[x], prev[x], stab)) all_ok = false;
  }
  return all_ok;
}

// Same for TWO message rows at once (the first NA elements belong to row a, the rest to row b; N even,
// NA may be odd — a binary factor's two half rows of D/2 values): both rows hold a previous message.
// ma / mb <- whether every element of row a / row b matches.
template <typename T, int N, int NA>
__device__ __forceinline__ void damp_match_pairs2(T (&cand)[N], const T (&prev)[N], bool damp_side, T lam, T oml, T stab,
                                                  bool &ma, bool &mb) {
  static_assert(N % 2 == 0 && NA > 0 && NA < N, "pairs");
  using P = typename Pair<T>::type;
  const P lam2 = pmake<T>(lam, lam), oml2 = pmake<T>(oml, oml), stab2 = pmake<T>(stab, stab);
  const P two2 = pmake<T>((T)2, (T)2);
  const P lo2 = pmake<T>(MatchEps<T>::lo(), MatchEps<T>::lo()), hi2 = pmake<T>(MatchEps<T>::hi(), MatchEps<T>::hi());
  bool ok_a = true, ok_b = true, unsure = !(stab > (T)0);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const P p = pmake<T>(prev[2 * i], prev[2 * i + 1]);
    P c = pmake<T>(cand[2 * i], cand[2 * i + 1]);
    if (damp_side) c = padd(pmul(lam2, p), pmul(oml2, c));
    cand[2 * i] = c.x;
    cand[2 * i + 1] = c.y;
    const P s = padd(p, c);
    const P d2 = pmul(two2, psub(p, c));
    const P rhs = pmul(stab2, s);
    const P rl = pmul(rhs, lo2), rh = pmul(rhs, hi2);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const T ad = fg_abs<T>(k ? d2.y : d2.x), ar = fg_abs<T>(k ? rhs.y : rhs.x);
      const T al = fg_abs<T>(k ? rl.y : rl.x), ah = fg_abs<T>(k ? rh.y : rh.x);
      const bool eq = (k ? p.y : p.x) == (k ? c.y : c.x);
      const bool safe = (ar > MatchEps<T>::tiny()) && (ar < Inf<T>::pos());
      const bool lt = ad < al, gt = ad > ah;
      unsure = unsure || (!eq && !(safe && (lt || gt)));
      if (2 * i + k < NA) ok_a = ok_a && (eq || lt);
      else ok_b = ok_b && (eq || lt);
    }
  }
  if (unsure) {  // rare
    ok_a = ok_b = true;
#pragma unroll
    for (int x = 0; x < N; ++x)
      if (!approx_match1<T>(cand[x], prev[x], stab)) { if (x < NA) ok_a = false; else ok_b = false; }
  }
  ma = ok_a;
  mb = ok_b;
}
