// Philox4x32-10, the injected-draw generator of the DSA parity definition (oracle/philox.py).
#pragma once
#include <stdint.h>

__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                       uint32_t c3, uint32_t k0, uint32_t k1,
                                                       uint32_t out[4]) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

#define FG_PHILOX_INIT_CYCLE 0xFFFFFFFFu

// u in [0,1) with 53 bits
__host__ __device__ __forceinline__ double philox_u53(const uint32_t b[4]) {
  return ((double)(b[0] >> 5) * 67108864.0 + (double)(b[1] >> 6)) / 9007199254740992.0;
}
__host__ __device__ __forceinline__ int philox_choice(const uint32_t b[4], int n) {
  return (int)(((uint64_t)b[2] * (uint64_t)n) >> 32);
}

// block of counter (var, cycle, purpose, 0): one stream per kind of decision (MGM-2); purpose 0 is
// the block every existing draw uses
__host__ __device__ __forceinline__ void philox_draw(uint32_t var, uint32_t cycle, uint32_t purpose, uint64_t seed,
                                                     uint32_t out[4]) {
  philox4x32_10(var, cycle, purpose, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), out);
}

// Philox key of internal variable v: its own entry of var_seed (a batch of problems, each with its own seed), or the
// run's one seed when var_seed is NULL.  Read at the draw only, so the paths that draw nothing load nothing.
__host__ __device__ __forceinline__ uint64_t fg_var_seed(const uint64_t *var_seed, int v, uint64_t seed) {
  return var_seed ? var_seed[v] : seed;
}

// Parameter set of internal variable v: its entry of the set table (a batch of problems, each with its own algorithm
// parameters; the table is the device copy fg_upload_psets made).  Callers read it only when var_pset is not NULL and
// take the descriptor's scalars otherwise.
template <class P>
__host__ __device__ __forceinline__ const P &fg_pset(const uint16_t *var_pset, const P *psets, int v) {
  return psets[var_pset[v]];
}
