// 8-bit storage of integer cost tables (DESIGN.md §3): the one rule that decides whether a table entry may be
// stored as a signed byte.  Host and device share it; it includes nothing of the engine, so a CPU test can compile
// it with g++ (__host__ / __device__ defined away).
#pragma once
#include <math.h>

// true when int8 code (int8_t)v decodes back to exactly the bits of v: an integer in [-128, 127] that is not -0.0
// (code 0 decodes to +0.0).  NaN and +/-inf fail the range test; denormals and other fractions fail the integer test.
template <typename T>
__host__ __device__ inline bool fg_table_entry_fits_i8(T v) {
  const double x = (double)v;   // exact for float and double
  if (!(x >= -128.0 && x <= 127.0)) return false;
  if ((double)(int)x != x) return false;
  return x != 0.0 || copysign(1.0, x) > 0.0;
}
