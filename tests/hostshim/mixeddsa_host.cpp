// TEST INFRASTRUCTURE: runs the MixedDSA CUDA kernel SOURCE (pydcop_b200/csrc/mixeddsa_kernels.cuh, and
// k_dsa_con_opt of dsa_generic.cuh) on the CPU, one "thread" after the other, in the launch order of mixeddsa.cu, so
// its logic can be compared with the oracle and the reference trajectories without a GPU.  Nothing in the product
// links or calls this.
//   g++ -O1 -std=c++17 -ffp-contract=off -I <cuda>/include -shared -fPIC -o mixeddsa_host.so mixeddsa_host.cpp
// The descriptor is the C-ABI's fg_mixeddsa_desc_t with HOST pointers.
#include <math.h>
#include <stdint.h>
#include <string.h>

struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 blockIdx, blockDim, threadIdx;
#define __launch_bounds__(...)
static inline float __int_as_float(unsigned x) { float f; memcpy(&f, &x, 4); return f; }
static inline double __longlong_as_double(unsigned long long x) { double f; memcpy(&f, &x, 8); return f; }

#include "../../pydcop_b200/csrc/dsa_generic.cuh"
#include "../../pydcop_b200/csrc/mixeddsa_kernels.cuh"

template <typename F>
static void launch(int64_t n, int block, F body) {
  blockDim = Dim3{(unsigned)block, 1, 1};
  for (int64_t b = 0; b < (n + block - 1) / block; ++b)
    for (unsigned t = 0; t < (unsigned)block; ++t) {
      blockIdx = Dim3{(unsigned)b, 0, 0};
      threadIdx = Dim3{t, 0, 0};
      body();
    }
}

static MgmSide side(const fg_mixeddsa_desc_t *d) {
  return MgmSide{d->classes, d->dev_dom_size, d->dev_var_id, nullptr, d->dev_edge_var, d->dev_edge_class,
                 d->dev_var_ptr, d->dev_slot_edge, d->dev_nbr_ptr, d->dev_nbr_idx, d->dev_unary_off};
}

template <typename T>
static void init_t(const fg_mixeddsa_desc_t *d) {
  for (int ci = 0; ci < d->n_classes; ++ci) {
    const fg_class_t &c = d->classes[ci];
    if (!c.n_factors) continue;
    launch(c.n_factors, 128, [&] { k_dsa_con_opt<T>(c, (const T *)d->dev_tables, (T *)d->dev_con_opt, d->mode_max); });
  }
  launch(d->n_vars, 128, [&] {
    k_mixeddsa_init(side(d), d->n_vars, d->dev_init_value, d->seed, d->dev_value[0], d->dev_has_cost);
  });
}

template <typename T, int DMAX>
static void round_t(const fg_mixeddsa_desc_t *d, int64_t done) {
  int32_t *vin = d->dev_value[done & 1], *vout = d->dev_value[(done + 1) & 1];
  launch(d->n_vars, 128, [&] {
    k_mixeddsa_step<T, DMAX>(side(d), d->n_vars, (const T *)d->dev_tables, (const T *)d->dev_unary, d->dev_soft_end,
                             (const T *)d->dev_con_opt, vin, vout, (T *)d->dev_cost, d->dev_has_cost, d->dev_h_best,
                             d->dev_branch, d->mode_max, d->variant, d->proba_hard, d->proba_soft, (T)INFINITY,
                             d->seed, (uint32_t)(done + 1));
  });
}

template <typename T>
static void cycle_t(const fg_mixeddsa_desc_t *d, int64_t done) {
  if (mixeddsa_dmax(d->classes, d->n_classes) <= 32) round_t<T, 32>(d, done);
  else round_t<T, FG_MAX_DOM>(d, done);
}

extern "C" {
void mixeddsa_host_init(const fg_mixeddsa_desc_t *d) {
  if (d->precision == FG_F64) init_t<double>(d);
  else init_t<float>(d);
}

void mixeddsa_host_cycle(const fg_mixeddsa_desc_t *d, int64_t done) {
  if (d->precision == FG_F64) cycle_t<double>(d, done);
  else cycle_t<float>(d, done);
}
}  // extern "C"
