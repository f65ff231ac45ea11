// TEST INFRASTRUCTURE: runs the GDBA CUDA kernel SOURCE (pydcop_b200/csrc/gdba_kernels.cuh) on the
// CPU, one "thread" after the other, so its logic can be compared with the oracle and the reference
// trajectories without a GPU.  Nothing in the product links or calls this.
//   g++ -O1 -std=c++17 -ffp-contract=off -shared -fPIC -o gdba_host.so gdba_host.cpp
// The descriptor is the C-ABI's fg_gdba_desc_t with HOST pointers.
#include <stdint.h>
#include <string.h>

struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 blockIdx, blockDim, threadIdx;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

#include "../../pydcop_b200/csrc/gdba_kernels.cuh"

template <typename F>
static void launch(int n, int block, F body) {
  blockDim = Dim3{(unsigned)block, 1, 1};
  for (unsigned b = 0; b < (unsigned)((n + block - 1) / block); ++b)
    for (unsigned t = 0; t < (unsigned)block; ++t) {
      blockIdx = Dim3{b, 0, 0};
      threadIdx = Dim3{t, 0, 0};
      body();
    }
}

static MgmSide side(const fg_gdba_desc_t *d) {
  return MgmSide{d->classes, d->dev_dom_size, d->dev_var_id, d->dev_var_rank, d->dev_edge_var, d->dev_edge_class,
                 d->dev_var_ptr, d->dev_slot_edge, d->dev_nbr_ptr, d->dev_nbr_idx, nullptr};
}

// the two launches of gdba.cu; each kernel boundary is a full pass over the "threads"
template <typename T>
static void cycle_t(const fg_gdba_desc_t *d, int64_t done) {
  const MgmSide g = side(d);
  const int n = d->n_vars;
  int32_t *vin = d->dev_value[done & 1], *vout = d->dev_value[(done + 1) & 1];
  const int64_t *mod_off = d->increase_mode == FG_GDBA_INCREASE_T ? nullptr : d->dev_mod_off;
  const uint32_t cyc = (uint32_t)(done + 1);
  launch(n, 128, [&] {
    k_gdba_eval<T>(g, n, (const T *)d->dev_tables, (const T *)d->dev_unary, d->dev_unary_off,
                   (const T *)d->dev_viol_ref, d->dev_mod, mod_off, d->modifier, d->violation, vin, (T *)d->dev_cost,
                   d->dev_has_cost, (T *)d->dev_improve, d->dev_new_value, d->dev_violated, d->mode_max, d->seed, cyc);
  });
  launch(n, 256, [&] {
    k_gdba_decide<T>(g, n, (const T *)d->dev_improve, d->dev_new_value, d->dev_violated, d->dev_mod, mod_off,
                     d->increase_mode, d->mode_max, vin, vout, (T *)d->dev_cost, d->dev_breakout);
  });
}

extern "C" {
void gdba_host_init(const fg_gdba_desc_t *d) {
  if (d->mod_size > 0) memset(d->dev_mod, 0, sizeof(int32_t) * (size_t)d->mod_size);
  launch(d->n_vars, 128, [&] {
    k_mgm_init(side(d), d->n_vars, d->dev_init_value, d->seed, d->dev_value[0], d->dev_has_cost);
  });
}

void gdba_host_cycle(const fg_gdba_desc_t *d, int64_t done) {
  if (d->precision == FG_F64) cycle_t<double>(d, done);
  else cycle_t<float>(d, done);
}
}  // extern "C"
