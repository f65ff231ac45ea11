// TEST INFRASTRUCTURE: runs the MGM-2 CUDA kernel SOURCE (pydcop_b200/csrc/mgm2_kernels.cuh) on the
// CPU, one "thread" after the other, so its logic can be compared with the oracle and the
// reference trajectories without a GPU.  Nothing in the product links or calls this.
//   g++ -O1 -std=c++17 -ffp-contract=off -shared -fPIC -o mgm2_host.so mgm2_host.cpp
// The descriptor is the C-ABI's fg_mgm2_desc_t with HOST pointers.
#include <stdint.h>

struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 blockIdx, blockDim, threadIdx;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

#include "../../pydcop_b200/csrc/mgm2_kernels.cuh"

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

static MgmSide side(const fg_mgm2_desc_t *d) {
  return MgmSide{d->classes, d->dev_dom_size, d->dev_var_id, d->dev_var_rank, d->dev_edge_var, d->dev_edge_class,
                 d->dev_var_ptr, d->dev_slot_edge, d->dev_nbr_ptr, d->dev_nbr_idx, nullptr};
}

template <typename T>
static void init_t(const fg_mgm2_desc_t *d) {
  launch(d->n_vars, 128, [&] {
    k_mgm2_init<T>(side(d), d->n_vars, (const T *)d->dev_tables, d->dev_init_value, d->mode_max, d->seed,
                   d->dev_value, (T *)d->dev_cost, d->dev_has_cost);
  });
}

// the five launches of mgm2.cu; each kernel boundary is a full pass over the "threads"
template <typename T>
static void cycle_t(const fg_mgm2_desc_t *d, uint32_t cyc) {
  const MgmSide g = side(d);
  const int n = d->n_vars;
  T *cost = (T *)d->dev_cost, *local = (T *)d->dev_local_cost, *gain = (T *)d->dev_gain;
  launch(n, 128, [&] {
    k_mgm2_value<T>(g, n, (const T *)d->dev_tables, d->dev_value, cost, d->dev_has_cost, local, gain,
                    d->dev_potential_value, d->dev_offerer, d->dev_partner, d->dev_committed, d->dev_answer,
                    d->dev_offer_off, (T *)d->dev_offer, d->mode_max, d->threshold, d->seed, cyc);
  });
  launch(n, 128, [&] {
    k_mgm2_answer<T>(g, n, (const T *)d->dev_tables, d->dev_value, local, gain, d->dev_potential_value,
                     d->dev_offerer, d->dev_partner, d->dev_committed, d->dev_answer, d->dev_answer_value,
                     (T *)d->dev_answer_gain, d->dev_offer_off, (const T *)d->dev_offer, d->mode_max, d->favor,
                     d->seed, cyc);
  });
  launch(n, 256, [&] {
    k_mgm2_commit<T>(n, d->dev_offerer, d->dev_answer, d->dev_answer_value, (const T *)d->dev_answer_gain, gain,
                     d->dev_potential_value, d->dev_committed);
  });
  launch(n, 256, [&] {
    k_mgm2_gain<T>(g, n, gain, d->dev_potential_value, d->dev_committed, d->dev_partner, d->dev_go, d->dev_value,
                   cost);
  });
  launch(n, 256, [&] {
    k_mgm2_go<T>(n, d->dev_committed, d->dev_partner, d->dev_go, gain, d->dev_potential_value, d->dev_value, cost);
  });
}

extern "C" {
void mgm2_host_init(const fg_mgm2_desc_t *d) {
  if (d->precision == FG_F64) init_t<double>(d);
  else init_t<float>(d);
}

void mgm2_host_cycle(const fg_mgm2_desc_t *d, uint32_t cycle) {
  if (d->precision == FG_F64) cycle_t<double>(d, cycle);
  else cycle_t<float>(d, cycle);
}
}  // extern "C"
