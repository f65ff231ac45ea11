// TEST INFRASTRUCTURE: runs the DBA CUDA kernel SOURCE (pydcop_b200/csrc/dba_kernels.cuh) on the CPU, one "thread"
// after the other, so its logic can be compared with the oracle and the reference trajectories without a GPU.
// Nothing in the product links or calls this.
//   g++ -O1 -std=c++17 -ffp-contract=off -shared -fPIC -o dba_host.so dba_host.cpp
// The descriptor is the C-ABI's fg_dba_desc_t with HOST pointers.
#include <stdint.h>

struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 blockIdx, blockDim, threadIdx;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

#include "../../pydcop_b200/csrc/dba_kernels.cuh"

template <typename F>
static void launch(int64_t n, int block, F body) {
  blockDim = Dim3{(unsigned)block, 1, 1};
  for (unsigned b = 0; b < (unsigned)((n + block - 1) / block); ++b)
    for (unsigned t = 0; t < (unsigned)block; ++t) {
      blockIdx = Dim3{b, 0, 0};
      threadIdx = Dim3{t, 0, 0};
      body();
    }
}

static MgmSide side(const fg_dba_desc_t *d) {
  return MgmSide{d->classes, d->dev_dom_size, d->dev_var_id, d->dev_var_rank, d->dev_edge_var, d->dev_edge_class,
                 d->dev_var_ptr, d->dev_slot_edge, d->dev_nbr_ptr, d->dev_nbr_idx, nullptr};
}

template <typename T>
static void bits_t(const fg_dba_desc_t *d) {
  launch(d->n_words, 256, [&] {
    k_dba_bits<T>(side(d), d->n_edges, (const T *)d->dev_tables, d->dev_bit_off, d->n_words, (T)d->infinity,
                  d->dev_bits);
  });
}

extern "C" {
// fg_dba_init's two launches
void dba_host_init(const fg_dba_desc_t *d) {
  if (d->n_edges) {
    if (d->precision == FG_F64) bits_t<double>(d);
    else bits_t<float>(d);
  }
  launch(d->n_vars > 0 ? d->n_vars : 1, 128, [&] {
    k_dba_init(side(d), d->n_vars, d->seed, d->n_live, d->dev_value[0], d->dev_has_cost, d->dev_counter_own,
               d->dev_finish_phase, d->dev_weight, d->dev_status, d->dev_unresolved);
  });
}

// the two launches of round done + 1 (dba.cu); each kernel boundary is a full pass over the "threads"
void dba_host_cycle(const fg_dba_desc_t *d, int64_t done) {
  const MgmSide g = side(d);
  const int n = d->n_vars;
  const int32_t k = (int32_t)(done + 1);
  int32_t *vin = d->dev_value[done & 1], *vout = d->dev_value[(done + 1) & 1];
  launch(n, 128, [&] {
    auto ok = dba_eval_dmax(d->classes, d->n_classes) <= 32 ? k_dba_ok<32> : k_dba_ok<FG_MAX_DOM>;
    ok(g, n, d->dev_bits, d->dev_bit_off, d->dev_weight, vin, d->infinity, d->seed, k, d->dev_finish_phase,
       d->dev_status, d->dev_counter_own, d->dev_eval, d->dev_improve, d->dev_counter, d->dev_new_value,
       d->dev_can_move, d->dev_qlm, d->dev_consistent, d->dev_violated, d->dev_cost, d->dev_has_cost,
       d->dev_unresolved);
  });
  launch(n, 256, [&] {
    k_dba_improve(g, n, d->dev_eval, d->dev_improve, d->dev_counter, d->dev_new_value, d->max_distance, k,
                  d->dev_finish_phase, d->dev_status, d->dev_violated, vin, vout, d->dev_counter_own, d->dev_can_move,
                  d->dev_qlm, d->dev_consistent, d->dev_weight, d->dev_cost);
  });
}
}  // extern "C"
