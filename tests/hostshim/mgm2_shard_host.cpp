// TEST INFRASTRUCTURE: runs the sharded MGM-2 kernel SOURCE (pydcop_b200/csrc/mgm2_shard_kernels.cuh) on the CPU,
// one "thread" after the other, so the sharded host logic can be compared with the single-process run without a GPU.
// Nothing in the product links or calls this.
//   g++ -O1 -std=c++17 -ffp-contract=off -shared -fPIC -o mgm2_shard_host.so mgm2_shard_host.cpp
// The descriptor and the shard plan are the C-ABI's fg_mgm2_desc_t / fg_mgm2_shard_plan_t with HOST pointers.  The
// sequence of launches is mgm2.cu's (mgm2_shard_init_t, mgm2_phase_t, mgm2_unpack_t).
#include <stdint.h>

struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 blockIdx, blockDim, threadIdx;
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

#include "../../pydcop_b200/csrc/mgm2_shard_kernels.cuh"

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

static MgmSide side(const fg_mgm2_desc_t *d) {
  return MgmSide{d->classes, d->dev_dom_size, d->dev_var_id, d->dev_var_rank, d->dev_edge_var, d->dev_edge_class,
                 d->dev_var_ptr, d->dev_slot_edge, d->dev_nbr_ptr, d->dev_nbr_idx, nullptr};
}

template <typename T>
static Mgm2State<T> state(const fg_mgm2_desc_t *d) {
  return Mgm2State<T>{d->dev_value, d->dev_offerer, d->dev_partner, d->dev_answer, d->dev_answer_value,
                      (T *)d->dev_answer_gain, (T *)d->dev_gain, d->dev_go, d->dev_offer_off, (T *)d->dev_offer};
}

template <typename T>
static void pack_t(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int x) {
  const fg_mgm2_xfer_t &q = p->x[x];
  const Mgm2List<T> l{q.n_send, q.dev_send_var, q.dev_send_off, (T *)q.dev_send_buf};
  const Mgm2Xlat xl{p->dev_send_peer, p->dev_owner_rank, p->dev_owner_local};
  launch(l.n, 256, [&] { k_mgm2x_pack<T>(x, l, state<T>(d), xl); });
}

template <typename T>
static void unpack_t(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int x) {
  const fg_mgm2_xfer_t &q = p->x[x];
  const Mgm2List<T> l{q.n_recv, q.dev_recv_var, q.dev_recv_off, (T *)q.dev_recv_buf};
  launch(l.n, 256, [&] { k_mgm2x_unpack<T>(x, l, state<T>(d)); });
}

template <typename T>
static void init_t(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p) {
  launch(d->n_vars, 128, [&] {
    k_mgm2s_init<T>(side(d), d->n_vars, p->dev_ghost, (const T *)d->dev_tables, d->dev_init_value, d->mode_max,
                    d->seed, d->dev_value, (T *)d->dev_cost, d->dev_has_cost);
  });
  pack_t<T>(d, p, MGM2X_VALUES);
}

template <typename T>
static void phase_t(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int x, uint32_t cyc) {
  const MgmSide g = side(d);
  const int n = d->n_vars;
  const uint8_t *gh = p->dev_ghost;
  T *cost = (T *)d->dev_cost, *local = (T *)d->dev_local_cost, *gain = (T *)d->dev_gain;
  switch (x) {
    case MGM2X_OFFERS:
      launch(n, 128, [&] {
        k_mgm2s_value<T>(g, n, gh, (const T *)d->dev_tables, d->dev_value, cost, d->dev_has_cost, local, gain,
                         d->dev_potential_value, d->dev_offerer, d->dev_partner, d->dev_committed, d->dev_answer,
                         d->dev_offer_off, (T *)d->dev_offer, d->mode_max, d->threshold, d->seed, cyc);
      });
      break;
    case MGM2X_ANSWERS:
      launch(n, 128, [&] {
        k_mgm2s_answer<T>(g, n, gh, (const T *)d->dev_tables, d->dev_value, local, gain, d->dev_potential_value,
                          d->dev_offerer, d->dev_partner, d->dev_committed, d->dev_answer, d->dev_answer_value,
                          (T *)d->dev_answer_gain, d->dev_offer_off, (const T *)d->dev_offer, d->mode_max, d->favor,
                          d->seed, cyc);
      });
      break;
    case MGM2X_GAINS:
      launch(n, 256, [&] {
        k_mgm2s_commit<T>(n, gh, d->dev_offerer, d->dev_answer, d->dev_answer_value, (const T *)d->dev_answer_gain,
                          gain, d->dev_potential_value, d->dev_committed);
      });
      break;
    case MGM2X_GO:
      launch(n, 256, [&] {
        k_mgm2s_gain<T>(g, n, gh, gain, d->dev_potential_value, d->dev_committed, d->dev_partner, d->dev_go,
                        d->dev_value, cost);
      });
      break;
    default:
      launch(n, 256, [&] {
        k_mgm2s_go<T>(n, gh, d->dev_committed, d->dev_partner, d->dev_go, gain, d->dev_potential_value, d->dev_value,
                      cost);
      });
      break;
  }
  pack_t<T>(d, p, x);
}

extern "C" {
void mgm2_shard_host_init(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p) {
  if (d->precision == FG_F64) init_t<double>(d, p);
  else init_t<float>(d, p);
}

// cycle: the 1-based round the phase kernels draw with
void mgm2_shard_host_phase(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int32_t x, uint32_t cycle) {
  if (d->precision == FG_F64) phase_t<double>(d, p, x, cycle);
  else phase_t<float>(d, p, x, cycle);
}

void mgm2_shard_host_unpack(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int32_t x) {
  if (d->precision == FG_F64) unpack_t<double>(d, p, x);
  else unpack_t<float>(d, p, x);
}
}  // extern "C"
