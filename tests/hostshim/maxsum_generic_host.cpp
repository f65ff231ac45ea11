// TEST INFRASTRUCTURE: runs the generic MaxSum CUDA kernel SOURCE (pydcop_b200/csrc/maxsum_generic.cuh,
// unmodified) on the CPU, one "thread" after the other, with the launch order of
// maxsum_init_t / maxsum_compute_t in engine.cu (generic kernels only, as with PYDCOP_B200_NO_FAST=1).
// Lets the kernels be compared with the oracle on shapes the GPU tests do not reach.  Nothing in the
// product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/maxsum_generic.cuh"

template <typename F>
static void launch(int64_t n, F body) {
  blockDim = Dim3{128, 1, 1};
  for (int64_t b = 0; b < (n + 127) / 128; ++b)
    for (unsigned t = 0; t < 128; ++t) {
      blockIdx = Dim3{(unsigned)b, 0, 0};
      threadIdx = Dim3{t, 0, 0};
      body();
    }
}

extern "C" {
struct ms_host {
  const fg_class_t *classes;
  const fg_varclass_t *varclasses;
  int32_t n_classes, n_varclasses, n_vars, n_edges, precision;
  int64_t n_msg_r, n_msg_q;
  const void *tables, *unary;
  const int32_t *dom_size, *var_ptr, *slot_edge, *slot_var, *init_value;
  const int64_t *unary_off, *var_qbase, *slot_roff, *edge_qoff;
  void *q[2], *r[2];
  uint8_t *q_valid, *r_valid, *q_cnt, *r_cnt, *q_sent, *r_sent;
  int32_t *value;
  void *value_cost;
  int32_t mode_max, damp_vars, damp_factors, start_messages;
  double damping, stability;
};
}

template <typename T>
static void init_t(const ms_host *h) {
  for (int b = 0; b < 2; ++b) {
    memset(h->q[b], 0, (size_t)h->n_msg_q * sizeof(T));
    memset(h->r[b], 0, (size_t)h->n_msg_r * sizeof(T));
  }
  uint8_t *bytes[] = {h->q_valid, h->r_valid, h->q_cnt, h->r_cnt, h->q_sent, h->r_sent};
  for (uint8_t *p : bytes)
    if (p && h->n_edges) memset(p, 0, (size_t)h->n_edges);
  VarSide g{h->dom_size, h->unary_off, h->var_ptr, h->var_qbase, h->slot_roff, h->slot_edge, h->slot_var};
  launch(h->n_vars, [&] {
    k_v2f_start<T>(g, h->n_vars, (const T *)h->unary, h->init_value, (T *)h->q[0], h->q_valid, h->q_sent, h->value,
                   (T *)h->value_cost, h->mode_max, h->start_messages);
  });
  for (int ci = 0; ci < h->n_classes; ++ci) {
    const fg_class_t &c = h->classes[ci];
    bool posts = (c.arity == 1 && h->start_messages <= FG_START_LEAFS_VARS) || h->start_messages == FG_START_ALL;
    if (!posts || c.n_factors == 0 || (c.flags & FG_CLASS_GHOST)) continue;
    launch((int64_t)c.n_factors * c.arity, [&] {
      k_f2v_start<T>(c, (const T *)h->tables, (T *)h->r[0], h->r_valid, h->r_sent, h->mode_max);
    });
  }
}

template <typename T, int FIRST>
static void cycle_t(const ms_host *h, int cur) {
  const int nxt = cur ^ 1;
  MaxSumParams p{h->mode_max, h->damp_vars, h->damp_factors, h->damping, 1.0 - h->damping, h->stability};
  const T *q_cur = (const T *)h->q[cur], *r_cur = (const T *)h->r[cur];
  T *q_next = (T *)h->q[nxt], *r_next = (T *)h->r[nxt];
  for (int ci = 0; ci < h->n_classes; ++ci) {
    const fg_class_t &c = h->classes[ci];
    if (c.n_factors == 0 || (c.flags & FG_CLASS_GHOST)) continue;
    launch((int64_t)c.n_factors * c.arity, [&] {
      k_f2v_generic<T, FIRST>(c, (const T *)h->tables, q_cur, r_cur, r_next, h->edge_qoff, h->q_valid, h->r_cnt,
                              h->r_sent, p);
    });
  }
  VarSide g{h->dom_size, h->unary_off, h->var_ptr, h->var_qbase, h->slot_roff, h->slot_edge, h->slot_var};
  for (int vi = 0; vi < h->n_varclasses; ++vi) {
    const fg_varclass_t &vc = h->varclasses[vi];
    if (vc.n_slots == 0 || (vc.flags & FG_CLASS_GHOST)) continue;
    launch(vc.n_slots, [&] {
      k_v2f_generic<T, FIRST>(g, vc.first_slot, vc.n_slots, (const T *)h->unary, r_cur, q_cur, q_next, h->r_valid,
                              h->q_cnt, h->q_sent, h->value, (T *)h->value_cost, p);
    });
  }
  if (FIRST && h->n_edges) {
    memset(h->q_valid, 1, (size_t)h->n_edges);
    memset(h->r_valid, 1, (size_t)h->n_edges);
  }
}

extern "C" void ms_host_init(const ms_host *h) {
  if (h->precision == FG_F64) init_t<double>(h); else init_t<float>(h);
}

extern "C" void ms_host_cycle(const ms_host *h, int cur, int first) {
  if (h->precision == FG_F64) { if (first) cycle_t<double, 1>(h, cur); else cycle_t<double, 0>(h, cur); }
  else { if (first) cycle_t<float, 1>(h, cur); else cycle_t<float, 0>(h, cur); }
}
