// MGM-2 for all variables at once: C-ABI entry points fg_mgm2_* and their kernels
// (csrc/mgm2_kernels.cuh).  Its own translation unit, so the MaxSum / DSA / MGM code in engine.cu
// and mgm.cu is compiled exactly as before.
//
// Floating-point operand order follows pydcop/algorithms/mgm2.py so that the f64 build equals the
// reference's Python floats and the f32 build the f32 oracle (tests/_mgm2_oracle.py):
//   cost of an assignment = ((0 + c1) + c2) + ...    in node.constraints order (assignment_cost)
//   offer gain            = current_cost - cost                                   (:553)
//   global gain           = (current_cost - cost over the other constraints) + offer gain (:593)
//   cost after a move     = current_cost - potential_gain                         (:941, :986)
#include "handle.cuh"
#include "mgm2_kernels.cuh"

struct fg_mgm2 : fg_handle_base {
  fg_mgm2_desc_t d;
};

static inline unsigned mgm2_blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

static MgmSide mgm2_side(const fg_mgm2 *h) {
  const fg_mgm2_desc_t &d = h->d;
  return MgmSide{h->dev_classes, d.dev_dom_size, d.dev_var_id, d.dev_var_rank, d.dev_edge_var, d.dev_edge_class,
                 d.dev_var_ptr, d.dev_slot_edge, d.dev_nbr_ptr, d.dev_nbr_idx, nullptr};
}

extern "C" int fg_mgm2_create(const fg_mgm2_desc_t *desc, fg_mgm2_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_mgm2 *h = *out;
  if (desc->favor < FG_MGM2_FAVOR_UNILATERAL || desc->favor > FG_MGM2_FAVOR_COORDINATED) {
    snprintf(h->err, sizeof(h->err), "favor %d is not one of unilateral (0), no (1), coordinated (2)", desc->favor);
    return FG_ERR_ARG;
  }
  if (!(desc->threshold >= 0.0 && desc->threshold <= 1.0)) {
    snprintf(h->err, sizeof(h->err), "threshold %g is not in [0, 1]", desc->threshold);
    return FG_ERR_ARG;
  }
  if (desc->stop_cycle < 0) {
    snprintf(h->err, sizeof(h->err), "negative stop_cycle %d", desc->stop_cycle);
    return FG_ERR_ARG;
  }
  if (desc->n_vars > 0 &&
      (!desc->dev_tables || !desc->dev_dom_size || !desc->dev_var_id || !desc->dev_var_rank || !desc->dev_var_ptr ||
       !desc->dev_nbr_ptr || !desc->dev_nbr_idx || !desc->dev_value || !desc->dev_cost || !desc->dev_has_cost ||
       !desc->dev_gain || !desc->dev_potential_value || !desc->dev_local_cost || !desc->dev_offerer ||
       !desc->dev_partner || !desc->dev_committed || !desc->dev_go || !desc->dev_answer || !desc->dev_answer_value ||
       !desc->dev_answer_gain || !desc->dev_offer_off || !desc->dev_offer)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_edges > 0 && (!desc->dev_edge_var || !desc->dev_edge_class || !desc->dev_slot_edge)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_mgm2_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id),
                             FG_FIELD(d, dev_var_rank), FG_FIELD(d, dev_edge_var), FG_FIELD(d, dev_edge_class),
                             FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_nbr_ptr),
                             FG_FIELD(d, dev_nbr_idx), FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_value),
                             FG_FIELD(d, dev_cost), FG_FIELD(d, dev_has_cost), FG_FIELD(d, dev_gain),
                             FG_FIELD(d, dev_potential_value), FG_FIELD(d, dev_local_cost), FG_FIELD(d, dev_offerer),
                             FG_FIELD(d, dev_partner), FG_FIELD(d, dev_committed), FG_FIELD(d, dev_go),
                             FG_FIELD(d, dev_answer), FG_FIELD(d, dev_answer_value), FG_FIELD(d, dev_answer_gain),
                             FG_FIELD(d, dev_offer_off), FG_FIELD(d, dev_offer)});
  if (rc != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_mgm2_destroy(fg_mgm2_t h) { return fg_close(h); }

extern "C" const char *fg_mgm2_last_error(fg_mgm2_t h) { return fg_last_error(h); }

template <typename T>
static void mgm2_init_t(fg_mgm2 *h, cudaStream_t st) {
  const fg_mgm2_desc_t &d = h->d;
  k_mgm2_init<T><<<mgm2_blocks(d.n_vars, 128), 128, 0, st>>>(mgm2_side(h), d.n_vars, (const T *)d.dev_tables,
                                                             d.dev_init_value, d.mode_max, d.seed, d.dev_value,
                                                             (T *)d.dev_cost, d.dev_has_cost);
}

extern "C" int fg_mgm2_init(fg_mgm2_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  const fg_mgm2_desc_t &d = h->d;
  cudaStream_t st = (cudaStream_t)stream;
  if (d.n_vars) {
    if (d.precision == FG_F64) mgm2_init_t<double>(h, st);
    else mgm2_init_t<float>(h, st);
    ++h->launches;
  }
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

template <typename T>
static int mgm2_cycle_t(fg_mgm2 *h, cudaStream_t st) {
  const fg_mgm2_desc_t &d = h->d;
  if (d.n_vars) {
    const MgmSide g = mgm2_side(h);
    const uint32_t cyc = (uint32_t)(h->cycle + 1);
    const int n = d.n_vars;
    T *cost = (T *)d.dev_cost, *local = (T *)d.dev_local_cost, *gain = (T *)d.dev_gain;
    k_mgm2_value<T><<<mgm2_blocks(n, 128), 128, 0, st>>>(
        g, n, (const T *)d.dev_tables, d.dev_value, cost, d.dev_has_cost, local, gain, d.dev_potential_value,
        d.dev_offerer, d.dev_partner, d.dev_committed, d.dev_answer, d.dev_offer_off, (T *)d.dev_offer, d.mode_max,
        d.threshold, d.seed, cyc);
    k_mgm2_answer<T><<<mgm2_blocks(n, 128), 128, 0, st>>>(
        g, n, (const T *)d.dev_tables, d.dev_value, local, gain, d.dev_potential_value, d.dev_offerer, d.dev_partner,
        d.dev_committed, d.dev_answer, d.dev_answer_value, (T *)d.dev_answer_gain, d.dev_offer_off,
        (const T *)d.dev_offer, d.mode_max, d.favor, d.seed, cyc);
    k_mgm2_commit<T><<<mgm2_blocks(n, 256), 256, 0, st>>>(n, d.dev_offerer, d.dev_answer, d.dev_answer_value,
                                                          (const T *)d.dev_answer_gain, gain, d.dev_potential_value,
                                                          d.dev_committed);
    k_mgm2_gain<T><<<mgm2_blocks(n, 256), 256, 0, st>>>(g, n, gain, d.dev_potential_value, d.dev_committed,
                                                        d.dev_partner, d.dev_go, d.dev_value, cost);
    k_mgm2_go<T><<<mgm2_blocks(n, 256), 256, 0, st>>>(n, d.dev_committed, d.dev_partner, d.dev_go, gain,
                                                      d.dev_potential_value, d.dev_value, cost);
    h->launches += 5;
  }
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return FG_OK;
}

extern "C" int fg_mgm2_step(fg_mgm2_t h, int32_t n_cycles, void *stream) {
  return fg_step(h, n_cycles, stream, mgm2_cycle_t<float>, mgm2_cycle_t<double>);
}

extern "C" int fg_mgm2_current(fg_mgm2_t h, int64_t *cycle, int32_t *finished) { return fg_current(h, cycle, finished); }

extern "C" int64_t fg_mgm2_launch_count(fg_mgm2_t h) { return fg_launch_count(h); }
