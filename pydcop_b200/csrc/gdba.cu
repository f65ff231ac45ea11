// GDBA for all variables at once: C-ABI entry points fg_gdba_* and their kernels
// (csrc/gdba_kernels.cuh, which states the floating-point operand order).  Its own translation unit,
// so the MaxSum / DSA / MGM / MGM-2 code is compiled exactly as before.
#include "handle.cuh"
#include "gdba_kernels.cuh"

struct fg_gdba : fg_handle_base {
  fg_gdba_desc_t d;
};

extern "C" int fg_gdba_create(const fg_gdba_desc_t *desc, fg_gdba_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_gdba *h = *out;
  if (desc->modifier != FG_GDBA_MODIFIER_A && desc->modifier != FG_GDBA_MODIFIER_M) {
    snprintf(h->err, sizeof(h->err), "modifier %d is not one of A (0), M (1)", desc->modifier);
    return FG_ERR_ARG;
  }
  if (desc->violation < FG_GDBA_VIOLATION_NZ || desc->violation > FG_GDBA_VIOLATION_MX) {
    snprintf(h->err, sizeof(h->err), "violation %d is not one of NZ (0), NM (1), MX (2)", desc->violation);
    return FG_ERR_ARG;
  }
  if (desc->increase_mode < FG_GDBA_INCREASE_E || desc->increase_mode > FG_GDBA_INCREASE_T) {
    snprintf(h->err, sizeof(h->err), "increase_mode %d is not one of E (0), R (1), C (2), T (3)",
             desc->increase_mode);
    return FG_ERR_ARG;
  }
  if (desc->stop_cycle < 0) {
    snprintf(h->err, sizeof(h->err), "negative stop_cycle %d", desc->stop_cycle);
    return FG_ERR_ARG;
  }
  if (desc->mod_size < 0 || (desc->increase_mode == FG_GDBA_INCREASE_T && desc->mod_size < desc->n_edges)) {
    snprintf(h->err, sizeof(h->err), "mod_size %lld too small", (long long)desc->mod_size);
    return FG_ERR_ARG;
  }
  if (desc->n_vars > 0 &&
      (!desc->dev_tables || !desc->dev_unary || !desc->dev_unary_off || !desc->dev_dom_size || !desc->dev_var_id ||
       !desc->dev_var_rank || !desc->dev_var_ptr || !desc->dev_nbr_ptr || !desc->dev_nbr_idx || !desc->dev_value[0] ||
       !desc->dev_value[1] || !desc->dev_cost || !desc->dev_has_cost || !desc->dev_improve ||
       !desc->dev_new_value || !desc->dev_breakout)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_edges > 0 &&
      (!desc->dev_edge_var || !desc->dev_edge_class || !desc->dev_slot_edge || !desc->dev_violated ||
       !desc->dev_mod || (desc->increase_mode != FG_GDBA_INCREASE_T && !desc->dev_mod_off) ||
       (desc->violation != FG_GDBA_VIOLATION_NZ && !desc->dev_viol_ref))) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_gdba_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_unary), FG_FIELD(d, dev_unary_off),
                             FG_FIELD(d, dev_viol_ref), FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id),
                             FG_FIELD(d, dev_var_rank), FG_FIELD(d, dev_edge_var), FG_FIELD(d, dev_edge_class),
                             FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_nbr_ptr),
                             FG_FIELD(d, dev_nbr_idx), FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_value[0]),
                             FG_FIELD(d, dev_value[1]), FG_FIELD(d, dev_cost), FG_FIELD(d, dev_has_cost),
                             FG_FIELD(d, dev_improve), FG_FIELD(d, dev_new_value), FG_FIELD(d, dev_violated),
                             FG_FIELD(d, dev_breakout), FG_FIELD(d, dev_mod), FG_FIELD(d, dev_mod_off),
                             FG_FIELD(d, dev_var_seed)});
  if (rc != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_gdba_destroy(fg_gdba_t h) { return fg_close(h); }

extern "C" const char *fg_gdba_last_error(fg_gdba_t h) { return fg_last_error(h); }

extern "C" int fg_gdba_init(fg_gdba_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  fg_launcher launch(h, (cudaStream_t)stream);
  gdba_init(h->d, h->dev_classes, launch);
  if (int rc = launch.status()) return rc;
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

template <typename T>
static int gdba_cycle_t(fg_gdba *h, cudaStream_t st) {
  fg_launcher launch(h, st);
  if (h->d.n_vars) gdba_cycle<T>(h->d, h->dev_classes, h->cycle, launch);
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return FG_OK;
}

extern "C" int fg_gdba_step(fg_gdba_t h, int32_t n_cycles, void *stream) {
  return fg_step(h, n_cycles, stream, gdba_cycle_t<float>, gdba_cycle_t<double>);
}

extern "C" int fg_gdba_current(fg_gdba_t h, int64_t *cycle, int32_t *finished) { return fg_current(h, cycle, finished); }

extern "C" int64_t fg_gdba_launch_count(fg_gdba_t h) { return fg_launch_count(h); }
