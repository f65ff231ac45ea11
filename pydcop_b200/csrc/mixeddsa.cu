// MixedDSA for all variables at once: C-ABI entry points fg_mixeddsa_* and their kernels (csrc/mixeddsa_kernels.cuh,
// which states the floating-point operand order).  Its own translation unit, so the other families' code is compiled
// exactly as before.
#include "handle.cuh"
#include "philox.cuh"

// k_dsa_con_opt for the constraint optima; with internal linkage, as mgm_kernels.cuh in mixeddsa_kernels.cuh, so the
// DSA kernels engine.cu defines are not defined twice (the includes above must stay above the namespace)
namespace {
#include "dsa_generic.cuh"
}
#include "mixeddsa_kernels.cuh"

struct fg_mixeddsa : fg_handle_base {
  fg_mixeddsa_desc_t d;
  int dmax = FG_MAX_DOM;  // mixeddsa_dmax of the class table: which k_mixeddsa_step instance runs
};

// stop_cycle as fg_dsa_*: a run ends after stop_cycle rounds (dsa.py:352)
static bool mixeddsa_finished(const fg_mixeddsa *h) { return h->d.stop_cycle && h->cycle >= h->d.stop_cycle; }

extern "C" int fg_mixeddsa_create(const fg_mixeddsa_desc_t *desc, fg_mixeddsa_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_mixeddsa *h = *out;
  if (desc->variant < FG_DSA_A || desc->variant > FG_DSA_C) {
    snprintf(h->err, sizeof(h->err), "variant %d is not one of A (0), B (1), C (2)", desc->variant);
    return FG_ERR_ARG;
  }
  if (desc->mode_max != 0 && desc->mode_max != 1) {
    snprintf(h->err, sizeof(h->err), "mode_max %d is not 0 (min) or 1 (max)", desc->mode_max);
    return FG_ERR_ARG;
  }
  if (desc->stop_cycle < 0) {
    snprintf(h->err, sizeof(h->err), "negative stop_cycle %d", desc->stop_cycle);
    return FG_ERR_ARG;
  }
  if (desc->n_vars > 0 &&
      (!desc->dev_unary || !desc->dev_unary_off || !desc->dev_dom_size || !desc->dev_var_id || !desc->dev_var_ptr ||
       !desc->dev_soft_end || !desc->dev_nbr_ptr || !desc->dev_nbr_idx || !desc->dev_value[0] ||
       !desc->dev_value[1] || !desc->dev_cost || !desc->dev_has_cost || !desc->dev_h_best || !desc->dev_branch)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_edges > 0 &&
      (!desc->dev_tables || !desc->dev_edge_var || !desc->dev_edge_class || !desc->dev_slot_edge)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_factors > 0 && !desc->dev_con_opt) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  h->dmax = mixeddsa_dmax(h->classes.data(), (int)h->classes.size());
  rc = fg_check_psets(h, [](const fg_mixeddsa_pset_t &p) -> const char * {
    if (p.variant < FG_DSA_A || p.variant > FG_DSA_C) return "variant is not an FG_DSA_* value";
    if (!fg_unit_interval(p.proba_hard)) return "proba_hard is not in [0, 1]";
    return fg_unit_interval(p.proba_soft) ? nullptr : "proba_soft is not in [0, 1]";
  });
  if (rc != FG_OK) return rc;
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_mixeddsa_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_unary), FG_FIELD(d, dev_unary_off),
                             FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id), FG_FIELD(d, dev_edge_var),
                             FG_FIELD(d, dev_edge_class), FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_slot_edge),
                             FG_FIELD(d, dev_soft_end), FG_FIELD(d, dev_nbr_ptr), FG_FIELD(d, dev_nbr_idx),
                             FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_con_opt), FG_FIELD(d, dev_value[0]),
                             FG_FIELD(d, dev_value[1]), FG_FIELD(d, dev_cost), FG_FIELD(d, dev_has_cost),
                             FG_FIELD(d, dev_h_best), FG_FIELD(d, dev_branch), FG_FIELD(d, dev_var_seed),
                             FG_FIELD(d, dev_var_pset)});
  if (rc != FG_OK || (rc = fg_upload_psets(h)) != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_mixeddsa_destroy(fg_mixeddsa_t h) { return fg_close(h); }

extern "C" const char *fg_mixeddsa_last_error(fg_mixeddsa_t h) { return fg_last_error(h); }

extern "C" int fg_mixeddsa_init(fg_mixeddsa_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  fg_launcher launch(h, (cudaStream_t)stream);
  if (h->d.precision == FG_F64) mixeddsa_init<double>(h->d, h->dev_classes, launch);
  else mixeddsa_init<float>(h->d, h->dev_classes, launch);
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

template <typename T>
static int mixeddsa_round_t(fg_mixeddsa *h, cudaStream_t st) {
  fg_launcher launch(h, st);
  if (h->d.n_vars) mixeddsa_cycle<T>(h->d, h->dev_classes, h->dmax, h->cycle, launch);
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return fg_trace_cycle(h, h->d.dev_value[h->cycle % 2], st);
}

extern "C" int fg_mixeddsa_step(fg_mixeddsa_t h, int32_t n_cycles, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n_cycles; ++i) {
    if (mixeddsa_finished(h)) break;
    int rc = h->d.precision == FG_F64 ? mixeddsa_round_t<double>(h, st) : mixeddsa_round_t<float>(h, st);
    if (rc != FG_OK) return rc;
  }
  return FG_OK;
}

extern "C" int fg_mixeddsa_current(fg_mixeddsa_t h, int64_t *cycle, int32_t *finished) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (cycle) *cycle = h->cycle;
  if (finished) *finished = mixeddsa_finished(h) ? 1 : 0;
  return FG_OK;
}

extern "C" int64_t fg_mixeddsa_launch_count(fg_mixeddsa_t h) { return fg_launch_count(h); }

extern "C" int fg_mixeddsa_set_trace(fg_mixeddsa_t h, fg_trace_t tr) { return fg_set_trace(h, tr); }
