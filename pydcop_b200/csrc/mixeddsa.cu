// MixedDSA for all variables at once: C-ABI entry points fg_mixeddsa_* and their kernels (csrc/mixeddsa_kernels.cuh,
// which states the floating-point operand order).  Its own translation unit, so the other families' code is compiled
// exactly as before.
#include <limits>

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

static inline unsigned mixeddsa_blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

static MgmSide mixeddsa_side(const fg_mixeddsa *h) {
  const fg_mixeddsa_desc_t &d = h->d;
  return MgmSide{h->dev_classes, d.dev_dom_size, d.dev_var_id, nullptr, d.dev_edge_var, d.dev_edge_class,
                 d.dev_var_ptr, d.dev_slot_edge, d.dev_nbr_ptr, d.dev_nbr_idx, d.dev_unary_off,
                 d.dev_var_seed};
}

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
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_mixeddsa_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_unary), FG_FIELD(d, dev_unary_off),
                             FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id), FG_FIELD(d, dev_edge_var),
                             FG_FIELD(d, dev_edge_class), FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_slot_edge),
                             FG_FIELD(d, dev_soft_end), FG_FIELD(d, dev_nbr_ptr), FG_FIELD(d, dev_nbr_idx),
                             FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_con_opt), FG_FIELD(d, dev_value[0]),
                             FG_FIELD(d, dev_value[1]), FG_FIELD(d, dev_cost), FG_FIELD(d, dev_has_cost),
                             FG_FIELD(d, dev_h_best), FG_FIELD(d, dev_branch), FG_FIELD(d, dev_var_seed)});
  if (rc != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_mixeddsa_destroy(fg_mixeddsa_t h) { return fg_close(h); }

extern "C" const char *fg_mixeddsa_last_error(fg_mixeddsa_t h) { return fg_last_error(h); }

template <typename T>
static void mixeddsa_con_opt_t(fg_mixeddsa *h, cudaStream_t st) {
  for (const fg_class_t &c : h->classes) {
    if (!c.n_factors) continue;
    k_dsa_con_opt<T><<<mixeddsa_blocks(c.n_factors, 128), 128, 0, st>>>(c, (const T *)h->d.dev_tables,
                                                                         (T *)h->d.dev_con_opt, h->d.mode_max);
    ++h->launches;
  }
}

extern "C" int fg_mixeddsa_init(fg_mixeddsa_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  const fg_mixeddsa_desc_t &d = h->d;
  cudaStream_t st = (cudaStream_t)stream;
  if (d.precision == FG_F64) mixeddsa_con_opt_t<double>(h, st);
  else mixeddsa_con_opt_t<float>(h, st);
  if (d.n_vars) {
    k_mixeddsa_init<<<mixeddsa_blocks(d.n_vars, 128), 128, 0, st>>>(mixeddsa_side(h), d.n_vars, d.dev_init_value,
                                                                    d.seed, d.dev_value[0], d.dev_has_cost);
    ++h->launches;
  }
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

template <typename T>
static int mixeddsa_round_t(fg_mixeddsa *h, cudaStream_t st) {
  const fg_mixeddsa_desc_t &d = h->d;
  if (d.n_vars) {
    const int n = d.n_vars;
    int32_t *vin = d.dev_value[h->cycle & 1], *vout = d.dev_value[(h->cycle + 1) & 1];
    auto step = h->dmax <= 32 ? k_mixeddsa_step<T, 32> : k_mixeddsa_step<T, FG_MAX_DOM>;
    step<<<mixeddsa_blocks(n, 128), 128, 0, st>>>(
        mixeddsa_side(h), n, (const T *)d.dev_tables, (const T *)d.dev_unary, d.dev_soft_end,
        (const T *)d.dev_con_opt, vin, vout, (T *)d.dev_cost, d.dev_has_cost, d.dev_h_best, d.dev_branch, d.mode_max,
        d.variant, d.proba_hard, d.proba_soft, std::numeric_limits<T>::infinity(), d.seed, (uint32_t)(h->cycle + 1));
    ++h->launches;
  }
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return FG_OK;
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
