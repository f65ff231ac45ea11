// MGM for all variables at once (SURVEY.md §8f.4): C-ABI entry points fg_mgm_* and their kernels.
// Separate translation unit: the MaxSum / DSA code in engine.cu is not recompiled differently.
//
// One thread per variable, any arity / domain sizes (the generic shape of k_dsa_step_generic).
// Floating-point operand order follows pydcop/algorithms/mgm.py so that the f64 build equals the
// reference's Python floats and the f32 build equals the f32 oracle (oracle/dcop_oracle_impl.h):
//   relation value of x  = ((f1(x) + f2(x)) + f3(x)) ...   in node.constraints order (mgm.py:443)
//   evaluation           = best + own cost(CURRENT value) + neighbours' costs       (:446-452)
//   gain                 = current_cost - evaluation                                (:381)
#include "handle.cuh"
#include "mgm_kernels.cuh"
#include "mgm_fast_kernels.cuh"
#include "mgm_cached_kernels.cuh"

struct fg_mgm : fg_handle_base {
  fg_mgm_desc_t d;
};

extern "C" int fg_mgm_create(const fg_mgm_desc_t *desc, fg_mgm_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_mgm *h = *out;
  if (desc->n_vars > 0 && (!desc->dev_nbr_ptr || !desc->dev_value || !desc->dev_cost || !desc->dev_has_cost ||
                           !desc->dev_gain || !desc->dev_new_value || !desc->dev_var_rank || !desc->dev_var_id)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_mgm_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_unary), FG_FIELD(d, dev_unary_off),
                             FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id), FG_FIELD(d, dev_var_rank),
                             FG_FIELD(d, dev_edge_var), FG_FIELD(d, dev_edge_class), FG_FIELD(d, dev_var_ptr),
                             FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_nbr_ptr), FG_FIELD(d, dev_nbr_idx),
                             FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_value), FG_FIELD(d, dev_cost),
                             FG_FIELD(d, dev_has_cost), FG_FIELD(d, dev_gain), FG_FIELD(d, dev_new_value),
                             FG_FIELD(d, dev_tables_or), FG_FIELD(d, dev_slot_nbr), FG_FIELD(d, dev_slot_tab),
                             FG_FIELD(d, dev_row_cache), FG_FIELD(d, dev_slot_last), FG_FIELD(d, dev_var_seed)});
  if (rc != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_mgm_destroy(fg_mgm_t h) { return fg_close(h); }

extern "C" const char *fg_mgm_last_error(fg_mgm_t h) { return fg_last_error(h); }

extern "C" int fg_mgm_init(fg_mgm_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  const fg_mgm_desc_t &d = h->d;
  cudaStream_t st = (cudaStream_t)stream;
  fg_launcher launch(h, st);
  if (d.n_vars) mgm_init(d, h->dev_classes, launch);
  if (d.dev_slot_last && d.n_edges)   // active-row array: no row has been read yet
    CUDA_TRY(h, cudaMemsetAsync(d.dev_slot_last, 0xFF, (size_t)d.n_edges, st));
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

template <typename T, int D>
static void mgm_gain_cached_launch(fg_mgm *h, cudaStream_t st) {
  const fg_mgm_desc_t &d = h->d;
  using Cfg = MgmCachedCfg<T, D>;
  static_assert(sizeof(T) * Cfg::CH * D + 2 * Cfg::CH + 4 * (Cfg::NV + 1) + 16 <= 48 * 1024, "static shared memory");
  k_mgm_gain_cached<T, D><<<(unsigned)((d.n_vars + Cfg::NV - 1) / Cfg::NV), Cfg::THREADS, 0, st>>>(
      mgm_side(d, h->dev_classes), d.n_vars, d.dev_slot_nbr, d.dev_slot_tab, (const T *)d.dev_tables_or,
      (const T *)d.dev_unary, d.dev_value, (T *)d.dev_cost, d.dev_has_cost, (T *)d.dev_gain, d.dev_new_value,
      d.mode_max, d.seed, (uint32_t)(h->cycle + 1), (T *)d.dev_row_cache, d.dev_slot_last);
  ++h->launches;
}

// the active-row value phase (a block per Cfg::NV variables, so not a launch of the shared sequence) when the
// descriptor carries the active-row arrays over oriented tables, else false
template <typename T>
static bool mgm_gain_cached(fg_mgm *h, cudaStream_t st) {
  const fg_mgm_desc_t &d = h->d;
  if (!d.dev_row_cache || !d.dev_slot_last || !mgm_fast_shape(d)) return false;
  switch (d.fast_dom) {
#define FG_MGM_CC(n) case n: mgm_gain_cached_launch<T, n>(h, st); return true;
    FG_MGM_CC(4) FG_MGM_CC(8) FG_MGM_CC(10) FG_MGM_CC(16) FG_MGM_CC(20)
#undef FG_MGM_CC
  }
  return false;
}

template <typename T>
static int mgm_cycle_t(fg_mgm *h, cudaStream_t st) {
  const fg_mgm_desc_t &d = h->d;
  fg_launcher launch(h, st);
  if (d.n_vars) {
    if (!mgm_gain_cached<T>(h, st)) mgm_gain<T>(d, h->dev_classes, h->cycle, launch);
    mgm_decide<T>(d, h->dev_classes, launch);
  }
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return fg_trace_cycle(h, d.dev_value, st);
}

extern "C" int fg_mgm_step(fg_mgm_t h, int32_t n_cycles, void *stream) {
  return fg_step(h, n_cycles, stream, mgm_cycle_t<float>, mgm_cycle_t<double>);
}

extern "C" int fg_mgm_current(fg_mgm_t h, int64_t *cycle, int32_t *finished) { return fg_current(h, cycle, finished); }

extern "C" int64_t fg_mgm_launch_count(fg_mgm_t h) { return fg_launch_count(h); }

extern "C" int fg_mgm_set_trace(fg_mgm_t h, fg_trace_t tr) { return fg_set_trace(h, tr); }
