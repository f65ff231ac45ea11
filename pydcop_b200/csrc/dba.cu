// DBA for all variables at once: C-ABI entry points fg_dba_* and their kernels (csrc/dba_kernels.cuh).  Its own
// translation unit, so the other families' code is compiled exactly as before.
#include "handle.cuh"
#include "dba_kernels.cuh"

struct fg_dba : fg_handle_base {
  fg_dba_desc_t d;
  cudaStream_t last_stream = nullptr;  // where the last init / step enqueued its work
  bool started = false;                // fg_dba_init ran: dev_status is meaningful
  bool ended = false;                  // fg_dba_current saw every variable with neighbours finished
  int32_t end_round = FG_DBA_LIVE;
  int eval_dmax = FG_MAX_DOM;          // dba_eval_dmax of the class table: which k_dba_ok instance runs
};

// stop_cycle as fg_gdba_*: rounds stop once cycle + 1 >= stop_cycle
static bool dba_finished(const fg_dba *h) {
  return h->ended || (h->d.stop_cycle && h->cycle + 1 >= h->d.stop_cycle);
}

extern "C" int fg_dba_create(const fg_dba_desc_t *desc, fg_dba_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_dba *h = *out;
  if (desc->max_distance < 0) {
    snprintf(h->err, sizeof(h->err), "negative max_distance %d", desc->max_distance);
    return FG_ERR_ARG;
  }
  if (desc->stop_cycle < 0) {
    snprintf(h->err, sizeof(h->err), "negative stop_cycle %d", desc->stop_cycle);
    return FG_ERR_ARG;
  }
  if (desc->n_live < 0 || desc->n_live > desc->n_vars) {
    snprintf(h->err, sizeof(h->err), "n_live %d not in [0, n_vars]", desc->n_live);
    return FG_ERR_ARG;
  }
  if (desc->n_words < desc->n_edges) {  // every slot has at least one row of one word
    snprintf(h->err, sizeof(h->err), "bit-row size n_words %lld too small for %d slots", (long long)desc->n_words,
             desc->n_edges);
    return FG_ERR_ARG;
  }
  if (!desc->dev_status || !desc->dev_unresolved ||
      (desc->n_vars > 0 &&
       (!desc->dev_dom_size || !desc->dev_var_id || !desc->dev_var_rank || !desc->dev_var_ptr ||
        !desc->dev_nbr_ptr || !desc->dev_nbr_idx || !desc->dev_value[0] || !desc->dev_value[1] ||
        !desc->dev_cost || !desc->dev_has_cost || !desc->dev_eval || !desc->dev_improve || !desc->dev_counter ||
        !desc->dev_counter_own || !desc->dev_new_value || !desc->dev_can_move || !desc->dev_qlm ||
        !desc->dev_consistent || !desc->dev_finish_phase))) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_edges > 0 && (!desc->dev_tables || !desc->dev_edge_var || !desc->dev_edge_class ||
                            !desc->dev_slot_edge || !desc->dev_bit_off || !desc->dev_bits || !desc->dev_weight ||
                            !desc->dev_violated)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  h->eval_dmax = dba_eval_dmax(h->classes.data(), (int)h->classes.size());
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_dba_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id),
                             FG_FIELD(d, dev_var_rank), FG_FIELD(d, dev_edge_var), FG_FIELD(d, dev_edge_class),
                             FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_nbr_ptr),
                             FG_FIELD(d, dev_nbr_idx), FG_FIELD(d, dev_bit_off), FG_FIELD(d, dev_bits),
                             FG_FIELD(d, dev_value[0]), FG_FIELD(d, dev_value[1]), FG_FIELD(d, dev_cost),
                             FG_FIELD(d, dev_has_cost), FG_FIELD(d, dev_eval), FG_FIELD(d, dev_improve),
                             FG_FIELD(d, dev_counter), FG_FIELD(d, dev_counter_own), FG_FIELD(d, dev_new_value),
                             FG_FIELD(d, dev_can_move), FG_FIELD(d, dev_qlm), FG_FIELD(d, dev_consistent),
                             FG_FIELD(d, dev_finish_phase), FG_FIELD(d, dev_weight), FG_FIELD(d, dev_violated),
                             FG_FIELD(d, dev_status), FG_FIELD(d, dev_unresolved)});
  if (rc != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_dba_destroy(fg_dba_t h) { return fg_close(h); }

extern "C" const char *fg_dba_last_error(fg_dba_t h) { return fg_last_error(h); }

extern "C" int fg_dba_init(fg_dba_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  fg_launcher launch(h, st);
  if (h->d.precision == FG_F64) dba_init<double>(h->d, h->dev_classes, launch);
  else dba_init<float>(h->d, h->dev_classes, launch);
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  h->started = true;
  h->ended = false;
  h->end_round = FG_DBA_LIVE;
  h->last_stream = st;
  return FG_OK;
}

static int dba_round(fg_dba *h, cudaStream_t st) {
  fg_launcher launch(h, st);
  if (h->d.n_vars) dba_cycle(h->d, h->dev_classes, h->eval_dmax, h->cycle, launch);
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return fg_trace_cycle(h, h->d.dev_value[h->cycle % 2], st);
}

extern "C" int fg_dba_step(fg_dba_t h, int32_t n_cycles, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n_cycles; ++i) {
    if (dba_finished(h)) break;
    if (h->cycle >= INT32_MAX / 2 - 1) {  // phase stamps are int32
      snprintf(h->err, sizeof(h->err), "round count exceeds %d", INT32_MAX / 2 - 1);
      return FG_ERR_ARG;
    }
    int rc = dba_round(h, st);
    if (rc != FG_OK) return rc;
    h->last_stream = st;
  }
  return FG_OK;
}

extern "C" int fg_dba_current(fg_dba_t h, int64_t *cycle, int32_t *finished) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (h->started && !h->ended) {
    int32_t status[2];
    CUDA_TRY(h, cudaMemcpyAsync(status, h->d.dev_status, sizeof(status), cudaMemcpyDeviceToHost, h->last_stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->last_stream));
    if (status[1] != FG_DBA_LIVE) {
      h->ended = true;
      h->end_round = status[1];
    }
  }
  if (cycle) *cycle = h->ended && h->end_round < h->cycle ? h->end_round : h->cycle;
  if (finished) *finished = dba_finished(h) ? 1 : 0;
  return FG_OK;
}

extern "C" int64_t fg_dba_launch_count(fg_dba_t h) { return fg_launch_count(h); }

extern "C" int fg_dba_set_trace(fg_dba_t h, fg_trace_t tr) { return fg_set_trace(h, tr); }
