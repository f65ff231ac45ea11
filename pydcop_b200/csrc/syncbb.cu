// SyncBB for the whole chain: C-ABI entry points fg_syncbb_* and their kernels (csrc/syncbb_kernels.cuh).  Its own
// translation unit, so the other families' code is compiled exactly as before.
#include "handle.cuh"
#include "syncbb_kernels.cuh"

// the path's values and costs live in shared memory while they fit in the default 48 KB with the kernel's static
// arrays; longer chains read them from global memory
static const size_t SBB_SMEM_PATH_MAX = 40 * 1024;

struct fg_syncbb : fg_handle_base {
  fg_syncbb_desc_t d;
  cudaStream_t last_stream = nullptr;   // where the last init / step enqueued its work
  bool started = false;
};

template <typename T>
static SbbSide<T> sbb_side(const fg_syncbb *h) {
  const fg_syncbb_desc_t &d = h->d;
  return SbbSide<T>{d.n_vars, d.mode_max, d.dev_dom, d.dev_elt_ptr, d.dev_elt_pos, d.dev_elt_tab,
                    (const T *)d.dev_pair, (T *)d.dev_ub, d.dev_sel, d.dev_path_val, (T *)d.dev_path_cost,
                    (T *)d.dev_path_sum, (T *)d.dev_path_comp, d.dev_msg, (T *)d.dev_msg_ub, d.dev_count, d.dev_cycles};
}

static size_t sbb_path_bytes(const fg_syncbb_desc_t &d) {
  return (size_t)d.n_vars * ((d.precision == FG_F64 ? sizeof(double) : sizeof(float)) + sizeof(int32_t));
}

extern "C" int fg_syncbb_create(const fg_syncbb_desc_t *desc, fg_syncbb_t *out) {
  if (!desc || !out) return FG_ERR_ARG;
  *out = nullptr;
  if (desc->precision != FG_F32 && desc->precision != FG_F64) return FG_ERR_ARG;
  fg_syncbb *h = fg_alloc(desc, out);
  if (!h) return FG_ERR_ARG;
  if (desc->n_vars < 2) {
    snprintf(h->err, sizeof(h->err), "n_vars %d: SyncBB needs a chain of at least two variables", desc->n_vars);
    return FG_ERR_ARG;
  }
  if (desc->mode_max != 0 && desc->mode_max != 1) {
    snprintf(h->err, sizeof(h->err), "mode_max %d not 0 or 1", desc->mode_max);
    return FG_ERR_ARG;
  }
  if (desc->n_elts < 0 || desc->n_pair < 0 || (desc->n_elts > 0) != (desc->n_pair > 0)) {
    snprintf(h->err, sizeof(h->err), "n_elts %lld / n_pair %lld inconsistent", (long long)desc->n_elts,
             (long long)desc->n_pair);
    return FG_ERR_ARG;
  }
  if (!desc->dev_dom || !desc->dev_elt_ptr || !desc->dev_ub || !desc->dev_sel || !desc->dev_path_val ||
      !desc->dev_path_cost || !desc->dev_path_sum || !desc->dev_path_comp || !desc->dev_msg || !desc->dev_msg_ub ||
      !desc->dev_count || !desc->dev_cycles || (desc->n_elts > 0 && (!desc->dev_elt_pos || !desc->dev_elt_tab || !desc->dev_pair))) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  int rc = fg_require_device(h);
  if (rc != FG_OK) return rc;
  const fg_syncbb_desc_t &d = *desc;
  return fg_check_resident(h, {FG_FIELD(d, dev_dom), FG_FIELD(d, dev_elt_ptr), FG_FIELD(d, dev_elt_pos),
                               FG_FIELD(d, dev_elt_tab), FG_FIELD(d, dev_pair), FG_FIELD(d, dev_ub),
                               FG_FIELD(d, dev_sel), FG_FIELD(d, dev_path_val), FG_FIELD(d, dev_path_cost),
                               FG_FIELD(d, dev_path_sum), FG_FIELD(d, dev_path_comp), FG_FIELD(d, dev_msg),
                               FG_FIELD(d, dev_msg_ub), FG_FIELD(d, dev_count),
                               FG_FIELD(d, dev_cycles)});
}

extern "C" int fg_syncbb_destroy(fg_syncbb_t h) { return fg_close(h); }

extern "C" const char *fg_syncbb_last_error(fg_syncbb_t h) { return fg_last_error(h); }

extern "C" int fg_syncbb_init(fg_syncbb_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((h->d.n_vars + 255) / 256 < 1024 ? (h->d.n_vars + 255) / 256 : 1024);
  if (h->d.precision == FG_F64) k_syncbb_init<double><<<blocks, 256, 0, st>>>(sbb_side<double>(h));
  else k_syncbb_init<float><<<blocks, 256, 0, st>>>(sbb_side<float>(h));
  ++h->launches;
  CUDA_TRY(h, cudaGetLastError());
  h->started = true;
  h->last_stream = st;
  return FG_OK;
}

extern "C" int fg_syncbb_step(fg_syncbb_t h, int64_t n_steps, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (!h->started) {
    snprintf(h->err, sizeof(h->err), "fg_syncbb_step before fg_syncbb_init");
    return FG_ERR_ARG;
  }
  if (n_steps <= 0) return FG_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = sbb_path_bytes(h->d);
  const int smem_path = bytes <= SBB_SMEM_PATH_MAX;
  const size_t dyn = smem_path ? bytes : 0;
  if (h->d.precision == FG_F64) k_syncbb<double><<<1, SBB_THREADS, dyn, st>>>(sbb_side<double>(h), n_steps, smem_path);
  else k_syncbb<float><<<1, SBB_THREADS, dyn, st>>>(sbb_side<float>(h), n_steps, smem_path);
  ++h->launches;
  CUDA_TRY(h, cudaGetLastError());
  h->last_stream = st;
  return FG_OK;
}

extern "C" int fg_syncbb_current(fg_syncbb_t h, int64_t *steps, int64_t *messages, int32_t *finished) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  int64_t count[2] = {0, 0};
  int32_t msg[4] = {0, 0, 0, 0};
  if (h->started) {
    CUDA_TRY(h, cudaMemcpyAsync(count, h->d.dev_count, sizeof(count), cudaMemcpyDeviceToHost, h->last_stream));
    CUDA_TRY(h, cudaMemcpyAsync(msg, h->d.dev_msg, sizeof(msg), cudaMemcpyDeviceToHost, h->last_stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->last_stream));
  }
  if (steps) *steps = count[0];
  if (messages) *messages = count[1];
  if (finished) *finished = msg[3];
  return FG_OK;
}

extern "C" int64_t fg_syncbb_launch_count(fg_syncbb_t h) { return fg_launch_count(h); }
