// DPOP: C-ABI entry points fg_dpop_* and their kernels (csrc/dpop_kernels.cuh, which states the
// floating-point operand order).  Its own translation unit, so the other families are compiled exactly
// as before.
#include "handle.cuh"
#include "dpop_kernels.cuh"

struct fg_dpop : fg_handle_base {   // no class table: classes stays empty
  fg_dpop_desc_t d;
  std::vector<fg_dpop_launch_t> util_launches, value_launches;
  int n_sm = 132;
};

static DpopNodes dpop_nodes(const fg_dpop_desc_t &d) {
  return DpopNodes{d.dev_dom_size, d.dev_unary_off, d.dev_util_off, d.dev_util_size, d.dev_sep_ptr,
                   d.dev_sep_var, d.dev_term_ptr, d.dev_term_kind, d.dev_term_base, d.dev_term_own,
                   d.dev_tdim_ptr, d.dev_tdim_pos, d.dev_tdim_stride};
}

static bool dpop_check_launches(fg_dpop *h, const std::vector<fg_dpop_launch_t> &ls, int n_segs, bool allow_big,
                                const char *phase) {
  for (const auto &l : ls) {
    bool ok;
    if (l.kind == 0) ok = l.first >= 0 && l.count >= 0 && (int64_t)l.first + l.count <= n_segs;
    else ok = allow_big && l.kind == 1 && l.first >= 0 && l.first < h->d.n_vars;
    if (!ok) {
      snprintf(h->err, sizeof(h->err), "%s launch (kind %d, first %d, count %d) out of range", phase, l.kind,
               l.first, l.count);
      return false;
    }
  }
  return true;
}

extern "C" int fg_dpop_create(const fg_dpop_desc_t *desc, fg_dpop_t *out) {
  fg_dpop *h = fg_alloc(desc, out);
  if (!h) return FG_ERR_ARG;
  if (desc->precision != FG_F32 && desc->precision != FG_F64) {
    snprintf(h->err, sizeof(h->err), "precision %d is not FG_F32 (0) or FG_F64 (1)", desc->precision);
    return FG_ERR_ARG;
  }
  if (desc->n_vars < 0 || desc->n_util_segs < 0 || desc->n_value_segs < 0 || desc->n_util_launches < 0 ||
      desc->n_value_launches < 0 || desc->arena_size < 0) {
    snprintf(h->err, sizeof(h->err), "negative size in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->max_sep < 0 || desc->max_sep > FG_DPOP_MAX_SEP) {
    snprintf(h->err, sizeof(h->err), "separator of %d variables: the kernels decode at most %d", desc->max_sep,
             FG_DPOP_MAX_SEP);
    return FG_ERR_ARG;
  }
  if ((desc->n_util_launches && !desc->util_launches) || (desc->n_value_launches && !desc->value_launches)) {
    snprintf(h->err, sizeof(h->err), "missing launch list in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_vars > 0 &&
      (!desc->dev_unary || !desc->dev_arena || !desc->dev_dom_size || !desc->dev_unary_off || !desc->dev_util_off ||
       !desc->dev_util_size || !desc->dev_sep_ptr || !desc->dev_term_ptr || !desc->dev_util_nodes ||
       !desc->dev_util_seg_ptr || !desc->dev_value_nodes || !desc->dev_value_seg_ptr || !desc->dev_value ||
       !desc->dev_cost || !desc->dev_unresolved || (desc->n_terms > 0 && (!desc->dev_term_kind ||
       !desc->dev_term_base || !desc->dev_term_own || !desc->dev_tdim_ptr)) ||
       (desc->n_tdims > 0 && (!desc->dev_tdim_pos || !desc->dev_tdim_stride || !desc->dev_sep_var)))) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  h->util_launches.assign(desc->util_launches, desc->util_launches + desc->n_util_launches);
  h->value_launches.assign(desc->value_launches, desc->value_launches + desc->n_value_launches);
  h->d.util_launches = h->util_launches.data();
  h->d.value_launches = h->value_launches.data();
  if (!dpop_check_launches(h, h->util_launches, desc->n_util_segs, true, "UTIL") ||
      !dpop_check_launches(h, h->value_launches, desc->n_value_segs, false, "VALUE"))
    return FG_ERR_ARG;
  int rc = fg_require_device(h);
  if (rc != FG_OK) return rc;
  const fg_dpop_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_unary), FG_FIELD(d, dev_tables), FG_FIELD(d, dev_arena),
                             FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_unary_off), FG_FIELD(d, dev_util_off),
                             FG_FIELD(d, dev_util_size), FG_FIELD(d, dev_sep_ptr), FG_FIELD(d, dev_sep_var),
                             FG_FIELD(d, dev_term_ptr), FG_FIELD(d, dev_term_kind), FG_FIELD(d, dev_term_base),
                             FG_FIELD(d, dev_term_own), FG_FIELD(d, dev_tdim_ptr), FG_FIELD(d, dev_tdim_pos),
                             FG_FIELD(d, dev_tdim_stride), FG_FIELD(d, dev_util_nodes), FG_FIELD(d, dev_util_seg_ptr),
                             FG_FIELD(d, dev_value_nodes), FG_FIELD(d, dev_value_seg_ptr), FG_FIELD(d, dev_value),
                             FG_FIELD(d, dev_cost), FG_FIELD(d, dev_unresolved)});
  if (rc != FG_OK) return rc;
  CUDA_TRY(h, cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, h->device));
  return FG_OK;
}

extern "C" int fg_dpop_destroy(fg_dpop_t h) { return fg_close(h); }

extern "C" const char *fg_dpop_last_error(fg_dpop_t h) { return fg_last_error(h); }

static inline unsigned dpop_warp_blocks(int n_warps) { return (unsigned)((n_warps + 3) / 4); }

template <typename T>
static int dpop_run_t(fg_dpop *h, cudaStream_t st) {
  const fg_dpop_desc_t &d = h->d;
  const DpopNodes g = dpop_nodes(d);
  const DpopData<T> a{(const T *)d.dev_unary, (const T *)d.dev_tables, (T *)d.dev_arena};
  for (const auto &l : h->util_launches) {
    if (l.kind == 0) {
      if (!l.count) continue;
      k_dpop_util_walk<T><<<dpop_warp_blocks(l.count), 128, 0, st>>>(g, a, d.dev_util_nodes, d.dev_util_seg_ptr,
                                                                   l.first, l.count, d.mode_max);
    } else {
      k_dpop_util_big<T><<<(unsigned)(h->n_sm * 8), 256, 0, st>>>(g, a, l.first, d.mode_max);
    }
    ++h->launches;
  }
  for (const auto &l : h->value_launches) {
    if (!l.count) continue;
    k_dpop_value_walk<T><<<dpop_warp_blocks(l.count), 128, 0, st>>>(g, a, d.dev_value_nodes, d.dev_value_seg_ptr,
                                                                  l.first, l.count, d.mode_max, d.dev_value,
                                                                  (T *)d.dev_cost, d.dev_unresolved);
    ++h->launches;
  }
  CUDA_TRY(h, cudaGetLastError());
  return FG_OK;
}

extern "C" int fg_dpop_run(fg_dpop_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  if (h->d.n_vars == 0) return FG_OK;
  CUDA_TRY(h, cudaMemsetAsync(h->d.dev_unresolved, 0, sizeof(int32_t), st));
  return h->d.precision == FG_F64 ? dpop_run_t<double>(h, st) : dpop_run_t<float>(h, st);
}

extern "C" int64_t fg_dpop_launch_count(fg_dpop_t h) { return fg_launch_count(h); }
