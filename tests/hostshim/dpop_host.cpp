// TEST INFRASTRUCTURE: runs the DPOP CUDA kernel SOURCE (pydcop_b200/csrc/dpop_kernels.cuh) on the CPU:
// the UTIL launches of the schedule in order, each segment's nodes bottom-up with dpop_util_entry on every
// UTIL entry, then the VALUE paths top-down with dpop_value_node, so its logic can be compared with the
// oracle and the reference's messages without a GPU.  Nothing in the product links or calls this.
// The descriptor is the C-ABI's fg_dpop_desc_t with HOST pointers.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/dpop_kernels.cuh"

static DpopNodes nodes(const fg_dpop_desc_t *d) {
  return DpopNodes{d->dev_dom_size, d->dev_unary_off, d->dev_util_off, d->dev_util_size, d->dev_sep_ptr,
                   d->dev_sep_var, d->dev_term_ptr, d->dev_term_kind, d->dev_term_base, d->dev_term_own,
                   d->dev_tdim_ptr, d->dev_tdim_pos, d->dev_tdim_stride};
}

template <typename T>
static void run_t(const fg_dpop_desc_t *d) {
  const DpopNodes g = nodes(d);
  const DpopData<T> a{(const T *)d->dev_unary, (const T *)d->dev_tables, (T *)d->dev_arena};
  *d->dev_unresolved = 0;
  for (int k = 0; k < d->n_util_launches; ++k) {
    const fg_dpop_launch_t &l = d->util_launches[k];
    if (l.kind == 1) {
      for (int64_t i = 0; i < d->dev_util_size[l.first]; ++i) dpop_util_entry(g, a, l.first, i, d->mode_max);
      continue;
    }
    for (int s = l.first; s < l.first + l.count; ++s)
      for (int i = d->dev_util_seg_ptr[s]; i < d->dev_util_seg_ptr[s + 1]; ++i) {
        const int u = d->dev_util_nodes[i];
        for (int64_t e = 0; e < d->dev_util_size[u]; ++e) dpop_util_entry(g, a, u, e, d->mode_max);
      }
  }
  for (int k = 0; k < d->n_value_launches; ++k) {
    const fg_dpop_launch_t &l = d->value_launches[k];
    for (int s = l.first; s < l.first + l.count; ++s)
      for (int i = d->dev_value_seg_ptr[s]; i < d->dev_value_seg_ptr[s + 1]; ++i)
        dpop_value_node(g, a, d->dev_value_nodes[i], d->mode_max, d->dev_value, (T *)d->dev_cost,
                        d->dev_unresolved);
  }
}

extern "C" void dpop_host_run(const fg_dpop_desc_t *d) {
  if (d->precision == FG_F64) run_t<double>(d);
  else run_t<float>(d);
}
