// TEST INFRASTRUCTURE: runs fg_dba_init / fg_dba_step's launch sequence (pydcop_b200/csrc/dba_kernels.cuh) on the
// CPU.  The descriptor is the C-ABI's fg_dba_desc_t with HOST pointers.  Nothing in the product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/dba_kernels.cuh"

extern "C" {
int64_t dba_host_init(const fg_dba_desc_t *d) {
  fg_host_launcher launch;
  if (d->precision == FG_F64) dba_init<double>(*d, d->classes, launch);
  else dba_init<float>(*d, d->classes, launch);
  return launch.launches;
}

// round done + 1
int64_t dba_host_cycle(const fg_dba_desc_t *d, int64_t done) {
  fg_host_launcher launch;
  if (d->n_vars) dba_cycle(*d, d->classes, dba_eval_dmax(d->classes, d->n_classes), done, launch);
  return launch.launches;
}
}  // extern "C"
