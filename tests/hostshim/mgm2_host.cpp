// TEST INFRASTRUCTURE: runs fg_mgm2_init / fg_mgm2_step's launch sequence (pydcop_b200/csrc/mgm2_kernels.cuh) on the
// CPU.  The descriptor is the C-ABI's fg_mgm2_desc_t with HOST pointers.  Nothing in the product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/mgm2_kernels.cuh"

extern "C" {
int64_t mgm2_host_init(const fg_mgm2_desc_t *d) {
  fg_host_launcher launch;
  if (d->n_vars) {
    if (d->precision == FG_F64) mgm2_init<double>(*d, d->classes, launch);
    else mgm2_init<float>(*d, d->classes, launch);
  }
  return launch.launches;
}

// round done + 1
int64_t mgm2_host_cycle(const fg_mgm2_desc_t *d, int64_t done) {
  fg_host_launcher launch;
  if (d->n_vars) {
    if (d->precision == FG_F64) mgm2_cycle<double>(*d, d->classes, done, launch);
    else mgm2_cycle<float>(*d, d->classes, done, launch);
  }
  return launch.launches;
}
}  // extern "C"
