// TEST INFRASTRUCTURE: runs fg_gdba_init / fg_gdba_step's launch sequence (pydcop_b200/csrc/gdba_kernels.cuh) on the
// CPU.  The descriptor is the C-ABI's fg_gdba_desc_t with HOST pointers.  Nothing in the product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/gdba_kernels.cuh"

extern "C" {
int64_t gdba_host_init(const fg_gdba_desc_t *d) {
  fg_host_launcher launch;
  gdba_init(*d, d->classes, launch);
  return launch.launches;
}

// round done + 1
int64_t gdba_host_cycle(const fg_gdba_desc_t *d, int64_t done) {
  fg_host_launcher launch;
  if (d->n_vars) {
    if (d->precision == FG_F64) gdba_cycle<double>(*d, d->classes, done, launch);
    else gdba_cycle<float>(*d, d->classes, done, launch);
  }
  return launch.launches;
}
}  // extern "C"
