// TEST INFRASTRUCTURE: runs fg_mixeddsa_init / fg_mixeddsa_step's launch sequence
// (pydcop_b200/csrc/mixeddsa_kernels.cuh) on the CPU.  The descriptor is the C-ABI's fg_mixeddsa_desc_t with HOST
// pointers.  Nothing in the product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/dsa_generic.cuh"
#include "../../pydcop_b200/csrc/mixeddsa_kernels.cuh"

extern "C" {
int64_t mixeddsa_host_init(const fg_mixeddsa_desc_t *d) {
  fg_host_launcher launch;
  if (d->precision == FG_F64) mixeddsa_init<double>(*d, d->classes, launch);
  else mixeddsa_init<float>(*d, d->classes, launch);
  return launch.launches;
}

// round done + 1
int64_t mixeddsa_host_cycle(const fg_mixeddsa_desc_t *d, int64_t done) {
  fg_host_launcher launch;
  const int dmax = mixeddsa_dmax(d->classes, d->n_classes);
  if (d->n_vars) {
    if (d->precision == FG_F64) mixeddsa_cycle<double>(*d, d->classes, dmax, done, launch);
    else mixeddsa_cycle<float>(*d, d->classes, dmax, done, launch);
  }
  return launch.launches;
}
}  // extern "C"
