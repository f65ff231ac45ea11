// TEST INFRASTRUCTURE: runs fg_dsa_init / fg_dsa_cycle_compute's generic launch sequence
// (pydcop_b200/csrc/dsa_generic.cuh) on the CPU.  The descriptor is the C-ABI's fg_dsa_desc_t with HOST pointers.
// Nothing in the product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/dsa_generic.cuh"

extern "C" {
int64_t dsa_host_init(const fg_dsa_desc_t *d) {
  fg_host_launcher launch;
  if (d->precision == FG_F64) dsa_init<double>(*d, d->classes, launch);
  else dsa_init<float>(*d, d->classes, launch);
  return launch.launches;
}

// round done, from buffer done & 1 (fg_dsa_current's buf_index) into the other one
int64_t dsa_host_cycle(const fg_dsa_desc_t *d, int64_t done) {
  fg_host_launcher launch;
  if (d->n_vars) {
    if (d->precision == FG_F64) dsa_step<double>(*d, d->classes, (int)(done & 1), (uint32_t)done, launch);
    else dsa_step<float>(*d, d->classes, (int)(done & 1), (uint32_t)done, launch);
  }
  return launch.launches;
}
}  // extern "C"
