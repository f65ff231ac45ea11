// TEST INFRASTRUCTURE: runs fg_mgm_init / fg_mgm_step's launch sequence (pydcop_b200/csrc/mgm_fast_kernels.cuh) on
// the CPU.  The descriptor is the C-ABI's fg_mgm_desc_t with HOST pointers.  Nothing in the product links or calls
// this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/mgm_fast_kernels.cuh"

extern "C" {
int64_t mgm_host_init(const fg_mgm_desc_t *d) {
  fg_host_launcher launch;
  if (d->n_vars) mgm_init(*d, d->classes, launch);
  return launch.launches;
}

// round done + 1; -1 with the active-row arrays (dev_row_cache): that value phase is block-cooperative and has no
// thread-by-thread run
int64_t mgm_host_cycle(const fg_mgm_desc_t *d, int64_t done) {
  if (d->dev_row_cache) return -1;
  fg_host_launcher launch;
  if (d->n_vars) {
    if (d->precision == FG_F64) {
      mgm_gain<double>(*d, d->classes, done, launch);
      mgm_decide<double>(*d, d->classes, launch);
    } else {
      mgm_gain<float>(*d, d->classes, done, launch);
      mgm_decide<float>(*d, d->classes, launch);
    }
  }
  return launch.launches;
}
}  // extern "C"
