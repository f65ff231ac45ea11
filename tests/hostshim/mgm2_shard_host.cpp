// TEST INFRASTRUCTURE: runs fg_mgm2_shard_init / _phase / _unpack's launch sequences
// (pydcop_b200/csrc/mgm2_shard_kernels.cuh) on the CPU, so the sharded host logic can be compared with the
// single-process run without a GPU.  The descriptor and the shard plan are the C-ABI's fg_mgm2_desc_t /
// fg_mgm2_shard_plan_t with HOST pointers.  Nothing in the product links or calls this.
#include "cuda_host.h"
#include "../../pydcop_b200/csrc/mgm2_shard_kernels.cuh"

extern "C" {
int64_t mgm2_shard_host_init(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p) {
  fg_host_launcher launch;
  if (d->precision == FG_F64) mgm2s_init<double>(*d, d->classes, *p, launch);
  else mgm2s_init<float>(*d, d->classes, *p, launch);
  return launch.launches;
}

// exchange x of round done + 1
int64_t mgm2_shard_host_phase(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int32_t x, int64_t done) {
  fg_host_launcher launch;
  if (d->precision == FG_F64) mgm2s_phase<double>(*d, d->classes, *p, x, done, launch);
  else mgm2s_phase<float>(*d, d->classes, *p, x, done, launch);
  return launch.launches;
}

int64_t mgm2_shard_host_unpack(const fg_mgm2_desc_t *d, const fg_mgm2_shard_plan_t *p, int32_t x) {
  fg_host_launcher launch;
  if (d->precision == FG_F64) mgm2x_unpack<double>(*d, *p, x, launch);
  else mgm2x_unpack<float>(*d, *p, x, launch);
  return launch.launches;
}
}  // extern "C"
