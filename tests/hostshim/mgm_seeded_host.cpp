// TEST INFRASTRUCTURE: mgm_host.cpp's launches with a per-variable Philox key (MgmSide::var_seed), so the kernel
// SOURCE of a batch whose problems have seeds of their own runs on the CPU.  Nothing in the product links or calls
// this.  var_seed: internal order, NULL = a->seed for every variable.
#include "mgm_host.cpp"

static MgmSide seeded_side(const mgm_host_arrays *a, const uint64_t *var_seed) {
  MgmSide g = side(a);
  g.var_seed = var_seed;
  return g;
}

template <typename T>
static void seeded_cycle_t(const mgm_host_arrays *a, uint32_t cycle, const uint64_t *var_seed) {
  launch(a->n_vars, 128, [&] {
    k_mgm_gain<T>(seeded_side(a, var_seed), a->n_vars, (const T *)a->tables, (const T *)a->unary, a->value,
                  (T *)a->cost, a->has_cost, (T *)a->gain, a->new_value, a->mode_max, a->seed, cycle);
  });
  launch(a->n_vars, 256, [&] {
    k_mgm_decide<T>(side(a), a->n_vars, (const T *)a->gain, a->new_value, a->value, (T *)a->cost);
  });
}

extern "C" {
void mgm_host_init_seeded(const mgm_host_arrays *a, const uint64_t *var_seed) {
  launch(a->n_vars, 128, [&] {
    k_mgm_init(seeded_side(a, var_seed), a->n_vars, a->init_value, a->seed, a->value, a->has_cost);
  });
}

void mgm_host_cycle_seeded(const mgm_host_arrays *a, uint32_t cycle, const uint64_t *var_seed) {
  if (a->precision == FG_F64) seeded_cycle_t<double>(a, cycle, var_seed);
  else seeded_cycle_t<float>(a, cycle, var_seed);
}
}  // extern "C"
