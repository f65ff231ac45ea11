// TEST INFRASTRUCTURE: dsa_generic_host.cpp's launches with a per-variable Philox key (DsaSide::var_seed), so the
// kernel SOURCE of a batch whose problems have seeds of their own runs on the CPU.  Nothing in the product links or
// calls this.  var_seed: internal order, NULL = h->seed for every variable.
#include "dsa_generic_host.cpp"

static DsaSide seeded_side(const dsa_host *h, const uint64_t *var_seed) {
  DsaSide g = side(h);
  g.var_seed = var_seed;
  return g;
}

template <typename T>
static void seeded_init_t(const dsa_host *h, const uint64_t *var_seed) {
  for (int ci = 0; ci < h->n_classes; ++ci) {
    const fg_class_t &c = h->classes[ci];
    if (!c.n_factors) continue;
    launch(c.n_factors, [&] { k_dsa_con_opt<T>(c, (const T *)h->tables, (T *)h->con_opt, h->mode_max); });
  }
  launch(h->n_vars, [&] { k_dsa_init(seeded_side(h, var_seed), h->n_vars, h->seed, h->value[0]); });
  memcpy(h->value[1], h->value[0], sizeof(int32_t) * (size_t)h->n_vars);
}

template <typename T>
static void seeded_step_t(const dsa_host *h, int cur, uint32_t cycle, const uint64_t *var_seed) {
  launch(h->n_vars, [&] {
    k_dsa_step_generic<T>(seeded_side(h, var_seed), h->n_vars, (const T *)h->tables, (const T *)h->con_opt,
                          h->value[cur], h->value[cur ^ 1], (T *)h->value_cost, h->mode_max, h->variant, h->seed,
                          cycle, (const T *)h->var_cost, h->unary_off);
  });
}

extern "C" void dsa_host_init_seeded(const dsa_host *h, const uint64_t *var_seed) {
  if (h->precision == FG_F64) seeded_init_t<double>(h, var_seed); else seeded_init_t<float>(h, var_seed);
}
extern "C" void dsa_host_step_seeded(const dsa_host *h, int cur, uint32_t cycle, const uint64_t *var_seed) {
  if (h->precision == FG_F64) seeded_step_t<double>(h, cur, cycle, var_seed);
  else seeded_step_t<float>(h, cur, cycle, var_seed);
}
