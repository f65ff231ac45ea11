// TEST INFRASTRUCTURE: mixeddsa_host.cpp's launches with the descriptor's per-variable Philox key (dev_var_seed into
// MgmSide::var_seed), under the same entry-point names, so the kernel SOURCE of a batch whose problems have seeds of
// their own runs on the CPU.  Nothing in the product links or calls this.
#define mixeddsa_host_init mixeddsa_host_init_unseeded
#define mixeddsa_host_cycle mixeddsa_host_cycle_unseeded
#include "mixeddsa_host.cpp"
#undef mixeddsa_host_init
#undef mixeddsa_host_cycle

static MgmSide seeded_side(const fg_mixeddsa_desc_t *d) {
  MgmSide g = side(d);
  g.var_seed = d->dev_var_seed;
  return g;
}

template <typename T>
static void seeded_init_t(const fg_mixeddsa_desc_t *d) {
  for (int ci = 0; ci < d->n_classes; ++ci) {
    const fg_class_t &c = d->classes[ci];
    if (!c.n_factors) continue;
    launch(c.n_factors, 128, [&] { k_dsa_con_opt<T>(c, (const T *)d->dev_tables, (T *)d->dev_con_opt, d->mode_max); });
  }
  launch(d->n_vars, 128, [&] {
    k_mixeddsa_init(seeded_side(d), d->n_vars, d->dev_init_value, d->seed, d->dev_value[0], d->dev_has_cost);
  });
}

template <typename T, int DMAX>
static void seeded_round_t(const fg_mixeddsa_desc_t *d, int64_t done) {
  int32_t *vin = d->dev_value[done & 1], *vout = d->dev_value[(done + 1) & 1];
  launch(d->n_vars, 128, [&] {
    k_mixeddsa_step<T, DMAX>(seeded_side(d), d->n_vars, (const T *)d->dev_tables, (const T *)d->dev_unary,
                             d->dev_soft_end, (const T *)d->dev_con_opt, vin, vout, (T *)d->dev_cost, d->dev_has_cost,
                             d->dev_h_best, d->dev_branch, d->mode_max, d->variant, d->proba_hard, d->proba_soft,
                             (T)INFINITY, d->seed, (uint32_t)(done + 1));
  });
}

template <typename T>
static void seeded_cycle_t(const fg_mixeddsa_desc_t *d, int64_t done) {
  if (mixeddsa_dmax(d->classes, d->n_classes) <= 32) seeded_round_t<T, 32>(d, done);
  else seeded_round_t<T, FG_MAX_DOM>(d, done);
}

extern "C" {
void mixeddsa_host_init(const fg_mixeddsa_desc_t *d) {
  if (d->precision == FG_F64) seeded_init_t<double>(d);
  else seeded_init_t<float>(d);
}

void mixeddsa_host_cycle(const fg_mixeddsa_desc_t *d, int64_t done) {
  if (d->precision == FG_F64) seeded_cycle_t<double>(d, done);
  else seeded_cycle_t<float>(d, done);
}
}  // extern "C"
