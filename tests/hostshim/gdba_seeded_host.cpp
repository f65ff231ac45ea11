// TEST INFRASTRUCTURE: gdba_host.cpp's launches with the descriptor's per-variable Philox key (dev_var_seed into
// MgmSide::var_seed), under the same entry-point names, so the kernel SOURCE of a batch whose problems have seeds of
// their own runs on the CPU.  Nothing in the product links or calls this.
#define gdba_host_init gdba_host_init_unseeded
#define gdba_host_cycle gdba_host_cycle_unseeded
#include "gdba_host.cpp"
#undef gdba_host_init
#undef gdba_host_cycle

static MgmSide seeded_side(const fg_gdba_desc_t *d) {
  MgmSide g = side(d);
  g.var_seed = d->dev_var_seed;
  return g;
}

template <typename T>
static void seeded_cycle_t(const fg_gdba_desc_t *d, int64_t done) {
  const MgmSide g = seeded_side(d);
  const int n = d->n_vars;
  int32_t *vin = d->dev_value[done & 1], *vout = d->dev_value[(done + 1) & 1];
  const int64_t *mod_off = d->increase_mode == FG_GDBA_INCREASE_T ? nullptr : d->dev_mod_off;
  const uint32_t cyc = (uint32_t)(done + 1);
  launch(n, 128, [&] {
    k_gdba_eval<T>(g, n, (const T *)d->dev_tables, (const T *)d->dev_unary, d->dev_unary_off,
                   (const T *)d->dev_viol_ref, d->dev_mod, mod_off, d->modifier, d->violation, vin, (T *)d->dev_cost,
                   d->dev_has_cost, (T *)d->dev_improve, d->dev_new_value, d->dev_violated, d->mode_max, d->seed, cyc);
  });
  launch(n, 256, [&] {
    k_gdba_decide<T>(g, n, (const T *)d->dev_improve, d->dev_new_value, d->dev_violated, d->dev_mod, mod_off,
                     d->increase_mode, d->mode_max, vin, vout, (T *)d->dev_cost, d->dev_breakout);
  });
}

extern "C" {
void gdba_host_init(const fg_gdba_desc_t *d) {
  if (d->mod_size > 0) memset(d->dev_mod, 0, sizeof(int32_t) * (size_t)d->mod_size);
  launch(d->n_vars, 128, [&] {
    k_mgm_init(seeded_side(d), d->n_vars, d->dev_init_value, d->seed, d->dev_value[0], d->dev_has_cost);
  });
}

void gdba_host_cycle(const fg_gdba_desc_t *d, int64_t done) {
  if (d->precision == FG_F64) seeded_cycle_t<double>(d, done);
  else seeded_cycle_t<float>(d, done);
}
}  // extern "C"
