// TEST INFRASTRUCTURE: mgm2_host.cpp's launches with the descriptor's per-variable Philox key (dev_var_seed into
// MgmSide::var_seed), under the same entry-point names, so the kernel SOURCE of a batch whose problems have seeds of
// their own runs on the CPU.  Nothing in the product links or calls this.
#define mgm2_host_init mgm2_host_init_unseeded
#define mgm2_host_cycle mgm2_host_cycle_unseeded
#include "mgm2_host.cpp"
#undef mgm2_host_init
#undef mgm2_host_cycle

static MgmSide seeded_side(const fg_mgm2_desc_t *d) {
  MgmSide g = side(d);
  g.var_seed = d->dev_var_seed;
  return g;
}

template <typename T>
static void seeded_init_t(const fg_mgm2_desc_t *d) {
  launch(d->n_vars, 128, [&] {
    k_mgm2_init<T>(seeded_side(d), d->n_vars, (const T *)d->dev_tables, d->dev_init_value, d->mode_max, d->seed,
                   d->dev_value, (T *)d->dev_cost, d->dev_has_cost);
  });
}

template <typename T>
static void seeded_cycle_t(const fg_mgm2_desc_t *d, uint32_t cyc) {
  const MgmSide g = seeded_side(d);
  const int n = d->n_vars;
  T *cost = (T *)d->dev_cost, *local = (T *)d->dev_local_cost, *gain = (T *)d->dev_gain;
  launch(n, 128, [&] {
    k_mgm2_value<T>(g, n, (const T *)d->dev_tables, d->dev_value, cost, d->dev_has_cost, local, gain,
                    d->dev_potential_value, d->dev_offerer, d->dev_partner, d->dev_committed, d->dev_answer,
                    d->dev_offer_off, (T *)d->dev_offer, d->mode_max, d->threshold, d->seed, cyc);
  });
  launch(n, 128, [&] {
    k_mgm2_answer<T>(g, n, (const T *)d->dev_tables, d->dev_value, local, gain, d->dev_potential_value,
                     d->dev_offerer, d->dev_partner, d->dev_committed, d->dev_answer, d->dev_answer_value,
                     (T *)d->dev_answer_gain, d->dev_offer_off, (const T *)d->dev_offer, d->mode_max, d->favor,
                     d->seed, cyc);
  });
  launch(n, 256, [&] {
    k_mgm2_commit<T>(n, d->dev_offerer, d->dev_answer, d->dev_answer_value, (const T *)d->dev_answer_gain, gain,
                     d->dev_potential_value, d->dev_committed);
  });
  launch(n, 256, [&] {
    k_mgm2_gain<T>(g, n, gain, d->dev_potential_value, d->dev_committed, d->dev_partner, d->dev_go, d->dev_value,
                   cost);
  });
  launch(n, 256, [&] {
    k_mgm2_go<T>(n, d->dev_committed, d->dev_partner, d->dev_go, gain, d->dev_potential_value, d->dev_value, cost);
  });
}

extern "C" {
void mgm2_host_init(const fg_mgm2_desc_t *d) {
  if (d->precision == FG_F64) seeded_init_t<double>(d);
  else seeded_init_t<float>(d);
}

void mgm2_host_cycle(const fg_mgm2_desc_t *d, uint32_t cycle) {
  if (d->precision == FG_F64) seeded_cycle_t<double>(d, cycle);
  else seeded_cycle_t<float>(d, cycle);
}
}  // extern "C"
