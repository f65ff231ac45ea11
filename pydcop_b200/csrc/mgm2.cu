// MGM-2 for all variables at once: C-ABI entry points fg_mgm2_* and their kernels
// (csrc/mgm2_kernels.cuh).  Its own translation unit, so the MaxSum / DSA / MGM code in engine.cu
// and mgm.cu is compiled exactly as before.
//
// Floating-point operand order follows pydcop/algorithms/mgm2.py so that the f64 build equals the
// reference's Python floats and the f32 build the f32 oracle (tests/_mgm2_oracle.py):
//   cost of an assignment = ((0 + c1) + c2) + ...    in node.constraints order (assignment_cost)
//   offer gain            = current_cost - cost                                   (:553)
//   global gain           = (current_cost - cost over the other constraints) + offer gain (:593)
//   cost after a move     = current_cost - potential_gain                         (:941, :986)
#include <type_traits>

#include "handle.cuh"
#include "mgm2_shard_kernels.cuh"

// engine.cu defines the barrier kernels of peer_sync.cuh; here they get internal linkage (no duplicate host stubs at
// link time).  Its includes (<cuda_runtime.h>, <stdint.h>, <type_traits>, pydcop_b200.h) come before the namespace.
namespace {
#include "peer_sync.cuh"
}

struct fg_mgm2_shard;

struct fg_mgm2 : fg_handle_base {
  fg_mgm2_desc_t d;
  fg_mgm2_shard *shard = nullptr;   // fg_mgm2_shard_attach: this handle runs one rank of a sharded problem
  ~fg_mgm2();
};

extern "C" int fg_mgm2_create(const fg_mgm2_desc_t *desc, fg_mgm2_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_mgm2 *h = *out;
  if (desc->favor < FG_MGM2_FAVOR_UNILATERAL || desc->favor > FG_MGM2_FAVOR_COORDINATED) {
    snprintf(h->err, sizeof(h->err), "favor %d is not one of unilateral (0), no (1), coordinated (2)", desc->favor);
    return FG_ERR_ARG;
  }
  if (!(desc->threshold >= 0.0 && desc->threshold <= 1.0)) {
    snprintf(h->err, sizeof(h->err), "threshold %g is not in [0, 1]", desc->threshold);
    return FG_ERR_ARG;
  }
  if (desc->stop_cycle < 0) {
    snprintf(h->err, sizeof(h->err), "negative stop_cycle %d", desc->stop_cycle);
    return FG_ERR_ARG;
  }
  if (desc->n_vars > 0 &&
      (!desc->dev_tables || !desc->dev_dom_size || !desc->dev_var_id || !desc->dev_var_rank || !desc->dev_var_ptr ||
       !desc->dev_nbr_ptr || !desc->dev_nbr_idx || !desc->dev_value || !desc->dev_cost || !desc->dev_has_cost ||
       !desc->dev_gain || !desc->dev_potential_value || !desc->dev_local_cost || !desc->dev_offerer ||
       !desc->dev_partner || !desc->dev_committed || !desc->dev_go || !desc->dev_answer || !desc->dev_answer_value ||
       !desc->dev_answer_gain || !desc->dev_offer_off || !desc->dev_offer)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if (desc->n_edges > 0 && (!desc->dev_edge_var || !desc->dev_edge_class || !desc->dev_slot_edge)) {
    snprintf(h->err, sizeof(h->err), "missing device array in the descriptor");
    return FG_ERR_ARG;
  }
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_mgm2_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id),
                             FG_FIELD(d, dev_var_rank), FG_FIELD(d, dev_edge_var), FG_FIELD(d, dev_edge_class),
                             FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_nbr_ptr),
                             FG_FIELD(d, dev_nbr_idx), FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_value),
                             FG_FIELD(d, dev_cost), FG_FIELD(d, dev_has_cost), FG_FIELD(d, dev_gain),
                             FG_FIELD(d, dev_potential_value), FG_FIELD(d, dev_local_cost), FG_FIELD(d, dev_offerer),
                             FG_FIELD(d, dev_partner), FG_FIELD(d, dev_committed), FG_FIELD(d, dev_go),
                             FG_FIELD(d, dev_answer), FG_FIELD(d, dev_answer_value), FG_FIELD(d, dev_answer_gain),
                             FG_FIELD(d, dev_offer_off), FG_FIELD(d, dev_offer), FG_FIELD(d, dev_var_seed)});
  if (rc != FG_OK) return rc;
  return fg_upload_classes(h);
}

extern "C" int fg_mgm2_destroy(fg_mgm2_t h) { return fg_close(h); }

extern "C" const char *fg_mgm2_last_error(fg_mgm2_t h) { return fg_last_error(h); }

extern "C" int fg_mgm2_init(fg_mgm2_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  fg_launcher launch(h, (cudaStream_t)stream);
  if (h->d.n_vars) {
    if (h->d.precision == FG_F64) mgm2_init<double>(h->d, h->dev_classes, launch);
    else mgm2_init<float>(h->d, h->dev_classes, launch);
  }
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

template <typename T>
static int mgm2_cycle_t(fg_mgm2 *h, cudaStream_t st) {
  fg_launcher launch(h, st);
  if (h->d.n_vars) mgm2_cycle<T>(h->d, h->dev_classes, h->cycle, launch);
  CUDA_TRY(h, cudaGetLastError());
  ++h->cycle;
  return FG_OK;
}

extern "C" int fg_mgm2_step(fg_mgm2_t h, int32_t n_cycles, void *stream) {
  return fg_step(h, n_cycles, stream, mgm2_cycle_t<float>, mgm2_cycle_t<double>);
}

extern "C" int fg_mgm2_current(fg_mgm2_t h, int64_t *cycle, int32_t *finished) { return fg_current(h, cycle, finished); }

extern "C" int64_t fg_mgm2_launch_count(fg_mgm2_t h) { return fg_launch_count(h); }

// ---------------------------------------------------------------------------------------------
// Sharded MGM-2 (include/pydcop_b200.h: fg_mgm2_shard_*; kernels in csrc/mgm2_shard_kernels.cuh)
// ---------------------------------------------------------------------------------------------

struct fg_mgm2_shard {
  fg_mgm2_shard_plan_t plan;
  fg_mgm2_peer_plan_t peer;
  bool has_peer = false;
  uint64_t epoch = 0;
};

fg_mgm2::~fg_mgm2() { delete shard; }

// the phase kernel that produces exchange x, on the owned variables, then the pack of x
template <typename T>
static int mgm2_phase_t(fg_mgm2 *h, int x, cudaStream_t st) {
  fg_launcher launch(h, st);
  mgm2s_phase<T>(h->d, h->dev_classes, h->shard->plan, x, h->cycle, launch);
  CUDA_TRY(h, cudaGetLastError());
  if (x == MGM2X_VALUES) ++h->cycle;
  return FG_OK;
}

// NVLink transport of one exchange: every thread stores one 4-byte word of a peer's block into the peer's receive
// buffer; the last block to finish releases `epoch` to every peer (the ordering argument of csrc/peer_sync.cuh)
struct Mgm2Blocks {
  int n;
  int64_t word0[FG_MAX_PEERS + 1];      // prefix sums of the blocks' words
  const uint32_t *src[FG_MAX_PEERS];
  uint32_t *dst[FG_MAX_PEERS];
};

__global__ void __launch_bounds__(256) k_mgm2x_push(Mgm2Blocks b, uint32_t *__restrict__ counter, PeerSlots ps,
                                                    uint64_t epoch) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < b.word0[b.n]) {
    int k = 0;
    while (b.word0[k + 1] <= t) ++k;
    const int64_t w = t - b.word0[k];
    b.dst[k][w] = b.src[k][w];
  }
  __threadfence_system();   // my stores are ordered before the release below
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(counter, 1u);
    if (prev == gridDim.x - 1) {
      *counter = 0;          // ready for the next launch (stream-ordered)
      peer_release_all(ps, epoch);
    }
  }
}

template <typename T>
static int mgm2_push(fg_mgm2 *h, int x, cudaStream_t st) {
  fg_mgm2_shard *s = h->shard;
  const fg_mgm2_peer_plan_t &pp = s->peer;
  const int wpe = (int)(sizeof(T) / 4);
  Mgm2Blocks b;
  b.n = pp.n_blocks[x];
  b.word0[0] = 0;
  for (int k = 0; k < b.n; ++k) {
    b.src[k] = (const uint32_t *)((const T *)s->plan.x[x].dev_send_buf + pp.src[x][k]);
    b.dst[k] = (uint32_t *)(uintptr_t)pp.dst[x][k];
    b.word0[k + 1] = b.word0[k] + pp.n_elems[x][k] * wpe;
  }
  const int64_t words = b.word0[b.n];
  const unsigned blocks = (unsigned)(words > 0 ? (words + 255) / 256 : 1);
  k_mgm2x_push<<<blocks, 256, 0, st>>>(b, pp.dev_counter, peer_slots_of(pp.sync), s->epoch + 1);
  ++h->launches;
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

template <typename T>
static int mgm2_shard_cycle_t(fg_mgm2 *h, cudaStream_t st) {
  fg_mgm2_shard *s = h->shard;
  for (int x = 0; x < MGM2X_N; ++x) {
    int rc = mgm2_phase_t<T>(h, x, st);
    if (rc != FG_OK) return rc;
    if (s->peer.sync.n_peers) {
      rc = mgm2_push<T>(h, x, st);
      if (rc == FG_OK) rc = peer_wait_launch(s->peer.sync, s->epoch + 1, st, h->launches);
      if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push / wait launch failed"); return rc; }
      ++s->epoch;
    }
    fg_launcher launch(h, st);
    mgm2x_unpack<T>(h->d, s->plan, x, launch);
  }
  CUDA_TRY(h, cudaGetLastError());
  return FG_OK;
}

template <typename T>
static int mgm2_preload() {
  cudaFuncAttributes a;
  const void *fns[] = {(const void *)k_mgm2s_value<T>, (const void *)k_mgm2s_answer<T>, (const void *)k_mgm2s_commit<T>,
                       (const void *)k_mgm2s_gain<T>,  (const void *)k_mgm2s_go<T>,     (const void *)k_mgm2x_pack<T>,
                       (const void *)k_mgm2x_unpack<T>, (const void *)k_mgm2x_push,     (const void *)k_peer_wait};
  for (const void *f : fns)
    if (cudaFuncGetAttributes(&a, f) != cudaSuccess) { cudaGetLastError(); return FG_ERR_CUDA; }
  return FG_OK;
}

static int mgm2_xfer_check(const fg_mgm2_xfer_t &x) {
  if (x.n_send < 0 || x.n_recv < 0) return FG_ERR_ARG;
  if (x.n_send && (!x.dev_send_var || !x.dev_send_off || !x.dev_send_buf)) return FG_ERR_ARG;
  if (x.n_recv && (!x.dev_recv_var || !x.dev_recv_off || !x.dev_recv_buf)) return FG_ERR_ARG;
  return FG_OK;
}

extern "C" int fg_mgm2_shard_attach(fg_mgm2_t h, const fg_mgm2_shard_plan_t *plan, const fg_mgm2_peer_plan_t *peer) {
  if (!h || !plan) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (h->d.n_vars && (!plan->dev_ghost || !plan->dev_owner_rank || !plan->dev_owner_local)) {
    snprintf(h->err, sizeof(h->err), "shard plan: missing ghost mask or owner arrays");
    return FG_ERR_ARG;
  }
  for (int x = 0; x < MGM2X_N; ++x) {
    if (mgm2_xfer_check(plan->x[x]) != FG_OK) {
      snprintf(h->err, sizeof(h->err), "shard plan: exchange %d has a missing array or a negative count", x);
      return FG_ERR_ARG;
    }
  }
  if (plan->x[MGM2X_OFFERS].n_send && !plan->dev_send_peer) {
    snprintf(h->err, sizeof(h->err), "shard plan: missing dev_send_peer");
    return FG_ERR_ARG;
  }
  if (peer) {
    if (peer_sync_check(&peer->sync) != FG_OK || (peer->sync.n_peers && !peer->dev_counter)) {
      snprintf(h->err, sizeof(h->err), "invalid peer plan");
      return FG_ERR_ARG;
    }
    const int64_t es = h->d.precision == FG_F64 ? 8 : 4;
    for (int x = 0; x < MGM2X_N; ++x) {
      if (peer->n_blocks[x] < 0 || peer->n_blocks[x] > FG_MAX_PEERS) {
        snprintf(h->err, sizeof(h->err), "peer plan: exchange %d has %d blocks", x, peer->n_blocks[x]);
        return FG_ERR_ARG;
      }
      for (int k = 0; k < peer->n_blocks[x]; ++k) {
        if (peer->src[x][k] < 0 || peer->n_elems[x][k] < 0 || (peer->n_elems[x][k] && !peer->dst[x][k]) ||
            peer->dst[x][k] % (uint64_t)es) {
          snprintf(h->err, sizeof(h->err), "peer plan: exchange %d block %d is malformed", x, k);
          return FG_ERR_ARG;
        }
      }
    }
  }
  if (peer) {
    // Load every kernel of the device-side cycle now: with lazy module loading, the first launch of a kernel may wait
    // for the device to go idle, which never happens while this rank's barrier wait spins for a peer driven by the same
    // host thread (several shards in one process).
    const int rc = h->d.precision == FG_F64 ? mgm2_preload<double>() : mgm2_preload<float>();
    if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "cannot load the sharded MGM-2 kernels"); return rc; }
  }
  if (!h->shard) h->shard = new (std::nothrow) fg_mgm2_shard();
  if (!h->shard) { snprintf(h->err, sizeof(h->err), "out of host memory"); return FG_ERR_ARG; }
  h->shard->plan = *plan;
  h->shard->has_peer = peer != nullptr;
  if (peer) h->shard->peer = *peer;
  else h->shard->peer = fg_mgm2_peer_plan_t{};
  return FG_OK;
}

template <typename T>
static int mgm2_shard_init_t(fg_mgm2 *h, cudaStream_t st) {
  fg_launcher launch(h, st);
  mgm2s_init<T>(h->d, h->dev_classes, h->shard->plan, launch);
  CUDA_TRY(h, cudaGetLastError());
  h->cycle = 0;
  return FG_OK;
}

extern "C" int fg_mgm2_shard_init(fg_mgm2_t h, void *stream) {
  if (!h || !h->shard) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  return h->d.precision == FG_F64 ? mgm2_shard_init_t<double>(h, st) : mgm2_shard_init_t<float>(h, st);
}

extern "C" int fg_mgm2_shard_phase(fg_mgm2_t h, int32_t x, void *stream) {
  if (!h || !h->shard || x < 0 || x >= MGM2X_N) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  return h->d.precision == FG_F64 ? mgm2_phase_t<double>(h, x, st) : mgm2_phase_t<float>(h, x, st);
}

extern "C" int fg_mgm2_shard_unpack(fg_mgm2_t h, int32_t x, void *stream) {
  if (!h || !h->shard || x < 0 || x >= MGM2X_N) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  fg_launcher launch(h, (cudaStream_t)stream);
  if (h->d.precision == FG_F64) mgm2x_unpack<double>(h->d, h->shard->plan, x, launch);
  else mgm2x_unpack<float>(h->d, h->shard->plan, x, launch);
  CUDA_TRY(h, cudaGetLastError());
  return FG_OK;
}

extern "C" int fg_mgm2_shard_step(fg_mgm2_t h, int32_t n_cycles, void *stream) {
  if (!h || !h->shard || !h->shard->has_peer) return FG_ERR_ARG;
  return fg_step(h, n_cycles, stream, mgm2_shard_cycle_t<float>, mgm2_shard_cycle_t<double>);
}
