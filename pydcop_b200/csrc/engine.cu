// C-ABI of the pydcop_b200 engine (include/pydcop_b200.h): handle management and kernel launch
// sequencing.  No torch, no host-side arithmetic on messages, no CPU fallback.
#include <cstring>
#include <type_traits>

#include "handle.cuh"
#include "dsa_generic.cuh"
#include "maxsum_generic.cuh"
#include "maxsum_fast.cuh"
#include "maxsum_warp.cuh"
#include "maxsum_tiled_rt.cuh"
#include "selftest.cuh"
#include "dsa_fast.cuh"
#include "dsa_cached.cuh"
#include "peer_sync.cuh"

namespace {

template <typename T> constexpr size_t tsize() { return sizeof(T); }
inline size_t prec_size(int precision) { return precision == FG_F64 ? 8 : 4; }
inline unsigned blocks_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace

struct fg_maxsum : fg_handle_base {   // dev_classes unused: the plans own their device tables
  cudaStream_t side_stream = nullptr;   // variable side runs here, concurrently with the factor side
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  fg_maxsum_desc_t d;
  std::vector<fg_varclass_t> varclasses;
  MaxSumFastPlan fast;
  MaxSumWarpPlan warp;   // warp-autonomous kernels (round 2) over the same classes
  TiledRtPlan tiled_rt;  // factor classes of other shapes on the runtime-dimension tiled kernel (maxsum_tiled_rt.cuh)
  bool fast_first = true;   // tiled kernels in cycle 1 as well (PYDCOP_B200_FAST_FIRST=0: generic kernels)
  int cur = 0;
  // multi-GPU: push plan + device-side barrier (fg_maxsum_shard_*)
  bool has_halo = false;
  bool split_push = true;   // r rows right behind the factor side, q rows on the side stream (PYDCOP_B200_PUSH_SPLIT=0: one push after the join)
  bool fused_push = false;  // boundary rows stored to the peers by the warp kernels themselves (fg_halo_plan_t::dev_edge_dst_r)
  bool chain_push = true;   // split mode: the q push waits for the r push, then releases the epoch AND waits for the peers'
                            // releases in its last block — no separate release / wait kernels (PYDCOP_B200_PUSH_CHAIN=0: off)
  bool chained_now = false; // the cycle being enqueued was closed inside phase 0
  cudaEvent_t ev_r = nullptr;
  // early q push (EXPERIMENT, PYDCOP_B200_PUSH_EARLY=1|2): the variable classes with a remote factor (FG_CLASS_BOUNDARY) are
  // launched first and their rows leave while the interior classes are still being computed.  Many back-to-back
  // enqueued cycles run slower with it, for a reason not understood yet, so it is off by default
  bool early_q = false;
  int early_mode = 1;   // 1: the q push follows the r push on the main stream; 2: on a third stream (PYDCOP_B200_PUSH_EARLY=2)
  cudaStream_t push_stream = nullptr;
  cudaEvent_t ev_vb = nullptr, ev_q = nullptr;
  fg_halo_plan_t halo;
  uint64_t epoch = 0;
  cudaEvent_t *prof = nullptr;   // fg_maxsum_shard_profile: 8 timing events recorded inside a cycle
};

struct fg_dsa : fg_handle_base {
  fg_dsa_desc_t d;
  int cur = 0;
  bool has_halo = false;
  fg_halo_plan_t halo;
  uint64_t epoch = 0;
};

extern "C" int fg_abi_version(void) { return FG_ABI_VERSION; }

extern "C" int fg_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// ---------------------------------------------------------------------------------------------
// MaxSum
// ---------------------------------------------------------------------------------------------
extern "C" int fg_maxsum_create(const fg_maxsum_desc_t *desc, fg_maxsum_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_maxsum *h = *out;
  if (desc->n_varclasses > 0 && desc->varclasses)
    h->varclasses.assign(desc->varclasses, desc->varclasses + desc->n_varclasses);
  h->d.varclasses = h->varclasses.data();
  int64_t covered = 0;
  for (auto &vc : h->varclasses) covered += vc.n_slots;
  if (covered != desc->n_edges) {
    snprintf(h->err, sizeof(h->err), "variable classes cover %lld slots, expected %d", (long long)covered, desc->n_edges);
    return FG_ERR_ARG;
  }
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_maxsum_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_unary), FG_FIELD(d, dev_dom_size),
                             FG_FIELD(d, dev_unary_off), FG_FIELD(d, dev_var_ptr), FG_FIELD(d, dev_var_qbase),
                             FG_FIELD(d, dev_slot_roff), FG_FIELD(d, dev_edge_qoff), FG_FIELD(d, dev_slot_roff32),
                             FG_FIELD(d, dev_edge_qoff32), FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_slot_var),
                             FG_FIELD(d, dev_init_value), FG_FIELD(d, dev_q[0]), FG_FIELD(d, dev_q[1]),
                             FG_FIELD(d, dev_r[0]), FG_FIELD(d, dev_r[1]), FG_FIELD(d, dev_q_valid),
                             FG_FIELD(d, dev_r_valid), FG_FIELD(d, dev_q_cnt), FG_FIELD(d, dev_r_cnt),
                             FG_FIELD(d, dev_q_sent), FG_FIELD(d, dev_r_sent), FG_FIELD(d, dev_value),
                             FG_FIELD(d, dev_value_cost)});
  if (rc != FG_OK) return rc;
  maxsum_fast_plan(h->d, h->classes, h->varclasses, h->fast);
  if (maxsum_warp_plan(h->d, h->varclasses, h->fast, h->warp) != FG_OK) {
    snprintf(h->err, sizeof(h->err), "tile descriptors of the variable side: %s", cudaGetErrorString(cudaGetLastError()));
    return FG_ERR_CUDA;
  }
  maxsum_warp_plan_f2v(h->d, h->classes, h->fast, h->warp);
  if (maxsum_warp_plan_tab8(h->d, h->classes, h->warp) != FG_OK) {
    snprintf(h->err, sizeof(h->err), "8-bit table copy of the factor side: %s", cudaGetErrorString(cudaGetLastError()));
    return FG_ERR_CUDA;
  }
  {
    std::vector<uint8_t> skip(h->classes.size(), 0);
    for (size_t i = 0; i < h->classes.size(); ++i) skip[i] = h->fast.f2v[i] || h->warp.f2v[i];
    if (tiled_rt_plan(h->d, h->classes, skip, !fg_fast_disabled() && !fg_env_is("PYDCOP_B200_TILED_RT", '0'), h->tiled_rt) != FG_OK) {
      snprintf(h->err, sizeof(h->err), "tile table of the runtime-dimension factor kernel: %s", cudaGetErrorString(cudaGetLastError()));
      return FG_ERR_CUDA;
    }
  }
  { const char *e = getenv("PYDCOP_B200_FAST_FIRST"); h->fast_first = !(e && e[0] == '0'); }
  if (!fg_env_int("PYDCOP_B200_SERIAL", 0)) {
    CUDA_TRY(h, cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
  }
  return FG_OK;
}

extern "C" int fg_maxsum_destroy(fg_maxsum_t h) {
  if (h) {
    fg_device_scope on(h);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->ev_r) cudaEventDestroy(h->ev_r);
    if (h->ev_vb) cudaEventDestroy(h->ev_vb);
    if (h->ev_q) cudaEventDestroy(h->ev_q);
    if (h->push_stream) cudaStreamDestroy(h->push_stream);
    if (h->side_stream) cudaStreamDestroy(h->side_stream);
    if (h->warp.dev_classes) cudaFree(h->warp.dev_classes);
    if (h->warp.tab8) cudaFree(h->warp.tab8);
    tiled_rt_free(h->tiled_rt);
  }
  delete h;
  return FG_OK;
}

extern "C" const char *fg_maxsum_last_error(fg_maxsum_t h) { return fg_last_error(h); }

template <typename T>
static int maxsum_init_t(fg_maxsum *h, cudaStream_t st) {
  const fg_maxsum_desc_t &d = h->d;
  const size_t mbq = (size_t)d.n_msg_q * sizeof(T), mbr = (size_t)d.n_msg_r * sizeof(T);
  for (int b = 0; b < 2; ++b) {
    if (mbq) CUDA_TRY(h, cudaMemsetAsync(d.dev_q[b], 0, mbq, st));
    if (mbr) CUDA_TRY(h, cudaMemsetAsync(d.dev_r[b], 0, mbr, st));
  }
  uint8_t *bytes[] = {d.dev_q_valid, d.dev_r_valid, d.dev_q_cnt, d.dev_r_cnt, d.dev_q_sent, d.dev_r_sent};
  for (uint8_t *p : bytes)
    if (p && d.n_edges) CUDA_TRY(h, cudaMemsetAsync(p, 0, (size_t)d.n_edges, st));
  VarSide g{d.dev_dom_size, d.dev_unary_off, d.dev_var_ptr, d.dev_var_qbase, d.dev_slot_roff, d.dev_slot_edge, d.dev_slot_var};
  if (d.n_vars) {
    k_v2f_start<T><<<blocks_for(d.n_vars, 128), 128, 0, st>>>(
        g, d.n_vars, (const T *)d.dev_unary, d.dev_init_value, (T *)d.dev_q[0], d.dev_q_valid,
        d.dev_q_sent, d.dev_value, (T *)d.dev_value_cost, d.mode_max, d.start_messages);
    ++h->launches;
  }
  for (const fg_class_t &c : h->classes) {
    bool posts = (c.arity == 1 && d.start_messages <= FG_START_LEAFS_VARS) || d.start_messages == FG_START_ALL;
    if (!posts || c.n_factors == 0 || (c.flags & FG_CLASS_GHOST)) continue;
    k_f2v_start<T><<<blocks_for((int64_t)c.n_factors * c.arity, 128), 128, 0, st>>>(
        c, (const T *)d.dev_tables, (T *)d.dev_r[0], d.dev_r_valid, d.dev_r_sent, d.mode_max);
    ++h->launches;
  }
  CUDA_TRY(h, cudaGetLastError());
  h->cur = 0;
  h->cycle = 0;
  return FG_OK;
}

extern "C" int fg_maxsum_init(fg_maxsum_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  return h->d.precision == FG_F64 ? maxsum_init_t<double>(h, st) : maxsum_init_t<float>(h, st);
}

// push_split: multi-GPU only — the boundary r rows leave right behind the factor side (main stream), the q
// rows right behind the variable side (side stream), each overlapping the other side's compute
template <typename T>
static int maxsum_compute_t(fg_maxsum *h, cudaStream_t st, bool push_split = false) {
  const fg_maxsum_desc_t &d = h->d;
  const int cur = h->cur, nxt = cur ^ 1;
  // The generic kernels of cycle 1 consult the validity arrays.  The buffers are zero-filled at init and
  // a never-sent message counts as zeros in every sum (maxsum.py:430-436, 656-661), so the tiled
  // kernels, which read every row, compute the same values in cycle 1 too (default; checked against the
  // generic kernels and the oracle by tests/test_gpu_zz_fast_first.py).
  const bool first = (h->cycle == 0) && !h->fast_first;
  const bool first_cycle = (h->cycle == 0);
  MaxSumParams p{d.mode_max, d.damp_vars, d.damp_factors, d.damping, 1.0 - d.damping, d.stability, nullptr, nullptr};
  const bool fused = push_split && h->fused_push && !first;   // the warp kernels store the boundary rows themselves
  if (fused) { p.edge_dst = h->halo.dev_edge_dst_r[nxt]; p.slot_dst = h->halo.dev_slot_dst_q[nxt]; }
  const T *q_cur = (const T *)d.dev_q[cur], *r_cur = (const T *)d.dev_r[cur];
  T *q_next = (T *)d.dev_q[nxt], *r_next = (T *)d.dev_r[nxt];
  // fork BEFORE anything of this cycle is enqueued, so the side stream only waits for the past
  cudaStream_t st_f = st;
  const bool fork = !first && h->side_stream != nullptr && d.n_edges > 0;
  if (fork) {
    CUDA_TRY(h, cudaEventRecord(h->ev_fork, st_f));
    CUDA_TRY(h, cudaStreamWaitEvent(h->side_stream, h->ev_fork, 0));
  }
  // factor -> variable
  for (size_t ci = 0; ci < h->classes.size(); ++ci) {
    const fg_class_t &c = h->classes[ci];
    if (c.n_factors == 0 || (c.flags & FG_CLASS_GHOST)) continue;
    if (!first && h->warp.f2v[ci]) {
      if (launch_f2v_warp_class<T>(h->warp, ci, c, d, q_cur, r_cur, r_next, p, st)) { ++h->launches; continue; }
      if (fused) {   // no other kernel stores boundary rows to the peers: never drop them silently
        snprintf(h->err, sizeof(h->err), "fused halo: no peer-store factor kernel for class %zu", ci);
        return FG_ERR_ARG;
      }
    }
    if (!first && maxsum_fast_f2v<T>(h->fast, (int)ci, c, d, q_cur, r_cur, r_next, p, st, h->launches)) continue;
    if (!first && h->tiled_rt.on[ci]) continue;   // below, one launch per arity
    const int64_t n = (int64_t)c.n_factors * c.arity;
    if (first)
      k_f2v_generic<T, 1><<<blocks_for(n, 128), 128, 0, st>>>(c, (const T *)d.dev_tables, q_cur, r_cur, r_next,
                                                             d.dev_edge_qoff, d.dev_q_valid, d.dev_r_cnt, d.dev_r_sent, p);
    else
      k_f2v_generic<T, 0><<<blocks_for(n, 128), 128, 0, st>>>(c, (const T *)d.dev_tables, q_cur, r_cur, r_next,
                                                             d.dev_edge_qoff, d.dev_q_valid, d.dev_r_cnt, d.dev_r_sent, p);
    ++h->launches;
  }
  if (!first) h->launches += dispatch_f2v_tiled_rt<T>(h->tiled_rt, d, q_cur, r_cur, r_next, p, st);
  if (h->prof) cudaEventRecord(h->prof[1], st);
  if (push_split && !fused && h->halo.n_r > 0) {
    int rc = halo_push_launch(h->halo, r_next, q_next, nxt, h->halo.n_r, 0, 0, 0, st, h->launches);
    if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push (r rows) failed"); return rc; }
  }
  const bool chain = push_split && h->chain_push && fork;   // the side stream's last launch closes the cycle
  h->chained_now = chain;
  const bool early = chain && h->early_q && !fused;         // q rows of the boundary classes leave before the interior ones are done
  const int early_mode = early ? h->early_mode : 0;
  if (chain && early_mode != 1) CUDA_TRY(h, cudaEventRecord(h->ev_r, st));   // mode 1: recorded behind the early q push
  bool early_done = false;
  // enqueue the q push behind the boundary classes (recorded on the side stream `sv`): on the main stream after the r
  // push (mode 1) or on the push stream (mode 2)
  auto early_push = [&](cudaStream_t sv) -> int {
    if (cudaEventRecord(h->ev_vb, sv) != cudaSuccess) return FG_ERR_CUDA;
    cudaStream_t ps = early_mode == 2 ? h->push_stream : st_f;
    if (cudaStreamWaitEvent(ps, h->ev_vb, 0) != cudaSuccess) return FG_ERR_CUDA;
    int rc = halo_push_launch(h->halo, r_next, q_next, nxt, 0, h->halo.n_q, 0, 0, ps, h->launches);
    if (rc != FG_OK) return rc;
    if (cudaEventRecord(early_mode == 2 ? h->ev_q : h->ev_r, ps) != cudaSuccess) return FG_ERR_CUDA;
    early_done = true;
    return FG_OK;
  };
  if (h->prof) cudaEventRecord(h->prof[2], st);
  // variable -> factor (+ value selection).  Both sides only READ the current buffers and WRITE
  // disjoint next buffers (Jacobi), so from cycle 2 on the variable side runs on a second stream,
  // concurrently with the factor side: one is HBM-streaming, the other gather/latency-bound.
  if (fork) st = h->side_stream;
  if (d.n_edges) {
    VarSide g{d.dev_dom_size, d.dev_unary_off, d.dev_var_ptr, d.dev_var_qbase, d.dev_slot_roff, d.dev_slot_edge, d.dev_slot_var};
    if (first) {
      for (const fg_varclass_t &vc : h->varclasses) {
        if (vc.n_slots == 0 || (vc.flags & FG_CLASS_GHOST)) continue;
        k_v2f_generic<T, 1><<<blocks_for(vc.n_slots, 128), 128, 0, st>>>(
            g, vc.first_slot, vc.n_slots, (const T *)d.dev_unary, r_cur, q_cur, q_next, d.dev_r_valid, d.dev_q_cnt,
            d.dev_q_sent, d.dev_value, (T *)d.dev_value_cost, p);
        ++h->launches;
      }
    } else {
      if (h->warp.v2f_on) {
        bool in_boundary = true;
        for (const WTileRange &rg : h->warp.v2f) {
          if (early && in_boundary && !rg.boundary) {   // every boundary class is enqueued: their q rows may leave now
            in_boundary = false;
            int rc = early_push(st);
            if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push (q rows, early) failed"); return rc; }
          }
          if (dispatch_v2f_warp<T>(h->warp.dev_classes, rg, d, r_cur, q_cur, q_next, p, st)) ++h->launches;
        }
        if (early && !early_done) {   // no interior range followed: push behind the last boundary launch
          int rc = early_push(st);
          if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push (q rows, early) failed"); return rc; }
        }
      } else {
        for (size_t li = 0; li < h->fast.v2f.size(); ++li)
          if (dispatch_v2f_classes<T>(h->fast.v2f_dom[li], h->fast.v2f[li], d, r_cur, q_cur, q_next, p, st)) ++h->launches;
      }
      // classes without a tiled kernel: one launch per RUN of adjacent slot ranges (the kernel works per slot)
      for (size_t k = 0; k < h->fast.slow_varclasses.size();) {
        const fg_varclass_t &vc = h->varclasses[h->fast.slow_varclasses[k]];
        int64_t begin = vc.first_slot, n = vc.n_slots;
        for (++k; k < h->fast.slow_varclasses.size(); ++k) {
          const fg_varclass_t &nx = h->varclasses[h->fast.slow_varclasses[k]];
          if (nx.first_slot != begin + n) break;
          n += nx.n_slots;
        }
        k_v2f_generic<T, 0><<<blocks_for(n, 128), 128, 0, st>>>(
            g, (int)begin, (int)n, (const T *)d.dev_unary, r_cur, q_cur, q_next, d.dev_r_valid, d.dev_q_cnt,
            d.dev_q_sent, d.dev_value, (T *)d.dev_value_cost, p);
        ++h->launches;
      }
    }
  }
  if (h->prof) cudaEventRecord(h->prof[3], st);
  if (chain && early_mode == 1 && !early_done) CUDA_TRY(h, cudaEventRecord(h->ev_r, st_f));   // (no warp launch ran)
  if (chain) {   // everything this rank sends in this cycle is on its way once the r push is done as well
    CUDA_TRY(h, cudaStreamWaitEvent(st, h->ev_r, 0));
    if (early_done && early_mode == 2) CUDA_TRY(h, cudaStreamWaitEvent(st, h->ev_q, 0));
    int rc = halo_push_launch(h->halo, r_next, q_next, nxt, 0, (fused || early_done) ? 0 : h->halo.n_q, 1, h->epoch + 1, st, h->launches, 1);
    if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push (q rows, release, wait) failed"); return rc; }
  } else if (push_split && !fused && h->halo.n_q > 0) {  // q list only: the kernel indexes rows >= n_r as q rows
    int rc = halo_push_launch(h->halo, r_next, q_next, nxt, 0, h->halo.n_q, 0, 0, st, h->launches);
    if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push (q rows) failed"); return rc; }
  }
  if (h->prof) cudaEventRecord(h->prof[4], st);
  if (fork) {
    CUDA_TRY(h, cudaEventRecord(h->ev_join, h->side_stream));
    CUDA_TRY(h, cudaStreamWaitEvent(st_f, h->ev_join, 0));
    st = st_f;
  }
  if (first_cycle && d.n_edges) {  // every edge has posted in cycle 1: all messages are valid from now on
    CUDA_TRY(h, cudaMemsetAsync(d.dev_q_valid, 1, (size_t)d.n_edges, st));
    CUDA_TRY(h, cudaMemsetAsync(d.dev_r_valid, 1, (size_t)d.n_edges, st));
  }
  CUDA_TRY(h, cudaGetLastError());
  return FG_OK;
}

extern "C" int fg_maxsum_cycle_compute(fg_maxsum_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  return h->d.precision == FG_F64 ? maxsum_compute_t<double>(h, st) : maxsum_compute_t<float>(h, st);
}

extern "C" int fg_maxsum_cycle_commit(fg_maxsum_t h) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  h->cur ^= 1;
  ++h->cycle;
  return FG_OK;
}

extern "C" int fg_maxsum_step(fg_maxsum_t h, int32_t n_cycles, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  for (int i = 0; i < n_cycles; ++i) {
    int rc = fg_maxsum_cycle_compute(h, stream);
    if (rc != FG_OK) return rc;
    fg_maxsum_cycle_commit(h);
  }
  return FG_OK;
}

extern "C" int fg_maxsum_current(fg_maxsum_t h, int32_t *buf_index, int64_t *cycle) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (buf_index) *buf_index = h->cur;
  if (cycle) *cycle = h->cycle;
  return FG_OK;
}

extern "C" int64_t fg_maxsum_launch_count(fg_maxsum_t h) { return fg_launch_count(h); }

extern "C" int fg_maxsum_kernel_plan(fg_maxsum_t h, int32_t *family, int32_t n_classes) {
  if (!h || !family || n_classes != (int32_t)h->classes.size()) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  for (int32_t i = 0; i < n_classes; ++i) {
    const fg_class_t &c = h->classes[i];
    family[i] = (c.flags & FG_CLASS_GHOST) ? -1 : h->warp.f2v[i] ? FG_KERNEL_WARP : h->fast.f2v[i] ? FG_KERNEL_PIPE
              : h->tiled_rt.on[i] ? FG_KERNEL_TILED_RT : FG_KERNEL_GENERIC;
  }
  return FG_OK;
}

extern "C" int fg_maxsum_table_width(fg_maxsum_t h, int32_t *bytes, int32_t n_classes) {
  if (!h || !bytes || n_classes != (int32_t)h->classes.size()) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  const int32_t full = (int32_t)prec_size(h->d.precision);
  for (int32_t i = 0; i < n_classes; ++i)
    bytes[i] = (!h->warp.tab8_base.empty() && h->warp.tab8_base[i] >= 0) ? 1 : full;
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------
// multi-GPU cycle on the device: compute -> peer push (+ release) -> wait -> commit
// ---------------------------------------------------------------------------------------------
static int halo_plan_check(const fg_halo_plan_t *p) {
  if (!p || p->dom < 1 || (p->elem_bytes != 4 && p->elem_bytes != 8) || p->n_r < 0 || p->n_q < 0) return FG_ERR_ARG;
  if (p->n_r && (!p->dev_src_r_off || !p->dev_dst_r[0] || !p->dev_dst_r[1])) return FG_ERR_ARG;
  if (p->n_q && (!p->dev_src_q_off || !p->dev_dst_q[0] || !p->dev_dst_q[1])) return FG_ERR_ARG;
  if (!p->dev_counter) return FG_ERR_ARG;
  return peer_sync_check(&p->sync);
}

extern "C" int fg_peer_signal(const fg_peer_sync_t *ps, uint64_t epoch, void *stream) {
  if (peer_sync_check(ps) != FG_OK) return FG_ERR_ARG;
  if (!ps->n_peers) return FG_OK;
  k_peer_signal<<<1, 32, 0, (cudaStream_t)stream>>>(peer_slots_of(*ps), epoch);
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

extern "C" int fg_peer_wait(const fg_peer_sync_t *ps, uint64_t epoch, void *stream) {
  if (peer_sync_check(ps) != FG_OK) return FG_ERR_ARG;
  int64_t n = 0;
  return peer_wait_launch(*ps, epoch, (cudaStream_t)stream, n);
}

extern "C" int fg_maxsum_shard_attach(fg_maxsum_t h, const fg_halo_plan_t *plan) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (halo_plan_check(plan) != FG_OK) { snprintf(h->err, sizeof(h->err), "invalid halo plan"); return FG_ERR_ARG; }
  if ((size_t)plan->elem_bytes != prec_size(h->d.precision)) { snprintf(h->err, sizeof(h->err), "halo plan element size"); return FG_ERR_ARG; }
  h->halo = *plan;
  h->has_halo = true;
  h->epoch = 0;
  { const char *e = getenv("PYDCOP_B200_PUSH_SPLIT"); h->split_push = !(e && e[0] == '0'); }   // default on
  // fused halo: every class that produces rows must run on a warp kernel (they carry the peer stores)
  bool all_warp = plan->dev_edge_dst_r[0] && plan->dev_edge_dst_r[1] && plan->dev_slot_dst_q[0] && plan->dev_slot_dst_q[1] &&
                  h->warp.v2f_on && h->fast.slow_varclasses.empty() && fg_env_is("PYDCOP_B200_PUSH_FUSED", '1') &&
                  fg_env_int("PYDCOP_B200_F2VW_NS", 2) == 2 && fg_env_int("PYDCOP_B200_V2FW_NS", 2) == 2;   // opt-in: the stores stall the
                  // compute kernels more as the cut grows
  for (size_t i = 0; all_warp && i < h->classes.size(); ++i)
    if (h->classes[i].n_factors && !(h->classes[i].flags & FG_CLASS_GHOST) && !h->warp.f2v[i]) all_warp = false;
  h->fused_push = all_warp;
  h->chain_push = !fg_env_is("PYDCOP_B200_PUSH_CHAIN", '0') && h->side_stream != nullptr;
  if (h->chain_push && !h->ev_r) CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_r, cudaEventDisableTiming));
  // every boundary class must be in one of the warp launches (they come first in the plan) for its rows to leave early
  bool early = h->chain_push && h->split_push && !h->fused_push && h->warp.v2f_on && plan->n_q > 0 &&
               (fg_env_is("PYDCOP_B200_PUSH_EARLY", '1') || fg_env_is("PYDCOP_B200_PUSH_EARLY", '2'));   // opt-in, see DESIGN.md §6
  h->early_mode = fg_env_is("PYDCOP_B200_PUSH_EARLY", '2') ? 2 : 1;
  bool any_boundary = false;
  for (const fg_varclass_t &vc : h->varclasses) {
    if (!(vc.flags & FG_CLASS_BOUNDARY) || (vc.flags & FG_CLASS_GHOST) || vc.n_slots == 0) continue;
    any_boundary = true;
    if (!(fg_fast_dom(vc.dom) && vc.degree >= 1 && vc.degree <= 32)) early = false;
  }
  h->early_q = early && any_boundary;
  if (h->early_q && !h->push_stream) {
    CUDA_TRY(h, cudaStreamCreateWithFlags(&h->push_stream, cudaStreamNonBlocking));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_vb, cudaEventDisableTiming));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_q, cudaEventDisableTiming));
  }
  return FG_OK;
}

extern "C" int fg_maxsum_shard_fused(fg_maxsum_t h) { return (h && h->has_halo && h->fused_push) ? 1 : 0; }

extern "C" int fg_maxsum_shard_phase(fg_maxsum_t h, int32_t phase, void *stream) {
  if (!h || !h->has_halo) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  const int nxt = h->cur ^ 1;
  switch (phase) {
    case 0: {
      const bool split = (h->split_push || h->fused_push) && h->cycle > 0;
      return h->d.precision == FG_F64 ? maxsum_compute_t<double>(h, st, split) : maxsum_compute_t<float>(h, st, split);
    }
    case 1: {
      if (h->chained_now) return FG_OK;   // released (and waited) by the q push of phase 0
      const bool split = (h->split_push || h->fused_push) && h->cycle > 0;   // rows already on their way: release only
      return halo_push_launch(h->halo, h->d.dev_r[nxt], h->d.dev_q[nxt], nxt, split ? 0 : h->halo.n_r,
                              split ? 0 : h->halo.n_q, 1, h->epoch + 1, st, h->launches);
    }
    case 2: return h->chained_now ? FG_OK : peer_wait_launch(h->halo.sync, h->epoch + 1, st, h->launches);
    case 3: ++h->epoch; h->chained_now = false; return fg_maxsum_cycle_commit(h);
  }
  return FG_ERR_ARG;
}

// Device-time profile of a sharded cycle (diagnostics; bench.py's `breakdown`): n_cycles cycles with timing
// events inside, averaged, in microseconds:
//   out[0] factor side   out[1] push of the r rows (split mode)   out[2] variable side (from the cycle start)
//   out[3] push of the q rows (split mode)   out[4] join -> push (+ release) done   out[5] wait   out[6] whole cycle
extern "C" int fg_maxsum_shard_profile(fg_maxsum_t h, int32_t n_cycles, void *stream, double *out_us) {
  if (!h || !h->has_halo || !out_us || n_cycles < 1) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  cudaEvent_t ev[8];
  for (auto &e : ev) CUDA_TRY(h, cudaEventCreate(&e));
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};
  int rc = FG_OK;
  for (int i = 0; i < n_cycles && rc == FG_OK; ++i) {
    cudaEventRecord(ev[0], st);
    h->prof = ev;
    rc = fg_maxsum_shard_phase(h, 0, stream);
    h->prof = nullptr;
    cudaEventRecord(ev[5], st);
    if (rc == FG_OK) rc = fg_maxsum_shard_phase(h, 1, stream);
    cudaEventRecord(ev[6], st);
    if (rc == FG_OK) rc = fg_maxsum_shard_phase(h, 2, stream);
    cudaEventRecord(ev[7], st);
    if (rc == FG_OK) rc = fg_maxsum_shard_phase(h, 3, stream);
    if (cudaStreamSynchronize(st) != cudaSuccess) rc = FG_ERR_CUDA;
    if (h->side_stream) cudaStreamSynchronize(h->side_stream);
    if (rc != FG_OK) break;
    auto ms = [&](int a, int b) { float t = 0; cudaEventElapsedTime(&t, ev[a], ev[b]); return (double)t * 1e3; };
    acc[0] += ms(0, 1); acc[1] += ms(1, 2); acc[2] += ms(0, 3); acc[3] += ms(3, 4);
    acc[4] += ms(5, 6); acc[5] += ms(6, 7); acc[6] += ms(0, 7);
  }
  for (auto &e : ev) cudaEventDestroy(e);
  cudaGetLastError();
  for (int k = 0; k < 7; ++k) out_us[k] = acc[k] / n_cycles;
  return rc;
}

extern "C" int fg_maxsum_shard_step(fg_maxsum_t h, int32_t n_cycles, void *stream) {
  if (!h || !h->has_halo) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  for (int i = 0; i < n_cycles; ++i)
    for (int ph = 0; ph < 4; ++ph) {
      int rc = fg_maxsum_shard_phase(h, ph, stream);
      if (rc != FG_OK) return rc;
    }
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------
// halo pack / unpack: one warp per boundary row
// ---------------------------------------------------------------------------------------------
template <typename T, bool PACK>
__global__ void k_halo_rows(T *__restrict__ arr, T *__restrict__ packed, const int64_t *__restrict__ row_off,
                            const int64_t *__restrict__ packed_off, const int32_t *__restrict__ row_len,
                            int64_t n_rows) {
  int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (w >= n_rows) return;
  const int64_t a = row_off[w], b = packed_off[w];
  const int n = row_len[w];
  for (int x = lane; x < n; x += 32) {
    if (PACK) packed[b + x] = arr[a + x];
    else arr[a + x] = packed[b + x];
  }
}

template <bool PACK>
static int halo_rows(int32_t precision, void *arr, void *packed, const int64_t *row_off,
                     const int64_t *packed_off, const int32_t *row_len, int64_t n_rows, void *stream) {
  if (n_rows <= 0) return FG_OK;
  if (!fg_on_current_device(arr) || !fg_on_current_device(packed)) return FG_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned blocks = blocks_for(n_rows * 32, 256);
  if (precision == FG_F64)
    k_halo_rows<double, PACK><<<blocks, 256, 0, st>>>((double *)arr, (double *)packed, row_off, packed_off, row_len, n_rows);
  else
    k_halo_rows<float, PACK><<<blocks, 256, 0, st>>>((float *)arr, (float *)packed, row_off, packed_off, row_len, n_rows);
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

extern "C" int fg_halo_pack(int32_t precision, const void *dev_src, void *dev_packed, const int64_t *dev_row_off,
                            const int64_t *dev_packed_off, const int32_t *dev_row_len, int64_t n_rows, void *stream) {
  return halo_rows<true>(precision, const_cast<void *>(dev_src), dev_packed, dev_row_off, dev_packed_off, dev_row_len, n_rows, stream);
}

extern "C" int fg_halo_unpack(int32_t precision, void *dev_dst, const void *dev_packed, const int64_t *dev_row_off,
                              const int64_t *dev_packed_off, const int32_t *dev_row_len, int64_t n_rows, void *stream) {
  return halo_rows<false>(precision, dev_dst, const_cast<void *>(dev_packed), dev_row_off, dev_packed_off, dev_row_len, n_rows, stream);
}

struct HaloPeers {
  int n;
  int64_t r_start[17], q_start[17], base[16];
};

// one thread per (row, 4/8/16-byte piece): r rows first, then q rows
template <int PB, bool PACK>
__global__ void __launch_bounds__(256)
k_halo_rows_uniform(unsigned char *__restrict__ arr_r, unsigned char *__restrict__ arr_q,
                    unsigned char *__restrict__ packed, const int64_t *__restrict__ off_r,
                    const int64_t *__restrict__ off_q, int64_t n_r, int64_t n_q, int row_bytes, int elem,
                    HaloPeers hp) {
  const int ppr = row_bytes / PB;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = t / ppr;
  const int piece = (int)(t - row * ppr);
  if (row >= n_r + n_q) return;
  const bool is_q = row >= n_r;
  const int64_t i = is_q ? row - n_r : row;
  const int64_t *start = is_q ? hp.q_start : hp.r_start;
  int p = 0;
#pragma unroll 1
  while (p + 1 < hp.n && i >= start[p + 1]) ++p;
  int64_t pk = hp.base[p] * elem + (i - start[p]) * row_bytes;            // byte offset in the packed buffer
  if (is_q) pk += (hp.r_start[p + 1] - hp.r_start[p]) * (int64_t)row_bytes;  // after the peer's r rows
  unsigned char *a = (is_q ? arr_q : arr_r) + (is_q ? off_q[i] : off_r[i]) * elem + piece * PB;
  unsigned char *b = packed + pk + piece * PB;
  using V = typename std::conditional<PB == 16, uint4, typename std::conditional<PB == 8, uint2, uint32_t>::type>::type;
  if (PACK) *reinterpret_cast<V *>(b) = *reinterpret_cast<const V *>(a);
  else *reinterpret_cast<V *>(a) = *reinterpret_cast<const V *>(b);
}

extern "C" int fg_halo_rows_uniform(int32_t precision, int32_t pack, void *dev_r, void *dev_q, void *dev_packed,
                                    const int64_t *dev_row_off_r, const int64_t *dev_row_off_q, int64_t n_r, int64_t n_q,
                                    int32_t dom, int32_t n_peers, const int64_t *peer_r_start, const int64_t *peer_q_start,
                                    const int64_t *peer_base, void *stream) {
  if (n_r + n_q <= 0) return FG_OK;
  if (n_peers < 1 || n_peers > 16 || dom < 1) return FG_ERR_ARG;
  if (!fg_on_current_device(dev_packed)) return FG_ERR_ARG;
  HaloPeers hp;
  hp.n = n_peers;
  for (int i = 0; i <= n_peers; ++i) { hp.r_start[i] = peer_r_start[i]; hp.q_start[i] = peer_q_start[i]; }
  for (int i = 0; i < n_peers; ++i) hp.base[i] = peer_base[i];
  const int elem = precision == FG_F64 ? 8 : 4;
  const int row_bytes = dom * elem;
  const int pb = (row_bytes % 16 == 0) ? 16 : ((row_bytes % 8 == 0) ? 8 : 4);
  const int64_t threads = (n_r + n_q) * (row_bytes / pb);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char *r = (unsigned char *)dev_r, *q = (unsigned char *)dev_q, *pk = (unsigned char *)dev_packed;
  const unsigned blocks = blocks_for(threads, 256);
#define FG_HALO_LAUNCH(PB_)                                                                                                    \
  if (pack) k_halo_rows_uniform<PB_, true><<<blocks, 256, 0, st>>>(r, q, pk, dev_row_off_r, dev_row_off_q, n_r, n_q, row_bytes, elem, hp); \
  else k_halo_rows_uniform<PB_, false><<<blocks, 256, 0, st>>>(r, q, pk, dev_row_off_r, dev_row_off_q, n_r, n_q, row_bytes, elem, hp);
  if (pb == 16) { FG_HALO_LAUNCH(16) } else if (pb == 8) { FG_HALO_LAUNCH(8) } else { FG_HALO_LAUNCH(4) }
#undef FG_HALO_LAUNCH
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

// rows -> absolute (peer) addresses: stores travel over NVLink
template <int PB>
__global__ void __launch_bounds__(256)
k_halo_push(const unsigned char *__restrict__ arr_r, const unsigned char *__restrict__ arr_q,
            const int64_t *__restrict__ off_r, const int64_t *__restrict__ off_q,
            const int64_t *__restrict__ dst_r, const int64_t *__restrict__ dst_q, int64_t n_r, int64_t n_q,
            int row_bytes, int elem) {
  const int ppr = row_bytes / PB;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = t / ppr;
  const int piece = (int)(t - row * ppr);
  if (row >= n_r + n_q) return;
  const bool is_q = row >= n_r;
  const int64_t i = is_q ? row - n_r : row;
  const unsigned char *a = (is_q ? arr_q : arr_r) + (is_q ? off_q[i] : off_r[i]) * elem + piece * PB;
  unsigned char *b = reinterpret_cast<unsigned char *>(is_q ? dst_q[i] : dst_r[i]) + piece * PB;
  using V = typename std::conditional<PB == 16, uint4, typename std::conditional<PB == 8, uint2, uint32_t>::type>::type;
  *reinterpret_cast<V *>(b) = *reinterpret_cast<const V *>(a);
}

extern "C" int fg_enable_peer_access(int32_t peer_device) {
  int cur = 0, can = 0;
  if (cudaGetDevice(&cur) != cudaSuccess) return FG_ERR_CUDA;
  if (cur == peer_device) return FG_OK;
  if (cudaDeviceCanAccessPeer(&can, cur, peer_device) != cudaSuccess || !can) { cudaGetLastError(); return FG_ERR_UNSUPPORTED; }
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return FG_OK; }
  return e == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

// cuMemGetAddressRange through dlopen: the library must load on boxes without a driver
#include <dlfcn.h>
extern "C" int fg_ipc_export(const void *dev_ptr, unsigned char handle_out[64], int64_t *offset_out) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  typedef int (*range_fn)(unsigned long long *, size_t *, unsigned long long);
  static range_fn get_range = nullptr;
  if (!get_range) {
    void *lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) return FG_ERR_UNSUPPORTED;
    get_range = (range_fn)dlsym(lib, "cuMemGetAddressRange_v2");
    if (!get_range) return FG_ERR_UNSUPPORTED;
  }
  unsigned long long base = 0;
  size_t size = 0;
  if (get_range(&base, &size, (unsigned long long)dev_ptr) != 0) return FG_ERR_CUDA;
  cudaIpcMemHandle_t h;
  if (cudaIpcGetMemHandle(&h, (void *)base) != cudaSuccess) { cudaGetLastError(); return FG_ERR_CUDA; }
  memcpy(handle_out, &h, 64);
  *offset_out = (int64_t)((unsigned long long)dev_ptr - base);
  return FG_OK;
}

extern "C" int fg_ipc_import(const unsigned char handle[64], void **base_out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  void *p = nullptr;
  if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); return FG_ERR_CUDA; }
  *base_out = p;
  return FG_OK;
}

extern "C" int fg_ipc_close(void *base) {
  return cudaIpcCloseMemHandle(base) == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

extern "C" int fg_halo_push(int32_t precision, const void *dev_r, const void *dev_q, const int64_t *dev_row_off_r,
                            const int64_t *dev_row_off_q, const int64_t *dev_dst_r, const int64_t *dev_dst_q, int64_t n_r,
                            int64_t n_q, int32_t dom, void *stream) {
  if (n_r + n_q <= 0) return FG_OK;
  if (dom < 1) return FG_ERR_ARG;
  const int elem = precision == FG_F64 ? 8 : 4;
  const int row_bytes = dom * elem;
  const int pb = (row_bytes % 16 == 0) ? 16 : ((row_bytes % 8 == 0) ? 8 : 4);
  const int64_t threads = (n_r + n_q) * (row_bytes / pb);
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned char *r = (const unsigned char *)dev_r, *q = (const unsigned char *)dev_q;
  const unsigned blocks = blocks_for(threads, 256);
  if (pb == 16) k_halo_push<16><<<blocks, 256, 0, st>>>(r, q, dev_row_off_r, dev_row_off_q, dev_dst_r, dev_dst_q, n_r, n_q, row_bytes, elem);
  else if (pb == 8) k_halo_push<8><<<blocks, 256, 0, st>>>(r, q, dev_row_off_r, dev_row_off_q, dev_dst_r, dev_dst_q, n_r, n_q, row_bytes, elem);
  else k_halo_push<4><<<blocks, 256, 0, st>>>(r, q, dev_row_off_r, dev_row_off_q, dev_dst_r, dev_dst_q, n_r, n_q, row_bytes, elem);
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------------
// DSA
// ---------------------------------------------------------------------------------------------
extern "C" int fg_dsa_create(const fg_dsa_desc_t *desc, fg_dsa_t *out) {
  int rc = fg_open(desc, out);
  if (rc != FG_OK) return rc;
  fg_dsa *h = *out;
  if ((rc = fg_require_device(h)) != FG_OK) return rc;
  const fg_dsa_desc_t &d = *desc;
  rc = fg_check_resident(h, {FG_FIELD(d, dev_tables), FG_FIELD(d, dev_dom_size), FG_FIELD(d, dev_var_id),
                             FG_FIELD(d, dev_edge_var), FG_FIELD(d, dev_edge_class), FG_FIELD(d, dev_var_ptr),
                             FG_FIELD(d, dev_slot_edge), FG_FIELD(d, dev_has_nbr), FG_FIELD(d, dev_prob),
                             FG_FIELD(d, dev_con_opt), FG_FIELD(d, dev_tables_or), FG_FIELD(d, dev_slot_nbr),
                             FG_FIELD(d, dev_slot_tab), FG_FIELD(d, dev_slot_opt), FG_FIELD(d, dev_value[0]),
                             FG_FIELD(d, dev_value[1]), FG_FIELD(d, dev_value_cost), FG_FIELD(d, dev_var_cost),
                             FG_FIELD(d, dev_unary_off), FG_FIELD(d, dev_row_cache), FG_FIELD(d, dev_slot_last),
                             FG_FIELD(d, dev_var_seed)});
  if (rc != FG_OK) return rc;
  {  // experiment knob: L2 -> DRAM fetch granularity hint (32 | 64 | 128 bytes) for the sparse row reads
    const int g = fg_env_int("PYDCOP_B200_L2_FETCH", 0);
    if (g == 32 || g == 64 || g == 128) { cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)g); cudaGetLastError(); }
  }
  return fg_upload_classes(h);
}

extern "C" int fg_dsa_destroy(fg_dsa_t h) { return fg_close(h); }

extern "C" const char *fg_dsa_last_error(fg_dsa_t h) { return fg_last_error(h); }

extern "C" int fg_dsa_init(fg_dsa_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  fg_launcher launch(h, (cudaStream_t)stream);
  if (h->d.precision == FG_F64) dsa_init<double>(h->d, h->dev_classes, launch);
  else dsa_init<float>(h->d, h->dev_classes, launch);
  if (int rc = launch.status()) return rc;
  CUDA_TRY(h, cudaGetLastError());
  h->cur = 0;
  h->cycle = 0;
  return FG_OK;
}

template <typename T>
static int dsa_compute_t(fg_dsa *h, cudaStream_t st) {
  const fg_dsa_desc_t &d = h->d;
  if (!d.n_vars) return FG_OK;
  const int32_t *val = d.dev_value[h->cur];
  int32_t *val_next = d.dev_value[h->cur ^ 1];
  if (dsa_cached_step<T>(h->d, val, val_next, (uint32_t)h->cycle, st, h->launches)) {
  } else if (!dsa_fast_step<T>(h->d, h->classes, val, val_next, (uint32_t)h->cycle, st, h->launches)) {
    fg_launcher launch(h, st);
    dsa_step<T>(d, h->dev_classes, h->cur, (uint32_t)h->cycle, launch);
  }
  CUDA_TRY(h, cudaGetLastError());
  return FG_OK;
}

extern "C" int fg_dsa_cycle_compute(fg_dsa_t h, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (h->d.stop_cycle && h->cycle >= h->d.stop_cycle) return FG_OK;
  cudaStream_t st = (cudaStream_t)stream;
  return h->d.precision == FG_F64 ? dsa_compute_t<double>(h, st) : dsa_compute_t<float>(h, st);
}

extern "C" int fg_dsa_cycle_commit(fg_dsa_t h) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (h->d.stop_cycle && h->cycle >= h->d.stop_cycle) return FG_OK;
  h->cur ^= 1;
  ++h->cycle;
  return FG_OK;
}

extern "C" int fg_dsa_step(fg_dsa_t h, int32_t n_cycles, void *stream) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  for (int i = 0; i < n_cycles; ++i) {
    if (h->d.stop_cycle && h->cycle >= h->d.stop_cycle) break;
    int rc = fg_dsa_cycle_compute(h, stream);
    if (rc != FG_OK) return rc;
    fg_dsa_cycle_commit(h);
  }
  return FG_OK;
}

extern "C" int fg_dsa_current(fg_dsa_t h, int32_t *buf_index, int64_t *cycle) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (buf_index) *buf_index = h->cur;
  if (cycle) *cycle = h->cycle;
  return FG_OK;
}

extern "C" int64_t fg_dsa_launch_count(fg_dsa_t h) { return fg_launch_count(h); }

extern "C" int fg_dsa_shard_attach(fg_dsa_t h, const fg_halo_plan_t *plan) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (halo_plan_check(plan) != FG_OK || plan->elem_bytes != 4 || plan->dom != 1 || plan->n_q != 0) {
    snprintf(h->err, sizeof(h->err), "invalid halo plan (DSA pushes single 4-byte values, list r only)");
    return FG_ERR_ARG;
  }
  h->halo = *plan;
  h->has_halo = true;
  h->epoch = 0;
  return FG_OK;
}

// whole DSA cycles of one shard on the device: evaluate_cycle -> boundary values into the peers' ghost
// entries of `next` (+ release) -> wait -> commit.  Ghost (frozen) variables are never written locally.
extern "C" int fg_dsa_shard_step(fg_dsa_t h, int32_t n_cycles, void *stream) {
  if (!h || !h->has_halo) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n_cycles; ++i) {
    if (h->d.stop_cycle && h->cycle >= h->d.stop_cycle) break;
    int rc = fg_dsa_cycle_compute(h, stream);
    if (rc != FG_OK) return rc;
    const int nxt = h->cur ^ 1;
    rc = halo_push_launch(h->halo, h->d.dev_value[nxt], h->d.dev_value[nxt], nxt, h->halo.n_r, 0, 1, h->epoch + 1, st,
                          h->launches);
    if (rc == FG_OK) rc = peer_wait_launch(h->halo.sync, h->epoch + 1, st, h->launches);
    if (rc != FG_OK) { snprintf(h->err, sizeof(h->err), "peer push / wait launch failed"); return rc; }
    ++h->epoch;
    fg_dsa_cycle_commit(h);
  }
  return FG_OK;
}

// ---------------------------------------------------------------------------------------------
// solution cost (dcop.py:319-367): costs equal to `infinity` are COUNTED, the others summed —
// constraints and variable costs alike.  `seg` (optional) gives every factor / variable the problem it belongs to
// (fg_solution_cost_segmented); NULL puts everything in segment 0.
// ---------------------------------------------------------------------------------------------

// Adds the warp's (cost, violation) pairs into out[2 * s], out[2 * s + 1].  Without segments: a butterfly and one
// atomic pair per warp.  With segments: an inclusive scan inside each run of consecutive lanes with the same segment,
// and one atomic pair per run from its last lane, so any order is correct and runs (the usual case: a problem's
// factors and variables lie in runs of the internal order) cost one atomic pair per warp and run.  A lane with
// s < 0 adds nothing.
__device__ __forceinline__ void cost_warp_add(double cst, double viol, int s, bool segmented, double *__restrict__ out) {
  const unsigned lane = threadIdx.x & 31;
  if (!segmented) {
    for (int o = 16; o; o >>= 1) { cst += __shfl_xor_sync(0xffffffffu, cst, o); viol += __shfl_xor_sync(0xffffffffu, viol, o); }
    if (lane == 0) { if (cst != 0.0) atomicAdd(out, cst); if (viol != 0.0) atomicAdd(out + 1, viol); }
    return;
  }
  const int prev = __shfl_up_sync(0xffffffffu, s, 1);
  const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || prev != s);
  const unsigned run_start = 31u - __clz(heads & (0xffffffffu >> (31u - lane)));   // highest head at or below lane
  for (unsigned o = 1; o < 32; o <<= 1) {
    const double c = __shfl_up_sync(0xffffffffu, cst, o), v = __shfl_up_sync(0xffffffffu, viol, o);
    if (lane >= run_start + o) { cst += c; viol += v; }
  }
  const bool run_end = lane == 31 || ((heads >> (lane + 1)) & 1u);
  if (run_end && s >= 0) {
    if (cst != 0.0) atomicAdd(out + 2 * (int64_t)s, cst);
    if (viol != 0.0) atomicAdd(out + 2 * (int64_t)s + 1, viol);
  }
}

template <typename T>
__global__ void k_cost_factors(const fg_class_t c, const T *__restrict__ tables, const int32_t *__restrict__ edge_var,
                               const int32_t *__restrict__ value, const uint8_t *__restrict__ skip, T infinity,
                               const int32_t *__restrict__ seg, int32_t n_seg, double *__restrict__ out) {
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  double cst = 0.0, viol = 0.0;
  int s = -1;
  if (f < c.n_factors) {
    s = seg ? seg[c.first_factor + f] : 0;
    if (s >= n_seg) s = -1;
  }
  if (s >= 0 && !(skip && skip[c.first_factor + f])) {
    int64_t idx = 0, stride = 1;
    const int e0 = c.first_edge + f * c.arity;
    for (int i = c.arity - 1; i >= 0; --i) { idx += (int64_t)value[edge_var[e0 + i]] * stride; stride *= c.dom[i]; }
    const T t = tables[c.table_base + (int64_t)f * c.table_size + idx];
    if (t != infinity) cst = (double)t; else viol = 1.0;   // `r_cost != infinity`, dcop.py:355
  }
  cost_warp_add(cst, viol, s, seg != nullptr, out);
}

template <typename T>
__global__ void k_cost_unary(const T *__restrict__ unary, const int64_t *__restrict__ unary_off,
                             const int32_t *__restrict__ value, int n_vars, const uint8_t *__restrict__ skip,
                             T infinity, const int32_t *__restrict__ seg, int32_t n_seg, double *__restrict__ out) {
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  double cst = 0.0, viol = 0.0;
  int s = -1;
  if (v < n_vars) {
    s = seg ? seg[v] : 0;
    if (s >= n_seg) s = -1;
  }
  if (s >= 0 && !(skip && skip[v])) {
    const T t = unary[unary_off[v] + value[v]];
    if (t != infinity) cst = (double)t; else viol = 1.0;   // `cost_for_val != infinity`, dcop.py:363
  }
  cost_warp_add(cst, viol, s, seg != nullptr, out);
}

static int solution_cost_launch(int32_t precision, int32_t n_classes, const fg_class_t *classes, const void *dev_tables,
                                const int32_t *dev_edge_var, const int32_t *dev_value, const void *dev_unary,
                                const int64_t *dev_unary_off, int32_t n_vars, const uint8_t *dev_factor_skip,
                                const uint8_t *dev_var_skip, const int32_t *dev_factor_seg, const int32_t *dev_var_seg,
                                int32_t n_seg, double infinity, double *dev_out, void *stream) {
  if (!fg_on_current_device(dev_out) || (dev_value && !fg_on_current_device(dev_value))) return FG_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(dev_out, 0, 2 * sizeof(double) * (size_t)n_seg, st) != cudaSuccess) return FG_ERR_CUDA;
  for (int i = 0; i < n_classes; ++i) {
    const fg_class_t &c = classes[i];
    if (!c.n_factors || (c.flags & FG_CLASS_GHOST)) continue;   // halo stubs stand for another rank's factors
    if (precision == FG_F64) k_cost_factors<double><<<blocks_for(c.n_factors, 128), 128, 0, st>>>(c, (const double *)dev_tables, dev_edge_var, dev_value, dev_factor_skip, infinity, dev_factor_seg, n_seg, dev_out);
    else k_cost_factors<float><<<blocks_for(c.n_factors, 128), 128, 0, st>>>(c, (const float *)dev_tables, dev_edge_var, dev_value, dev_factor_skip, (float)infinity, dev_factor_seg, n_seg, dev_out);
  }
  if (dev_unary && n_vars) {
    if (precision == FG_F64) k_cost_unary<double><<<blocks_for(n_vars, 128), 128, 0, st>>>((const double *)dev_unary, dev_unary_off, dev_value, n_vars, dev_var_skip, infinity, dev_var_seg, n_seg, dev_out);
    else k_cost_unary<float><<<blocks_for(n_vars, 128), 128, 0, st>>>((const float *)dev_unary, dev_unary_off, dev_value, n_vars, dev_var_skip, (float)infinity, dev_var_seg, n_seg, dev_out);
  }
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

extern "C" int fg_solution_cost(int32_t precision, int32_t n_classes, const fg_class_t *classes, const void *dev_tables,
                                const int32_t *dev_edge_var, const int32_t *dev_value, const void *dev_unary,
                                const int64_t *dev_unary_off, int32_t n_vars, const uint8_t *dev_factor_skip,
                                const uint8_t *dev_var_skip, double infinity, double *dev_out, void *stream) {
  return solution_cost_launch(precision, n_classes, classes, dev_tables, dev_edge_var, dev_value, dev_unary,
                              dev_unary_off, n_vars, dev_factor_skip, dev_var_skip, nullptr, nullptr, 1, infinity,
                              dev_out, stream);
}

extern "C" int fg_solution_cost_segmented(int32_t precision, int32_t n_classes, const fg_class_t *classes,
                                          const void *dev_tables, const int32_t *dev_edge_var, const int32_t *dev_value,
                                          const void *dev_unary, const int64_t *dev_unary_off, int32_t n_vars,
                                          const uint8_t *dev_factor_skip, const uint8_t *dev_var_skip,
                                          const int32_t *dev_factor_seg, const int32_t *dev_var_seg, int32_t n_seg,
                                          double infinity, double *dev_out, void *stream) {
  if (n_seg < 1 || !dev_factor_seg || !dev_var_seg) return FG_ERR_ARG;
  if (!fg_on_current_device(dev_factor_seg) || !fg_on_current_device(dev_var_seg)) return FG_ERR_ARG;
  return solution_cost_launch(precision, n_classes, classes, dev_tables, dev_edge_var, dev_value, dev_unary,
                              dev_unary_off, n_vars, dev_factor_skip, dev_var_skip, dev_factor_seg, dev_var_seg, n_seg,
                              infinity, dev_out, stream);
}

// one 16-, 8- or 4-byte word per thread and step: rows of C2's f32 tables (400 bytes) move as 25 16-byte words
template <typename W>
__global__ void k_gather_rows(W *__restrict__ dst, const W *__restrict__ src, const int64_t *__restrict__ rows,
                              int64_t n_rows, int64_t row_words) {
  const int64_t n = n_rows * row_words;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / row_words;
    dst[i] = src[rows[r] * row_words + (i - r * row_words)];
  }
}

extern "C" int fg_gather_rows(int32_t precision, void *dev_dst, const void *dev_src, const int64_t *dev_rows,
                              int64_t n_rows, int64_t row_elems, void *stream) {
  if (n_rows <= 0 || row_elems <= 0) return FG_OK;
  if (!dev_dst || !dev_src || !dev_rows || !fg_on_current_device(dev_dst) || !fg_on_current_device(dev_src))
    return FG_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t row_bytes = row_elems * (precision == FG_F64 ? 8 : 4);
  const uintptr_t al = (uintptr_t)dev_dst | (uintptr_t)dev_src | (uintptr_t)row_bytes;
  const unsigned blocks = (unsigned)std::min<int64_t>((n_rows * row_bytes / 4 + 255) / 256, 8192);
  if (al % 16 == 0)
    k_gather_rows<int4><<<blocks, 256, 0, st>>>((int4 *)dev_dst, (const int4 *)dev_src, dev_rows, n_rows, row_bytes / 16);
  else if (al % 8 == 0)
    k_gather_rows<int2><<<blocks, 256, 0, st>>>((int2 *)dev_dst, (const int2 *)dev_src, dev_rows, n_rows, row_bytes / 8);
  else
    k_gather_rows<int32_t><<<blocks, 256, 0, st>>>((int32_t *)dev_dst, (const int32_t *)dev_src, dev_rows, n_rows, row_bytes / 4);
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------------
// diagnostics
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_selftest_match(int64_t n, const T *__restrict__ c, const T *__restrict__ prev, T stab,
                                 uint8_t *__restrict__ out_fast, uint8_t *__restrict__ out_exact) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out_fast[i] = approx_match_fast<T>(c[i], prev[i], stab) ? 1 : 0;
  out_exact[i] = approx_match1<T>(c[i], prev[i], stab) ? 1 : 0;
}

extern "C" int fg_selftest_approx_match(int32_t precision, int64_t n, const void *dev_c, const void *dev_prev,
                                        double stability, uint8_t *dev_out_fast, uint8_t *dev_out_exact, void *stream) {
  if (n <= 0) return FG_OK;
  if (!fg_on_current_device(dev_c)) return FG_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == FG_F64)
    k_selftest_match<double><<<blocks_for(n, 256), 256, 0, st>>>(n, (const double *)dev_c, (const double *)dev_prev, stability, dev_out_fast, dev_out_exact);
  else
    k_selftest_match<float><<<blocks_for(n, 256), 256, 0, st>>>(n, (const float *)dev_c, (const float *)dev_prev, (float)stability, dev_out_fast, dev_out_exact);
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}

extern "C" int fg_selftest_gather(const void *dev_base, int64_t region_bytes, int32_t row_bytes, int32_t stride_bytes,
                                  int64_t n_threads, int32_t rows_per_thread, float *dev_out, void *stream) {
  if (!dev_base || !dev_out || row_bytes <= 0 || row_bytes % 16 || stride_bytes < row_bytes || stride_bytes % 16 ||
      region_bytes < stride_bytes || n_threads <= 0)
    return FG_ERR_ARG;
  if (!fg_on_current_device(dev_base)) return FG_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const uint64_t n_slots = (uint64_t)(region_bytes / stride_bytes);
  const unsigned blocks = blocks_for(n_threads, 128);
  switch (rows_per_thread) {
#define X(n) case n: k_selftest_gather<n><<<blocks, 128, 0, st>>>((const uint8_t *)dev_base, n_slots, row_bytes, stride_bytes, n_threads, dev_out); break;
    X(1) X(2) X(3) X(6)
#undef X
    default: return FG_ERR_ARG;
  }
  return cudaGetLastError() == cudaSuccess ? FG_OK : FG_ERR_CUDA;
}
