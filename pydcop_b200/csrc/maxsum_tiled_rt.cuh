// Factor side for the shapes the compile-time kernels do not cover: mixed domain sizes, domain sizes
// outside the compiled set, arity up to FG_MAX_ARITY.  factor_costs_for_var (maxsum.py:382-447) +
// the factor's on_new_cycle (maxsum.py:339-379) with RUNTIME dimensions and compile-time arity.
//
// The one-thread-per-edge kernel (maxsum_generic.cuh) reads each table `arity` times with a stride of one
// table between neighbouring threads, and a class of few large tables (arity 4 over 12 values: 83 KB each) keeps a handful of threads busy for
// tens of milliseconds.  Here a CTA owns a run of consecutive factors of one class: their tables, their
// previous messages and their output rows are CONTIGUOUS in the class-major layout, so every byte crosses
// HBM once, in coalesced requests; only the incoming q rows are gathered (one row per edge, via edge_qoff).
//
// Work is split by OUTPUT VALUE (factor f, scope position j, value x_j) with the lanes of a warp always
// running along the LAST scope dimension — the one with stride 1 in the table — so neighbouring lanes
// read neighbouring table elements (conflict-free in shared memory, coalesced when the table is too
// large for shared memory and is read in place):
//   j <  A-1 : G lanes (G = the power of two >= min(d_last, 32)) share one output; lane g takes
//              x_last = g, g + G, ..., walks the remaining dimensions and the G partial optima are
//              combined with shuffles (an optimum of floats is exact: the split changes no bit);
//   j == A-1 : one lane per value x_last; for arity >= 3 the slice is cut into d_0 parts (x_0 fixed per
//              part) so that these lanes do not become the critical path; the parts are combined when
//              the edge's message is finished.
// The sum over the other positions keeps the reference's order (scope order, left to right):
// ((0 + q_a[x_a]) + q_b[x_b]) + ..., then table + sum, strict optimum; damping / approx_match / send gate
// per edge.  Bit-identical to k_f2v_generic and to the oracle (tests/test_gpu_tiled_rt.py).
// Message rows may be padded (fg_class_t::row_off is aligned, row_total >= sum(dom)): padding is carried over.
// ONE launch per arity and size group over every class (tile table on the device): a mixed-domain problem
// has |domains|^arity classes.
#pragma once
#include <algorithm>

#include "common.cuh"

// one CTA's work: `nf` factors of class `cls` from factor `f0` on; sp = table stride in shared memory, or
// 0 when the table does not fit and is read in place
struct RtTile { int32_t cls, f0, nf, sp; };

constexpr int FG_TILED_RT_THREADS = 256;
constexpr size_t FG_TILED_RT_SMEM = 72 * 1024;         // 3 CTAs per SM
constexpr size_t FG_TILED_RT_SMEM_BIG = 200 * 1024;    // tables between 72 and 200 KB: 1 CTA per SM

struct TiledRtCfg {
  int nf_tile = 0;   // factors per CTA (0: the class is not taken)
  int sp = 0;        // table stride in shared memory, 0 = read in place
  int group = 0;     // 0: FG_TILED_RT_SMEM launch, 1: FG_TILED_RT_SMEM_BIG launch
};

inline int tiled_rt_pow2_ge(int d) { int g = 1; while (g < d && g < 32) g *= 2; return g; }
// tables up to this many entries: one lane per output value walks its whole slice (the lane-group / parts split
// costs more in index arithmetic and shuffles than the bank conflicts of a small table)
constexpr int64_t FG_TILED_RT_WIDE = 2048;

// SMs of the current device (queried once per device): the tile size spreads a class over about 6 tiles per SM
inline int tiled_rt_n_sm() {
  static std::vector<int> per_dev;
  int &n_sm = fg_per_device(per_dev);
  if (!n_sm) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n_sm <= 0) n_sm = 1;
  }
  return n_sm;
}

inline TiledRtCfg tiled_rt_cfg(const fg_class_t &c, size_t elem) {
  TiledRtCfg r;
  const int a = c.arity;
  const int64_t S = c.table_size, RT = c.row_total;
  if (S <= 0 || a < 1) return r;
  const int d_last = c.dom[a - 1];
  const bool wide = S > FG_TILED_RT_WIDE;
  const int64_t parts = (wide && a >= 3) ? (int64_t)c.dom[0] * d_last : 0;   // partial optima of the j == A-1 outputs
  const int64_t rows = (3 * RT + parts) * (int64_t)elem;
  const int64_t sp = S | 1;       // odd: neighbouring factors start in different banks
  int64_t threads = ((wide && a >= 3) ? (int64_t)c.dom[0] : 1) * d_last;     // lanes a factor keeps busy
  for (int j = 0; j + 1 < a; ++j) threads += (int64_t)c.dom[j] * (wide ? tiled_rt_pow2_ge(d_last) : 1);
  const int64_t want = std::max<int64_t>(1, (2 * FG_TILED_RT_THREADS + threads - 1) / threads);
  const int64_t spread = std::max<int64_t>(1, c.n_factors / ((int64_t)tiled_rt_n_sm() * 6));
  const int64_t target = std::max(want, std::min<int64_t>(spread, 4 * want));
  const int64_t per = sp * (int64_t)elem + rows;
  if (per <= (int64_t)FG_TILED_RT_SMEM) {
    r.nf_tile = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)FG_TILED_RT_SMEM / per, target));
    r.sp = (int)sp;
  } else if (per <= (int64_t)FG_TILED_RT_SMEM_BIG) {
    r.nf_tile = 1;
    r.sp = (int)sp;
    r.group = 1;
  } else if (rows <= (int64_t)FG_TILED_RT_SMEM && S < (1ll << 30)) {
    r.nf_tile = 1;   // table read in place (coalesced along the last dimension, `arity` passes through L2)
    r.sp = 0;
  }
  return r;
}

// Launch plan: tiles ordered by (arity, size group), class order inside.
struct TiledRtPlan {
  std::vector<uint8_t> on;            // per class: taken by this kernel
  fg_class_t *dev_classes = nullptr;  // all classes of the problem (indexed by RtTile::cls)
  RtTile *dev_tiles = nullptr;
  int first_tile[2 * FG_MAX_ARITY + 3] = {0};   // tiles of (arity A, group g): [first_tile[2A + g], first_tile[2A + g + 1])
  bool any = false;
};

inline void tiled_rt_free(TiledRtPlan &plan) {
  if (plan.dev_classes) cudaFree(plan.dev_classes);
  if (plan.dev_tiles) cudaFree(plan.dev_tiles);
  plan.dev_classes = nullptr;
  plan.dev_tiles = nullptr;
}

// `skip[i]` != 0: class i already has a compile-time kernel
inline int tiled_rt_plan(const fg_maxsum_desc_t &d, const std::vector<fg_class_t> &classes, const std::vector<uint8_t> &skip,
                         bool enabled, TiledRtPlan &plan) {
  plan.on.assign(classes.size(), 0);
  plan.any = false;
  if (!enabled) return FG_OK;
  const size_t elem = d.precision == FG_F64 ? 8 : 4;
  std::vector<RtTile> tiles;
  plan.first_tile[0] = plan.first_tile[1] = 0;
  for (int a = 1; a <= FG_MAX_ARITY; ++a)
    for (int g = 0; g < 2; ++g) {
      plan.first_tile[2 * a + g] = (int)tiles.size();
      for (size_t i = 0; i < classes.size(); ++i) {
        const fg_class_t &c = classes[i];
        if (c.arity != a || c.n_factors == 0 || (c.flags & FG_CLASS_GHOST) || skip[i]) continue;
        const TiledRtCfg cfg = tiled_rt_cfg(c, elem);
        if (cfg.nf_tile == 0 || cfg.group != g) continue;
        plan.on[i] = 1;
        for (int f0 = 0; f0 < c.n_factors; f0 += cfg.nf_tile)
          tiles.push_back(RtTile{(int32_t)i, f0, std::min(cfg.nf_tile, c.n_factors - f0), cfg.sp});
      }
    }
  plan.first_tile[2 * FG_MAX_ARITY + 2] = (int)tiles.size();
  if (tiles.empty()) return FG_OK;
  plan.any = true;
  if (cudaMalloc(&plan.dev_classes, classes.size() * sizeof(fg_class_t)) != cudaSuccess) return FG_ERR_CUDA;
  if (cudaMalloc(&plan.dev_tiles, tiles.size() * sizeof(RtTile)) != cudaSuccess) return FG_ERR_CUDA;
  if (cudaMemcpy(plan.dev_classes, classes.data(), classes.size() * sizeof(fg_class_t), cudaMemcpyHostToDevice) != cudaSuccess) return FG_ERR_CUDA;
  if (cudaMemcpy(plan.dev_tiles, tiles.data(), tiles.size() * sizeof(RtTile), cudaMemcpyHostToDevice) != cudaSuccess) return FG_ERR_CUDA;
  return FG_OK;
}

template <typename T, int A>
__global__ void __launch_bounds__(FG_TILED_RT_THREADS)
k_f2v_tiled_rt(const fg_class_t *__restrict__ classes, const RtTile *__restrict__ tiles, const T *__restrict__ tables,
               const T *__restrict__ q_cur, const T *__restrict__ r_cur, T *__restrict__ r_next,
               const int64_t *__restrict__ edge_qoff, uint8_t *__restrict__ r_cnt, uint8_t *__restrict__ r_sent, MaxSumParams p) {
  extern __shared__ __align__(16) unsigned char fg_tiled_rt_smem[];
  const RtTile tile = tiles[blockIdx.x];
  const fg_class_t &c = classes[tile.cls];
  const int f0 = tile.f0, nf = tile.nf, sp = tile.sp;
  const bool staged = sp > 0;
  const int S = (int)c.table_size, RT = c.row_total;
  const int first_edge = c.first_edge;
  const int64_t table_base = c.table_base, msg_base = c.msg_base;
  const int tid = threadIdx.x, nt = blockDim.x;
  int dom[A], roff[A], stride[A];
  {
    int s = 1;
#pragma unroll
    for (int i = A - 1; i >= 0; --i) { dom[i] = c.dom[i]; roff[i] = c.row_off[i]; stride[i] = s; s *= c.dom[i]; }
  }
  const int d_last = dom[A - 1];
  const bool wide = S > (int)FG_TILED_RT_WIDE;       // small tables: one lane per output, no split
  const int P = (wide && A >= 3) ? dom[0] : 1;       // parts of a j == A-1 output
  int G = 1, logG = 0;                               // lanes per j < A-1 output
  while (wide && G < d_last && G < 32) { G *= 2; ++logG; }
  T *tab = reinterpret_cast<T *>(fg_tiled_rt_smem);   // nf x sp (staged tables)
  T *qs = tab + (staged ? (size_t)nf * sp : 0);       // nf x RT   incoming v->f rows, scope order
  T *cand = qs + (size_t)nf * RT;                     // nf x RT   new f->v rows
  T *prev = cand + (size_t)nf * RT;                   // nf x RT   previous f->v rows
  T *part = prev + (size_t)nf * RT;                   // nf x d_last x P   partial optima (A >= 3)
  const T *gtab = tables + table_base + (int64_t)f0 * S;
  // --- stage: tables and previous rows are contiguous runs; q rows are gathered per edge
  {
    if (staged) {
      const int n = nf * S;
      for (int i = tid; i < n; i += nt) {
        const int f = i / S, k = i - f * S;
        tab[f * sp + k] = gtab[i];
      }
    }
    const T *rp = r_cur + msg_base + (int64_t)f0 * RT;
    const int64_t *qo = edge_qoff + first_edge + (int64_t)f0 * A;
    const int m = nf * RT;
    for (int i = tid; i < m; i += nt) {
      const T pv = rp[i];
      prev[i] = pv;
      cand[i] = pv;   // padding between rows is carried over
      const int f = i / RT, k = i - f * RT;
      int j = 0, ro = 0, dj = dom[0];
#pragma unroll
      for (int t = 1; t < A; ++t)
        if (k >= roff[t]) { j = t; ro = roff[t]; dj = dom[t]; }
      qs[i] = (k - ro) < dj ? q_cur[qo[f * A + j] + (k - ro)] : (T)0;
    }
  }
  __syncthreads();
  // --- optima.  Thread slots: for j = 0 .. A-2 a segment of nf * d_j outputs x G lanes, then nf * P * d_last lanes
  {
    const bool mx = p.mode_max != 0;
    int seg_end[A];   // exclusive end of segment j (j == A-1: the one-lane-per-value segment)
    {
      int o = 0;
#pragma unroll
      for (int j = 0; j < A - 1; ++j) { o += nf * dom[j] * G; seg_end[j] = o; }
      o += nf * P * d_last;
      seg_end[A - 1] = o;
    }
    const int total = seg_end[A - 1];
    for (int base = 0; base < total; base += nt) {
      const int u = base + tid;
      const bool valid = u < total;
      int j = A - 1, seg0 = 0;
#pragma unroll
      for (int t = A - 2; t >= 0; --t)
        if (u < seg_end[t]) j = t;
#pragma unroll
      for (int t = 0; t < A - 1; ++t)
        if (j > t) seg0 = seg_end[t];
      const bool last_pos = j == A - 1;
      const int w = u - seg0;
      int f, xv, g = 0, part_id = 0, dj = d_last, sj = 1;
      if (last_pos) {
        xv = w % d_last;
        const int w2 = w / d_last;
        part_id = w2 % P;
        f = w2 / P;
      } else {
#pragma unroll
        for (int t = 0; t < A - 1; ++t)
          if (j == t) { dj = dom[t]; sj = stride[t]; }
        g = w & (G - 1);
        const int o = w >> logG;
        f = o / dj;
        xv = o - f * dj;
      }
      T opt = mx ? -Inf<T>::pos() : Inf<T>::pos();
      if (valid) {
        const T *tf = staged ? tab + f * sp : gtab + (int64_t)f * S;
        const T *qf = qs + f * RT;
        const bool fix0 = last_pos && P > 1;    // x_0 = part_id, not walked
        int x[A];
#pragma unroll
        for (int i = 0; i < A; ++i) x[i] = 0;
        int idx = xv * sj;                      // last_pos: sj == 1, xv is the last-dimension index
        if (fix0) { x[0] = part_id; idx += part_id * stride[0]; }
        for (;;) {
          T sum = (T)0;   // scope order, left to right: exactly the reference's additions
#pragma unroll
          for (int i = 0; i < A - 1; ++i)
            if (i != j) sum += qf[roff[i] + x[i]];
          if (last_pos) {
            opt_update(opt, tf[idx] + sum, mx);
          } else {
            for (int xl = g; xl < d_last; xl += G) opt_update(opt, tf[idx + xl] + (sum + qf[roff[A - 1] + xl]), mx);
          }
          bool more = false;
#pragma unroll
          for (int i = A - 2; i >= 0; --i) {
            if (more || i == j || (fix0 && i == 0)) continue;
            ++x[i];
            idx += stride[i];
            if (x[i] < dom[i]) { more = true; continue; }
            idx -= dom[i] * stride[i];
            x[i] = 0;
          }
          if (!more) break;
        }
      }
      // combine the G lanes of an output (all 32 lanes take part in the shuffles; G is uniform over the CTA)
      if (G > 1) {
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1) {
          const T other = __shfl_xor_sync(0xffffffffu, opt, m);
          if (!last_pos && m < G) opt_update(opt, other, mx);
        }
      }
      if (valid) {
        if (last_pos) {
          if (P > 1) part[(f * d_last + xv) * P + part_id] = opt;
          else cand[f * RT + roff[A - 1] + xv] = opt;
        } else if (g == 0) {
          int ro = roff[0];
#pragma unroll
          for (int t = 1; t < A - 1; ++t)
            if (j == t) ro = roff[t];
          cand[f * RT + ro + xv] = opt;
        }
      }
    }
  }
  __syncthreads();
  // --- per edge: damping, approx_match, send gate (maxsum.py:339-379, 679-710); results replace `cand`
  {
    const bool mx = p.mode_max != 0;
    const T lam = (T)p.damping, oml = (T)p.one_minus_damping, stab = (T)p.stability;
    const int ne = nf * A;
    for (int le = tid; le < ne; le += nt) {
      const int f = le / A, j = le - f * A;
      const int e = first_edge + (f0 + f) * A + j;
      int d = dom[0], ro = roff[0];
#pragma unroll
      for (int t = 1; t < A; ++t)
        if (j == t) { d = dom[t]; ro = roff[t]; }
      T *cr = cand + f * RT + ro;
      const T *pr = prev + f * RT + ro;
      const bool parts = P > 1 && j == A - 1;
      uint8_t cnt = r_cnt[e];
      const bool has_prev = cnt & 1;
      const bool damp = p.damp_factors && has_prev;
      bool match = has_prev;
      for (int xv = 0; xv < d; ++xv) {
        T v;
        if (parts) {
          const T *pp = part + (f * d_last + xv) * P;
          v = pp[0];
          for (int k = 1; k < P; ++k) opt_update(v, pp[k], mx);
        } else {
          v = cr[xv];
        }
        const T pv = pr[xv];
        if (damp) v = lam * pv + oml * v;
        if (has_prev && !approx_match1<T>(v, pv, stab)) match = false;
        cr[xv] = v;
      }
      const bool sent = gate_decide(match, cnt);
      if (!sent)
        for (int xv = 0; xv < d; ++xv) cr[xv] = pr[xv];
      r_cnt[e] = cnt;
      if (r_sent) r_sent[e] = sent ? 1 : 0;
    }
  }
  __syncthreads();
  {
    T *dst = r_next + msg_base + (int64_t)f0 * RT;
    const int m = nf * RT;
    for (int i = tid; i < m; i += nt) dst[i] = cand[i];
  }
}

// every class of the plan: one launch per (arity, size group) present
template <typename T, int A>
inline int launch_f2v_tiled_rt(const TiledRtPlan &plan, const fg_maxsum_desc_t &d, const T *q_cur, const T *r_cur, T *r_next,
                               const MaxSumParams &p, cudaStream_t st) {
  static std::vector<uint8_t> per_dev;   // per instantiation and device: the attribute is set
  int n = 0;
  for (int g = 0; g < 2; ++g) {
    const int t0 = plan.first_tile[2 * A + g], t1 = plan.first_tile[2 * A + g + 1];
    if (t1 <= t0) continue;
    uint8_t &attr_done = fg_per_device(per_dev);
    if (!attr_done) {
      cudaFuncSetAttribute(k_f2v_tiled_rt<T, A>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FG_TILED_RT_SMEM_BIG);
      attr_done = true;
    }
    const size_t smem = g ? FG_TILED_RT_SMEM_BIG : FG_TILED_RT_SMEM;
    k_f2v_tiled_rt<T, A><<<t1 - t0, FG_TILED_RT_THREADS, smem, st>>>(plan.dev_classes, plan.dev_tiles + t0, (const T *)d.dev_tables, q_cur,
                                                                     r_cur, r_next, d.dev_edge_qoff, d.dev_r_cnt, d.dev_r_sent, p);
    ++n;
  }
  return n;
}

template <typename T>
inline int dispatch_f2v_tiled_rt(const TiledRtPlan &plan, const fg_maxsum_desc_t &d, const T *q_cur, const T *r_cur, T *r_next,
                                 const MaxSumParams &p, cudaStream_t st) {
  int n = 0;
  if (!plan.any) return 0;
#define X(a) n += launch_f2v_tiled_rt<T, a>(plan, d, q_cur, r_cur, r_next, p, st);
  X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8)
#undef X
  return n;
}
