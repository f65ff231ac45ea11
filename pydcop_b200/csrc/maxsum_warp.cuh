// Warp-autonomous MaxSum kernels: every warp runs its OWN software pipeline over its own
// tiles — its own shared-memory stages, its own mbarriers and cp.async groups — so there is no
// block-wide barrier anywhere (the CTA-pipelined k_v2f_pipe spends much of its issue slots parked at
// __syncthreads), and the arithmetic is written for the issue slots it costs, so
//   * rows are handled as value pairs (packed.cuh) — every element gets the correctly rounded IEEE
//     operation of the scalar code;
//   * min / max is a template parameter, tile descriptors are arithmetic from a per-class table staged in
//     shared memory (no dependent global load on the critical path), lane -> (variable, slot) uses a
//     reciprocal from that table.
//
//  k_v2f_warp<T,D,NS,MX>   variable -> factor (+ select_value).  A tile = nv variables of one (D, K) class
//      = nv*K <= 32 consecutive slots, ONE SLOT PER LANE.  HBM side: the previous q rows and the unary
//      rows of a tile are contiguous (1-D bulk async copies, TMA, per-warp mbarrier), the K r rows of a
//      variable are gathered through slot_roff with cp.async — lanes mapped (row, 8/16-byte piece) so one
//      LDGSTS instruction touches ~7 rows instead of 32 — and the produced q rows leave with one bulk
//      store per tile (written in place over the staged previous rows).  NS stages per warp: tile k is
//      computed while tiles k+1 .. k+NS-1 load.
//      Arithmetic per lane (slot f of variable i): costs_for_factor (maxsum.py:623-676) in the
//      reference's operand order — value-major, then the OTHER factors in `links` order (the own factor
//      is skipped by addressing: row g = gg + (gg >= f), no select) — unrolled for K = 1..8; the lane of
//      the LAST slot holds ur + r_0 + ... + r_{K-2}, so select_value (maxsum.py:584-620) costs one more
//      add per value.
//
//  k_f2v_warp<T,D,NS,MX>   factor -> variable, binary factors over one even domain size (see below).
//
// Both kernels have a PEER instantiation (multi-GPU, opt-in fused halo, DESIGN.md §6): the lane that finishes a
// boundary row also stores it into the consuming rank's buffer (an IPC-mapped NVLink address per edge / per slot,
// MaxSumParams::edge_dst / slot_dst); PEER = false compiles that code out.
//
// Results are bit-identical to the generic kernels, the round-1 pipelined kernels and the CPU oracle
// of the same precision.
#pragma once
#include "maxsum_fast.cuh"
#include "packed.cuh"
#include "table_i8.cuh"

// ------------------------------------------------------------------------------------------------
// variable -> factor
// ------------------------------------------------------------------------------------------------
// one class of the variable side as the kernel sees it (host-built, 48 bytes, staged in shared memory): tile t
// of the launch belongs to the entry with tile_begin <= t < tile_end; everything of the tile is affine in it
struct WClassEntry {
  int32_t tile_begin, tile_end;
  int32_t nv_tile;   // variables per tile (nv_tile * K <= 32)
  int32_t K;         // degree
  int32_t n_vars, first_slot, first_var;
  int32_t kinv;      // ceil(65536 / K): lane / K == (lane * kinv) >> 16 for lane < 32
  uint32_t q_base, unary_base;   // element offsets (the fast plans require 32-bit message offsets)
  int32_t pad0, pad1;
};
static_assert(sizeof(WClassEntry) == 48, "three 16-byte loads");
#define FG_WARP_MAX_CLASSES 40   // degrees 1..16 x (own | other tags) of one domain size

struct WTileRange {   // one launch: the regular variable classes of one domain size
  int32_t dom, first, count;   // entries [first, first + count) of the plan's class table
  int32_t n_tiles;
  int32_t boundary;            // multi-GPU: classes of variables with a remote factor (FG_CLASS_BOUNDARY), launched first
};

struct WTile {
  int valid, K, nv, nslots, slot0, var0, kinv;
  uint32_t qoff, uoff;
};

// tile t; `ci` is a forward-only cursor of the calling ROLE (a warp visits its tiles in ascending order)
__device__ __forceinline__ WTile wtile_at(const WClassEntry *__restrict__ cls, int n_tiles, int t, int D, int &ci) {
  WTile o;
  o.valid = t < n_tiles;
  if (!o.valid) { o.K = 1; o.nv = o.nslots = o.slot0 = o.var0 = 0; o.kinv = 65536; o.qoff = o.uoff = 0; return o; }
  while (t >= cls[ci].tile_end) ++ci;
  const WClassEntry &e = cls[ci];
  const int v0 = (t - e.tile_begin) * e.nv_tile;
  o.K = e.K;
  o.kinv = e.kinv;
  o.nv = min(e.nv_tile, e.n_vars - v0);
  o.nslots = o.nv * e.K;
  o.slot0 = e.first_slot + v0 * e.K;
  o.var0 = e.first_var + v0;
  o.qoff = e.q_base + (uint32_t)(v0 * e.K * D);
  o.uoff = e.unary_base + (uint32_t)(v0 * D);
  return o;
}

#define FG_WARP_K_SWITCH(K_, CALL)                 \
  switch (K_) {                                    \
    case 1: { constexpr int KK = 1; CALL; } break; \
    case 2: { constexpr int KK = 2; CALL; } break; \
    case 3: { constexpr int KK = 3; CALL; } break; \
    case 4: { constexpr int KK = 4; CALL; } break; \
    case 5: { constexpr int KK = 5; CALL; } break; \
    case 6: { constexpr int KK = 6; CALL; } break; \
    case 7: { constexpr int KK = 7; CALL; } break; \
    case 8: { constexpr int KK = 8; CALL; } break; \
  }

// One lane = slot f of a variable whose K gathered r rows start at `col` (row g at col + g*D) and whose
// own costs are `ur`.  cand <- un-normalised message, returns sum_cost; best / best_c <- select_value over
// ur + ALL K rows, meaningful on the lane with f == K-1 only (its message chain is exactly the first
// K-1 terms of that sum).  KK > 0: compile-time degree; KK == 0: run-time degree k_rt.
template <typename T, int D, int KK, bool MX>
__device__ __forceinline__ T v2f_lane_msg(const T *__restrict__ col, const T *__restrict__ ur, int f, int k_rt,
                                          T (&cand)[D], int &best, T &best_c) {
  constexpr int VR = V2FCfg<T, D>::VR;
  using P = typename Pair<T>::type;
  T sum_cost = (T)0;
  best = 0;
  best_c = (T)0;
  if constexpr (KK > 0) {
    constexpr int KO = KK > 1 ? KK - 1 : 1;
    const T *rp[KO];   // the other factors' rows, in `links` order
#pragma unroll
    for (int gg = 0; gg < KK - 1; ++gg) rp[gg] = col + (gg + (gg >= f ? 1 : 0)) * D;
    const T *lastp = col + (KK - 1) * D;
#pragma unroll
    for (int x0 = 0; x0 < D; x0 += VR) {
      T u[VR], last[VR], c[KO][VR];
      ld_row<T, VR, VR>(ur + x0, u);
      ld_row<T, VR, VR>(lastp + x0, last);
#pragma unroll
      for (int gg = 0; gg < KK - 1; ++gg) ld_row<T, VR, VR>(rp[gg] + x0, c[gg]);
#pragma unroll
      for (int xx = 0; xx < VR; ++xx) {    // sum_cost: ONE chain, value-major then factor order
#pragma unroll
        for (int gg = 0; gg < KK - 1; ++gg) sum_cost += c[gg][xx];
      }
      if constexpr (VR % 2 == 0) {
#pragma unroll
        for (int xx = 0; xx < VR; xx += 2) {
          P m = pmake<T>(u[xx], u[xx + 1]);
#pragma unroll
          for (int gg = 0; gg < KK - 1; ++gg) m = padd(m, pmake<T>(c[gg][xx], c[gg][xx + 1]));
          cand[x0 + xx] = m.x;
          cand[x0 + xx + 1] = m.y;
          const P tot = padd(m, pmake<T>(last[xx], last[xx + 1]));   // lane f == K-1: ((ur + r_0) + ...) + r_{K-1}
          if (x0 + xx == 0 || (MX ? (tot.x > best_c) : (tot.x < best_c))) { best = x0 + xx; best_c = tot.x; }
          if (MX ? (tot.y > best_c) : (tot.y < best_c)) { best = x0 + xx + 1; best_c = tot.y; }
        }
      } else {
#pragma unroll
        for (int xx = 0; xx < VR; ++xx) {
          T m = u[xx];
#pragma unroll
          for (int gg = 0; gg < KK - 1; ++gg) m += c[gg][xx];
          cand[x0 + xx] = m;
          const T tot = m + last[xx];
          if (x0 + xx == 0 || (MX ? (tot > best_c) : (tot < best_c))) { best = x0 + xx; best_c = tot; }
        }
      }
    }
  } else {  // run-time degree (9..16): values unrolled, factors in a loop
#pragma unroll
    for (int x = 0; x < D; ++x) {
      T m = ur[x];
#pragma unroll 1
      for (int gg = 0; gg < k_rt - 1; ++gg) {
        const T cst = col[(gg + (gg >= f ? 1 : 0)) * D + x];
        sum_cost += cst;
        m += cst;
      }
      cand[x] = m;
      const T tot = m + col[(k_rt - 1) * D + x];
      if (x == 0 || (MX ? (tot > best_c) : (tot < best_c))) { best = x; best_c = tot; }
    }
  }
  return sum_cost;
}

#define FG_V2FW_WARPS 4   // warps per CTA (each warp is independent; the CTA is only a container)
#ifndef FG_V2FW_MINB
#define FG_V2FW_MINB 6   // register cap 65536 / (6 * 128) = 85
#endif

template <typename T, int D, int NS_>
struct V2FWarpCfg {
  static constexpr int VR = V2FCfg<T, D>::VR;
  static constexpr int VR_BYTES = V2FCfg<T, D>::VR_BYTES;
  static constexpr int PIECES = D / VR;                     // async-copy pieces per row
  static constexpr int STAGE = 3 * 32 * D;                  // rrow | qio | un   (elements)
  static constexpr int NS = NS_;
  static constexpr size_t WARP_SMEM = (size_t)NS * STAGE * sizeof(T);
  static constexpr size_t SMEM = FG_V2FW_WARPS * WARP_SMEM + FG_V2FW_WARPS * NS * sizeof(uint64_t) +
                                 FG_WARP_MAX_CLASSES * sizeof(WClassEntry) + 16;
  static constexpr bool OK = SMEM <= FG_SMEM_LIMIT;
};


// Fused halo (multi-GPU): a boundary row leaves for its consumer's buffer — an IPC-mapped address of another
// GPU, reached over NVLink — from the lane that produced it, while the rest of the tile is still being
// computed; interior rows have destination 0.  8-byte stores when the row size allows (rows are 8-byte
// aligned at both ends for even D), else element stores.
template <typename T, int D>
__device__ __forceinline__ void peer_store_row(int64_t dst, const T *row) {
  if (dst == 0) return;
  if constexpr ((D * sizeof(T)) % 8 == 0) {
    uint64_t *d = reinterpret_cast<uint64_t *>(dst);
    const uint64_t *s = reinterpret_cast<const uint64_t *>(row);
#pragma unroll
    for (int i = 0; i < (int)(D * sizeof(T) / 8); ++i) d[i] = s[i];
  } else {
    T *d = reinterpret_cast<T *>(dst);
#pragma unroll
    for (int i = 0; i < D; ++i) d[i] = row[i];
  }
}

template <typename T, int D, int NS_, bool MX, typename OffT, bool PEER = false>
__global__ void __launch_bounds__(FG_V2FW_WARPS * 32, FG_V2FW_MINB)
k_v2f_warp(const WClassEntry *__restrict__ classes, int n_classes, int n_tiles, const OffT *__restrict__ slot_roff,
           const T *__restrict__ unary, const T *__restrict__ r_cur, const T *__restrict__ q_cur,
           T *__restrict__ q_next, uint8_t *__restrict__ q_cnt, uint8_t *__restrict__ q_sent,
           int32_t *__restrict__ value, T *__restrict__ value_cost, MaxSumParams p) {
  using C = V2FWarpCfg<T, D, NS_>;
  // PEER (opt-in fused halo): per slot the peer address of its q row this cycle, 0 = interior
  const int64_t *__restrict__ slot_dst = PEER ? p.slot_dst : nullptr;
  constexpr int VR = C::VR, PIECES = C::PIECES, NS = C::NS;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  T *stage0 = reinterpret_cast<T *>(smem_raw + (size_t)wib * C::WARP_SMEM);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)FG_V2FW_WARPS * C::WARP_SMEM) + NS * wib;
  // the class table of the launch, staged once per CTA: tile descriptors are arithmetic from it, so no trip of
  // the loop waits for a descriptor to come from L2 (the first versions did: 18 % of the stall samples)
  WClassEntry *cls = reinterpret_cast<WClassEntry *>(smem_raw + (size_t)FG_V2FW_WARPS * C::WARP_SMEM +
                                                     FG_V2FW_WARPS * NS * sizeof(uint64_t));
  for (int i = threadIdx.x; i < n_classes * (int)(sizeof(WClassEntry) / 16); i += blockDim.x)
    reinterpret_cast<int4 *>(cls)[i] = reinterpret_cast<const int4 *>(classes)[i];
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    fence_mbar_init();
  }
  __syncthreads();   // the only block-wide barrier: the class table is in place

  // tiles are strided over the warps (t = gw + k * nw): the costly high-degree tiles come first in the order and
  // spread evenly (a contiguous run per warp left the first CTAs with all of them: 2x slower, r02 call 8)
  const int gw = (int)blockIdx.x * FG_V2FW_WARPS + wib;       // global warp id
  const int nw = (int)gridDim.x * FG_V2FW_WARPS;
  int cur_c = 0, cur_i = 0, cur_l = 0, cur_n = 0;   // one forward-only cursor per role
  auto tile_at = [&](int k, int &cursor) { return wtile_at(cls, n_tiles, gw + k * nw, D, cursor); };
  auto load_roff = [&](const WTile &t) -> OffT {
    return lane < t.nslots ? slot_roff[t.slot0 + lane] : (OffT)0;
  };
  auto load_cnt = [&](const WTile &t) -> uint8_t {
    return lane < t.nslots ? q_cnt[t.slot0 + lane] : (uint8_t)0;
  };
  auto load_dst = [&](const WTile &t) -> int64_t {
    if constexpr (!PEER) return (int64_t)0;
    return (slot_dst != nullptr && lane < t.nslots) ? slot_dst[t.slot0 + lane] : (int64_t)0;
  };
  // start every load of a tile into stage s (all lanes)
  auto issue = [&](int s, const WTile &t, OffT roff) {
    if (t.valid) {
      const int nslots = t.nslots, nv = t.nv;
      const uint32_t qoff = t.qoff, uoff = t.uoff;
      T *rrow = stage0 + s * C::STAGE;
      T *qio = rrow + 32 * D;
      T *un = qio + 32 * D;
      const uint32_t qbytes = (uint32_t)(nslots * D) * (uint32_t)sizeof(T);
      const uint32_t ubytes = (uint32_t)(nv * D) * (uint32_t)sizeof(T);
      const bool tma_q = (qbytes % 16 == 0) && ((((int64_t)qoff * (int64_t)sizeof(T)) & 15) == 0);
      const bool tma_u = (ubytes % 16 == 0) && ((((int64_t)uoff * (int64_t)sizeof(T)) & 15) == 0);
      if (lane == 0) {
        mbar_expect_tx(&bars[s], (tma_q ? qbytes : 0u) + (tma_u ? ubytes : 0u));
        if (tma_q) tma_load_1d(qio, q_cur + qoff, qbytes, &bars[s]);
        if (tma_u) tma_load_1d(un, unary + uoff, ubytes, &bars[s]);
      }
      if (!tma_q)
        for (int i = lane; i < nslots * D; i += 32) cp_async_b<(int)sizeof(T)>(qio + i, q_cur + qoff + i);
      if (!tma_u)
        for (int i = lane; i < nv * D; i += 32) cp_async_b<(int)sizeof(T)>(un + i, unary + uoff + i);
      // r rows: lane <-> (row, piece), consecutive lanes on consecutive pieces of one row
#pragma unroll
      for (int it = 0; it < PIECES; ++it) {
        const int pc = it * 32 + lane;
        const int row = pc / PIECES, piece = pc - row * PIECES;
        const OffT ro = __shfl_sync(0xffffffffu, roff, row & 31);
        if (row < nslots) cp_async_b<C::VR_BYTES>(rrow + row * D + piece * VR, r_cur + (int64_t)ro + piece * VR);
      }
    }
    cp_async_commit();  // one group per tile, even when empty: uniform accounting
  };

  const T lam = (T)p.damping, oml = (T)p.one_minus_damping, stab = (T)p.stability;

  // prologue: tiles 0 .. NS-2 in flight, gather indices of tile NS-1 and counters of tile 0 on their way
#pragma unroll 1
  for (int k = 0; k < NS - 1; ++k) {
    const WTile t = tile_at(k, cur_i);
    issue(k, t, load_roff(t));
    cur_l = cur_i;
  }
  OffT roff_n = load_roff(tile_at(NS - 1, cur_l));
  int cur_d = 0;
  uint8_t cnt = load_cnt(tile_at(0, cur_n));
  int64_t pdst = 0;
  if constexpr (PEER) pdst = load_dst(tile_at(0, cur_d));

#pragma unroll 1
  for (int k = 0;; ++k) {
    const WTile t = tile_at(k, cur_c);
    if (!t.valid) break;
    const int s = k % NS;
    // tile k+NS-1 goes into the stage tile k-1 held: its bulk store must have finished READING it
    if (lane == 0) tma_store_wait_read();
    __syncwarp();
    issue((k + NS - 1) % NS, tile_at(k + NS - 1, cur_i), roff_n);
    const OffT roff_n2 = load_roff(tile_at(k + NS, cur_l));
    const uint8_t cnt_n = load_cnt(tile_at(k + 1, cur_n));
    int64_t pdst_n = 0;
    if constexpr (PEER) pdst_n = load_dst(tile_at(k + 1, cur_d));
    cp_async_wait_group<NS - 1>();                  // my gathers of tile k have landed ...
    mbar_wait(&bars[s], (uint32_t)((k / NS) & 1));  // ... and so have its bulk copies
    __syncwarp();                                   // ... and every other lane's gathers

    const int K = t.K, nslots = t.nslots, slot0 = t.slot0;
    const uint32_t qoff = t.qoff;
    T *rrow = stage0 + s * C::STAGE;
    T *qio = rrow + 32 * D;
    const T *un = qio + 32 * D;
    if (lane < nslots) {
      const int i = (lane * t.kinv) >> 16, f = lane - i * K;
      const T *col = rrow + i * K * D;
      const T *ur = un + i * D;
      T cand[D], prev[D];
      int best = 0;
      T best_c = (T)0, sum_cost = (T)0;
      if (K <= 8) {
        FG_WARP_K_SWITCH(K, (sum_cost = v2f_lane_msg<T, D, KK, MX>(col, ur, f, K, cand, best, best_c)))
      } else {
        sum_cost = v2f_lane_msg<T, D, 0, MX>(col, ur, f, K, cand, best, best_c);
      }
      const T avg = sum_cost / (T)D;
      ld_row<T, D, VR>(qio + lane * D, prev);
      uint8_t c8 = cnt;
      bool match;
      if constexpr (D % 2 == 0) {
        using P = typename Pair<T>::type;
        const P avg2 = pmake<T>(avg, avg);
#pragma unroll
        for (int x = 0; x < D; x += 2) {
          const P v = psub(pmake<T>(cand[x], cand[x + 1]), avg2);
          cand[x] = v.x;
          cand[x + 1] = v.y;
        }
        match = damp_match_pairs<T, D>(cand, prev, (c8 & 1) != 0, p.damp_vars != 0, lam, oml, stab);
      } else {
#pragma unroll
        for (int x = 0; x < D; ++x) cand[x] = cand[x] - avg;
        match = damp_match_row<T, D>(cand, prev, (c8 & 1) != 0, p.damp_vars != 0, lam, oml, stab);
      }
      const bool sent = gate_decide(match, c8);
      if (!sent) {
#pragma unroll
        for (int x = 0; x < D; ++x) cand[x] = prev[x];
      }
      st_row<T, D, VR>(qio + lane * D, cand);
      if constexpr (PEER) peer_store_row<T, D>(pdst, cand);
      q_cnt[slot0 + lane] = c8;
      if (q_sent) q_sent[slot0 + lane] = sent ? 1 : 0;
      if (f == K - 1) {
        value[t.var0 + i] = best;
        value_cost[t.var0 + i] = best_c;
      }
    }
    const uint32_t obytes = (uint32_t)(nslots * D) * (uint32_t)sizeof(T);
    if ((obytes % 16 == 0) && ((((int64_t)qoff * (int64_t)sizeof(T)) & 15) == 0)) {
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        tma_store_1d(q_next + qoff, qio, obytes);
        tma_store_commit();
      }
    } else {
      __syncwarp();
      for (int i = lane; i < nslots * D; i += 32) q_next[qoff + i] = qio[i];
      __syncwarp();
    }
    roff_n = roff_n2;
    cnt = cnt_n;
    pdst = pdst_n;
  }
  cp_async_wait_all();
  if (lane == 0) tma_store_wait_read();
}

// ------------------------------------------------------------------------------------------------
// host side of the variable kernel
// ------------------------------------------------------------------------------------------------
// Class entries of the regular variable classes (degree 1..16, not ghosts) of domain size D, costly (high-degree)
// classes first.  nv per tile: as many variables as fit 32 lanes, rounded down to the number of rows that
// keeps every tile's q / unary offsets 16-byte aligned (bulk copies) when possible.  Returns the tile count.
inline int v2fw_build_classes(const std::vector<fg_varclass_t> &vcs, int D, size_t elem, std::vector<WClassEntry> &out,
                              int boundary) {
  std::vector<fg_varclass_t> order;
  for (const fg_varclass_t &vc : vcs)
    if (vc.dom == D && vc.degree >= 1 && vc.degree <= 32 && vc.n_vars > 0 && !(vc.flags & FG_CLASS_GHOST) &&
        (boundary < 0 || ((vc.flags & FG_CLASS_BOUNDARY) != 0) == (boundary != 0)))
      order.push_back(vc);
  std::stable_sort(order.begin(), order.end(),
                   [](const fg_varclass_t &a, const fg_varclass_t &b) { return a.degree > b.degree; });
  const int unit = 16 / fg_gcd(16, D * (int)elem);  // rows per 16-byte multiple
  int tiles = 0;
  for (const fg_varclass_t &vc : order) {
    const int K = vc.degree;
    int nv = 32 / K;
    if (nv >= unit) nv = nv / unit * unit;
    WClassEntry e;
    e.tile_begin = tiles;
    tiles += (vc.n_vars + nv - 1) / nv;
    e.tile_end = tiles;
    e.nv_tile = nv;
    e.K = K;
    e.n_vars = vc.n_vars;
    e.first_slot = vc.first_slot;
    e.first_var = vc.first_var;
    e.kinv = (65536 + K - 1) / K;
    e.q_base = (uint32_t)vc.q_base;
    e.unary_base = (uint32_t)vc.unary_base;
    e.pad0 = e.pad1 = 0;
    out.push_back(e);
  }
  return tiles;
}

struct MaxSumWarpPlan {
  std::vector<uint8_t> f2v;          // per factor class: warp kernel available (PYDCOP_B200_F2V != pipe)
  bool v2f_on = false;               // PYDCOP_B200_V2F != pipe
  std::vector<WTileRange> v2f;       // launches of the variable side
  WClassEntry *dev_classes = nullptr;   // library-owned: class table of every launch (48 bytes per class)
  // factor side: 8-bit copy of the integer tables (maxsum_warp_plan_tab8), library-owned; per class its byte offset
  // in it, -1 = the kernel reads dev_tables at full width
  int8_t *tab8 = nullptr;
  int64_t tab8_bytes = 0;
  std::vector<int64_t> tab8_base;
};

template <typename T, int D, int NS_, bool MX>
inline bool launch_v2f_warp_ns(const WClassEntry *dev_classes, const WTileRange &rg, const fg_maxsum_desc_t &d, const T *r_cur,
                               const T *q_cur, T *q_next, const MaxSumParams &p, cudaStream_t st) {
  using C = V2FWarpCfg<T, D, NS_>;
  if constexpr (!C::OK) {
    return false;
  } else {
    auto kern = k_v2f_warp<T, D, NS_, MX, uint32_t>;
    struct Launch { int per_sm = 0, n_sm = 0; bool peer_attr = false; };
    static std::vector<Launch> per_dev;  // one per instantiation and device
    Launch &L = fg_per_device(per_dev);
    if (!L.per_sm) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
      int dev = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&L.n_sm, cudaDevAttrMultiProcessorCount, dev);
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&L.per_sm, kern, FG_V2FW_WARPS * 32, C::SMEM);
      if (L.per_sm < 1) L.per_sm = 1;
      const int cap = fg_env_int("PYDCOP_B200_V2FW_CPS", 3);  // leaves room for the factor side (runs concurrently)
      if (L.per_sm > cap) L.per_sm = cap;
    }
    const int need = (rg.n_tiles + FG_V2FW_WARPS - 1) / FG_V2FW_WARPS;
    const unsigned blocks = (unsigned)std::min(need, L.n_sm * L.per_sm);
    if constexpr (NS_ == 2) {   // fused halo: same kernel with the peer stores compiled in (default depth only)
      if (p.slot_dst != nullptr) {
        auto kp = k_v2f_warp<T, D, NS_, MX, uint32_t, true>;
        if (!L.peer_attr) {
          cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
          L.peer_attr = true;
        }
        kp<<<blocks, FG_V2FW_WARPS * 32, C::SMEM, st>>>(dev_classes + rg.first, rg.count, rg.n_tiles, d.dev_slot_roff32,
                                                        (const T *)d.dev_unary, r_cur, q_cur, q_next, d.dev_q_cnt, d.dev_q_sent,
                                                        d.dev_value, (T *)d.dev_value_cost, p);
        return true;
      }
    }
    kern<<<blocks, FG_V2FW_WARPS * 32, C::SMEM, st>>>(dev_classes + rg.first, rg.count, rg.n_tiles,
                                                       d.dev_slot_roff32, (const T *)d.dev_unary, r_cur, q_cur, q_next,
                                                       d.dev_q_cnt, d.dev_q_sent, d.dev_value, (T *)d.dev_value_cost, p);
    return true;
  }
}

// pipeline depth: PYDCOP_B200_V2FW_NS = 2 | 3 | 4 stages per warp (default 2)
template <typename T, int D>
inline void launch_v2f_warp(const WClassEntry *dev_tiles, const WTileRange &rg, const fg_maxsum_desc_t &d, const T *r_cur,
                            const T *q_cur, T *q_next, const MaxSumParams &p, cudaStream_t st) {
  static const int ns = fg_env_int("PYDCOP_B200_V2FW_NS", 2);
#define FG_TRY(NS_)                                                                                              \
  if (p.mode_max ? launch_v2f_warp_ns<T, D, NS_, true>(dev_tiles, rg, d, r_cur, q_cur, q_next, p, st)            \
                 : launch_v2f_warp_ns<T, D, NS_, false>(dev_tiles, rg, d, r_cur, q_cur, q_next, p, st))          \
    return;
  if (ns >= 4) { FG_TRY(4) }
  if (ns >= 3) { FG_TRY(3) }
  FG_TRY(2)
#undef FG_TRY
}

template <typename T>
inline bool dispatch_v2f_warp(const WClassEntry *dev_tiles, const WTileRange &rg, const fg_maxsum_desc_t &d, const T *r_cur,
                              const T *q_cur, T *q_next, const MaxSumParams &p, cudaStream_t st) {
  switch (rg.dom) {
#define X(n) case n: launch_v2f_warp<T, n>(dev_tiles, rg, d, r_cur, q_cur, q_next, p, st); return true;
    FG_FAST_DOMS(X)
#undef X
  }
  return false;
}

// same class selection as maxsum_fast_plan (every regular class of a compiled domain size); uploads the
// tile descriptors (cudaMalloc: the device must be there)
inline int maxsum_warp_plan(const fg_maxsum_desc_t &d, const std::vector<fg_varclass_t> &vcs, const MaxSumFastPlan &fast,
                            MaxSumWarpPlan &plan) {
  plan.v2f.clear();
  const char *e = getenv("PYDCOP_B200_V2F");
  plan.v2f_on = fast.off32 && !fg_fast_disabled() && !(e && e[0] == 'p');
  if (!plan.v2f_on) return FG_OK;
  const size_t elem = d.precision == FG_F64 ? 8 : 4;
  std::vector<WClassEntry> all;
  std::vector<int> doms;
  for (const fg_varclass_t &vc : vcs)
    if (!(vc.flags & FG_CLASS_GHOST) && vc.degree >= 1 && fg_fast_dom(vc.dom) &&
        std::find(doms.begin(), doms.end(), vc.dom) == doms.end())
      doms.push_back(vc.dom);
  // PYDCOP_B200_PUSH_EARLY=1|2 (experiment): boundary classes first, in launches of their own, so that their rows can leave
  // while the rest computes; default: one launch per domain size over all classes, as on a single GPU
  const bool split_b = fg_env_is("PYDCOP_B200_PUSH_EARLY", '1') || fg_env_is("PYDCOP_B200_PUSH_EARLY", '2');
  for (int boundary = split_b ? 1 : -1; boundary >= (split_b ? 0 : -1); --boundary)
    for (int D : doms) {
      WTileRange rg;
      rg.dom = D;
      rg.boundary = boundary > 0;
      rg.first = (int32_t)all.size();
      rg.n_tiles = v2fw_build_classes(vcs, D, elem, all, boundary);
      rg.count = (int32_t)all.size() - rg.first;
      if (rg.count > FG_WARP_MAX_CLASSES) {   // (cannot happen: <= 16 degrees x 2 tags) — whole side back on the pipelined kernels
        plan.v2f.clear();
        plan.v2f_on = false;
        return FG_OK;
      }
      if (rg.count) plan.v2f.push_back(rg);
    }
  if (!all.empty()) {
    if (cudaMalloc(reinterpret_cast<void **>(&plan.dev_classes), all.size() * sizeof(WClassEntry)) != cudaSuccess) return FG_ERR_CUDA;
    if (cudaMemcpy(plan.dev_classes, all.data(), all.size() * sizeof(WClassEntry), cudaMemcpyHostToDevice) != cudaSuccess)
      return FG_ERR_CUDA;
  }
  return FG_OK;
}

// ------------------------------------------------------------------------------------------------
//  k_f2v_warp<T,D,NS,MX>   factor -> variable, binary factors over one (even) domain size D.
//      A tile = 16 factors = 32 directed edges, TWO LANES PER FACTOR: lane (f, h) owns half of the table
//      rows and walks them ONCE, producing from the same shared-memory read
//        - its D/2 values of the marginal towards position 0 (row optimum of T[x0][.] + q1), and
//        - partial optima over its rows of the marginal towards position 1 (T[.][x1] + q0[x0]),
//      which the two lanes of a factor complete with D/2 shuffles (the optimum of a set of floats is
//      exact, so the split changes no bit).  Rows are taken in PAIRS (two rows = 2*D contiguous elements,
//      16-byte aligned: 128-bit shared-memory loads): for D/2 even lane h owns rows [h*D/2, (h+1)*D/2); for
//      D/2 odd it owns the pairs [h*(D/2-1), (h+1)*(D/2-1)) and the single row D-2+h.  Adds are packed
//      (FADD2), optima 3-input (FMNMX3).  Round 1's kernel read every table twice (once per directed edge).
//      HBM side per warp and stage: tables and previous r rows of the tile are contiguous (1-D bulk
//      async copies on a per-warp mbarrier), the 32 q rows are gathered through edge_qoff with
//      cp.async (lanes <-> (row, piece)), the produced r rows are written in place over the staged
//      previous rows and leave with one bulk store.  NS stages: tile k computes while k+1 .. k+NS-1 load.
//      TT = the table storage type: T, or int8_t for the classes whose every entry passes fg_table_entry_fits_i8
//      (table_i8.cuh; a copy the engine makes at creation, MaxSumWarpPlan::tab8): the same body, only the table
//      loads decode bytes to T exactly (tab_decode), so every message keeps its bits.
// ------------------------------------------------------------------------------------------------
template <typename T, typename TT, int D, int NS_>
struct F2VWarpCfg {
  static constexpr int S = D * D, HD = D / 2, NF = 16;
  static constexpr int NPAIR = (HD % 2 == 0) ? HD / 2 : (HD - 1) / 2;   // row pairs per lane
  static constexpr bool SINGLE = (HD % 2) != 0;                          // plus one single row
  static constexpr bool NARROW = sizeof(TT) < sizeof(T);                 // 8-bit table codes
  static constexpr int VR = V2FCfg<T, D>::VR;          // elements per row vector (row = D elements)
  static constexpr int VR_BYTES = V2FCfg<T, D>::VR_BYTES;
  static constexpr int PIECES = D / VR;
  static constexpr int V2_BYTES = fg_gcd(16, 2 * D * (int)sizeof(T));   // a pair of rows / a factor's 2 message rows
  static constexpr int V2 = V2_BYTES / (int)sizeof(T);
  // table loads, in bytes: a row pair starts at fl*S + ra*D entries (ra even), the single row at fl*S + (D-2+h)*D.
  // Full width: as the message rows.  8-bit: the alignment those offsets guarantee (D = 10: 4-byte pairs — the
  // factor stride of 25 words is odd, so a half-warp's 16 factors hit 16 banks — and 2-byte single rows)
  static constexpr int TV2_BYTES = NARROW ? fg_gcd(fg_gcd(16, 2 * D), S) : V2_BYTES;
  static constexpr int TV1_BYTES = NARROW ? fg_gcd(16, D) : VR_BYTES;
  static constexpr int TAB_BYTES = NF * S * (int)sizeof(TT);           // a multiple of 16: rt stays 16-byte aligned
  static constexpr int STAGE_BYTES = TAB_BYTES + 2 * NF * 2 * D * (int)sizeof(T);   // tab | rt (previous r rows) | qt
  static constexpr int OUT = NF * 2 * D;                             // produced r rows, double-buffered per warp
  static constexpr int NS = NS_;
  static constexpr size_t WARP_SMEM = (size_t)NS * STAGE_BYTES + (size_t)2 * OUT * sizeof(T);
  static constexpr size_t smem_for(int w) { return (size_t)w * WARP_SMEM + (size_t)w * NS * sizeof(uint64_t) + 16; }
  // warps per CTA: the CTA is only a container of independent warps
  static constexpr int WARPS = smem_for(2) <= FG_SMEM_LIMIT ? 2 : (smem_for(1) <= FG_SMEM_LIMIT ? 1 : 0);
  static constexpr size_t SMEM = smem_for(WARPS > 0 ? WARPS : 1);
  static constexpr bool OK = (D % 2 == 0) && D >= 4 && WARPS > 0;
};

// Byte k of w (a signed 8-bit table code, already XOR-ed with 0x80, i.e. biased by +128) as T, exactly: the biased
// byte becomes the low mantissa bits of 2^23 (2^52), and one correctly rounded subtract of 2^23 + 128 leaves the
// integer in [-128, 127] (every intermediate is an integer below 2^24).  A PRMT and an add per entry.
template <typename T> __device__ __forceinline__ T tab_decode(uint32_t wb, int k);
template <> __device__ __forceinline__ float tab_decode<float>(uint32_t wb, int k) {
  return __fsub_rn(__uint_as_float(__byte_perm(wb, 0x4B000000u, 0x7440u | (uint32_t)k)), 8388736.0f);
}
template <> __device__ __forceinline__ double tab_decode<double>(uint32_t wb, int k) {
  return __dsub_rn(__hiloint2double(0x43300000, (int)__byte_perm(wb, 0u, 0x4440u | (uint32_t)k)), 4503599627370624.0);
}

// N consecutive table entries at p, VB-byte aligned, as T: full-width tables load as message rows do, 8-bit codes
// load as 16-bit (VB = 2) or 32/64/128-bit words and are decoded
template <typename T, int N, int VB>
__device__ __forceinline__ void ld_tab(const T *__restrict__ p, T (&out)[N]) {
  ld_row<T, N, VB / (int)sizeof(T)>(p, out);
}
template <typename T, int N, int VB>
__device__ __forceinline__ void ld_tab(const int8_t *__restrict__ p, T (&out)[N]) {
  static_assert(N % VB == 0 && (VB == 2 || VB == 4 || VB == 8 || VB == 16), "table load width");
  if constexpr (VB == 2) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
      const uint32_t wb = (uint32_t)*reinterpret_cast<const uint16_t *>(p + 2 * i) ^ 0x8080u;
      out[2 * i] = tab_decode<T>(wb, 0);
      out[2 * i + 1] = tab_decode<T>(wb, 1);
    }
  } else {
    constexpr int W = VB / 4;   // 32-bit words per load
#pragma unroll
    for (int i = 0; i < N / VB; ++i) {
      uint32_t w[W];
      if constexpr (W == 1) {
        w[0] = *reinterpret_cast<const uint32_t *>(p + VB * i);
      } else if constexpr (W == 2) {
        const uint2 v = *reinterpret_cast<const uint2 *>(p + VB * i);
        w[0] = v.x; w[1] = v.y;
      } else {
        const uint4 v = *reinterpret_cast<const uint4 *>(p + VB * i);
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const uint32_t wb = w[j] ^ 0x80808080u;
#pragma unroll
        for (int k = 0; k < 4; ++k) out[VB * i + 4 * j + k] = tab_decode<T>(wb, k);
      }
    }
  }
}

// table row index of the i-th row lane h owns (i < D/2); see the kernel comment
template <int D>
__host__ __device__ constexpr int f2vw_row(int h, int i) {
  return ((D / 2) % 2 == 0) ? h * (D / 2) + i : (i < D / 2 - 1 ? h * (D / 2 - 1) + i : 2 * (D / 2 - 1) + h);
}

template <typename T, typename TT, int D, int NS_, bool MX, typename OffT, bool PEER = false>
__global__ void __launch_bounds__(F2VWarpCfg<T, TT, D, NS_>::WARPS > 0 ? F2VWarpCfg<T, TT, D, NS_>::WARPS * 32 : 32)
k_f2v_warp(const fg_class_t c, const TT *__restrict__ tables, const T *__restrict__ q_cur,
           const T *__restrict__ r_cur, T *__restrict__ r_next, const OffT *__restrict__ edge_qoff,
           uint8_t *__restrict__ r_cnt, uint8_t *__restrict__ r_sent, MaxSumParams p) {
  using C = F2VWarpCfg<T, TT, D, NS_>;
  // PEER (opt-in fused halo): per edge the peer address of its r row this cycle, 0 = interior
  const int64_t *__restrict__ edge_dst = PEER ? p.edge_dst : nullptr;
  using P = typename Pair<T>::type;
  constexpr int S = C::S, HD = C::HD, NF = C::NF, NS = C::NS, PIECES = C::PIECES, R = 2 * D;
  constexpr int VR = C::VR;
  constexpr int WARPS = C::WARPS > 0 ? C::WARPS : 1;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  unsigned char *stage0 = smem_raw + (size_t)wib * C::WARP_SMEM;
  // stage s: table (TT) | previous r rows (T) | gathered q rows (T)
  auto stage_tab = [&](int s) { return reinterpret_cast<TT *>(stage0 + (size_t)s * C::STAGE_BYTES); };
  auto stage_rt = [&](int s) { return reinterpret_cast<T *>(stage0 + (size_t)s * C::STAGE_BYTES + C::TAB_BYTES); };
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)WARPS * C::WARP_SMEM) + NS * wib;
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    fence_mbar_init();
  }
  __syncwarp();

  const int gw = (int)blockIdx.x * WARPS + wib;
  const int nw = (int)gridDim.x * WARPS;
  const int n_tiles = (c.n_factors + NF - 1) / NF;
  const int n_my = gw < n_tiles ? (n_tiles - 1 - gw) / nw + 1 : 0;

  // lane = local edge le = 2 f + j of my k-th tile: gather offset / gate counter
  auto load_qo = [&](int k) -> OffT {
    if (k < n_my) {
      const int f0 = (gw + k * nw) * NF;
      if (lane < 2 * min(NF, c.n_factors - f0)) return edge_qoff[c.first_edge + f0 * 2 + lane];
    }
    return (OffT)0;
  };
  auto load_cnt = [&](int k) -> uint8_t {
    if (k < n_my) {
      const int f0 = (gw + k * nw) * NF;
      if (lane < 2 * min(NF, c.n_factors - f0)) return r_cnt[c.first_edge + f0 * 2 + lane];
    }
    return (uint8_t)0;
  };
  auto load_dst = [&](int k) -> int64_t {   // lane = local edge 2 f + j
    if constexpr (!PEER) return (int64_t)0;
    if (edge_dst != nullptr && k < n_my) {
      const int f0 = (gw + k * nw) * NF;
      if (lane < 2 * min(NF, c.n_factors - f0)) return edge_dst[c.first_edge + f0 * 2 + lane];
    }
    return (int64_t)0;
  };
  auto issue = [&](int k, OffT qo) {
    if (k < n_my) {
      const int s = k % NS;
      const int f0 = (gw + k * nw) * NF;
      const int nf = min(NF, c.n_factors - f0);
      TT *tab = stage_tab(s);
      T *rt = stage_rt(s);
      T *qt = rt + NF * R;
      const TT *gtab = tables + c.table_base + (int64_t)f0 * S;
      const T *grow = r_cur + c.msg_base + (int64_t)f0 * R;
      // 8-bit codes: every class is padded to whole tiles (maxsum_warp_plan_tab8), so the tail tile loads all NF
      // tables too and its size stays a multiple of 16 (there is no 1-byte cp.async to fall back on)
      const uint32_t tb = (uint32_t)((C::NARROW ? NF : nf) * S) * (uint32_t)sizeof(TT);
      const uint32_t rb = (uint32_t)(nf * R) * (uint32_t)sizeof(T);
      const bool tma_t = (tb % 16 == 0), tma_r = (rb % 16 == 0);   // bases are 128-byte aligned, tiles 16 factors
      if (lane == 0) {
        mbar_expect_tx(&bars[s], (tma_t ? tb : 0u) + (tma_r ? rb : 0u));
        if (tma_t) tma_load_1d(tab, gtab, tb, &bars[s]);
        if (tma_r) tma_load_1d(rt, grow, rb, &bars[s]);
      }
      if constexpr (!C::NARROW)
        if (!tma_t) for (int i = lane; i < nf * S; i += 32) cp_async_b<(int)sizeof(T)>(tab + i, gtab + i);
      if (!tma_r) for (int i = lane; i < nf * R; i += 32) cp_async_b<(int)sizeof(T)>(rt + i, grow + i);
#pragma unroll
      for (int it = 0; it < PIECES; ++it) {
        const int pc = it * 32 + lane;
        const int row = pc / PIECES, piece = pc - row * PIECES;
        const OffT ro = __shfl_sync(0xffffffffu, qo, row & 31);
        if (row < 2 * nf) cp_async_b<C::VR_BYTES>(qt + row * D + piece * VR, q_cur + (int64_t)ro + piece * VR);
      }
    }
    cp_async_commit();
  };

  const T lam = (T)p.damping, oml = (T)p.one_minus_damping, stab = (T)p.stability;
  const T init = MX ? -Inf<T>::pos() : Inf<T>::pos();
  // lane -> (factor, half): the 16 lanes of a half-warp walk 16 different factors, whose stride (D*D elements = an
  // odd number of 16-byte units for D = 6, 10) spreads a quarter-warp's 128-bit reads over all 32 banks; the first
  // mapping (half in the low lane bit) had 43 % conflict wavefronts.  The partner of a lane is lane ^ 16.
  const int fl = lane & 15, h = lane >> 4;
  T *out0 = reinterpret_cast<T *>(stage0 + (size_t)NS * C::STAGE_BYTES);

  // prologue: tiles 0 .. NS-2 in flight, gather offsets of tile NS-1 and counters of tile 0 on their way
#pragma unroll 1
  for (int k = 0; k < NS - 1; ++k) issue(k, load_qo(k));
  OffT qo_next = load_qo(NS - 1);
  uint8_t cnt = load_cnt(0);
  int64_t pdst = 0;
  if constexpr (PEER) pdst = load_dst(0);

#pragma unroll 1
  for (int k = 0; k < n_my; ++k) {
    const int s = k % NS;
    // tile k+NS-1 goes into the stage tile k-1 held (all lanes are past its reads: they met at the __syncwarp
    // before its store); the OUTPUT buffer of this trip was last used by tile k-2: at most one store pending
    if (lane == 0) tma_store_wait_read1();
    __syncwarp();
    issue(k + NS - 1, qo_next);
    const OffT qo_n2 = load_qo(k + NS);
    const uint8_t cnt_n = load_cnt(k + 1);
    int64_t pdst_n = 0;
    if constexpr (PEER) pdst_n = load_dst(k + 1);
    cp_async_wait_group<NS - 1>();                  // my gathers of tile k have landed ...
    mbar_wait(&bars[s], (uint32_t)((k / NS) & 1));  // ... and its bulk copies
    __syncwarp();                                   // ... and every other lane's gathers

    const int f0 = (gw + k * nw) * NF;
    const int nf = min(NF, c.n_factors - f0);
    const TT *tab = stage_tab(s);
    T *rt = stage_rt(s);
    const T *qt = rt + NF * R;
    const bool act = fl < nf;
    // counters were loaded lane = edge index (2 f + j): fetch both edges of my factor
    uint8_t c0 = (uint8_t)__shfl_sync(0xffffffffu, (unsigned)cnt, 2 * fl);
    uint8_t c1 = (uint8_t)__shfl_sync(0xffffffffu, (unsigned)cnt, 2 * fl + 1);
    // cc / pp: [0, HD) = my values of the message towards position 0 (at my ROW indices), [HD, 2 HD) = my
    // half of the message towards position 1
    T cc[2 * HD], pp[2 * HD];
    T part[D];   // optima over MY rows of T[x0][x1] + q0[x0], per x1
#pragma unroll
    for (int x = 0; x < D; ++x) part[x] = init;
#pragma unroll
    for (int i = 0; i < 2 * HD; ++i) { cc[i] = init; pp[i] = (T)0; }
    if (act) {
      const TT *tf = tab + fl * S;
      T q0[D], q1[D];
      {
        T qq[2 * D];
        ld_row<T, 2 * D, C::V2>(qt + (2 * fl) * D, qq);   // the factor's two q rows are adjacent
#pragma unroll
        for (int x = 0; x < D; ++x) { q0[x] = qq[x]; q1[x] = qq[D + x]; }
      }
      // pairs of rows: one vector read of 2*D elements, both marginals from it
#pragma unroll
      for (int pi = 0; pi < C::NPAIR; ++pi) {
        constexpr int dummy = 0;
        (void)dummy;
        const int ra = h == 0 ? f2vw_row<D>(0, 2 * pi) : f2vw_row<D>(1, 2 * pi);   // rows ra, ra + 1
        T rows[2 * D];
        ld_tab<T, 2 * D, C::TV2_BYTES>(tf + ra * D, rows);
        // q0[ra], q0[ra + 1] with static register indices: h selects between two compile-time candidates
        const T qa = h == 0 ? q0[f2vw_row<D>(0, 2 * pi)] : q0[f2vw_row<D>(1, 2 * pi)];
        const T qb = h == 0 ? q0[f2vw_row<D>(0, 2 * pi) + 1] : q0[f2vw_row<D>(1, 2 * pi) + 1];
        const P qa2 = pmake<T>(qa, qa), qb2 = pmake<T>(qb, qb);
        T a0[D], a1[D];
#pragma unroll
        for (int x = 0; x < D; x += 2) {
          const P ta = pmake<T>(rows[x], rows[x + 1]), tb2 = pmake<T>(rows[D + x], rows[D + x + 1]);
          const P q1p = pmake<T>(q1[x], q1[x + 1]);
          const P sa = padd(ta, q1p), sb = padd(tb2, q1p);     // towards position 0: T + q1[x1]
          a0[x] = sa.x; a0[x + 1] = sa.y;
          a1[x] = sb.x; a1[x + 1] = sb.y;
          const P ua = padd(ta, qa2), ub = padd(tb2, qb2);     // towards position 1: T + q0[x0]
          part[x] = opt3<MX>(part[x], ua.x, ub.x);
          part[x + 1] = opt3<MX>(part[x + 1], ua.y, ub.y);
        }
        // from the +/-inf start like the reference: an output whose candidates are all NaN stays +/-inf
        cc[2 * pi] = opt2<MX>(init, opt_tree3<MX, T, D>(a0));
        cc[2 * pi + 1] = opt2<MX>(init, opt_tree3<MX, T, D>(a1));
      }
      if constexpr (C::SINGLE) {
        const int ra = h == 0 ? f2vw_row<D>(0, HD - 1) : f2vw_row<D>(1, HD - 1);
        T row[D], a0[D];
        ld_tab<T, D, C::TV1_BYTES>(tf + ra * D, row);
        const T qa = h == 0 ? q0[f2vw_row<D>(0, HD - 1)] : q0[f2vw_row<D>(1, HD - 1)];
        const P qa2 = pmake<T>(qa, qa);
#pragma unroll
        for (int x = 0; x < D; x += 2) {
          const P ta = pmake<T>(row[x], row[x + 1]);
          const P sa = padd(ta, pmake<T>(q1[x], q1[x + 1]));
          a0[x] = sa.x; a0[x + 1] = sa.y;
          const P ua = padd(ta, qa2);
          part[x] = opt2<MX>(part[x], ua.x);
          part[x + 1] = opt2<MX>(part[x + 1], ua.y);
        }
        cc[HD - 1] = opt2<MX>(init, opt_tree3<MX, T, D>(a0));
      }
    }
    // complete position 1: I keep x1 in [h*HD, (h+1)*HD), the partner lane sends its partial optima for it
#pragma unroll
    for (int i = 0; i < HD; ++i) {
      const T mine = h == 0 ? part[i] : part[HD + i];
      const T give = h == 0 ? part[HD + i] : part[i];
      const T got = __shfl_xor_sync(0xffffffffu, give, 16);
      cc[HD + i] = opt2<MX>(mine, got);
    }
    bool m0 = false, m1 = false;
    if (act) {
      // previous messages: position 0 at my ROW indices, position 1 at my half
#pragma unroll
      for (int i = 0; i < HD; ++i) {
        const int x0 = h == 0 ? f2vw_row<D>(0, i) : f2vw_row<D>(1, i);
        pp[i] = rt[fl * R + x0];
        pp[HD + i] = rt[fl * R + D + h * HD + i];
      }
      if ((c0 & c1 & 1) != 0) {   // both edges hold a previous message (every cycle but the first ones)
        damp_match_pairs2<T, 2 * HD, HD>(cc, pp, p.damp_factors != 0, lam, oml, stab, m0, m1);
      } else {
        T ca[HD], cb[HD], pa[HD], pb[HD];
#pragma unroll
        for (int i = 0; i < HD; ++i) { ca[i] = cc[i]; cb[i] = cc[HD + i]; pa[i] = pp[i]; pb[i] = pp[HD + i]; }
        m0 = damp_match_row<T, HD>(ca, pa, (c0 & 1) != 0, p.damp_factors != 0, lam, oml, stab);
        m1 = damp_match_row<T, HD>(cb, pb, (c1 & 1) != 0, p.damp_factors != 0, lam, oml, stab);
#pragma unroll
        for (int i = 0; i < HD; ++i) { cc[i] = ca[i]; cc[HD + i] = cb[i]; }
      }
    }
    const unsigned mm = (m0 ? 1u : 0u) | (m1 ? 2u : 0u);
    const unsigned mo = __shfl_xor_sync(0xffffffffu, mm, 16);
    T *ot = out0 + (k & 1) * C::OUT;   // the bulk store of tile k-2 has finished reading it (waited above: <= 1 pending)
    if (act) {
      const bool s0 = gate_decide((mm & mo & 1u) != 0, c0);
      const bool s1 = gate_decide((mm & mo & 2u) != 0, c1);
#pragma unroll
      for (int i = 0; i < HD; ++i) {
        const int x0 = h == 0 ? f2vw_row<D>(0, i) : f2vw_row<D>(1, i);
        ot[fl * R + x0] = s0 ? cc[i] : pp[i];
        ot[fl * R + D + h * HD + i] = s1 ? cc[HD + i] : pp[HD + i];
      }
      const int e = c.first_edge + f0 * 2 + 2 * fl + h;   // edge (f, j = h)
      r_cnt[e] = h == 0 ? c0 : c1;
      if (r_sent) r_sent[e] = (h == 0 ? s0 : s1) ? 1 : 0;
    }
    const uint32_t ob = (uint32_t)(nf * R) * (uint32_t)sizeof(T);
    T *gout = r_next + c.msg_base + (int64_t)f0 * R;
    if (ob % 16 == 0) {
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        tma_store_1d(gout, ot, ob);
        tma_store_commit();
      }
    } else {
      __syncwarp();
      for (int i = lane; i < nf * R; i += 32) gout[i] = ot[i];
      __syncwarp();
    }
    if constexpr (PEER) peer_store_row<T, D>(pdst, ot + lane * D);   // lane = local edge 2 f + j: its finished row (all lanes met above)
    qo_next = qo_n2;
    cnt = cnt_n;
    pdst = pdst_n;
  }
  cp_async_wait_all();
  if (lane == 0) tma_store_wait_read();
}

// Launch shape of the 8-bit table instantiations (PYDCOP_B200_F2VW_CPS / _NS override both widths): a stage is half
// the size of a full-width one, so more CTAs and stages keep the same bytes in flight (sweep on C2: DESIGN.md §5)
#define FG_F2VW8_CPS 4
#define FG_F2VW8_NS 3
// the fused halo's peer-store kernel (PEER = true) is compiled at the default depth of each table width only
#define FG_F2VW_PEER_NS(T, TT) (sizeof(TT) < sizeof(T) ? FG_F2VW8_NS : 2)

// tables: dev_tables (TT = T) or the 8-bit copy (TT = int8_t; c.table_base is then the class's byte offset in it)
template <typename T, typename TT, int D, int NS_, bool MX>
inline bool launch_f2v_warp_ns(bool probe, const fg_class_t &c, const TT *tables, const fg_maxsum_desc_t &d, const T *q_cur,
                               const T *r_cur, T *r_next, const MaxSumParams &p, cudaStream_t st) {
  using C = F2VWarpCfg<T, TT, D, NS_>;
  if constexpr (!C::OK) {
    return false;
  } else {
    if (probe) return true;
    auto kern = k_f2v_warp<T, TT, D, NS_, MX, uint32_t>;
    struct Launch { int per_sm = 0, n_sm = 0; bool peer_attr = false; };
    static std::vector<Launch> per_dev;  // one per instantiation and device
    Launch &L = fg_per_device(per_dev);
    if (!L.per_sm) {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
      int dev = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&L.n_sm, cudaDevAttrMultiProcessorCount, dev);
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&L.per_sm, kern, C::WARPS * 32, C::SMEM);
      if (L.per_sm < 1) L.per_sm = 1;
      // CTAs of 2 warps; the variable side shares the SMs
      const int cap = fg_env_int("PYDCOP_B200_F2VW_CPS", C::NARROW ? FG_F2VW8_CPS : 3);
      if (L.per_sm > cap) L.per_sm = cap;
    }
    const int n_tiles = (c.n_factors + C::NF - 1) / C::NF;
    const int need = (n_tiles + C::WARPS - 1) / C::WARPS;
    const unsigned blocks = (unsigned)std::min(need, L.n_sm * L.per_sm);
    if (p.edge_dst != nullptr) {   // fused halo: only the PEER instantiation stores the boundary rows
      if constexpr (NS_ == FG_F2VW_PEER_NS(T, TT)) {
        auto kp = k_f2v_warp<T, TT, D, NS_, MX, uint32_t, true>;
        if (!L.peer_attr) {
          cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
          L.peer_attr = true;
        }
        kp<<<blocks, C::WARPS * 32, C::SMEM, st>>>(c, tables, q_cur, r_cur, r_next, d.dev_edge_qoff32,
                                                  d.dev_r_cnt, d.dev_r_sent, p);
        return true;
      } else {
        return false;   // not compiled at this depth (launch_f2v_warp never asks): the caller reports an error
      }
    }
    kern<<<blocks, C::WARPS * 32, C::SMEM, st>>>(c, tables, q_cur, r_cur, r_next, d.dev_edge_qoff32,
                                                d.dev_r_cnt, d.dev_r_sent, p);
    return true;
  }
}

// pipeline depth: PYDCOP_B200_F2VW_NS = 2 | 3 | 4 stages per warp (default 2, FG_F2VW8_NS for 8-bit tables),
// shallower when it does not fit.  A fused-halo launch (p.edge_dst set) always runs at the depth its peer-store kernel
// is compiled at.
template <typename T, typename TT, int D>
inline bool launch_f2v_warp(bool probe, const fg_class_t &c, const TT *tables, const fg_maxsum_desc_t &d, const T *q_cur,
                            const T *r_cur, T *r_next, const MaxSumParams &p, cudaStream_t st) {
  constexpr int NSP = FG_F2VW_PEER_NS(T, TT);
  static_assert(!F2VWarpCfg<T, TT, D, 2>::OK || F2VWarpCfg<T, TT, D, NSP>::OK,
                "every shape of the warp kernel has its peer-store instantiation");
  if (!probe && p.edge_dst != nullptr)
    return p.mode_max ? launch_f2v_warp_ns<T, TT, D, NSP, true>(false, c, tables, d, q_cur, r_cur, r_next, p, st)
                      : launch_f2v_warp_ns<T, TT, D, NSP, false>(false, c, tables, d, q_cur, r_cur, r_next, p, st);
  static const int ns = fg_env_int("PYDCOP_B200_F2VW_NS", sizeof(TT) < sizeof(T) ? FG_F2VW8_NS : 2);
#define FG_TRY(NS_)                                                                                              \
  if (p.mode_max ? launch_f2v_warp_ns<T, TT, D, NS_, true>(probe, c, tables, d, q_cur, r_cur, r_next, p, st)    \
                 : launch_f2v_warp_ns<T, TT, D, NS_, false>(probe, c, tables, d, q_cur, r_cur, r_next, p, st))  \
    return true;
  if (ns >= 4) { FG_TRY(4) }
  if (ns >= 3) { FG_TRY(3) }
  FG_TRY(2)
#undef FG_TRY
  return false;
}

// binary classes over one even domain size; probe == true: only report whether the kernel exists.
// tab8 != nullptr: the class's tables are read from the 8-bit copy at byte offset tab8_base
template <typename T>
inline bool dispatch_f2v_warp(bool probe, const fg_class_t &c, const fg_maxsum_desc_t &d, const int8_t *tab8, int64_t tab8_base,
                              const T *q_cur, const T *r_cur, T *r_next, const MaxSumParams &p, cudaStream_t st) {
  if (c.arity != 2 || c.dom[0] != c.dom[1]) return false;
  fg_class_t c8 = c;
  c8.table_base = tab8_base;
  switch (c.dom[0]) {
#define X(n)                                                                                               \
  case n:                                                                                                  \
    return tab8 ? launch_f2v_warp<T, int8_t, n>(probe, c8, tab8, d, q_cur, r_cur, r_next, p, st)           \
                : launch_f2v_warp<T, T, n>(probe, c, (const T *)d.dev_tables, d, q_cur, r_cur, r_next, p, st);
    X(4) X(6) X(8) X(10) X(16) X(20)
#undef X
  }
  return false;
}

// the factor side of class ci on the warp kernel, from the 8-bit copy when the class has one
template <typename T>
inline bool launch_f2v_warp_class(const MaxSumWarpPlan &plan, size_t ci, const fg_class_t &c, const fg_maxsum_desc_t &d,
                                  const T *q_cur, const T *r_cur, T *r_next, const MaxSumParams &p, cudaStream_t st) {
  const bool narrow = plan.tab8 != nullptr && plan.tab8_base[ci] >= 0;
  return dispatch_f2v_warp<T>(false, c, d, narrow ? plan.tab8 : nullptr, narrow ? plan.tab8_base[ci] : 0, q_cur, r_cur,
                              r_next, p, st);
}

// Every entry of a class's tables fits int8 (fg_table_entry_fits_i8): *ok stays 1, else it is cleared
template <typename T>
__global__ void k_tab8_check(const T *__restrict__ t, int64_t n, int32_t *__restrict__ ok) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!fg_table_entry_fits_i8<T>(t[i])) { *ok = 0; return; }
}

template <typename T>
__global__ void k_tab8_encode(const T *__restrict__ t, int64_t n, int8_t *__restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int8_t)(int)t[i];
}

// 8-bit copy of the tables of every warp-kernel class whose entries all fit (engine creation; the device must be
// there).  Each class starts on a 128-byte boundary and is padded with zeros to whole 16-factor tiles.  dev_tables
// is left as it is for every other reader.  Synchronises the device: the tables may have been uploaded on any stream.
template <typename T>
inline int maxsum_warp_plan_tab8_t(const fg_maxsum_desc_t &d, const std::vector<fg_class_t> &classes, MaxSumWarpPlan &plan) {
  const size_t n = classes.size();
  plan.tab8_base.assign(n, -1);
  std::vector<size_t> cand;
  for (size_t i = 0; i < n; ++i)
    if (plan.f2v[i] && classes[i].n_factors > 0) cand.push_back(i);
  if (cand.empty()) return FG_OK;
  if (cudaDeviceSynchronize() != cudaSuccess) return FG_ERR_CUDA;
  int32_t *dev_ok = nullptr;
  if (cudaMalloc(reinterpret_cast<void **>(&dev_ok), cand.size() * sizeof(int32_t)) != cudaSuccess) return FG_ERR_CUDA;
  std::vector<int32_t> ok(cand.size(), 1);
  int rc = FG_OK;
  const T *tables = (const T *)d.dev_tables;
  auto grid = [](int64_t m) { return (unsigned)std::min<int64_t>((m + 255) / 256, 4096); };
  if (cudaMemcpy(dev_ok, ok.data(), ok.size() * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) rc = FG_ERR_CUDA;
  for (size_t k = 0; rc == FG_OK && k < cand.size(); ++k) {
    const fg_class_t &c = classes[cand[k]];
    const int64_t m = (int64_t)c.n_factors * c.table_size;
    k_tab8_check<T><<<grid(m), 256>>>(tables + c.table_base, m, dev_ok + k);
  }
  if (rc == FG_OK && cudaMemcpy(ok.data(), dev_ok, ok.size() * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess)
    rc = FG_ERR_CUDA;
  cudaFree(dev_ok);
  if (rc != FG_OK) return rc;
  int64_t total = 0;
  for (size_t k = 0; k < cand.size(); ++k) {
    if (!ok[k]) continue;
    const fg_class_t &c = classes[cand[k]];
    plan.tab8_base[cand[k]] = total;
    total += ((int64_t)(c.n_factors + 15) / 16 * 16 * c.table_size + 127) / 128 * 128;
  }
  if (total == 0) return FG_OK;
  if (cudaMalloc(reinterpret_cast<void **>(&plan.tab8), (size_t)total) != cudaSuccess) return FG_ERR_CUDA;
  plan.tab8_bytes = total;
  if (cudaMemset(plan.tab8, 0, (size_t)total) != cudaSuccess) return FG_ERR_CUDA;
  for (size_t k = 0; k < cand.size(); ++k) {
    if (!ok[k]) continue;
    const fg_class_t &c = classes[cand[k]];
    const int64_t m = (int64_t)c.n_factors * c.table_size;
    k_tab8_encode<T><<<grid(m), 256>>>(tables + c.table_base, m, plan.tab8 + plan.tab8_base[cand[k]]);
  }
  if (cudaDeviceSynchronize() != cudaSuccess) return FG_ERR_CUDA;
  return FG_OK;
}

inline int maxsum_warp_plan_tab8(const fg_maxsum_desc_t &d, const std::vector<fg_class_t> &classes, MaxSumWarpPlan &plan) {
  return d.precision == FG_F64 ? maxsum_warp_plan_tab8_t<double>(d, classes, plan)
                               : maxsum_warp_plan_tab8_t<float>(d, classes, plan);
}

// factor classes the warp kernel takes over from the round-1 pipelined kernel
inline void maxsum_warp_plan_f2v(const fg_maxsum_desc_t &d, const std::vector<fg_class_t> &classes,
                                 const MaxSumFastPlan &fast, MaxSumWarpPlan &plan) {
  plan.f2v.assign(classes.size(), 0);
  const char *e = getenv("PYDCOP_B200_F2V");
  if (!fast.off32 || fg_fast_disabled() || (e && e[0] == 'p')) return;
  MaxSumParams dummy{};
  for (size_t i = 0; i < classes.size(); ++i) {
    if (classes[i].flags & FG_CLASS_GHOST) continue;
    const bool ok = d.precision == FG_F64
                        ? dispatch_f2v_warp<double>(true, classes[i], d, nullptr, 0, nullptr, nullptr, nullptr, dummy, nullptr)
                        : dispatch_f2v_warp<float>(true, classes[i], d, nullptr, 0, nullptr, nullptr, nullptr, dummy, nullptr);
    if (ok) plan.f2v[i] = 1;
  }
}
