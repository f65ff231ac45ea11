/* pydcop_b200 — C-ABI of the factor-graph message-passing engine (H100, sm_90a).
 *
 * The reference (Orange-OpenSource/pyDcop) is pure Python and has NO FFI: its boundary for this
 * path is the algorithm-module surface `pydcop.algorithms.<name>` (GRAPH_TYPE / algo_params /
 * build_computation / computation_memory / communication_load,
 * pydcop/algorithms/__init__.py:508-566, pydcop/infrastructure/computations.py:1156-1165).
 * pydcop_b200/algorithms/{maxsum_gpu,dsa_gpu}.py implement that surface; THIS header is the
 * boundary one level below it: what a reference maintainer binds with ctypes (INTEGRATION.md) to
 * replace, for all edges at once, the per-computation Python hot loops cited on each entry point.
 *
 * Conventions
 *   - plain C, opaque handles, int return codes (0 = FG_OK), no exceptions, no torch types;
 *   - every `dev_*` pointer is CALLER-OWNED DEVICE memory (the Python host passes
 *     torch.Tensor.data_ptr()); the only device memory the library owns is the DSA handle's copy
 *     of the class table (a few hundred bytes) and a MaxSum handle's class table of the variable side
 *     (48 bytes per (domain, degree) class); a MaxSum handle also owns one side stream + 2 events;
 *   - a handle belongs to the device current when fg_*_create is called: every call on the handle
 *     runs on that device (it is made current for the call, the caller's device restored on
 *     return), and every non-NULL dev_* array of its descriptor must be device memory of that
 *     device — create returns FG_ERR_ARG, naming the field, for host memory or another device's;
 *     calls without a handle run on the current device and refuse a main array that lives
 *     elsewhere; fg_enable_peer_access / fg_ipc_import / fg_halo_push take the current device as
 *     the accessor by design;
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream), a stream
 *     of the handle's device;
 *   - all calls are asynchronous on `stream`; the caller synchronises;
 *   - value type T is float (precision = FG_F32) or double (FG_F64) for every cost/message array;
 *   - there is NO CPU fallback: without a CUDA device every launch entry point returns
 *     FG_ERR_CUDA and fg_last_error() says why.
 *
 * Data layout (DESIGN.md §3): factors are grouped into CLASSES of identical shape
 * (arity, domain sizes).  Inside a class everything is affine in the factor index f:
 *   table of f        = dev_tables + table_base + f * table_size          (row-major, axis i <->
 *                                                                           scope position i)
 *   message row (f,j) = msg_base + f * row_total + row_off[j], length dom[j]
 *                       (rows of a class whose positions have DIFFERENT domain sizes start on
 *                       4-element boundaries; uniform classes are dense: row_off[j] = j * dom)
 * (this is the layout of the factor->variable array r, written by the factor side).  The variable
 * side owns a CSR: variable v has slots [var_ptr[v], var_ptr[v+1]) in the reference's `links` order
 * (pydcop/algorithms/maxsum.py:466); the variable->factor array q is stored in SLOT order:
 *   q row of slot s   = var_qbase[v] + (s - var_ptr[v]) * dom_size[v]
 * so each side WRITES its own messages with perfectly coalesced stores and reads the other side's
 * through one gather index: edge_qoff[e] (factor side reads q), slot_roff[s] (variable side reads r).
 * Variables are stored class-major too (classes of identical (domain size, degree), fg_varclass_t);
 * dev_value / dev_value_cost are in that internal variable order (the Python host keeps the
 * permutation, pydcop_b200/layout.py).
 */
#ifndef PYDCOP_B200_H
#define PYDCOP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FG_ABI_VERSION 3
#define FG_MAX_ARITY 8
#define FG_MAX_DOM 256

enum { FG_OK = 0, FG_ERR_ARG = 1, FG_ERR_CUDA = 2, FG_ERR_UNSUPPORTED = 3 };
enum { FG_F32 = 0, FG_F64 = 1 };
enum { FG_START_LEAFS = 0, FG_START_LEAFS_VARS = 1, FG_START_ALL = 2 }; /* maxsum.py:219 */
enum { FG_DSA_A = 0, FG_DSA_B = 1, FG_DSA_C = 2 };                      /* dsa.py:133 */
#define FG_MAX_PSETS 65535   /* parameter sets of one handle: indices are uint16 */
enum { FG_CLASS_GHOST = 1, FG_CLASS_BOUNDARY = 2 };

/* One class of same-shaped factors (constraints). */
typedef struct {
  int32_t arity;                 /* 1..FG_MAX_ARITY */
  int32_t dom[FG_MAX_ARITY];     /* domain size per scope position */
  int32_t row_off[FG_MAX_ARITY]; /* offset of position j's message row inside a factor's rows */
  int32_t row_total;             /* elements of one factor's rows: sum(dom), or with every row padded to 4 elements when the scope mixes domain sizes */
  int32_t n_factors;
  int32_t flags;                 /* FG_CLASS_GHOST: rows exist but the class is never computed
                                    (multi-GPU halo stubs, filled by the exchange) */
  int32_t first_factor;          /* global factor index of the first factor of the class */
  int32_t first_edge;            /* global edge index of its first edge; edge(f,j)=first_edge+f*arity+j */
  int64_t table_size;            /* prod(dom) */
  int64_t table_base;            /* element offset into dev_tables */
  int64_t msg_base;              /* element offset into the message arrays */
} fg_class_t;

/* One class of same-shaped variables: identical domain size and degree.  Variables are stored in
 * class-major ("internal") order; inside a class everything is affine in the variable's rank i:
 *   unary row   = dev_unary + unary_base + i * dom
 *   slots       = first_slot + i * degree + g            (g = 0..degree-1, the `links` order)
 *   q row (i,g) = q_base + (i * degree + g) * dom
 * degree == -1 marks the irregular class (variables of degree > 16): CSR through dev_var_ptr,
 * q rows still dense from q_base in slot order. */
typedef struct {
  int32_t dom, degree;
  int32_t n_vars, first_var, first_slot;
  int32_t n_slots;     /* total slots of the class */
  int32_t flags, reserved;  /* FG_CLASS_GHOST as above */
  int64_t unary_base;
  int64_t q_base;
} fg_varclass_t;

/* ------------------------------------------------------------------------------------------
 * MaxSum  (replaces MaxSumFactorComputation.on_new_cycle maxsum.py:339-379 +
 * factor_costs_for_var :382-447, MaxSumVariableComputation.on_new_cycle :525-565 +
 * select_value :584-620 + costs_for_factor :623-676, apply_damping :679-685, approx_match
 * :688-710, and both on_start methods :305-328, :495-523 — for ALL factors/variables at once)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t abi_version; /* FG_ABI_VERSION */
  int32_t precision;   /* FG_F32 | FG_F64 */
  int32_t n_vars, n_factors, n_edges, n_classes;
  int64_t n_msg_r;     /* elements of each r buffer (class-major edge order, padded bases) */
  int64_t n_msg_q;     /* elements of each q buffer (slot order) */
  int32_t uniform_dom; /* D if every variable has domain size D, else 0 (enables fast kernels) */
  int32_t max_degree;  /* largest number of factors on one variable */
  const fg_class_t *classes; /* HOST array [n_classes], copied by fg_maxsum_create */
  int32_t n_varclasses, reserved0;
  const fg_varclass_t *varclasses; /* HOST array [n_varclasses], copied by fg_maxsum_create */

  /* problem (device, read-only) */
  const void *dev_tables;       /* T[sum table_size] */
  const void *dev_unary;        /* T[sum dom_size]  variable costs (+noise), maxsum.py:477-487 */
  const int32_t *dev_dom_size;  /* [n_vars] */
  const int64_t *dev_unary_off; /* [n_vars+1] */
  const int32_t *dev_var_ptr;   /* [n_vars+1] */
  const int64_t *dev_var_qbase; /* [n_vars+1] q offset of the first slot of v */
  const int64_t *dev_slot_roff; /* [n_edges] slot order: offset in r of the row of slot s's edge */
  const int64_t *dev_edge_qoff; /* [n_edges] edge order: offset in q of the row of edge e */
  const uint32_t *dev_slot_roff32; /* same as 32-bit offsets, or NULL when they do not fit */
  const uint32_t *dev_edge_qoff32;
  const int32_t *dev_slot_edge; /* [n_edges] edge id of slot s */
  const int32_t *dev_slot_var;  /* [n_edges] variable of slot s */
  const int32_t *dev_init_value; /* [n_vars] initial_value index or -1 (maxsum.py:497-500) */

  /* state (device, read-write).  q = variable->factor, r = factor->variable; [0]/[1] are the
   * Jacobi double buffers, the engine tracks which one is current. */
  void *dev_q[2], *dev_r[2];       /* T[n_msg_q] / T[n_msg_r] each */
  uint8_t *dev_q_valid, *dev_r_valid; /* [n_edges] edge order: receiver holds a message */
  uint8_t *dev_q_cnt;              /* [n_edges] SLOT order: bit0 has-prev, bits1.. send count */
  uint8_t *dev_r_cnt;              /* [n_edges] edge order: same encoding */
  uint8_t *dev_q_sent, *dev_r_sent; /* [n_edges] q_sent SLOT order, r_sent edge order: message
                                       posted in the last cycle (may be NULL: not recorded) */
  int32_t *dev_value;              /* [n_vars] selected value index (select_value) */
  void *dev_value_cost;            /* T[n_vars] its cost */

  /* algorithm parameters (maxsum.py:212-220) */
  int32_t mode_max;      /* 0 'min', 1 'max' */
  int32_t damp_vars, damp_factors; /* damping_nodes in {vars,both} / {factors,both} */
  int32_t start_messages; /* FG_START_* */
  double damping, stability;
} fg_maxsum_desc_t;

typedef struct fg_maxsum *fg_maxsum_t;

int fg_abi_version(void);
/* Number of CUDA devices visible to the library (0 when none / driver missing). */
int fg_device_count(void);

int fg_maxsum_create(const fg_maxsum_desc_t *desc, fg_maxsum_t *out);
int fg_maxsum_destroy(fg_maxsum_t h);
const char *fg_maxsum_last_error(fg_maxsum_t h);
/* cycle 0: every computation's on_start (maxsum.py:305-328, 495-523). */
int fg_maxsum_init(fg_maxsum_t h, void *stream);
/* n_cycles synchronous cycles (one = every factor's and every variable's on_new_cycle). */
int fg_maxsum_step(fg_maxsum_t h, int32_t n_cycles, void *stream);
/* Split-phase variant for the multi-GPU host loop: launch the compute of ONE cycle (writes the
 * `next` buffers), let the caller exchange halos on them, then commit (swap buffers). */
int fg_maxsum_cycle_compute(fg_maxsum_t h, void *stream);
int fg_maxsum_cycle_commit(fg_maxsum_t h);
/* Index (0/1) of the CURRENT message buffers and the number of cycles done so far. */
int fg_maxsum_current(fg_maxsum_t h, int32_t *buf_index, int64_t *cycle);
/* Number of kernel launches issued by this handle so far (bench.py's gpu_launches). */
int64_t fg_maxsum_launch_count(fg_maxsum_t h);
/* Which kernel family computes each factor class from cycle 2 on (diagnostic; -1 = ghost class, never computed):
 * generic one-thread-per-edge, round-1 CTA-pipelined (compile-time shape), warp-autonomous (binary, even domain),
 * runtime-dimension tiled (any other shape whose table fits shared memory). */
enum { FG_KERNEL_GENERIC = 0, FG_KERNEL_PIPE = 1, FG_KERNEL_WARP = 2, FG_KERNEL_TILED_RT = 3 };
int fg_maxsum_kernel_plan(fg_maxsum_t h, int32_t *family, int32_t n_classes);

/* Bytes per stored table entry that the factor side reads for each class (diagnostic): 1 where the warp kernel reads
 * an 8-bit copy made at creation — every entry of the class an integer in [-128, 127], none -0.0, NaN or inf, so the
 * messages are the same bit for bit — else the value width (4 or 8).  The copy is taken once by fg_maxsum_create:
 * writes to dev_tables after creation are not seen by those classes. */
int fg_maxsum_table_width(fg_maxsum_t h, int32_t *bytes, int32_t n_classes);

/* Gather / scatter of boundary message rows for the halo exchange (replaces
 * Messaging.post_msg for cut edges, pydcop/infrastructure/communication.py:588-698).
 * rows: `n_rows` (offset,len) pairs in dev_row_off/dev_row_len; packed back to back. */
int fg_halo_pack(int32_t precision, const void *dev_src, void *dev_packed,
                 const int64_t *dev_row_off, const int64_t *dev_packed_off,
                 const int32_t *dev_row_len, int64_t n_rows, void *stream);
int fg_halo_unpack(int32_t precision, void *dev_dst, const void *dev_packed,
                   const int64_t *dev_row_off, const int64_t *dev_packed_off,
                   const int32_t *dev_row_len, int64_t n_rows, void *stream);

/* Uniform-domain fast form of the two calls above, r and q rows in ONE launch.  The packed
 * buffer is the all_to_all buffer: for peer p the block [r rows for p | q rows for p] starts at
 * element peer_base[p]; rows of the r list [peer_r_start[p], peer_r_start[p+1]) and of the q list
 * [peer_q_start[p], peer_q_start[p+1]) belong to peer p (HOST arrays of n_peers+1 / n_peers
 * entries, n_peers <= 16).  pack != 0: arrays -> packed; pack == 0: packed -> arrays. */
int fg_halo_rows_uniform(int32_t precision, int32_t pack, void *dev_r, void *dev_q, void *dev_packed,
                         const int64_t *dev_row_off_r, const int64_t *dev_row_off_q, int64_t n_r,
                         int64_t n_q, int32_t dom, int32_t n_peers, const int64_t *peer_r_start,
                         const int64_t *peer_q_start, const int64_t *peer_base, void *stream);

/* Direct halo push over NVLink peer memory (uniform domain): row i of the r list
 * (dev_r + row_off_r[i], `dom` elements) is stored at the ABSOLUTE device address dst_r[i] — a
 * location inside the consuming rank's `next` buffer, mapped into this process through CUDA IPC —
 * and likewise for the q list.  One launch replaces pack -> NCCL all_to_all -> unpack; the caller
 * closes the cycle with a barrier. */
/* Enable stores from the CURRENT device into `peer_device`'s memory (cudaDeviceEnablePeerAccess);
 * returns FG_ERR_UNSUPPORTED when the pair has no peer path. */
int fg_enable_peer_access(int32_t peer_device);
/* CUDA IPC for the peer push: export = IPC handle (64 bytes) of the allocation containing dev_ptr
 * and dev_ptr's byte offset inside it; import = map a peer's allocation into THIS process with the
 * current device as accessor (cudaIpcMemLazyEnablePeerAccess), returning its base address. */
int fg_ipc_export(const void *dev_ptr, unsigned char handle_out[64], int64_t *offset_out);
int fg_ipc_import(const unsigned char handle[64], void **base_out);
int fg_ipc_close(void *base);
int fg_halo_push(int32_t precision, const void *dev_r, const void *dev_q, const int64_t *dev_row_off_r,
                 const int64_t *dev_row_off_q, const int64_t *dev_dst_r, const int64_t *dev_dst_q,
                 int64_t n_r, int64_t n_q, int32_t dom, void *stream);

/* ------------------------------------------------------------------------------------------
 * DSA  (replaces DsaComputation.on_start dsa.py:277-299 and evaluate_cycle :320-357 with
 * find_optimal relations.py:1594-1638, assignment_cost :1479-1532, variant_a/b/c dsa.py:359-405,
 * probabilistic_change :407-417, exists_violated_constraint :419-431, find_optimum
 * relations.py:1367-1400 — for ALL variables at once).  Random draws are Philox4x32-10 keyed by
 * (seed; variable, cycle): u = 53-bit uniform, choice = (word*n)>>32 (oracle/philox.py).
 * ------------------------------------------------------------------------------------------ */
/* one parameter set of a DSA / A-DSA handle: the decision rule (the probability reaches the kernels as dev_prob) */
typedef struct {
  int32_t variant;               /* FG_DSA_* */
} fg_dsa_pset_t;

typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_factors, n_edges, n_classes;
  const fg_class_t *classes;     /* HOST [n_classes] */
  const void *dev_tables;        /* T[...] */
  const int32_t *dev_dom_size;   /* [n_vars] */
  const int32_t *dev_var_id;     /* [n_vars] caller's (canonical) id of each internal variable: the
                                    Philox counter, so draws do not depend on the internal order */
  const int32_t *dev_edge_var;   /* [n_edges] variable of edge e (class-major edge order) */
  const int32_t *dev_edge_class; /* [n_edges] class of edge e */
  const int32_t *dev_var_ptr;    /* [n_vars+1] */
  const int32_t *dev_slot_edge;  /* [n_edges] incident edges of v in node.constraints order */
  const uint8_t *dev_has_nbr;    /* [n_vars] 1: variable has >= 1 neighbour (dsa.py:278); 0: isolated, its
                                    value is carried over; 2: ghost of a variable another rank owns (multi-GPU):
                                    never written by the kernels, filled by the owner's push / halo unpack */
  const double *dev_prob;        /* [n_vars] change threshold (p_mode fixed|arity, dsa.py:252-263) */
  void *dev_con_opt;             /* T[n_factors] per-constraint optimum, filled by fg_dsa_init */
  /* optional fast path: every constraint binary over one domain size `fast_dom` (else NULL / 0).
   * Per slot (variable v, incident constraint c, neighbour u): the table of c ORIENTED so that
   * row y = value of u is contiguous over v's values (position-0 slots read a transposed copy):
   *   cost_v[x] += dev_tables_or[slot_tab[s] + y * fast_dom + x] */
  const void *dev_tables_or;     /* T[...] original tables followed by the transposed copies */
  const int32_t *dev_slot_nbr;   /* [n_edges] neighbour variable of slot s */
  const int64_t *dev_slot_tab;   /* [n_edges] element offset of the oriented table of slot s */
  const void *dev_slot_opt;      /* T[n_edges] optimum of the slot's constraint (variant B) */
  int32_t fast_dom, reserved1;
  int32_t *dev_value[2];         /* [n_vars] current / next value index (double buffer) */
  void *dev_value_cost;          /* T[n_vars] cost reported with the last selection */
  int32_t mode_max, variant;     /* FG_DSA_* */
  int32_t stop_cycle;            /* 0 = never (dsa.py:134,352) */
  uint64_t seed;
  /* A-DSA (pydcop/algorithms/adsa.py:344-377): non-NULL = the variables' own costs T[sum dom] (internal variable
   * order, row of v at dev_unary_off[v]) are added to every CANDIDATE's cost; the current cost (adsa.py:262) and
   * DSA itself (the variable-cost branch of find_optimal is dead code, relations.py:1630) do not use them. */
  const void *dev_var_cost;
  const int64_t *dev_unary_off;  /* [n_vars+1] */
  /* optional, fast path only (csrc/dsa_cached.cuh): the row each slot read last, slot-major T[n_edges * fast_dom],
   * and the neighbour value it belongs to (0xFF = none yet; reset by fg_dsa_init).  A cycle streams these rows and
   * goes to the oriented tables only for the slots whose neighbour changed; results are identical. */
  void *dev_row_cache;
  uint8_t *dev_slot_last;        /* [n_edges] */
  const uint64_t *dev_var_seed;  /* [n_vars] optional: the Philox key of internal variable v, in place of `seed`
                                   (a batch of problems, each run with its own seed); NULL = `seed` for all */
  /* optional parameter sets (a batch of problems, each with its own algorithm parameters): dev_var_pset[v] is the
   * set of internal variable v, an index into the HOST table psets[0 .. n_psets).  create validates every set and
   * copies the table into device memory the handle owns; the kernels read it there.  Both NULL (n_psets 0, anything
   * else is refused): every variable takes the scalar fields above. */
  const uint16_t *dev_var_pset;  /* [n_vars] */
  const fg_dsa_pset_t *psets;
  int32_t n_psets, reserved_ps;
} fg_dsa_desc_t;

typedef struct fg_dsa *fg_dsa_t;

int fg_dsa_create(const fg_dsa_desc_t *desc, fg_dsa_t *out);
int fg_dsa_destroy(fg_dsa_t h);
const char *fg_dsa_last_error(fg_dsa_t h);
/* on_start: per-constraint optima + random initial values (isolated variables keep the value
 * the host stored in dev_value[0], dsa.py:278-289). */
int fg_dsa_init(fg_dsa_t h, void *stream);
/* up to n_cycles evaluate_cycle rounds (stops at stop_cycle). */
int fg_dsa_step(fg_dsa_t h, int32_t n_cycles, void *stream);
int fg_dsa_cycle_compute(fg_dsa_t h, void *stream);
int fg_dsa_cycle_commit(fg_dsa_t h);
int fg_dsa_current(fg_dsa_t h, int32_t *buf_index, int64_t *cycle);
int64_t fg_dsa_launch_count(fg_dsa_t h);

/* ------------------------------------------------------------------------------------------
 * Device-side cycle barrier + fused peer push (multi-GPU; replaces the per-cycle NCCL all_reduce and
 * the host-driven compute -> push -> barrier chain; reference counterpart: the cycle_id handshake of
 * SynchronousComputationMixin, pydcop/infrastructure/computations.py:696-718, and Messaging.post_msg
 * for cut edges, communication.py:588-698).
 *
 * Every rank owns an array of `world` 64-bit EPOCH FLAGS in its own device memory, mapped into the
 * peers through CUDA IPC; slot p is written only by rank p.  After its boundary rows of a cycle are
 * stored in the peers' buffers, a rank releases (fence.sys + st.release.sys) the new epoch into its
 * slot on every peer; before it reads rows the peers wrote it acquires (ld.acquire.sys, spinning)
 * the same epoch from every peer's slot in its own array.  No host round trip, no collective.
 * A wait that does not complete within `timeout_ns` stores peer rank + 1 in *dev_error and returns,
 * so a lost peer cannot hang the device.
 * ------------------------------------------------------------------------------------------ */
#define FG_MAX_PEERS 16
typedef struct {
  int32_t n_peers;                    /* ranks this rank exchanges with (<= FG_MAX_PEERS) */
  int32_t my_rank;
  const uint64_t *dev_flags;          /* MY flag array [world], zeroed by the caller at creation */
  int32_t peer_rank[FG_MAX_PEERS];    /* slot of dev_flags written by peer i */
  uint64_t *peer_slot[FG_MAX_PEERS];  /* address, as mapped into THIS process, of slot my_rank in
                                         peer i's flag array */
  int32_t *dev_error;                 /* one int32, zeroed by the caller */
  uint64_t timeout_ns;                /* 0 = 20 s */
} fg_peer_sync_t;

int fg_peer_signal(const fg_peer_sync_t *ps, uint64_t epoch, void *stream);
int fg_peer_wait(const fg_peer_sync_t *ps, uint64_t epoch, void *stream);

/* Rows a rank pushes every cycle: row i of list r is `dom` elements at dev_r + src_r_off[i] and is
 * stored at the absolute (peer) address dst_r[b][i] when the cycle writes buffer b; likewise q.
 * For DSA the "rows" are single 4-byte values (dom = 1, list r only). */
typedef struct {
  int32_t elem_bytes, dom;
  int64_t n_r, n_q;
  const int64_t *dev_src_r_off, *dev_src_q_off;
  const int64_t *dev_dst_r[2], *dev_dst_q[2];
  uint32_t *dev_counter;              /* one zeroed uint32: last-block detection of the push kernel */
  fg_peer_sync_t sync;
  /* Optional (NULL / 0 = one thread per 4/8/16-byte piece of a row): the push lists cut into RUNS of rows
   * whose destinations are consecutive addresses — the rows one peer receives land in dense blocks of its
   * buffers — so that the kernel can issue whole 16-byte aligned stores over NVLink whatever the row
   * size (rows of 40 bytes would otherwise leave as 8-byte stores).  Per list and buffer index b:
   * dev_runs[b] = int64 [n_runs][4] = (first destination address, index of the run's first row in the
   * list, bytes in the run, index of the run's first 16-byte destination unit), units = total units.
   * Needs row bytes % 8 == 0. */
  const int64_t *dev_runs_r[2], *dev_runs_q[2];
  int32_t n_runs_r[2], n_runs_q[2];
  int64_t units_r[2], units_q[2];
  /* Optional, MaxSum only (NULL = off): FUSED halo.  Per buffer index b, for every edge (class-major order) the
   * address in its consumer's r[b] of the f->v row the factor side produces, and for every slot the address in
   * its consumer's q[b] of the v->f row the variable side produces; 0 = the row stays on this GPU.  When every
   * non-ghost class of the shard runs on the warp-autonomous kernels (csrc/maxsum_warp.cuh), those kernels store
   * each boundary row to its peer from the lane that produced it — the transfer overlaps the rest of the cycle's
   * arithmetic tile by tile and the two push launches disappear; otherwise the push kernels above are used. */
  const int64_t *dev_edge_dst_r[2], *dev_slot_dst_q[2];
} fg_halo_plan_t;

/* Attach a push plan to an engine (copied).  From then on fg_*_shard_step runs whole cycles on the
 * device without the host: compute -> push boundary rows into the peers' `next` buffers, the last
 * block of the push kernel releasing epoch+1 -> wait for every peer's epoch+1 -> commit.  The epoch
 * counter only grows (it survives fg_*_init), so every rank must run the same number of cycles. */
int fg_maxsum_shard_attach(fg_maxsum_t h, const fg_halo_plan_t *plan);
/* 1 when the attached plan runs in FUSED mode (boundary rows stored by the warp kernels), else 0. */
int fg_maxsum_shard_fused(fg_maxsum_t h);
int fg_maxsum_shard_step(fg_maxsum_t h, int32_t n_cycles, void *stream);
/* One phase of a cycle, for timing breakdowns: 0 compute, 1 push + signal, 2 wait, 3 commit. */
int fg_maxsum_shard_phase(fg_maxsum_t h, int32_t phase, void *stream);
/* Diagnostics: n_cycles whole cycles with CUDA timing events INSIDE the cycle (no host work between the
 * kernels), averaged, microseconds: out_us[0] factor side, [1] push of the r rows (split mode),
 * [2] variable side, [3] push of the q rows (split mode), [4] push / release after the join, [5] wait
 * for the peers, [6] whole cycle.  Synchronises the stream after every cycle. */
int fg_maxsum_shard_profile(fg_maxsum_t h, int32_t n_cycles, void *stream, double *out_us);
int fg_dsa_shard_attach(fg_dsa_t h, const fg_halo_plan_t *plan);
int fg_dsa_shard_step(fg_dsa_t h, int32_t n_cycles, void *stream);

/* ------------------------------------------------------------------------------------------
 * MGM  (next-tier row §8f.4; replaces MgmComputation.on_start mgm.py:283-310, the value phase
 * _handle_value_message :343-397 with _compute_best_value :434-455 and find_arg_optimal
 * relations.py:1554-1591, and the gain phase _handle_gain_message :497-537 with the lexicographic
 * tie break :574-591 — for ALL variables at once).  Same constraint-hypergraph arrays as DSA.
 * One cycle = two launches: every variable's best local gain, then every variable's decision.
 * Draws: Philox4x32-10 keyed (seed; canonical variable id, cycle) — cycle 0xffffffff for the
 * initial value, else the 1-based round (the reference's cycle_count when it draws).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_factors, n_edges, n_classes;
  const fg_class_t *classes;      /* HOST [n_classes] */
  const void *dev_tables;         /* T[...] */
  const void *dev_unary;          /* T[...] variable costs (cost_for_val) */
  const int64_t *dev_unary_off;   /* [n_vars+1] */
  const int32_t *dev_dom_size;    /* [n_vars] */
  const int32_t *dev_var_id;      /* [n_vars] canonical id = Philox counter */
  const int32_t *dev_var_rank;    /* [n_vars] position of the variable's NAME in sorted order */
  const int32_t *dev_edge_var;    /* [n_edges] */
  const int32_t *dev_edge_class;  /* [n_edges] */
  const int32_t *dev_var_ptr;     /* [n_vars+1] */
  const int32_t *dev_slot_edge;   /* [n_edges] incident edges of v in node.constraints order */
  const int32_t *dev_nbr_ptr;     /* [n_vars+1] distinct neighbours (mgm.py:245-252) */
  const int32_t *dev_nbr_idx;     /* [nbr_ptr[n_vars]] */
  const int32_t *dev_init_value;  /* [n_vars] value index or -1 (random), may be NULL */
  int32_t *dev_value;             /* [n_vars] in/out; variables without neighbours are preset by the
                                     host (optimal_cost_value, relations.py:1641-1669) */
  void *dev_cost;                 /* T[n_vars] current_cost (preset for isolated variables) */
  uint8_t *dev_has_cost;          /* [n_vars] current_cost is not None */
  void *dev_gain;                 /* T[n_vars] */
  int32_t *dev_new_value;         /* [n_vars] */
  int32_t mode_max;
  int32_t stop_cycle;             /* 0 = never; a run ends when round + 1 >= stop_cycle (mgm.py:404) */
  uint64_t seed;
  /* optional fast shape (opt-in experiment): every constraint binary over one domain size `fast_dom`
   * in {4, 8, 10, 16, 20}; the oriented tables of the DSA fast path (fg_dsa_desc_t) and the number of
   * incidences handled per trip (2 | 4).  All NULL / 0 = the generic value-phase kernel. */
  const void *dev_tables_or;      /* T[...] */
  const int32_t *dev_slot_nbr;    /* [n_edges] */
  const int64_t *dev_slot_tab;    /* [n_edges] */
  int32_t fast_dom, fast_chunk;
  /* optional with the fast shape (csrc/mgm_cached_kernels.cuh): the row each slot read last, slot-major
   * T[n_edges * fast_dom], and the neighbour value it belongs to (0xFF = none yet; reset by fg_mgm_init): the value
   * phase streams these rows and reads the oriented tables only where a neighbour moved; results are identical. */
  void *dev_row_cache;
  uint8_t *dev_slot_last;         /* [n_edges] */
  const uint64_t *dev_var_seed;   /* [n_vars] optional: Philox key of internal variable v; NULL = `seed` */
} fg_mgm_desc_t;

typedef struct fg_mgm *fg_mgm_t;

int fg_mgm_create(const fg_mgm_desc_t *desc, fg_mgm_t *out);
int fg_mgm_destroy(fg_mgm_t h);
const char *fg_mgm_last_error(fg_mgm_t h);
/* on_start for the variables that have neighbours: initial_value or an injected random choice. */
int fg_mgm_init(fg_mgm_t h, void *stream);
/* up to n_cycles value+gain rounds (stops as the reference does at stop_cycle). */
int fg_mgm_step(fg_mgm_t h, int32_t n_cycles, void *stream);
int fg_mgm_current(fg_mgm_t h, int64_t *cycle, int32_t *finished);
int64_t fg_mgm_launch_count(fg_mgm_t h);

/* ------------------------------------------------------------------------------------------
 * MGM-2  (pydcop/algorithms/mgm2.py: coordinated moves of neighbour pairs, for ALL variables at
 * once).  Same constraint-hypergraph arrays as MGM; variable costs are never counted (mgm2.py uses
 * assignment_cost without them).  One cycle = five launches, in the order of the data they need:
 *   1. value phase (:742-785): current cost, best unilateral move, offerer coin and partner pick,
 *      the offerer's table of improving joint moves (own value x partner value, all its constraints)
 *   2. answers (:787-856): every non-offerer scores the offers it got over its constraints that do
 *      not contain the offerer and commits to the best one (favor rule) or to none
 *   3. commit (:858-890): an accepted offerer takes the receiver's value and global gain
 *   4. gain phase (:892-972): GO flags of committed variables, unilateral moves of the others
 *   5. go (:974-1001): a committed pair moves when both sent GO.
 * Draws: Philox4x32-10, counter (canonical variable id, cycle, purpose, 0) — cycle 0xffffffff for
 * the start values (purpose 0), else the 1-based round; purposes 1 offerer coin + partner pick,
 * 2 unilateral value pick, 3 favor "no" coin, 4 offer pick (philox_draw, csrc/philox.cuh).
 * ------------------------------------------------------------------------------------------ */
enum { FG_MGM2_FAVOR_UNILATERAL = 0, FG_MGM2_FAVOR_NO = 1, FG_MGM2_FAVOR_COORDINATED = 2 };

/* one parameter set of an MGM-2 handle */
typedef struct {
  double threshold;               /* finite, in [0, 1] */
  int32_t favor;                  /* FG_MGM2_FAVOR_* */
  int32_t reserved0;
} fg_mgm2_pset_t;

typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_factors, n_edges, n_classes;
  const fg_class_t *classes;      /* HOST [n_classes] */
  const void *dev_tables;         /* T[...] */
  const int32_t *dev_dom_size;    /* [n_vars] */
  const int32_t *dev_var_id;      /* [n_vars] canonical id = Philox counter */
  const int32_t *dev_var_rank;    /* [n_vars] position of the variable's NAME in sorted order */
  const int32_t *dev_edge_var;    /* [n_edges] */
  const int32_t *dev_edge_class;  /* [n_edges] */
  const int32_t *dev_var_ptr;     /* [n_vars+1] */
  const int32_t *dev_slot_edge;   /* [n_edges] incident edges of v in node.constraints order */
  const int32_t *dev_nbr_ptr;     /* [n_vars+1] distinct neighbours, first-appearance order */
  const int32_t *dev_nbr_idx;     /* [nbr_ptr[n_vars]] */
  const int32_t *dev_init_value;  /* [n_vars] value index or -1 (random), may be NULL */
  int32_t *dev_value;             /* [n_vars] in/out */
  void *dev_cost;                 /* T[n_vars] current_cost */
  uint8_t *dev_has_cost;          /* [n_vars] current_cost is not None */
  void *dev_gain;                 /* T[n_vars] potential_gain */
  int32_t *dev_potential_value;   /* [n_vars] */
  void *dev_local_cost;           /* T[n_vars] cost computed in the value phase */
  uint8_t *dev_offerer;           /* [n_vars] the variable made an offer this cycle */
  int32_t *dev_partner;           /* [n_vars] offerer: its partner; committed receiver: its offerer; else -1 */
  uint8_t *dev_committed;         /* [n_vars] */
  uint8_t *dev_go;                /* [n_vars] a committed variable sent GO */
  uint8_t *dev_answer;            /* [n_vars] by offerer: accepted by its partner */
  int32_t *dev_answer_value;      /* [n_vars] by offerer: its value in the accepted joint move */
  void *dev_answer_gain;          /* T[n_vars] by offerer: the receiver's global gain */
  const int64_t *dev_offer_off;   /* [n_vars] start of v's offer table in dev_offer */
  void *dev_offer;                /* T[...] v's table: dom(v) x max dom of its neighbours entries, row
                                     stride dom(partner); an entry not offered holds 0 (an offered gain
                                     is > 0 in min mode, < 0 in max mode) */
  int32_t mode_max;
  int32_t favor;                  /* FG_MGM2_FAVOR_* */
  double threshold;               /* offerer when u < threshold */
  int32_t stop_cycle;             /* 0 = never; a run ends when round + 1 >= stop_cycle (mgm2.py:613) */
  int32_t reserved0;
  uint64_t seed;
  const uint64_t *dev_var_seed;   /* [n_vars] optional: Philox key of internal variable v; NULL = `seed` */
  /* optional parameter sets, as fg_dsa_desc_t's */
  const uint16_t *dev_var_pset;  /* [n_vars] */
  const fg_mgm2_pset_t *psets;
  int32_t n_psets, reserved_ps;
} fg_mgm2_desc_t;

typedef struct fg_mgm2 *fg_mgm2_t;

int fg_mgm2_create(const fg_mgm2_desc_t *desc, fg_mgm2_t *out);
int fg_mgm2_destroy(fg_mgm2_t h);
const char *fg_mgm2_last_error(fg_mgm2_t h);
/* on_start: start values of the variables with neighbours (initial_value or a draw); a variable
 * without neighbours takes a drawn value among its best over its (unary) constraints and is done. */
int fg_mgm2_init(fg_mgm2_t h, void *stream);
/* up to n_cycles cycles (stops as the reference does at stop_cycle). */
int fg_mgm2_step(fg_mgm2_t h, int32_t n_cycles, void *stream);
int fg_mgm2_current(fg_mgm2_t h, int64_t *cycle, int32_t *finished);
int64_t fg_mgm2_launch_count(fg_mgm2_t h);

/* Sharded MGM-2 (multi-GPU; pydcop_b200/multigpu_mgm2.py).  The handle's problem is one rank's closed local
 * problem: its own variables with all their constraints plus a GHOST for every remote variable in their scopes
 * (dev_var_id = GLOBAL ids, so the draws equal the single-GPU run's).  The phase kernels run on the owned variables
 * only; a cycle has five exchanges, each one pack -> transport -> unpack over per-exchange buffers of T elements:
 *   0 offers  owner -> holders (offerer, partner as the receiver's id or -1, the first len - 1 offer entries)
 *   1 answers holder -> owner (accepted value or -1, the receiver's global gain), merged into the owner's flags
 *   2 gains, 3 GO flags, 4 values: owner -> holders (one element each).
 * Entry i of a list moves variable var[i] in record buf[off[i] .. off[i+1]); the lists of one transport peer are
 * consecutive, so a peer's block is one contiguous run of each buffer. */
typedef struct {
  int64_t n_send, n_recv;
  const int32_t *dev_send_var, *dev_recv_var;   /* internal local ids */
  const int64_t *dev_send_off, *dev_recv_off;   /* [n + 1] record starts, elements of the run's precision */
  void *dev_send_buf, *dev_recv_buf;            /* T[send_off[n_send]], T[recv_off[n_recv]] */
} fg_mgm2_xfer_t;

#define FG_MGM2_EXCHANGES 5
typedef struct {
  fg_mgm2_xfer_t x[FG_MGM2_EXCHANGES];
  const uint8_t *dev_ghost;        /* [n_vars] 1 = another rank's variable: never computed here */
  const int32_t *dev_send_peer;    /* [x[0].n_send] rank each offer record goes to */
  const int32_t *dev_owner_rank;   /* [n_vars] rank owning the variable */
  const int32_t *dev_owner_local;  /* [n_vars] the variable's internal id on that rank */
} fg_mgm2_shard_plan_t;

/* Transport over NVLink peer memory: for exchange x, block b copies n_elems[x][b] elements from send_buf + src[x][b]
 * to the absolute (peer-mapped) address dst[x][b]; the last block of the copy kernel releases the next epoch to every
 * peer of `sync` (csrc/peer_sync.cuh), then the rank waits for the same epoch from every peer and unpacks. */
typedef struct {
  int32_t n_blocks[FG_MGM2_EXCHANGES];
  int32_t reserved0;
  int64_t src[FG_MGM2_EXCHANGES][FG_MAX_PEERS];
  int64_t n_elems[FG_MGM2_EXCHANGES][FG_MAX_PEERS];
  uint64_t dst[FG_MGM2_EXCHANGES][FG_MAX_PEERS];
  uint32_t *dev_counter;           /* one zeroed uint32 */
  fg_peer_sync_t sync;
} fg_mgm2_peer_plan_t;

/* Attach the shard plan (copied) and, when `peer` is not NULL, the NVLink transport (copied); attaching again
 * replaces both.  The epoch counter starts at 0 and only grows: every rank runs the same number of cycles. */
int fg_mgm2_shard_attach(fg_mgm2_t h, const fg_mgm2_shard_plan_t *plan, const fg_mgm2_peer_plan_t *peer);
/* init on the owned variables, then pack exchange 4 (values); the caller transports and calls unpack(4). */
int fg_mgm2_shard_init(fg_mgm2_t h, void *stream);
/* Host-transported cycles (NCCL): phase x runs the kernel that produces exchange x (0 value, 1 answer, 2 commit,
 * 3 gain, 4 go) and packs it; phase 4 ends the cycle.  unpack(x) after the transport.  A cycle is phases 0..4 in
 * order, each followed by its transport and unpack; check fg_mgm2_current's `finished` before starting one. */
int fg_mgm2_shard_phase(fg_mgm2_t h, int32_t x, void *stream);
int fg_mgm2_shard_unpack(fg_mgm2_t h, int32_t x, void *stream);
/* Up to n_cycles whole cycles on the device with the NVLink transport (stops at stop_cycle as fg_mgm2_step):
 * per exchange kernel -> pack -> copy + release -> wait -> unpack; five epochs per cycle. */
int fg_mgm2_shard_step(fg_mgm2_t h, int32_t n_cycles, void *stream);

/* ------------------------------------------------------------------------------------------
 * GDBA  (pydcop/algorithms/gdba.py: distributed breakout with constraint modifiers, for ALL
 * variables at once).  Same constraint-hypergraph arrays as MGM.  One round = two launches:
 *   1. ok phase (:352-387): effective evaluation of every value (base cost combined with the
 *      variable's modifier, plus the variable-cost terms), violated constraints at the current
 *      value, improve and the value an improving variable would take
 *   2. improve phase (:493-541): an improving variable that wins its neighbourhood moves; a variable
 *      that cannot improve, when no neighbour's improve exceeds 0, raises its own modifiers on its
 *      violated constraints.  Values are double-buffered: round k reads dev_value[(k-1) % 2] and
 *      writes dev_value[k % 2], so a breakout reads the values the round was evaluated on.
 * Modifier counts (int32, converted to T at use; reset by fg_gdba_init): increase mode T keeps one
 * count per slot; E / R / C keep a table of the constraint's entries only for a slot whose constraint
 * spans {variable} + all its neighbours — the only constraints where the reference ever reads what those
 * modes write (:585-588 vs :634-654).
 * Draws: Philox4x32-10 keyed as MGM's: counter (canonical variable id, cycle, 0, 0), cycle 0xffffffff
 * for the start value, else the 1-based round.
 * ------------------------------------------------------------------------------------------ */
enum { FG_GDBA_MODIFIER_A = 0, FG_GDBA_MODIFIER_M = 1 };
enum { FG_GDBA_VIOLATION_NZ = 0, FG_GDBA_VIOLATION_NM = 1, FG_GDBA_VIOLATION_MX = 2 };
enum { FG_GDBA_INCREASE_E = 0, FG_GDBA_INCREASE_R = 1, FG_GDBA_INCREASE_C = 2, FG_GDBA_INCREASE_T = 3 };

/* one parameter set of a GDBA handle (increase_mode stays one per handle: it decides the modifier layout); with
 * NM / MX the factors of the variables of a set read their dev_viol_ref entry of that set's mode */
typedef struct {
  int32_t modifier;               /* FG_GDBA_MODIFIER_* */
  int32_t violation;              /* FG_GDBA_VIOLATION_* */
} fg_gdba_pset_t;

typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_factors, n_edges, n_classes;
  const fg_class_t *classes;      /* HOST [n_classes] */
  const void *dev_tables;         /* T[...] */
  const void *dev_unary;          /* T[...] variable costs (cost_for_val) */
  const int64_t *dev_unary_off;   /* [n_vars+1] */
  const void *dev_viol_ref;       /* T[n_factors] internal factor order: min (NM) / max (MX) of the base
                                     table (:252-274); may be NULL with NZ */
  const int32_t *dev_dom_size;    /* [n_vars] */
  const int32_t *dev_var_id;      /* [n_vars] canonical id = Philox counter */
  const int32_t *dev_var_rank;    /* [n_vars] position of the variable's NAME in sorted order */
  const int32_t *dev_edge_var;    /* [n_edges] */
  const int32_t *dev_edge_class;  /* [n_edges] */
  const int32_t *dev_var_ptr;     /* [n_vars+1] */
  const int32_t *dev_slot_edge;   /* [n_edges] incident edges of v in node.constraints order */
  const int32_t *dev_nbr_ptr;     /* [n_vars+1] distinct neighbours, first-appearance order */
  const int32_t *dev_nbr_idx;     /* [nbr_ptr[n_vars]] */
  const int32_t *dev_init_value;  /* [n_vars] value index or -1 (random), may be NULL */
  int32_t *dev_value[2];          /* [n_vars] each; dev_value[0] holds the preset values of the variables
                                     without neighbours (optimal_cost_value), the others are set by init */
  void *dev_cost;                 /* T[n_vars] current_cost (preset for isolated variables) */
  uint8_t *dev_has_cost;          /* [n_vars] current_cost is not None */
  void *dev_improve;              /* T[n_vars] */
  int32_t *dev_new_value;         /* [n_vars] */
  uint8_t *dev_violated;          /* [n_edges] per slot: violated at the current value (last round) */
  uint8_t *dev_breakout;          /* [n_vars] the last round raised a modifier */
  int32_t *dev_mod;               /* modifier counts: [n_edges] (T) or the spanning tables (E / R / C) */
  const int64_t *dev_mod_off;     /* [n_edges] E / R / C: start of the slot's table in dev_mod, -1 = none;
                                     NULL with T */
  int32_t mode_max;
  int32_t modifier;               /* FG_GDBA_MODIFIER_* */
  int32_t violation;              /* FG_GDBA_VIOLATION_* */
  int32_t increase_mode;          /* FG_GDBA_INCREASE_* */
  int32_t stop_cycle;             /* 0 = never; a run ends when round + 1 >= stop_cycle (as fg_mgm_desc_t) */
  int32_t reserved0;
  int64_t mod_size;               /* elements of dev_mod */
  uint64_t seed;
  const uint64_t *dev_var_seed;   /* [n_vars] optional: Philox key of internal variable v; NULL = `seed` */
  /* optional parameter sets, as fg_dsa_desc_t's */
  const uint16_t *dev_var_pset;  /* [n_vars] */
  const fg_gdba_pset_t *psets;
  int32_t n_psets, reserved_ps;
} fg_gdba_desc_t;

typedef struct fg_gdba *fg_gdba_t;

int fg_gdba_create(const fg_gdba_desc_t *desc, fg_gdba_t *out);
int fg_gdba_destroy(fg_gdba_t h);
const char *fg_gdba_last_error(fg_gdba_t h);
/* on_start: start values of the variables with neighbours (initial_value or a draw), every modifier
 * back to its base. */
int fg_gdba_init(fg_gdba_t h, void *stream);
/* up to n_cycles rounds (stops at stop_cycle). */
int fg_gdba_step(fg_gdba_t h, int32_t n_cycles, void *stream);
/* rounds run; the current values are in dev_value[cycle % 2]. */
int fg_gdba_current(fg_gdba_t h, int64_t *cycle, int32_t *finished);
int64_t fg_gdba_launch_count(fg_gdba_t h);

/* ------------------------------------------------------------------------------------------
 * DPOP  (pydcop/algorithms/dpop.py: exact UTIL / VALUE propagation over a DFS pseudo-tree).  Every
 * per-node array is in CANONICAL variable order; the tree, the separators, the term descriptors and
 * the schedule come from the host (pydcop_b200/pseudotree.py), so a run is a fixed sequence of
 * launches with nothing read back in between:
 *   UTIL  util_launches in order: kind 0 = one warp per segment [first, first + count) of
 *         dev_util_seg_ptr, walking its nodes bottom-up; kind 1 = node `first` on the whole grid
 *   VALUE value_launches in order (kind 0 only): one warp per heavy path, top down
 * Summation order, argopt and the unresolved rule: csrc/dpop_kernels.cuh.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t kind, first, count, reserved;
} fg_dpop_launch_t;

typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, mode_max;
  int64_t n_terms, n_tdims;
  int64_t arena_size;              /* T elements of dev_arena */
  const void *dev_unary;           /* T[...] the layout's variable costs (internal order) */
  const void *dev_tables;          /* T[...] the layout's class-major constraint tables */
  void *dev_arena;                 /* T[arena_size] every node's UTIL */
  const int32_t *dev_dom_size;     /* [n_vars] */
  const int64_t *dev_unary_off;    /* [n_vars] */
  const int64_t *dev_util_off;     /* [n_vars] */
  const int64_t *dev_util_size;    /* [n_vars] */
  const int32_t *dev_sep_ptr;      /* [n_vars+1] */
  const int32_t *dev_sep_var;      /* separators, root side first, at most FG_DPOP_MAX_SEP (32) each */
  const int32_t *dev_term_ptr;     /* [n_vars+1] */
  const int32_t *dev_term_kind;    /* [n_terms] 0 = child UTIL (arena), 1 = constraint (tables) */
  const int64_t *dev_term_base;    /* [n_terms] */
  const int64_t *dev_term_own;     /* [n_terms] */
  const int32_t *dev_tdim_ptr;     /* [n_terms+1] */
  const int32_t *dev_tdim_pos;     /* [n_tdims] */
  const int64_t *dev_tdim_stride;  /* [n_tdims] */
  const int32_t *dev_util_nodes;   /* UTIL segments' nodes, bottom-up */
  const int32_t *dev_util_seg_ptr; /* [n_util_segs+1] */
  const int32_t *dev_value_nodes;  /* heavy paths' nodes, top-down */
  const int32_t *dev_value_seg_ptr; /* [n_value_segs+1] */
  int32_t n_util_segs, n_value_segs;
  int32_t n_util_launches, n_value_launches;
  const fg_dpop_launch_t *util_launches;   /* HOST */
  const fg_dpop_launch_t *value_launches;  /* HOST */
  int32_t *dev_value;              /* [n_vars] chosen value index */
  void *dev_cost;                  /* T[n_vars] the chosen value's joined entry (NaN when unresolved) */
  int32_t *dev_unresolved;         /* [1] nodes where no value reached the best (the reference raises) */
  int32_t max_sep, reserved0;
} fg_dpop_desc_t;

typedef struct fg_dpop *fg_dpop_t;

int fg_dpop_create(const fg_dpop_desc_t *desc, fg_dpop_t *out);
int fg_dpop_destroy(fg_dpop_t h);
const char *fg_dpop_last_error(fg_dpop_t h);
/* both phases: every UTIL launch, then every VALUE launch; the unresolved count is reset first. */
int fg_dpop_run(fg_dpop_t h, void *stream);
int64_t fg_dpop_launch_count(fg_dpop_t h);

/* ------------------------------------------------------------------------------------------
 * DBA  (pydcop/algorithms/dba.py: Yokoo and Hirayama's distributed breakout, for ALL variables at
 * once).  Same constraint-hypergraph arrays as MGM.  DBA reads a table only through
 * `entry >= infinity` (:478), so fg_dba_init evaluates that predicate once, in the tables' precision,
 * into VIOLATION BIT ROWS: slot s (variable v at scope position j of constraint f) owns
 * table_size / dom(v) rows, indexed by the mixed-radix index of the OTHER scope variables' values in
 * scope order; a row is ceil(dom(v) / 32) words and bit x of word x / 32 is entry(v = x) >= infinity.
 * Slot s's rows start at word dev_bit_off[s].  Later writes to dev_tables are not seen.
 * One round = two launches (phases: ok of round k = 2k, improve = 2k + 1, k from 1):
 *   1. ok (:366-420): eval of every value = sum of the slot weights whose bit is set; best below
 *      `infinity`, improve, consistency, the posted counter, the violated slots at the current value
 *   2. improve (:504-562): counter minimum, the contest (larger improve, then smaller name), the stop
 *      test (counter == max_distance), the move or the weight raise.
 * End flood (:578-588): a variable finishes at phase p, and does nothing else, iff a neighbour's
 * dev_finish_phase < p; a stopping variable finishes at its improve phase.  dev_status = {live,
 * end_round}: live counts the unfinished variables with neighbours, end_round (INT32_MAX while live > 0)
 * the round in which it reached 0; rounds after end_round change no state.  Variables without
 * neighbours never evaluate, move or finish.
 * Draws: Philox4x32-10 counter (canonical variable id, cycle, 0, 0); cycle 0xffffffff for the start
 * value of EVERY variable (initial values are ignored), else the reference's cycle_count, k - 1.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_factors, n_edges, n_classes;
  const fg_class_t *classes;      /* HOST [n_classes] */
  const void *dev_tables;         /* T[...] read once, by fg_dba_init */
  const int32_t *dev_dom_size;    /* [n_vars] */
  const int32_t *dev_var_id;      /* [n_vars] canonical id = Philox counter */
  const int32_t *dev_var_rank;    /* [n_vars] position of the variable's NAME in sorted order */
  const int32_t *dev_edge_var;    /* [n_edges] */
  const int32_t *dev_edge_class;  /* [n_edges] */
  const int32_t *dev_var_ptr;     /* [n_vars+1] */
  const int32_t *dev_slot_edge;   /* [n_edges] incident edges of v in node.constraints order */
  const int32_t *dev_nbr_ptr;     /* [n_vars+1] distinct neighbours */
  const int32_t *dev_nbr_idx;     /* [nbr_ptr[n_vars]] */
  const int64_t *dev_bit_off;     /* [n_edges+1] first word of every slot's bit rows; [n_edges] = n_words */
  uint32_t *dev_bits;             /* [n_words] violation bit rows (written by fg_dba_init) */
  int32_t *dev_value[2];          /* [n_vars] each: round k reads dev_value[(k-1) % 2], writes dev_value[k % 2] */
  int64_t *dev_cost;              /* [n_vars] current_cost: eval(current) after an ok phase, eval - improve after
                                     a move (the reference assigns the field in both places, :385 and :558) */
  uint8_t *dev_has_cost;          /* [n_vars] current_cost is not None (an ok phase has run) */
  int64_t *dev_eval;              /* [n_vars] posted eval(current value) */
  int64_t *dev_improve;           /* [n_vars] posted improve */
  int32_t *dev_counter;           /* [n_vars] posted termination counter */
  int32_t *dev_counter_own;       /* [n_vars] counter after the improve phase */
  int32_t *dev_new_value;         /* [n_vars] value drawn among the best, -1 without a draw */
  uint8_t *dev_can_move, *dev_qlm, *dev_consistent;   /* [n_vars] each */
  int32_t *dev_finish_phase;      /* [n_vars] INT32_MAX while live */
  int32_t *dev_weight;            /* [n_edges] per slot, from 1 */
  uint8_t *dev_violated;          /* [n_edges] per slot: violated at the current value (last ok phase) */
  int32_t *dev_status;            /* [2] live, end_round */
  int32_t *dev_unresolved;        /* [1] improve > 0 with no value below infinity (the reference raises) */
  int64_t n_words;                /* uint32 words of dev_bits */
  int64_t infinity;
  int32_t max_distance;           /* >= 0; 0 never stops */
  int32_t stop_cycle;             /* 0 = never; a run ends when round + 1 >= stop_cycle (as fg_gdba_desc_t) */
  int32_t n_live;                 /* variables with neighbours */
  int32_t reserved0;
  uint64_t seed;
} fg_dba_desc_t;

typedef struct fg_dba *fg_dba_t;

int fg_dba_create(const fg_dba_desc_t *desc, fg_dba_t *out);
int fg_dba_destroy(fg_dba_t h);
const char *fg_dba_last_error(fg_dba_t h);
/* bit rows from dev_tables, start values of every variable, weights 1, counters 0, status reset. */
int fg_dba_init(fg_dba_t h, void *stream);
/* up to n_cycles rounds; none once `finished` has been observed by fg_dba_current. */
int fg_dba_step(fg_dba_t h, int32_t n_cycles, void *stream);
/* waits for the work already enqueued; cycle = min(rounds enqueued, end_round), finished = every variable
 * with neighbours finished, or stop_cycle reached.  The current values are in dev_value[cycle % 2]. */
int fg_dba_current(fg_dba_t h, int64_t *cycle, int32_t *finished);
int64_t fg_dba_launch_count(fg_dba_t h);

/* ------------------------------------------------------------------------------------------
 * SyncBB  (pydcop/algorithms/syncbb.py: synchronous branch and bound over the variables sorted by
 * name, ordered_graph.py:173).  The search is a token walk: one message is in flight at any time.
 * ONE CTA runs the whole search, message after message, and leaves every piece of state in the
 * caller's arrays, so a run may be split into launches anywhere with the same result.
 * Everything is indexed by CHAIN POSITION p (the variable's rank in name order).  The path is always
 * a prefix of the chain: path element q is (chain variable q, dev_path_val[q], dev_path_cost[q]).
 * Per step, threads cover the candidates of the receiver; each sums its candidate's path elements
 * sequentially in path order (get_next_assignment, :415-473):
 *   ass(q) = dev_pair[dev_elt_tab[k] + val_q * dom(p) + x] for the earlier neighbour at q (slot k),
 *            0 for any other element
 *   min mode: element q fails when cc + ass >= ub(p) or ass + path_cost(q) >= ub(p); a candidate
 *            is rejected iff its FIRST element fails, else accepted with cc up to the last passing
 *            element.  Max mode accepts every candidate with its full sum.
 * A block reduction picks the first accepted candidate, or at the last variable the first strict
 * best of psum + cost (psum = the path's costs summed as CPython's sum() does, Neumaier-compensated,
 * kept per prefix in dev_path_sum / dev_path_comp).  Unary constraints and variable costs are not
 * part of the plan (SyncBB never reads them); constraints of arity > 2 are refused by the host.
 * dev_msg = {type (0 forward, 1 backward, 2 terminate), receiver, path length, finished}.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars;                 /* chain length, >= 2 */
  int32_t mode_max;
  const int32_t *dev_dom;         /* [n_vars] domain size per chain position, 1..FG_MAX_DOM; the kernel covers
                                     FG_MAX_DOM candidates per step and cannot check these device values, so a
                                     larger domain is undefined behaviour (SyncbbEngine's layout refuses it) */
  const int32_t *dev_elt_ptr;     /* [n_vars+1] earlier neighbours of chain position p */
  const int32_t *dev_elt_pos;     /* [n_elts] their chain positions, ascending within p */
  const int64_t *dev_elt_tab;     /* [n_elts] first entry of the pair table [val_u][x] in dev_pair */
  const void *dev_pair;           /* T[n_pair] every binary constraint between p and u summed from 0 in
                                     node.constraints order */
  void *dev_ub;                   /* T[n_vars] per-variable upper_bound */
  int32_t *dev_sel;               /* [n_vars] last value_selection, -1 before any */
  int32_t *dev_path_val;          /* [n_vars] */
  void *dev_path_cost;            /* T[n_vars] */
  void *dev_path_sum;             /* T[n_vars] compensated prefix sum of path_cost[0..q] */
  void *dev_path_comp;            /* T[n_vars] its compensation */
  int32_t *dev_msg;               /* [4] */
  void *dev_msg_ub;               /* T[1] bound carried by the message in flight */
  int64_t *dev_count;             /* [2] steps (messages delivered), messages posted */
  int64_t *dev_cycles;            /* [n_vars] the reference's new_cycle count per variable: messages received,
                                     plus one for the first variable's start (syncbb.py:211) */
  int64_t n_elts, n_pair;
} fg_syncbb_desc_t;

typedef struct fg_syncbb *fg_syncbb_t;

int fg_syncbb_create(const fg_syncbb_desc_t *desc, fg_syncbb_t *out);
int fg_syncbb_destroy(fg_syncbb_t h);
const char *fg_syncbb_last_error(fg_syncbb_t h);
/* bounds +-inf, no selection, the first variable's start message [(x0, 0, 0)] to chain position 1. */
int fg_syncbb_init(fg_syncbb_t h, void *stream);
/* one launch delivering up to n_steps messages; none once the last terminate message is delivered. */
int fg_syncbb_step(fg_syncbb_t h, int64_t n_steps, void *stream);
/* waits for the work already enqueued. */
int fg_syncbb_current(fg_syncbb_t h, int64_t *steps, int64_t *messages, int32_t *finished);
int64_t fg_syncbb_launch_count(fg_syncbb_t h);

/* ------------------------------------------------------------------------------------------
 * MixedDSA  (pydcop/algorithms/mixeddsa.py, MixedDsaComputation: DSA for problems that mix hard
 * constraints, a table with a +inf or -inf entry, with soft ones; for ALL variables at once).  Same
 * constraint-hypergraph arrays as MGM, except that dev_slot_edge lists each variable's SOFT slots first and
 * its HARD slots after dev_soft_end[v], each group in node.constraints order (the host classifies the
 * constraints in the tables' precision).  One round = one launch, one thread per variable:
 *   C(x) = (((0 + soft slots) + own cost at x) + neighbours' costs) + hard entries that are not +inf
 *   H(x) = hard entries equal to +inf
 * then the lexicographic best (H, then C strictly, ties in domain order) and the five-way decision of
 * mixeddsa.py:300-358 (csrc/mixeddsa_kernels.cuh).  Values are double-buffered: round k reads
 * dev_value[(k-1) % 2] and writes dev_value[k % 2].  A variable without neighbours evaluates in round 1
 * only.  dev_con_opt is written by fg_mixeddsa_init (the whole-table optimum of every constraint).
 * Draws: Philox4x32-10 counter (canonical variable id, cycle, 0, 0): cycle 0xffffffff for the start value
 * of EVERY variable without an initial value, else the 1-based round; u (philox_u53) for the probability
 * test and the choice among the best values from the same block.
 * ------------------------------------------------------------------------------------------ */
enum { FG_MIXEDDSA_BRANCH_NONE = 0, FG_MIXEDDSA_BRANCH_HARD = 1, FG_MIXEDDSA_BRANCH_SOFT = 2,
       FG_MIXEDDSA_BRANCH_STUCK_HARD = 3, FG_MIXEDDSA_BRANCH_STUCK_SOFT = 4, FG_MIXEDDSA_BRANCH_IDLE = 5,
       FG_MIXEDDSA_MOVED = 8 };

/* one parameter set of a MixedDSA handle */
typedef struct {
  double proba_hard, proba_soft;  /* finite, in [0, 1] */
  int32_t variant;                /* FG_DSA_* */
  int32_t reserved0;
} fg_mixeddsa_pset_t;

typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_factors, n_edges, n_classes;
  const fg_class_t *classes;      /* HOST [n_classes] */
  const void *dev_tables;         /* T[...] */
  const void *dev_unary;          /* T[...] variable costs (cost_for_val) */
  const int64_t *dev_unary_off;   /* [n_vars+1] */
  const int32_t *dev_dom_size;    /* [n_vars] */
  const int32_t *dev_var_id;      /* [n_vars] canonical id = Philox counter */
  const int32_t *dev_edge_var;    /* [n_edges] */
  const int32_t *dev_edge_class;  /* [n_edges] */
  const int32_t *dev_var_ptr;     /* [n_vars+1] */
  const int32_t *dev_slot_edge;   /* [n_edges] v's soft slots, then its hard slots */
  const int32_t *dev_soft_end;    /* [n_vars] end of v's soft slots: var_ptr[v] <= soft_end[v] <= var_ptr[v+1] */
  const int32_t *dev_nbr_ptr;     /* [n_vars+1] distinct neighbours, first-appearance order */
  const int32_t *dev_nbr_idx;     /* [nbr_ptr[n_vars]] */
  const int32_t *dev_init_value;  /* [n_vars] value index or -1 (random), may be NULL */
  void *dev_con_opt;              /* T[n_factors] internal factor order (written by init) */
  int32_t *dev_value[2];          /* [n_vars] each */
  void *dev_cost;                 /* T[n_vars] current_cost: the eff_cost of the last move */
  uint8_t *dev_has_cost;          /* [n_vars] current_cost is not None (the variable has moved) */
  int32_t *dev_h_best;            /* [n_vars] H of the best values in the last round, -1 without an evaluation */
  uint8_t *dev_branch;            /* [n_vars] FG_MIXEDDSA_BRANCH_* of the last round, | FG_MIXEDDSA_MOVED */
  double proba_hard, proba_soft;
  int32_t mode_max;
  int32_t variant;                /* FG_DSA_A | FG_DSA_B | FG_DSA_C (C acts as B, mixeddsa.py:342) */
  int32_t stop_cycle;             /* 0 = never; a run ends after stop_cycle rounds (as fg_dsa_desc_t) */
  int32_t reserved0;
  uint64_t seed;
  const uint64_t *dev_var_seed;   /* [n_vars] optional: Philox key of internal variable v; NULL = `seed` */
  /* optional parameter sets, as fg_dsa_desc_t's */
  const uint16_t *dev_var_pset;  /* [n_vars] */
  const fg_mixeddsa_pset_t *psets;
  int32_t n_psets, reserved_ps;
} fg_mixeddsa_desc_t;

typedef struct fg_mixeddsa *fg_mixeddsa_t;

int fg_mixeddsa_create(const fg_mixeddsa_desc_t *desc, fg_mixeddsa_t *out);
int fg_mixeddsa_destroy(fg_mixeddsa_t h);
const char *fg_mixeddsa_last_error(fg_mixeddsa_t h);
/* constraint optima, start value of every variable (initial_value or a draw), no cost yet. */
int fg_mixeddsa_init(fg_mixeddsa_t h, void *stream);
/* up to n_cycles rounds (none once stop_cycle rounds have run). */
int fg_mixeddsa_step(fg_mixeddsa_t h, int32_t n_cycles, void *stream);
/* rounds run; the current values are in dev_value[cycle % 2]. */
int fg_mixeddsa_current(fg_mixeddsa_t h, int64_t *cycle, int32_t *finished);
int64_t fg_mixeddsa_launch_count(fg_mixeddsa_t h);

/* Solution cost (next-tier row §8f.1; pydcop/dcop/dcop.py:319-367 `solution_cost`, called by the
 * orchestrator at the end of a run and at every metric tick, orchestrator.py:1229-1231): over the factors
 * of every non-ghost class the table entry at the assignment, over the first n_vars variables
 * dev_unary[unary_off[v] + value[v]]; an entry EQUAL to `infinity` (compared in the tables' precision) is
 * counted as a violation, every other entry is summed: dev_out[0] = cost (double), dev_out[1] =
 * violations.  dev_unary holds the variables' OWN costs in internal variable order (without MaxSum's
 * noise, which is not part of the problem's cost); NULL skips the variable costs.  A shard counts only
 * what it owns — n_vars leading variables, and the optional byte masks dev_factor_skip[internal factor]
 * / dev_var_skip[internal variable] (non-zero = not mine; NULL = none) — and the caller all-reduces
 * dev_out over the ranks. */
int fg_solution_cost(int32_t precision, int32_t n_classes, const fg_class_t *classes,
                     const void *dev_tables, const int32_t *dev_edge_var,
                     const int32_t *dev_value, const void *dev_unary,
                     const int64_t *dev_unary_off, int32_t n_vars, const uint8_t *dev_factor_skip,
                     const uint8_t *dev_var_skip, double infinity, double *dev_out, void *stream);

/* Solution cost per problem of a batch (pydcop_b200.solve.solve_batch: several problems packed into one layout as a
 * disjoint union): fg_solution_cost's sums, split by dev_factor_seg[internal factor] and dev_var_seg[internal
 * variable], the problem each belongs to, in 0..n_seg-1 (an id outside that range is not counted).  dev_out[2 * s] =
 * cost, dev_out[2 * s + 1] = violations of problem s, n_seg pairs of doubles.  Any segment order is correct; each warp
 * adds one atomic pair per run of consecutive factors (variables) of the same problem.  Both segment arrays are
 * required, on the current device. */
int fg_solution_cost_segmented(int32_t precision, int32_t n_classes, const fg_class_t *classes,
                               const void *dev_tables, const int32_t *dev_edge_var,
                               const int32_t *dev_value, const void *dev_unary,
                               const int64_t *dev_unary_off, int32_t n_vars, const uint8_t *dev_factor_skip,
                               const uint8_t *dev_var_skip, const int32_t *dev_factor_seg,
                               const int32_t *dev_var_seg, int32_t n_seg, double infinity, double *dev_out,
                               void *stream);

/* ------------------------------------------------------------------------------------------
 * Cost trace (pydcop solve --collect_on cycle_change, orchestrator.py:802-884): with a trace attached to an
 * iterative family's handle, its fg_<family>_step enqueues, after every committed cycle and on the step's stream,
 * one record of fg_solution_cost(_segmented)'s sums over the family's current values: record k (k = 0, 1, ...)
 * adds into row k, dev_rows[(k * n_seg + s) * 2] = cost and [... + 1] = violations of segment s, and stamps
 * dev_stamp[k + 1] with the device's global timer (ns) when the whole row is summed.  A record is ONE launch over a
 * block map built at create (the factor ranges of every non-ghost class, then the variables); it never
 * synchronises.  Once `capacity` rows are recorded no more are: the caller attaches a fresh trace to go on.
 * Records count in neither the family's launch count nor its cycles.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t abi_version, precision;
  int32_t n_vars, n_classes;
  const fg_class_t *classes;      /* HOST [n_classes], copied by fg_trace_create */
  const void *dev_tables;         /* T[...] the family's tables */
  const int32_t *dev_edge_var;    /* [n_edges] */
  const void *dev_unary;          /* T[...] the variables' OWN costs, internal order (MaxSum: without noise); NULL:
                                     variable costs are not added */
  const int64_t *dev_unary_off;   /* [n_vars+1] */
  const int32_t *dev_factor_seg;  /* [n_factors] optional, as fg_solution_cost_segmented; NULL (both): one segment */
  const int32_t *dev_var_seg;     /* [n_vars] */
  int32_t n_seg, reserved0;
  double infinity;                /* an entry equal to it counts as a violation */
  double *dev_rows;               /* [capacity * n_seg * 2] */
  int64_t *dev_stamp;             /* [capacity + 1] stamp 0 written by fg_trace_start */
  int64_t capacity;               /* rows */
} fg_trace_desc_t;

typedef struct fg_trace *fg_trace_t;

int fg_trace_create(const fg_trace_desc_t *desc, fg_trace_t *out);
/* a trace still attached to a handle must be detached first */
int fg_trace_destroy(fg_trace_t tr);
const char *fg_trace_last_error(fg_trace_t tr);
/* zeroes every row, writes stamp 0 and the row count back to 0, on `stream` */
int fg_trace_start(fg_trace_t tr, void *stream);
/* rows enqueued since fg_trace_start (a host count: no synchronisation) */
int fg_trace_rows(fg_trace_t tr, int64_t *n_rows);
/* Keep, per segment, the best row the trace records and the values of that cycle (the anytime result of a run):
 * the first record sets it, a later row replaces it only when strictly better (fewer violations; at equal
 * violations a cost < the best's in min mode, > in max mode; a NaN cost never beats a non-NaN one), so ties keep
 * the earlier cycle.  dev_best: [n_seg * 2] doubles (cost, violations), the row's own; dev_best_cycle: [n_seg]
 * int64, 0 = none yet, else the record number (1-based, counted since this call, NOT reset by fg_trace_start);
 * dev_best_value: [n_vars] int32, internal order, the values the record summed.  Resets them on `stream`.  All three
 * NULL: detach.  A record then adds at most one launch (the values of the segments it improved), counted by the
 * trace; a full trace records, and so keeps, nothing. */
int fg_trace_set_best(fg_trace_t tr, int32_t mode_max, double *dev_best, int64_t *dev_best_cycle,
                      int32_t *dev_best_value, void *stream);
/* Attach `tr` (NULL: detach) to a handle of the same device, precision and variable count.  Records the values of
 * MaxSum's dev_value, DSA's dev_value[cur], MGM's and MGM-2's dev_value, and GDBA's, DBA's and MixedDSA's
 * dev_value[cycle % 2]; the sharded step loops record nothing. */
int fg_maxsum_set_trace(fg_maxsum_t h, fg_trace_t tr);
int fg_dsa_set_trace(fg_dsa_t h, fg_trace_t tr);
int fg_mgm_set_trace(fg_mgm_t h, fg_trace_t tr);
int fg_mgm2_set_trace(fg_mgm2_t h, fg_trace_t tr);
int fg_gdba_set_trace(fg_gdba_t h, fg_trace_t tr);
int fg_dba_set_trace(fg_dba_t h, fg_trace_t tr);
int fg_mixeddsa_set_trace(fg_mixeddsa_t h, fg_trace_t tr);

/* Row permutation on the device (engine creation): dev_dst[i * row_elems + k] = dev_src[dev_rows[i] * row_elems + k]
 * for i < n_rows, k < row_elems, elements of the given precision.  MaxSumEngine packs a one-class layout's tables with it
 * when the factor order permutes them (layout.FactorGraphLayout.table_rows): the caller's array is uploaded as it is and
 * the host makes no copy. */
int fg_gather_rows(int32_t precision, void *dev_dst, const void *dev_src, const int64_t *dev_rows, int64_t n_rows,
                   int64_t row_elems, void *stream);

/* Diagnostic: evaluates the send-gate predicate approx_match (maxsum.py:688-710) on n pairs with
 * the division-free fast form used by the tiled kernels (out_fast) and the literal form
 * (out_exact); the two must agree on every input.  T arrays of n elements, uint8 outputs. */
int fg_selftest_approx_match(int32_t precision, int64_t n, const void *dev_c, const void *dev_prev,
                             double stability, uint8_t *dev_out_fast, uint8_t *dev_out_exact,
                             void *stream);

/* Diagnostic: HBM throughput of the DSA / MGM table access pattern alone — `n_threads` threads each read
 * `rows_per_thread` (1, 2, 3 or 6) rows of `row_bytes` (multiple of 16) at pseudo-random multiples of `stride_bytes`
 * inside [dev_base, dev_base + region_bytes), all loads independent; dev_out[n_threads] receives a checksum.
 * Timed by the caller (tools/gather_peak.py): the ceiling those kernels are measured against in DESIGN.md. */
int fg_selftest_gather(const void *dev_base, int64_t region_bytes, int32_t row_bytes, int32_t stride_bytes,
                       int64_t n_threads, int32_t rows_per_thread, float *dev_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PYDCOP_B200_H */
