// Host-side scaffolding shared by the fg_<family>_* handles (engine.cu, mgm.cu, mgm2.cu, gdba.cu, dpop.cu): opening a
// handle over a copy of its descriptor, the class-table checks and upload, the device a handle belongs to, closing,
// the step loop of the families that stop at cycle + 1 >= stop_cycle, and the launcher the kernel headers' shared
// launch sequences run on.  No device code.
#pragma once

#include <cstdio>
#include <initializer_list>
#include <new>
#include <vector>

#include "common.cuh"

struct fg_trace;

struct fg_handle_base {
  std::vector<fg_class_t> classes;      // the descriptor's class table, copied (d.classes points here)
  fg_class_t *dev_classes = nullptr;    // its device copy (fg_upload_classes)
  int device = -1;                      // the device current at create (fg_require_device); -1 before
  int64_t cycle = 0;
  int64_t launches = 0;
  fg_trace *trace = nullptr;            // fg_<family>_set_trace: a record after every cycle of the step loop
  void *dev_psets = nullptr;            // device copy of the descriptor's parameter sets (fg_upload_psets)
  mutable char err[512] = {0};        // written by const readers too (fg_device_scope)
};

// engine.cu: the checks of fg_<family>_set_trace (FG_ERR_ARG, the reason in err) and one record of `value` on the
// stream, counted by the trace alone
int fg_trace_check(const fg_trace *tr, int device, int32_t precision, int32_t n_vars, char *err, size_t n);
int fg_trace_record(fg_trace *tr, const int32_t *value, cudaStream_t st);

// Runs the rest of an entry point on the handle's device and gives the caller's device back on exit, so a handle
// works whichever device the calling thread has current.  No-op for a null handle or one without a device yet.
// A failed switch leaves ok false and its reason in the handle's err.
struct fg_device_scope {
  int prev = -1;
  bool ok = true;
  explicit fg_device_scope(const fg_handle_base *h) {
    if (!h || h->device < 0) return;
    int cur = 0;
    cudaError_t e = cudaGetDevice(&cur);
    if (e == cudaSuccess && cur == h->device) return;
    if (e == cudaSuccess) e = cudaSetDevice(h->device);
    if (e != cudaSuccess) {
      cudaGetLastError();
      snprintf(h->err, sizeof(h->err), "cannot make the handle's device %d current: %s", h->device,
               cudaGetErrorString(e));
      ok = false;
      return;
    }
    prev = cur;
  }
  ~fg_device_scope() {
    if (prev >= 0) cudaSetDevice(prev);
  }
  fg_device_scope(const fg_device_scope &) = delete;
  fg_device_scope &operator=(const fg_device_scope &) = delete;
};

#define FG_ON_DEVICE(h)                      \
  fg_device_scope fg_device_scope_(h);       \
  if (!fg_device_scope_.ok) return FG_ERR_CUDA

// Where `p` lives, for messages: "device memory of device N", "pinned host memory", ...; *dev = the device of
// device memory, else -1
static inline const char *fg_memory_kind(const void *p, int *dev) {
  cudaPointerAttributes a;
  *dev = -1;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return "pageable host memory"; }
  switch (a.type) {
    case cudaMemoryTypeDevice: *dev = a.device; return "device memory";
    case cudaMemoryTypeHost: return "pinned host memory";
    case cudaMemoryTypeManaged: return "managed memory";
    default: return "pageable host memory";
  }
}

// true when `p` is device memory of the current device (the handle-less entry points' check of their main array)
static inline bool fg_on_current_device(const void *p) {
  int cur = 0, dev = -1;
  if (cudaGetDevice(&cur) != cudaSuccess) { cudaGetLastError(); return false; }
  fg_memory_kind(p, &dev);
  return dev == cur;
}

struct fg_field {
  const char *name;
  const void *ptr;
};
#define FG_FIELD(d, x) fg_field{#x, (const void *)(d).x}

// Every non-null array of a descriptor must be device memory of the handle's device: FG_ERR_ARG naming the first one
// that is not, and where it lives.  After fg_require_device.
static inline int fg_check_resident(fg_handle_base *h, std::initializer_list<fg_field> fields) {
  for (const fg_field &f : fields) {
    if (!f.ptr) continue;
    int dev = -1;
    const char *kind = fg_memory_kind(f.ptr, &dev);
    if (dev == h->device) continue;
    if (dev >= 0)
      snprintf(h->err, sizeof(h->err), "%s is device memory of device %d, the handle belongs to device %d", f.name, dev,
               h->device);
    else
      snprintf(h->err, sizeof(h->err), "%s is %s, not device memory of the handle's device %d", f.name, kind, h->device);
    return FG_ERR_ARG;
  }
  return FG_OK;
}

static inline int check_class(const fg_class_t &c, char *err, size_t n) {
  if (c.arity < 1 || c.arity > FG_MAX_ARITY) { snprintf(err, n, "class arity %d out of range", c.arity); return FG_ERR_ARG; }
  int64_t ts = 1; int rt = 0;
  for (int i = 0; i < c.arity; ++i) {
    if (c.dom[i] < 1 || c.dom[i] > FG_MAX_DOM) { snprintf(err, n, "domain size %d out of range", c.dom[i]); return FG_ERR_ARG; }
    if (c.row_off[i] < rt) { snprintf(err, n, "row_off overlaps the previous row"); return FG_ERR_ARG; }
    ts *= c.dom[i]; rt = c.row_off[i] + c.dom[i];
  }
  if (ts != c.table_size || rt > c.row_total) { snprintf(err, n, "class size mismatch"); return FG_ERR_ARG; }
  return FG_OK;
}

// Null and ABI checks, then a new handle holding a copy of the descriptor, also stored in *out.  nullptr (with *out
// cleared where there is one) when any of that fails.
template <class H, class D>
static inline H *fg_alloc(const D *desc, H **out) {
  if (!desc || !out) return nullptr;
  *out = nullptr;
  if (desc->abi_version != FG_ABI_VERSION) return nullptr;
  H *h = new (std::nothrow) H();
  if (!h) return nullptr;
  h->d = *desc;
  return *out = h;
}

// fg_alloc for the families with a class table: a precision other than FG_F32 / FG_F64 gets no handle; the classes
// are copied into the handle and checked one by one, a bad one leaving its message in the handle's err.
template <class H, class D>
static inline int fg_open(const D *desc, H **out) {
  if (!desc || !out) return FG_ERR_ARG;
  *out = nullptr;
  if (desc->precision != FG_F32 && desc->precision != FG_F64) return FG_ERR_ARG;
  H *h = fg_alloc(desc, out);
  if (!h) return FG_ERR_ARG;
  h->classes.assign(desc->classes, desc->classes + desc->n_classes);
  h->d.classes = h->classes.data();
  for (const fg_class_t &c : h->classes) {
    int rc = check_class(c, h->err, sizeof(h->err));
    if (rc != FG_OK) return rc;
  }
  return FG_OK;
}

static inline int fg_require_device(fg_handle_base *h) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    snprintf(h->err, sizeof(h->err), "no CUDA device visible: pydcop_b200 has no CPU fallback");
    return FG_ERR_CUDA;
  }
  CUDA_TRY(h, cudaGetDevice(&h->device));   // the handle belongs to this device from now on
  return FG_OK;
}

// the class table is a device allocation the library owns (a few hundred bytes), as the parameter sets are
static inline int fg_upload_classes(fg_handle_base *h) {
  size_t bytes = sizeof(fg_class_t) * (h->classes.empty() ? 1 : h->classes.size());
  CUDA_TRY(h, cudaMalloc(&h->dev_classes, bytes));
  if (!h->classes.empty())
    CUDA_TRY(h, cudaMemcpy(h->dev_classes, h->classes.data(), sizeof(fg_class_t) * h->classes.size(), cudaMemcpyHostToDevice));
  return FG_OK;
}

// The descriptor's parameter sets (dev_var_pset, psets[n_psets]): both or neither, at most FG_MAX_PSETS, and every
// set accepted by valid(set) -> NULL or the reason it is refused.  Host memory only: runs before fg_require_device.
template <class H, class V>
static inline int fg_check_psets(H *h, V valid) {
  const auto &d = h->d;
  if (!d.dev_var_pset && !d.psets && !d.n_psets) return FG_OK;
  if (!d.dev_var_pset || !d.psets || d.n_psets < 1 || d.n_psets > FG_MAX_PSETS) {
    snprintf(h->err, sizeof(h->err), "dev_var_pset and psets go together, with 1 <= n_psets <= %d (n_psets %d)",
             FG_MAX_PSETS, d.n_psets);
    return FG_ERR_ARG;
  }
  for (int i = 0; i < d.n_psets; ++i) {
    if (const char *why = valid(d.psets[i])) {
      snprintf(h->err, sizeof(h->err), "parameter set %d: %s", i, why);
      return FG_ERR_ARG;
    }
  }
  return FG_OK;
}

// the checked parameter sets into device memory the handle owns; the handle's descriptor points at that copy
template <class H>
static inline int fg_upload_psets(H *h) {
  if (!h->d.psets) return FG_OK;
  const size_t bytes = sizeof(*h->d.psets) * (size_t)h->d.n_psets;
  CUDA_TRY(h, cudaMalloc(&h->dev_psets, bytes));
  CUDA_TRY(h, cudaMemcpy(h->dev_psets, h->d.psets, bytes, cudaMemcpyHostToDevice));
  h->d.psets = (decltype(h->d.psets))h->dev_psets;
  return FG_OK;
}

static inline bool fg_unit_interval(double p) { return p >= 0.0 && p <= 1.0; }   // false for NaN too

template <class H>
static inline int fg_close(H *h) {
  {
    fg_device_scope on(h);
    if (h && h->dev_classes) cudaFree(h->dev_classes);
    if (h && h->dev_psets) cudaFree(h->dev_psets);
  }
  delete h;
  return FG_OK;
}

// The launcher the shared host sequences of the kernel headers run on (mgm_kernels.cuh & co.; tests/hostshim/
// cuda_host.h is the other one, on the CPU): L(n, block, kernel, args...) launches ceil(n / block) blocks of `block`
// threads on the stream and counts the launch; fill / copy are cudaMemsetAsync / cudaMemcpyAsync.  After the first
// failed fill or copy every call does nothing, and status() reports it as CUDA_TRY would.
struct fg_launcher {
  fg_handle_base *h;
  cudaStream_t st;
  cudaError_t e = cudaSuccess;
  const char *what = nullptr;

  fg_launcher(fg_handle_base *h, cudaStream_t st) : h(h), st(st) {}
  template <class... P, class... A>
  void operator()(int64_t n, int block, void (*kernel)(P...), const A &...args) {
    if (e != cudaSuccess) return;
    kernel<<<(unsigned)((n + block - 1) / block), block, 0, st>>>(args...);
    ++h->launches;
  }
  void fill(void *p, int byte, size_t bytes) {
    if (e == cudaSuccess && (e = cudaMemsetAsync(p, byte, bytes, st)) != cudaSuccess) what = "cudaMemsetAsync";
  }
  void copy(void *dst, const void *src, size_t bytes) {
    if (e == cudaSuccess && (e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
      what = "cudaMemcpyAsync";
  }
  int status() const {
    if (e == cudaSuccess) return FG_OK;
    snprintf(h->err, sizeof(h->err), "%s: %s", what, cudaGetErrorString(e));
    return FG_ERR_CUDA;
  }
};

static inline const char *fg_last_error(const fg_handle_base *h) { return h ? h->err : "invalid handle"; }

static inline int64_t fg_launch_count(const fg_handle_base *h) { return h ? h->launches : -1; }

template <class H>
static inline int fg_set_trace(H *h, fg_trace *tr) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (tr && fg_trace_check(tr, h->device, h->d.precision, h->d.n_vars, h->err, sizeof(h->err)) != FG_OK)
    return FG_ERR_ARG;
  h->trace = tr;
  return FG_OK;
}

// the record of a committed cycle whose values are `value`, when a trace is attached
static inline int fg_trace_cycle(fg_handle_base *h, const int32_t *value, cudaStream_t st) {
  if (!h->trace) return FG_OK;
  int rc = fg_trace_record(h->trace, value, st);
  if (rc != FG_OK) snprintf(h->err, sizeof(h->err), "trace record: %s", fg_trace_last_error(h->trace));
  return rc;
}

// MGM, MGM-2 and GDBA: rounds stop once cycle + 1 >= stop_cycle (0 = never)
template <class H>
static inline bool fg_finished(const H *h) { return h->d.stop_cycle && h->cycle + 1 >= h->d.stop_cycle; }

template <class H>
static inline int fg_current(const H *h, int64_t *cycle, int32_t *finished) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  if (cycle) *cycle = h->cycle;
  if (finished) *finished = fg_finished(h) ? 1 : 0;
  return FG_OK;
}

// up to n_cycles rounds of `cycle` in the handle's precision, stopping early at fg_finished
template <class H>
static inline int fg_step(H *h, int32_t n_cycles, void *stream, int (*cycle_f32)(H *, cudaStream_t),
                          int (*cycle_f64)(H *, cudaStream_t)) {
  if (!h) return FG_ERR_ARG;
  FG_ON_DEVICE(h);
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n_cycles; ++i) {
    if (fg_finished(h)) break;
    int rc = h->d.precision == FG_F64 ? cycle_f64(h, st) : cycle_f32(h, st);
    if (rc != FG_OK) return rc;
  }
  return FG_OK;
}
