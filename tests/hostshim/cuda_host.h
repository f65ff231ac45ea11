// TEST INFRASTRUCTURE: what a host shim needs to compile CUDA kernel SOURCE with g++ and run it on the CPU, one
// "thread" after the other.  Nothing in the product links or calls this.
//   g++ -O1 -std=c++17 -ffp-contract=off -I<cuda>/include -shared -fPIC -o <family>_host.so <family>_host.cpp
// <cuda_runtime.h> compiled by a host compiler defines __global__, __device__ and __host__ away and provides the
// vector types; the thread indices are per-launch globals here.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#define __launch_bounds__(...)

struct Dim3 { unsigned x, y, z; };
static thread_local Dim3 blockIdx, blockDim, threadIdx, gridDim;

static inline float __int_as_float(unsigned x) { float f; memcpy(&f, &x, 4); return f; }
static inline double __longlong_as_double(unsigned long long x) { double f; memcpy(&f, &x, 8); return f; }

// The launcher of the kernel headers' shared sequences (csrc/handle.cuh has the device one): L(n, block, kernel,
// args...) runs ceil(n / block) blocks of `block` threads in order, each kernel boundary a full pass over the threads.
struct fg_host_launcher {
  int64_t launches = 0;

  template <class K, class... A>
  void operator()(int64_t n, int block, K kernel, const A &...args) {
    const int64_t blocks = (n + block - 1) / block;
    gridDim = Dim3{(unsigned)blocks, 1, 1};
    blockDim = Dim3{(unsigned)block, 1, 1};
    for (int64_t b = 0; b < blocks; ++b)
      for (unsigned t = 0; t < (unsigned)block; ++t) {
        blockIdx = Dim3{(unsigned)b, 0, 0};
        threadIdx = Dim3{t, 0, 0};
        kernel(args...);
      }
    ++launches;
  }
  void fill(void *p, int byte, size_t bytes) { memset(p, byte, bytes); }
  void copy(void *dst, const void *src, size_t bytes) { memcpy(dst, src, bytes); }
};
