// Shared host/device helpers for libnnconv_b200 (error reporting, integer utilities, launch checks).
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#include "../../include/nnconv_b200.h"   // status codes (NNCONV_OK, NNCONV_ERR_*)

namespace nnc {

void set_error(const char* fmt, ...);

#define NNC_CHECK_CUDA(expr)                                                                  \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::nnc::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return NNCONV_ERR_CUDA;                                                          \
    }                                                                                         \
  } while (0)

#define NNC_CHECK_LAUNCH() NNC_CHECK_CUDA(cudaGetLastError())

#define NNC_REQUIRE(cond, code, ...)     \
  do {                                   \
    if (!(cond)) {                       \
      ::nnc::set_error(__VA_ARGS__);     \
      return (code);                     \
    }                                    \
  } while (0)

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int64_t round_up64(int64_t a, int64_t b) { return ceil_div64(a, b) * b; }
__host__ __device__ inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// Bump allocator over a caller-provided device workspace (the library never calls cudaMalloc).
struct Carver {
  char* base;
  size_t cap;
  size_t off;
  Carver(void* p, size_t bytes) : base(static_cast<char*>(p)), cap(bytes), off(0) {}
  template <typename T>
  T* take(size_t count) {
    size_t bytes = round_up64(static_cast<int64_t>(count * sizeof(T)), 1024);
    size_t o = off;
    off += bytes;
    return reinterpret_cast<T*>(base ? base + o : nullptr);
  }
  bool ok() const { return off <= cap; }
};

constexpr int kTileEdges = 128;   // edges per contraction tile (two m64 wgmma halves)

// Optional per-kernel-class timing with CUDA events (bench.py roofline numbers); off by default.
enum ProfKind : int { PK_LAYER1 = 0, PK_HIDDEN_GEMM = 1, PK_NODE_PREP = 2, PK_Y_GEMM = 3, PK_CONV = 4, PK_APPLY_FUSED = 5, PK_COUNT = 6 };
bool prof_enabled();
void prof_mark(int kind, cudaStream_t st, bool begin);
struct ProfScope {
  int kind;
  cudaStream_t st;
  bool on;
  ProfScope(int k, cudaStream_t s) : kind(k), st(s), on(prof_enabled()) { if (on) prof_mark(kind, st, true); }
  ~ProfScope() { if (on) prof_mark(kind, st, false); }
};

}  // namespace nnc
