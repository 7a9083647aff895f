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

// aggr = max (DESIGN 5): every (node, channel) reduces a uint64 key.  High word: the message's bits in an order-
// preserving unsigned form, after -0 -> +0 and every NaN -> one canonical NaN (which orders above +inf); low word:
// 0xFFFFFFFF - caller edge index.  One unsigned 64-bit max then yields the largest message and, among equal ones,
// the smallest caller index, independent of the order the edges arrive in.  Key 0 (below every message) = no edge.
__device__ __forceinline__ unsigned long long max_key(float m, uint32_t caller_edge) {
  uint32_t u = __float_as_uint(m);
  if (m == 0.f) u = 0u;
  else if (m != m) u = 0x7FC00000u;
  const uint32_t o = (u & 0x80000000u) ? ~u : (u ^ 0x80000000u);
  return (static_cast<unsigned long long>(o) << 32) | (0xFFFFFFFFu - caller_edge);
}

// caller edge index of the sorted edge e (perm == nullptr: the caller's list was already grouped by source)
__device__ __forceinline__ uint32_t caller_edge(const int* perm, int64_t e) {
  return static_cast<uint32_t>(perm ? __ldg(perm + e) : e);
}

// bytes of the key array of an aggr = max application ([N, cout] uint64, rounded to 1 KiB)
inline size_t max_keys_bytes(int64_t N, int cout) {
  return static_cast<size_t>(round_up64(N * cout * 8, 1024));
}

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
