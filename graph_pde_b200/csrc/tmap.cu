#include "tmap.h"

#include <cudaTypedefs.h>
#include <cstdlib>

#include "kernels.h"
#include "options.h"
#include <mutex>

namespace nnc {

namespace {
PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
std::once_flag g_once;
int g_status = NNCONV_OK;
}  // namespace

int tmap_init() {
  std::call_once(g_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr) {
      set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
      g_status = NNCONV_ERR_CUDA;
      return;
    }
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  });
  return g_status;
}

namespace {
// cuTensorMapEncodeTiled costs microseconds; one conv application issues hundreds of launches that reuse a
// handful of (base, shape, box) combinations, so encoded descriptors are memoised per host thread.
struct TmapKey {
  const void* base;
  uint64_t rows, cols;
  uint32_t box_rows;
  int bf;
  int kind;   // 0: [box_rows x 64] SWIZZLE_128B operand tiles, 1: [16 x 32] SWIZZLE_64B store panels
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && box_rows == o.box_rows && bf == o.bf &&
           kind == o.kind;
  }
};
struct TmapEntry {
  TmapKey key;
  CUtensorMap map;
};
constexpr int kTmapCache = 128;
thread_local TmapEntry t_cache[kTmapCache];
thread_local int t_cache_n = 0;
thread_local int t_cache_next = 0;
}  // namespace

static int make_tmap_kind(CUtensorMap* out, int is_bf16, const void* base, uint64_t rows, uint64_t cols,
                          uint32_t box_rows, int kind) {
  const TmapKey key{base, rows, cols, box_rows, is_bf16, kind};
  for (int i = 0; i < t_cache_n; ++i) {
    if (t_cache[i].key == key) {
      *out = t_cache[i].map;
      return NNCONV_OK;
    }
  }
  int s = tmap_init();
  if (s != NNCONV_OK) return s;
  NNC_REQUIRE(cols % 64 == 0 && rows > 0 && box_rows >= 1 && box_rows <= 256 && rows < (1ull << 31), NNCONV_ERR_ARG,
              "tmap: bad shape rows=%llu cols=%llu box_rows=%u", (unsigned long long)rows,
              (unsigned long long)cols, box_rows);
  NNC_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, NNCONV_ERR_ARG, "tmap: base not 16B aligned");
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * 2};
  cuuint32_t box[2] = {kind == 1 ? 32u : 64u, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                        const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        kind == 1 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                        options().tmap_promo == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE
                        : options().tmap_promo == 1 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                                    : CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  NNC_REQUIRE(r == CUDA_SUCCESS, NNCONV_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  TmapEntry& e = t_cache[t_cache_next];
  e.key = key;
  e.map = *out;
  t_cache_next = (t_cache_next + 1) % kTmapCache;
  if (t_cache_n < kTmapCache) ++t_cache_n;
  return NNCONV_OK;
}

int make_tmap_2d_16b(CUtensorMap* out, int is_bf16, const void* base, uint64_t rows, uint64_t cols,
                     uint32_t box_rows) {
  return make_tmap_kind(out, is_bf16, base, rows, cols, box_rows, 0);
}

int make_tmap_store_16b(CUtensorMap* out, int is_bf16, const void* base, uint64_t rows, uint64_t cols) {
  return make_tmap_kind(out, is_bf16, base, rows, cols, 16, 1);
}

// ---- tracing buffer (debug) ------------------------------------------------------------------------
namespace {
TraceHandle g_trace{nullptr, nullptr, 0};
bool g_trace_checked = false;
}
TraceHandle trace_get() {
  if (!g_trace_checked) {
    g_trace_checked = true;
    if (options().trace > 0) {
      const unsigned int cap = 1u << 20;
      if (cudaMalloc(&g_trace.rec, static_cast<size_t>(cap) * 6 * sizeof(unsigned long long)) == cudaSuccess &&
          cudaMalloc(&g_trace.count, sizeof(unsigned int)) == cudaSuccess) {
        cudaMemset(g_trace.count, 0, sizeof(unsigned int));
        g_trace.cap = cap;
      } else {
        g_trace = TraceHandle{nullptr, nullptr, 0};
      }
    }
  }
  return g_trace;
}
int trace_dump(unsigned long long* host_rec, unsigned int max_rec, unsigned int* n_out) {
  *n_out = 0;
  if (!g_trace.rec) return NNCONV_OK;
  NNC_CHECK_CUDA(cudaDeviceSynchronize());
  unsigned int n = 0;
  NNC_CHECK_CUDA(cudaMemcpy(&n, g_trace.count, sizeof(n), cudaMemcpyDeviceToHost));
  if (n > g_trace.cap) n = g_trace.cap;
  if (n > max_rec) n = max_rec;
  NNC_CHECK_CUDA(cudaMemcpy(host_rec, g_trace.rec, static_cast<size_t>(n) * 6 * sizeof(unsigned long long),
                            cudaMemcpyDeviceToHost));
  NNC_CHECK_CUDA(cudaMemset(g_trace.count, 0, sizeof(unsigned int)));
  *n_out = n;
  return NNCONV_OK;
}

}  // namespace nnc
