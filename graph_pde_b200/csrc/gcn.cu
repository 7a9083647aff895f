// GCNConv (Kipf & Welling; the PyG 1.x operator of the reference's neurips4_GCN.py baseline, DESIGN 4.8):
//   out = A_hat x Theta + bias,   A_hat[n, m] = sum_{e: dst_e = n, src_e = m} norm_e  +  [n == m] self_n
// The graph (built once per edge_index) holds A_hat twice without its diagonal -- a CSR by destination for the forward
// and one by source for the backward, rows stable in the caller's edge order -- plus the diagonal self_n.
// Forward: z = A_hat x gathered row by row, then z Theta; backward: w = A_hat^T g, dx = w Theta^T, dTheta = x^T w,
// dbias = sum_n g_n.  Every row is written once and every sum runs in a fixed order: no atomics, so forward and backward
// are bitwise reproducible run to run.
//
// 16-bit precisions (in, out multiples of 16 in [16, 128]): k_gcn_tc, one persistent kernel per application.  Eight
// producer warps gather 128-row tiles of z (or w) in fp32, divide each row by the power of two >= its max-abs (range
// safety, as k_src_prep) and store it 16-bit into a double-buffered SWIZZLE_128B A tile; Theta stays resident as the B
// operand; one consumer warpgroup runs wgmma and writes fp32 out with the row scale multiplied back.  Everything else
// (precision fp32, other shapes, dTheta and dbias) runs on the CUDA cores.
#include <cub/cub.cuh>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "kernels.h"
#include "tc05.cuh"

namespace nnc {

struct GcnGraph {
  int64_t N, E;          // E: caller edges (self loops included; they leave the CSRs)
  int flags;
  const int* fwd_ptr;    // [N + 1] by destination
  const int* fwd_idx;    // source node of each entry
  const float* fwd_norm;
  const int* bwd_ptr;    // [N + 1] by source
  const int* bwd_idx;    // destination node of each entry
  const float* bwd_norm;
  const float* self;     // [N] diagonal of A_hat
};

namespace {

constexpr int kGcnTb = 256;
constexpr int kGcnRows = 128;                 // rows (nodes) per tensor-core tile
constexpr int kGcnThreads = 128 + 256;        // consumer warpgroup + two producer warpgroups
constexpr int kProducerRegs = 120, kConsumerRegs = 232;   // 2 x 128 x 120 + 128 x 232 <= 384 x 168
constexpr int kGcnChunks = 128;               // row chunks of the deterministic dTheta / dbias reduction
enum { BAR_FULL = 1, BAR_EMPTY = 3 };         // named barriers FULL + s, EMPTY + s of the two A stages

__device__ __forceinline__ void named_bar_arrive(int id, int n) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// power of two >= m (m finite, >= 0; 1 for m == 0), as k_src_prep
__device__ __forceinline__ float pow2_ceil(float m) {
  if (!(m > 0.f && m <= 3.0e38f)) return 1.f;
  int e;
  const float f = frexpf(m, &e);
  e = f == 0.5f ? e - 1 : e;
  e = e < -100 ? -100 : (e > 126 ? 126 : e);
  return ldexpf(1.f, e);
}

// ---------------------------------------------------------------- graph build
__global__ void k_gcn_count(const int64_t* __restrict__ src, const int64_t* __restrict__ dst, int64_t E, int64_t N,
                            int* __restrict__ indeg, int* __restrict__ loops, int* __restrict__ keys_d,
                            int* __restrict__ keys_s, int* __restrict__ vals, int* __restrict__ flags) {
  const int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (e >= E) return;
  const int64_t s = src[e], d = dst[e];
  vals[e] = static_cast<int>(e);
  if (s < 0 || s >= N || d < 0 || d >= N) {
    atomicOr(flags, 1);
    keys_d[e] = keys_s[e] = static_cast<int>(N);
    return;
  }
  if (s == d) {                                  // a caller's self loop leaves the edge list (sorted past the rows)
    atomicAdd(&loops[d], 1);
    keys_d[e] = keys_s[e] = static_cast<int>(N);
  } else {
    atomicAdd(&indeg[d], 1);
    keys_d[e] = static_cast<int>(d);
    keys_s[e] = static_cast<int>(s);
  }
}

// per node: the loop weight w (add_remaining_self_loops: 1 if the caller had a loop, else fill; without added loops or
// normalisation: the caller's loops, each of weight 1), deg = in-degree + w, dinv = deg^-1/2 (0 for deg 0), self.
__global__ void k_gcn_deg(const int* __restrict__ indeg, const int* __restrict__ loops, int64_t N, int flags,
                          float* __restrict__ dinv, float* __restrict__ self) {
  const int64_t n = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (n >= N) return;
  const bool normalize = !(flags & NNCONV_GCN_NO_NORMALIZE);
  const bool add_loops = normalize && !(flags & NNCONV_GCN_NO_SELF_LOOPS);
  const float fill = (flags & NNCONV_GCN_IMPROVED) ? 2.f : 1.f;
  const float w = add_loops ? (loops[n] > 0 ? 1.f : fill) : static_cast<float>(loops[n]);
  if (!normalize) {
    dinv[n] = 1.f;
    self[n] = w;
    return;
  }
  const float deg = static_cast<float>(indeg[n]) + w;
  const float di = deg > 0.f ? 1.f / sqrtf(deg) : 0.f;
  dinv[n] = di;
  self[n] = di * w * di;
}

__global__ void k_gcn_outdeg(const int* __restrict__ keys_s, int64_t E, int* __restrict__ outdeg, int64_t N) {
  const int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (e >= E) return;
  const int s = keys_s[e];
  if (s < N) atomicAdd(&outdeg[s], 1);
}

// CSR entries: sorted position p (< ptr[N]: the loops sorted past the rows) -> caller edge perm[p]
__global__ void k_gcn_fill(const int64_t* __restrict__ src, const int64_t* __restrict__ dst, const int* __restrict__ perm,
                           int64_t E, const int* __restrict__ ptr, int64_t N, int by_src, const float* __restrict__ dinv,
                           int* __restrict__ idx, float* __restrict__ norm) {
  const int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (p >= E || p >= ptr[N]) return;
  const int e = perm[p];
  const int s = static_cast<int>(src[e]), d = static_cast<int>(dst[e]);
  idx[p] = by_src ? d : s;
  norm[p] = dinv[s] * dinv[d];
}

size_t cub_bytes(int64_t E, int64_t N) {
  size_t a = 0, b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, a, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                static_cast<int>(N + 1));
  cub::DeviceRadixSort::SortPairs(nullptr, b, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                  static_cast<int*>(nullptr), static_cast<int*>(nullptr), static_cast<int>(E + 1));
  return a > b ? a : b;
}

struct GcnLayout {
  int *fwd_ptr, *fwd_idx, *bwd_ptr, *bwd_idx;
  float *fwd_norm, *bwd_norm, *self;
  size_t bytes;
};
GcnLayout carve_graph(void* ws, int64_t E, int64_t N) {
  Carver c(ws, ~size_t(0));
  GcnLayout L;
  L.fwd_ptr = c.take<int>(N + 1);
  L.fwd_idx = c.take<int>(E + 1);
  L.fwd_norm = c.take<float>(E + 1);
  L.bwd_ptr = c.take<int>(N + 1);
  L.bwd_idx = c.take<int>(E + 1);
  L.bwd_norm = c.take<float>(E + 1);
  L.self = c.take<float>(N + 1);
  L.bytes = c.off;
  return L;
}
struct GcnTmp {
  int *indeg, *outdeg, *loops, *flags, *keys_d, *keys_s, *keys_out, *vals, *perm;
  float* dinv;
  void* cub_tmp;
  size_t cub_bytes, bytes;
};
GcnTmp carve_tmp(void* tmp, int64_t E, int64_t N) {
  Carver c(tmp, ~size_t(0));
  GcnTmp T;
  T.indeg = c.take<int>(N + 1);
  T.outdeg = c.take<int>(N + 1);
  T.loops = c.take<int>(N + 1);
  T.flags = c.take<int>(8);
  T.keys_d = c.take<int>(E + 1);
  T.keys_s = c.take<int>(E + 1);
  T.keys_out = c.take<int>(E + 1);
  T.vals = c.take<int>(E + 1);
  T.perm = c.take<int>(E + 1);
  T.dinv = c.take<float>(N + 1);
  T.cub_bytes = cub_bytes(E, N);
  T.cub_tmp = c.take<char>(T.cub_bytes + 256);
  T.bytes = c.off;
  return T;
}

// ---------------------------------------------------------------- CUDA-core kernels
// z[n, :] = self_n v[n, :] + sum_{p in row n} norm_p v[idx_p, :]   (one warp per row, fixed order)
__global__ void __launch_bounds__(256) k_gcn_gather(const int* __restrict__ ptr, const int* __restrict__ idx,
                                                    const float* __restrict__ norm, const float* __restrict__ self,
                                                    const float* __restrict__ v, int64_t N, int C, float* __restrict__ z) {
  const int64_t n = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  const int p0 = __ldg(ptr + n), p1 = __ldg(ptr + n + 1);
  const float sn = __ldg(self + n);
  for (int c = lane; c < C; c += 32) {
    float acc = sn * __ldg(v + n * C + c);
    for (int p = p0; p < p1; ++p) acc = fmaf(__ldg(norm + p), __ldg(v + static_cast<int64_t>(__ldg(idx + p)) * C + c), acc);
    z[n * C + c] = acc;
  }
}

__global__ void k_gcn_transpose(const float* __restrict__ src, int R, int C, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * C) return;
  const int r = i / C, c = i - r * C;
  dst[static_cast<int64_t>(c) * R + r] = src[i];
}

__global__ void k_gcn_bias(float* __restrict__ out, int64_t N, int C, const float* __restrict__ bias) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= N * C) return;
  out[i] += bias[i % C];
}

// partial[chunk][m][n] = sum_{r in chunk} A[r, m] B[r, n]  (A [R, M], B [R, Nc] fp32 row-major; 64 x 64 output tiles)
__global__ void __launch_bounds__(256) k_gcn_sgemm_tn(const float* __restrict__ A, int M, const float* __restrict__ B,
                                                      int Nc, int64_t R, int64_t rows_per_chunk,
                                                      float* __restrict__ partial) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.z * 64;
  const int64_t r0 = blockIdx.x * rows_per_chunk;
  const int64_t r1 = r0 + rows_per_chunk < R ? r0 + rows_per_chunk : R;
  float acc[4][4] = {};
  for (int64_t k0 = r0; k0 < r1; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int kk = i / 64, c = i % 64;
      const int64_t r = k0 + kk;
      As[kk][c] = (r < r1 && m0 + c < M) ? A[r * M + m0 + c] : 0.f;
      Bs[kk][c] = (r < r1 && n0 + c < Nc) ? B[r * Nc + n0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* P = partial + static_cast<int64_t>(blockIdx.x) * M * Nc;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < Nc) P[static_cast<int64_t>(m) * Nc + n] = acc[i][j];
    }
  }
}

// pb[chunk][c] = sum_{r in chunk} g[r, c]
__global__ void k_gcn_colsum(const float* __restrict__ g, int C, int64_t R, int64_t rows_per_chunk, float* __restrict__ pb) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int64_t r0 = blockIdx.x * rows_per_chunk;
  const int64_t r1 = r0 + rows_per_chunk < R ? r0 + rows_per_chunk : R;
  float acc = 0.f;
  for (int64_t r = r0; r < r1; ++r) acc += g[r * C + c];
  pb[static_cast<int64_t>(blockIdx.x) * C + c] = acc;
}

// dst[q] = sum_chunk partial[chunk][q] in chunk order, for q < n (and the same for the bias partials, nullable)
__global__ void k_gcn_reduce(const float* __restrict__ partial, int64_t n, const float* __restrict__ pb, int nb, int chunks,
                             float* __restrict__ dst, float* __restrict__ dbias) {
  const int64_t q = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (q < n) {
    float acc = 0.f;
    for (int c = 0; c < chunks; ++c) acc += partial[c * n + q];
    dst[q] = acc;
  } else if (dbias != nullptr && q < n + nb) {
    const int64_t j = q - n;
    float acc = 0.f;
    for (int c = 0; c < chunks; ++c) acc += pb[c * nb + j];
    dbias[j] = acc;
  }
}

// ---------------------------------------------------------------- tensor-core application
struct GcnTcArgs {
  const int* ptr;
  const int* idx;
  const float* norm;
  const float* self;
  const float* v;        // gathered rows [N, K] fp32: x (forward) or g (backward)
  const float* theta;    // [cin, cout] fp32
  const float* bias;     // [NO] or nullptr
  float* out;            // [N, NO]
  float* wrows;          // backward: the gathered fp32 rows [N, K] (dTheta = x^T w), else nullptr
  int64_t N;
  int K;                 // reduction width: cin (forward) or cout (backward)
  int n_tiles;
};

template <int FMT>
struct GcnT;
template <>
struct GcnT<0> { using T = __half; static __device__ T cvt(float v) { return __float2half_rn(v); } };
template <>
struct GcnT<1> { using T = __nv_bfloat16; static __device__ T cvt(float v) { return __float2bfloat16_rn(v); } };
template <>
struct GcnT<2> { using T = __half; static __device__ T cvt(float v) { return __float2half_rn(v); } };

__device__ __forceinline__ uint32_t pack2(__half a, __half b) {
  return static_cast<uint32_t>(__half_as_ushort(a)) | (static_cast<uint32_t>(__half_as_ushort(b)) << 16);
}
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
}

// byte offset of element (row r, column c) in a SWIZZLE_128B K-major panel set of `rows` rows per 64-column panel
__device__ __forceinline__ uint32_t sw128_off(int r, int c, int rows) {
  return static_cast<uint32_t>((c >> 6) * rows * 128 + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
}

// dynamic shared memory of k_gcn_tc (+ 1 KB to align the base to the 128B swizzle atom)
__host__ __device__ inline size_t gcn_tc_smem(int fmt, int K, int NO) {
  const int kp = (K + 63) / 64;
  const int split = fmt == 2;
  return static_cast<size_t>(kp) * (split ? 3 : 1) * NO * 128 + 2 * static_cast<size_t>(kp) * (split ? 2 : 1) * kGcnRows * 128 +
         2 * kGcnRows * 4 + 128 + 1024;
}

// FMT 0 fp16, 1 bf16, 2 f16x2 (A = [hi | lo], B = [hi | lo | hi] of the pre-scaled Theta: hi*hi + hi*lo + lo*hi).
// BWD: B[n][k] = Theta[n][k] (dx = w Theta^T), else B[n][k] = Theta[k][n] (out = z Theta).
template <int FMT, int NO, bool BWD>
__global__ void __launch_bounds__(kGcnThreads, 1) k_gcn_tc(GcnTcArgs a) {
  using T = typename GcnT<FMT>::T;
  constexpr int SPLIT = FMT == 2;
  constexpr int WF = FMT == 1 ? 1 : 0;          // wgmma operand format
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int K = a.K;
  const int kp = (K + 63) / 64;
  unsigned char* Bs = smem;
  const uint32_t b_bytes = static_cast<uint32_t>(kp * (SPLIT ? 3 : 1) * NO * 128);
  const uint32_t a_stage = static_cast<uint32_t>(kp * (SPLIT ? 2 : 1) * kGcnRows * 128);
  unsigned char* As = smem + b_bytes;
  float* rs = reinterpret_cast<float*>(As + 2 * a_stage);     // [2][kGcnRows] row scales
  float* red = rs + 2 * kGcnRows;                              // [32] reduction scratch
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cin = BWD ? NO : K, cout = BWD ? K : NO;

  // Theta pre-scaled by the power of two s with max|Theta| s in [0.5, 1): exact, and the lo halves of f16x2 stay normal
  float m = 0.f;
  for (int i = tid; i < cin * cout; i += kGcnThreads) m = fmaxf(m, fabsf(__ldg(a.theta + i)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  float mm = 0.f;
  for (int w = 0; w < kGcnThreads / 32; ++w) mm = fmaxf(mm, red[w]);
  int te = 0;                                    // s = 2^-e with max|Theta| = f 2^e, f in [0.5, 1)
  if (mm > 0.f && mm <= 3.0e38f) frexpf(mm, &te);
  te = te < -100 ? -100 : (te > 100 ? 100 : te);
  const float ts = ldexpf(1.f, -te), inv_ts = ldexpf(1.f, te);
  for (int i = tid; i < NO * K; i += kGcnThreads) {
    const int n = i / K, k = i - n * K;
    const float v = (BWD ? __ldg(a.theta + static_cast<int64_t>(n) * cout + k) : __ldg(a.theta + static_cast<int64_t>(k) * cout + n)) * ts;
    const T hi = GcnT<FMT>::cvt(v);
    *reinterpret_cast<T*>(Bs + sw128_off(n, k, NO)) = hi;
    if constexpr (SPLIT) {
      const uint32_t blk = static_cast<uint32_t>(kp * NO * 128);
      *reinterpret_cast<T*>(Bs + blk + sw128_off(n, k, NO)) = GcnT<FMT>::cvt(v - __half2float(hi));
      *reinterpret_cast<T*>(Bs + 2 * blk + sw128_off(n, k, NO)) = hi;
    }
  }
  tc05::fence_proxy_async_smem();
  __syncthreads();

  // registers: the launch gives every thread 168 (384 threads, one CTA per SM); the producers hand registers to the
  // consumer, whose [128 x NO] fp32 accumulator alone takes 128 of them at NO = 128 (no spill at f16x2)
  if (warp >= 4) {
    tc05::warpgroup_reg_dealloc<kProducerRegs>();
    // ---------------- producers: 8 warps, each row gathered by the lanes of a power-of-two group, 4 columns per lane
    const int pw = warp - 4;
    int lpr = 4;
    while (lpr * 4 < K) lpr *= 2;
    const int rpw = 32 / lpr;
    const int sub = lane / lpr, cl = lane % lpr;
    const bool active = cl * 4 < K;
    const unsigned gmask = (lpr == 32 ? 0xffffffffu : ((1u << lpr) - 1u)) << (sub * lpr);
    int it = 0;
    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x, ++it) {
      const int s = it & 1;
      if (it >= 2) tc05::named_bar_sync(BAR_EMPTY + s, kGcnThreads);
      unsigned char* A = As + s * a_stage;
      // two rows per row slot in flight: their neighbour loads overlap
      for (int rr = pw * rpw + sub; rr < kGcnRows; rr += 2 * 8 * rpw) {
        const int rows[2] = {rr, rr + 8 * rpw};
        float4 acc[2];
        int p[2], pe[2];
        int64_t n[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          n[u] = static_cast<int64_t>(tile) * kGcnRows + rows[u];
          acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          p[u] = pe[u] = 0;
          if (rows[u] < kGcnRows && n[u] < a.N) {
            p[u] = __ldg(a.ptr + n[u]);
            pe[u] = __ldg(a.ptr + n[u] + 1);
            if (active) {
              const float sn = __ldg(a.self + n[u]);
              const float4 xv = __ldg(reinterpret_cast<const float4*>(a.v + n[u] * K) + cl);
              acc[u] = make_float4(sn * xv.x, sn * xv.y, sn * xv.z, sn * xv.w);
            }
          }
        }
        if (active) {
          while (p[0] < pe[0] || p[1] < pe[1]) {
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              if (p[u] < pe[u]) {
                const float w = __ldg(a.norm + p[u]);
                const int j = __ldg(a.idx + p[u]);
                const float4 xv = __ldg(reinterpret_cast<const float4*>(a.v + static_cast<int64_t>(j) * K) + cl);
                acc[u].x = fmaf(w, xv.x, acc[u].x);
                acc[u].y = fmaf(w, xv.y, acc[u].y);
                acc[u].z = fmaf(w, xv.z, acc[u].z);
                acc[u].w = fmaf(w, xv.w, acc[u].w);
                ++p[u];
              }
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int r = rows[u];
          float mx = fmaxf(fmaxf(fabsf(acc[u].x), fabsf(acc[u].y)), fmaxf(fabsf(acc[u].z), fabsf(acc[u].w)));
          for (int o = lpr / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(gmask, mx, o));
          if (r >= kGcnRows) continue;
          const float sc = pow2_ceil(mx), inv = 1.f / sc;
          if (cl == 0) rs[s * kGcnRows + r] = sc;
          if (!active) continue;
          if (BWD && a.wrows != nullptr && n[u] < a.N) reinterpret_cast<float4*>(a.wrows + n[u] * K)[cl] = acc[u];
          const float v0 = acc[u].x * inv, v1 = acc[u].y * inv, v2 = acc[u].z * inv, v3 = acc[u].w * inv;
          const T h0 = GcnT<FMT>::cvt(v0), h1 = GcnT<FMT>::cvt(v1), h2 = GcnT<FMT>::cvt(v2), h3 = GcnT<FMT>::cvt(v3);
          const uint32_t off = sw128_off(r, 4 * cl, kGcnRows);
          *reinterpret_cast<uint2*>(A + off) = make_uint2(pack2(h0, h1), pack2(h2, h3));
          if constexpr (SPLIT) {
            const T l0 = GcnT<FMT>::cvt(v0 - __half2float(h0)), l1 = GcnT<FMT>::cvt(v1 - __half2float(h1));
            const T l2 = GcnT<FMT>::cvt(v2 - __half2float(h2)), l3 = GcnT<FMT>::cvt(v3 - __half2float(h3));
            *reinterpret_cast<uint2*>(A + kp * kGcnRows * 128 + off) = make_uint2(pack2(l0, l1), pack2(l2, l3));
          }
        }
      }
      tc05::fence_proxy_async_smem();
      named_bar_arrive(BAR_FULL + s, kGcnThreads);
    }
  } else {
    tc05::warpgroup_reg_alloc<kConsumerRegs>();
    // ---------------- consumer warpgroup: wgmma over the tile, epilogue straight from the accumulator fragments
    tc05::Acc<NO> acc;
    const uint32_t b_base = tc05::smem_u32(Bs);
    const int ksteps = K / 16;
    int it = 0;
    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x, ++it) {
      const int s = it & 1;
      tc05::named_bar_sync(BAR_FULL + s, kGcnThreads);
      const uint32_t a_base = tc05::smem_u32(As + s * a_stage);
      tc05::wgmma_fence();
#pragma unroll
      for (int pass = 0; pass < (SPLIT ? 3 : 1); ++pass) {
        const uint32_t ap = a_base + (pass == 2 ? kp * kGcnRows * 128 : 0);
        const uint32_t bp = b_base + pass * kp * NO * 128;
#pragma unroll 1
        for (int kk = 0; kk < ksteps; ++kk) {
          const uint64_t ad = tc05::smem_desc_sw128(ap + (kk >> 2) * kGcnRows * 128 + (kk & 3) * 32);
          const uint64_t bd = tc05::smem_desc_sw128(bp + (kk >> 2) * NO * 128 + (kk & 3) * 32);
          const int sd = (pass > 0 || kk > 0) ? 1 : 0;
          tc05::wgmma<NO, WF>(acc.d[0], ad, bd, sd);
          tc05::wgmma<NO, WF>(acc.d[1], ad + 512, bd, sd);   // rows 64..127: +8 KB
        }
      }
      tc05::wgmma_commit();
      tc05::wgmma_wait<0>();
      const int r0 = 16 * warp + (lane >> 2);
      float sc[4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        sc[2 * h] = rs[s * kGcnRows + 64 * h + r0] * inv_ts;
        sc[2 * h + 1] = rs[s * kGcnRows + 64 * h + r0 + 8] * inv_ts;
      }
      if (tile + 2 * static_cast<int>(gridDim.x) < a.n_tiles) named_bar_arrive(BAR_EMPTY + s, kGcnThreads);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int64_t n = static_cast<int64_t>(tile) * kGcnRows + 64 * h + r0 + 8 * half;
          if (n >= a.N) continue;
          const float f = sc[2 * h + half];
          float* orow = a.out + n * NO;
#pragma unroll
          for (int j = 0; j < NO / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            float2 v = make_float2(acc.d[h][4 * j + 2 * half] * f, acc.d[h][4 * j + 2 * half + 1] * f);
            if (a.bias != nullptr) {
              v.x += __ldg(a.bias + c);
              v.y += __ldg(a.bias + c + 1);
            }
            *reinterpret_cast<float2*>(orow + c) = v;
          }
        }
      }
    }
  }
}

bool gcn_tc_shape(int cin, int cout) {
  return cin % 16 == 0 && cout % 16 == 0 && cin >= 16 && cin <= 128 && cout >= 16 && cout <= 128;
}

template <int FMT, int NO, bool BWD>
int launch_gcn_tc_t(const GcnTcArgs& a, cudaStream_t st) {
  const size_t smem = gcn_tc_smem(FMT, a.K, NO);
  static int attr_set = 0;   // per instantiation: the largest dynamic shared memory any K needs
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_gcn_tc<FMT, NO, BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(gcn_tc_smem(FMT, 128, NO))));
    attr_set = 1;
  }
  int dev = 0, sms = 0;
  NNC_CHECK_CUDA(cudaGetDevice(&dev));
  NNC_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = a.n_tiles < sms ? a.n_tiles : sms;
  k_gcn_tc<FMT, NO, BWD><<<grid, kGcnThreads, smem, st>>>(a);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

template <int FMT, bool BWD>
int launch_gcn_tc_no(const GcnTcArgs& a, int NO, cudaStream_t st) {
  switch (NO) {
    case 16: return launch_gcn_tc_t<FMT, 16, BWD>(a, st);
    case 32: return launch_gcn_tc_t<FMT, 32, BWD>(a, st);
    case 48: return launch_gcn_tc_t<FMT, 48, BWD>(a, st);
    case 64: return launch_gcn_tc_t<FMT, 64, BWD>(a, st);
    case 80: return launch_gcn_tc_t<FMT, 80, BWD>(a, st);
    case 96: return launch_gcn_tc_t<FMT, 96, BWD>(a, st);
    case 112: return launch_gcn_tc_t<FMT, 112, BWD>(a, st);
    case 128: return launch_gcn_tc_t<FMT, 128, BWD>(a, st);
  }
  set_error("gcn: unsupported width %d", NO);
  return NNCONV_ERR_UNSUPPORTED;
}

int launch_gcn_tc(int prec, bool bwd, const GcnTcArgs& a, int NO, cudaStream_t st) {
  const int fmt = prec == PREC_F16 ? 0 : prec == PREC_BF16 ? 1 : 2;
  if (fmt == 0) return bwd ? launch_gcn_tc_no<0, true>(a, NO, st) : launch_gcn_tc_no<0, false>(a, NO, st);
  if (fmt == 1) return bwd ? launch_gcn_tc_no<1, true>(a, NO, st) : launch_gcn_tc_no<1, false>(a, NO, st);
  return bwd ? launch_gcn_tc_no<2, true>(a, NO, st) : launch_gcn_tc_no<2, false>(a, NO, st);
}

int64_t gcn_rows_per_chunk(int64_t N) { return ceil_div64(N, kGcnChunks); }

size_t gcn_apply_ws(const GcnGraph* G, int prec, int cin, int cout) {
  if (prec != PREC_FP32 && gcn_tc_shape(cin, cout)) return 0;
  return static_cast<size_t>(round_up64(G->N * cin * 4, 1024) + round_up64(static_cast<int64_t>(cin) * cout * 4, 1024));
}

size_t gcn_backward_ws(const GcnGraph* G, int cin, int cout) {
  return static_cast<size_t>(round_up64(G->N * cout * 4, 1024) + round_up64(static_cast<int64_t>(kGcnChunks) * cin * cout * 4, 1024) +
                             round_up64(static_cast<int64_t>(kGcnChunks) * cout * 4, 1024));
}

int gcn_check(const GcnGraph* G, int prec, int cin, int cout) {
  NNC_REQUIRE(G != nullptr, NNCONV_ERR_ARG, "gcn: null graph");
  NNC_REQUIRE(prec >= PREC_FP32 && prec <= PREC_F16X2, NNCONV_ERR_ARG, "gcn: unknown precision %d", prec);
  NNC_REQUIRE(cin >= 1 && cout >= 1, NNCONV_ERR_ARG, "gcn: need in, out >= 1 (got %d, %d)", cin, cout);
  NNC_REQUIRE(prec == PREC_FP32 || gcn_tc_shape(cin, cout), NNCONV_ERR_UNSUPPORTED,
              "GCNConv: in=%d, out=%d is not covered by the tensor-core kernel (multiples of 16 in [16, 128]); use "
              "precision 'fp32'", cin, cout);
  return NNCONV_OK;
}

}  // namespace

int gcn_graph_sizes(int64_t E, int64_t N, size_t* ws_bytes, size_t* tmp_bytes) {
  NNC_REQUIRE(ws_bytes && tmp_bytes, NNCONV_ERR_ARG, "null output pointer");
  NNC_REQUIRE(E >= 0 && N >= 1, NNCONV_ERR_ARG, "gcn graph: need E >= 0 and N >= 1");
  *ws_bytes = carve_graph(nullptr, E, N).bytes;
  *tmp_bytes = carve_tmp(nullptr, E, N).bytes;
  return NNCONV_OK;
}

int gcn_graph_build(GcnGraph* G, const int64_t* row0, const int64_t* row1, int64_t E, int64_t N, int flow, int flags,
                    void* ws, size_t ws_bytes, void* tmp, size_t tmp_bytes, cudaStream_t st) {
  NNC_REQUIRE(E >= 0 && N >= 1, NNCONV_ERR_ARG, "gcn graph: need E >= 0 and N >= 1 (got E=%lld N=%lld)", (long long)E,
              (long long)N);
  NNC_REQUIRE(E < (int64_t(1) << 31) - 256 && N < (int64_t(1) << 31) - 256, NNCONV_ERR_UNSUPPORTED,
              "gcn graph: E and N must fit int32");
  NNC_REQUIRE(flow == 0 || flow == 1, NNCONV_ERR_ARG, "gcn graph: flow must be 0 (source_to_target) or 1");
  NNC_REQUIRE((flags & ~7) == 0, NNCONV_ERR_ARG, "gcn graph: unknown flags 0x%x", flags);
  NNC_REQUIRE(ws != nullptr && tmp != nullptr, NNCONV_ERR_ARG, "gcn graph: null workspace");
  const GcnLayout L = carve_graph(ws, E, N);
  const GcnTmp T = carve_tmp(tmp, E, N);
  NNC_REQUIRE(L.bytes <= ws_bytes && T.bytes <= tmp_bytes, NNCONV_ERR_WORKSPACE,
              "gcn graph: workspace too small (need %zu + %zu bytes)", L.bytes, T.bytes);
  const int64_t* src = flow == 0 ? row0 : row1;
  const int64_t* dst = flow == 0 ? row1 : row0;
  const int TB = kGcnTb;
  NNC_CHECK_CUDA(cudaMemsetAsync(T.indeg, 0, (N + 1) * sizeof(int), st));
  NNC_CHECK_CUDA(cudaMemsetAsync(T.outdeg, 0, (N + 1) * sizeof(int), st));
  NNC_CHECK_CUDA(cudaMemsetAsync(T.loops, 0, (N + 1) * sizeof(int), st));
  NNC_CHECK_CUDA(cudaMemsetAsync(T.flags, 0, 8 * sizeof(int), st));
  if (E > 0) {
    k_gcn_count<<<(unsigned)ceil_div64(E, TB), TB, 0, st>>>(src, dst, E, N, T.indeg, T.loops, T.keys_d, T.keys_s, T.vals,
                                                            T.flags);
    NNC_CHECK_LAUNCH();
  }
  int h_flag = 0;
  NNC_CHECK_CUDA(cudaMemcpyAsync(&h_flag, T.flags, sizeof(int), cudaMemcpyDeviceToHost, st));
  NNC_CHECK_CUDA(cudaStreamSynchronize(st));
  NNC_REQUIRE(h_flag == 0, NNCONV_ERR_ARG, "gcn graph: edge_index has entries outside [0, N)");
  k_gcn_deg<<<(unsigned)ceil_div64(N, TB), TB, 0, st>>>(T.indeg, T.loops, N, flags, T.dinv, L.self);
  NNC_CHECK_LAUNCH();
  size_t cb = T.cub_bytes;
  NNC_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(T.cub_tmp, cb, T.indeg, L.fwd_ptr, static_cast<int>(N + 1), st));
  if (E > 0) {
    k_gcn_outdeg<<<(unsigned)ceil_div64(E, TB), TB, 0, st>>>(T.keys_s, E, T.outdeg, N);
    NNC_CHECK_LAUNCH();
  }
  cb = T.cub_bytes;
  NNC_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(T.cub_tmp, cb, T.outdeg, L.bwd_ptr, static_cast<int>(N + 1), st));
  if (E > 0) {
    int bits = 1;
    while ((int64_t(1) << bits) <= N) ++bits;    // keys in [0, N]: N marks a self loop
    for (int by_src = 0; by_src < 2; ++by_src) {
      cb = T.cub_bytes;
      // stable: within a row the entries keep the caller's edge order
      NNC_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(T.cub_tmp, cb, by_src ? T.keys_s : T.keys_d, T.keys_out, T.vals,
                                                     T.perm, static_cast<int>(E), 0, bits, st));
      k_gcn_fill<<<(unsigned)ceil_div64(E, TB), TB, 0, st>>>(src, dst, T.perm, E, by_src ? L.bwd_ptr : L.fwd_ptr, N, by_src,
                                                             T.dinv, by_src ? L.bwd_idx : L.fwd_idx,
                                                             by_src ? L.bwd_norm : L.fwd_norm);
      NNC_CHECK_LAUNCH();
    }
  }
  G->N = N;
  G->E = E;
  G->flags = flags;
  G->fwd_ptr = L.fwd_ptr;
  G->fwd_idx = L.fwd_idx;
  G->fwd_norm = L.fwd_norm;
  G->bwd_ptr = L.bwd_ptr;
  G->bwd_idx = L.bwd_idx;
  G->bwd_norm = L.bwd_norm;
  G->self = L.self;
  return NNCONV_OK;
}

int gcn_apply(const GcnGraph* G, int prec, int cin, int cout, const float* x, const float* theta, const float* bias,
              float* out, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches) {
  int s = gcn_check(G, prec, cin, cout);
  if (s) return s;
  NNC_REQUIRE(x && theta && out, NNCONV_ERR_ARG, "gcn apply: null x, weight or out");
  NNC_REQUIRE(ws_bytes >= gcn_apply_ws(G, prec, cin, cout) && (ws != nullptr || gcn_apply_ws(G, prec, cin, cout) == 0),
              NNCONV_ERR_WORKSPACE, "gcn apply: workspace too small (use nnconv_gcn_apply_sizes)");
  const int64_t N = G->N;
  int64_t n_l = 0;
  if (prec != PREC_FP32) {
    NNC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, NNCONV_ERR_ARG,
                "gcn apply: x and out must be 16-byte aligned");
    GcnTcArgs a{G->fwd_ptr, G->fwd_idx, G->fwd_norm, G->self, x, theta, bias, out, nullptr, N, cin,
                static_cast<int>(ceil_div64(N, kGcnRows))};
    s = launch_gcn_tc(prec, false, a, cout, st);
    if (s) return s;
    n_l = 1;
  } else {
    float* z = static_cast<float*>(ws);
    float* tt = reinterpret_cast<float*>(static_cast<char*>(ws) + round_up64(N * cin * 4, 1024));
    k_gcn_gather<<<(unsigned)ceil_div64(N * 32, 256), 256, 0, st>>>(G->fwd_ptr, G->fwd_idx, G->fwd_norm, G->self, x, N, cin, z);
    NNC_CHECK_LAUNCH();
    k_gcn_transpose<<<ceil_div(cin * cout, 256), 256, 0, st>>>(theta, cin, cout, tt);
    NNC_CHECK_LAUNCH();
    s = launch_sgemm_store(z, cin, tt, cin, out, cout, static_cast<int>(N), cout, cin, nullptr, st);
    if (s) return s;
    n_l = 3;
    if (bias != nullptr) {
      k_gcn_bias<<<(unsigned)ceil_div64(N * cout, 256), 256, 0, st>>>(out, N, cout, bias);
      NNC_CHECK_LAUNCH();
      ++n_l;
    }
  }
  if (launches) *launches += n_l;
  return NNCONV_OK;
}

int gcn_backward(const GcnGraph* G, int prec, int cin, int cout, const float* x, const float* theta, const float* gout,
                 float* dx, float* dtheta, float* dbias, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches) {
  int s = gcn_check(G, prec, cin, cout);
  if (s) return s;
  NNC_REQUIRE(x && theta && gout && dx && dtheta, NNCONV_ERR_ARG, "gcn backward: null x, weight, grad_out, grad_x or grad_weight");
  NNC_REQUIRE(ws != nullptr && ws_bytes >= gcn_backward_ws(G, cin, cout), NNCONV_ERR_WORKSPACE,
              "gcn backward: workspace too small (use nnconv_gcn_backward_sizes)");
  const int64_t N = G->N;
  float* w = static_cast<float*>(ws);
  float* partial = reinterpret_cast<float*>(static_cast<char*>(ws) + round_up64(N * cout * 4, 1024));
  float* pb = partial + round_up64(static_cast<int64_t>(kGcnChunks) * cin * cout * 4, 1024) / 4;
  int64_t n_l = 0;
  if (prec != PREC_FP32) {
    NNC_REQUIRE(((reinterpret_cast<uintptr_t>(gout) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0, NNCONV_ERR_ARG,
                "gcn backward: grad_out and grad_x must be 16-byte aligned");
    // w = A_hat^T g gathered over the by-source CSR; dx = w Theta^T on the tensor cores, w kept in fp32 for dTheta
    GcnTcArgs a{G->bwd_ptr, G->bwd_idx, G->bwd_norm, G->self, gout, theta, nullptr, dx, w, N, cout,
                static_cast<int>(ceil_div64(N, kGcnRows))};
    s = launch_gcn_tc(prec, true, a, cin, st);
    if (s) return s;
    n_l = 1;
  } else {
    k_gcn_gather<<<(unsigned)ceil_div64(N * 32, 256), 256, 0, st>>>(G->bwd_ptr, G->bwd_idx, G->bwd_norm, G->self, gout, N,
                                                                     cout, w);
    NNC_CHECK_LAUNCH();
    s = launch_sgemm_store(w, cout, theta, cout, dx, cin, static_cast<int>(N), cin, cout, nullptr, st);
    if (s) return s;
    n_l = 2;
  }
  // dTheta = x^T w and dbias = sum_n g_n: per-chunk partials, then one fixed-order sum over the chunks
  const int64_t rpc = gcn_rows_per_chunk(N);
  k_gcn_sgemm_tn<<<dim3(kGcnChunks, ceil_div(cin, 64), ceil_div(cout, 64)), 256, 0, st>>>(x, cin, w, cout, N, rpc, partial);
  NNC_CHECK_LAUNCH();
  n_l += 2;
  if (dbias != nullptr) {
    k_gcn_colsum<<<dim3(kGcnChunks, ceil_div(cout, 128)), 128, 0, st>>>(gout, cout, N, rpc, pb);
    NNC_CHECK_LAUNCH();
    ++n_l;
  }
  const int64_t nq = static_cast<int64_t>(cin) * cout + (dbias ? cout : 0);
  k_gcn_reduce<<<(unsigned)ceil_div64(nq, 256), 256, 0, st>>>(partial, static_cast<int64_t>(cin) * cout, pb, cout, kGcnChunks,
                                                               dtheta, dbias);
  NNC_CHECK_LAUNCH();
  if (launches) *launches += n_l;
  return NNCONV_OK;
}

}  // namespace nnc

using namespace nnc;

struct nnconv_gcn_graph {
  GcnGraph g;
};

extern "C" {

int nnconv_gcn_graph_sizes(int64_t E, int64_t N, size_t* ws_bytes, size_t* tmp_bytes) {
  return gcn_graph_sizes(E, N, ws_bytes, tmp_bytes);
}

int nnconv_gcn_graph_create(const int64_t* row0, const int64_t* row1, int64_t E, int64_t N, int flow, int flags, void* ws,
                            size_t ws_bytes, void* tmp, size_t tmp_bytes, void* stream, nnconv_gcn_graph_t** out) {
  NNC_REQUIRE(out != nullptr, NNCONV_ERR_ARG, "null output pointer");
  *out = nullptr;
  nnconv_gcn_graph* h = new (std::nothrow) nnconv_gcn_graph();
  NNC_REQUIRE(h != nullptr, NNCONV_ERR_ARG, "out of host memory");
  const int s = gcn_graph_build(&h->g, row0, row1, E, N, flow, flags, ws, ws_bytes, tmp, tmp_bytes,
                                static_cast<cudaStream_t>(stream));
  if (s != NNCONV_OK) {
    delete h;
    return s;
  }
  *out = h;
  return NNCONV_OK;
}

void nnconv_gcn_graph_destroy(nnconv_gcn_graph_t* graph) { delete graph; }

int nnconv_gcn_apply_sizes(const nnconv_gcn_graph_t* graph, int precision, int in_channels, int out_channels,
                           size_t* ws_bytes) {
  NNC_REQUIRE(graph && ws_bytes, NNCONV_ERR_ARG, "null argument");
  const int s = gcn_check(&graph->g, precision, in_channels, out_channels);
  if (s) return s;
  *ws_bytes = gcn_apply_ws(&graph->g, precision, in_channels, out_channels);
  return NNCONV_OK;
}

int nnconv_gcn_apply(const nnconv_gcn_graph_t* graph, int precision, int in_channels, int out_channels, const float* x,
                     const float* weight, const float* bias, float* out, void* ws, size_t ws_bytes, void* stream,
                     int64_t* launches) {
  NNC_REQUIRE(graph != nullptr, NNCONV_ERR_ARG, "null graph");
  return gcn_apply(&graph->g, precision, in_channels, out_channels, x, weight, bias, out, ws, ws_bytes,
                   static_cast<cudaStream_t>(stream), launches);
}

int nnconv_gcn_backward_sizes(const nnconv_gcn_graph_t* graph, int precision, int in_channels, int out_channels,
                              size_t* ws_bytes) {
  NNC_REQUIRE(graph && ws_bytes, NNCONV_ERR_ARG, "null argument");
  const int s = gcn_check(&graph->g, precision, in_channels, out_channels);
  if (s) return s;
  *ws_bytes = gcn_backward_ws(&graph->g, in_channels, out_channels);
  return NNCONV_OK;
}

int nnconv_gcn_backward(const nnconv_gcn_graph_t* graph, int precision, int in_channels, int out_channels, const float* x,
                        const float* weight, const float* grad_out, float* grad_x, float* grad_weight, float* grad_bias,
                        void* ws, size_t ws_bytes, void* stream, int64_t* launches) {
  NNC_REQUIRE(graph != nullptr, NNCONV_ERR_ARG, "null graph");
  return gcn_backward(&graph->g, precision, in_channels, out_channels, x, weight, grad_out, grad_x, grad_weight, grad_bias,
                      ws, ws_bytes, static_cast<cudaStream_t>(stream), launches);
}

}  // extern "C"
