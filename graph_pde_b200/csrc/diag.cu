// Diagonal-kernel NNConv (formulation D, DESIGN 4.7): the reference's graph-neural-operator/nn_conv.py:8-96 NNConv,
// whose message is x_j . diag(k_e) with k_e = nn(edge_attr_e) in R^out (in == out):
//   d_e = W_L h_e + b_L                         x-independent: built once per (edge_attr, parameters), fp32 [E, out]
//   out_n = aggr_{e: dst_e = n} x_src(e) * d_e  +  x_n root + bias
// diag_build computes d chunk by chunk from edge_attr (edge_features_rows, then one GEMM per chunk), so only d lives in
// device memory.  Each application is one pass over d (4 * out bytes per edge) with fp32 reductions into out.
#include <cuda_fp16.h>

#include "kernels.h"
#include "options.h"

namespace nnc {

namespace {

constexpr size_t kDiagHeader = 1024;   // ws[0]: fp16 range counter of the chunks (nnconv_edge_features_overflow)

// d[r, o] = sum_k h[r, k] WL[o, k] + bL[o] for the rows r < n of a chunk (CUDA cores, fp32 accumulation).
// SPLIT = 0: h fp32 row-major [n, Kp] (precision fp32); SPLIT = 1: h fp16 (hi, lo) pairs in chunk-major panels of hpad
// rows, the lo panels after the Kp / 64 hi panels (precision f16x2).  WL fp32 [cout, Kp], zero past K.
template <int SPLIT>
__global__ void __launch_bounds__(256) k_diag_build(const void* __restrict__ h, int n, int64_t hpad, int Kp,
                                                    const float* __restrict__ WL, const float* __restrict__ bL, int cout,
                                                    float* __restrict__ d) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < Kp; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i / 16, kk = i % 16;
      const int gm = m0 + r, gn = n0 + r, gk = k0 + kk;
      float a = 0.f;
      if (gm < n) {
        if (SPLIT) {
          const __half* hh = static_cast<const __half*>(h);
          const int64_t idx = (static_cast<int64_t>(gk / 64) * hpad + gm) * 64 + gk % 64;
          a = __half2float(hh[idx]) + __half2float(hh[idx + static_cast<int64_t>(Kp / 64) * hpad * 64]);
        } else {
          a = static_cast<const float*>(h)[static_cast<int64_t>(gm) * Kp + gk];
        }
      }
      As[kk][r] = a;
      Bs[kk][r] = gn < cout ? WL[static_cast<int64_t>(gn) * Kp + gk] : 0.f;
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
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= n) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn < cout) d[static_cast<int64_t>(gm) * cout + gn] = acc[i][j] + bL[gn];
    }
  }
}

// One warp per plan tile (<= 128 edges of one source, so a hub source spreads over many warps): for every edge e of the
// tile and channel o, m = x_src[o] * d_e[o] (times inv_deg[dst] for mean) is added into out[dst, o] (AGGR 0 add, 1
// mean) or reduced into the max key of (dst, o) (AGGR 2).  VEC: out % 4 == 0, 16-byte loads of d and x and one
// red.global.add.v4.f32 per four channels.
template <int AGGR, bool VEC>
__global__ void __launch_bounds__(256) k_apply_diag(const float* __restrict__ d, const float* __restrict__ x, int cout,
                                                    int n_tiles, const int* __restrict__ tile_c,
                                                    const int* __restrict__ tile_e0, const int* __restrict__ tile_cnt,
                                                    const int* __restrict__ src_nodes, const int* __restrict__ dst_sorted,
                                                    const float* __restrict__ inv_deg, const int* __restrict__ perm,
                                                    float* __restrict__ out, unsigned long long* __restrict__ keys) {
  const int t = static_cast<int>((blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const int e0 = __ldg(tile_e0 + t), cnt = __ldg(tile_cnt + t);
  const float* xs = x + static_cast<int64_t>(__ldg(src_nodes + __ldg(tile_c + t))) * cout;
  const int q = VEC ? cout / 4 : cout;
  for (int i = lane; i < cnt * q; i += 32) {
    const int p = i / q, j = i - p * q;
    const int64_t e = e0 + p;
    const int dn = __ldg(dst_sorted + e);
    const float w = AGGR == 1 ? __ldg(inv_deg + dn) : 1.f;
    if (VEC) {
      const float4 dv = __ldcs(reinterpret_cast<const float4*>(d + e * cout) + j);
      const float4 xv = __ldg(reinterpret_cast<const float4*>(xs) + j);
      float4 m = make_float4(xv.x * dv.x, xv.y * dv.y, xv.z * dv.z, xv.w * dv.w);
      if (AGGR == 1) m = make_float4(m.x * w, m.y * w, m.z * w, m.w * w);
      if (AGGR == 2) {
        const uint32_t ce = caller_edge(perm, e);
        unsigned long long* k = keys + static_cast<int64_t>(dn) * cout + 4 * j;
        atomicMax(k, max_key(m.x, ce));
        atomicMax(k + 1, max_key(m.y, ce));
        atomicMax(k + 2, max_key(m.z, ce));
        atomicMax(k + 3, max_key(m.w, ce));
      } else {
        atomicAdd(reinterpret_cast<float4*>(out + static_cast<int64_t>(dn) * cout) + j, m);
      }
    } else {
      float m = __ldg(xs + j) * __ldcs(d + e * cout + j);
      if (AGGR == 1) m *= w;
      if (AGGR == 2) atomicMax(keys + static_cast<int64_t>(dn) * cout + j, max_key(m, caller_edge(perm, e)));
      else atomicAdd(out + static_cast<int64_t>(dn) * cout + j, m);
    }
  }
}

bool diag_tc_build(const Weights* W) { return W->prec == PREC_F16 || W->prec == PREC_BF16; }

size_t diag_h_row_bytes(const Weights* W) { return W->prec == PREC_FP32 ? static_cast<size_t>(W->Kp) * 4 : h_row_bytes(W); }

}  // namespace

size_t diag_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes) {
  const size_t row = diag_h_row_bytes(W) + ef_row_bytes(W);
  const int64_t all = round_up64(P->E > 0 ? P->E : 1, 128);
  int64_t rows = static_cast<int64_t>(want_bytes / row) / 128 * 128;
  if (rows < 128) rows = 128;
  if (rows > all) rows = all;
  return kDiagHeader + static_cast<size_t>(rows) * row + 2 * 4096 + 1024;
}

int diag_build(const Plan* P, const Weights* W, const float* edge_attr, float* d, void* ws, size_t ws_bytes, cudaStream_t st,
               int64_t* launches) {
  NNC_REQUIRE(W->diag, NNCONV_ERR_ARG, "diag_build: weights not prepared as a diagonal kernel");
  NNC_REQUIRE(W->prec == PREC_FP32 || (tc_shapes_supported(W) && (W->split || W->cout % 64 == 0)), NNCONV_ERR_UNSUPPORTED,
              "diagonal kernel: out=%d, K=%d not supported by the tensor-core edge network; use precision fp32",
              W->cout, W->K);
  NNC_REQUIRE(ws != nullptr && ws_bytes >= kDiagHeader, NNCONV_ERR_WORKSPACE, "diag_build: workspace too small");
  int* overflow = static_cast<int*>(ws);
  NNC_CHECK_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int), st));
  if (P->E == 0) return NNCONV_OK;
  if (!options().overflow_check) overflow = nullptr;
  const size_t hrow = diag_h_row_bytes(W), row = hrow + ef_row_bytes(W);
  const int64_t rows = static_cast<int64_t>((ws_bytes - kDiagHeader - 2 * 4096 - 1024) / row) / 128 * 128;
  NNC_REQUIRE(ws_bytes > kDiagHeader + 2 * 4096 + 1024 && rows >= 128, NNCONV_ERR_WORKSPACE,
              "diag_build: workspace too small (use nnconv_diag_sizes)");
  char* hbuf = static_cast<char*>(ws) + kDiagHeader;
  char* efws = hbuf + round_up64(static_cast<int64_t>(rows * hrow), 1024);
  const size_t ef_bytes = ws_bytes - static_cast<size_t>(efws - static_cast<char*>(ws));
  for (int64_t e0 = 0; e0 < P->E; e0 += rows) {
    const int n = static_cast<int>(P->E - e0 < rows ? P->E - e0 : rows);
    const int64_t hpad = round_up64(n, 128);
    int s = edge_features_rows(P, W, edge_attr, e0, n, hbuf, efws, ef_bytes, overflow, st, launches, nullptr);
    if (s) return s;
    float* drows = d + e0 * W->cout;
    if (diag_tc_build(W)) {
      // wgmma with the fp32 epilogue: d = h W_L^T + b_L, A = the chunk-major h of the chunk
      s = launch_gemm_tc(W->prec, hbuf, n, 0, n, W->Kp, W->W3n, W->cout, W->B3, 0, drows, W->cout, st, nullptr, 0, 0, 0,
                         nullptr, nullptr, 0, 1, hpad);
      if (s) return s;
    } else {
      const dim3 grid(ceil_div(n, 64), ceil_div(W->cout, 64));
      const float* WL = static_cast<const float*>(W->W3n);
      if (W->split) k_diag_build<1><<<grid, 256, 0, st>>>(hbuf, n, hpad, W->Kp, WL, W->B3, W->cout, drows);
      else k_diag_build<0><<<grid, 256, 0, st>>>(hbuf, n, 0, W->Kp, WL, W->B3, W->cout, drows);
      NNC_CHECK_LAUNCH();
    }
    if (launches) ++*launches;
  }
  return NNCONV_OK;
}

int apply_diag(const Plan* P, const Weights* W, const float* d, const float* x, const float* root, const float* bias,
               int aggr, float* out, int* argmax, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches) {
  NNC_REQUIRE(W->diag, NNCONV_ERR_ARG, "apply_diag: weights not prepared as a diagonal kernel");
  NNC_REQUIRE(aggr >= 0 && aggr <= 2, NNCONV_ERR_ARG, "apply_diag: unknown aggr %d", aggr);
  if (int sb = check_bipartite_root(P, root, 0)) return sb;
  const int cout = W->cout;
  unsigned long long* keys = nullptr;
  if (aggr == 2) {
    NNC_REQUIRE(argmax != nullptr && ws != nullptr && ws_bytes >= max_keys_bytes(P->N_dst, cout), NNCONV_ERR_WORKSPACE,
                "apply_diag: aggr max needs argmax and a workspace of nnconv_apply_diag_sizes bytes");
    keys = static_cast<unsigned long long*>(ws);
    NNC_CHECK_CUDA(cudaMemsetAsync(keys, 0, sizeof(unsigned long long) * P->N_dst * cout, st));
  }
  int s = launch_out_init(x, root, bias, P->N_dst, cout, cout, out, st, 0);
  if (s) return s;
  int64_t n_l = 1;
  if (P->E > 0 && P->n_tiles > 0) {
    const unsigned grid = static_cast<unsigned>(ceil_div64(static_cast<int64_t>(P->n_tiles) * 32, 256));
    // 16-byte accesses need x, d and out rows 16-byte aligned (a caller's x may start at any float)
    const bool vec = cout % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(d) |
                                        reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const float* inv_deg = P->inv_deg;
#define NNC_DIAG_LAUNCH(A, V)                                                                                          \
  k_apply_diag<A, V><<<grid, 256, 0, st>>>(d, x, cout, P->n_tiles, P->tile_c, P->tile_e0, P->tile_cnt, P->src_nodes,  \
                                           P->dst_sorted, inv_deg, P->perm, out, keys)
    if (vec) {
      if (aggr == 0) NNC_DIAG_LAUNCH(0, true);
      else if (aggr == 1) NNC_DIAG_LAUNCH(1, true);
      else NNC_DIAG_LAUNCH(2, true);
    } else {
      if (aggr == 0) NNC_DIAG_LAUNCH(0, false);
      else if (aggr == 1) NNC_DIAG_LAUNCH(1, false);
      else NNC_DIAG_LAUNCH(2, false);
    }
#undef NNC_DIAG_LAUNCH
    NNC_CHECK_LAUNCH();
    ++n_l;
  }
  if (aggr == 2) {
    s = launch_max_finalize(keys, P->N_dst * cout, out, argmax, st);
    if (s) return s;
    ++n_l;
  }
  if (launches) *launches += n_l;
  return NNCONV_OK;
}

}  // namespace nnc
