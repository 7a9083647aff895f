// Tensor-core backward of the NNConv path (SURVEY 8(a) row a11; what autograd generates for
// graph-neural-operator/nn_conv.py:267-282 + utilities.py:223-227), for the shapes of the GKN / MGKN
// training configurations (out_channels = 64, in_channels <= 64, operand precisions f16, bf16 and f16x2; the split
// variant of each kernel is described next to it).
//
// Notation (DESIGN.md section 2): h_e = edge features (cached by the forward), Y_c = x_c (x) W_L per source,
// G_e = g[dst_e] / max(deg_in(dst_e),1) (mean) or g[dst_e] (add), g = dL/dout.
//
//   per APPLICATION (backward_apply_tc, needs g of that application):
//     dY_c[k,o]  = sum_{e in c} h_e[k] G_e[o]            k_dy:   per-source reduction over edges, MN-major wgmma
//     dx_c       = dY_c : W_L + B_L Gs_c                  k_gemm_tc (K = Kp*out) + scatter
//     dW_L      += x_c (x) dY_c                           k_gemm_tn over sources
//     droot, dbias, dx += g root^T, dB_L                  CUDA cores (N x in x out, negligible)
//   ONCE per (edge_attr, parameters) for all T applications of a shared conv (backward_mlp_tc): h_e does not
//   depend on x, so the gradient w.r.t. h is the SUM over the applications,
//     dh_e[k]    = sum_t sum_o G^t_e[o] Y^t_src(e)[o,k]   k_dh:   one contraction with K = T*out per edge tile,
//   followed by ONE backward pass through the hidden layers (k_gemm_tc with the ReLU-mask epilogue for
//   dz_{l-1} = (dz_l W_l) * [h_{l-1} > 0]; k_gemm_tn for dW_l = dz_l^T h_{l-1} and, against the split-precision
//   first-layer image A1, for db_l and dW_1).  The reference pays that pass T times.
//   On request the same pass also yields the gradient w.r.t. edge_attr, d ea_e = dz_1[e, :] . W_1 (k_ea_grad, one
//   read of dz_1 per batch, rows scattered back to the caller's edge order).
//
// Partially resident h (E_res < E, DESIGN.md section 3): k_dy and k_dh read h through a row window (h_e_base, h_rows);
// source batches past the resident prefix recompute their edges' h (per application) or h_{L-1} (MLP pass) first.
//
// 16-bit range: gradients are normalised by powers of two computed on the device (no host sync): G by the
// largest |G| of the application(s), x by its largest magnitude; the fp32 epilogues multiply the scales back.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "act.cuh"
#include "kernels.h"
#include "tc05.cuh"
#include "tmap.h"

namespace nnc {

int tc_num_sms();

namespace {

using namespace tc05;

constexpr int kMaxApps = 8;     // applications of one shared conv folded into one dh pass

template <int FMT>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if (FMT == 0) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}

// PREC_F16X2: (a, b) as fp16 pairs, hi = fp16(v), lo = fp16(v - hi)
__device__ __forceinline__ void pack2_split(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

struct Maps8 {
  CUtensorMap m[8];
};

// =====================================================================================================
// scales (device scalars, no host round trip)
//   scal[0] = max |G|      scal[1] = gs = pow2 >= scal[0]      scal[2] = 1 / gs
//   scal[3] = max |x|      scal[4] = xs (pow2)                 scal[5] = 1 / xs
//   scal[6] = gs * xs      (multiplier of the dW_L accumulator)
// =====================================================================================================
__device__ __forceinline__ float pow2_ge(float m) {
  if (!(m > 0.f) || !(m <= 3.0e38f)) return 1.f;
  int e;
  const float f = frexpf(m, &e);
  e = f == 0.5f ? e - 1 : e;
  e = e < -100 ? -100 : (e > 100 ? 100 : e);
  return ldexpf(1.f, e);
}

// amax over rows n of |v[n, :]| * w[n]   (w nullable); rows optionally through an index list
__global__ void k_absmax_rows(const float* __restrict__ v, const float* __restrict__ w, const int* __restrict__ idx,
                              int64_t rows, int cols, float* __restrict__ out) {
  float m = 0.f;
  const int64_t total = rows * cols;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols;
    const int c = static_cast<int>(i % cols);
    const int64_t n = idx ? idx[r] : r;
    float a = fabsf(v[n * cols + c]);
    if (w) a *= w[n];
    if (a <= 3.0e38f) m = fmaxf(m, a);
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

__global__ void k_apply_scales(float* scal) {
  scal[1] = pow2_ge(scal[0]);
  scal[2] = 1.f / scal[1];
  scal[4] = pow2_ge(scal[3]);
  scal[5] = 1.f / scal[4];
  scal[6] = scal[1] * scal[4];
}

// mlp pass: s = pow2 >= max_t gmax_t * xsmax_t ; scal[0..T) = gmax_t, scal[8..8+T) = xsmax_t
__global__ void k_mlp_scales(float* scal, int T) {
  float m = 0.f;
  for (int t = 0; t < T; ++t) m = fmaxf(m, scal[t] * scal[8 + t]);
  scal[16] = pow2_ge(m);
  scal[17] = 1.f / scal[16];
}

// =====================================================================================================
// node-level terms
// =====================================================================================================
// out[i, o] += sum_r X[row(r), i] * V[r, o]      row(r) = idx ? idx[r] : r      (droot = x^T g, dB_L = x_src^T Gs)
__global__ void __launch_bounds__(256) k_xtv(const float* __restrict__ X, const int* __restrict__ idx,
                                             const float* __restrict__ V, int64_t R, int cin, int cout,
                                             float* __restrict__ out) {
  extern __shared__ float sm[];
  constexpr int kRows = 32;
  float* sx = sm;                  // [kRows][cin]
  float* sv = sm + kRows * cin;    // [kRows][cout]
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kRows;
  const int nr = static_cast<int>(min(static_cast<int64_t>(kRows), R - r0));
  for (int i = threadIdx.x; i < nr * cin; i += blockDim.x) {
    const int r = i / cin, c = i % cin;
    const int64_t n = idx ? idx[r0 + r] : (r0 + r);
    sx[i] = X[n * cin + c];
  }
  for (int i = threadIdx.x; i < nr * cout; i += blockDim.x) sv[i] = V[(r0 + i / cout) * cout + i % cout];
  __syncthreads();
  for (int p = threadIdx.x; p < cin * cout; p += blockDim.x) {
    const int i = p / cout, o = p % cout;
    float acc = 0.f;
    for (int r = 0; r < nr; ++r) acc = fmaf(sx[r * cin + i], sv[r * cout + o], acc);
    atomicAdd(out + p, acc);
  }
}

// dx[n, i] = sum_o g[n, o] * root[i, o]
__global__ void k_g_rootT(const float* __restrict__ g, const float* __restrict__ root, int64_t N, int cin, int cout,
                          float* __restrict__ dx) {
  extern __shared__ float sroot[];   // [cin][cout + 1]: consecutive threads (i) hit consecutive banks
  const int ld = cout + 1;
  for (int i = threadIdx.x; i < cin * cout; i += blockDim.x) sroot[(i / cout) * ld + i % cout] = root[i];
  __syncthreads();
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (idx >= N * cin) return;
  const int64_t n = idx / cin;
  const int i = static_cast<int>(idx % cin);
  const float* gr = g + n * cout;
  float acc = 0.f;
  for (int o = 0; o < cout; ++o) acc = fmaf(__ldg(gr + o), sroot[i * ld + o], acc);
  dx[idx] = acc;
}

__global__ void k_colsum(const float* __restrict__ g, int64_t N, int C, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  for (int64_t n = blockIdx.y * 8 + threadIdx.y; n < N; n += 8 * gridDim.y)
    if (col < C) s += g[n * C + col];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < C) {
    float t = 0.f;
    for (int r = 0; r < 8; ++r) t += red[r][threadIdx.x];
    atomicAdd(out + col, t);
  }
}

// G16[t*128 + r, o] = (g[dst, o] * inv_deg[dst]) / gs  for r < cnt_t, zero rows up to 128 (cout == 64)
// and, in the same pass, Gs[c, o] += sum of the tile's UNSCALED G rows (Gs zero-initialised by the caller)
// SPLIT (PREC_F16X2, T16 = __half): G16 holds the hi halves, the lo halves follow at row n_tiles*128 (one block per tile)
// MAX (aggr = max, inv_deg = nullptr): g[dst, o] only where argmax[dst, o] is the edge's caller index, else 0
template <typename T16, int SPLIT = 0, bool MAX = false>
__global__ void __launch_bounds__(256) k_gather_g16(const float* __restrict__ g, const int* __restrict__ dst_sorted,
                                                    const float* __restrict__ inv_deg, const int* __restrict__ tile_c,
                                                    const int* __restrict__ tile_e0,
                                                    const int* __restrict__ tile_cnt, const float* __restrict__ scal,
                                                    T16* __restrict__ G16, float* __restrict__ Gs,
                                                    const int* __restrict__ argmax, const int* __restrict__ perm) {
  __shared__ float s_sum[32][65];
  const int t = blockIdx.x;
  const int e0 = tile_e0[t], cnt = tile_cnt[t];
  const float inv_gs = scal[2];
  float colsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  // thread -> (row r = threadIdx / 8 + 32 * pass, 8 columns)
  for (int pass = 0; pass < 4; ++pass) {
    const int r = pass * 32 + threadIdx.x / 8, c0 = (threadIdx.x % 8) * 8;
    uint32_t w[4] = {0u, 0u, 0u, 0u}, wl[4] = {0u, 0u, 0u, 0u};
    if (r < cnt) {
      const int d = dst_sorted[e0 + r];
      const float dsc = inv_deg ? inv_deg[d] : 1.f;
      const float sc = dsc * inv_gs;
      float4 a = *reinterpret_cast<const float4*>(g + static_cast<int64_t>(d) * 64 + c0);
      float4 b = *reinterpret_cast<const float4*>(g + static_cast<int64_t>(d) * 64 + c0 + 4);
      if constexpr (MAX) {
        const int ce = static_cast<int>(caller_edge(perm, e0 + r));
        const int4 ma = *reinterpret_cast<const int4*>(argmax + static_cast<int64_t>(d) * 64 + c0);
        const int4 mb = *reinterpret_cast<const int4*>(argmax + static_cast<int64_t>(d) * 64 + c0 + 4);
        a = make_float4(ma.x == ce ? a.x : 0.f, ma.y == ce ? a.y : 0.f, ma.z == ce ? a.z : 0.f, ma.w == ce ? a.w : 0.f);
        b = make_float4(mb.x == ce ? b.x : 0.f, mb.y == ce ? b.y : 0.f, mb.z == ce ? b.z : 0.f, mb.w == ce ? b.w : 0.f);
      }
      colsum[0] += a.x * dsc; colsum[1] += a.y * dsc; colsum[2] += a.z * dsc; colsum[3] += a.w * dsc;
      colsum[4] += b.x * dsc; colsum[5] += b.y * dsc; colsum[6] += b.z * dsc; colsum[7] += b.w * dsc;
      if (SPLIT) {
        pack2_split(a.x * sc, a.y * sc, w[0], wl[0]); pack2_split(a.z * sc, a.w * sc, w[1], wl[1]);
        pack2_split(b.x * sc, b.y * sc, w[2], wl[2]); pack2_split(b.z * sc, b.w * sc, w[3], wl[3]);
      } else if (std::is_same<T16, __half>::value) {
        w[0] = pack2<0>(a.x * sc, a.y * sc); w[1] = pack2<0>(a.z * sc, a.w * sc);
        w[2] = pack2<0>(b.x * sc, b.y * sc); w[3] = pack2<0>(b.z * sc, b.w * sc);
      } else {
        w[0] = pack2<1>(a.x * sc, a.y * sc); w[1] = pack2<1>(a.z * sc, a.w * sc);
        w[2] = pack2<1>(b.x * sc, b.y * sc); w[3] = pack2<1>(b.z * sc, b.w * sc);
      }
    }
    *reinterpret_cast<uint4*>(G16 + (static_cast<int64_t>(t) * 128 + r) * 64 + c0) = make_uint4(w[0], w[1], w[2], w[3]);
    if (SPLIT)
      *reinterpret_cast<uint4*>(G16 + (static_cast<int64_t>(gridDim.x + t) * 128 + r) * 64 + c0) =
          make_uint4(wl[0], wl[1], wl[2], wl[3]);
  }
  // thread (rr = threadIdx / 8, cg = threadIdx % 8) holds the sums of rows rr, rr+32, rr+64, rr+96 for 8 columns
  {
    const int rr = threadIdx.x / 8, c0 = (threadIdx.x % 8) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) s_sum[rr][c0 + j] = colsum[j];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr) s += s_sum[rr][threadIdx.x];
    atomicAdd(Gs + static_cast<int64_t>(tile_c[t]) * 64 + threadIdx.x, s);
  }
}

// Xg16[c, i] = x[src_c, i] / xs   (global power-of-two scale, zero padded to cin_p)
// SPLIT (PREC_F16X2, T16 = __half): rows of 2 * cin_p, [hi | lo]
template <typename T16, int SPLIT = 0>
__global__ void k_prep_xg(const float* __restrict__ x, const int* __restrict__ src_nodes, int S, int cin, int cin_p,
                          const float* __restrict__ scal, T16* __restrict__ Xg) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(S) * cin_p) return;
  const int c = static_cast<int>(i / cin_p), ii = static_cast<int>(i % cin_p);
  const float v = ii < cin ? x[static_cast<int64_t>(src_nodes[c]) * cin + ii] * scal[5] : 0.f;
  if (SPLIT) {
    const __half hi = __float2half_rn(v);
    __half* row = reinterpret_cast<__half*>(Xg) + static_cast<int64_t>(c) * 2 * cin_p;
    row[ii] = hi;
    row[cin_p + ii] = __float2half_rn(v - __half2float(hi));
  } else if (std::is_same<T16, __half>::value) reinterpret_cast<__half*>(Xg)[i] = __float2half_rn(v);
  else reinterpret_cast<__nv_bfloat16*>(Xg)[i] = __float2bfloat16_rn(v);
}

// dx[src_{c0+c}, i] += gs * winv * dxp[c, i] + sum_o B3[i, o] * Gs[c0+c, o]
// (winv: the inverse power of two of a pre-scaled split W3t image, nullptr = 1)
__global__ void k_scatter_dx_tc(const float* __restrict__ dxp, int ld, const float* __restrict__ Gs,
                                const float* __restrict__ B3, const int* __restrict__ src_nodes, int c0, int nb,
                                int cin, int cout, const float* __restrict__ scal, const float* __restrict__ winv,
                                float* __restrict__ dx) {
  extern __shared__ float sb3[];     // [cin][cout + 1]
  const int ldb = cout + 1;
  for (int t = threadIdx.x; t < cin * cout; t += blockDim.x) sb3[(t / cout) * ldb + t % cout] = B3[t];
  __syncthreads();
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(nb) * cin) return;
  const int c = static_cast<int>(i / cin), ii = static_cast<int>(i % cin);
  float acc = dxp[static_cast<int64_t>(c) * ld + ii] * (winv ? scal[1] * winv[0] : scal[1]);
  const float* gs = Gs + static_cast<int64_t>(c0 + c) * cout;
  for (int o = 0; o < cout; ++o) acc = fmaf(sb3[ii * ldb + o], __ldg(gs + o), acc);
  dx[static_cast<int64_t>(src_nodes[c0 + c]) * cin + ii] += acc;
}

// dW_L[(i*cout + o), k] = mult * acc[(k*cout + o), i]        acc: [Kp*cout, cin_p]
__global__ void k_unpermute_w3q(const float* __restrict__ acc, int cin, int cout, int K, int cin_p,
                                const float* __restrict__ scal, int scal_idx, float* __restrict__ dWL) {
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<int64_t>(cin) * cout * K) return;
  const int k = static_cast<int>(idx % K);
  const int64_t io = idx / K;
  const int o = static_cast<int>(io % cout), i = static_cast<int>(io / cout);
  dWL[idx] = acc[(static_cast<int64_t>(k) * cout + o) * cin_p + i] * scal[scal_idx];
}

// dst[r, c] (R x C) = mult * src[r * ld + c0 + c]
__global__ void k_scale_unpad(const float* __restrict__ src, int64_t ld, int c0, const float* __restrict__ scal,
                              int scal_idx, float* __restrict__ dst, int R, int C) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(R) * C) return;
  const int r = static_cast<int>(i / C), c = static_cast<int>(i % C);
  dst[i] = src[static_cast<int64_t>(r) * ld + c0 + c] * scal[scal_idx];
}

// first layer from D1 = dz_1^T A1 ([kp1, 64]; A1 = [hi(ea) | lo(ea) | hi(ea) | 1 | 1]):
//   dW_1[j, i] = s * (D1[j, i] + D1[j, k_in + i]),   db_1[j] = s * D1[j, 3 k_in]
__global__ void k_fold_w1(const float* __restrict__ D1, int k1, int k_in, const float* __restrict__ scal, int scal_idx,
                          float* __restrict__ dW1, float* __restrict__ db1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k1 * (k_in + 1)) return;
  const int j = i / (k_in + 1), c = i % (k_in + 1);
  const float s = scal[scal_idx];
  if (c < k_in) dW1[j * k_in + c] = s * (D1[j * 64 + c] + D1[j * 64 + k_in + c]);
  else db1[j] = s * D1[j * 64 + 3 * k_in];
}

// Ghat[e - e_base, t*64 + o] = g_t[dst_e, o] * inv_deg[dst_e] * xs_t[src(e)] / s      (one block per tile)
struct GatherGArgs {
  const float* g[kMaxApps];
  const float* xs[kMaxApps];    // [S] per-source power-of-two scale of the forward's Y operand
  int T;
};
// aggr = max: the argmax [N, 64] of every application's forward and the plan's perm (nullable)
struct GatherMaxArgs {
  const int* argmax[kMaxApps];
  const int* perm;
};
// SPLIT (PREC_F16X2, T16 = __half): rows of 2 * T * 64, the hi halves in columns [0, T*64), the lo halves after them
// MAX (aggr = max, inv_deg = nullptr): application a's g[dst, o] only where its argmax[dst, o] is the edge's caller index
template <typename T16, int SPLIT = 0, bool MAX = false>
__global__ void __launch_bounds__(256) k_gather_ghat(GatherGArgs ga, const int* __restrict__ dst_sorted,
                                                     const float* __restrict__ inv_deg, const int* __restrict__ tile_c,
                                                     const int* __restrict__ tile_e0, const int* __restrict__ tile_cnt,
                                                     int tile0, int e_base, const float* __restrict__ scal,
                                                     T16* __restrict__ Gh, GatherMaxArgs gm) {
  const int t = tile0 + blockIdx.x;
  const int e0 = tile_e0[t], cnt = tile_cnt[t], c = tile_c[t];
  const float inv_s = scal[17];
  const int ld = (SPLIT ? 2 : 1) * ga.T * 64;
  for (int a = 0; a < ga.T; ++a) {
    const float xsc = ga.xs[a][c] * inv_s;
    const float* g = ga.g[a];
    for (int pass = 0; pass < 4; ++pass) {
      const int r = pass * 32 + threadIdx.x / 8, c0 = (threadIdx.x % 8) * 8;
      if (r >= cnt) continue;
      const int d = dst_sorted[e0 + r];
      const float sc = (inv_deg ? inv_deg[d] : 1.f) * xsc;
      float4 p = *reinterpret_cast<const float4*>(g + static_cast<int64_t>(d) * 64 + c0);
      float4 q = *reinterpret_cast<const float4*>(g + static_cast<int64_t>(d) * 64 + c0 + 4);
      if constexpr (MAX) {
        const int ce = static_cast<int>(caller_edge(gm.perm, e0 + r));
        const int* am = gm.argmax[a] + static_cast<int64_t>(d) * 64 + c0;
        const int4 mp = *reinterpret_cast<const int4*>(am);
        const int4 mq = *reinterpret_cast<const int4*>(am + 4);
        p = make_float4(mp.x == ce ? p.x : 0.f, mp.y == ce ? p.y : 0.f, mp.z == ce ? p.z : 0.f, mp.w == ce ? p.w : 0.f);
        q = make_float4(mq.x == ce ? q.x : 0.f, mq.y == ce ? q.y : 0.f, mq.z == ce ? q.z : 0.f, mq.w == ce ? q.w : 0.f);
      }
      uint32_t w[4], wl[4];
      if (SPLIT) {
        pack2_split(p.x * sc, p.y * sc, w[0], wl[0]); pack2_split(p.z * sc, p.w * sc, w[1], wl[1]);
        pack2_split(q.x * sc, q.y * sc, w[2], wl[2]); pack2_split(q.z * sc, q.w * sc, w[3], wl[3]);
      } else if (std::is_same<T16, __half>::value) {
        w[0] = pack2<0>(p.x * sc, p.y * sc); w[1] = pack2<0>(p.z * sc, p.w * sc);
        w[2] = pack2<0>(q.x * sc, q.y * sc); w[3] = pack2<0>(q.z * sc, q.w * sc);
      } else {
        w[0] = pack2<1>(p.x * sc, p.y * sc); w[1] = pack2<1>(p.z * sc, p.w * sc);
        w[2] = pack2<1>(q.x * sc, q.y * sc); w[3] = pack2<1>(q.z * sc, q.w * sc);
      }
      T16* row = Gh + static_cast<int64_t>(e0 - e_base + r) * ld + a * 64 + c0;
      *reinterpret_cast<uint4*>(row) = make_uint4(w[0], w[1], w[2], w[3]);
      if (SPLIT) *reinterpret_cast<uint4*>(row + ga.T * 64) = make_uint4(wl[0], wl[1], wl[2], wl[3]);
    }
  }
}

__global__ void k_max_f(const float* __restrict__ v, int n, float* __restrict__ out) {
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(v[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(reinterpret_cast<unsigned int*>(out), __float_as_uint(m));
}

// =====================================================================================================
// k_dy: dY_c^T[k, o] = sum_{e in c} h_e[k] G_e[o] for the sources [c0, c1)   (out = 64)
//   wgmma M = 128 k's (two 64-column chunk panels of h, MN-major A), N = 64 (G tile, MN-major B), K = edges.
//   One (source, 128-k block) at a time per CTA, its [128 x 64] accumulator in the registers of the warpgroup; a
//   stage holds the k block's two h boxes and the G box of one tile of the source.
//   roles: warps 0..3 consumer warpgroup (wgmma, then 16-bit -> dY[c, k*64 + o]) | warp 4 TMA producer
// SPLIT (PREC_F16X2): h and G are fp16 pairs (the lo panels of h start at panel nk, the lo rows of G at g_lo_row);
//   every tile is three stages of the same shape, (h_hi, G_hi), (h_hi, G_lo), (h_lo, G_hi), accumulated into one
//   fp32 tile, i.e. the reduction over edges runs three times as long; dY rows are [hi | lo] pairs (2 * Kp * 64).
// =====================================================================================================
constexpr int kDyStage = 48 * 1024;    // two [<=128 rows x 128 B] h boxes + one G box
constexpr int kDyStages = 4;
constexpr int kDySmem = kDyStages * kDyStage + 4 * acc_scratch_bytes<32>() + 1024;

struct DyArgs {
  const int* tile_ptr;
  const int* tile_e0;
  const int* tile_cnt;
  int c0, c1;
  int h_e_base, h_rows;     // h holds the sorted edges [h_e_base, ...) in chunk panels of h_rows rows
  int nk;                   // nk = Kp / 64 chunk panels
  int num_mt;               // ceil(nk / 2)
  int Kp;
  int g_lo_row;             // SPLIT: first row of the lo halves of G (n_tiles * 128)
  uint16_t* dY;             // [c1 - c0, Kp * 64]   (SPLIT: [c1 - c0, 2 * Kp * 64])
};

template <int FMT, int SPLIT = 0>
__global__ void __launch_bounds__(160, 1)
k_dy(const __grid_constant__ Maps8 tmH, const __grid_constant__ Maps8 tmG, DyArgs a) {
  constexpr int kTerms = SPLIT ? 3 : 1;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  float* scratch = reinterpret_cast<float*>(smem + kDyStages * kDyStage);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kDyStages * kDyStage + 4 * acc_scratch_bytes<32>());
  uint64_t* full = bars;
  uint64_t* empty = full + kDyStages;
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x / 32), 0), lane = threadIdx.x % 32;

  if (warp == 4 && lane == 0) {
    for (int i = 0; i < 8; ++i) { prefetch_tmap(&tmH.m[i]); prefetch_tmap(&tmG.m[i]); }
    for (int s = 0; s < kDyStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    int stage = 0;
    uint32_t phase = 0;
    for (int c = a.c0 + blockIdx.x; c < a.c1; c += gridDim.x) {
      const int t0 = __ldg(a.tile_ptr + c), t1 = __ldg(a.tile_ptr + c + 1);
      for (int m = 0; m < a.num_mt; ++m) {
        const bool two = 2 * m + 1 < a.nk;
        for (int t = t0; t < t1; ++t) {
          const int e0 = __ldg(a.tile_e0 + t);
          const int box = (__ldg(a.tile_cnt + t) + 15) >> 4;       // 16-row units, 1..8
          const uint32_t box_bytes = static_cast<uint32_t>(box) * 16u * 128u;
          for (int term = 0; term < kTerms; ++term) {
            const int hp = 2 * m + (term == 2 ? a.nk : 0);           // h panel (hi, or lo for the lo*hi term)
            const int gr = t * 128 + (term == 1 ? a.g_lo_row : 0);   // G rows (hi, or lo for the hi*lo term)
            // the h_hi boxes of the second term were loaded by the first: keep them for it (evict-first otherwise)
            const uint64_t hpol = (SPLIT && term == 0) ? kEvictNormal : kEvictFirst;
            mbar_wait(&empty[stage], phase ^ 1u);
            if (elect_one()) {
              uint8_t* st = smem + stage * kDyStage;
              mbar_arrive_expect_tx(&full[stage], (two ? 3u : 2u) * box_bytes);
              const int hr = e0 - a.h_e_base;
              tma_load_2d(st, &tmH.m[box - 1], &full[stage], 0, hp * a.h_rows + hr, hpol);
              if (two) tma_load_2d(st + 16384, &tmH.m[box - 1], &full[stage], 0, (hp + 1) * a.h_rows + hr, hpol);
              tma_load_2d(st + 32768, &tmG.m[box - 1], &full[stage], 0, gr, kEvictFirst);
            }
            __syncwarp();
            if (++stage == kDyStages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else {
    const int quarter = warp;
    float* wb = scratch + warp * (acc_scratch_bytes<32>() / 4);
    Acc<64> acc;
    int stage = 0;
    uint32_t phase = 0;
    for (int c = a.c0 + blockIdx.x; c < a.c1; c += gridDim.x) {
      const int t0 = __ldg(a.tile_ptr + c), t1 = __ldg(a.tile_ptr + c + 1);
      uint16_t* yrow = a.dY + static_cast<int64_t>(c - a.c0) * (SPLIT ? 2 : 1) * a.Kp * 64;
      for (int m = 0; m < a.num_mt; ++m) {
        for (int t = t0; t < t1; ++t) {
          const int ksteps = (__ldg(a.tile_cnt + t) + 15) >> 4;
          for (int term = 0; term < kTerms; ++term) {
            mbar_wait(&full[stage], phase);
            const uint32_t st = smem_u32(smem + stage * kDyStage);
            // second m64 half = the second h box (+16 KB); 16 edges = two 8-row groups of 1024 B (+128 units)
            mma_block<64, FMT, 1, 1>(acc, smem_desc_mn_sw128(st, 16384), smem_desc_mn_sw128(st + 32768, 16384),
                                     16384 >> 4, 128, ksteps, t != t0 || term != 0);
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == kDyStages) { stage = 0; phase ^= 1u; }
          }
        }
        const int k = m * 128 + acc_row(quarter, lane);
#pragma unroll
        for (int cc = 0; cc < 64; cc += 32) {
          uint32_t v[32];
          acc_rows<64, 32>(acc, cc, wb, v);
          if (k < a.Kp) {
            uint32_t pk[16], pl[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              if (SPLIT) pack2_split(__uint_as_float(v[2 * j]), __uint_as_float(v[2 * j + 1]), pk[j], pl[j]);
              else pk[j] = pack2<FMT>(__uint_as_float(v[2 * j]), __uint_as_float(v[2 * j + 1]));
            }
            uint16_t* dst = yrow + static_cast<int64_t>(k) * 64 + cc;
            st_global_32b(dst, pk);
            st_global_32b(dst + 16, pk + 8);
            if (SPLIT) {
              st_global_32b(dst + static_cast<int64_t>(a.Kp) * 64, pl);
              st_global_32b(dst + static_cast<int64_t>(a.Kp) * 64 + 16, pl + 8);
            }
          }
        }
      }
    }
  }
}

// =====================================================================================================
// k_dh: dz[e, k] = [h_e[k] > 0] * sum_{t<T} sum_o Ghat[e, t*64 + o] * Yt[(t, c(e), k), o]     for the tiles of a batch
//   wgmma M = 128 edges (A = Ghat tile, K-major, resident for the tile: T chunks of 64),
//         N = BN k's  (B = rows (t, c, k) of the per-application Y^T matrices, K-major [BN x 64] boxes),
//         K = T * 64; the accumulator lives in the registers of the consumer warpgroup (warps 0..3, warp 4 = TMA
//   producer), which runs the epilogue: ReLU mask from the chunk-major h -> 16-bit -> dz[e - e_base, k].
// SPLIT (PREC_F16X2): Ghat and Y^T are fp16 pairs.  Resident pairs would need 32 KB per application (256 KB at
//   kMaxApps), more than shared memory holds beside the B ring, so A is streamed with B instead: a stage holds the
//   (hi, lo) Ghat chunks of application j and the (hi, lo) Y^T boxes of (j, k block) -- 2 x 16 KB + 2 x BN x 128 B --
//   and runs the three MMA blocks hi*hi, hi*lo, lo*hi.  The Ghat chunks are re-read once per k block (L2 hits: a tile's
//   2 x T x 16 KB stay hot while its k blocks run).  dz rows are [hi | lo] pairs (2 * Kp); the mask is h's hi half.
// =====================================================================================================
constexpr int kDhAChunk = 16 * 1024;
constexpr int kDhBStages = 3;

struct DhArgs {
  const int* tile_c;
  const int* tile_e0;
  const int* tile_cnt;
  int tile0, tile1;
  int c0, Sb;               // batch of sources [c0, c0 + Sb)
  int e_base;               // first sorted edge of the batch
  int h_e_base, h_rows;     // h holds the sorted edges [h_e_base, ...) in chunk panels of h_rows rows
  int T, Kp, n_nb;          // n_nb = Kp / BN
  const uint16_t* h;        // chunk-major edge features (the ReLU mask)
  uint16_t* dz;             // [batch edges, Kp] row-major (SPLIT: [batch edges, 2 * Kp], [hi | lo])
  // optional fused bias gradient: colsum[k * colsum_stride] += sum over the batch's edges of dz[e, k] (fp32, unscaled by
  // the caller's power-of-two factor like dz itself).  Column sums are formed per warp piece through a [32][33] shared
  // transpose and accumulated in a per-warp shared array; needs 4 * (4224 + 4 * Kp) extra bytes of shared memory.
  float* colsum;
  int colsum_stride;
  float act_q0, act_q1, act_q2;   // v[0 .. 2] of MODE's activation parameter block (ActParams), all act_grad reads
};

constexpr int kDhScratch = 4 * acc_scratch_bytes<32>();

// bytes of the operand stages of k_dh (everything before its barriers)
__host__ __device__ constexpr int dh_pipe_bytes(int split, int BN, int T) {
  return split ? kDhBStages * (2 * kDhAChunk + 2 * BN * 128) : T * kDhAChunk + kDhBStages * BN * 128;
}

// MODE = SPLIT | ACT << 1: ACT is the hidden activation (act.cuh).  ReLU (ACT 0) masks with h > 0 as above; another
// activation multiplies by act_grad<ACT>(h) (SPLIT: of h's hi + lo halves), so the ReLU kernels keep their names.
template <int FMT, int BN, int MODE = 0>
__global__ void __launch_bounds__(160, 1)
k_dh(const __grid_constant__ Maps8 tmA, const __grid_constant__ CUtensorMap tmB, DhArgs a) {
  constexpr int SPLIT = MODE & 1, kAct = MODE >> 1;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const int b_stage_bytes = BN * 128;
  constexpr int kSplitStage = 2 * kDhAChunk + 2 * BN * 128;  // SPLIT: [A hi | A lo | B hi | B lo]
  uint8_t* smem_a = smem;                                   // [kMaxApps? T] chunks of 16 KB
  uint8_t* smem_b = SPLIT ? smem : smem + a.T * kDhAChunk;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + dh_pipe_bytes(SPLIT, BN, a.T));
  uint64_t* a_full = bars;                   // [kMaxApps]
  uint64_t* a_empty = a_full + kMaxApps;
  uint64_t* b_full = a_empty + kMaxApps;
  uint64_t* b_empty = b_full + kDhBStages;
  float* scratch = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 1024);  // [4] accumulator transposes
  float* s_tr = scratch + kDhScratch / 4;                                               // [4][32][33]  (colsum only)
  float* s_cs = s_tr + 4 * 32 * 33;                                                     // [4][Kp]
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x / 32), 0), lane = threadIdx.x % 32;

  if (warp == 4 && lane == 0) {
    for (int i = 0; i < 8; ++i) prefetch_tmap(&tmA.m[i]);
    prefetch_tmap(&tmB);
    for (int s = 0; s < kMaxApps; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4); }
    for (int s = 0; s < kDhBStages; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4 && SPLIT) {
    int bs = 0;
    uint32_t bph = 0;
    for (int t = a.tile0 + blockIdx.x; t < a.tile1; t += gridDim.x) {
      const int e0 = __ldg(a.tile_e0 + t);
      const int box = (__ldg(a.tile_cnt + t) + 15) >> 4;
      const int cl = __ldg(a.tile_c + t) - a.c0;
      const uint32_t a_bytes = static_cast<uint32_t>(box) * 16u * 128u;
      for (int nb = 0; nb < a.n_nb; ++nb) {
        for (int j = 0; j < a.T; ++j) {
          mbar_wait(&b_empty[bs], bph ^ 1u);
          if (elect_one()) {
            uint8_t* sp = smem + bs * kSplitStage;
            const int yrow = (j * a.Sb + cl) * 2 * a.Kp + nb * BN;      // Y^T rows of (j, c): [hi Kp | lo Kp]
            mbar_arrive_expect_tx(&b_full[bs], 2u * a_bytes + 2u * static_cast<uint32_t>(b_stage_bytes));
            tma_load_2d(sp, &tmA.m[box - 1], &b_full[bs], j * 64, e0 - a.e_base, kEvictNormal);
            tma_load_2d(sp + kDhAChunk, &tmA.m[box - 1], &b_full[bs], (a.T + j) * 64, e0 - a.e_base, kEvictNormal);
            tma_load_2d(sp + 2 * kDhAChunk, &tmB, &b_full[bs], 0, yrow, kEvictLast);
            tma_load_2d(sp + 2 * kDhAChunk + b_stage_bytes, &tmB, &b_full[bs], 0, yrow + a.Kp, kEvictLast);
          }
          __syncwarp();
          if (++bs == kDhBStages) { bs = 0; bph ^= 1u; }
        }
      }
    }
  } else if (warp == 4) {
    int bs = 0;
    uint32_t bph = 0, aph = 0;
    for (int t = a.tile0 + blockIdx.x; t < a.tile1; t += gridDim.x, aph ^= 1u) {
      const int e0 = __ldg(a.tile_e0 + t);
      const int box = (__ldg(a.tile_cnt + t) + 15) >> 4;
      const int cl = __ldg(a.tile_c + t) - a.c0;
      for (int j = 0; j < a.T; ++j) {                       // the tile's Ghat chunks (resident until its last k block)
        mbar_wait(&a_empty[j], aph ^ 1u);
        if (elect_one()) {
          mbar_arrive_expect_tx(&a_full[j], static_cast<uint32_t>(box) * 16u * 128u);
          tma_load_2d(smem_a + j * kDhAChunk, &tmA.m[box - 1], &a_full[j], j * 64, e0 - a.e_base, kEvictFirst);
        }
        __syncwarp();
      }
      for (int nb = 0; nb < a.n_nb; ++nb) {
        for (int j = 0; j < a.T; ++j) {
          mbar_wait(&b_empty[bs], bph ^ 1u);
          if (elect_one()) {
            mbar_arrive_expect_tx(&b_full[bs], static_cast<uint32_t>(b_stage_bytes));
            tma_load_2d(smem_b + bs * b_stage_bytes, &tmB, &b_full[bs], 0, (j * a.Sb + cl) * a.Kp + nb * BN, kEvictLast);
          }
          __syncwarp();
          if (++bs == kDhBStages) { bs = 0; bph ^= 1u; }
        }
      }
    }
  } else {
    const int quarter = warp % 4;
    float* my_tr = s_tr + quarter * 32 * 33;
    float* my_cs = s_cs + quarter * a.Kp;
    if (a.colsum != nullptr)
      for (int k = lane; k < a.Kp; k += 32) my_cs[k] = 0.f;
    __syncwarp();
    float* wb = scratch + quarter * (acc_scratch_bytes<32>() / 4);
    Acc<BN> acc;
    int bs = 0;
    uint32_t bph = 0, aph = 0;
    for (int t = a.tile0 + blockIdx.x; t < a.tile1; t += gridDim.x, aph ^= 1u) {
      const int e0 = __ldg(a.tile_e0 + t), cnt = __ldg(a.tile_cnt + t);
      const int r = acc_row(quarter, lane);
      const bool ok = r < cnt;
      for (int nb = 0; nb < a.n_nb; ++nb) {
        for (int j = 0; j < a.T; ++j) {
          if (SPLIT) {
            mbar_wait(&b_full[bs], bph);
            const uint32_t sp = smem_u32(smem + bs * kSplitStage);
            const uint64_t ah = smem_desc_sw128(sp), al = smem_desc_sw128(sp + kDhAChunk);
            const uint64_t bh = smem_desc_sw128(sp + 2 * kDhAChunk), bl = smem_desc_sw128(sp + 2 * kDhAChunk + b_stage_bytes);
            mma_block<BN, FMT>(acc, ah, bh, 512, 2, 4, j != 0);
            mma_block<BN, FMT>(acc, ah, bl, 512, 2, 4, true);
            mma_block<BN, FMT>(acc, al, bh, 512, 2, 4, true);
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&b_empty[bs]);
          } else {
            if (nb == 0) mbar_wait(&a_full[j], aph);
            mbar_wait(&b_full[bs], bph);
            mma_block<BN, FMT>(acc, smem_desc_sw128(smem_u32(smem_a + j * kDhAChunk)),
                               smem_desc_sw128(smem_u32(smem_b + bs * b_stage_bytes)), 512, 2, 4, j != 0);
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) {
              mbar_arrive(&b_empty[bs]);
              if (nb == a.n_nb - 1) mbar_arrive(&a_empty[j]);
            }
          }
          if (++bs == kDhBStages) { bs = 0; bph ^= 1u; }
        }
#pragma unroll
        for (int cc = 0; cc < BN; cc += 32) {
          uint32_t v[32];
          acc_rows<BN, 32>(acc, cc, wb, v);
          const int k0 = nb * BN + cc;
          if (ok) {
            // (SPLIT: the hi panels of h come first, so this is the hi half)
            const uint16_t* hp = a.h + (static_cast<int64_t>(k0 >> 6) * a.h_rows + (e0 - a.h_e_base) + r) * 64 + (k0 & 63);
            uint32_t pk[16], pl[16];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const uint4 mk = __ldg(reinterpret_cast<const uint4*>(hp) + q);
              const uint32_t mw[4] = {mk.x, mk.y, mk.z, mk.w};
              uint32_t lw[4] = {0u, 0u, 0u, 0u};
              if (SPLIT && kAct != ACT_RELU) {   // the lo panels follow the Kp / 64 hi panels
                const uint4 ml = __ldg(reinterpret_cast<const uint4*>(hp + static_cast<int64_t>(a.Kp) * a.h_rows) + q);
                lw[0] = ml.x; lw[1] = ml.y; lw[2] = ml.z; lw[3] = ml.w;
              }
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float f0, f1;
                if (kAct == ACT_RELU) {
                  f0 = (mw[j] & 0x7FFFu) ? __uint_as_float(v[8 * q + 2 * j]) : 0.f;
                  f1 = (mw[j] & 0x7FFF0000u) ? __uint_as_float(v[8 * q + 2 * j + 1]) : 0.f;
                } else {
                  float2 y = unpack2<FMT>(mw[j]);
                  if (SPLIT) {
                    const float2 yl = unpack2<FMT>(lw[j]);
                    y.x += yl.x;
                    y.y += yl.y;
                  }
                  const ActParams aq{{a.act_q0, a.act_q1, a.act_q2}};
                  f0 = __uint_as_float(v[8 * q + 2 * j]) * act_grad<kAct>(y.x, aq);
                  f1 = __uint_as_float(v[8 * q + 2 * j + 1]) * act_grad<kAct>(y.y, aq);
                }
                if (SPLIT) pack2_split(f0, f1, pk[4 * q + j], pl[4 * q + j]);
                else pk[4 * q + j] = pack2<FMT>(f0, f1);
                v[8 * q + 2 * j] = __float_as_uint(f0);
                v[8 * q + 2 * j + 1] = __float_as_uint(f1);
              }
            }
            uint16_t* dst = a.dz + static_cast<int64_t>(e0 - a.e_base + r) * (SPLIT ? 2 : 1) * a.Kp + k0;
            st_global_32b(dst, pk);
            st_global_32b(dst + 16, pk + 8);
            if (SPLIT) {
              st_global_32b(dst + a.Kp, pl);
              st_global_32b(dst + a.Kp + 16, pl + 8);
            }
          }
          if (a.colsum != nullptr) {          // column sums of this warp's [32 rows x 32 columns] piece
#pragma unroll
            for (int j = 0; j < 32; ++j) my_tr[lane * 33 + j] = ok ? __uint_as_float(v[j]) : 0.f;
            __syncwarp();
            float cs = 0.f;
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) cs += my_tr[rr * 33 + lane];
            my_cs[k0 + lane] += cs;
            __syncwarp();
          }
        }
      }
    }
    if (a.colsum != nullptr) {
      __syncwarp();
      for (int k = lane; k < a.Kp; k += 32) {
        const float v = my_cs[k];
        if (v != 0.f) atomicAdd(a.colsum + static_cast<int64_t>(k) * a.colsum_stride, v);
      }
    }
  }
}

// k_dh with another hidden activation (the ReLU launches below set their attributes once, together)
template <int FMT, int BN, int MODE>
int launch_dh(const Maps8& tmA, const CUtensorMap& tmB, const DhArgs& a, int grid, int smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<FMT, BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  k_dh<FMT, BN, MODE><<<grid, 160, smem, st>>>(tmA, tmB, a);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

// =====================================================================================================
// k_ea_grad: grad_edge_attr[perm[e_base + r], i] = s * sum_j dz_1[r, j] W_1[j, i]   for the rows r < n of a batch
//   (edge_attr enters the op only through the first Linear).  dz_1 is 16-bit [n, kp1] row-major, scaled by 1 / s like
//   every gradient of the pass, and read once; W_1 (fp32 [kp1, k_in], zero rows past k_1) sits transposed in shared
//   memory.  Eight lanes share a row (64 consecutive columns per step, 16-byte loads), each lane carries kEaRows rows,
//   so a warp covers 4 * kEaRows rows and a row's sum needs three shuffles.  Padding rows [n, n_pad) are never read.
//   SPLIT (PREC_F16X2): dz_1 rows are [hi | lo] pairs (2 * kp1), summed in fp32 as they are read.
// =====================================================================================================
constexpr int kEaRows = 2;
constexpr int kEaRowsPerBlock = 8 * 4 * kEaRows;   // 256 threads

template <int FMT>
__device__ __forceinline__ void unpack8(const uint4 u, float* v) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float2 f;
    if (FMT == 0) f = __half22float2(*reinterpret_cast<const __half2*>(&w[k]));
    else f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[k]));
    v[2 * k] = f.x;
    v[2 * k + 1] = f.y;
  }
}

template <int FMT, int KMAX, int SPLIT = 0>
__global__ void __launch_bounds__(256) k_ea_grad(const uint16_t* __restrict__ dz, int n, int kp1,
                                                 const float* __restrict__ W1, int k_in, const int* __restrict__ perm,
                                                 int e_base, const float* __restrict__ scal, int scal_idx,
                                                 float* __restrict__ out) {
  extern __shared__ __align__(16) float sw[];     // [k_in][kp1]: sw[i * kp1 + j] = W1[j, i]
  for (int t = threadIdx.x; t < k_in * kp1; t += blockDim.x) sw[(t % k_in) * kp1 + t / k_in] = W1[t];
  __syncthreads();
  const float s = scal[scal_idx];
  const int lane = threadIdx.x & 31, grp = lane >> 3, q = lane & 7;
  const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t r0 = warp * 4 * kEaRows; r0 < n; r0 += n_warps * 4 * kEaRows) {
    int64_t row[kEaRows];
    float acc[kEaRows][KMAX];
#pragma unroll
    for (int rr = 0; rr < kEaRows; ++rr) {
      row[rr] = r0 + grp * kEaRows + rr;
#pragma unroll
      for (int i = 0; i < KMAX; ++i) acc[rr][i] = 0.f;
    }
    for (int j0 = q * 8; j0 < kp1; j0 += 64) {
      float v[kEaRows][8];
#pragma unroll
      for (int rr = 0; rr < kEaRows; ++rr) {
        uint4 u = make_uint4(0u, 0u, 0u, 0u), ul = make_uint4(0u, 0u, 0u, 0u);
        const uint16_t* zr = dz + row[rr] * (SPLIT ? 2 : 1) * kp1 + j0;
        if (row[rr] < n) {
          u = __ldcs(reinterpret_cast<const uint4*>(zr));
          if (SPLIT) ul = __ldcs(reinterpret_cast<const uint4*>(zr + kp1));
        }
        unpack8<FMT>(u, v[rr]);
        if (SPLIT) {
          float vl[8];
          unpack8<FMT>(ul, vl);
#pragma unroll
          for (int k = 0; k < 8; ++k) v[rr][k] += vl[k];
        }
      }
#pragma unroll
      for (int i = 0; i < KMAX; ++i) {
        if (i >= k_in) break;
        const float4 w0 = *reinterpret_cast<const float4*>(sw + i * kp1 + j0);
        const float4 w1 = *reinterpret_cast<const float4*>(sw + i * kp1 + j0 + 4);
#pragma unroll
        for (int rr = 0; rr < kEaRows; ++rr) {
          float a = acc[rr][i];
          a = fmaf(v[rr][0], w0.x, a); a = fmaf(v[rr][1], w0.y, a); a = fmaf(v[rr][2], w0.z, a);
          a = fmaf(v[rr][3], w0.w, a); a = fmaf(v[rr][4], w1.x, a); a = fmaf(v[rr][5], w1.y, a);
          a = fmaf(v[rr][6], w1.z, a); a = fmaf(v[rr][7], w1.w, a);
          acc[rr][i] = a;
        }
      }
    }
#pragma unroll
    for (int rr = 0; rr < kEaRows; ++rr) {
#pragma unroll
      for (int i = 0; i < KMAX; ++i) {
        if (i >= k_in) break;
        float a = acc[rr][i];
        a += __shfl_xor_sync(0xffffffffu, a, 4);
        a += __shfl_xor_sync(0xffffffffu, a, 2);
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        acc[rr][i] = a;
      }
      if (row[rr] < n) {
        const int64_t e = e_base + row[rr];
        const int64_t dst = perm ? perm[e] : e;
#pragma unroll
        for (int i = 0; i < KMAX; ++i)
          if (i < k_in && (i & 7) == q) out[dst * k_in + i] = acc[rr][i] * s;
      }
    }
  }
}

}  // namespace

// =====================================================================================================
// host side
// =====================================================================================================
bool backward_tc_supported(const Weights* W) {
  if (W->prec != PREC_F16 && W->prec != PREC_BF16 && W->prec != PREC_F16X2) return false;
  if (W->cout != 64 || W->cin > 64 || W->n_layers < 2 || W->W1aug == nullptr) return false;
  if (W->W3q == nullptr || W->W3t == nullptr) return false;
  for (int l = 2; l <= W->n_layers - 1; ++l)
    if (W->WhT[l] == nullptr) return false;
  return true;
}

namespace {

struct ApplyBwdLayout {
  size_t off_scal, off_Xg, off_Gs, off_G16, off_dW3, off_dxp, off_dY, fixed, per_src;
};

ApplyBwdLayout apply_bwd_layout(const Plan* P, const Weights* W) {
  Carver c(nullptr, ~size_t(0));
  ApplyBwdLayout L{};
  const size_t S = P->n_src > 0 ? P->n_src : 1;
  const size_t pm = W->split ? 2 : 1;      // PREC_F16X2: x, G and dY as [hi | lo] pairs
  L.off_scal = c.off; c.take<float>(64);
  L.off_Xg = c.off; c.take<char>((S + 128) * W->cin_p * 2 * pm);
  L.off_Gs = c.off; c.take<float>(S * W->cout);
  L.off_G16 = c.off; c.take<char>(static_cast<size_t>(P->n_tiles > 0 ? P->n_tiles : 1) * 128 * 64 * 2 * pm);
  L.off_dW3 = c.off; c.take<float>(static_cast<size_t>(W->Kp) * W->cout * W->cin_p);
  L.fixed = c.off;
  L.per_src = static_cast<size_t>(W->Kp) * W->cout * 2 * pm + static_cast<size_t>(W->cin_p) * 4;   // dY row + dxp row
  return L;
}

// C[M, N] += sum_{r < R} A[r, m] B[r, n] (see launch_gemm_tn).  PREC_F16X2: A and B are [hi | lo] pairs whose lo halves
// start at columns a_lo / b_lo (b_lo < 0: B is a single operand, e.g. the split first-layer image A1), and the product
// is hi*hi + hi*lo + lo*hi as accumulating fp16 calls (hi*hi + lo*hi when B is single)
int gemm_tn_pairs(const Weights* W, const void* A, int64_t lda, int a_lo, const void* B, int64_t ldb, int b_lo, int64_t R,
                  int M, int N, float* C, int64_t ldc, cudaStream_t st) {
  if (!W->split) return launch_gemm_tn(W->prec, A, lda, 0, B, ldb, 0, R, M, N, C, ldc, 1.f, nullptr, st);
  const int cols[3][2] = {{0, 0}, {a_lo, 0}, {0, b_lo}};
  for (int i = 0; i < (b_lo < 0 ? 2 : 3); ++i) {
    const int s = launch_gemm_tn(PREC_F16, A, lda, cols[i][0], B, ldb, cols[i][1], R, M, N, C, ldc, 1.f, nullptr, st);
    if (s) return s;
  }
  return NNCONV_OK;
}

// ---- streamed edge features (E_res < E): the sources whose edges all lie in the resident prefix [0, E_res) run
// against it; every later source batch first recomputes the h of its edges into a chunk buffer.  Batches are aligned to
// sources, not units: k_dy writes dY_c from registers, so all edges of one source go through one launch.
constexpr int64_t kBwdEfRows = 8192;     // rows of the edge-feature scratch of the chunk recomputation

size_t bwd_ef_bytes(const Plan* P, const Weights* W, int64_t E_res) {
  if (E_res >= P->E) return 0;
  const int64_t rows = std::min<int64_t>(kBwdEfRows, round_up64(P->E, 128));
  return static_cast<size_t>(round_up64(static_cast<int64_t>(rows * ef_row_bytes(W)) + 4096, 1024));
}

// first compact source with an edge at or past E_res (sources [0, c) lie in the resident prefix)
int first_streamed_src(const Plan* P, int64_t E_res) {
  if (E_res >= P->E) return P->n_src;
  const int* g = P->h_group_ptr;
  return static_cast<int>(std::upper_bound(g, g + P->n_src + 1, static_cast<int>(E_res)) - g) - 1;
}

// end of the streamed batch starting at c0: sources while their dxp / dY rows and the chunk-major h of their edges fit
// the pool (c0 = not even one source fits)
int apply_stream_batch_end(const Plan* P, const Weights* W, const ApplyBwdLayout& L, int c0, size_t pool) {
  const int* g = P->h_group_ptr;
  const size_t hrow = h_row_bytes(W);
  int c1 = c0;
  while (c1 < P->n_src) {
    const size_t need = static_cast<size_t>(c1 + 1 - c0 + 128) * L.per_src +
                        static_cast<size_t>(round_up64(g[c1 + 1] - g[c0], 128)) * hrow;
    if (need > pool) break;
    ++c1;
  }
  return c1;
}

}  // namespace

int node_terms_rows(const float* x, const float* root, const float* gout, int64_t N, int cin, int cout, float* dx,
                    float* droot, float* dbias, cudaStream_t st, int64_t* launches) {
  const size_t smem_xtv = sizeof(float) * 32 * (cin + cout), smem_rootT = sizeof(float) * cin * (cout + 1);
  if (smem_xtv > 48 * 1024 || smem_rootT > 48 * 1024)
    return backward_node_terms(x, root, gout, N, cin, cout, dx, droot, dbias, st, launches);
  if (dbias) {
    NNC_CHECK_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float) * cout, st));
    k_colsum<<<dim3(ceil_div(cout, 32), 64), dim3(32, 8), 0, st>>>(gout, N, cout, dbias);
    NNC_CHECK_LAUNCH();
    ++*launches;
  }
  if (root != nullptr) {
    NNC_CHECK_CUDA(cudaMemsetAsync(droot, 0, sizeof(float) * cin * cout, st));
    k_xtv<<<(unsigned)ceil_div64(N, 32), 256, smem_xtv, st>>>(x, nullptr, gout, N, cin, cout, droot);
    NNC_CHECK_LAUNCH();
    k_g_rootT<<<(unsigned)ceil_div64(N * cin, 256), 256, smem_rootT, st>>>(gout, root, N, cin, cout, dx);
    NNC_CHECK_LAUNCH();
    *launches += 2;
  } else if (dx != nullptr) {
    NNC_CHECK_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * N * cin, st));
  }
  return NNCONV_OK;
}

size_t backward_apply_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes, int64_t E_res, size_t chunk_ws_bytes) {
  ApplyBwdLayout L = apply_bwd_layout(P, W);
  const size_t S = P->n_src > 0 ? P->n_src : 1;
  size_t nb = want_bytes > L.fixed ? (want_bytes - L.fixed) / L.per_src : 0;
  if (nb < 128) nb = 128;
  if (nb > S) nb = S;
  const size_t cached = L.fixed + (nb + 128) * L.per_src + 4096;
  if (E_res < 0 || E_res >= P->E) return cached;
  // chunk rows: about chunk_ws_bytes of h, and at least every edge of the largest source (one batch holds whole sources)
  const size_t hrow = h_row_bytes(W);
  const int64_t all_rows = round_up64(P->E, 128);
  int64_t rows = static_cast<int64_t>(chunk_ws_bytes / hrow) / 128 * 128;
  const int64_t deg_rows = round_up64(P->max_out_deg > 0 ? P->max_out_deg : 1, 128);
  if (rows > all_rows) rows = all_rows;
  if (rows < deg_rows) rows = deg_rows;
  return cached + bwd_ef_bytes(P, W, E_res) + static_cast<size_t>(rows) * hrow;
}

int backward_apply_tc(const Plan* P, const Weights* W, const float* edge_attr, const void* h, int64_t E_res,
                      const float* x, const float* root, int aggr_mean, const float* gout, float* dx, float* dWL,
                      float* dbL, float* droot, float* dbias, void* ws, size_t ws_bytes, cudaStream_t st,
                      int64_t* launches, const int* argmax) {
  NNC_REQUIRE(backward_tc_supported(W), NNCONV_ERR_UNSUPPORTED, "tensor-core backward: unsupported shape / precision");
  const int cin = W->cin, cout = W->cout, Kp = W->Kp, cin_p = W->cin_p;
  const int64_t N = P->N_dst;   // rows of gout; dx has N_src rows (square plans: the same)
  const int bf = W->prec == PREC_BF16;
  const int sp = W->split;
  const bool streamed = E_res < P->E;
  NNC_REQUIRE(!streamed || edge_attr != nullptr, NNCONV_ERR_ARG, "backward_apply: streamed edge features need edge_attr");
  auto count = [&](int64_t k) { if (launches) *launches += k; };
  int s = check_bipartite_root(P, root, 0);
  if (s) return s;
  s = tc_init();
  if (s) return s;
  // ---- node-level terms
  if (dbias) {
    NNC_CHECK_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float) * cout, st));
    k_colsum<<<dim3(ceil_div(cout, 32), 64), dim3(32, 8), 0, st>>>(gout, N, cout, dbias);
    NNC_CHECK_LAUNCH();
    count(1);
  }
  if (root != nullptr) {
    NNC_CHECK_CUDA(cudaMemsetAsync(droot, 0, sizeof(float) * cin * cout, st));
    k_xtv<<<(unsigned)ceil_div64(N, 32), 256, sizeof(float) * 32 * (cin + cout), st>>>(x, nullptr, gout, N, cin, cout, droot);
    NNC_CHECK_LAUNCH();
    k_g_rootT<<<(unsigned)ceil_div64(N * cin, 256), 256, sizeof(float) * cin * (cout + 1), st>>>(gout, root, N, cin, cout, dx);
    NNC_CHECK_LAUNCH();
    count(2);
  } else {
    NNC_CHECK_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * P->N_src * cin, st));
  }
  NNC_CHECK_CUDA(cudaMemsetAsync(dbL, 0, sizeof(float) * cin * cout, st));
  const int64_t nWL = static_cast<int64_t>(cin) * cout * W->K;
  if (P->E == 0 || P->n_src == 0) {
    NNC_CHECK_CUDA(cudaMemsetAsync(dWL, 0, sizeof(float) * nWL, st));
    return NNCONV_OK;
  }
  ApplyBwdLayout L = apply_bwd_layout(P, W);
  const size_t ef_bytes = bwd_ef_bytes(P, W, E_res);      // 0 when h is whole
  NNC_REQUIRE(ws != nullptr && ws_bytes >= L.fixed + ef_bytes + 128 * L.per_src, NNCONV_ERR_WORKSPACE,
              "backward_apply: workspace too small");
  char* base = static_cast<char*>(ws);
  float* scal = reinterpret_cast<float*>(base + L.off_scal);
  void* Xg = base + L.off_Xg;
  float* Gs = reinterpret_cast<float*>(base + L.off_Gs);
  void* G16 = base + L.off_G16;
  float* dW3 = reinterpret_cast<float*>(base + L.off_dW3);
  const int S = P->n_src;
  const size_t pool = ws_bytes - L.fixed - ef_bytes - 4096;   // dxp, dY (and the chunk h) of one source batch
  int64_t nb_max = static_cast<int64_t>(pool / L.per_src) - 128;
  if (nb_max > S) nb_max = S;
  NNC_REQUIRE(nb_max >= 1, NNCONV_ERR_WORKSPACE, "backward_apply: workspace too small");
  char* ef_ws = base + L.fixed;
  char* dyn = base + L.fixed + ef_bytes;
  float* dxp = reinterpret_cast<float*>(dyn);
  uint16_t* dY = reinterpret_cast<uint16_t*>(dyn + round_up64(static_cast<int64_t>(nb_max + 128) * cin_p * 4, 1024));
  const float* inv_deg = aggr_mean ? P->inv_deg : nullptr;

  // ---- scales, G tiles, per-source sums, globally scaled x
  NNC_CHECK_CUDA(cudaMemsetAsync(scal, 0, sizeof(float) * 64, st));
  k_absmax_rows<<<592, 256, 0, st>>>(gout, inv_deg, nullptr, N, cout, scal + 0);
  NNC_CHECK_LAUNCH();
  k_absmax_rows<<<592, 256, 0, st>>>(x, nullptr, P->src_nodes, S, cin, scal + 3);
  NNC_CHECK_LAUNCH();
  k_apply_scales<<<1, 1, 0, st>>>(scal);
  NNC_CHECK_LAUNCH();
  NNC_CHECK_CUDA(cudaMemsetAsync(Gs, 0, sizeof(float) * static_cast<size_t>(S) * cout, st));
  {
    auto gather = [&](auto t16, auto split, auto mx) {
      using T16 = decltype(t16);
      k_gather_g16<T16, decltype(split)::value, decltype(mx)::value><<<P->n_tiles, 256, 0, st>>>(
          gout, P->dst_sorted, inv_deg, P->tile_c, P->tile_e0, P->tile_cnt, scal, static_cast<T16*>(G16), Gs, argmax,
          P->perm);
    };
    auto by_max = [&](auto t16, auto split) {
      if (argmax != nullptr) gather(t16, split, std::true_type());
      else gather(t16, split, std::false_type());
    };
    if (sp) by_max(__half(), std::integral_constant<int, 1>());
    else if (bf) by_max(__nv_bfloat16(), std::integral_constant<int, 0>());
    else by_max(__half(), std::integral_constant<int, 0>());
  }
  NNC_CHECK_LAUNCH();
  if (sp) k_prep_xg<__half, 1><<<(unsigned)ceil_div64(static_cast<int64_t>(S) * cin_p, 256), 256, 0, st>>>(
      x, P->src_nodes, S, cin, cin_p, scal, static_cast<__half*>(Xg));
  else if (bf) k_prep_xg<__nv_bfloat16><<<(unsigned)ceil_div64(static_cast<int64_t>(S) * cin_p, 256), 256, 0, st>>>(
      x, P->src_nodes, S, cin, cin_p, scal, static_cast<__nv_bfloat16*>(Xg));
  else k_prep_xg<__half><<<(unsigned)ceil_div64(static_cast<int64_t>(S) * cin_p, 256), 256, 0, st>>>(
      x, P->src_nodes, S, cin, cin_p, scal, static_cast<__half*>(Xg));
  NNC_CHECK_LAUNCH();
  NNC_CHECK_CUDA(cudaMemsetAsync(dW3, 0, sizeof(float) * static_cast<size_t>(Kp) * cout * cin_p, st));
  // dB_L = x_src^T Gs
  k_xtv<<<(unsigned)ceil_div(S, 32), 256, sizeof(float) * 32 * (cin + cout), st>>>(x, P->src_nodes, Gs, S, cin, cout, dbL);
  NNC_CHECK_LAUNCH();
  count(6);

  Maps8 tmG;
  for (int i = 0; i < 8; ++i) {
    s = make_tmap_2d_16b(&tmG.m[i], bf, G16, static_cast<uint64_t>((sp ? 2 : 1) * P->n_tiles) * 128, 64, 16 * (i + 1));
    if (s) return s;
  }
  static bool attr_set = false;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dy<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDySmem));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dy<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDySmem));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dy<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDySmem));
    attr_set = true;
  }
  const int NY = Kp * cout;
  const int panels = (sp ? 2 : 1) * Kp / 64;
  // sources [c0, c0 + nb) against h holding the sorted edges [h_e_base, ...) in panels of h_rows rows
  auto run_batch = [&](int64_t c0, int nb, const void* hb, int64_t h_e_base, int64_t h_rows, float* dxp_b,
                       uint16_t* dY_b) -> int {
    Maps8 tmH;
    for (int i = 0; i < 8; ++i) {
      int r = make_tmap_2d_16b(&tmH.m[i], bf, hb, static_cast<uint64_t>(panels) * h_rows, 64, 16 * (i + 1));
      if (r) return r;
    }
    DyArgs a;
    a.tile_ptr = P->tile_ptr; a.tile_e0 = P->tile_e0; a.tile_cnt = P->tile_cnt;
    a.c0 = static_cast<int>(c0); a.c1 = static_cast<int>(c0) + nb;
    a.h_e_base = static_cast<int>(h_e_base); a.h_rows = static_cast<int>(h_rows);
    a.nk = Kp / 64; a.num_mt = (a.nk + 1) / 2;
    a.Kp = Kp; a.g_lo_row = P->n_tiles * 128; a.dY = dY_b;
    const int grid = nb < tc_num_sms() ? nb : tc_num_sms();
    if (sp) k_dy<0, 1><<<grid, 160, kDySmem, st>>>(tmH, tmG, a);
    else if (bf) k_dy<1><<<grid, 160, kDySmem, st>>>(tmH, tmG, a);
    else k_dy<0><<<grid, 160, kDySmem, st>>>(tmH, tmG, a);
    NNC_CHECK_LAUNCH();
    // dxp[c, i] = sum_n dY[c, n] W3t[i, n]      (fp32 out; PREC_F16X2: split A against the pre-scaled split W3t)
    int r = launch_gemm_tc(W->prec, dY_b, nb, 0, nb, (sp ? 3 : 1) * NY, W->W3t, cin_p, nullptr, 0, dxp_b, cin_p, st, nullptr,
                           0, 0, sp ? GEMM_A_SPLIT : 0, nullptr, nullptr, 0, 1);
    if (r) return r;
    k_scatter_dx_tc<<<(unsigned)ceil_div64(static_cast<int64_t>(nb) * cin, 256), 256, sizeof(float) * cin * (cout + 1), st>>>(
        dxp_b, cin_p, Gs, W->B3, P->src_nodes, static_cast<int>(c0), nb, cin, cout, scal,
        sp ? W->wscale + 2 * W->n_layers + 1 : nullptr, dx);
    NNC_CHECK_LAUNCH();
    // dW3[(k,o), i] += sum_c dY[c, (k,o)] Xg[c0 + c, i]
    r = gemm_tn_pairs(W, dY_b, (sp ? 2 : 1) * NY, NY,
                      static_cast<const char*>(Xg) + static_cast<size_t>(c0) * cin_p * 2 * (sp ? 2 : 1), (sp ? 2 : 1) * cin_p,
                      cin_p, nb, NY, cin_p, dW3, cin_p, st);
    count(sp ? 6 : 4);
    return r;
  };
  // sources inside the resident prefix (all of them when h is whole)
  const int c_res = first_streamed_src(P, E_res);
  for (int64_t c0 = 0; c0 < c_res; c0 += nb_max) {
    const int nb = static_cast<int>((c_res - c0) < nb_max ? (c_res - c0) : nb_max);
    s = run_batch(c0, nb, h, 0, round_up64(E_res, 128), dxp, dY);
    if (s) return s;
  }
  // the other sources: recompute the h of each batch's edges [g[c0], g[c1]) into the chunk buffer after its dY rows.
  // Its padding rows are zeroed (TMA boxes reach them; the G rows they meet are zero)
  const int* g = P->h_group_ptr;
  for (int c0 = c_res; c0 < S;) {
    const int c1 = apply_stream_batch_end(P, W, L, c0, pool);
    NNC_REQUIRE(c1 > c0, NNCONV_ERR_WORKSPACE,
                "backward_apply: workspace too small for one source (use nnconv_backward_apply_streamed_sizes)");
    const int nb = c1 - c0;
    const int64_t e_lo = g[c0], n = g[c1] - g[c0];
    uint16_t* dY_b = reinterpret_cast<uint16_t*>(dyn + round_up64(static_cast<int64_t>(nb + 128) * cin_p * 4, 1024));
    char* hc = reinterpret_cast<char*>(dY_b) + round_up64(static_cast<int64_t>(nb) * NY * 2 * (sp ? 2 : 1), 1024);
    s = edge_features_rows(P, W, edge_attr, e_lo, n, hc, ef_ws, ef_bytes, nullptr, st, launches, nullptr);
    if (s) return s;
    s = run_batch(c0, nb, hc, e_lo, round_up64(n, 128), dxp, dY_b);
    if (s) return s;
    c0 = c1;
  }
  k_unpermute_w3q<<<(unsigned)ceil_div64(nWL, 256), 256, 0, st>>>(dW3, cin, cout, W->K, cin_p, scal, 6, dWL);
  NNC_CHECK_LAUNCH();
  count(1);
  return NNCONV_OK;
}

// -----------------------------------------------------------------------------------------------------
// deferred pass over the hidden layers
// -----------------------------------------------------------------------------------------------------
namespace {
struct MlpBwdLayout {
  size_t off_scal, off_Xc[kMaxApps], off_xs[kMaxApps], off_cvec, off_dW[kMaxLayers], off_D[kMaxLayers], fixed;
  size_t per_edge, per_src;
};

MlpBwdLayout mlp_bwd_layout(const Plan* P, const Weights* W, int T, bool streamed) {
  Carver c(nullptr, ~size_t(0));
  MlpBwdLayout L{};
  const size_t S = P->n_src > 0 ? P->n_src : 1;
  const int nl = W->n_layers;
  const size_t pm = W->split ? 2 : 1;      // PREC_F16X2: [hi | lo] pairs (Xc: [hi | hi | lo], see launch_src_prep)
  L.off_scal = c.off; c.take<float>(64);
  for (int t = 0; t < T; ++t) {
    L.off_Xc[t] = c.off; c.take<char>((S + 128) * W->cin_p * 2 * (W->split ? 3 : 1));
    L.off_xs[t] = c.off; c.take<float>(S);
  }
  L.off_cvec = c.off; c.take<float>(S * W->cout);
  for (int l = 1; l <= nl - 1; ++l) {
    if (l >= 2) { L.off_dW[l] = c.off; c.take<float>(static_cast<size_t>(W->kp[l]) * W->kp[l - 1]); }
    L.off_D[l] = c.off; c.take<float>(static_cast<size_t>(W->kp[l]) * 64);
  }
  L.fixed = c.off;
  size_t acts = 0, maxkp = 0;
  for (int l = 1; l <= nl - 1; ++l) {
    if (l <= nl - 2) acts += W->kp[l];
    maxkp = static_cast<size_t>(W->kp[l]) > maxkp ? W->kp[l] : maxkp;
  }
  // Ghat row + dz ping/pong + stored hidden activations h_1..h_{L-2} + A1 row
  L.per_edge = (static_cast<size_t>(T) * 128 + 2 * maxkp * 2 + acts * 2) * pm + 128;
  // streamed edge features: + the recomputed h_{L-1} of a batch (its ReLU mask), chunk-major
  if (streamed) L.per_edge += static_cast<size_t>(W->Kp) * 2 * pm;
  L.per_src = static_cast<size_t>(T) * W->Kp * 64 * 2 * pm;      // Y^T rows of the T applications
  return L;
}

// end of the source batch starting at c0: sources while their Y^T rows and per-edge buffers fit avail (c0 = not even
// one source group fits)
int mlp_batch_end(const Plan* P, const MlpBwdLayout& L, int c0, size_t avail) {
  const int* hgp = P->h_group_ptr;
  int c1 = c0;
  size_t used = 0;
  while (c1 < P->n_src) {
    const size_t add = L.per_src + L.per_edge * static_cast<size_t>(hgp[c1 + 1] - hgp[c1]);
    if (used + add + L.per_edge * 256 > avail) break;
    used += add;
    ++c1;
  }
  return c1;
}
}  // namespace

int64_t backward_streamed_chunks(const Plan* P, const Weights* W, int T, int64_t E_res, size_t ws_bytes) {
  if (E_res >= P->E || P->n_src == 0) return 0;
  int64_t n = 0;
  if (T == 0) {
    const ApplyBwdLayout L = apply_bwd_layout(P, W);
    const size_t fixed = L.fixed + bwd_ef_bytes(P, W, E_res) + 4096;
    if (ws_bytes <= fixed) return 0;
    for (int c0 = first_streamed_src(P, E_res); c0 < P->n_src; ++n) {
      const int c1 = apply_stream_batch_end(P, W, L, c0, ws_bytes - fixed);
      if (c1 == c0) return 0;
      c0 = c1;
    }
    return n;
  }
  const MlpBwdLayout L = mlp_bwd_layout(P, W, T, true);
  if (ws_bytes <= L.fixed + (1 << 16)) return 0;
  for (int c0 = 0; c0 < P->n_src;) {
    const int c1 = mlp_batch_end(P, L, c0, ws_bytes - L.fixed - (1 << 16));
    if (c1 == c0) return 0;
    if (P->h_group_ptr[c1] > E_res) ++n;
    c0 = c1;
  }
  return n;
}

size_t backward_mlp_ws_bytes(const Plan* P, const Weights* W, int T, size_t want_bytes, int64_t E_res) {
  MlpBwdLayout L = mlp_bwd_layout(P, W, T, E_res >= 0 && E_res < P->E);
  const size_t deg = P->max_out_deg > 0 ? P->max_out_deg : 1;
  const size_t need_min = L.fixed + L.per_src + L.per_edge * (deg + 256) + (1 << 16);
  const size_t all = L.fixed + L.per_src * (P->n_src > 0 ? P->n_src : 1) + L.per_edge * (static_cast<size_t>(P->E) + 256) +
                     (1 << 16);
  size_t w = want_bytes < need_min ? need_min : want_bytes;
  return w < all ? w : all;
}

int backward_mlp_tc(const Plan* P, const Weights* W, const float* edge_attr, const void* h, int64_t E_res, int T,
                    const float* const* gouts, const float* const* xs_in, int aggr_mean, float* const* dWs,
                    float* const* dbs, void* ws, size_t ws_bytes, cudaStream_t st, const void* acts, float* grad_ea,
                    const int* const* argmax) {
  NNC_REQUIRE(backward_tc_supported(W), NNCONV_ERR_UNSUPPORTED, "tensor-core backward: unsupported shape / precision");
  const bool streamed = E_res < P->E;
  if (streamed || (acts != nullptr && edge_acts_bytes(P, W) == 0)) acts = nullptr;
  NNC_REQUIRE(T >= 1 && T <= kMaxApps, NNCONV_ERR_ARG, "backward_mlp: 1..%d applications per pass", kMaxApps);
  const int nl = W->n_layers;
  const int cin = W->cin, cout = W->cout, Kp = W->Kp, cin_p = W->cin_p, k_in = W->dims[0];
  const int bf = W->prec == PREC_BF16;
  // PREC_F16X2: every 16-bit buffer of the pass holds [hi | lo] pairs (pm = 2), the GEMMs read split operands
  // (K tripled, kmul = 3) against the pre-scaled split weight images, whose power of two the epilogues undo
  const int sp = W->split, pm = sp ? 2 : 1, kmul = sp ? 3 : 1;
  int s = tc_init();
  if (s) return s;
  // gradient w.r.t. edge_attr: W_1 transposed in shared memory (k_in <= 20 on this path)
  const int ea_smem = static_cast<int>(sizeof(float)) * k_in * W->kp[1];
  NNC_REQUIRE(grad_ea == nullptr || (k_in <= 20 && ea_smem <= 227 * 1024), NNCONV_ERR_UNSUPPORTED,
              "backward_mlp: edge_attr gradient needs k_in * k_1 <= 58112 (first Linear in shared memory)");
  // zero gradients for an empty graph
  if (P->E == 0 || P->n_src == 0) {
    for (int l = 1; l <= nl - 1; ++l) {
      NNC_CHECK_CUDA(cudaMemsetAsync(dWs[l - 1], 0, sizeof(float) * W->dims[l] * W->dims[l - 1], st));
      NNC_CHECK_CUDA(cudaMemsetAsync(dbs[l - 1], 0, sizeof(float) * W->dims[l], st));
    }
    return NNCONV_OK;
  }
  MlpBwdLayout L = mlp_bwd_layout(P, W, T, streamed);
  NNC_REQUIRE(ws != nullptr && ws_bytes >= L.fixed + L.per_src + L.per_edge * 256, NNCONV_ERR_WORKSPACE,
              "backward_mlp: workspace too small");
  char* base = static_cast<char*>(ws);
  float* scal = reinterpret_cast<float*>(base + L.off_scal);
  const int S = P->n_src;
  const float* inv_deg = aggr_mean ? P->inv_deg : nullptr;
  NNC_CHECK_CUDA(cudaMemsetAsync(base, 0, L.fixed, st));        // scales and every accumulator
  GatherGArgs ga{};
  ga.T = T;
  GatherMaxArgs gm{};
  gm.perm = P->perm;
  if (argmax != nullptr)
    for (int t = 0; t < T; ++t) gm.argmax[t] = argmax[t];
  float* cvec = reinterpret_cast<float*>(base + L.off_cvec);
  for (int t = 0; t < T; ++t) {
    void* Xc = base + L.off_Xc[t];
    float* xs = reinterpret_cast<float*>(base + L.off_xs[t]);
    s = launch_src_prep(W->prec, xs_in[t], P->src_nodes, S, cin, cin_p, cout, W->B3, Xc, cvec, xs, st);
    if (s) return s;
    k_absmax_rows<<<592, 256, 0, st>>>(gouts[t], inv_deg, nullptr, P->N_dst, cout, scal + t);
    NNC_CHECK_LAUNCH();
    k_max_f<<<64, 256, 0, st>>>(xs, S, scal + 8 + t);
    NNC_CHECK_LAUNCH();
    ga.g[t] = gouts[t];
    ga.xs[t] = xs;
  }
  k_mlp_scales<<<1, 1, 0, st>>>(scal, T);
  NNC_CHECK_LAUNCH();

  // ---- batches of sources: [c0, c1) with edges [e_base, e_base + n)
  const int* hgp = P->h_group_ptr;
  const int* htp = P->h_tile_ptr;
  const size_t avail = ws_bytes - L.fixed - (1 << 16);
  const int64_t h_rows_res = round_up64(E_res, 128);     // panel height of h (the whole h: round_up(E, 128))
  const int BN = Kp % 128 == 0 ? 128 : 64;   // k block of k_dh (Kp is a multiple of 64; <= 128 accumulator registers)
  int maxkp = 0;
  for (int l = 1; l <= nl - 1; ++l) maxkp = W->kp[l] > maxkp ? W->kp[l] : maxkp;
  static bool attr_set = false;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<0, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<1, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<0, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<1, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_ea_grad<0, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_ea_grad<1, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_ea_grad<0, 20>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_ea_grad<1, 20>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<0, 64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_dh<0, 128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_ea_grad<0, 8, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_ea_grad<0, 20, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  int dh_smem = dh_pipe_bytes(sp, BN, T) + 1024 + kDhScratch;
  NNC_REQUIRE(dh_smem <= 227 * 1024, NNCONV_ERR_UNSUPPORTED, "backward_mlp: T=%d applications do not fit shared memory", T);
  // bias gradient of the top hidden layer fused into k_dh (one pass over dz_{L-1} saved) when the transpose + column
  // accumulators fit next to the operand stages; layer 1 (nl == 2) needs the full dz^T A1 product anyway
  const int cs_bytes = 4 * (32 * 33 * 4 + 4 * Kp);
  const bool fuse_colsum = nl >= 3 && dh_smem + cs_bytes <= 227 * 1024;
  if (fuse_colsum) dh_smem += cs_bytes;
  int c0 = 0;
  while (c0 < S) {
    const int c1 = mlp_batch_end(P, L, c0, avail);
    NNC_REQUIRE(c1 > c0, NNCONV_ERR_WORKSPACE, "backward_mlp: workspace too small for one source group");
    const int nb = c1 - c0, e_base = hgp[c0], n = hgp[c1] - hgp[c0];
    const int64_t n_pad = round_up64(n, 128) + 128;
    // a batch with edges past the resident prefix recomputes its own h_{L-1} (the ReLU mask of k_dh) from the hidden
    // activations below, with the forward's GEMMs (same bits as the h the forward contracted)
    const bool stream_h = e_base + n > E_res;
    Carver cv(base + L.fixed, avail + (1 << 16));
    uint16_t* Yt = cv.take<uint16_t>(static_cast<size_t>(T) * nb * Kp * 64 * pm);
    uint16_t* Gh = cv.take<uint16_t>(static_cast<size_t>(n_pad) * T * 64 * pm);
    uint16_t* dzA = cv.take<uint16_t>(static_cast<size_t>(n_pad) * maxkp * pm);
    uint16_t* dzB = cv.take<uint16_t>(static_cast<size_t>(n_pad) * maxkp * pm);
    uint16_t* A1 = cv.take<uint16_t>(static_cast<size_t>(n_pad) * 64);
    uint16_t* act[kMaxLayers + 1] = {nullptr};
    for (int l = 1; l <= nl - 2; ++l) {
      if (acts != nullptr)   // kept by the forward (nnconv_edge_features_keep): rows [e_base, e_base + n) of layer l
        act[l] = const_cast<uint16_t*>(reinterpret_cast<const uint16_t*>(static_cast<const char*>(acts) + edge_acts_offset(P, W, l))) +
                 static_cast<size_t>(e_base) * W->kp[l];
      else
        act[l] = cv.take<uint16_t>(static_cast<size_t>(n_pad) * W->kp[l] * pm);
    }
    uint16_t* hb = stream_h ? cv.take<uint16_t>(static_cast<size_t>(n_pad) * Kp * pm) : nullptr;
    NNC_REQUIRE(cv.ok(), NNCONV_ERR_WORKSPACE, "backward_mlp: workspace carve overflow");
    // ---- the hidden activations h_1 .. h_{L-2} of the batch (16-bit, row-major) and A1
    auto recompute_acts = [&]() -> int {
      int r = launch_build_a1(W->prec, edge_attr, P->perm, e_base, n, k_in, A1, st);
      if (r) return r;
      if (nl >= 3 && acts == nullptr) {
        r = launch_gemm_tc(W->prec, A1, n, 0, n, 64, W->W1aug, W->kp[1], nullptr, 1, act[1], pm * W->kp[1], st, nullptr, 0, 0,
                           sp ? GEMM_C_SPLIT : 0, nullptr, nullptr, 0, 0, 0, nullptr, W->act);
        if (r) return r;
        for (int l = 2; l <= nl - 2; ++l) {
          r = launch_gemm_tc(W->prec, act[l - 1], n, 0, n, kmul * W->kp[l - 1], W->Wh[l], W->kp[l], W->bh[l], 1, act[l],
                             pm * W->kp[l], st, nullptr, 0, 0, sp ? (GEMM_A_SPLIT | GEMM_C_SPLIT) : 0, nullptr, nullptr, 0, 0,
                             0, sp ? W->wscale + 2 * l + 1 : nullptr, W->act);
          if (r) return r;
        }
      }
      return NNCONV_OK;
    };
    if (stream_h) {
      s = recompute_acts();
      if (s) return s;
      // h_{L-1} of the batch into chunk-major panels of round_up(n, 128) rows (edge_features_rows' last GEMM)
      const int64_t hpad = round_up64(n, 128);
      if (nl == 2)
        s = launch_gemm_tc(W->prec, A1, n, 0, n, 64, W->W1aug, W->kp[1], nullptr, 1, hb, pm * W->kp[1], st, nullptr, hpad, 0,
                           sp ? GEMM_C_SPLIT : 0, nullptr, nullptr, 0, 0, 0, nullptr, W->act);
      else
        s = launch_gemm_tc(W->prec, act[nl - 2], n, 0, n, kmul * W->kp[nl - 2], W->Wh[nl - 1], W->kp[nl - 1], W->bh[nl - 1], 1,
                           hb, pm * W->kp[nl - 1], st, nullptr, hpad, 0, sp ? (GEMM_A_SPLIT | GEMM_C_SPLIT) : 0, nullptr,
                           nullptr, 0, 0, 0, sp ? W->wscale + 2 * (nl - 1) + 1 : nullptr, W->act);
      if (s) return s;
    }
    // ---- Y^T of the batch for every application: Yt[t][(c, k), o] = sum_i Xc_t[c, i] W_L[i*out + o, k]
    //      (PREC_F16X2: row c of application t is [hi | lo], 2 * Kp * 64)
    for (int t = 0; t < T; ++t) {
      s = launch_gemm_tc(W->prec, base + L.off_Xc[t], S, c0, nb, kmul * cin_p, W->W3q, Kp * 64, nullptr, 0,
                         Yt + static_cast<size_t>(t) * nb * Kp * 64 * pm, static_cast<int64_t>(pm) * Kp * 64, st, nullptr, 0,
                         0, sp ? GEMM_C_SPLIT : 0, nullptr, nullptr, 0, 0, 0, sp ? W->wscale + 2 * nl + 1 : nullptr);
      if (s) return s;
    }
    // ---- Ghat rows of the batch
    {
      const int nt = htp[c1] - htp[c0];
      auto gather = [&](auto t16, auto split, auto mx) {
        using T16 = decltype(t16);
        k_gather_ghat<T16, decltype(split)::value, decltype(mx)::value><<<nt, 256, 0, st>>>(
            ga, P->dst_sorted, inv_deg, P->tile_c, P->tile_e0, P->tile_cnt, htp[c0], e_base, scal,
            reinterpret_cast<T16*>(Gh), gm);
      };
      auto by_max = [&](auto t16, auto split) {
        if (argmax != nullptr) gather(t16, split, std::true_type());
        else gather(t16, split, std::false_type());
      };
      if (sp) by_max(__half(), std::integral_constant<int, 1>());
      else if (bf) by_max(__nv_bfloat16(), std::integral_constant<int, 0>());
      else by_max(__half(), std::integral_constant<int, 0>());
      NNC_CHECK_LAUNCH();
    }
    // ---- dz_{L-1} = [h > 0] * (Ghat . Yt)
    {
      Maps8 tmA;
      CUtensorMap tmB;
      for (int i = 0; i < 8; ++i) {
        s = make_tmap_2d_16b(&tmA.m[i], bf, Gh, static_cast<uint64_t>(n_pad), static_cast<uint64_t>(pm) * T * 64, 16 * (i + 1));
        if (s) return s;
      }
      s = make_tmap_2d_16b(&tmB, bf, Yt, static_cast<uint64_t>(pm) * T * nb * Kp, 64, BN);
      if (s) return s;
      DhArgs a;
      a.tile_c = P->tile_c; a.tile_e0 = P->tile_e0; a.tile_cnt = P->tile_cnt;
      a.tile0 = htp[c0]; a.tile1 = htp[c1]; a.c0 = c0; a.Sb = nb; a.e_base = e_base;
      a.h_e_base = stream_h ? e_base : 0;
      a.h_rows = static_cast<int>(stream_h ? round_up64(n, 128) : h_rows_res);
      a.T = T; a.Kp = Kp; a.n_nb = Kp / BN;
      a.h = stream_h ? hb : static_cast<const uint16_t*>(h); a.dz = dzA;
      a.colsum = fuse_colsum ? reinterpret_cast<float*>(base + L.off_D[nl - 1]) + 3 * k_in : nullptr;
      a.colsum_stride = 64;
      const int tiles = a.tile1 - a.tile0;
      const int grid = tiles < tc_num_sms() ? tiles : tc_num_sms();
      a.act_q0 = W->act.p.v[0]; a.act_q1 = W->act.p.v[1]; a.act_q2 = W->act.p.v[2];
      if (W->act.kind != ACT_RELU) {
        s = act_dispatch(W->act.kind, [&](auto k) {
          constexpr int M = decltype(k)::value << 1;
          if (sp) return BN == 128 ? launch_dh<0, 128, M | 1>(tmA, tmB, a, grid, dh_smem, st)
                                   : launch_dh<0, 64, M | 1>(tmA, tmB, a, grid, dh_smem, st);
          if (BN == 128) return bf ? launch_dh<1, 128, M>(tmA, tmB, a, grid, dh_smem, st)
                                   : launch_dh<0, 128, M>(tmA, tmB, a, grid, dh_smem, st);
          return bf ? launch_dh<1, 64, M>(tmA, tmB, a, grid, dh_smem, st) : launch_dh<0, 64, M>(tmA, tmB, a, grid, dh_smem, st);
        });
        if (s) return s;
      } else if (sp) {
        if (BN == 128) k_dh<0, 128, 1><<<grid, 160, dh_smem, st>>>(tmA, tmB, a);
        else k_dh<0, 64, 1><<<grid, 160, dh_smem, st>>>(tmA, tmB, a);
      } else if (BN == 128) {
        if (bf) k_dh<1, 128><<<grid, 160, dh_smem, st>>>(tmA, tmB, a);
        else k_dh<0, 128><<<grid, 160, dh_smem, st>>>(tmA, tmB, a);
      } else {
        if (bf) k_dh<1, 64><<<grid, 160, dh_smem, st>>>(tmA, tmB, a);
        else k_dh<0, 64><<<grid, 160, dh_smem, st>>>(tmA, tmB, a);
      }
      NNC_CHECK_LAUNCH();
    }
    if (!stream_h) {
      s = recompute_acts();
      if (s) return s;
    }
    // ---- down through the layers
    uint16_t* cur = dzA;
    uint16_t* nxt = dzB;
    for (int l = nl - 1; l >= 1; --l) {
      float* Dl = reinterpret_cast<float*>(base + L.off_D[l]);
      // D_l[j, :] += dz_l^T A1   (column 3*k_in = the bias gradient; for l = 1 also dW_1 in split form); the top
      // layer's column comes out of k_dh when fused
      if (!(fuse_colsum && l == nl - 1)) {
        s = gemm_tn_pairs(W, cur, pm * W->kp[l], W->kp[l], A1, 64, -1, n, W->kp[l], 64, Dl, 64, st);
        if (s) return s;
      }
      if (l >= 2) {
        float* dWl = reinterpret_cast<float*>(base + L.off_dW[l]);
        s = gemm_tn_pairs(W, cur, pm * W->kp[l], W->kp[l], act[l - 1], pm * W->kp[l - 1], W->kp[l - 1], n, W->kp[l],
                          W->kp[l - 1], dWl, W->kp[l - 1], st);
        if (s) return s;
        // dz_{l-1} = (dz_l W_l) * [h_{l-1} > 0]   (PREC_F16X2: the mask is the hi half of the activation pair); another
        // activation multiplies by f'(h_{l-1}) instead (PREC_F16X2: of hi + lo)
        s = launch_gemm_tc(W->prec, cur, n, 0, n, kmul * W->kp[l], W->WhT[l], W->kp[l - 1], nullptr, 0, nxt,
                           pm * W->kp[l - 1], st, nullptr, 0, 0, sp ? (GEMM_A_SPLIT | GEMM_C_SPLIT) : 0, nullptr, act[l - 1],
                           pm * W->kp[l - 1], 0, 0, sp ? W->wscale + 2 * l + 1 : nullptr, W->act);
        if (s) return s;
        uint16_t* tmp = cur; cur = nxt; nxt = tmp;
      }
    }
    // ---- cur = dz_1 of the batch (summed over the applications): grad_edge_attr rows of its edges
    if (grad_ea != nullptr) {
      auto kern = sp ? (k_in <= 8 ? k_ea_grad<0, 8, 1> : k_ea_grad<0, 20, 1>)
                     : k_in <= 8 ? (bf ? k_ea_grad<1, 8> : k_ea_grad<0, 8>) : (bf ? k_ea_grad<1, 20> : k_ea_grad<0, 20>);
      // as many resident CTAs as fit (a bandwidth-bound stream: every resident warp keeps loads in flight)
      int per_sm = 0;
      NNC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, ea_smem));
      const int64_t resident = static_cast<int64_t>(per_sm > 0 ? per_sm : 1) * tc_num_sms();
      const unsigned grid = static_cast<unsigned>(std::min<int64_t>(ceil_div64(n, kEaRowsPerBlock), resident));
      kern<<<grid, 256, ea_smem, st>>>(cur, n, W->kp[1], W->W1, k_in, P->perm, e_base, scal, 16, grad_ea);
      NNC_CHECK_LAUNCH();
    }
    c0 = c1;
  }
  // ---- scale back and write the caller's gradient tensors
  for (int l = 2; l <= nl - 1; ++l) {
    const int R = W->dims[l], C = W->dims[l - 1];
    k_scale_unpad<<<(unsigned)ceil_div64(static_cast<int64_t>(R) * C, 256), 256, 0, st>>>(
        reinterpret_cast<const float*>(base + L.off_dW[l]), W->kp[l - 1], 0, scal, 16, dWs[l - 1], R, C);
    NNC_CHECK_LAUNCH();
    k_scale_unpad<<<ceil_div(R, 256), 256, 0, st>>>(reinterpret_cast<const float*>(base + L.off_D[l]), 64, 3 * k_in, scal, 16,
                                                    dbs[l - 1], R, 1);
    NNC_CHECK_LAUNCH();
  }
  k_fold_w1<<<ceil_div(W->dims[1] * (k_in + 1), 256), 256, 0, st>>>(reinterpret_cast<const float*>(base + L.off_D[1]),
                                                                    W->dims[1], k_in, scal, 16, dWs[0], dbs[0]);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

}  // namespace nnc
