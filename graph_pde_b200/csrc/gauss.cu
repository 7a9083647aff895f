// Gaussian-kernel NNConv (DESIGN 4.9): the reference's graph-neural-operator/nn_conv.py:99-194 NNConv_Gaussian, whose
// message is x_j . diag(d_e) with a diagonal that depends on three edge attributes and one width-C vector sigma:
//   a_e  = 1 / sqrt(|p_e1 * p_e2|)          d_ec = a_e * exp(-p_e0^2 / sigma_c^2)          (p_e = edge_attr row e)
//   out_n = aggr_{e: dst_e = n} x_src(e),c * d_ec  +  x_n root + bias
// d is computed in registers inside the application and the backward, never stored: one pass reads x, three attributes
// per edge and sigma, and reduces the messages into out in fp32.  The rounding follows torch's fp32 order (IEEE sqrt
// and reciprocal for a, IEEE division for p0^2 / sigma^2, then exp, a * exp, x * d), so with p0 = 0 and p1 * p2 a power
// of four every message is exact.
#include "kernels.h"

namespace nnc {

namespace {

constexpr int kGaussWarps = 8;   // warps per CTA (256 threads)

// a_e = 1 / sqrt(|p1 p2|), IEEE-rounded at each step as torch's fp32 ops round it
__device__ __forceinline__ float gauss_amp(float p1, float p2) { return __frcp_rn(__fsqrt_rn(fabsf(p1 * p2))); }

// d = a * exp(-(p0^2) / sigma^2), nsq = -(p0 * p0)
__device__ __forceinline__ float gauss_d(float a, float nsq, float s2) { return a * expf(__fdiv_rn(nsq, s2)); }

// One warp per plan tile (<= 128 edges of one source), the schedule of k_apply_diag: for every edge e of the tile and
// channel c, m = x_src[c] * d_ec (times inv_deg[dst] for mean) is added into out[dst, c] (AGGR 0 add, 1 mean) or reduced
// into the max key of (dst, c) (AGGR 2).  The three attributes of e are read from the caller-order edge_attr (row stride
// k_in) through the plan's permutation.  VEC: C % 4 == 0, 16-byte loads of x and one red.global.add.v4.f32 per four
// channels.  Dynamic shared memory: sigma_c^2 [C].
template <int AGGR, bool VEC>
__global__ void __launch_bounds__(256) k_apply_gauss(const float* __restrict__ ea, int k_in, const float* __restrict__ sigma,
                                                     const float* __restrict__ x, int C, int n_tiles,
                                                     const int* __restrict__ tile_c, const int* __restrict__ tile_e0,
                                                     const int* __restrict__ tile_cnt, const int* __restrict__ src_nodes,
                                                     const int* __restrict__ dst_sorted, const float* __restrict__ inv_deg,
                                                     const int* __restrict__ perm, float* __restrict__ out,
                                                     unsigned long long* __restrict__ keys) {
  extern __shared__ float s2[];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float s = __ldg(sigma + c);
    s2[c] = s * s;
  }
  __syncthreads();
  const int t = static_cast<int>((blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const int e0 = __ldg(tile_e0 + t), cnt = __ldg(tile_cnt + t);
  const float* xs = x + static_cast<int64_t>(__ldg(src_nodes + __ldg(tile_c + t))) * C;
  const int q = VEC ? C / 4 : C;
  for (int i = lane; i < cnt * q; i += 32) {
    const int p = i / q, j = i - p * q;
    const int64_t e = e0 + p;
    const int dn = __ldg(dst_sorted + e);
    const uint32_t ce = caller_edge(perm, e);
    const float* pe = ea + static_cast<int64_t>(ce) * k_in;
    const float p0 = __ldg(pe), a = gauss_amp(__ldg(pe + 1), __ldg(pe + 2));
    const float nsq = -(p0 * p0);
    const float w = AGGR == 1 ? __ldg(inv_deg + dn) : 1.f;
    if (VEC) {
      const float4 xv = __ldg(reinterpret_cast<const float4*>(xs) + j);
      const float* sj = s2 + 4 * j;
      float4 m = make_float4(xv.x * gauss_d(a, nsq, sj[0]), xv.y * gauss_d(a, nsq, sj[1]),
                             xv.z * gauss_d(a, nsq, sj[2]), xv.w * gauss_d(a, nsq, sj[3]));
      if (AGGR == 1) m = make_float4(m.x * w, m.y * w, m.z * w, m.w * w);
      if (AGGR == 2) {
        unsigned long long* k = keys + static_cast<int64_t>(dn) * C + 4 * j;
        atomicMax(k, max_key(m.x, ce));
        atomicMax(k + 1, max_key(m.y, ce));
        atomicMax(k + 2, max_key(m.z, ce));
        atomicMax(k + 3, max_key(m.w, ce));
      } else {
        atomicAdd(reinterpret_cast<float4*>(out + static_cast<int64_t>(dn) * C) + j, m);
      }
    } else {
      float m = __ldg(xs + j) * gauss_d(a, nsq, s2[j]);
      if (AGGR == 1) m *= w;
      if (AGGR == 2) atomicMax(keys + static_cast<int64_t>(dn) * C + j, max_key(m, ce));
      else atomicAdd(out + static_cast<int64_t>(dn) * C + j, m);
    }
  }
}

// Backward of one application over the same tiles.  G_ec = g[dst_e, c] (add), times inv_deg[dst_e] (mean), or masked
// by the forward's argmax (max); u_ec = G_ec * x_src,c * d_ec.  Per tile:
//   dx[src, c]  += sum_e G_ec d_ec                        one atomic per channel
//   dsigma_c    += 2 / sigma_c^3 * sum_e u_ec p_e0^2        one atomic per channel (dsig nullable)
//   dea[e, 0]    = -2 p_e0 sum_c u_ec / sigma_c^2           written once per edge into the caller's row (dea nullable;
//   dea[e, 1|2]  = -(sum_c u_ec) / (2 p_e1|2)               columns 3 and up get 0)
// Lanes per edge lp = min(32, next power of two of q) (q = C / 4 with VEC, else C), so 32 / lp edges run side by side;
// the per-edge channel sums are reduced across an edge's lanes with shuffles and kept in shared memory until every
// channel block has run.  VEC: 16-byte loads of x, g (and argmax) and one 16-byte atomic per four channels of dx.
// Dynamic shared memory: sigma_c^2 [C], then 1 / sigma_c^2 [C].
template <int AGGR, bool VEC>
__global__ void __launch_bounds__(256) k_bwd_gauss(const float* __restrict__ ea, int k_in, const float* __restrict__ sigma,
                                                   const float* __restrict__ x, const float* __restrict__ gout, int C,
                                                   int n_tiles, const int* __restrict__ tile_c,
                                                   const int* __restrict__ tile_e0, const int* __restrict__ tile_cnt,
                                                   const int* __restrict__ src_nodes, const int* __restrict__ dst_sorted,
                                                   const float* __restrict__ inv_deg, const int* __restrict__ argmax,
                                                   const int* __restrict__ perm, float* __restrict__ dx,
                                                   float* __restrict__ dsig, float* __restrict__ dea) {
  constexpr int V = VEC ? 4 : 1;
  extern __shared__ float sh[];
  float* s2 = sh;
  float* is2 = sh + C;
  __shared__ float esum[kGaussWarps][kTileEdges][2];   // per edge of the warp's tile: sum_c u / sigma^2, sum_c u
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float s = __ldg(sigma + c);
    s2[c] = s * s;
    is2[c] = 1.f / (s * s);
  }
  __syncthreads();
  const int t = static_cast<int>((blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (t >= n_tiles) return;
  const int e0 = __ldg(tile_e0 + t), cnt = __ldg(tile_cnt + t);
  const int64_t s = __ldg(src_nodes + __ldg(tile_c + t));
  const int q = C / V;
  int lp = 1;
  while (lp < q && lp < 32) lp *= 2;
  const int r = 32 / lp, sub = lane / lp, jl = lane % lp;
  const bool want_ea = dea != nullptr;
  float (*es)[2] = esum[warp];
  if (want_ea) {
    for (int p = lane; p < cnt; p += 32) es[p][0] = es[p][1] = 0.f;
    __syncwarp();
  }
  for (int jb = 0; jb < q; jb += lp) {
    const int j = jb + jl;
    const bool jok = j < q;
    float xv[V], adx[V], asg[V];
#pragma unroll
    for (int v = 0; v < V; ++v) { xv[v] = 0.f; adx[v] = 0.f; asg[v] = 0.f; }
    if (jok) {
      if (VEC) {
        const float4 t4 = __ldg(reinterpret_cast<const float4*>(x + s * C) + j);
        xv[0] = t4.x; xv[1] = t4.y; xv[2] = t4.z; xv[V - 1] = t4.w;
      } else {
        xv[0] = __ldg(x + s * C + j);
      }
    }
    for (int pb = 0; pb < cnt; pb += r) {
      const int p = pb + sub;
      float su = 0.f, sw = 0.f;
      if (p < cnt && jok) {
        const int64_t e = e0 + p;
        const int dn = __ldg(dst_sorted + e);
        const uint32_t ce = caller_edge(perm, e);
        const float* pe = ea + static_cast<int64_t>(ce) * k_in;
        const float p0 = __ldg(pe), a = gauss_amp(__ldg(pe + 1), __ldg(pe + 2));
        const float psq = p0 * p0, nsq = -psq;
        const int64_t k = static_cast<int64_t>(dn) * C + j * V;
        float g[V];
        if (VEC) {
          const float4 g4 = __ldg(reinterpret_cast<const float4*>(gout + k));
          g[0] = g4.x; g[1] = g4.y; g[2] = g4.z; g[V - 1] = g4.w;
        } else {
          g[0] = __ldg(gout + k);
        }
        if (AGGR == 1) {
          const float w = __ldg(inv_deg + dn);
#pragma unroll
          for (int v = 0; v < V; ++v) g[v] *= w;
        }
        if (AGGR == 2) {
          int am[V];
          if (VEC) {
            const int4 a4 = __ldg(reinterpret_cast<const int4*>(argmax + k));
            am[0] = a4.x; am[1] = a4.y; am[2] = a4.z; am[V - 1] = a4.w;
          } else {
            am[0] = __ldg(argmax + k);
          }
#pragma unroll
          for (int v = 0; v < V; ++v)
            if (static_cast<uint32_t>(am[v]) != ce) g[v] = 0.f;
        }
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const int c = j * V + v;
          const float d = gauss_d(a, nsq, s2[c]);
          adx[v] = fmaf(g[v], d, adx[v]);
          const float u = g[v] * xv[v] * d;
          asg[v] = fmaf(u, psq, asg[v]);
          su += u;
          sw = fmaf(u, is2[c], sw);
        }
      }
      if (want_ea) {
        for (int o = lp / 2; o > 0; o /= 2) {
          su += __shfl_xor_sync(0xffffffffu, su, o);
          sw += __shfl_xor_sync(0xffffffffu, sw, o);
        }
        if (jl == 0 && p < cnt) {
          es[p][0] += sw;
          es[p][1] += su;
        }
      }
    }
    // the r edge groups of the warp hold partial sums of the same channels: reduce across them
    for (int o = lp; o < 32; o *= 2) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        adx[v] += __shfl_xor_sync(0xffffffffu, adx[v], o);
        asg[v] += __shfl_xor_sync(0xffffffffu, asg[v], o);
      }
    }
    if (sub == 0 && jok) {
      float* dxs = dx + s * C + j * V;
      if (VEC) atomicAdd(reinterpret_cast<float4*>(dxs), make_float4(adx[0], adx[1], adx[2], adx[V - 1]));
      else atomicAdd(dxs, adx[0]);
      if (dsig != nullptr) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const int c = j * V + v;
          atomicAdd(dsig + c, 2.f * asg[v] / (s2[c] * __ldg(sigma + c)));
        }
      }
    }
  }
  if (want_ea) {
    __syncwarp();
    for (int p = lane; p < cnt; p += 32) {
      const uint32_t ce = caller_edge(perm, e0 + p);
      const float* pe = ea + static_cast<int64_t>(ce) * k_in;
      float* de = dea + static_cast<int64_t>(ce) * k_in;
      const float sw = es[p][0], su = es[p][1];
      de[0] = -2.f * __ldg(pe) * sw;
      de[1] = -su / (2.f * __ldg(pe + 1));
      de[2] = -su / (2.f * __ldg(pe + 2));
      for (int k = 3; k < k_in; ++k) de[k] = 0.f;
    }
  }
}

size_t gauss_smem_bytes(int C, int arrays) { return static_cast<size_t>(C) * arrays * sizeof(float); }

bool gauss_aligned(const void* a, const void* b, const void* c, const void* d = nullptr) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
           reinterpret_cast<uintptr_t>(d)) & 15) == 0;
}

}  // namespace

size_t gauss_apply_ws_bytes(const Plan* P, int C, int aggr) { return aggr == 2 ? max_keys_bytes(P->N_dst, C) : 1024; }

int apply_gauss(const Plan* P, const float* edge_attr, int k_in, const float* sigma, int C, const float* x,
                const float* root, const float* bias, int aggr, float* out, int* argmax, void* ws, size_t ws_bytes,
                cudaStream_t st, int64_t* launches) {
  NNC_REQUIRE(aggr >= 0 && aggr <= 2, NNCONV_ERR_ARG, "apply_gauss: unknown aggr %d", aggr);
  if (int sb = check_bipartite_root(P, root, 0)) return sb;
  NNC_REQUIRE(C >= 1 && C <= kGaussMaxChannels, NNCONV_ERR_UNSUPPORTED, "apply_gauss: channels %d not in [1, %d]", C,
              kGaussMaxChannels);
  NNC_REQUIRE(k_in >= 3, NNCONV_ERR_ARG, "apply_gauss: edge_attr needs at least 3 columns, got %d", k_in);
  unsigned long long* keys = nullptr;
  if (aggr == 2) {
    NNC_REQUIRE(argmax != nullptr && ws != nullptr && ws_bytes >= max_keys_bytes(P->N_dst, C), NNCONV_ERR_WORKSPACE,
                "apply_gauss: aggr max needs argmax and a workspace of nnconv_gauss_apply_sizes bytes");
    keys = static_cast<unsigned long long*>(ws);
    NNC_CHECK_CUDA(cudaMemsetAsync(keys, 0, sizeof(unsigned long long) * P->N_dst * C, st));
  }
  int s = launch_out_init(x, root, bias, P->N_dst, C, C, out, st, 0);
  if (s) return s;
  int64_t n_l = 1;
  if (P->E > 0 && P->n_tiles > 0) {
    const unsigned grid = static_cast<unsigned>(ceil_div64(static_cast<int64_t>(P->n_tiles) * 32, 256));
    const size_t smem = gauss_smem_bytes(C, 1);
    // 16-byte accesses need x and out rows 16-byte aligned (a caller's x may start at any float)
    const bool vec = C % 4 == 0 && gauss_aligned(x, out, x);
#define NNC_GAUSS_LAUNCH(A, V)                                                                                         \
  k_apply_gauss<A, V><<<grid, 256, smem, st>>>(edge_attr, k_in, sigma, x, C, P->n_tiles, P->tile_c, P->tile_e0,        \
                                               P->tile_cnt, P->src_nodes, P->dst_sorted, P->inv_deg, P->perm, out, keys)
    if (vec) {
      if (aggr == 0) NNC_GAUSS_LAUNCH(0, true);
      else if (aggr == 1) NNC_GAUSS_LAUNCH(1, true);
      else NNC_GAUSS_LAUNCH(2, true);
    } else {
      if (aggr == 0) NNC_GAUSS_LAUNCH(0, false);
      else if (aggr == 1) NNC_GAUSS_LAUNCH(1, false);
      else NNC_GAUSS_LAUNCH(2, false);
    }
#undef NNC_GAUSS_LAUNCH
    NNC_CHECK_LAUNCH();
    ++n_l;
  }
  if (aggr == 2) {
    s = launch_max_finalize(keys, P->N_dst * C, out, argmax, st);
    if (s) return s;
    ++n_l;
  }
  if (launches) *launches += n_l;
  return NNCONV_OK;
}

int backward_gauss(const Plan* P, const float* edge_attr, int k_in, const float* sigma, int C, const float* x,
                   const float* root, int aggr, const int* argmax, const float* gout, float* dx, float* droot,
                   float* dbias, float* dsigma, float* dea, cudaStream_t st, int64_t* launches) {
  NNC_REQUIRE(aggr >= 0 && aggr <= 2 && (aggr != 2 || argmax != nullptr), NNCONV_ERR_ARG,
              "backward_gauss: aggr %d (max needs the forward's argmax)", aggr);
  if (int sb = check_bipartite_root(P, root, 0)) return sb;
  NNC_REQUIRE(C >= 1 && C <= kGaussMaxChannels, NNCONV_ERR_UNSUPPORTED, "backward_gauss: channels %d not in [1, %d]", C,
              kGaussMaxChannels);
  NNC_REQUIRE(k_in >= 3, NNCONV_ERR_ARG, "backward_gauss: edge_attr needs at least 3 columns, got %d", k_in);
  int64_t n_l = 0;
  int s = backward_node_terms(x, root, gout, P->N_dst, C, C, root ? dx : nullptr, droot, dbias, st, &n_l);
  if (s) return s;
  if (root == nullptr) NNC_CHECK_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * P->N_src * C, st));   // dx: the sources
  if (dsigma) NNC_CHECK_CUDA(cudaMemsetAsync(dsigma, 0, sizeof(float) * C, st));
  if (P->E > 0 && P->n_tiles > 0) {
    const unsigned grid = static_cast<unsigned>(ceil_div64(static_cast<int64_t>(P->n_tiles) * 32, 256));
    const size_t smem = gauss_smem_bytes(C, 2);
    const bool vec = C % 4 == 0 && gauss_aligned(x, gout, dx, aggr == 2 ? static_cast<const void*>(argmax) : x);
#define NNC_GAUSS_BWD(A, V)                                                                                            \
  k_bwd_gauss<A, V><<<grid, 256, smem, st>>>(edge_attr, k_in, sigma, x, gout, C, P->n_tiles, P->tile_c, P->tile_e0,    \
                                             P->tile_cnt, P->src_nodes, P->dst_sorted, P->inv_deg, argmax, P->perm, dx, \
                                             dsigma, dea)
    if (vec) {
      if (aggr == 0) NNC_GAUSS_BWD(0, true);
      else if (aggr == 1) NNC_GAUSS_BWD(1, true);
      else NNC_GAUSS_BWD(2, true);
    } else {
      if (aggr == 0) NNC_GAUSS_BWD(0, false);
      else if (aggr == 1) NNC_GAUSS_BWD(1, false);
      else NNC_GAUSS_BWD(2, false);
    }
#undef NNC_GAUSS_BWD
    NNC_CHECK_LAUNCH();
    ++n_l;
  }
  if (launches) *launches += n_l;
  return NNCONV_OK;
}

}  // namespace nnc
