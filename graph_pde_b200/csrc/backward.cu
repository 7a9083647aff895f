// Backward of one NNConv application (SURVEY 8(a) row a11: what autograd generates for
// graph-neural-operator/nn_conv.py:267-282 + utilities.py:223-227), fp32 on CUDA cores, for arbitrary shapes.
// This round's backward is the CORRECTNESS path (it makes the op trainable on the reference's training
// configurations, which are sub-sampled graphs of 10^2..10^3 nodes); it is not the tuned tensor-core path.
//
// With c_n = max(deg_in(n),1) (mean) or 1 (add), g = dL/dout, G_e = g[dst_e] / c_dst_e, and the hoisted /
// reassociated forward of DESIGN.md section 2 (h = MLP without its last Linear W_L,b_L; Y_c = x_c (x) W_L):
//   dbias = sum_n g_n            droot = x^T g               dx  = g root^T
//   dY_c[o,k] = sum_{e in c} G_e[o] h_e[k]                   Gs_c = sum_{e in c} G_e
//   dW_L[i*out+o, k] = sum_c x_c[i] dY_c[o,k]                db_L.view(in,out) = sum_c x_c (x) Gs_c
//   dx_c += dY_c : W_L  +  B_L Gs_c
//   dh_e[k] = sum_o G_e[o] Y_c[o,k]        then the usual MLP backward through ReLU for layers L-1 .. 1,
//   d ea_e  = dz_1[e, :] . W_1             (on request; dh_e[:k_in] for a single-Linear edge network).
// Sources are processed in batches (contiguous sorted edges) so that activations are recomputed and freed
// batch by batch; parameter gradients accumulate across batches.
#include "act.cuh"
#include "kernels.h"

namespace nnc {

namespace {

// C[m,n] = beta*C[m,n] + sum_k A[m*sa_m + k*sa_k] * B[k*sb_k + n*sb_n]      (64x64x16 tiles, 256 threads)
// grouped != nullptr: blockIdx.z = source index in the batch; rows/cols/K and base offsets come from the group.
struct AnyGemm {
  const float* A;
  int64_t sa_m, sa_k;
  const float* B;
  int64_t sb_k, sb_n;
  float* C;
  int64_t ldc;
  int M, N, K;
  float beta;
  // grouped mode
  const int* group_ptr;   // [S+1] sorted-edge offsets
  int c0;                 // first compact source of the batch
  int e_base;             // first sorted edge of the batch (buffers are batch-local)
  int mode;               // 0 plain, 1 = K runs over the group's edges (dY), 2 = M runs over the group's edges (dh)
  int64_t a_group, b_group, c_group;   // per-source strides of A/B/C in elements (mode dependent)
};

__global__ void __launch_bounds__(256) k_sgemm_any(AnyGemm g) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const float* A = g.A;
  const float* B = g.B;
  float* C = g.C;
  int M = g.M, K = g.K;
  if (g.mode != 0) {
    const int c = blockIdx.z;
    const int e0 = g.group_ptr[g.c0 + c] - g.e_base, e1 = g.group_ptr[g.c0 + c + 1] - g.e_base;
    if (g.mode == 1) {          // contraction over the group's edges
      K = e1 - e0;
      A += static_cast<int64_t>(e0) * g.a_group;
      B += static_cast<int64_t>(e0) * g.b_group;
      C += static_cast<int64_t>(c) * g.c_group;
    } else {                    // rows are the group's edges
      M = e1 - e0;
      A += static_cast<int64_t>(e0) * g.a_group;
      B += static_cast<int64_t>(c) * g.b_group;
      C += static_cast<int64_t>(e0) * g.c_group;
    }
  }
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  if (m0 >= M) return;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i / 16, kk = i % 16;
      const int gm = m0 + r, gn = n0 + r, gk = k0 + kk;
      As[kk][r] = (gm < M && gk < K) ? A[gm * g.sa_m + gk * g.sa_k] : 0.f;
      Bs[kk][r] = (gn < g.N && gk < K) ? B[gk * g.sb_k + gn * g.sb_n] : 0.f;
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
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= g.N) continue;
      float* c = C + static_cast<int64_t>(gm) * g.ldc + gn;
      *c = (g.beta != 0.f ? g.beta * *c : 0.f) + acc[i][j];
    }
  }
}

int gemm_any(const float* A, int64_t sa_m, int64_t sa_k, const float* B, int64_t sb_k, int64_t sb_n, float* C,
             int64_t ldc, int M, int N, int K, float beta, cudaStream_t st) {
  if (M <= 0 || N <= 0) return NNCONV_OK;
  AnyGemm g{};
  g.A = A; g.sa_m = sa_m; g.sa_k = sa_k; g.B = B; g.sb_k = sb_k; g.sb_n = sb_n; g.C = C; g.ldc = ldc;
  g.M = M; g.N = N; g.K = K; g.beta = beta; g.mode = 0;
  dim3 grid(ceil_div(M, 64), ceil_div(N, 64), 1);
  k_sgemm_any<<<grid, 256, 0, st>>>(g);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

// G[p, o] = g[dst[p], o] * inv_deg[dst[p]]          (p local to the batch)
// MAX (aggr = max): G[p, o] = g[dst[p], o] if argmax[dst[p], o] is the caller index of edge e0 + p, else 0
template <bool MAX = false>
__global__ void k_gather_g(const float* __restrict__ gout, const int* __restrict__ dst_sorted,
                           const float* __restrict__ inv_deg, int e0, int ne, int cout, float* __restrict__ G,
                           const int* __restrict__ argmax, const int* __restrict__ perm) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(ne) * cout) return;
  const int p = static_cast<int>(i / cout), o = static_cast<int>(i % cout);
  const int d = dst_sorted[e0 + p];
  if constexpr (MAX) {
    const int64_t k = static_cast<int64_t>(d) * cout + o;
    G[i] = static_cast<uint32_t>(argmax[k]) == caller_edge(perm, e0 + p) ? gout[k] : 0.f;
  } else {
    G[i] = gout[static_cast<int64_t>(d) * cout + o] * (inv_deg ? inv_deg[d] : 1.f);
  }
}

// Gs[c, o] = sum over the group's edges of G[p, o]
__global__ void k_group_sum(const float* __restrict__ G, const int* __restrict__ group_ptr, int c0, int e_base,
                            int nb, int cout, float* __restrict__ Gs) {
  const int c = blockIdx.x;
  if (c >= nb) return;
  const int e0 = group_ptr[c0 + c] - e_base, e1 = group_ptr[c0 + c + 1] - e_base;
  for (int o = threadIdx.x; o < cout; o += blockDim.x) {
    float s = 0.f;
    for (int p = e0; p < e1; ++p) s += G[static_cast<int64_t>(p) * cout + o];
    Gs[static_cast<int64_t>(c) * cout + o] = s;
  }
}

// dz = dh * (act > 0), in place; column sums accumulate into db (one block per 32 columns).  k_act_grad_colsum<ACT>
// multiplies by f'(act) of another hidden activation (act.cuh) instead, with its parameter block as the last argument.
template <int ACT>
__device__ __forceinline__ void act_grad_colsum(float* __restrict__ dh, const float* __restrict__ act, int ne, int kp,
                                                float* __restrict__ db, const ActParams& act_p) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  for (int p = threadIdx.y; p < ne; p += 8) {
    if (col < kp) {
      const int64_t i = static_cast<int64_t>(p) * kp + col;
      const float v = ACT == ACT_RELU ? (act[i] > 0.f ? dh[i] : 0.f) : dh[i] * act_grad<ACT>(act[i], act_p);
      dh[i] = v;
      s += v;
    }
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < kp) {
    float t = 0.f;
    for (int r = 0; r < 8; ++r) t += red[r][threadIdx.x];
    db[col] += t;
  }
}

__global__ void k_relu_mask_colsum(float* __restrict__ dh, const float* __restrict__ act, int ne, int kp,
                                   float* __restrict__ db) {
  act_grad_colsum<ACT_RELU>(dh, act, ne, kp, db, ActParams{});
}

template <int ACT>
__global__ void k_act_grad_colsum(float* __restrict__ dh, const float* __restrict__ act, int ne, int kp,
                                  float* __restrict__ db, ActParams act_p) {
  act_grad_colsum<ACT>(dh, act, ne, kp, db, act_p);
}

__global__ void k_gather_ea(const float* __restrict__ edge_attr, const int* __restrict__ perm, int e0, int ne,
                            int k_in, float* __restrict__ out) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(ne) * k_in) return;
  const int p = static_cast<int>(i / k_in), c = static_cast<int>(i % k_in);
  const int64_t src = perm ? perm[e0 + p] : (e0 + p);
  out[i] = edge_attr[src * k_in + c];
}

// grad_edge_attr[perm[e0 + p], i] = sum_{j < kw} dz[p, j] W1[j, i]      (W1 == nullptr: identity features, dz[p, i])
__global__ void k_ea_grad_fp32(const float* __restrict__ dz, int ne, int ld, const float* __restrict__ W1, int kw,
                               int k_in, const int* __restrict__ perm, int e0, float* __restrict__ out) {
  int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<int64_t>(ne) * k_in) return;
  const int p = static_cast<int>(idx / k_in), i = static_cast<int>(idx % k_in);
  const float* row = dz + static_cast<int64_t>(p) * ld;
  float acc = 0.f;
  if (W1 == nullptr) acc = row[i];
  else
    for (int j = 0; j < kw; ++j) acc = fmaf(row[j], W1[static_cast<int64_t>(j) * k_in + i], acc);
  const int64_t e = static_cast<int64_t>(e0) + p;
  out[(perm ? perm[e] : e) * k_in + i] = acc;
}

// dx[src_nodes[c0 + c], i] += dXc[c, i]
__global__ void k_scatter_dx(const float* __restrict__ dXc, const int* __restrict__ src_nodes, int c0, int nb, int cin,
                             int cin_p, float* __restrict__ dx) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(nb) * cin) return;
  const int c = static_cast<int>(i / cin), ii = static_cast<int>(i % cin);
  dx[static_cast<int64_t>(src_nodes[c0 + c]) * cin + ii] += dXc[static_cast<int64_t>(c) * cin_p + ii];
}

// dst[r, c] (R x C, unpadded) = src[r, c] (Rp x Cp padded)
__global__ void k_unpad(const float* __restrict__ src, int Cp, float* __restrict__ dst, int R, int C) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(R) * C) return;
  const int r = static_cast<int>(i / C), c = static_cast<int>(i % C);
  dst[i] = src[static_cast<int64_t>(r) * Cp + c];
}

// dW_L[(i*cout + o), k] = dW3p[(o*Kp + k), i]
__global__ void k_unpermute_w3(const float* __restrict__ dW3p, int cin, int cout, int K, int Kp, int cin_p,
                               float* __restrict__ dWL) {
  int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<int64_t>(cin) * cout * K) return;
  const int k = static_cast<int>(idx % K);
  const int64_t io = idx / K;
  const int o = static_cast<int>(io % cout), i = static_cast<int>(io / cout);
  dWL[idx] = dW3p[(static_cast<int64_t>(o) * Kp + k) * cin_p + i];
}

__global__ void k_colsum_rows(const float* __restrict__ g, int64_t N, int C, float* __restrict__ out) {
  // out[c] = sum_n g[n, c]; one block per column group of 32, 8 row lanes
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  for (int64_t n = threadIdx.y; n < N; n += 8)
    if (col < C) s += g[n * C + col];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < C) {
    float t = 0.f;
    for (int r = 0; r < 8; ++r) t += red[r][threadIdx.x];
    out[col] = t;
  }
}

// dh = the gradient w.r.t. h_{L-1} of the sorted edges [e0, e0 + ne) in cur ([ne, Kp] fp32; nxt: a buffer of the same
// size): back through the hidden layers with the activation derivatives f'(act[1 .. L-1]) (recomputed fp32
// activations; the ReLU mask for ReLU), adding into
// the padded accumulators dW[l], db[l], and, with grad_ea, the gradient w.r.t. the batch's edge_attr rows.  ea: scratch
// of ne * k_in floats.
int mlp_backward_rows(const Plan* P, const Weights* W, const float* edge_attr, int e0, int ne, float* const* act, float* ea,
                      float* cur, float* nxt, float* const* dW, float* const* db, float* grad_ea, cudaStream_t st) {
  const int nl = W->n_layers;
  const int TB = 256;
  int s;
  if (nl >= 2) {
    k_gather_ea<<<(unsigned)ceil_div64(static_cast<int64_t>(ne) * W->kp[0], TB), TB, 0, st>>>(
        edge_attr, P->perm, e0, ne, W->kp[0], ea);
    NNC_CHECK_LAUNCH();
  }
  for (int l = nl - 1; l >= 1; --l) {
    if (W->act.kind == ACT_RELU)
      k_relu_mask_colsum<<<ceil_div(W->kp[l], 32), dim3(32, 8), 0, st>>>(cur, act[l], ne, W->kp[l], db[l]);
    else
      act_dispatch(W->act.kind, [&](auto k) {
        k_act_grad_colsum<decltype(k)::value><<<ceil_div(W->kp[l], 32), dim3(32, 8), 0, st>>>(cur, act[l], ne, W->kp[l],
                                                                                              db[l], W->act.p);
      });
    NNC_CHECK_LAUNCH();
    const float* prev = l == 1 ? ea : act[l - 1];
    const int kprev = W->kp[l - 1];
    // dW_l += dz^T prev
    s = gemm_any(cur, 1, W->kp[l], prev, kprev, 1, dW[l], kprev, W->kp[l], kprev, ne, 1.f, st);
    if (s) return s;
    if (l > 1) {   // dh_{l-1} = dz W_l
      s = gemm_any(cur, W->kp[l], 1, reinterpret_cast<const float*>(W->Wh[l]), kprev, 1, nxt, kprev, ne, kprev,
                   W->kp[l], 0.f, st);
      if (s) return s;
      float* t = cur; cur = nxt; nxt = t;
    }
  }
  // ---- cur = dz_1 (masked, [ne, kp1]) or, for a single Linear, dh ([ne, Kp]): edge_attr rows of the batch
  if (grad_ea != nullptr) {
    k_ea_grad_fp32<<<(unsigned)ceil_div64(static_cast<int64_t>(ne) * W->dims[0], TB), TB, 0, st>>>(
        cur, ne, nl >= 2 ? W->kp[1] : W->Kp, nl >= 2 ? W->W1 : nullptr, nl >= 2 ? W->dims[1] : 0, W->dims[0], P->perm,
        e0, grad_ea);
    NNC_CHECK_LAUNCH();
  }
  return NNCONV_OK;
}

// recomputes the fp32 activations act[1 .. L-1] of the sorted edges [e0, e0 + ne) (a single Linear: the identity
// features into hid) and returns h_{L-1}
const float* recompute_acts_fp32(const Plan* P, const Weights* W, const float* edge_attr, int e0, int ne, float* const* act,
                                 float* hid, cudaStream_t st, int* status) {
  const int nl = W->n_layers;
  int s;
  if (nl == 1) {
    s = launch_edge_layer1(PREC_FP32, edge_attr, P->perm, e0, ne, W->dims[0], nullptr, nullptr, W->Kp, 1, hid, st);
    *status = s;
    return hid;
  }
  s = launch_edge_layer1(PREC_FP32, edge_attr, P->perm, e0, ne, W->dims[0], W->W1, W->b1, W->kp[1], 0, act[1], st, 0, 0,
                         nullptr, W->act);
  for (int l = 2; l <= nl - 1 && s == NNCONV_OK; ++l)
    s = launch_sgemm_store(act[l - 1], W->kp[l - 1], reinterpret_cast<const float*>(W->Wh[l]), W->kp[l - 1], act[l],
                           W->kp[l], ne, W->kp[l], W->kp[l - 1], W->bh[l], st, W->act);
  *status = s;
  return act[nl - 1];
}

struct BwdLayout {
  // persistent over the call (padded fp32 gradient accumulators)
  size_t off_dW[kMaxLayers + 1], off_db[kMaxLayers + 1], off_dW3p, off_dB3, off_Xc, off_cvec;
  size_t fixed;
  // per batch
  size_t per_edge, per_node;
};

BwdLayout bwd_layout(const Plan* P, const Weights* W) {
  Carver c(nullptr, ~size_t(0));
  BwdLayout L{};
  const int nl = W->n_layers;
  for (int l = 1; l <= nl - 1; ++l) {
    L.off_dW[l] = c.off; c.take<float>(static_cast<size_t>(W->kp[l]) * W->kp[l - 1]);
    L.off_db[l] = c.off; c.take<float>(W->kp[l]);
  }
  L.off_dW3p = c.off; c.take<float>(static_cast<size_t>(W->cout) * W->Kp * W->cin_p);
  L.off_dB3 = c.off; c.take<float>(static_cast<size_t>(W->cin) * W->cout);
  const size_t S = P->n_src > 0 ? P->n_src : 1;
  L.off_Xc = c.off; c.take<float>((S + 128) * W->cin_p);
  L.off_cvec = c.off; c.take<float>(S * W->cout);
  L.fixed = c.off;
  size_t acts = 0;
  int maxkp = W->kp[0];
  for (int l = 1; l <= nl - 1; ++l) { acts += W->kp[l]; maxkp = W->kp[l] > maxkp ? W->kp[l] : maxkp; }
  if (nl == 1) acts = W->Kp;
  // activations of every hidden layer + two dh ping-pong buffers + G + gathered edge_attr
  L.per_edge = sizeof(float) * (acts + 2 * static_cast<size_t>(maxkp > W->Kp ? maxkp : W->Kp) + W->cout + W->kp[0]) + 64;
  // Y, dY, Gs, dXc
  L.per_node = sizeof(float) * (2 * static_cast<size_t>(W->cout) * W->Kp + W->cout + W->cin_p) + 64;
  return L;
}

}  // namespace

size_t backward_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes) {
  BwdLayout L = bwd_layout(P, W);
  const size_t per_src = L.per_node + L.per_edge * static_cast<size_t>(P->max_out_deg > 0 ? P->max_out_deg : 1);
  size_t need_min = L.fixed + per_src + 4096;
  size_t all = L.fixed + L.per_node * static_cast<size_t>(P->n_src > 0 ? P->n_src : 1) +
               L.per_edge * static_cast<size_t>(P->E > 0 ? P->E : 1) + 4096;
  size_t w = want_bytes < need_min ? need_min : want_bytes;
  return w < all ? w : all;
}

int backward_fp32(const Plan* P, const Weights* W, const float* edge_attr, const float* x, const float* root,
                  int aggr_mean, const float* gout, float* dx, float* const* dWs, float* const* dbs, float* droot,
                  float* dbias, void* ws, size_t ws_bytes, cudaStream_t st, float* grad_ea, const int* argmax) {
  NNC_REQUIRE(W->prec == PREC_FP32, NNCONV_ERR_ARG, "backward needs weights prepared with precision fp32");
  const int nl = W->n_layers;
  const int cin = W->cin, cout = W->cout, Kp = W->Kp, cin_p = W->cin_p;
  const int64_t N = P->N_dst;   // rows of gout; dx has N_src rows (square plans: the same)
  const int NY = cout * Kp;
  int s = check_bipartite_root(P, root, 0);
  if (s) return s;
  const int TB = 256;
  // ---- node-level terms: dbias, droot, dx = g root^T
  if (dbias) {
    k_colsum_rows<<<ceil_div(cout, 32), dim3(32, 8), 0, st>>>(gout, N, cout, dbias);
    NNC_CHECK_LAUNCH();
  }
  if (root != nullptr) {
    // droot[i,o] = sum_n x[n,i] g[n,o]
    s = gemm_any(x, 1, cin, gout, cout, 1, droot, cout, cin, cout, static_cast<int>(N), 0.f, st);
    if (s) return s;
    // dx[n,i] = sum_o g[n,o] root[i,o]
    s = gemm_any(gout, cout, 1, root, 1, cout, dx, cin, static_cast<int>(N), cin, cout, 0.f, st);
    if (s) return s;
  } else {
    NNC_CHECK_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * P->N_src * cin, st));
  }
  BwdLayout L = bwd_layout(P, W);
  NNC_REQUIRE(ws != nullptr && ws_bytes >= L.fixed, NNCONV_ERR_WORKSPACE, "backward: workspace too small");
  char* base = static_cast<char*>(ws);
  NNC_CHECK_CUDA(cudaMemsetAsync(base, 0, L.fixed, st));      // zero every accumulator
  float* dW3p = reinterpret_cast<float*>(base + L.off_dW3p);
  float* dB3 = reinterpret_cast<float*>(base + L.off_dB3);
  float* Xc = reinterpret_cast<float*>(base + L.off_Xc);
  float* cvec = reinterpret_cast<float*>(base + L.off_cvec);
  if (P->E > 0 && P->n_src > 0) {
    s = launch_src_prep(PREC_FP32, x, P->src_nodes, P->n_src, cin, cin_p, cout, W->B3, Xc, cvec, nullptr, st);
    if (s) return s;
    // batch of sources bounded by the workspace
    const int* hgp = P->h_group_ptr;
    size_t avail = ws_bytes - L.fixed;
    int c0 = 0;
    while (c0 < P->n_src) {
      int c1 = c0;
      size_t used = 0;
      while (c1 < P->n_src && c1 - c0 < 65535) {    // the grouped GEMMs put the source index on grid.z (<= 65535)
        const size_t add = L.per_node + L.per_edge * static_cast<size_t>(hgp[c1 + 1] - hgp[c1]);
        if (used + add + 4096 > avail && c1 > c0) break;
        NNC_REQUIRE(used + add + 4096 <= avail, NNCONV_ERR_WORKSPACE, "backward: workspace too small for one source group");
        used += add;
        ++c1;
      }
      const int nb = c1 - c0, e0 = hgp[c0], ne = hgp[c1] - hgp[c0];
      Carver cv(base + L.fixed, avail);
      float* act[kMaxLayers + 1] = {nullptr};
      for (int l = 1; l <= nl - 1; ++l) act[l] = cv.take<float>(static_cast<size_t>(ne) * W->kp[l]);
      int maxkp = Kp;
      for (int l = 1; l <= nl - 1; ++l) maxkp = W->kp[l] > maxkp ? W->kp[l] : maxkp;
      float* hid = nl == 1 ? cv.take<float>(static_cast<size_t>(ne) * Kp) : nullptr;   // identity features
      float* dhA = cv.take<float>(static_cast<size_t>(ne) * maxkp);
      float* dhB = cv.take<float>(static_cast<size_t>(ne) * maxkp);
      float* G = cv.take<float>(static_cast<size_t>(ne) * cout);
      float* ea = cv.take<float>(static_cast<size_t>(ne) * W->kp[0]);
      float* Y = cv.take<float>(static_cast<size_t>(nb) * NY);
      float* dY = cv.take<float>(static_cast<size_t>(nb) * NY);
      float* Gs = cv.take<float>(static_cast<size_t>(nb) * cout);
      float* dXc = cv.take<float>(static_cast<size_t>(nb) * cin_p);
      NNC_REQUIRE(cv.ok(), NNCONV_ERR_WORKSPACE, "backward: workspace carve overflow");
      // ---- recompute the edge features of this batch (fp32)
      const float* h = recompute_acts_fp32(P, W, edge_attr, e0, ne, act, hid, st, &s);
      if (s) return s;
      // ---- Y of the batch
      s = launch_sgemm_store(Xc + static_cast<int64_t>(c0) * cin_p, cin_p, reinterpret_cast<const float*>(W->W3p), cin_p,
                             Y, NY, nb, NY, cin_p, nullptr, st);
      if (s) return s;
      // ---- G, Gs
      if (argmax != nullptr)
        k_gather_g<true><<<(unsigned)ceil_div64(static_cast<int64_t>(ne) * cout, TB), TB, 0, st>>>(
            gout, P->dst_sorted, nullptr, e0, ne, cout, G, argmax, P->perm);
      else
        k_gather_g<<<(unsigned)ceil_div64(static_cast<int64_t>(ne) * cout, TB), TB, 0, st>>>(
            gout, P->dst_sorted, aggr_mean ? P->inv_deg : nullptr, e0, ne, cout, G, nullptr, nullptr);
      NNC_CHECK_LAUNCH();
      k_group_sum<<<nb, 64, 0, st>>>(G, P->group_ptr, c0, e0, nb, cout, Gs);
      NNC_CHECK_LAUNCH();
      // ---- dY_c = G_c^T h_c   (grouped, K = edges of the group)
      {
        AnyGemm g{};
        g.A = G; g.sa_m = 1; g.sa_k = cout; g.B = h; g.sb_k = Kp; g.sb_n = 1; g.C = dY; g.ldc = Kp;
        g.M = cout; g.N = Kp; g.K = 0; g.beta = 0.f; g.mode = 1; g.group_ptr = P->group_ptr; g.c0 = c0; g.e_base = e0;
        g.a_group = cout; g.b_group = Kp; g.c_group = NY;
        dim3 grid(ceil_div(cout, 64), ceil_div(Kp, 64), nb);
        k_sgemm_any<<<grid, 256, 0, st>>>(g);
        NNC_CHECK_LAUNCH();
      }
      // ---- dW3p += dY^T Xc ; dB3 += Xc^T Gs
      s = gemm_any(dY, 1, NY, Xc + static_cast<int64_t>(c0) * cin_p, cin_p, 1, dW3p, cin_p, NY, cin_p, nb, 1.f, st);
      if (s) return s;
      s = gemm_any(Xc + static_cast<int64_t>(c0) * cin_p, 1, cin_p, Gs, cout, 1, dB3, cout, cin, cout, nb, 1.f, st);
      if (s) return s;
      // ---- dXc = dY W3p + Gs B3^T ; scatter into dx
      s = gemm_any(dY, NY, 1, reinterpret_cast<const float*>(W->W3p), cin_p, 1, dXc, cin_p, nb, cin_p, NY, 0.f, st);
      if (s) return s;
      s = gemm_any(Gs, cout, 1, W->B3, 1, cout, dXc, cin_p, nb, cin, cout, 1.f, st);
      if (s) return s;
      k_scatter_dx<<<(unsigned)ceil_div64(static_cast<int64_t>(nb) * cin, TB), TB, 0, st>>>(dXc, P->src_nodes, c0, nb, cin,
                                                                                          cin_p, dx);
      NNC_CHECK_LAUNCH();
      if (nl >= 2 || grad_ea != nullptr) {
        // ---- dh = G_c Y_c (grouped, rows = edges of the group); with a single Linear (identity features) the
        // gradient w.r.t. edge_attr is its first k_in columns
        {
          AnyGemm g{};
          g.A = G; g.sa_m = cout; g.sa_k = 1; g.B = Y; g.sb_k = Kp; g.sb_n = 1; g.C = dhA; g.ldc = Kp;
          g.M = 0; g.N = Kp; g.K = cout; g.beta = 0.f; g.mode = 2; g.group_ptr = P->group_ptr; g.c0 = c0; g.e_base = e0;
          g.a_group = cout; g.b_group = NY; g.c_group = Kp;
          dim3 grid(ceil_div(P->max_out_deg, 64), ceil_div(Kp, 64), nb);
          k_sgemm_any<<<grid, 256, 0, st>>>(g);
          NNC_CHECK_LAUNCH();
        }
        // ---- MLP backward through the hidden layers
        float* dWp[kMaxLayers + 1] = {nullptr};
        float* dbp[kMaxLayers + 1] = {nullptr};
        for (int l = 1; l <= nl - 1; ++l) {
          dWp[l] = reinterpret_cast<float*>(base + L.off_dW[l]);
          dbp[l] = reinterpret_cast<float*>(base + L.off_db[l]);
        }
        s = mlp_backward_rows(P, W, edge_attr, e0, ne, act, ea, dhA, dhB, dWp, dbp, grad_ea, st);
        if (s) return s;
      }
      c0 = c1;
    }
  }
  // ---- un-pad / un-permute the parameter gradients into the caller's tensors
  for (int l = 1; l <= nl - 1; ++l) {
    const int R = W->dims[l], C = W->dims[l - 1];
    k_unpad<<<(unsigned)ceil_div64(static_cast<int64_t>(R) * C, TB), TB, 0, st>>>(
        reinterpret_cast<const float*>(base + L.off_dW[l]), W->kp[l - 1], dWs[l - 1], R, C);
    NNC_CHECK_LAUNCH();
    k_unpad<<<ceil_div(R, TB), TB, 0, st>>>(reinterpret_cast<const float*>(base + L.off_db[l]), R, dbs[l - 1], 1, R);
    NNC_CHECK_LAUNCH();
  }
  k_unpermute_w3<<<(unsigned)ceil_div64(static_cast<int64_t>(cin) * cout * W->K, TB), TB, 0, st>>>(
      dW3p, cin, cout, W->K, Kp, cin_p, dWs[nl - 1]);
  NNC_CHECK_LAUNCH();
  NNC_CHECK_CUDA(cudaMemcpyAsync(dbs[nl - 1], dB3, sizeof(float) * cin * cout, cudaMemcpyDeviceToDevice, st));
  return NNCONV_OK;
}

// ------------------------------------------------------------------------------------------------
// diagonal-kernel conv (formulation D, diag.cu).  Per application, with G_e = g[dst_e] * inv_deg[dst_e] (mean), g[dst_e]
// (add) or g[dst_e] masked by the forward's argmax (max):
//   dx_n = g_n root^T + sum_{e: src_e = n} G_e * d_e          dd_e += x_src(e) * G_e   (summed over the applications)
// and once per (edge_attr, parameters): dW_L = dd^T h, db_L = sum_e dd_e, dh = dd W_L, then the hidden layers.
// ------------------------------------------------------------------------------------------------
namespace {

// one warp per plan tile (one source): lane o of each 32-channel block keeps x_src[o] and the tile's dx sum in registers
// (dd nullable: no gradient reaches the edge network)
template <int AGGR>
__global__ void __launch_bounds__(256) k_bwd_diag_edges(const float* __restrict__ d, const float* __restrict__ x,
                                                        const float* __restrict__ gout, int cout, int n_tiles,
                                                        const int* __restrict__ tile_c, const int* __restrict__ tile_e0,
                                                        const int* __restrict__ tile_cnt, const int* __restrict__ src_nodes,
                                                        const int* __restrict__ dst_sorted,
                                                        const float* __restrict__ inv_deg, const int* __restrict__ argmax,
                                                        const int* __restrict__ perm, float* __restrict__ dx,
                                                        float* __restrict__ dd) {
  const int t = static_cast<int>((blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const int e0 = tile_e0[t], cnt = tile_cnt[t];
  const int64_t s = src_nodes[tile_c[t]];
  for (int o = lane; o < cout; o += 32) {
    const float xv = x[s * cout + o];
    float acc = 0.f;
    for (int p = 0; p < cnt; ++p) {
      const int64_t e = e0 + p;
      const int dn = dst_sorted[e];
      const int64_t k = static_cast<int64_t>(dn) * cout + o;
      float g = gout[k];
      if (AGGR == 1) g *= inv_deg[dn];
      if (AGGR == 2 && static_cast<uint32_t>(argmax[k]) != caller_edge(perm, e)) g = 0.f;
      acc = fmaf(g, d[e * cout + o], acc);
      if (dd != nullptr) dd[e * cout + o] += xv * g;
    }
    atomicAdd(dx + s * cout + o, acc);
  }
}

// out[c] += sum_n g[n, c]
__global__ void k_colsum_rows_add(const float* __restrict__ g, int64_t N, int C, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  for (int64_t n = threadIdx.y; n < N; n += 8)
    if (col < C) s += g[n * C + col];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < C) {
    float t = 0.f;
    for (int r = 0; r < 8; ++r) t += red[r][threadIdx.x];
    out[col] += t;
  }
}

constexpr size_t kDiagCarveSlack = 16 * 1024;

struct DiagBwdLayout {
  size_t off_dW[kMaxLayers + 1], off_db[kMaxLayers + 1], off_dWL, off_dbL, fixed, per_edge;
};

DiagBwdLayout diag_bwd_layout(const Weights* W) {
  Carver c(nullptr, ~size_t(0));
  DiagBwdLayout L{};
  const int nl = W->n_layers;
  for (int l = 1; l <= nl - 1; ++l) {
    L.off_dW[l] = c.off; c.take<float>(static_cast<size_t>(W->kp[l]) * W->kp[l - 1]);
    L.off_db[l] = c.off; c.take<float>(W->kp[l]);
  }
  L.off_dWL = c.off; c.take<float>(static_cast<size_t>(W->cout) * W->Kp);
  L.off_dbL = c.off; c.take<float>(W->cout);
  L.fixed = c.off;
  size_t acts = 0;
  int maxkp = W->Kp;
  for (int l = 1; l <= nl - 1; ++l) { acts += W->kp[l]; maxkp = W->kp[l] > maxkp ? W->kp[l] : maxkp; }
  if (nl == 1) acts = W->Kp;
  // activations of every hidden layer + two dh ping-pong buffers + gathered edge_attr
  L.per_edge = sizeof(float) * (acts + 2 * static_cast<size_t>(maxkp) + W->kp[0]);
  return L;
}

}  // namespace

int backward_node_terms(const float* x, const float* root, const float* gout, int64_t N, int cin, int cout, float* dx,
                        float* droot, float* dbias, cudaStream_t st, int64_t* launches) {
  if (dbias) {
    k_colsum_rows<<<ceil_div(cout, 32), dim3(32, 8), 0, st>>>(gout, N, cout, dbias);
    NNC_CHECK_LAUNCH();
    ++*launches;
  }
  if (root != nullptr) {
    int s = gemm_any(x, 1, cin, gout, cout, 1, droot, cout, cin, cout, static_cast<int>(N), 0.f, st);   // droot = x^T g
    if (s) return s;
    s = gemm_any(gout, cout, 1, root, 1, cout, dx, cin, static_cast<int>(N), cin, cout, 0.f, st);       // dx = g root^T
    if (s) return s;
    *launches += 2;
  }
  return NNCONV_OK;
}

int backward_apply_diag(const Plan* P, const Weights* W, const float* d, const float* x, const float* root, int aggr,
                        const int* argmax, const float* gout, float* dx, float* droot, float* dbias, float* dd,
                        cudaStream_t st, int64_t* launches) {
  NNC_REQUIRE(W->diag, NNCONV_ERR_ARG, "backward_apply_diag: weights not prepared as a diagonal kernel");
  NNC_REQUIRE(aggr >= 0 && aggr <= 2 && (aggr != 2 || argmax != nullptr), NNCONV_ERR_ARG,
              "backward_apply_diag: aggr %d (max needs the forward's argmax)", aggr);
  const int C = W->cout;
  int64_t n_l = 0;
  if (int sb = check_bipartite_root(P, root, 0)) return sb;
  const int s = backward_node_terms(x, root, gout, P->N_dst, C, C, root ? dx : nullptr, droot, dbias, st, &n_l);
  if (s) return s;
  if (root == nullptr) NNC_CHECK_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * P->N_src * C, st));   // dx: the sources
  if (P->E > 0 && P->n_tiles > 0) {
    const unsigned grid = static_cast<unsigned>(ceil_div64(static_cast<int64_t>(P->n_tiles) * 32, 256));
#define NNC_DIAG_BWD(A)                                                                                               \
  k_bwd_diag_edges<A><<<grid, 256, 0, st>>>(d, x, gout, C, P->n_tiles, P->tile_c, P->tile_e0, P->tile_cnt, P->src_nodes, \
                                            P->dst_sorted, P->inv_deg, argmax, P->perm, dx, dd)
    if (aggr == 0) NNC_DIAG_BWD(0);
    else if (aggr == 1) NNC_DIAG_BWD(1);
    else NNC_DIAG_BWD(2);
#undef NNC_DIAG_BWD
    NNC_CHECK_LAUNCH();
    ++n_l;
  }
  if (launches) *launches += n_l;
  return NNCONV_OK;
}

size_t backward_mlp_diag_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes) {
  const DiagBwdLayout L = diag_bwd_layout(W);
  const size_t need_min = L.fixed + L.per_edge * 128 + kDiagCarveSlack;
  const size_t all = L.fixed + L.per_edge * static_cast<size_t>(P->E > 0 ? P->E : 1) + kDiagCarveSlack;
  size_t w = want_bytes < need_min ? need_min : want_bytes;
  return w < all ? w : all;
}

int backward_mlp_diag(const Plan* P, const Weights* W, const float* edge_attr, const float* dd, float* const* dWs,
                      float* const* dbs, void* ws, size_t ws_bytes, cudaStream_t st, float* grad_ea) {
  NNC_REQUIRE(W->diag && W->prec == PREC_FP32, NNCONV_ERR_ARG,
              "backward_mlp_diag: needs diagonal weights prepared with precision fp32");
  const int nl = W->n_layers, C = W->cout, Kp = W->Kp;
  const DiagBwdLayout L = diag_bwd_layout(W);
  NNC_REQUIRE(ws != nullptr && ws_bytes >= L.fixed + L.per_edge * 128 + kDiagCarveSlack, NNCONV_ERR_WORKSPACE,
              "backward_mlp_diag: workspace too small");
  char* base = static_cast<char*>(ws);
  NNC_CHECK_CUDA(cudaMemsetAsync(base, 0, L.fixed, st));
  float* dWL = reinterpret_cast<float*>(base + L.off_dWL);
  float* dbL = reinterpret_cast<float*>(base + L.off_dbL);
  float* dWp[kMaxLayers + 1] = {nullptr};
  float* dbp[kMaxLayers + 1] = {nullptr};
  for (int l = 1; l <= nl - 1; ++l) {
    dWp[l] = reinterpret_cast<float*>(base + L.off_dW[l]);
    dbp[l] = reinterpret_cast<float*>(base + L.off_db[l]);
  }
  const size_t avail = ws_bytes - L.fixed;
  int64_t rows = static_cast<int64_t>((avail - kDiagCarveSlack) / L.per_edge);   // slack: the carver's 1 KiB rounding
  if (rows > P->E) rows = P->E;
  int s;
  for (int64_t e0 = 0; e0 < P->E; e0 += rows) {
    const int ne = static_cast<int>(P->E - e0 < rows ? P->E - e0 : rows);
    Carver cv(base + L.fixed, avail);
    float* act[kMaxLayers + 1] = {nullptr};
    for (int l = 1; l <= nl - 1; ++l) act[l] = cv.take<float>(static_cast<size_t>(ne) * W->kp[l]);
    int maxkp = Kp;
    for (int l = 1; l <= nl - 1; ++l) maxkp = W->kp[l] > maxkp ? W->kp[l] : maxkp;
    float* hid = nl == 1 ? cv.take<float>(static_cast<size_t>(ne) * Kp) : nullptr;
    float* dhA = cv.take<float>(static_cast<size_t>(ne) * maxkp);
    float* dhB = cv.take<float>(static_cast<size_t>(ne) * maxkp);
    float* ea = cv.take<float>(static_cast<size_t>(ne) * W->kp[0]);
    NNC_REQUIRE(cv.ok(), NNCONV_ERR_WORKSPACE, "backward_mlp_diag: workspace carve overflow");
    const float* h = recompute_acts_fp32(P, W, edge_attr, static_cast<int>(e0), ne, act, hid, st, &s);
    if (s) return s;
    const float* ddb = dd + e0 * C;
    // dW_L += dd^T h ; db_L += sum_e dd_e ; dh = dd W_L
    s = gemm_any(ddb, 1, C, h, Kp, 1, dWL, Kp, C, Kp, ne, 1.f, st);
    if (s) return s;
    k_colsum_rows_add<<<ceil_div(C, 32), dim3(32, 8), 0, st>>>(ddb, ne, C, dbL);
    NNC_CHECK_LAUNCH();
    s = gemm_any(ddb, C, 1, static_cast<const float*>(W->W3n), Kp, 1, dhA, Kp, ne, Kp, C, 0.f, st);
    if (s) return s;
    s = mlp_backward_rows(P, W, edge_attr, static_cast<int>(e0), ne, act, ea, dhA, dhB, dWp, dbp, grad_ea, st);
    if (s) return s;
  }
  const int TB = 256;
  for (int l = 1; l <= nl - 1; ++l) {
    const int R = W->dims[l], Cl = W->dims[l - 1];
    k_unpad<<<(unsigned)ceil_div64(static_cast<int64_t>(R) * Cl, TB), TB, 0, st>>>(dWp[l], W->kp[l - 1], dWs[l - 1], R, Cl);
    NNC_CHECK_LAUNCH();
    k_unpad<<<ceil_div(R, TB), TB, 0, st>>>(dbp[l], R, dbs[l - 1], 1, R);
    NNC_CHECK_LAUNCH();
  }
  k_unpad<<<(unsigned)ceil_div64(static_cast<int64_t>(C) * W->K, TB), TB, 0, st>>>(dWL, Kp, dWs[nl - 1], C, W->K);
  NNC_CHECK_LAUNCH();
  NNC_CHECK_CUDA(cudaMemcpyAsync(dbs[nl - 1], dbL, sizeof(float) * C, cudaMemcpyDeviceToDevice, st));
  return NNCONV_OK;
}

}  // namespace nnc
