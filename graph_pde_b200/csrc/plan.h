// Internal (C++) view of the opaque handles exported through include/nnconv_b200.h.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace nnc {

constexpr int kMaxLayers = 8;

enum Precision : int { PREC_FP32 = 0, PREC_F16 = 1, PREC_BF16 = 2, PREC_F16X2 = 3 };
// PREC_F16X2: every tensor-core operand is carried as an fp16 pair (hi, lo) with hi = fp16(v), lo = fp16(v - hi)
// (~22 mantissa bits) and every product as hi*hi + hi*lo + lo*hi in the fp32 accumulator: fp32-grade results on
// the fp16 tensor pipe at 3x the MMA work and 2x the activation bytes.
inline bool prec_is_bf16(int prec) { return prec == PREC_BF16; }
inline bool prec_is_split(int prec) { return prec == PREC_F16X2; }

struct Plan {
  int64_t E;
  // node counts of the two roles: sources (x rows gathered by the messages) and targets (rows of out).  A square plan
  // has N_src == N_dst; a bipartite one (DESIGN 4.10) maps x_src [N_src, in] to out [N_dst, out]
  int64_t N_src, N_dst;
  int flow;
  int n_src;        // S: sources with at least one out-edge (compact index c in [0,S))
  int n_tiles;      // T: tiles of <= 128 edges, never spanning two sources
  int max_out_deg;
  int src_sorted;   // caller's edge list was already grouped by source (perm == identity, not stored)
  const int* perm;        // [E] sorted position -> original edge id, nullptr = identity
  const int* dst_sorted;  // [E]
  const int* src_nodes;   // [S] node id of compact source c
  const int* group_ptr;   // [S+1] first sorted edge of source c
  const int* tile_ptr;    // [S+1] first tile of source c
  const int* tile_c;      // [T]
  const int* tile_e0;     // [T]
  const int* tile_cnt;    // [T]
  const int* unit_ptr;    // [S+1] first unit of source c (unit = <= 2 consecutive tiles of one source)
  const int* unit_t;      // [U] first tile of the unit
  const int* unit_u;      // [U] tiles in the unit (1 or 2)
  int n_units;
  const float* inv_deg;   // [N_dst] 1/max(in_degree,1)
  const int* h_tile_ptr;  // HOST mirror of tile_ptr ([S+1]) owned by the C handle
  const int* h_group_ptr; // HOST mirror of group_ptr ([S+1]) owned by the C handle
  const int* h_unit_ptr;  // HOST copy of unit_ptr ([S+1]) owned by the C handle
};

void plan_sizes(int64_t E, int64_t N_src, int64_t N_dst, size_t* ws_bytes, size_t* tmp_bytes);
int plan_build(Plan* P, const int64_t* row0, const int64_t* row1, int64_t E, int64_t N_src, int64_t N_dst, int flow, void* ws,
               size_t ws_bytes, void* tmp, size_t tmp_bytes, cudaStream_t st);
// a bipartite plan (N_src != N_dst) takes root = NULL and no NNCONV_APPLY_RESIDUAL in the message entry points of every
// conv (NNConv, diagonal, Gaussian): the root term reads x_dst, not x_src (root_term / node_terms_rows)
int check_bipartite_root(const Plan* P, const float* root, unsigned node_flags);

// parameter block of the edge MLP's hidden activation (act.cuh); act_grad reads v[0 .. 2] only, unused entries are 0:
//   NNCONV_ACT_LEAKY_RELU  v[0] = slope
//   NNCONV_ACT_ELU         v[0] = alpha
//   NNCONV_ACT_CLAMP       v = a, lo_img, hi_img, b, lo, hi   (the bounds' images in the weights' storage format)
//   NNCONV_ACT_SCALED_ELU  v = lambda, c, lambda * alpha, alpha
constexpr int kActParams = 6;
struct ActParams {
  float v[kActParams];
};

// hidden activation of the edge MLP: kind = NNCONV_ACT_* (0 = ReLU) and its parameter block
struct Act {
  int kind;
  ActParams p;
};

// Prepared (padded / permuted / down-converted) snapshot of the edge-MLP parameters.
struct Weights {
  int n_layers;                 // Linear layers of the edge MLP (DenseNet)
  int dims[kMaxLayers + 1];     // k_in, k_1, ..., cin*cout
  int kp[kMaxLayers + 1];       // padded widths (multiples of 64) of the activations h_1 .. h_{L-1}; kp[0] = k_in
  int cin, cout, cin_p;
  int K, Kp;                    // width of the hoisted per-edge feature h_last (= dims[L-1]) and its padding
  int prec;
  int split;                    // PREC_F16X2: activations are [hi | lo] pairs (2 x width), weights [hi | lo | hi] (3 x K)
  size_t esize;                 // bytes per element of activations / tensor-core operands
  const float* W1;              // [kp[1], k_in] fp32 (zero padded rows); nullptr when n_layers == 1
  const float* b1;              // [kp[1]]
  const void* W1aug;            // [kp[1], 64] in `prec`: split hi/lo first layer incl. bias (tensor-core path), or nullptr
  const void* Wh[kMaxLayers];   // hidden layers l = 2 .. L-1: [kp[l], kp[l-1]] in `prec` (split: [kp[l], 3*kp[l-1]])
  const float* bh[kMaxLayers];  // [kp[l]] fp32
  const void* W3p;              // [cout*Kp, cin_p] in `prec`:  W3p[(o*Kp + k), i] = W_L[i*cout + o, k] (split: 3*cin_p columns)
  const float* B3;              // [cin, cout] fp32 = b_L viewed (in, out)
  // extra images for the tensor-core backward (16-bit precisions; PREC_F16X2: split [hi | lo | hi] along the reduction
  // dimension and pre-scaled by wscale like W3p / Wh; nullptr when the backward does not cover the shape)
  // PREC_F16X2: every split weight matrix is stored multiplied by a power of two that brings its largest entry
  // into [0.5, 1) -- the lo halves of U(+-1/32)-sized weights would otherwise be fp16 subnormals (8 instead of 11
  // bits) -- and the epilogue multiplies the fp32 accumulator by the inverse.  wscale[2*l] = scale of layer l's
  // matrix (l = n_layers: the last Linear), wscale[2*l + 1] = its inverse; device floats, nullptr when not split.
  const float* wscale;
  const void* W3n;              // [cin*cout, Kp]: the last Linear in its own layout, padded (per-edge kernel matrices)
  const void* W3q;              // [Kp*cout, cin_p]:  W3q[(k*cout + o), i] = W_L[i*cout + o, k]   (Y^T rows per source; split: 3*cin_p)
  const void* W3t;              // [cin_p, Kp*cout]:  W3t[i, (k*cout + o)] = W_L[i*cout + o, k]   (dx = dY : W_L; split: 3*Kp*cout)
  const void* WhT[kMaxLayers];  // hidden layers l = 2 .. L-1 transposed: [kp[l-1], kp[l]]  (dz_{l-1} = dz_l W_l; split: 3*kp[l])
  // diagonal-kernel conv (formulation D, DESIGN 4.7): the last Linear maps h to one value per channel, d_e = W_L h_e +
  // b_L with cin == cout == dims[L].  Only the hidden layers, W3n and B3 are prepared: W3n = W_L [cout, Kp] zero padded,
  // 16-bit at f16 / bf16 (tensor-core build of d), fp32 at f16x2 and fp32 (CUDA-core build); B3 = b_L [cout] fp32.
  int diag;
  Act act;                      // hidden activation of the edge MLP, see act.cuh
};

size_t weights_bytes(int n_layers, const int* dims, int cin, int cout, int prec, int diag = 0);
int weights_prepare(Weights* W, int n_layers, const int* dims, int cin, int cout, int prec,
                    const float* const* Wsrc, const float* const* bsrc, void* buf, size_t buf_bytes,
                    cudaStream_t st, int diag = 0);

// edge features: h_last[p, :] for every sorted edge p  (x-independent prefix of the edge MLP)
size_t edge_features_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes);
// acts (nullable, training): keeps the hidden activations h_1 .. h_{L-2} of ALL edges (16-bit row-major, layer l at
// edge_acts_offset(l)) instead of recycling them chunk by chunk, so that the backward need not recompute them
size_t edge_acts_bytes(const Plan* P, const Weights* W);
size_t edge_acts_offset(const Plan* P, const Weights* W, int l);
// n_edges >= 0: only the sorted edges [0, n_edges) (a unit boundary), into panels of round_up(n_edges, 128) rows
int edge_features(const Plan* P, const Weights* W, const float* edge_attr, void* h, void* ws, size_t ws_bytes,
                  cudaStream_t st, int64_t* launches, void* acts = nullptr, int64_t n_edges = -1);

// one conv application given h_last of every edge: apply_streamed's application with E_res = E (one driver, api.cu)
size_t apply_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes);
int apply(const Plan* P, const Weights* W, const void* h, const float* x, const float* root, const float* bias,
          int aggr_mean, float* out, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches,
          unsigned node_flags = 0);

// partially resident edge features (16-bit precisions): the edge features of the sorted edges [0, E_res) are cached by
// the caller (edge_features with n_edges = E_res), those of [E_res, E) are recomputed chunk by chunk inside every
// application, each chunk contracted as the resident prefix is.  stream_split picks the largest unit-aligned E_res whose h fits resident_bytes and sizes the workspace
// of apply_streamed for chunks of chunk_ws_bytes (h rows + edge-feature workspace).
int stream_split(const Plan* P, const Weights* W, size_t resident_bytes, size_t chunk_ws_bytes, int64_t* E_res,
                 size_t* h_res_bytes, size_t* ws_bytes, int64_t* n_chunks);
bool is_unit_boundary(const Plan* P, int64_t e);
// h of the sorted edges [e_begin, e_begin + E) into the chunk-major panels of round_up(E, 128) rows at h (padding rows
// zeroed); ws: scratch of ef_row_bytes(W) per row plus 4096 bytes; overflow and launches nullable, acts as above
int edge_features_rows(const Plan* P, const Weights* W, const float* edge_attr, int64_t e_begin, int64_t E, void* h,
                       void* ws, size_t ws_bytes, int* overflow, cudaStream_t st, int64_t* launches, void* acts);
size_t ef_row_bytes(const Weights* W);
size_t h_row_bytes(const Weights* W);      // bytes of one edge's cached h (16-bit: Kp * 2, twice that at f16x2)
int apply_streamed(const Plan* P, const Weights* W, const float* edge_attr, const void* h_res, int64_t E_res,
                   const float* x, const float* root, const float* bias, int aggr_mean, float* out, void* ws,
                   size_t ws_bytes, cudaStream_t st, int64_t* launches, unsigned node_flags,
                   unsigned long long* max_keys = nullptr, int* argmax = nullptr);
// aggr = max (DESIGN 5): the application of h_res / E_res (E_res = E: a whole h, else apply_streamed's chunks) with
// ws = [max_keys_bytes(N, cout) of keys | the add / mean workspace]; writes out and argmax [N, cout] (caller edge
// indices, -1 for a node without in-edges)
int apply_max(const Plan* P, const Weights* W, const float* edge_attr, const void* h_res, int64_t E_res, const float* x,
              const float* root, const float* bias, float* out, int* argmax, void* ws, size_t ws_bytes, cudaStream_t st,
              int64_t* launches, unsigned node_flags);

// tensor-core backward (backward_tc.cu): per application (dx, dW_L, db_L, droot, dbias) and, once per
// (edge_attr, parameters) for all T applications of a shared conv, the pass through the hidden layers.
// grad_ea (nullable): [E, k_in] fp32 in the caller's edge order, WRITTEN -- the gradient w.r.t. edge_attr.
// h holds the edge features of the sorted edges [0, E_res) (a unit boundary; E_res = E: the whole cached h).  With
// E_res < E the h of the other edges is recomputed from edge_attr per source batch into a chunk buffer of the
// workspace (backward_*_ws_bytes with that E_res), and kept activations (acts) are not used.
bool backward_tc_supported(const Weights* W);
size_t backward_apply_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes, int64_t E_res = -1,
                               size_t chunk_ws_bytes = 0);
int backward_apply_tc(const Plan* P, const Weights* W, const float* edge_attr, const void* h, int64_t E_res,
                      const float* x, const float* root, int aggr_mean, const float* gout, float* dx, float* dWL,
                      float* dbL, float* droot, float* dbias, void* ws, size_t ws_bytes, cudaStream_t st,
                      int64_t* launches = nullptr, const int* argmax = nullptr);
size_t backward_mlp_ws_bytes(const Plan* P, const Weights* W, int T, size_t want_bytes, int64_t E_res = -1);
int backward_mlp_tc(const Plan* P, const Weights* W, const float* edge_attr, const void* h, int64_t E_res, int T,
                    const float* const* gouts, const float* const* xs_in, int aggr_mean, float* const* dWs,
                    float* const* dbs, void* ws, size_t ws_bytes, cudaStream_t st, const void* acts = nullptr,
                    float* grad_ea = nullptr, const int* const* argmax = nullptr);
// source batches whose edge features the call with this workspace recomputes (T = 0: backward_apply_tc)
int64_t backward_streamed_chunks(const Plan* P, const Weights* W, int T, int64_t E_res, size_t ws_bytes);

// per-edge kernel matrices for low out-degree graphs (formulation B): Kmat [E, cin*cout] 16-bit in sorted edge order
size_t edge_kernels_bytes(const Plan* P, const Weights* W);
bool edge_kernels_supported(const Weights* W);
int edge_kernels(const Plan* P, const Weights* W, const void* h, void* Kmat, cudaStream_t st);
int apply_edge(const Plan* P, const Weights* W, const void* Kmat, const float* x, const float* root, const float* bias,
               int aggr_mean, float* out, cudaStream_t st, unsigned node_flags = 0);

// diagonal-kernel conv (formulation D, diag.cu; weights prepared with diag = 1):
//   out_n = aggr_{e: dst_e = n} (x_src(e) * d_e) + x_n root + bias,   d_e = W_L h_e + b_L   (fp32 [E, cout], sorted order)
// diag_build computes d chunk by chunk from edge_attr (only d is kept); ws: diag_ws_bytes, its header holds the fp16
// range counter of the chunks' hidden activations (nnconv_edge_features_overflow).  apply_diag: aggr 0 add, 1 mean,
// 2 max (ws: max_keys_bytes of keys, argmax written).  backward_apply_diag: dx, droot, dbias of one application, and
// dd_e += x_src(e) * G_e accumulated over the applications (bipartite plans: root NULL; out, argmax and gout have N_dst
// rows, x and dx N_src, and dx is zeroed over them); backward_mlp_diag (weights prepared at fp32): every
// Linear's gradient from dd, the activations recomputed in fp32 batch by batch.
size_t diag_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes);
int diag_build(const Plan* P, const Weights* W, const float* edge_attr, float* d, void* ws, size_t ws_bytes, cudaStream_t st,
               int64_t* launches);
int apply_diag(const Plan* P, const Weights* W, const float* d, const float* x, const float* root, const float* bias,
               int aggr, float* out, int* argmax, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches);
int backward_apply_diag(const Plan* P, const Weights* W, const float* d, const float* x, const float* root, int aggr,
                        const int* argmax, const float* gout, float* dx, float* droot, float* dbias, float* dd,
                        cudaStream_t st, int64_t* launches);
size_t backward_mlp_diag_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes);
int backward_mlp_diag(const Plan* P, const Weights* W, const float* edge_attr, const float* dd, float* const* dWs,
                      float* const* dbs, void* ws, size_t ws_bytes, cudaStream_t st, float* grad_ea);

// node-level gradients of the root term x root + bias over N rows (x [N, cin], g [N, cout]), backward.cu:
// dbias = sum_n g_n (dbias nullable), droot = x^T g and dx = g root^T (root NULL: dx untouched, dx nullable then)
int backward_node_terms(const float* x, const float* root, const float* gout, int64_t N, int cin, int cout, float* dx,
                        float* droot, float* dbias, cudaStream_t st, int64_t* launches);
// the same terms with the tensor-core backward's node-level kernels (k_colsum, k_xtv, k_g_rootT: parallel over the
// rows) when their shared memory fits, else backward_node_terms (backward_tc.cu)
int node_terms_rows(const float* x, const float* root, const float* gout, int64_t N, int cin, int cout, float* dx,
                    float* droot, float* dbias, cudaStream_t st, int64_t* launches);
// out[n, :] += bias + x[n, :] root over N rows (kernels_simt.cu): the root term of a bipartite application, added
// after the messages (root or bias nullable)
int root_term(const float* x, const float* root, const float* bias, int64_t N, int cin, int cout, float* out,
              cudaStream_t st);

// Gaussian-kernel conv (gauss.cu, DESIGN 4.9): d_ec = exp(-p_e0^2 / sigma_c^2) / sqrt(|p_e1 p_e2|) computed in registers
//   out_n = aggr_{e: dst_e = n} x_src(e) * d_e + x_n root + bias          (C == in == out, 1 <= C <= kGaussMaxChannels)
// edge_attr [E, k_in] (k_in >= 3) in the caller's order, sigma [C].  apply_gauss: aggr 0 add, 1 mean, 2 max (ws:
// max_keys_bytes of keys, argmax written).  backward_gauss: dx, droot, dbias, and the nullable dsigma [C] and dea
// [E, k_in] (written, columns 3 and up 0) of one application.  Bipartite plans as for apply_diag / backward_apply_diag.
constexpr int kGaussMaxChannels = 4096;
size_t gauss_apply_ws_bytes(const Plan* P, int C, int aggr);
int apply_gauss(const Plan* P, const float* edge_attr, int k_in, const float* sigma, int C, const float* x,
                const float* root, const float* bias, int aggr, float* out, int* argmax, void* ws, size_t ws_bytes,
                cudaStream_t st, int64_t* launches);
int backward_gauss(const Plan* P, const float* edge_attr, int k_in, const float* sigma, int C, const float* x,
                   const float* root, int aggr, const int* argmax, const float* gout, float* dx, float* droot,
                   float* dbias, float* dsigma, float* dea, cudaStream_t st, int64_t* launches);

// backward of one application (fp32 CUDA-core path), backward.cu; grad_ea as for backward_mlp_tc.
// aggr = max (all three backward calls): argmax [N, cout] of the forward (backward_mlp_tc: one per application) routes
// each g[n, o] to the winning edge only, G_e[o] = g[dst_e, o] if argmax[dst_e, o] == caller index of e, else 0
size_t backward_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes);
int backward_fp32(const Plan* P, const Weights* W, const float* edge_attr, const float* x, const float* root,
                  int aggr_mean, const float* gout, float* dx, float* const* dWs, float* const* dbs, float* droot,
                  float* dbias, void* ws, size_t ws_bytes, cudaStream_t st, float* grad_ea = nullptr,
                  const int* argmax = nullptr);

}  // namespace nnc
