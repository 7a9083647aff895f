// C-ABI of libnnconv_b200 (declared in include/nnconv_b200.h) and the host-side sequencing of the
// kernels.  No device allocation and no device synchronisation happens here except in
// nnconv_plan_create (one-time per graph, returns counts to the host).
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "common.cuh"
#include "kernels.h"
#include "options.h"

namespace nnc {

namespace {
thread_local char g_err[512] = "";
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---- optional event-based profiling ------------------------------------------------------------
namespace {
struct ProfRec { int kind; cudaEvent_t a, b; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
cudaEvent_t g_prof_open[PK_COUNT];
}
bool prof_enabled() { return g_prof_on; }
void prof_mark(int kind, cudaStream_t st, bool begin) {
  cudaEvent_t e;
  if (cudaEventCreate(&e) != cudaSuccess) return;
  cudaEventRecord(e, st);
  if (begin) g_prof_open[kind] = e;
  else g_prof.push_back(ProfRec{kind, g_prof_open[kind], e});
}

static size_t esize_of(int prec) { return prec == PREC_FP32 ? 4 : 2; }

// ------------------------------------------------------------------------------------------------
// prepared weights
// ------------------------------------------------------------------------------------------------
struct WeightsLayout {
  size_t off_W1, off_b1, off_W1aug, off_Wh[kMaxLayers], off_bh[kMaxLayers], off_W3p, off_B3, bytes;
  size_t off_W3q, off_W3t, off_WhT[kMaxLayers], off_W3n, off_wscale;
  bool bwd;
};

static int fill_dims(Weights* W, int n_layers, const int* dims, int cin, int cout, int prec) {
  NNC_REQUIRE(n_layers >= 1 && n_layers <= kMaxLayers, NNCONV_ERR_ARG, "edge MLP must have 1..%d Linear layers", kMaxLayers);
  NNC_REQUIRE(prec >= PREC_FP32 && prec <= PREC_F16X2, NNCONV_ERR_ARG, "unknown precision %d", prec);
  NNC_REQUIRE(cin >= 1 && cout >= 1, NNCONV_ERR_ARG, "bad channel counts");
  NNC_REQUIRE(dims[n_layers] == cin * cout, NNCONV_ERR_ARG,
              "edge MLP output width %d != in_channels*out_channels = %d", dims[n_layers], cin * cout);
  memset(W, 0, sizeof(*W));
  W->n_layers = n_layers;
  for (int l = 0; l <= n_layers; ++l) {
    NNC_REQUIRE(dims[l] >= 1, NNCONV_ERR_ARG, "bad layer width");
    W->dims[l] = dims[l];
    W->kp[l] = l == 0 ? dims[0] : round_up(dims[l], 64);
  }
  W->cin = cin;
  W->cout = cout;
  W->cin_p = round_up(cin, 64);
  W->K = dims[n_layers - 1];
  W->Kp = round_up(W->K, 64);
  W->prec = prec;
  W->split = prec_is_split(prec) ? 1 : 0;
  W->esize = esize_of(prec);
  if (W->split) {
    NNC_REQUIRE(n_layers >= 2 && 3 * dims[0] + 2 <= 64, NNCONV_ERR_UNSUPPORTED,
                "precision f16x2 needs an edge MLP with >= 2 Linear layers and k_in <= 20 (tensor-core first layer)");
  }
  return NNCONV_OK;
}

static WeightsLayout layout_weights(const Weights* W) {
  Carver c(nullptr, ~size_t(0));
  WeightsLayout L{};
  const int nl = W->n_layers;
  if (nl >= 2) {
    L.off_W1 = c.off; c.take<float>(static_cast<size_t>(W->kp[1]) * W->dims[0]);
    L.off_b1 = c.off; c.take<float>(W->kp[1]);
    L.off_W1aug = c.off; c.take<char>(static_cast<size_t>(W->kp[1]) * 64 * 2);
  }
  for (int l = 2; l <= nl - 1; ++l) {
    L.off_Wh[l] = c.off; c.take<char>(static_cast<size_t>(W->kp[l]) * W->kp[l - 1] * W->esize * (W->split ? 3 : 1));
    L.off_bh[l] = c.off; c.take<float>(W->kp[l]);
  }
  L.off_wscale = c.off; c.take<float>(2 * (kMaxLayers + 2));
  L.off_W3p = c.off; c.take<char>(static_cast<size_t>(W->cout) * W->Kp * W->cin_p * W->esize * (W->split ? 3 : 1));
  L.off_B3 = c.off; c.take<float>(static_cast<size_t>(W->cin) * W->cout);
  // images for the tensor-core backward (same conditions as backward_tc_supported)
  L.bwd = (W->prec == PREC_F16 || W->prec == PREC_BF16) && W->cout == 64 && W->cin <= 64 && nl >= 2 &&
          3 * W->dims[0] + 2 <= 64;
  if (L.bwd) {
    L.off_W3q = c.off; c.take<char>(static_cast<size_t>(W->cout) * W->Kp * W->cin_p * 2);
    L.off_W3t = c.off; c.take<char>(static_cast<size_t>(W->cout) * W->Kp * W->cin_p * 2);
    for (int l = 2; l <= nl - 1; ++l) { L.off_WhT[l] = c.off; c.take<char>(static_cast<size_t>(W->kp[l]) * W->kp[l - 1] * 2); }
  }
  if (W->prec == PREC_F16 || W->prec == PREC_BF16) {
    L.off_W3n = c.off; c.take<char>(static_cast<size_t>(W->cin) * W->cout * W->Kp * 2);
  }
  L.bytes = c.off;
  return L;
}

size_t weights_bytes(int n_layers, const int* dims, int cin, int cout, int prec) {
  Weights W;
  if (fill_dims(&W, n_layers, dims, cin, cout, prec) != NNCONV_OK) return 0;
  return layout_weights(&W).bytes;
}

int weights_prepare(Weights* W, int n_layers, const int* dims, int cin, int cout, int prec,
                    const float* const* Wsrc, const float* const* bsrc, void* buf, size_t buf_bytes,
                    cudaStream_t st) {
  int s = fill_dims(W, n_layers, dims, cin, cout, prec);
  if (s != NNCONV_OK) return s;
  WeightsLayout L = layout_weights(W);
  NNC_REQUIRE(buf != nullptr && L.bytes <= buf_bytes, NNCONV_ERR_WORKSPACE, "weights buffer too small (need %zu)", L.bytes);
  char* base = static_cast<char*>(buf);
  const int nl = n_layers;
  if (nl >= 2) {
    float* W1 = reinterpret_cast<float*>(base + L.off_W1);
    float* b1 = reinterpret_cast<float*>(base + L.off_b1);
    s = launch_pad_convert(PREC_FP32, Wsrc[0], dims[1], dims[0], W1, W->kp[1], dims[0], st);
    if (s) return s;
    s = launch_pad_convert(PREC_FP32, bsrc[0], 1, dims[1], b1, 1, W->kp[1], st);
    if (s) return s;
    W->W1 = W1;
    W->b1 = b1;
    if (prec != PREC_FP32 && 3 * dims[0] + 2 <= 64) {   // split-precision first layer on the tensor cores
      void* aug = base + L.off_W1aug;
      s = launch_w1aug(prec, W1, b1, dims[1], W->kp[1], dims[0], aug, st);
      if (s) return s;
      W->W1aug = aug;
    }
  }
  float* wscale = reinterpret_cast<float*>(base + L.off_wscale);
  if (W->split) W->wscale = wscale;
  for (int l = 2; l <= nl - 1; ++l) {
    void* Wh = base + L.off_Wh[l];
    float* bh = reinterpret_cast<float*>(base + L.off_bh[l]);
    if (W->split) {
      s = launch_pow2_scale(Wsrc[l - 1], static_cast<int64_t>(dims[l]) * dims[l - 1], wscale + 2 * l, st);
      if (s) return s;
      s = launch_pad_convert_split3(Wsrc[l - 1], dims[l], dims[l - 1], Wh, W->kp[l], W->kp[l - 1], wscale + 2 * l, st);
    } else {
      s = launch_pad_convert(prec, Wsrc[l - 1], dims[l], dims[l - 1], Wh, W->kp[l], W->kp[l - 1], st);
    }
    if (s) return s;
    s = launch_pad_convert(PREC_FP32, bsrc[l - 1], 1, dims[l], bh, 1, W->kp[l], st);
    if (s) return s;
    W->Wh[l] = Wh;
    W->bh[l] = bh;
  }
  void* W3p = base + L.off_W3p;
  float* B3 = reinterpret_cast<float*>(base + L.off_B3);
  if (W->split) {
    s = launch_pow2_scale(Wsrc[nl - 1], static_cast<int64_t>(dims[nl]) * dims[nl - 1], wscale + 2 * nl, st);
    if (s) return s;
  }
  s = launch_w3p(prec, Wsrc[nl - 1], cin, cout, W->K, W->Kp, W->cin_p, W3p, st, W->split ? wscale + 2 * nl : nullptr);
  if (s) return s;
  s = launch_pad_convert(PREC_FP32, bsrc[nl - 1], 1, cin * cout, B3, 1, cin * cout, st);
  if (s) return s;
  W->W3p = W3p;
  W->B3 = B3;
  if (prec == PREC_F16 || prec == PREC_BF16) {
    s = launch_pad_convert(prec, Wsrc[nl - 1], cin * cout, W->K, base + L.off_W3n, cin * cout, W->Kp, st);
    if (s) return s;
    W->W3n = base + L.off_W3n;
  }
  if (L.bwd) {
    s = launch_w3q(prec, Wsrc[nl - 1], cin, cout, W->K, W->Kp, W->cin_p, 0, base + L.off_W3q, st);
    if (s) return s;
    s = launch_w3q(prec, Wsrc[nl - 1], cin, cout, W->K, W->Kp, W->cin_p, 1, base + L.off_W3t, st);
    if (s) return s;
    W->W3q = base + L.off_W3q;
    W->W3t = base + L.off_W3t;
    for (int l = 2; l <= nl - 1; ++l) {
      s = launch_transpose_pad(prec, Wsrc[l - 1], dims[l], dims[l - 1], base + L.off_WhT[l], W->kp[l], W->kp[l - 1], st);
      if (s) return s;
      W->WhT[l] = base + L.off_WhT[l];
    }
  }
  return NNCONV_OK;
}

// ------------------------------------------------------------------------------------------------
// edge features: h_last for every (source-sorted) edge
// ------------------------------------------------------------------------------------------------
static int max_hidden_kp(const Weights* W) {
  int m = 64;
  for (int l = 1; l <= W->n_layers - 1; ++l) m = W->kp[l] > m ? W->kp[l] : m;
  return m;
}

constexpr size_t kEfHeader = 1024;   // start of the edge-feature workspace: [0] = overflow counter (int)

static size_t ef_row_bytes(const Weights* W) {
  // per edge row of workspace: A1 (64 x 16-bit, tensor-core first layer) + ping/pong hidden activations
  // (PREC_F16X2: [hi | lo] pairs, twice the width)
  size_t row = 0;
  if (W->W1aug) row += 128;
  if (W->n_layers > 2) row += 2 * static_cast<size_t>(max_hidden_kp(W)) * W->esize * (W->split ? 2 : 1);
  return row;
}

size_t edge_features_ws_bytes(const Plan* P, const Weights* W, size_t want_bytes) {
  const size_t row = ef_row_bytes(W);
  if (row == 0) return kEfHeader + 1024;   // h_last is written directly by the CUDA-core first-layer kernel
  size_t rows_all = static_cast<size_t>(round_up64(P->E > 0 ? P->E : 1, 128));
  size_t rows = want_bytes / row;
  rows = rows / 128 * 128;
  if (rows < 128) rows = 128;
  if (rows > rows_all) rows = rows_all;
  return kEfHeader + rows * row + 8192;
}

size_t edge_acts_offset(const Plan* P, const Weights* W, int l) {
  const size_t rows = static_cast<size_t>(round_up64(P->E > 0 ? P->E : 1, 128));
  size_t off = 0;
  for (int j = 1; j < l; ++j) off += rows * W->kp[j] * 2;
  return off;
}

size_t edge_acts_bytes(const Plan* P, const Weights* W) {
  if (W->split || W->prec == PREC_FP32 || W->n_layers < 3) return 0;
  return edge_acts_offset(P, W, W->n_layers - 1) + 1024;
}

int edge_features(const Plan* P, const Weights* W, const float* edge_attr, void* h, void* ws, size_t ws_bytes,
                  cudaStream_t st, int64_t* launches, void* acts) {
  if (acts != nullptr && edge_acts_bytes(P, W) == 0) acts = nullptr;
  const int64_t E = P->E;
  NNC_REQUIRE(ws != nullptr && ws_bytes >= kEfHeader, NNCONV_ERR_WORKSPACE, "edge_features: workspace too small");
  int* overflow = static_cast<int*>(ws);
  NNC_CHECK_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int), st));
  if (options().l2_reset) cudaCtxResetPersistingL2Cache();   // experiment knob: drop the Y ring's persisting lines
  if (E == 0) return NNCONV_OK;
  if (!options().overflow_check) overflow = nullptr;
  ws = static_cast<char*>(ws) + kEfHeader;
  ws_bytes -= kEfHeader;
  const int nl = W->n_layers;
  const bool tc = tc_shapes_supported(W);
  NNC_REQUIRE(tc || W->prec == PREC_FP32, NNCONV_ERR_UNSUPPORTED,
              "shape not supported by the tensor-core path (out=%d, K=%d); use precision fp32", W->cout, W->K);
  int s;
  const int amul = W->split ? 2 : 1;   // activation width multiplier ([hi | lo])
  const int kmul = W->split ? 3 : 1;   // GEMM K multiplier ([hi | hi | lo] x [hi | lo | hi])
  // 16-bit path: h is chunk-major [amul*Kp/64][E_pad][64] (what the contraction kernel streams); fp32: row-major
  const int64_t hpad = W->prec == PREC_FP32 ? 0 : round_up64(E, 128);
  if (hpad > E) {
    // rows [E, E_pad) of every panel are read (never used) by TMA boxes that run past the last edge; the backward
    // multiplies them by zero, so they must not hold NaN bit patterns of a recycled allocation
    NNC_CHECK_CUDA(cudaMemset2DAsync(static_cast<char*>(h) + static_cast<size_t>(E) * 128, static_cast<size_t>(hpad) * 128,
                                     0, static_cast<size_t>(hpad - E) * 128, static_cast<size_t>(amul * W->Kp / 64), st));
  }
  if (nl == 1) {   // single Linear: h_last = edge_attr (padded)
    ProfScope ps(PK_LAYER1, st);
    s = launch_edge_layer1(W->prec, edge_attr, P->perm, 0, E, W->dims[0], nullptr, nullptr, W->Kp, 1, h, st, hpad, 0);
    if (launches) ++*launches;
    return s;
  }
  const size_t rowb = ef_row_bytes(W);
  if (rowb == 0) {   // CUDA-core first layer straight into h (fp32 path, 2-layer MLP)
    ProfScope ps(PK_LAYER1, st);
    s = launch_edge_layer1(W->prec, edge_attr, P->perm, 0, E, W->dims[0], W->W1, W->b1, W->kp[1], 0, h, st, hpad, 0);
    if (launches) ++*launches;
    return s;
  }
  NNC_REQUIRE(ws_bytes >= 128 * rowb + 4096, NNCONV_ERR_WORKSPACE, "edge_features: workspace too small");
  const int64_t rows = static_cast<int64_t>((ws_bytes - 4096) / rowb) / 128 * 128;
  const size_t hid = static_cast<size_t>(max_hidden_kp(W)) * W->esize * amul;
  char* a1 = static_cast<char*>(ws);
  char* bufA = a1 + (W->W1aug ? round_up64(rows * 128, 1024) : 0);
  char* bufB = bufA + round_up64(static_cast<int64_t>(rows * hid), 1024);
  for (int64_t e0 = 0; e0 < E; e0 += rows) {
    const int64_t n = (E - e0) < rows ? (E - e0) : rows;
    void* h_rows = hpad > 0 ? h : static_cast<void*>(static_cast<char*>(h) + static_cast<size_t>(e0) * W->Kp * W->esize);
    const int64_t h_pad_l1 = nl == 2 ? hpad : 0;     // first layer writes h directly only for 2-layer MLPs
    auto act_rows = [&](int l) -> char* {   // rows [e0, ...) of the kept activations of layer l
      return static_cast<char*>(acts) + edge_acts_offset(P, W, l) + static_cast<size_t>(e0) * W->kp[l] * 2;
    };
    void* dst1 = nl == 2 ? h_rows : (acts ? static_cast<void*>(act_rows(1)) : static_cast<void*>(bufA));
    {
      ProfScope ps(PK_LAYER1, st);
      if (W->W1aug) {
        s = launch_build_a1(W->prec, edge_attr, P->perm, e0, n, W->dims[0], a1, st);
        if (s) return s;
        s = launch_gemm_tc(W->prec, a1, n, 0, static_cast<int>(n), 64, W->W1aug, W->kp[1], nullptr, 1, dst1,
                           static_cast<int64_t>(amul) * W->kp[1], st, nullptr, h_pad_l1, e0,
                           W->split ? GEMM_C_SPLIT : 0, overflow);
        if (launches) ++*launches;
      } else {
        s = launch_edge_layer1(W->prec, edge_attr, P->perm, e0, n, W->dims[0], W->W1, W->b1, W->kp[1], 0, dst1, st,
                               h_pad_l1, e0);
      }
    }
    if (s) return s;
    if (launches) ++*launches;
    char* cur = acts ? act_rows(1) : bufA;
    char* nxt = bufB;
    for (int l = 2; l <= nl - 1; ++l) {
      const bool last = l == nl - 1;
      if (acts && !last) nxt = act_rows(l);
      void* dst = last ? h_rows : static_cast<void*>(nxt);
      ProfScope ps(PK_HIDDEN_GEMM, st);
      if (W->prec == PREC_FP32) {
        s = launch_sgemm_store(reinterpret_cast<const float*>(cur), W->kp[l - 1],
                               reinterpret_cast<const float*>(W->Wh[l]), W->kp[l - 1], static_cast<float*>(dst),
                               W->kp[l], static_cast<int>(n), W->kp[l], W->kp[l - 1], W->bh[l], st);
      } else {
        s = launch_gemm_tc(W->prec, cur, n, 0, static_cast<int>(n), kmul * W->kp[l - 1], W->Wh[l], W->kp[l], W->bh[l], 1,
                           dst, static_cast<int64_t>(amul) * W->kp[l], st, nullptr, last ? hpad : 0, e0,
                           W->split ? (GEMM_A_SPLIT | GEMM_C_SPLIT) : 0, overflow, nullptr, 0, 0, 0,
                           W->split ? W->wscale + 2 * l + 1 : nullptr);
      }
      if (s) return s;
      if (launches) ++*launches;
      char* tmp = cur; cur = nxt; nxt = acts ? bufB : tmp;
    }
  }
  return NNCONV_OK;
}

// ------------------------------------------------------------------------------------------------
// formulation B (SURVEY 8(d)): per-edge kernel matrices, for graphs whose sources have only a few out-edges.
// Formulation C spends one [out, Kp] matrix per SOURCE (128 KB at out=64, Kp=1024) and a 128-row wgmma tile per
// source; with 2-4 out-edges per node (the 1-D multipole hierarchy of config 5) that is as expensive as one kernel
// matrix per EDGE and the tiles are 97 % empty.  K_e = W_L h_e + b_L is x-independent like h: it is built once per
// (edge_attr, parameters) by the wgmma GEMM and every application is one bandwidth-bound pass over it.
// ------------------------------------------------------------------------------------------------
bool edge_kernels_supported(const Weights* W) {
  return (W->prec == PREC_F16 || W->prec == PREC_BF16) && W->W3n != nullptr && (W->cin * W->cout) % 64 == 0 &&
         W->cout % 2 == 0 && W->n_layers >= 2;
}

size_t edge_kernels_bytes(const Plan* P, const Weights* W) {
  return static_cast<size_t>(P->E > 0 ? P->E : 1) * W->cin * W->cout * 2 + 1024;
}

int edge_kernels(const Plan* P, const Weights* W, const void* h, void* Kmat, cudaStream_t st) {
  NNC_REQUIRE(edge_kernels_supported(W), NNCONV_ERR_UNSUPPORTED, "per-edge kernel matrices: unsupported shape / precision");
  if (P->E == 0) return NNCONV_OK;
  const int64_t hpad = round_up64(P->E, 128);
  const int NK = W->cin * W->cout;
  return launch_gemm_tc(W->prec, h, P->E, 0, static_cast<int>(P->E), W->Kp, W->W3n, NK, W->B3, 0, Kmat, NK, st, nullptr, 0, 0,
                        0, nullptr, nullptr, 0, 0, hpad);
}

int apply_edge(const Plan* P, const Weights* W, const void* Kmat, const float* x, const float* root, const float* bias,
               int aggr_mean, float* out, cudaStream_t st, unsigned node_flags) {
  NNC_REQUIRE(!(node_flags & NNCONV_APPLY_RESIDUAL) || W->cin == W->cout, NNCONV_ERR_ARG,
              "NNCONV_APPLY_RESIDUAL needs in_channels == out_channels");
  int s = launch_out_init(x, root, bias, P->N, W->cin, W->cout, out, st, node_flags);
  if (s) return s;
  if (P->E == 0 || P->n_src == 0) return NNCONV_OK;
  return launch_apply_edge(W->prec, P, W, Kmat, x, aggr_mean, out, st, node_flags);
}

// ------------------------------------------------------------------------------------------------
// one conv application
// ------------------------------------------------------------------------------------------------
struct ApplyLayout {
  size_t off_Xc, off_cvec, off_xs, off_flags, off_Y, fixed_bytes, per_node;
};
constexpr int kMaxPipeBatches = 1 << 14;   // flags: cntY, cntC, okY, okC per batch

static ApplyLayout layout_apply(const Plan* P, const Weights* W) {
  Carver c(nullptr, ~size_t(0));
  ApplyLayout L{};
  const size_t S = P->n_src > 0 ? P->n_src : 1;
  L.off_Xc = c.off; c.take<char>((S + 128) * W->cin_p * W->esize * (W->split ? 3 : 1));
  L.off_cvec = c.off; c.take<float>(S * W->cout);
  L.off_xs = c.off; c.take<float>(S);
  L.off_flags = c.off; c.take<int>(5 * kMaxPipeBatches);
  L.off_Y = c.off;
  L.fixed_bytes = c.off;
  L.per_node = static_cast<size_t>(W->cout) * W->Kp * W->esize * (W->split ? 2 : 1);
  return L;
}

size_t apply_ws_bytes(const Plan* P, const Weights* W, size_t want_y_bytes) {
  ApplyLayout L = layout_apply(P, W);
  size_t nodes = want_y_bytes / L.per_node;
  if (nodes < 1) nodes = 1;
  if (nodes > static_cast<size_t>(P->n_src > 0 ? P->n_src : 1)) nodes = P->n_src > 0 ? P->n_src : 1;
  return L.fixed_bytes + nodes * L.per_node + 1024;
}

int apply(const Plan* P, const Weights* W, const void* h, const float* x, const float* root, const float* bias,
          int aggr_mean, float* out, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches, unsigned node_flags) {
  int s;
  NNC_REQUIRE(!(node_flags & NNCONV_APPLY_RESIDUAL) || W->cin == W->cout, NNCONV_ERR_ARG,
              "NNCONV_APPLY_RESIDUAL needs in_channels == out_channels");
  if (P->E == 0 || P->n_src == 0) {
    ProfScope ps(PK_NODE_PREP, st);
    s = launch_out_init(x, root, bias, P->N, W->cin, W->cout, out, st, node_flags);
    if (s == NNCONV_OK && launches) ++*launches;
    return s;
  }
  const bool tc = tc_shapes_supported(W);
  NNC_REQUIRE(tc || W->prec == PREC_FP32, NNCONV_ERR_UNSUPPORTED,
              "shape not supported by the tensor-core path (out=%d, K=%d); use precision fp32", W->cout, W->K);
  ApplyLayout L = layout_apply(P, W);
  NNC_REQUIRE(ws != nullptr && ws_bytes >= L.fixed_bytes + L.per_node, NNCONV_ERR_WORKSPACE,
              "apply: workspace too small (need >= %zu bytes)", L.fixed_bytes + L.per_node);
  char* base = static_cast<char*>(ws);
  void* Xc = base + L.off_Xc;
  float* cvec = reinterpret_cast<float*>(base + L.off_cvec);
  float* xs = reinterpret_cast<float*>(base + L.off_xs);
  void* Y = base + L.off_Y;
  int64_t nodes_cap = static_cast<int64_t>((ws_bytes - L.fixed_bytes) / L.per_node);
  const Options& opt = options();
  // fused persistent kernel (below): its batch geometry is needed here because the node-prep launch also clears its flags
  const bool no_fuse_env = opt.no_fuse != 0 && !W->split;      // measurement / debugging knob
  bool fused = W->prec != PREC_FP32 && !no_fuse_env && apply_fused_supported(W);
  int ring = opt.ring;   // with dynamic unit scheduling 3 x 128 sources (48 MB at out=64, Kp=1024) is best
  int64_t nb = 0;
  if (fused) {
    if (opt.ring_deep && nodes_cap / 128 > ring) ring = nodes_cap / 128 < 16 ? static_cast<int>(nodes_cap / 128) : 16;
    if (nodes_cap < ring) ring = nodes_cap >= 2 ? static_cast<int>(nodes_cap) : 1;
    nb = nodes_cap / ring;
    if (nb >= 128) nb = nb / 128 * 128;
    if (nb > P->n_src) nb = P->n_src;
    fused = ceil_div64(P->n_src, nb) <= kMaxPipeBatches && ring >= 2;
  }
  int* flags = reinterpret_cast<int*>(base + L.off_flags);
  if (fused) {
    ProfScope ps(PK_NODE_PREP, st);
    s = launch_node_prep(W->prec, x, root, bias, P->N, out, P->src_nodes, P->n_src, W->cin, W->cin_p, W->cout, W->B3, Xc,
                         cvec, xs, flags, kMaxPipeBatches, static_cast<int>(ceil_div64(P->n_src, nb)), st, node_flags);
    if (s) return s;
    if (launches) ++*launches;
  } else {
    {
      ProfScope ps(PK_NODE_PREP, st);
      s = launch_out_init(x, root, bias, P->N, W->cin, W->cout, out, st, node_flags);
    }
    if (s) return s;
    {
      ProfScope ps(PK_NODE_PREP, st);
      s = launch_src_prep(W->prec, x, P->src_nodes, P->n_src, W->cin, W->cin_p, W->cout, W->B3, Xc, cvec, xs, st, node_flags);
    }
    if (s) return s;
    if (launches) *launches += 2;
  }
  // tile_ptr lives on the device; tile ranges per batch come from the host mirror kept in the plan handle
  const int* h_tile_ptr = P->h_tile_ptr;
  const int NY = W->cout * W->Kp;

  if (W->prec == PREC_FP32) {   // CUDA-core path: plain stream order, one Y buffer
    int64_t nb_max = nodes_cap > P->n_src ? P->n_src : nodes_cap;
    for (int64_t c0 = 0; c0 < P->n_src; c0 += nb_max) {
      const int nb = static_cast<int>((P->n_src - c0) < nb_max ? (P->n_src - c0) : nb_max);
      const int tb = h_tile_ptr[c0], te = h_tile_ptr[c0 + nb];
      {
        ProfScope ps(PK_Y_GEMM, st);
        s = launch_sgemm_store(reinterpret_cast<const float*>(Xc) + c0 * W->cin_p, W->cin_p,
                               reinterpret_cast<const float*>(W->W3p), W->cin_p, static_cast<float*>(Y), NY, nb, NY,
                               W->cin_p, nullptr, st);
      }
      if (s) return s;
      {
        ProfScope ps(PK_CONV, st);
        s = launch_sgemm_scatter(P, static_cast<const float*>(h), W->Kp, static_cast<const float*>(Y), W->cout, tb,
                                 te, static_cast<int>(c0), cvec, aggr_mean, out, st);
      }
      if (s) return s;
      if (launches) *launches += 2;
    }
    return NNCONV_OK;
  }

  // Tensor-core path, default: ONE persistent kernel per application (apply_tc.cu) in which every CTA runs
  // the Y GEMM pipeline and the contraction pipeline concurrently over a ring of L2-resident Y batches.
  if (fused) {
    {
      ProfScope ps(PK_APPLY_FUSED, st);
      s = launch_apply_tc(W->prec, P, W, h, Xc, Y, static_cast<int>(nb), ring, cvec, xs, aggr_mean, out, flags,
                          kMaxPipeBatches, st);
    }
    if (s == NNCONV_OK) {
      if (launches) ++*launches;
      return NNCONV_OK;
    }
    // the driver cannot co-schedule one CTA per SM (MPS / green-context partition): per-batch kernels below
    if (s != kApplyCannotCoSchedule) return s;
  }
  NNC_REQUIRE(!W->split, NNCONV_ERR_UNSUPPORTED,
              "precision f16x2 runs in the fused persistent kernel only (shape or workspace not supported)");

  // Fallback (NNCONV_NO_FUSE=1 or shapes the fused kernel does not cover): one Y GEMM + one contraction
  // kernel per batch of sources.  Batches of sources sized so that the Y buffers stay L2 resident; kernel order
  //   Y(0), Y(1), C(0), Y(2), C(1), ..., C(B-1)            (three Y buffers, b mod 3)
  // launched with programmatic stream serialization, so CTAs of the next kernel start on SMs as CTAs of
  // the running kernel retire; the true dependencies  C(b) <- Y(b)  and  Y(b) <- C(b-3) (buffer reuse)
  // are completion flags in global memory.  Profiling mode (events between kernels) falls back to plain
  // stream order so that per-kernel times are meaningful.
  const bool no_pipe_env = opt.no_pipe != 0;   // measurement / debugging knob
  const bool pipe = !prof_enabled() && !no_pipe_env && nodes_cap >= 3;
  int64_t nb_max = pipe ? nodes_cap / 3 : nodes_cap;
  if (nb_max > P->n_src) nb_max = P->n_src;
  int64_t n_batches = ceil_div64(P->n_src, nb_max);
  if (n_batches > kMaxPipeBatches) {   // keep the flag table bounded: grow batches past the L2 target
    NNC_REQUIRE(false, NNCONV_ERR_WORKSPACE, "apply: workspace too small for %lld source batches", (long long)n_batches);
  }
  int* cntY = flags;
  int* cntC = flags + kMaxPipeBatches;
  int* okY = flags + 2 * kMaxPipeBatches;
  int* okC = flags + 3 * kMaxPipeBatches;
  if (pipe) NNC_CHECK_CUDA(cudaMemsetAsync(flags, 0, sizeof(int) * 4 * kMaxPipeBatches, st));
  // three Y buffers: Y(b+2) is launched right after C(b) and reuses the buffer C(b-1) read, which has
  // retired by then -- with two buffers Y(b+2) would have to wait for the kernel it directly follows
  char* Ybuf[3] = {static_cast<char*>(Y), static_cast<char*>(Y) + (pipe ? nb_max * L.per_node : 0),
                   static_cast<char*>(Y) + (pipe ? 2 * nb_max * L.per_node : 0)};

  auto launch_y = [&](int64_t b) -> int {
    const int64_t c0 = b * nb_max;
    const int nb = static_cast<int>((P->n_src - c0) < nb_max ? (P->n_src - c0) : nb_max);
    PipeFlags pf{};
    pf.pdl = pipe && b > 0;
    pf.small_footprint = true;
    pf.wait_ok = (pipe && b >= 3) ? okC + (b - 3) : nullptr;
    pf.done_cnt = pipe ? cntY + b : nullptr;
    pf.done_ok = pipe ? okY + b : nullptr;
    ProfScope ps(PK_Y_GEMM, st);
    return launch_gemm_tc(W->prec, Xc, P->n_src, c0, nb, W->cin_p, W->W3p, NY, nullptr, 0, Ybuf[b % 3], NY, st, &pf);
  };
  auto launch_c = [&](int64_t b) -> int {
    const int64_t c0 = b * nb_max;
    const int nb = static_cast<int>((P->n_src - c0) < nb_max ? (P->n_src - c0) : nb_max);
    const int tb = h_tile_ptr[c0], te = h_tile_ptr[c0 + nb];
    PipeFlags pf{};
    pf.pdl = pipe;
    pf.wait_ok = pipe ? okY + b : nullptr;
    pf.done_cnt = pipe ? cntC + b : nullptr;
    pf.done_ok = pipe ? okC + b : nullptr;
    if (pipe && b == n_batches - 1) {   // last kernel of the chain: join every earlier conv kernel
      pf.join_ok = okC;
      pf.join_n = static_cast<int>(n_batches - 1);
    }
    ProfScope ps(PK_CONV, st);
    return launch_conv_tc(W->prec, P, h, W->Kp, Ybuf[b % 3], nb, W->cout, tb, te, static_cast<int>(c0), cvec, xs,
                          aggr_mean, out, st, pipe ? &pf : nullptr);
  };
  s = launch_y(0);
  if (s) return s;
  for (int64_t b = 0; b < n_batches; ++b) {
    if (b + 1 < n_batches) {
      s = launch_y(b + 1);
      if (s) return s;
    }
    s = launch_c(b);
    if (s) return s;
  }
  if (launches) *launches += 2 * n_batches;
  return NNCONV_OK;
}

}  // namespace nnc

// ==================================================================================================
// extern "C"
// ==================================================================================================
using namespace nnc;

struct nnconv_plan {
  Plan p;
  int* h_tile_ptr_storage;     // [2*(S+1)]: tile_ptr mirror, then group_ptr mirror
};
struct nnconv_weights {
  Weights w;
};

extern "C" {

const char* nnconv_last_error(void) { return nnc::g_err; }

int nnconv_abi_version(void) { return NNCONV_B200_ABI_VERSION; }

int nnconv_init(void) {
  (void)nnc::options();   // read the NNCONV_* environment once
  return tc_init();
}

int nnconv_set_option(const char* name, int value) {
  NNC_REQUIRE(name != nullptr && nnc::option_set(name, value) == 0, NNCONV_ERR_ARG, "unknown option '%s'", name ? name : "");
  return NNCONV_OK;
}

int nnconv_get_option(const char* name, int* value) {
  NNC_REQUIRE(name != nullptr && value != nullptr && nnc::option_get(name, value) == 0, NNCONV_ERR_ARG,
              "unknown option '%s'", name ? name : "");
  return NNCONV_OK;
}

int nnconv_plan_sizes(int64_t E, int64_t N, size_t* ws_bytes, size_t* tmp_bytes) {
  NNC_REQUIRE(ws_bytes && tmp_bytes, NNCONV_ERR_ARG, "null output pointer");
  NNC_REQUIRE(E >= 0 && N >= 1, NNCONV_ERR_ARG, "need E >= 0, N >= 1");
  plan_sizes(E, N, ws_bytes, tmp_bytes);
  return NNCONV_OK;
}

int nnconv_plan_create(const int64_t* row0, const int64_t* row1, int64_t E, int64_t N, int flow, void* ws, size_t ws_bytes,
                       void* tmp, size_t tmp_bytes, void* stream, nnconv_plan_t** out) {
  NNC_REQUIRE(out != nullptr, NNCONV_ERR_ARG, "null output pointer");
  *out = nullptr;
  nnconv_plan* h = new (std::nothrow) nnconv_plan();
  NNC_REQUIRE(h != nullptr, NNCONV_ERR_ARG, "out of host memory");
  h->h_tile_ptr_storage = nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int s = plan_build(&h->p, row0, row1, E, N, flow, ws, ws_bytes, tmp, tmp_bytes, st);
  if (s != NNCONV_OK) { delete h; return s; }
  // host mirror of tile_ptr (S+1 ints) so that batch tile ranges need no device read later
  const int S = h->p.n_src;
  h->h_tile_ptr_storage = new (std::nothrow) int[2 * (static_cast<size_t>(S) + 1)];
  if (!h->h_tile_ptr_storage) { delete h; set_error("out of host memory"); return NNCONV_ERR_ARG; }
  cudaError_t e = cudaMemcpyAsync(h->h_tile_ptr_storage, h->p.tile_ptr, (static_cast<size_t>(S) + 1) * sizeof(int),
                                  cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(h->h_tile_ptr_storage + S + 1, h->p.group_ptr, (static_cast<size_t>(S) + 1) * sizeof(int),
                        cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    set_error("plan: copying tile_ptr failed: %s", cudaGetErrorString(e));
    delete[] h->h_tile_ptr_storage;
    delete h;
    return NNCONV_ERR_CUDA;
  }
  h->p.h_tile_ptr = h->h_tile_ptr_storage;
  h->p.h_group_ptr = h->h_tile_ptr_storage + S + 1;
  *out = h;
  return NNCONV_OK;
}

void nnconv_plan_destroy(nnconv_plan_t* plan) {
  if (!plan) return;
  delete[] plan->h_tile_ptr_storage;
  delete plan;
}

int nnconv_plan_info(const nnconv_plan_t* plan, int64_t* info, int n_info) {
  NNC_REQUIRE(plan && info && n_info >= 7, NNCONV_ERR_ARG, "plan_info: need a plan and >= 7 slots");
  info[0] = plan->p.E;
  info[1] = plan->p.N;
  info[2] = plan->p.n_src;
  info[3] = plan->p.n_tiles;
  info[4] = plan->p.max_out_deg;
  info[5] = plan->p.src_sorted;
  info[6] = plan->p.flow;
  return NNCONV_OK;
}

int nnconv_weights_sizes(int n_layers, const int* dims, int in_channels, int out_channels, int precision,
                         size_t* bytes) {
  NNC_REQUIRE(bytes && dims, NNCONV_ERR_ARG, "null pointer");
  Weights W;
  int s = fill_dims(&W, n_layers, dims, in_channels, out_channels, precision);
  if (s) return s;
  *bytes = layout_weights(&W).bytes;
  return NNCONV_OK;
}

int nnconv_weights_create(int n_layers, const int* dims, int in_channels, int out_channels, int precision,
                          const float* const* W, const float* const* b, void* buf, size_t buf_bytes, void* stream,
                          nnconv_weights_t** out) {
  NNC_REQUIRE(out && dims && W && b, NNCONV_ERR_ARG, "null pointer");
  *out = nullptr;
  nnconv_weights* h = new (std::nothrow) nnconv_weights();
  NNC_REQUIRE(h != nullptr, NNCONV_ERR_ARG, "out of host memory");
  int s = weights_prepare(&h->w, n_layers, dims, in_channels, out_channels, precision, W, b, buf, buf_bytes,
                          static_cast<cudaStream_t>(stream));
  if (s != NNCONV_OK) { delete h; return s; }
  *out = h;
  return NNCONV_OK;
}

void nnconv_weights_destroy(nnconv_weights_t* w) { delete w; }

int nnconv_weights_tc_supported(const nnconv_weights_t* w) { return w && tc_shapes_supported(&w->w) ? 1 : 0; }

int nnconv_edge_features_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_ws_bytes,
                               size_t* h_bytes, size_t* ws_bytes) {
  NNC_REQUIRE(plan && w && h_bytes && ws_bytes, NNCONV_ERR_ARG, "null pointer");
  const int64_t rows = round_up64(plan->p.E > 0 ? plan->p.E : 1, 128);
  *h_bytes = static_cast<size_t>(rows) * w->w.Kp * w->w.esize * (w->w.split ? 2 : 1);
  *ws_bytes = edge_features_ws_bytes(&plan->p, &w->w, want_ws_bytes);
  return NNCONV_OK;
}

int nnconv_edge_features(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, void* h,
                         void* ws, size_t ws_bytes, void* stream, int64_t* launches) {
  NNC_REQUIRE(plan && w && (edge_attr || plan->p.E == 0) && h, NNCONV_ERR_ARG, "null pointer");
  return edge_features(&plan->p, &w->w, edge_attr, h, ws, ws_bytes, static_cast<cudaStream_t>(stream), launches);
}

int nnconv_edge_acts_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t* bytes) {
  NNC_REQUIRE(plan && w && bytes, NNCONV_ERR_ARG, "null pointer");
  *bytes = edge_acts_bytes(&plan->p, &w->w);
  return NNCONV_OK;
}

int nnconv_edge_features_keep(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, void* h,
                              void* acts, void* ws, size_t ws_bytes, void* stream, int64_t* launches) {
  NNC_REQUIRE(plan && w && (edge_attr || plan->p.E == 0) && h, NNCONV_ERR_ARG, "null pointer");
  return edge_features(&plan->p, &w->w, edge_attr, h, ws, ws_bytes, static_cast<cudaStream_t>(stream), launches, acts);
}

int nnconv_edge_features_overflow(const void* ws, void* stream, int64_t* count) {
  NNC_REQUIRE(ws && count, NNCONV_ERR_ARG, "null pointer");
  int v = 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  NNC_CHECK_CUDA(cudaMemcpyAsync(&v, ws, sizeof(int), cudaMemcpyDeviceToHost, st));
  NNC_CHECK_CUDA(cudaStreamSynchronize(st));
  *count = v;
  return NNCONV_OK;
}

int nnconv_edge_kernels_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t* bytes) {
  NNC_REQUIRE(plan && w && bytes, NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(edge_kernels_supported(&w->w), NNCONV_ERR_UNSUPPORTED, "per-edge kernel matrices: unsupported shape / precision");
  *bytes = edge_kernels_bytes(&plan->p, &w->w);
  return NNCONV_OK;
}

int nnconv_edge_kernels(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, void* kmat, void* stream) {
  NNC_REQUIRE(plan && w && kmat && (h || plan->p.E == 0), NNCONV_ERR_ARG, "null pointer");
  return edge_kernels(&plan->p, &w->w, h, kmat, static_cast<cudaStream_t>(stream));
}

int nnconv_apply_edge(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* kmat, const float* x,
                      const float* root, const float* bias, int aggr, float* out, void* stream) {
  NNC_REQUIRE(plan && w && x && out && (kmat || plan->p.E == 0), NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED, "aggr must be add or mean");
  return apply_edge(&plan->p, &w->w, kmat, x, root, bias, aggr == NNCONV_AGGR_MEAN, out, static_cast<cudaStream_t>(stream));
}

int nnconv_apply_edge_ex(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* kmat, const float* x,
                         const float* root, const float* bias, int aggr, unsigned flags, float* out, void* stream) {
  NNC_REQUIRE(plan && w && x && out && (kmat || plan->p.E == 0), NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED, "aggr must be add or mean");
  NNC_REQUIRE((flags & ~(NNCONV_APPLY_RELU_IN | NNCONV_APPLY_RESIDUAL)) == 0, NNCONV_ERR_ARG, "unknown apply flag");
  NNC_REQUIRE(x != out, NNCONV_ERR_ARG, "out must not alias x");
  return apply_edge(&plan->p, &w->w, kmat, x, root, bias, aggr == NNCONV_AGGR_MEAN, out, static_cast<cudaStream_t>(stream),
                    flags);
}

int nnconv_apply_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_y_bytes, size_t* ws_bytes) {
  NNC_REQUIRE(plan && w && ws_bytes, NNCONV_ERR_ARG, "null pointer");
  *ws_bytes = apply_ws_bytes(&plan->p, &w->w, want_y_bytes);
  return NNCONV_OK;
}

int nnconv_apply(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, const float* x,
                 const float* root, const float* bias, int aggr, float* out, void* ws, size_t ws_bytes, void* stream,
                 int64_t* launches) {
  NNC_REQUIRE(plan && w && x && out && (h || plan->p.E == 0), NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED,
              "aggr must be add (0) or mean (1); 'max' is used by no call site of the reference and is not built");
  return apply(&plan->p, &w->w, h, x, root, bias, aggr == NNCONV_AGGR_MEAN, out, ws, ws_bytes,
               static_cast<cudaStream_t>(stream), launches);
}

int nnconv_apply_ex(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, const float* x,
                    const float* root, const float* bias, int aggr, unsigned flags, float* out, void* ws, size_t ws_bytes,
                    void* stream, int64_t* launches) {
  NNC_REQUIRE(plan && w && x && out && (h || plan->p.E == 0), NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED,
              "aggr must be add (0) or mean (1); 'max' is used by no call site of the reference and is not built");
  NNC_REQUIRE((flags & ~(NNCONV_APPLY_RELU_IN | NNCONV_APPLY_RESIDUAL)) == 0, NNCONV_ERR_ARG, "unknown apply flag");
  NNC_REQUIRE(x != out, NNCONV_ERR_ARG, "out must not alias x");
  return apply(&plan->p, &w->w, h, x, root, bias, aggr == NNCONV_AGGR_MEAN, out, ws, ws_bytes,
               static_cast<cudaStream_t>(stream), launches, flags);
}

int nnconv_backward_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_bytes, size_t* ws_bytes) {
  NNC_REQUIRE(plan && w && ws_bytes, NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(w->w.prec == PREC_FP32, NNCONV_ERR_ARG, "backward needs weights prepared with NNCONV_PREC_FP32");
  *ws_bytes = backward_ws_bytes(&plan->p, &w->w, want_bytes);
  return NNCONV_OK;
}

int nnconv_backward(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const float* x,
                    const float* root, int aggr, const float* grad_out, float* grad_x, float* const* grad_W,
                    float* const* grad_b, float* grad_root, float* grad_bias, void* ws, size_t ws_bytes,
                    void* stream) {
  NNC_REQUIRE(plan && w && x && grad_out && grad_x && grad_W && grad_b, NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED, "aggr must be add or mean");
  NNC_REQUIRE((root == nullptr) == (grad_root == nullptr), NNCONV_ERR_ARG, "root / grad_root must both be given or both be NULL");
  return backward_fp32(&plan->p, &w->w, edge_attr, x, root, aggr == NNCONV_AGGR_MEAN, grad_out, grad_x, grad_W,
                       grad_b, grad_root, grad_bias, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

int nnconv_backward_tc_supported(const nnconv_weights_t* w) { return w && backward_tc_supported(&w->w) ? 1 : 0; }

int nnconv_backward_apply_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_bytes, size_t* ws_bytes) {
  NNC_REQUIRE(plan && w && ws_bytes, NNCONV_ERR_ARG, "null pointer");
  NNC_REQUIRE(backward_tc_supported(&w->w), NNCONV_ERR_UNSUPPORTED, "tensor-core backward: unsupported shape / precision");
  *ws_bytes = backward_apply_ws_bytes(&plan->p, &w->w, want_bytes);
  return NNCONV_OK;
}

int nnconv_backward_apply(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, const float* x,
                          const float* root, int aggr, const float* grad_out, float* grad_x, float* grad_W_last,
                          float* grad_b_last, float* grad_root, float* grad_bias, void* ws, size_t ws_bytes,
                          void* stream) {
  NNC_REQUIRE(plan && w && x && grad_out && grad_x && grad_W_last && grad_b_last && (h || plan->p.E == 0), NNCONV_ERR_ARG,
              "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED, "aggr must be add or mean");
  NNC_REQUIRE((root == nullptr) == (grad_root == nullptr), NNCONV_ERR_ARG, "root / grad_root must both be given or both be NULL");
  return backward_apply_tc(&plan->p, &w->w, h, x, root, aggr == NNCONV_AGGR_MEAN, grad_out, grad_x, grad_W_last,
                           grad_b_last, grad_root, grad_bias, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

int nnconv_backward_mlp_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, int n_apps, size_t want_bytes,
                              size_t* ws_bytes) {
  NNC_REQUIRE(plan && w && ws_bytes && n_apps >= 1, NNCONV_ERR_ARG, "bad arguments");
  NNC_REQUIRE(backward_tc_supported(&w->w), NNCONV_ERR_UNSUPPORTED, "tensor-core backward: unsupported shape / precision");
  *ws_bytes = backward_mlp_ws_bytes(&plan->p, &w->w, n_apps, want_bytes);
  return NNCONV_OK;
}

int nnconv_backward_mlp(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const void* h,
                        int n_apps, const float* const* grad_out, const float* const* x, int aggr, float* const* grad_W,
                        float* const* grad_b, void* ws, size_t ws_bytes, void* stream, const void* acts) {
  NNC_REQUIRE(plan && w && grad_out && x && grad_W && grad_b && ((edge_attr && h) || plan->p.E == 0), NNCONV_ERR_ARG,
              "null pointer");
  NNC_REQUIRE(aggr == NNCONV_AGGR_ADD || aggr == NNCONV_AGGR_MEAN, NNCONV_ERR_UNSUPPORTED, "aggr must be add or mean");
  return backward_mlp_tc(&plan->p, &w->w, edge_attr, h, n_apps, grad_out, x, aggr == NNCONV_AGGR_MEAN, grad_W, grad_b, ws,
                         ws_bytes, static_cast<cudaStream_t>(stream), acts);
}

int nnconv_gemm_tn_16b(int precision, const void* A, int64_t lda, const void* B, int64_t ldb, int64_t R, int M, int N,
                       float* C, int64_t ldc, float alpha, void* stream) {
  NNC_REQUIRE(A && B && C, NNCONV_ERR_ARG, "gemm_tn: null pointer");
  return launch_gemm_tn(precision, A, lda, 0, B, ldb, 0, R, M, N, C, ldc, alpha, nullptr, static_cast<cudaStream_t>(stream));
}

int nnconv_gemm_16b_ex(int precision, const void* A, int64_t M, int K, const void* B, int N, const float* bias, int relu,
                       void* C, int64_t ldc, const void* mask, int64_t mask_ld, int out_f32, void* stream) {
  NNC_REQUIRE(A && B && C && M >= 1 && M < (int64_t(1) << 31), NNCONV_ERR_ARG, "gemm: bad arguments");
  return launch_gemm_tc(precision, A, M, 0, static_cast<int>(M), K, B, N, bias, relu, C, ldc,
                        static_cast<cudaStream_t>(stream), nullptr, 0, 0, 0, nullptr, mask, mask_ld, out_f32);
}

int nnconv_halo_push(const float* out, int relu, int64_t n_local, int channels, int64_t own_lo, int64_t own_hi,
                     float* x_next, float* peer_up, int64_t up_src0, int64_t up_dst0, int64_t up_rows, float* peer_down,
                     int64_t dn_src0, int64_t dn_dst0, int64_t dn_rows, int* flag_up, int* flag_down, int seq,
                     void* stream) {
  return halo_push(out, relu, n_local, channels, own_lo, own_hi, x_next, peer_up, up_src0, up_dst0, up_rows, peer_down,
                   dn_src0, dn_dst0, dn_rows, flag_up, flag_down, seq, static_cast<cudaStream_t>(stream));
}

// Peer-visible buffers of the halo exchange.  They are the one place (besides the optional trace buffer) where the
// library allocates device memory itself: a CUDA IPC handle can only be taken of a whole cudaMalloc allocation, and
// the importing side must open it with ITS device current (cudaIpcMemLazyEnablePeerAccess then maps the memory for
// kernels of that device) -- memory imported through torch's tensor sharing is opened under the exporter's device and
// faulted when a kernel of the importing rank's device stored into it.
int nnconv_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64) {
  NNC_REQUIRE(dev_ptr && handle64 && bytes > 0, NNCONV_ERR_ARG, "ipc_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  void* p = nullptr;
  NNC_CHECK_CUDA(cudaMalloc(&p, bytes));
  NNC_CHECK_CUDA(cudaMemset(p, 0, bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    NNC_CHECK_CUDA(e);
  }
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return NNCONV_OK;
}

int nnconv_ipc_open(const unsigned char* handle64, void** dev_ptr) {
  NNC_REQUIRE(dev_ptr && handle64, NNCONV_ERR_ARG, "ipc_open: bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  NNC_CHECK_CUDA(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return NNCONV_OK;
}

int nnconv_ipc_close(void* dev_ptr) {
  if (dev_ptr) NNC_CHECK_CUDA(cudaIpcCloseMemHandle(dev_ptr));
  return NNCONV_OK;
}

int nnconv_ipc_free(void* dev_ptr) {
  if (dev_ptr) NNC_CHECK_CUDA(cudaFree(dev_ptr));
  return NNCONV_OK;
}

int nnconv_enable_peer_access(int peer_device) {
  int dev = 0;
  NNC_CHECK_CUDA(cudaGetDevice(&dev));
  if (peer_device == dev) return NNCONV_OK;
  int can = 0;
  NNC_CHECK_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
  NNC_REQUIRE(can, NNCONV_ERR_UNSUPPORTED, "device %d cannot access device %d (no P2P path)", dev, peer_device);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
  NNC_CHECK_CUDA(e);
  return NNCONV_OK;
}

int nnconv_halo_wait(const int* flag_from_up, const int* flag_from_down, int seq, void* stream) {
  return halo_wait(flag_from_up, flag_from_down, seq, static_cast<cudaStream_t>(stream));
}

int nnconv_loss_epilogue(const float* out, const float* y, const float* mean, const float* std_, float eps, int batch,
                         int64_t n, float grad_scale, float* grad_l1, float* results, float* ws, void* stream) {
  return loss_epilogue(out, y, mean, std_, eps, batch, n, grad_scale, grad_l1, results, ws, static_cast<cudaStream_t>(stream));
}

int nnconv_ball_count(const double* pa, int64_t na, const double* pb, int64_t nb, double radius, int* counts, void* stream) {
  NNC_REQUIRE(pa && pb && counts && na >= 0 && nb >= 0, NNCONV_ERR_ARG, "ball_count: bad arguments");
  return ball_count(pa, na, pb, nb, radius, counts, static_cast<cudaStream_t>(stream));
}

int nnconv_ball_fill(const double* pa, int64_t na, const double* pb, int64_t nb, double radius, const int64_t* offsets,
                     int64_t src_base, int64_t dst_base, int64_t* row0, int64_t* row1, const double* theta_a,
                     const double* theta_b, float* edge_attr, void* stream) {
  NNC_REQUIRE(pa && pb && offsets && row0 && row1 && (theta_a == nullptr) == (theta_b == nullptr), NNCONV_ERR_ARG,
              "ball_fill: bad arguments");
  return ball_fill(pa, na, pb, nb, radius, offsets, src_base, dst_base, row0, row1, theta_a, theta_b, edge_attr,
                   static_cast<cudaStream_t>(stream));
}

int nnconv_profile_begin(void) {
  for (auto& r : nnc::g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  nnc::g_prof.clear();
  nnc::g_prof_on = true;
  return NNCONV_OK;
}

int nnconv_profile_end(double* ms_by_kind, int64_t* launches_by_kind, int n_kinds) {
  nnc::g_prof_on = false;
  NNC_REQUIRE(ms_by_kind && launches_by_kind && n_kinds >= PK_COUNT, NNCONV_ERR_ARG, "profile_end: need >= %d slots", (int)PK_COUNT);
  NNC_CHECK_CUDA(cudaDeviceSynchronize());
  for (int k = 0; k < n_kinds; ++k) { ms_by_kind[k] = 0.0; launches_by_kind[k] = 0; }
  for (auto& r : nnc::g_prof) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { ms_by_kind[r.kind] += ms; launches_by_kind[r.kind] += 1; }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  nnc::g_prof.clear();
  return NNCONV_OK;
}

int nnconv_debug_trace_dump(unsigned long long* host_rec, unsigned int max_rec, unsigned int* n_out) {
  NNC_REQUIRE(host_rec && n_out, NNCONV_ERR_ARG, "null pointer");
  return trace_dump(host_rec, max_rec, n_out);
}

// test hook: `n_ctas` CTAs that each hold `smem_bytes` of shared memory and spin for `ns` nanoseconds
__global__ void k_debug_occupy(long long ns) {
  extern __shared__ char occ_smem[];
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  occ_smem[threadIdx.x] = 0;
  for (;;) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    if (static_cast<long long>(t - t0) >= ns) break;
    __nanosleep(1000);
  }
}

int nnconv_debug_occupy(int n_ctas, int smem_bytes, long long ns, void* stream) {
  NNC_REQUIRE(n_ctas >= 1 && smem_bytes >= 0 && smem_bytes <= 227 * 1024 && ns >= 0 && ns <= 2000000000ll, NNCONV_ERR_ARG,
              "debug_occupy: bad arguments");
  NNC_CHECK_CUDA(cudaFuncSetAttribute(k_debug_occupy, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  k_debug_occupy<<<n_ctas, 128, smem_bytes, static_cast<cudaStream_t>(stream)>>>(ns);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int nnconv_gemm_16b(int precision, const void* A, int64_t M, int K, const void* B, int N, const float* bias,
                    int relu, void* C, void* stream) {
  NNC_REQUIRE(A && B && C && M >= 1 && M < (int64_t(1) << 31), NNCONV_ERR_ARG, "gemm: bad arguments");
  return launch_gemm_tc(precision, A, M, 0, static_cast<int>(M), K, B, N, bias, relu, C, N,
                        static_cast<cudaStream_t>(stream));
}

}  // extern "C"
