// Kernel launchers shared between translation units (all return an NNCONV_* status).
#pragma once
#include "common.cuh"
#include "plan.h"

namespace nnc {

// ---- kernels_simt.cu (CUDA cores)
int launch_pad_convert(int prec, const float* src, int R, int C, void* dst, int Rp, int Cp, cudaStream_t st);
int launch_w3p(int prec, const float* WL, int cin, int cout, int K, int Kp, int cin_p, void* dst, cudaStream_t st,
               const float* scale = nullptr);
// scale2[0] = power of two s with max|src| * s in [0.5, 1), scale2[1] = 1 / s   (device floats)
int launch_pow2_scale(const float* src, int64_t n, float* scale2, cudaStream_t st);
// *sticky += *counter on the device (one thread; no host synchronisation, so it can be captured in a CUDA graph)
int launch_overflow_accumulate(const int* counter, int* sticky, cudaStream_t st);
int launch_pad_convert_split3(const float* src, int R, int C, void* dst, int Rp, int Cp, const float* scale, cudaStream_t st);
// backward images of the last Linear: transposed == 0 -> W3q [Kp*cout, cin_p], 1 -> W3t [cin_p, Kp*cout]
// (PREC_F16X2: the reduction dimension is tripled, [hi | lo | hi], and the values are multiplied by *scale first)
int launch_w3q(int prec, const float* WL, int cin, int cout, int K, int Kp, int cin_p, int transposed, void* dst,
               cudaStream_t st, const float* scale = nullptr);
// dst[Cp x Rp] (16-bit) = src[R x C]^T, zero padded (PREC_F16X2: [Cp x 3*Rp], [hi | lo | hi] of *scale times the value)
int launch_transpose_pad(int prec, const float* src, int R, int C, void* dst, int Rp, int Cp, cudaStream_t st,
                         const float* scale = nullptr);
int launch_edge_layer1(int prec, const float* edge_attr, const int* perm, int64_t e_begin, int64_t e_count, int k_in,
                       const float* W1, const float* b1, int kp1, int identity, void* out, cudaStream_t st,
                       int64_t chunk_rows_pad = 0, int64_t out_row0 = 0, int* overflow = nullptr, Act act = Act{});
int launch_build_a1(int prec, const float* edge_attr, const int* perm, int64_t e_begin, int64_t e_count, int k_in,
                    void* A1, cudaStream_t st);
int launch_w1aug(int prec, const float* W1, const float* b1, int k1, int kp1, int k_in, void* dst, cudaStream_t st);
// node_flags: NNCONV_APPLY_RELU_IN (1) = x holds pre-activations, read max(x, 0); NNCONV_APPLY_RESIDUAL (2) = add the
// input row to the output row (cin == cout)
int launch_out_init(const float* x, const float* root, const float* bias, int64_t N, int cin, int cout, float* out,
                    cudaStream_t st, unsigned node_flags = 0);
int launch_src_prep(int prec, const float* x, const int* src_nodes, int S, int cin, int cin_p, int cout,
                    const float* B3, void* Xc, float* cvec, float* xs, cudaStream_t st, unsigned node_flags = 0);
int launch_node_prep(int prec, const float* x, const float* root, const float* bias, int64_t N, float* out,
                     const int* src_nodes, int S, int cin, int cin_p, int cout, const float* B3, void* Xc, float* cvec,
                     float* xs, int* flags, int flags_stride, int n_batches, cudaStream_t st, unsigned node_flags,
                     unsigned long long* max_keys = nullptr);
int launch_sgemm_store(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M, int N,
                       int K, const float* bias_relu, cudaStream_t st, Act act = Act{});
int launch_sgemm_scatter(const Plan* P, const float* h, int Kp, const float* Y, int cout, int tile_begin,
                         int tile_end, int c0, const float* cvec, int aggr_mean, float* out, cudaStream_t st,
                         unsigned long long* max_keys = nullptr);
// aggr = max: max_keys (nullable everywhere above and below) are the [N, cout] keys of common.cuh max_key, which the
// scatter epilogues reduce instead of adding into out; k_node_prep clears them.  After the last contraction of the
// application launch_max_finalize adds the decoded max to out (nothing for a key 0) and writes the winning caller
// edge index (-1 for a node without in-edges) to argmax.
int launch_max_finalize(const unsigned long long* keys, int64_t n, float* out, int* argmax, cudaStream_t st);

// CTA timeline tracing (NNCONV_TRACE=1; measurement only).  The buffer is the one place where the library
// allocates device memory itself, and only when tracing is requested.
struct TraceHandle {
  unsigned long long* rec;
  unsigned int* count;
  unsigned int cap;
};
TraceHandle trace_get();          // {nullptr,..} when tracing is off
int trace_dump(unsigned long long* host_rec, unsigned int max_rec, unsigned int* n_out);

// Cross-kernel pipelining of one conv application (PDL + completion flags, see tc05.cuh).
struct PipeFlags {
  bool pdl;             // launch with programmatic stream serialization
  bool small_footprint; // GEMM only: ~101 KB configuration that can share an SM
  const int* wait_ok;   // flag that must be raised before this kernel touches its dependent buffer (or nullptr)
  int* done_cnt;        // per-kernel CTA counter (or nullptr)
  int* done_ok;         // raised by the last CTA
  const int* join_ok;   // conv only: flags [join_n] the LAST kernel of the chain waits for before it exits
  int join_n;
};

// ---- gemm_tc.cu (wgmma): C[M, N] (16-bit) = act(A[M, K] * B[N, K]^T + bias); A rows start at a_row0 of the
// tensor A_base[a_rows_total, K]; K, N multiples of 64.  bias == nullptr -> no bias, relu flag separate.
// split_flags (PREC_F16X2): GEMM_A_SPLIT -> A is [hi | lo] with 2K/3 columns and B is [hi | lo | hi] with K columns;
// GEMM_C_SPLIT -> C receives [hi | lo] pairs (2N columns / 2N/64 chunks).  overflow: device counter of output
// pieces that left the fp16 range (nullable).  act: the edge network's hidden activation, applied where relu != 0 and
// differentiated where mask != nullptr (C = acc * f'(mask), the ReLU mask for act.kind = NNCONV_ACT_RELU).
enum { GEMM_A_SPLIT = 1, GEMM_C_SPLIT = 2 };
int launch_gemm_tc(int prec, const void* A_base, int64_t a_rows_total, int64_t a_row0, int M, int K,
                   const void* B, int N, const float* bias, int relu, void* C, int64_t ldc, cudaStream_t st,
                   const PipeFlags* pf = nullptr, int64_t chunk_rows_pad = 0, int64_t c_row0 = 0,
                   int split_flags = 0, int* overflow = nullptr, const void* mask = nullptr, int64_t mask_ld = 0,
                   int out_f32 = 0, int64_t a_chunk_rows_pad = 0, const float* acc_scale = nullptr, Act act = Act{});

// ---- per-edge kernel matrices (formulation B, for graphs with few out-edges per source): K_e = W_L h_e + b_L once per
// (edge_attr, parameters), then out[dst] += x_src . K_e per application (kernels_simt.cu)
int launch_apply_edge(int prec, const Plan* P, const Weights* W, const void* Kmat, const float* x, int aggr_mean, float* out,
                      cudaStream_t st, unsigned node_flags = 0);

// ---- gemm_tn.cu (wgmma, MN-major operands): C[M, N] fp32 += alpha * sum_{r<R} A[r, a_col0 + m] * B[r, b_col0 + n]
// (A: [R, lda], B: [R, ldb] 16-bit row-major; C accumulates with fp32 atomics, the caller zero-initialises it)
int launch_gemm_tn(int prec, const void* A, int64_t lda, int a_col0, const void* B, int64_t ldb, int b_col0, int64_t R,
                   int M, int N, float* C, int64_t ldc, float alpha, const float* alpha_dev, cudaStream_t st);

// The part of an application that one contraction covers (api.cu: contract_range): units [u_begin, u_end) of sources
// [c_begin, c_end), with h holding the chunk-major rows of sorted edges [e_base, ...) in panels of h_rows rows.  A whole
// cached h is the range {0, n_units, 0, n_src, 0, round_up(E, 128)}.
struct UnitRange {
  int u_begin, u_end, c_begin, c_end;
  int64_t e_base, h_rows;
};

// ---- conv_tc.cu (wgmma): per-source contraction + scatter for tiles [tile_begin, tile_end); h_rows > 0: h holds the
// rows of sorted edges [e_base, e_base + h_rows) (default: every edge)
int launch_conv_tc(int prec, const Plan* P, const void* h, int Kp, const void* Y, int64_t y_nodes, int cout,
                   int tile_begin, int tile_end, int c0, const float* cvec, const float* xs, int aggr_mean, float* out,
                   cudaStream_t st, const PipeFlags* pf = nullptr, int64_t e_base = 0, int64_t h_rows = 0,
                   unsigned long long* max_keys = nullptr);

// ---- apply_tc.cu: ONE persistent kernel per unit range (Y GEMM + contraction pipelines in every CTA); flags: the
// range's batches of cntY, cntC, okY, okC, cntU at flags_stride
constexpr int kApplyCannotCoSchedule = 1000;   // private status of launch_apply_tc: cooperative launch impossible
bool apply_fused_supported(const Weights* W);
int launch_apply_tc(int prec, const Plan* P, const Weights* W, const void* h, const void* Xc, void* Yring, int nb,
                    int ring, const float* cvec, const float* xs, int aggr_mean, float* out, int* flags,
                    int flags_stride, cudaStream_t st, const UnitRange& R, unsigned long long* max_keys = nullptr);

// ---- graph_build.cu: ball graph (count / fill) on the device
int ball_count(const double* pa, int64_t na, const double* pb, int64_t nb, double radius, int* counts, cudaStream_t st);
int ball_fill(const double* pa, int64_t na, const double* pb, int64_t nb, double radius, const int64_t* offsets,
              int64_t src_base, int64_t dst_base, int64_t* row0, int64_t* row1, const double* theta_a,
              const double* theta_b, float* attr, cudaStream_t st);

// ---- loss.cu: fused loss / normaliser epilogue (ws: 2 + 2*batch floats, res: 4 floats)
int loss_epilogue(const float* out, const float* y, const float* mean, const float* std_, float eps, int batch, int64_t n,
                  float grad_scale, float* grad_l1, float* res, float* ws, cudaStream_t st);

// ---- halo.cu: strip-partition halo exchange by peer stores + sequence flags
int halo_push(const float* out, int relu, int64_t n_local, int C, int64_t own_lo, int64_t own_hi, float* x_next,
              float* peer_up, int64_t up_src0, int64_t up_dst0, int64_t up_rows, float* peer_down, int64_t dn_src0,
              int64_t dn_dst0, int64_t dn_rows, int* flag_up, int* flag_down, int seq, cudaStream_t st);
int halo_wait(const int* flag_a, const int* flag_b, int seq, cudaStream_t st);

bool tc_shapes_supported(const Weights* W);
int tc_init();   // resolves cuTensorMapEncodeTiled, sets kernel attributes; idempotent

}  // namespace nnc
