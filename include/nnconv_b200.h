/* nnconv_b200.h -- C ABI of libnnconv_b200.so: the NNConv (edge-conditioned convolution) hot path of
 * neuraloperator/graph-pde, hand-written for NVIDIA H100 (sm_90a).
 *
 * What it replaces (paths relative to the reference repo):
 *   graph-neural-operator/nn_conv.py:267-282   NNConv_old.forward / message / update
 *   graph-neural-operator/utilities.py:223-227 DenseNet.forward (the edge MLP evaluated inside message)
 *   torch_geometric MessagePassing.propagate + torch_scatter.scatter_{add,mean} (un-vendored third
 *   party reached from nn_conv.py:271)
 * and, through the same entry points, upstream torch_geometric.nn.NNConv as used by
 *   multipole-graph-neural-operator/neurips1_MGKN.py:41,49,57, MGKN_general_darcy2d.py:45,53,61,
 *   MGKN_orthogonal_burgers1d.py:37.
 *
 * Conventions
 *   - every function returns 0 on success or an NNCONV_ERR_* code; nnconv_last_error() returns a
 *     thread-local message.  No C++ exception crosses this boundary.
 *   - all data pointers are DEVICE pointers on the current CUDA device unless named host_*;
 *     `stream` is a cudaStream_t passed as void*.
 *   - the library never allocates device memory: callers query a size, allocate (e.g. through the
 *     PyTorch caching allocator) and pass the buffer.  Buffers handed to *_create calls must outlive
 *     the handle.
 *   - no call synchronises the device except nnconv_plan_create (one-time per graph).
 *   - re-entrant; no thread-local state apart from the error string.
 *
 * Math (identical to the reference up to floating-point association, see DESIGN.md):
 *   h_e    = DenseNet_without_last_Linear(edge_attr_e)                  (x independent, "edge features")
 *   K_e    = (W_L h_e + b_L).view(in, out)                              nn_conv.py:274
 *   m_e    = x[src_e] @ K_e                                             nn_conv.py:275
 *   out_n  = aggr_{e: dst_e = n} m_e  + x_n @ root + bias               nn_conv.py:277-282
 * with flow = source_to_target: src = edge_index[0], dst = edge_index[1]; mean of an empty
 * neighbourhood is 0.
 */
#ifndef NNCONV_B200_H_
#define NNCONV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NNCONV_B200_ABI_VERSION 2   /* 2: round-2 entry points (backward_apply / backward_mlp, f16x2, options, halo, ...) */

/* status codes */
#define NNCONV_OK 0
#define NNCONV_ERR_ARG 1
#define NNCONV_ERR_CUDA 2
#define NNCONV_ERR_WORKSPACE 3
#define NNCONV_ERR_UNSUPPORTED 4

/* precision of the tensor-core operands (accumulation is always fp32; x@root+bias and the first
 * MLP layer are always fp32 CUDA-core math) */
#define NNCONV_PREC_FP32 0 /* CUDA-core fp32 everywhere, any shape */
#define NNCONV_PREC_F16 1  /* wgmma f16, fp16 operands (10-bit mantissa, TF32-grade) */
#define NNCONV_PREC_BF16 2 /* wgmma bf16 operands */
/* fp32-grade results on the fp16 tensor pipe: every operand is an fp16 pair (hi, lo = fp16(v - hi)), every
 * product hi*hi + hi*lo + lo*hi in the fp32 accumulator (3x the MMA work, 2x the activation bytes) */
#define NNCONV_PREC_F16X2 3

#define NNCONV_AGGR_ADD 0
#define NNCONV_AGGR_MEAN 1

#define NNCONV_FLOW_SOURCE_TO_TARGET 0
#define NNCONV_FLOW_TARGET_TO_SOURCE 1

typedef struct nnconv_plan nnconv_plan_t;       /* per edge_index: source grouping, tiles, degrees */
typedef struct nnconv_weights nnconv_weights_t; /* per parameter version: padded/permuted MLP weights */

const char* nnconv_last_error(void);
int nnconv_abi_version(void);
/* checks the device (sm_90), resolves the TMA descriptor encoder and reads the NNCONV_* tuning
 * variables from the environment (once); idempotent */
int nnconv_init(void);
/* tuning / debugging knobs (csrc/options.h lists them: "no_fuse", "ring", "no_coop", ...).  The environment is
 * consulted only by the first nnconv_init; afterwards knobs change through nnconv_set_option.  A value below
 * -1000000 restores the built-in default. */
int nnconv_set_option(const char* name, int value);
int nnconv_get_option(const char* name, int* value);

/* ---- plan: replaces the implicit structure PyG derives from edge_index inside propagate() -------- */
int nnconv_plan_sizes(int64_t E, int64_t N, size_t* ws_bytes, size_t* tmp_bytes);
/* row0 / row1: the two int64 rows of edge_index [2, E] (nn_conv.py:267 argument); passing the rows
 * separately lets a column slice edge_index[:, a:b] (neurips1_MGKN.py:75) be used without a copy.
 * ws stays owned by the plan, tmp may be freed on return.  Synchronises `stream` (returns tile counts
 * to the host). */
int nnconv_plan_create(const int64_t* row0, const int64_t* row1, int64_t E, int64_t N, int flow, void* ws, size_t ws_bytes,
                       void* tmp, size_t tmp_bytes, void* stream, nnconv_plan_t** out);
void nnconv_plan_destroy(nnconv_plan_t* plan);
/* info[0..6] = E, N, #sources with out-edges, #tiles, max out-degree, already-grouped flag, flow */
int nnconv_plan_info(const nnconv_plan_t* plan, int64_t* info, int n_info);

/* ---- weights: snapshot of the edge MLP ("nn" argument of NNConv_old.__init__, nn_conv.py:234-246) -- */
/* dims[0..n_layers] = k_in, k_1, ..., in_channels*out_channels;  W[l]: [dims[l+1], dims[l]] fp32
 * (torch.nn.Linear layout, utilities.py:212-213), b[l]: [dims[l+1]].  W and b are HOST arrays of device
 * pointers. */
int nnconv_weights_sizes(int n_layers, const int* dims, int in_channels, int out_channels, int precision,
                         size_t* bytes);
int nnconv_weights_create(int n_layers, const int* dims, int in_channels, int out_channels, int precision,
                          const float* const* W, const float* const* b, void* buf, size_t buf_bytes, void* stream,
                          nnconv_weights_t** out);
void nnconv_weights_destroy(nnconv_weights_t* w);
int nnconv_weights_tc_supported(const nnconv_weights_t* w);

/* ---- hoisted, x-independent part of message(): h_e for every edge (utilities.py:223-227 minus the
 * last Linear).  Valid as long as edge_attr and the weights are unchanged, i.e. for all T applications
 * of the shared conv inside KernelNN.forward (UAI1_full_resolution.py:29-30). ------------------------ */
int nnconv_edge_features_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_ws_bytes,
                               size_t* h_bytes, size_t* ws_bytes);
int nnconv_edge_features(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr /*[E,k_in]*/,
                         void* h, void* ws, size_t ws_bytes, void* stream, int64_t* launches /*nullable*/);

/* Training variant: additionally KEEPS the hidden activations h_1 .. h_{L-2} of every edge in `acts`
 * (nnconv_edge_acts_sizes bytes; 0 = nothing to keep for this configuration, pass NULL) so that
 * nnconv_backward_mlp need not recompute them (2 KB per edge and kept layer at width 1024). */
int nnconv_edge_acts_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t* bytes);
int nnconv_edge_features_keep(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, void* h,
                              void* acts, void* ws, size_t ws_bytes, void* stream, int64_t* launches /*nullable*/);

/* Number of 32-column output pieces of the LAST nnconv_edge_features call on `ws` that left the fp16 range
 * (|v| > 65504 or NaN; fp16 precisions only, always 0 for bf16 / fp32 or with option overflow_check = 0).
 * Copies one int to the host and synchronises `stream`.  A non-zero count means h holds inf: use bf16 / fp32. */
int nnconv_edge_features_overflow(const void* ws, void* stream, int64_t* count);

/* The same counter without a host read: enqueues on `stream` one kernel that adds the int at `counter` (the first
 * word of an edge-feature or nnconv_apply_streamed workspace, or the last 1024 bytes of kmat, as for
 * nnconv_edge_features_overflow) into the device int `sticky`.  No host synchronisation: a CUDA graph can capture it,
 * and the caller reads `sticky` once after any number of passes. */
int nnconv_overflow_accumulate(const void* counter, int* sticky, void* stream);

/* ---- partially resident edge features, for graphs whose h does not fit the device (16-bit precisions):
 * the h of the sorted edges [0, E_res) is cached as above, and every application recomputes the h of [E_res, E)
 * chunk by chunk (same bits as the cached pass) and contracts each chunk right after computing it.
 *   nnconv_stream_split: E_res = the largest unit-aligned prefix whose h (h_res_bytes) fits resident_bytes
 *     (resident_bytes >= the whole h -> E_res = E); ws_bytes = workspace of nnconv_apply_streamed for chunks of
 *     about chunk_ws_bytes (chunk h + edge-feature workspace); n_chunks = chunks per application.
 *   nnconv_edge_features_prefix: h of [0, E_res) into h_res_bytes (ws of nnconv_edge_features_sizes).
 *   nnconv_apply_streamed: nnconv_apply_ex given that prefix.  No allocation, no host synchronisation (capturable);
 *     the first int of ws counts fp16 overflows of the streamed chunks (nnconv_edge_features_overflow(ws, ...)). */
int nnconv_stream_split(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t resident_bytes, size_t chunk_ws_bytes,
                        int64_t* E_res, size_t* h_res_bytes, size_t* ws_bytes, int64_t* n_chunks);
int nnconv_edge_features_prefix(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, int64_t E_res,
                                void* h, void* ws, size_t ws_bytes, void* stream, int64_t* launches /*nullable*/);
int nnconv_apply_streamed(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const void* h_res,
                          int64_t E_res, const float* x, const float* root, const float* bias, int aggr, unsigned flags,
                          float* out, void* ws, size_t ws_bytes, void* stream, int64_t* launches /*nullable*/);

/* ---- per-edge kernel matrices for graphs with few out-edges per source (the 1-D multipole hierarchy of
 * MGKN_orthogonal_burgers1d.py has 2-4): K_e = W_L h_e + b_L ([in, out] 16-bit per edge, sorted edge order) is as
 * x-independent as h, so it is built ONCE per (edge_attr, parameters) from the h of nnconv_edge_features
 * (nn_conv.py:274) and every application is nnconv_apply_edge: out[dst] (+)= x_src @ K_e, one bandwidth-bound pass
 * (nn_conv.py:275-282 incl. root / bias / mean).  Same result as nnconv_apply up to 16-bit rounding of K_e.
 * The last 1024 bytes of kmat hold the fp16 range counter of the build (nnconv_edge_features_overflow(kmat + bytes -
 * 1024, ...)): K_e carries b_L in 16 bits, where nnconv_apply keeps it in fp32, so a last-layer bias beyond the
 * fp16 range overflows here and not there. */
int nnconv_edge_kernels_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t* bytes);
int nnconv_edge_kernels(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, void* kmat, void* stream);
int nnconv_apply_edge(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* kmat, const float* x,
                      const float* root, const float* bias, int aggr, float* out, void* stream);
/* nnconv_apply_edge with the NNCONV_APPLY_* flags of nnconv_apply_ex (below). */
int nnconv_apply_edge_ex(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* kmat, const float* x,
                         const float* root, const float* bias, int aggr, unsigned flags, float* out, void* stream);

/* ---- one NNConv application: gather + last Linear + per-edge contraction + scatter + root + bias ---
 * want_y_bytes: bytes of per-source Y matrices the workspace holds; 0 = the library's default, sized from the
 * current device's L2 (what it holds beside the application's `out` rows, less headroom, but at least 128 sources per
 * ring slot up to the L2 size). */
int nnconv_apply_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_y_bytes, size_t* ws_bytes);
/* x [N,in] fp32, root [in,out] or NULL, bias [out] or NULL, out [N,out] fp32 (fully overwritten). */
int nnconv_apply(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, const float* x,
                 const float* root, const float* bias, int aggr, float* out, void* ws, size_t ws_bytes, void* stream,
                 int64_t* launches /*nullable*/);

/* One V-cycle step  x <- relu(x + conv(x))  (multipole-graph-neural-operator/neurips1_MGKN.py:76,81,84) without
 * elementwise kernels between the 52 dependent applications of a forward: the caller keeps the PRE-activation
 *   z_{k+1} = relu(z_k) + conv(relu(z_k))
 * and applies the last ReLU itself.  flags:
 *   NNCONV_APPLY_RELU_IN   x holds pre-activations; every read of x (gather, root term, residual) is max(x, 0)
 *   NNCONV_APPLY_RESIDUAL  out = (relu?)(x) + conv(...)   (in_channels == out_channels; out must not alias x)
 * flags = 0 is exactly nnconv_apply.  Forward only. */
#define NNCONV_APPLY_RELU_IN 1u
#define NNCONV_APPLY_RESIDUAL 2u
int nnconv_apply_ex(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, const float* x,
                    const float* root, const float* bias, int aggr, unsigned flags, float* out, void* ws, size_t ws_bytes,
                    void* stream, int64_t* launches /*nullable*/);

/* ---- backward of one application (what autograd generates for nn_conv.py:267-282 + utilities.py:223-227):
 * grad_x [N,in], grad_W[l] / grad_b[l] in the torch.nn.Linear layouts of the edge MLP, grad_root [in,out],
 * grad_bias [out] (NULL when the module has no root / bias).  fp32 CUDA-core path for arbitrary shapes: `w`
 * must have been created with NNCONV_PREC_FP32.  Gradients are WRITTEN (not accumulated).  edge_index receives no
 * gradient; edge_attr receives one through nnconv_backward_ex. ------------------------------------------------- */
int nnconv_backward_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_bytes, size_t* ws_bytes);
int nnconv_backward(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const float* x,
                    const float* root, int aggr, const float* grad_out, float* grad_x, float* const* grad_W,
                    float* const* grad_b, float* grad_root, float* grad_bias, void* ws, size_t ws_bytes,
                    void* stream);
/* nnconv_backward plus the gradient w.r.t. edge_attr: grad_edge_attr [E, k_in] fp32 in the caller's edge order,
 * WRITTEN (d edge_attr_e = dz_1[e] . W_1, dz_1 = gradient at the first hidden pre-activation; for a single-Linear
 * edge network the gradient w.r.t. the identity features).  NULL = exactly nnconv_backward: no extra launch, and the
 * workspace of nnconv_backward_sizes serves both. */
int nnconv_backward_ex(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const float* x,
                       const float* root, int aggr, const float* grad_out, float* grad_x, float* const* grad_W,
                       float* const* grad_b, float* grad_root, float* grad_bias, void* ws, size_t ws_bytes,
                       void* stream, float* grad_edge_attr /* nullable */);

/* ---- tensor-core backward (f16, bf16, f16x2; out_channels = 64, in_channels <= 64, edge MLP with >= 2 Linear
 * layers; nnconv_backward_tc_supported tells).  Split in two because the edge features h do not depend on x:
 *
 *   nnconv_backward_apply   one call per application, given that application's grad_out: writes grad_x,
 *                           grad of the LAST Linear (weight [in*out, K], bias [in*out]), grad_root, grad_bias.
 *   nnconv_backward_mlp     ONE call per (edge_attr, parameters) after the n_apps applications that shared them
 *                           (KernelNN applies one conv T times, UAI1_full_resolution.py:29-30): given every
 *                           application's grad_out and x (HOST arrays of device pointers), writes the gradients of
 *                           the hidden Linear layers 0 .. n_layers-2.  The reference's autograd runs this pass T times.
 *
 * `h` is the buffer nnconv_edge_features filled for the same (plan, w, edge_attr).  Gradients are WRITTEN. */
int nnconv_backward_tc_supported(const nnconv_weights_t* w);
int nnconv_backward_apply_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, size_t want_bytes, size_t* ws_bytes);
int nnconv_backward_apply(const nnconv_plan_t* plan, const nnconv_weights_t* w, const void* h, const float* x,
                          const float* root, int aggr, const float* grad_out, float* grad_x, float* grad_W_last,
                          float* grad_b_last, float* grad_root, float* grad_bias, void* ws, size_t ws_bytes,
                          void* stream);
int nnconv_backward_mlp_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, int n_apps, size_t want_bytes,
                              size_t* ws_bytes);
int nnconv_backward_mlp(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const void* h,
                        int n_apps, const float* const* grad_out, const float* const* x, int aggr, float* const* grad_W,
                        float* const* grad_b, void* ws, size_t ws_bytes, void* stream,
                        const void* acts /* from nnconv_edge_features_keep, or NULL = recompute */);
/* nnconv_backward_mlp plus the gradient w.r.t. edge_attr, summed over the n_apps applications: grad_edge_attr
 * [E, k_in] fp32 in the caller's edge order, WRITTEN (one extra pass per source batch that reads the 16-bit dz_1 once;
 * no host sync).  A conv applied more often than one call takes gets one call per group of applications, and the
 * caller sums the groups, as for grad_W / grad_b.  NULL = exactly nnconv_backward_mlp: no extra launch, and the
 * workspace of nnconv_backward_mlp_sizes serves both. */
int nnconv_backward_mlp_ex(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr, const void* h,
                           int n_apps, const float* const* grad_out, const float* const* x, int aggr,
                           float* const* grad_W, float* const* grad_b, void* ws, size_t ws_bytes, void* stream,
                           const void* acts, float* grad_edge_attr /* nullable */);

/* Tensor-core backward over partially resident edge features (training on graphs whose h does not fit the device):
 * h_res / E_res as for nnconv_apply_streamed (E_res a unit boundary; E_res = E is the cached call).  The sources whose
 * edges all lie in [0, E_res) run against h_res; the others run in source batches that first recompute the h of their
 * edges from edge_attr into a chunk buffer of the workspace (same bits as the cached pass).  The MLP pass recomputes
 * h_{L-1} of such batches for its ReLU mask.  Gradients are WRITTEN; no allocation, no host synchronisation.
 *   nnconv_backward_apply_streamed_sizes: want_bytes as for nnconv_backward_apply_sizes, plus chunk rows for about
 *     chunk_ws_bytes of h, never fewer than the edges of the largest source (a batch holds whole sources).
 *   nnconv_backward_streamed_chunks: source batches whose h the call with this workspace recomputes (n_apps = 0:
 *     nnconv_backward_apply_streamed, else nnconv_backward_mlp_streamed with n_apps applications); host only. */
int nnconv_backward_apply_streamed_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, int64_t E_res,
                                         size_t want_bytes, size_t chunk_ws_bytes, size_t* ws_bytes);
int nnconv_backward_apply_streamed(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr,
                                   const void* h_res, int64_t E_res, const float* x, const float* root, int aggr,
                                   const float* grad_out, float* grad_x, float* grad_W_last, float* grad_b_last,
                                   float* grad_root, float* grad_bias, void* ws, size_t ws_bytes, void* stream,
                                   int64_t* launches /*nullable*/);
int nnconv_backward_mlp_streamed_sizes(const nnconv_plan_t* plan, const nnconv_weights_t* w, int64_t E_res, int n_apps,
                                       size_t want_bytes, size_t* ws_bytes);
int nnconv_backward_mlp_streamed(const nnconv_plan_t* plan, const nnconv_weights_t* w, const float* edge_attr,
                                 const void* h_res, int64_t E_res, int n_apps, const float* const* grad_out,
                                 const float* const* x, int aggr, float* const* grad_W, float* const* grad_b, void* ws,
                                 size_t ws_bytes, void* stream, float* grad_edge_attr /* nullable */);
int nnconv_backward_streamed_chunks(const nnconv_plan_t* plan, const nnconv_weights_t* w, int64_t E_res, int n_apps,
                                    size_t ws_bytes, int64_t* n_chunks);

/* ---- halo exchange of the node-range (strip) partition by peer stores over NVLink (no NCCL call, no host round
 * trip between applications).  `out` [n_local, channels] is the result of one application on this rank (owned rows
 * [own_lo, own_hi) valid); the call writes relu?(out) of the owned rows into this rank's next-application buffer
 * x_next and the boundary rows [*_src0, +*_rows) into the neighbours' buffers (device pointers mapped with CUDA IPC,
 * NULL at the mesh border) at rows [*_dst0, ...), then stores `seq` into the neighbours' flag words.
 * nnconv_halo_wait makes `stream` wait until both local flag words are >= seq. */
int nnconv_halo_push(const float* out, int relu, int64_t n_local, int channels, int64_t own_lo, int64_t own_hi,
                     float* x_next, float* peer_up, int64_t up_src0, int64_t up_dst0, int64_t up_rows, float* peer_down,
                     int64_t dn_src0, int64_t dn_dst0, int64_t dn_rows, int* flag_up, int* flag_down, int seq,
                     void* stream);
int nnconv_halo_wait(const int* flag_from_up, const int* flag_from_down, int seq, void* stream);
/* Peer-visible device memory for the halo exchange: nnconv_ipc_alloc = cudaMalloc (zero-filled) + cudaIpcGetMemHandle
 * (64-byte handle to send to the neighbour processes); nnconv_ipc_open maps a neighbour's allocation for kernels of
 * the CURRENT device (cudaIpcOpenMemHandle with lazy peer access); _close / _free release them.  The only device
 * allocation the library performs on the caller's behalf. */
int nnconv_ipc_alloc(size_t bytes, void** dev_ptr, unsigned char* handle64);
int nnconv_ipc_open(const unsigned char* handle64, void** dev_ptr);
int nnconv_ipc_close(void* dev_ptr);
int nnconv_ipc_free(void* dev_ptr);
/* kernels of the CURRENT device may load / store memory of `peer_device` afterwards (cudaDeviceEnablePeerAccess;
 * needed once per neighbour before nnconv_halo_push writes into its IPC-mapped buffers) */
int nnconv_enable_peer_access(int peer_device);

/* ---- ball-graph construction on the device (replaces np.where(pairwise_distances(pa, pb) <= r), utilities.py:250-255
 * and multipole utilities.py:602-643, plus the attribute gather :269-285 / :672-706), two passes:
 *   nnconv_ball_count: counts[i] = #{j : |pa_i - pb_j| <= radius}        (pa [na,2], pb [nb,2] float64, device)
 *   (the caller turns counts into exclusive offsets)
 *   nnconv_ball_fill:  edges of source i at [offsets[i], ...) in ascending j: row0 = src_base + i, row1 = dst_base + j,
 *                      edge_attr (nullable) = [pa_i, pb_j] (+ [theta_a_i, theta_b_j] when the thetas are given), fp32.
 * Same float64 distance formula as sklearn (see csrc/graph_build.cu); edge order = np.where's row-major order. */
int nnconv_ball_count(const double* pa, int64_t na, const double* pb, int64_t nb, double radius, int* counts, void* stream);
int nnconv_ball_fill(const double* pa, int64_t na, const double* pb, int64_t nb, double radius, const int64_t* offsets,
                     int64_t src_base, int64_t dst_base, int64_t* row0, int64_t* row1, const double* theta_a,
                     const double* theta_b, float* edge_attr, void* stream);

/* ---- fused loss / normaliser epilogue after fc2 (UAI1_full_resolution.py:262-268, utilities.py:87-99,184-199):
 * out, y [batch, n] fp32; mean / std [n] of the UnitGaussianNormalizer (NULL = identity decode).  One pass writes
 * results[0] = mse_loss(out, y), [1] = ||out - y||_1, [2] = sum_b rel-L2 of the DECODED fields, [3] = their mean,
 * and, if grad_l1 != NULL, grad_l1 = grad_scale * sign(out - y) (the backward of results[1]).  ws: 2 + 2*batch floats.
 * Nothing is copied to the host. */
int nnconv_loss_epilogue(const float* out, const float* y, const float* mean, const float* std_, float eps, int batch,
                         int64_t n, float grad_scale, float* grad_l1, float* results, float* ws, void* stream);

/* ---- measurement hook (bench.py): while enabled, every kernel launch is bracketed by CUDA events on its
 * stream; profile_end synchronises the device and returns summed milliseconds / launch counts per kernel
 * class: 0 first MLP layer, 1 hidden-layer GEMM, 2 per-node prologue, 3 per-source Y GEMM (unfused path),
 * 4 contraction+scatter (unfused path), 5 fused persistent application kernel (Y GEMM + contraction).
 * Not thread safe; not for production use. */
#define NNCONV_PROFILE_KINDS 6
int nnconv_profile_begin(void);
int nnconv_profile_end(double* ms_by_kind, int64_t* launches_by_kind, int n_kinds);

/* ---- debugging aid: with NNCONV_TRACE=1 in the environment every tensor-core CTA records
 * {tag, blockIdx, smid, t_start, t_ready, t_end} (globaltimer ns); this copies the records to the host and
 * clears the buffer.  tag: 100 = K=64 GEMM, 101 = hidden GEMM, 200 = contraction. */
int nnconv_debug_trace_dump(unsigned long long* host_rec, unsigned int max_rec, unsigned int* n_out);

/* ---- test hook: occupy `n_ctas` CTA slots (each holding `smem_bytes` of shared memory) for `ns` nanoseconds on
 * `stream` -- used to check that the persistent application kernel tolerates concurrently resident kernels. */
int nnconv_debug_occupy(int n_ctas, int smem_bytes, long long ns, void* stream);

/* ---- unit-test hook for the wgmma GEMM used by the hidden layers and the per-source matrices:
 * C[M,N] (16-bit) = act(A[M,K] * B[N,K]^T + bias); K, N multiples of 64; bias nullable. ------------- */
int nnconv_gemm_16b(int precision, const void* A, int64_t M, int K, const void* B, int N, const float* bias,
                    int relu, void* C, void* stream);

/* ---- unit-test hooks for the backward GEMMs:
 * gemm_tn:  C[M,N] (fp32, ACCUMULATED with atomics) += alpha * sum_{r<R} A[r,m] * B[r,n]   (A [R,lda], B [R,ldb] 16-bit)
 * gemm_16b_ex: nnconv_gemm_16b with ldc, a ReLU-derivative mask (16-bit [M, mask_ld], keep where > 0) and fp32 output */
int nnconv_gemm_tn_16b(int precision, const void* A, int64_t lda, const void* B, int64_t ldb, int64_t R, int M, int N,
                       float* C, int64_t ldc, float alpha, void* stream);
int nnconv_gemm_16b_ex(int precision, const void* A, int64_t M, int K, const void* B, int N, const float* bias, int relu,
                       void* C, int64_t ldc, const void* mask, int64_t mask_ld, int out_f32, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NNCONV_B200_H_ */
