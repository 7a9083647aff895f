// Graph plan: one-time, per edge_index preprocessing for the NNConv hot path.
//
// The reference consumes edge_index [2,E] int64 as produced by np.where(pwd <= r)
// (graph-neural-operator/utilities.py:250-255): grouped by SOURCE node, unsorted in destination.  The
// contraction kernel wants exactly that grouping (all edges of one source share the per-source matrix
// Y_src), so the plan (a) verifies / establishes the source grouping (stable radix sort only when the
// caller's list is not already grouped), (b) compacts the sources that have out-edges, (c) cuts every
// source group into tiles of <= 128 edges (= one 128-row wgmma tile), (d) stores dst as int32 in sorted order
// and 1/max(in_degree,1) for the mean aggregation (PyG scatter_('mean'), empty set -> 0).  Sources and targets are
// counted separately (N_src, N_dst): equal for a square graph, two node sets for a bipartite one (DESIGN 4.10).  Every
// per-source array runs over N_src, the in-degrees and inv_deg over N_dst.
#include <cub/cub.cuh>

#include "common.cuh"
#include "plan.h"

namespace nnc {

namespace {

__global__ void k_count(const int64_t* __restrict__ src, const int64_t* __restrict__ dst, int64_t E, int64_t N_src,
                        int64_t N_dst, int* __restrict__ outdeg, int* __restrict__ indeg, int* __restrict__ flags) {
  int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (e >= E) return;
  int64_t s = src[e], d = dst[e];
  const bool bad_s = s < 0 || s >= N_src, bad_d = d < 0 || d >= N_dst;
  if (bad_s || bad_d) {       // index out of range: flags[1] source row, flags[2] target row
    if (bad_s) atomicOr(&flags[1], 1);
    if (bad_d) atomicOr(&flags[2], 1);
    return;
  }
  atomicAdd(&outdeg[s], 1);
  atomicAdd(&indeg[d], 1);
  if (e > 0 && src[e - 1] > s) atomicOr(&flags[0], 1);   // not grouped-by-source ascending
}

__global__ void k_keys(const int64_t* __restrict__ src, int64_t E, int* __restrict__ keys, int* __restrict__ vals) {
  int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (e >= E) return;
  keys[e] = static_cast<int>(src[e]);
  vals[e] = static_cast<int>(e);
}

__global__ void k_node_flags(const int* __restrict__ outdeg, int64_t N, int* __restrict__ nz, int* __restrict__ nt,
                             int* __restrict__ nu, int* __restrict__ maxdeg) {
  int64_t n = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (n >= N) return;
  int d = outdeg[n];
  nz[n] = d > 0 ? 1 : 0;
  nt[n] = (d + kTileEdges - 1) / kTileEdges;
  nu[n] = (nt[n] + 1) / 2;
  if (d > 0) atomicMax(maxdeg, d);
}

__global__ void k_compact(const int* __restrict__ outdeg, const int* __restrict__ rowptr, const int* __restrict__ cpos,
                          const int* __restrict__ tpos, const int* __restrict__ upos, int64_t N,
                          int* __restrict__ src_nodes, int* __restrict__ group_ptr, int* __restrict__ tile_ptr,
                          int* __restrict__ tile_c, int* __restrict__ tile_e0, int* __restrict__ tile_cnt,
                          int* __restrict__ unit_ptr, int* __restrict__ unit_t, int* __restrict__ unit_u) {
  int64_t n = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (n >= N) return;
  int d = outdeg[n];
  if (d <= 0) return;
  int c = cpos[n], t0 = tpos[n], e0 = rowptr[n];
  src_nodes[c] = static_cast<int>(n);
  group_ptr[c] = e0;
  tile_ptr[c] = t0;
  int nt = (d + kTileEdges - 1) / kTileEdges;
  for (int i = 0; i < nt; ++i) {
    tile_c[t0 + i] = c;
    tile_e0[t0 + i] = e0 + i * kTileEdges;
    tile_cnt[t0 + i] = min(kTileEdges, d - i * kTileEdges);
  }
  const int u0 = upos[n];
  unit_ptr[c] = u0;
  for (int i = 0; i < (nt + 1) / 2; ++i) {
    unit_t[u0 + i] = t0 + 2 * i;
    unit_u[u0 + i] = min(2, nt - 2 * i);
  }
}

__global__ void k_tail(int* group_ptr, int* tile_ptr, int* unit_ptr, const int* cpos, const int* tpos,
                       const int* upos, const int* outdeg, int64_t N, int64_t E, int* counts) {
  // totals = exclusive-scan value at N-1 plus the last element
  int S = cpos[N - 1] + (outdeg[N - 1] > 0 ? 1 : 0);
  int T = tpos[N - 1] + (outdeg[N - 1] + kTileEdges - 1) / kTileEdges;
  const int ntl = (outdeg[N - 1] + kTileEdges - 1) / kTileEdges;
  const int U = upos[N - 1] + (ntl + 1) / 2;
  group_ptr[S] = static_cast<int>(E);
  tile_ptr[S] = T;
  unit_ptr[S] = U;
  counts[0] = S;
  counts[1] = T;
  counts[3] = U;
}

__global__ void k_sorted_dst(const int64_t* __restrict__ dst, const int* __restrict__ perm, int64_t E,
                             int* __restrict__ dst_sorted) {
  int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (p >= E) return;
  int64_t e = perm ? perm[p] : p;
  dst_sorted[p] = static_cast<int>(dst[e]);
}

__global__ void k_inv_deg(const int* __restrict__ indeg, int64_t N, float* __restrict__ inv_deg) {
  int64_t n = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (n >= N) return;
  int d = indeg[n];
  inv_deg[n] = 1.0f / static_cast<float>(d > 1 ? d : 1);
}

size_t cub_scan_bytes(int64_t n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                static_cast<int>(n));
  return b;
}
size_t cub_sort_bytes(int64_t n) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                  static_cast<int*>(nullptr), static_cast<int*>(nullptr), static_cast<int>(n));
  return b;
}

struct PlanLayout {
  // persistent
  int *perm, *dst_sorted, *src_nodes, *group_ptr, *tile_ptr, *tile_c, *tile_e0, *tile_cnt, *unit_ptr, *unit_t, *unit_u;
  float* inv_deg;
  size_t ws_bytes;
};

PlanLayout carve_plan(void* ws, int64_t E, int64_t N_src, int64_t N_dst) {
  Carver c(ws, ~size_t(0));
  PlanLayout L;
  int64_t Smax = (N_src < E ? N_src : E) + 1;
  int64_t Tmax = E / kTileEdges + Smax + 1;
  L.perm = c.take<int>(E + 1);
  L.dst_sorted = c.take<int>(E + 1);
  L.src_nodes = c.take<int>(Smax);
  L.group_ptr = c.take<int>(Smax + 1);
  L.tile_ptr = c.take<int>(Smax + 1);
  L.tile_c = c.take<int>(Tmax);
  L.tile_e0 = c.take<int>(Tmax);
  L.tile_cnt = c.take<int>(Tmax);
  L.unit_ptr = c.take<int>(Smax + 1);
  L.unit_t = c.take<int>(Tmax);
  L.unit_u = c.take<int>(Tmax);
  L.inv_deg = c.take<float>(N_dst + 1);
  L.ws_bytes = c.off;
  return L;
}

struct TmpLayout {
  int *outdeg, *indeg, *rowptr, *nz, *nt, *nu, *cpos, *tpos, *upos, *flags, *counts, *keys_in, *keys_out, *vals_in;
  void* cub_tmp;
  size_t cub_bytes;
  size_t bytes;
};

TmpLayout carve_tmp(void* tmp, int64_t E, int64_t N_src, int64_t N_dst) {
  Carver c(tmp, ~size_t(0));
  TmpLayout L;
  const int64_t N = N_src;     // the per-source arrays
  L.outdeg = c.take<int>(N + 1);
  L.indeg = c.take<int>(N_dst + 1);
  L.rowptr = c.take<int>(N + 1);
  L.nz = c.take<int>(N + 1);
  L.nt = c.take<int>(N + 1);
  L.nu = c.take<int>(N + 1);
  L.upos = c.take<int>(N + 1);
  L.cpos = c.take<int>(N + 1);
  L.tpos = c.take<int>(N + 1);
  L.flags = c.take<int>(8);
  L.counts = c.take<int>(8);
  L.keys_in = c.take<int>(E + 1);
  L.keys_out = c.take<int>(E + 1);
  L.vals_in = c.take<int>(E + 1);
  size_t a = cub_scan_bytes(N + 1), b = cub_sort_bytes(E + 1);
  L.cub_bytes = a > b ? a : b;
  L.cub_tmp = c.take<char>(L.cub_bytes + 256);
  L.bytes = c.off;
  return L;
}

}  // namespace

void plan_sizes(int64_t E, int64_t N_src, int64_t N_dst, size_t* ws_bytes, size_t* tmp_bytes) {
  *ws_bytes = carve_plan(nullptr, E, N_src, N_dst).ws_bytes;
  *tmp_bytes = carve_tmp(nullptr, E, N_src, N_dst).bytes;
}

int plan_build(Plan* P, const int64_t* row0, const int64_t* row1, int64_t E, int64_t N_src, int64_t N_dst, int flow, void* ws,
               size_t ws_bytes, void* tmp, size_t tmp_bytes, cudaStream_t st) {
  NNC_REQUIRE(E >= 0 && N_src >= 1 && N_dst >= 1, NNCONV_ERR_ARG,
              "plan: need E >= 0, n_src >= 1 and n_dst >= 1 (got E=%lld n_src=%lld n_dst=%lld)", (long long)E,
              (long long)N_src, (long long)N_dst);
  NNC_REQUIRE(E < (int64_t(1) << 31) - 256 && N_src < (int64_t(1) << 31) - 256 && N_dst < (int64_t(1) << 31) - 256,
              NNCONV_ERR_UNSUPPORTED, "plan: E and N must fit int32");
  NNC_REQUIRE(flow == 0 || flow == 1, NNCONV_ERR_ARG, "plan: flow must be 0 (source_to_target) or 1");
  const int64_t N = N_src;     // every per-source array and kernel below
  PlanLayout L = carve_plan(ws, E, N_src, N_dst);
  TmpLayout T = carve_tmp(tmp, E, N_src, N_dst);
  NNC_REQUIRE(ws != nullptr && tmp != nullptr, NNCONV_ERR_ARG, "plan: null workspace");
  NNC_REQUIRE(L.ws_bytes <= ws_bytes && T.bytes <= tmp_bytes, NNCONV_ERR_WORKSPACE,
              "plan: workspace too small (need %zu + %zu bytes)", L.ws_bytes, T.bytes);
  // flow = source_to_target (PyG default, reference checkpoints): gather from row 0, aggregate at row 1
  const int64_t* src = flow == 0 ? row0 : row1;
  const int64_t* dst = flow == 0 ? row1 : row0;

  P->E = E;
  P->N_src = N_src;
  P->N_dst = N_dst;
  P->flow = flow;
  P->perm = nullptr;
  P->dst_sorted = L.dst_sorted;
  P->src_nodes = L.src_nodes;
  P->group_ptr = L.group_ptr;
  P->tile_ptr = L.tile_ptr;
  P->tile_c = L.tile_c;
  P->tile_e0 = L.tile_e0;
  P->tile_cnt = L.tile_cnt;
  P->unit_ptr = L.unit_ptr;
  P->unit_t = L.unit_t;
  P->unit_u = L.unit_u;
  P->n_units = 0;
  P->inv_deg = L.inv_deg;
  P->n_src = 0;
  P->n_tiles = 0;
  P->max_out_deg = 0;
  P->src_sorted = 1;

  const int TB = 256;
  NNC_CHECK_CUDA(cudaMemsetAsync(T.outdeg, 0, (N + 1) * sizeof(int), st));
  NNC_CHECK_CUDA(cudaMemsetAsync(T.indeg, 0, (N_dst + 1) * sizeof(int), st));
  NNC_CHECK_CUDA(cudaMemsetAsync(T.flags, 0, 8 * sizeof(int), st));
  NNC_CHECK_CUDA(cudaMemsetAsync(T.counts, 0, 8 * sizeof(int), st));
  if (E > 0) {
    k_count<<<(unsigned)ceil_div64(E, TB), TB, 0, st>>>(src, dst, E, N_src, N_dst, T.outdeg, T.indeg, T.flags);
    NNC_CHECK_LAUNCH();
  }
  int h_flags[3] = {0, 0, 0};
  NNC_CHECK_CUDA(cudaMemcpyAsync(h_flags, T.flags, 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
  NNC_CHECK_CUDA(cudaStreamSynchronize(st));
  // the rows are named as the caller passes them: flow 0 gathers from row 0, flow 1 from row 1
  NNC_REQUIRE(h_flags[1] == 0, NNCONV_ERR_ARG, "plan: edge_index row %d (source row) has entries outside [0, %lld)",
              flow == 0 ? 0 : 1, (long long)N_src);
  NNC_REQUIRE(h_flags[2] == 0, NNCONV_ERR_ARG, "plan: edge_index row %d (target row) has entries outside [0, %lld)",
              flow == 0 ? 1 : 0, (long long)N_dst);
  if (h_flags[0] != 0 && E > 0) {   // not grouped by source: stable sort by source, keep the permutation
    P->src_sorted = 0;
    P->perm = L.perm;
    k_keys<<<(unsigned)ceil_div64(E, TB), TB, 0, st>>>(src, E, T.keys_in, T.vals_in);
    NNC_CHECK_LAUNCH();
    size_t cb = T.cub_bytes;
    int bits = 1;
    while ((int64_t(1) << bits) < N) ++bits;
    NNC_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(T.cub_tmp, cb, T.keys_in, T.keys_out, T.vals_in, L.perm,
                                                   static_cast<int>(E), 0, bits, st));
  }
  size_t cb = T.cub_bytes;
  NNC_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(T.cub_tmp, cb, T.outdeg, T.rowptr, static_cast<int>(N), st));
  k_node_flags<<<(unsigned)ceil_div64(N, TB), TB, 0, st>>>(T.outdeg, N, T.nz, T.nt, T.nu, T.counts + 2);
  NNC_CHECK_LAUNCH();
  cb = T.cub_bytes;
  NNC_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(T.cub_tmp, cb, T.nz, T.cpos, static_cast<int>(N), st));
  cb = T.cub_bytes;
  NNC_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(T.cub_tmp, cb, T.nt, T.tpos, static_cast<int>(N), st));
  cb = T.cub_bytes;
  NNC_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(T.cub_tmp, cb, T.nu, T.upos, static_cast<int>(N), st));
  k_compact<<<(unsigned)ceil_div64(N, TB), TB, 0, st>>>(T.outdeg, T.rowptr, T.cpos, T.tpos, T.upos, N, L.src_nodes,
                                                        L.group_ptr, L.tile_ptr, L.tile_c, L.tile_e0, L.tile_cnt,
                                                        L.unit_ptr, L.unit_t, L.unit_u);
  NNC_CHECK_LAUNCH();
  k_tail<<<1, 1, 0, st>>>(L.group_ptr, L.tile_ptr, L.unit_ptr, T.cpos, T.tpos, T.upos, T.outdeg, N, E, T.counts);
  NNC_CHECK_LAUNCH();
  if (E > 0) {
    k_sorted_dst<<<(unsigned)ceil_div64(E, TB), TB, 0, st>>>(dst, P->perm, E, L.dst_sorted);
    NNC_CHECK_LAUNCH();
  }
  k_inv_deg<<<(unsigned)ceil_div64(N_dst, TB), TB, 0, st>>>(T.indeg, N_dst, L.inv_deg);
  NNC_CHECK_LAUNCH();
  int h_counts[4] = {0, 0, 0, 0};
  NNC_CHECK_CUDA(cudaMemcpyAsync(h_counts, T.counts, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  NNC_CHECK_CUDA(cudaStreamSynchronize(st));
  P->n_src = h_counts[0];
  P->n_tiles = h_counts[1];
  P->max_out_deg = h_counts[2];
  P->n_units = h_counts[3];
  return NNCONV_OK;
}

int check_bipartite_root(const Plan* P, const float* root, unsigned node_flags) {
  NNC_REQUIRE(P->N_src == P->N_dst || (root == nullptr && (node_flags & NNCONV_APPLY_RESIDUAL) == 0), NNCONV_ERR_ARG,
              "bipartite plan (n_src %lld, n_dst %lld): pass root = NULL and add x_dst root + bias with "
              "nnconv_root_term; NNCONV_APPLY_RESIDUAL needs a square plan", (long long)P->N_src, (long long)P->N_dst);
  return NNCONV_OK;
}

}  // namespace nnc
