// CUDA-core kernels of the NNConv path:
//   * parameter preparation (pad / convert / permute the last Linear layer into W3p)
//   * first edge-MLP layer (k_in is 4..6: no tensor-core shape) fused with the edge permutation
//   * per-node prologue: out = x@root + bias, compact fp16 copy of x, c = x @ B3
//   * a plain fp32 NT-GEMM with three epilogues: the PREC_FP32 path (any shape) of the hidden layers,
//     the per-source matrices Y and the per-edge contraction + scatter.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "act.cuh"
#include "common.cuh"
#include "kernels.h"

namespace nnc {

namespace {

template <typename T>
__device__ __forceinline__ T cvt(float v);
template <>
__device__ __forceinline__ float cvt<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half cvt<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 cvt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// dst[Rp x Cp] (T) <- src[R x C] fp32, zero padded
template <typename T>
__global__ void k_pad_convert(const float* __restrict__ src, int R, int C, T* __restrict__ dst, int Rp, int Cp) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(Rp) * Cp) return;
  int r = static_cast<int>(i / Cp), c = static_cast<int>(i % Cp);
  float v = (r < R && c < C) ? src[static_cast<int64_t>(r) * C + c] : 0.f;
  dst[i] = cvt<T>(v);
}

// W3p[(o*Kp + k) * cin_p + i] = W_L[(i*cout + o) * K + k]   (W_L is the last Linear: [cin*cout, K])
template <typename T>
__global__ void k_w3p(const float* __restrict__ WL, int cin, int cout, int K, int Kp, int cin_p, T* __restrict__ dst) {
  int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  int64_t total = static_cast<int64_t>(cout) * Kp * cin_p;
  if (idx >= total) return;
  int i = static_cast<int>(idx % cin_p);
  int64_t ok = idx / cin_p;
  int k = static_cast<int>(ok % Kp);
  int o = static_cast<int>(ok / Kp);
  float v = (i < cin && k < K) ? WL[(static_cast<int64_t>(i) * cout + o) * K + k] : 0.f;
  dst[idx] = cvt<T>(v);
}

// W3q[(k*cout + o) * cin_p + i] = W_L[(i*cout + o) * K + k]  /  W3t[i * (Kp*cout) + (k*cout + o)] = same
template <typename T>
__global__ void k_w3q(const float* __restrict__ WL, int cin, int cout, int K, int Kp, int cin_p, int transposed,
                      T* __restrict__ dst) {
  int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t NY = static_cast<int64_t>(Kp) * cout;
  if (idx >= NY * cin_p) return;
  int i;
  int64_t ko;
  if (transposed) { i = static_cast<int>(idx / NY); ko = idx % NY; }
  else { i = static_cast<int>(idx % cin_p); ko = idx / cin_p; }
  const int o = static_cast<int>(ko % cout), k = static_cast<int>(ko / cout);
  const float v = (i < cin && k < K) ? WL[(static_cast<int64_t>(i) * cout + o) * K + k] : 0.f;
  dst[idx] = cvt<T>(v);
}

// dst[c, r] (Cp x Rp) = src[r, c] (R x C), zero padded
template <typename T>
__global__ void k_transpose_pad(const float* __restrict__ src, int R, int C, T* __restrict__ dst, int Rp, int Cp) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(Rp) * Cp) return;
  const int c = static_cast<int>(i / Rp), r = static_cast<int>(i % Rp);
  dst[i] = cvt<T>((r < R && c < C) ? src[static_cast<int64_t>(r) * C + c] : 0.f);
}

// ---- PREC_F16X2 weight images: K is tripled, [hi(W) | lo(W) | hi(W)], to pair with activations read as
// [hi(a) | hi(a) | lo(a)]:  a.W ~= hi*hi + hi*lo + lo*hi  (the dropped lo*lo term is 2^-22 relative)
__device__ __forceinline__ __half split_part(float v, int part) {
  const __half hi = __float2half_rn(v);
  return part == 1 ? __float2half_rn(v - __half2float(hi)) : hi;
}
__global__ void k_pad_convert_split3(const float* __restrict__ src, int R, int C, __half* __restrict__ dst, int Rp,
                                     int Cp, const float* __restrict__ scale) {
  int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(Rp) * 3 * Cp) return;
  const int r = static_cast<int>(i / (3 * Cp)), cc = static_cast<int>(i % (3 * Cp));
  const int part = cc / Cp, c = cc % Cp;
  const float sc = scale ? scale[0] : 1.f;
  const float v = (r < R && c < C) ? src[static_cast<int64_t>(r) * C + c] * sc : 0.f;
  dst[i] = split_part(v, part);
}
// scale2[0] = 2^k with max|src| * 2^k in [0.5, 1) (1 for an all-zero / non-finite matrix), scale2[1] = 2^-k
__global__ void k_absmax_bits(const float* __restrict__ src, int64_t n, unsigned int* __restrict__ out) {
  float m = 0.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float a = fabsf(src[i]);
    if (a <= 3.0e38f) m = fmaxf(m, a);
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}
__global__ void k_pow2_from_max(float* scale2) {
  const float m = scale2[0];
  float s = 1.f;
  if (m > 0.f && m <= 3.0e38f) {
    int e;
    frexpf(m, &e);                  // m = f * 2^e, f in [0.5, 1)  ->  m * 2^-e in [0.5, 1)
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
    s = ldexpf(1.f, -e);
  }
  scale2[0] = s;
  scale2[1] = 1.f / s;
}
// *sticky += *counter: folds one pass's fp16 range counter into a word that outlives the pass's workspace
__global__ void k_overflow_accumulate(const int* __restrict__ counter, int* __restrict__ sticky) {
  const int v = *counter;
  if (v != 0) atomicAdd(sticky, v);
}
__global__ void k_w3p_split3(const float* __restrict__ WL, int cin, int cout, int K, int Kp, int cin_p,
                             __half* __restrict__ dst, const float* __restrict__ scale) {
  int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t total = static_cast<int64_t>(cout) * Kp * 3 * cin_p;
  if (idx >= total) return;
  const int ii = static_cast<int>(idx % (3 * cin_p));
  const int part = ii / cin_p, i = ii % cin_p;
  const int64_t ok = idx / (3 * cin_p);
  const int k = static_cast<int>(ok % Kp);
  const int o = static_cast<int>(ok / Kp);
  const float v = (i < cin && k < K) ? WL[(static_cast<int64_t>(i) * cout + o) * K + k] * (scale ? scale[0] : 1.f) : 0.f;
  dst[idx] = split_part(v, part);
}
// backward images of the split last Linear (see k_w3q), pre-scaled like W3p:
//   transposed == 0: W3q [Kp*cout, 3*cin_p], column part*cin_p + i;  1: W3t [cin_p, 3*Kp*cout], column part*NY + (k*cout + o)
__global__ void k_w3q_split3(const float* __restrict__ WL, int cin, int cout, int K, int Kp, int cin_p, int transposed,
                             __half* __restrict__ dst, const float* __restrict__ scale) {
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t NY = static_cast<int64_t>(Kp) * cout;
  if (idx >= 3 * NY * cin_p) return;
  int i, part;
  int64_t ko;
  if (transposed) {
    i = static_cast<int>(idx / (3 * NY));
    const int64_t cc = idx % (3 * NY);
    part = static_cast<int>(cc / NY);
    ko = cc % NY;
  } else {
    const int ii = static_cast<int>(idx % (3 * cin_p));
    part = ii / cin_p;
    i = ii % cin_p;
    ko = idx / (3 * cin_p);
  }
  const int o = static_cast<int>(ko % cout), k = static_cast<int>(ko / cout);
  const float v = (i < cin && k < K) ? WL[(static_cast<int64_t>(i) * cout + o) * K + k] * scale[0] : 0.f;
  dst[idx] = split_part(v, part);
}
// dst[c, part*Rp + r] ([Cp, 3*Rp]) = split part of scale * src[r, c] (src [R, C]), zero padded
__global__ void k_transpose_pad_split3(const float* __restrict__ src, int R, int C, __half* __restrict__ dst, int Rp,
                                       int Cp, const float* __restrict__ scale) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(Cp) * 3 * Rp) return;
  const int c = static_cast<int>(i / (3 * Rp)), rr = static_cast<int>(i % (3 * Rp));
  const int part = rr / Rp, r = rr % Rp;
  const float v = (r < R && c < C) ? src[static_cast<int64_t>(r) * C + c] * scale[0] : 0.f;
  dst[i] = split_part(v, part);
}

// First layer: h1[p, j] = relu(b1[j] + sum_c W1[j, c] * edge_attr[perm[p], c]),  j < kp1 (pad rows of W1/b1 are 0)
// identity (single-Linear MLP): h[p, j] = edge_attr[perm[p], j] (zero padded), no ReLU.
// overflow (fp16 output, nullable): +1 per block that wrote a value beyond the fp16 range or NaN.  Counted here, at the
// writer: the next layer's GEMM would turn an inf into NaN, which its ReLU turns into 0 before its own range check.
// k_edge_layer1 is the ReLU kernel; k_edge_layer1_act<ACT> applies another hidden activation (act.cuh, act_range for
// the range check) in its place, with its parameter block as the last argument; a 16-bit CLAMP output follows the
// store rule of act.cuh (act_store16).
constexpr int kL1Edges = 32;
template <int ACT, typename T>
__device__ __forceinline__ void edge_layer1(const float* __restrict__ edge_attr, const int* __restrict__ perm,
                                            int64_t e_begin, int64_t e_count, int k_in, const float* __restrict__ W1,
                                            const float* __restrict__ b1, int kp1, int identity, T* __restrict__ out,
                                            int64_t chunk_rows_pad, int64_t out_row0, int* __restrict__ overflow,
                                            const ActParams& act_p) {
  constexpr bool kRangeCheck = std::is_same<T, __half>::value;
  bool bad = false;
  extern __shared__ float sm[];
  float* s_ea = sm;                       // [kL1Edges][k_in]
  int64_t p0 = static_cast<int64_t>(blockIdx.x) * kL1Edges;
  int64_t rem = e_count - p0;
  int ne = rem < kL1Edges ? static_cast<int>(rem) : kL1Edges;
  for (int i = threadIdx.x; i < ne * k_in; i += blockDim.x) {
    int e = i / k_in, c = i % k_in;
    int64_t p = e_begin + p0 + e;
    int64_t src = perm ? perm[p] : p;
    s_ea[i] = edge_attr[src * k_in + c];
  }
  __syncthreads();
  // row-major [rows, kp1] or chunk-major [kp1/64][chunk_rows_pad][64] (see gemm_tc.cu)
  auto oidx = [&](int e, int j) -> int64_t {
    return chunk_rows_pad > 0 ? (static_cast<int64_t>(j >> 6) * chunk_rows_pad + out_row0 + p0 + e) * 64 + (j & 63)
                              : (p0 + e) * static_cast<int64_t>(kp1) + j;
  };
  for (int j = threadIdx.x; j < kp1; j += blockDim.x) {
    if (identity) {
      for (int e = 0; e < ne; ++e) {
        const float v = j < k_in ? s_ea[e * k_in + j] : 0.f;
        if (kRangeCheck) bad |= !(fabsf(v) <= 65504.f);
        out[oidx(e, j)] = cvt<T>(v);
      }
      continue;
    }
    float w[16];
    const bool small = k_in <= 16;
    if (small) {
#pragma unroll
      for (int c = 0; c < 16; ++c) w[c] = c < k_in ? W1[static_cast<int64_t>(j) * k_in + c] : 0.f;
    }
    float bj = b1[j];
    for (int e = 0; e < ne; ++e) {
      float acc = bj;
      if (small) {
#pragma unroll
        for (int c = 0; c < 16; ++c)
          if (c < k_in) acc = fmaf(w[c], s_ea[e * k_in + c], acc);
      } else {
        for (int c = 0; c < k_in; ++c) acc = fmaf(W1[static_cast<int64_t>(j) * k_in + c], s_ea[e * k_in + c], acc);
      }
      if (ACT == ACT_RELU) {
        const float v = fmaxf(acc, 0.f);
        if (kRangeCheck) bad |= !(v <= 65504.f);
        out[oidx(e, j)] = cvt<T>(v);
      } else {
        float v = act_fwd<ACT>(acc, act_p);
        if (kRangeCheck) bad |= !(act_range<ACT>(acc, v) <= 65504.f);
        if (std::is_same<T, __half>::value) v = act_store16<ACT, 0>(v, act_p);
        if (std::is_same<T, __nv_bfloat16>::value) v = act_store16<ACT, 1>(v, act_p);
        out[oidx(e, j)] = cvt<T>(v);
      }
    }
  }
  if (kRangeCheck && overflow != nullptr) {
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicAdd(overflow, 1);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
k_edge_layer1(const float* __restrict__ edge_attr, const int* __restrict__ perm, int64_t e_begin, int64_t e_count,
              int k_in, const float* __restrict__ W1, const float* __restrict__ b1, int kp1, int identity,
              T* __restrict__ out, int64_t chunk_rows_pad, int64_t out_row0, int* __restrict__ overflow) {
  edge_layer1<ACT_RELU>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1, identity, out, chunk_rows_pad, out_row0,
                        overflow, ActParams{});
}

template <int ACT, typename T>
__global__ void __launch_bounds__(256)
k_edge_layer1_act(const float* __restrict__ edge_attr, const int* __restrict__ perm, int64_t e_begin, int64_t e_count,
                  int k_in, const float* __restrict__ W1, const float* __restrict__ b1, int kp1, T* __restrict__ out,
                  int64_t chunk_rows_pad, int64_t out_row0, int* __restrict__ overflow, ActParams act_p) {
  edge_layer1<ACT>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1, 0, out, chunk_rows_pad, out_row0, overflow,
                   act_p);
}

// ---- first edge-MLP layer on the tensor cores with fp32-grade inputs -------------------------------
// v = hi + lo with hi = T(v), lo = T(v - hi): two 16-bit values carry ~22 mantissa bits.  With
//   A1[p, :] = [hi(ea) | lo(ea) | hi(ea) | 1 | 1 | 0...]            (64 columns, one wgmma K block)
//   B1[j, :] = [hi(W1_j) | hi(W1_j) | lo(W1_j) | hi(b1_j) | lo(b1_j) | 0...]
// A1 . B1^T = ea . W1_j + b1_j up to the dropped lo*lo terms (2^-22 relative): the first Linear keeps
// fp32-grade accuracy although it runs as a 16-bit wgmma GEMM (utilities.py:223-227, first layer).
template <typename T>
__device__ __forceinline__ float as_float(T v);
template <>
__device__ __forceinline__ float as_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ float as_float<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float as_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__global__ void k_build_a1(const float* __restrict__ edge_attr, const int* __restrict__ perm, int64_t e_begin,
                           int64_t e_count, int k_in, T* __restrict__ A1) {
  int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;   // one thread per 8 columns
  int64_t p = idx >> 3;
  if (p >= e_count) return;
  int c0 = static_cast<int>(idx & 7) * 8;
  int64_t src = perm ? perm[e_begin + p] : (e_begin + p);
  const float* ea = edge_attr + src * k_in;
  T v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = c0 + i;
    float out = 0.f;
    if (c < 3 * k_in) {
      float a = ea[c % k_in];
      T hi = cvt<T>(a);
      out = (c >= k_in && c < 2 * k_in) ? (a - as_float<T>(hi)) : as_float<T>(hi);
    } else if (c < 3 * k_in + 2) {
      out = 1.f;
    }
    v[i] = cvt<T>(out);
  }
  *reinterpret_cast<uint4*>(A1 + p * 64 + c0) = *reinterpret_cast<const uint4*>(v);
}

template <typename T>
__global__ void k_w1aug(const float* __restrict__ W1, const float* __restrict__ b1, int k1, int kp1, int k_in,
                        T* __restrict__ dst) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= kp1 * 64) return;
  int j = idx / 64, c = idx % 64;
  float out = 0.f;
  if (j < k1) {
    if (c < 3 * k_in) {
      float w = W1[j * k_in + (c % k_in)];
      T hi = cvt<T>(w);
      out = (c >= 2 * k_in) ? (w - as_float<T>(hi)) : as_float<T>(hi);
    } else if (c < 3 * k_in + 2) {
      float b = b1[j];
      T hi = cvt<T>(b);
      out = (c == 3 * k_in) ? as_float<T>(hi) : (b - as_float<T>(hi));
    }
  }
  dst[idx] = cvt<T>(out);
}

// out[n, o] = bias[o] + sum_i x[n, i] root[i, o]   (graph-neural-operator/nn_conv.py:277-282), or 0.
// node_flags (nnconv_b200.h NNCONV_APPLY_*): RELU_IN reads max(x, 0) -- the caller hands over the PRE-activation of the
// previous layer -- and RESIDUAL (cin == cout) adds that input row to the output row, so that one V-cycle step
// x <- relu(x + conv(x))  (multipole-graph-neural-operator/neurips1_MGKN.py:76) needs no elementwise kernel of its own.
__device__ __forceinline__ void out_init_rows(const float* __restrict__ x, const float* __restrict__ root,
                                              const float* __restrict__ bias, int64_t N, int cin, int cout,
                                              float* __restrict__ out, unsigned node_flags, int64_t row_block, float* sx) {
  const int npb = blockDim.y;
  int64_t n = row_block * npb + threadIdx.y;
  float* myx = sx + threadIdx.y * cin;
  const bool relu_in = (node_flags & 1u) != 0, residual = (node_flags & 2u) != 0;
  if ((root != nullptr || residual) && n < N)
    for (int i = threadIdx.x; i < cin; i += blockDim.x) {
      const float v = x[n * cin + i];
      myx[i] = relu_in ? fmaxf(v, 0.f) : v;
    }
  __syncthreads();
  if (n >= N) return;
  for (int o = threadIdx.x; o < cout; o += blockDim.x) {
    float acc = bias ? bias[o] : 0.f;
    if (residual) acc += myx[o];
    if (root)
      for (int i = 0; i < cin; ++i) acc = fmaf(myx[i], root[i * cout + o], acc);
    out[n * cout + o] = acc;
  }
}

__global__ void k_out_init(const float* __restrict__ x, const float* __restrict__ root, const float* __restrict__ bias,
                           int64_t N, int cin, int cout, float* __restrict__ out, unsigned node_flags) {
  extern __shared__ float sx[];   // [nodes_per_block][cin]
  out_init_rows(x, root, bias, N, cin, cout, out, node_flags, blockIdx.x, sx);
}

// out[n, o] += bias[o] + sum_i x[n, i] root[i, o]: the root term of a bipartite application (x = x_dst), added after
// its messages.  The sum is out_init_rows' (same order), so a probe exact in fp32 gets the square conv's bits.
__global__ void k_root_add(const float* __restrict__ x, const float* __restrict__ root, const float* __restrict__ bias,
                           int64_t N, int cin, int cout, float* __restrict__ out) {
  extern __shared__ float sx[];   // [nodes_per_block][cin]
  const int64_t n = static_cast<int64_t>(blockIdx.x) * blockDim.y + threadIdx.y;
  float* myx = sx + threadIdx.y * cin;
  if (root != nullptr && n < N)
    for (int i = threadIdx.x; i < cin; i += blockDim.x) myx[i] = x[n * cin + i];
  __syncthreads();
  if (n >= N) return;
  for (int o = threadIdx.x; o < cout; o += blockDim.x) {
    float acc = bias ? bias[o] : 0.f;
    if (root)
      for (int i = 0; i < cin; ++i) acc = fmaf(myx[i], root[i * cout + o], acc);
    out[n * cout + o] += acc;
  }
}

// per compact source c: Xc[c, :] = x[src_nodes[c], :] / xs[c] (converted, zero padded to cin_p),
//                       cvec[c, o] = sum_i x[n, i] * B3[i, o]       (bias of the last Linear, reassociated)
// xs[c] (16-bit paths only) = the power of two >= max_i |x[n, i]| (1 for an all-zero row): the contraction is
// linear in x, so the operand row is normalised to (0.5, 1] -- exactly, the scale only touches the exponent --
// and the epilogue multiplies the accumulator by xs[c].  Without it node features beyond the fp16 range
// (65504; an untrained MGKN V-cycle reaches 5e5 after 4 depth iterations) turned into inf/NaN.
// SPLIT (PREC_F16X2): Xc row = [hi | hi | lo] of the normalised row (3 * cin_p columns).
template <typename T, int SPLIT>
__device__ __forceinline__ void src_prep_rows(const float* __restrict__ x, const int* __restrict__ src_nodes, int S, int cin,
                                              int cin_p, int cout, const float* __restrict__ B3, T* __restrict__ Xc,
                                              float* __restrict__ cvec, float* __restrict__ xs, unsigned node_flags,
                                              int row_block, float* sx) {
  const int npb = blockDim.y;
  int c = row_block * npb + threadIdx.y;
  float* myx = sx + threadIdx.y * cin;
  int n = c < S ? src_nodes[c] : 0;
  const bool relu_in = (node_flags & 1u) != 0;
  if (c < S)
    for (int i = threadIdx.x; i < cin; i += blockDim.x) {
      const float v = x[static_cast<int64_t>(n) * cin + i];
      myx[i] = relu_in ? fmaxf(v, 0.f) : v;
    }
  __syncthreads();
  if (c >= S) return;
  float inv = 1.f;
  if (xs != nullptr) {
    float m = 0.f;
    for (int i = 0; i < cin; ++i) m = fmaxf(m, fabsf(myx[i]));
    float sc = 1.f;
    if (m > 0.f && m <= 3.0e38f) {                 // finite, non-zero: round up to a power of two
      int e;
      const float f = frexpf(m, &e);               // m = f * 2^e, f in [0.5, 1)
      e = f == 0.5f ? e - 1 : e;
      e = e < -100 ? -100 : (e > 126 ? 126 : e);
      sc = ldexpf(1.f, e);
    }
    inv = 1.f / sc;                                // exact (power of two)
    if (threadIdx.x == 0) xs[c] = sc;
  }
  if (SPLIT) {
    for (int i = threadIdx.x; i < cin_p; i += blockDim.x) {
      const float v = i < cin ? myx[i] * inv : 0.f;
      const T hi = cvt<T>(v);
      T* row = Xc + static_cast<int64_t>(c) * 3 * cin_p;
      row[i] = hi;
      row[cin_p + i] = hi;
      row[2 * cin_p + i] = cvt<T>(v - as_float<T>(hi));
    }
  } else {
    for (int i = threadIdx.x; i < cin_p; i += blockDim.x)
      Xc[static_cast<int64_t>(c) * cin_p + i] = cvt<T>(i < cin ? myx[i] * inv : 0.f);
  }
  for (int o = threadIdx.x; o < cout; o += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < cin; ++i) acc = fmaf(myx[i], B3[i * cout + o], acc);
    cvec[static_cast<int64_t>(c) * cout + o] = acc;
  }
}

template <typename T, int SPLIT = 0>
__global__ void k_src_prep(const float* __restrict__ x, const int* __restrict__ src_nodes, int S, int cin, int cin_p,
                           int cout, const float* __restrict__ B3, T* __restrict__ Xc, float* __restrict__ cvec,
                           float* __restrict__ xs, unsigned node_flags) {
  extern __shared__ float sx[];
  src_prep_rows<T, SPLIT>(x, src_nodes, S, cin, cin_p, cout, B3, Xc, cvec, xs, node_flags, blockIdx.x, sx);
}

// One launch for everything a 16-bit application needs before its contractions: blocks [0, g_out) initialise the
// output rows, blocks [g_out, g_out + g_src) prepare the source rows, and the grid clears the batch flags of the
// application (cntY / cntC / okY / okC / cntU [n_batches] at stride flags_stride; a grid-stride loop, because the
// batches of many streamed chunks are not bounded by the source count that sizes the grid) -- in the launch-bound
// MGKN regime (52 dependent applications per forward) every launch removed from the chain counts.
// MAX (aggr = max): the same grid also clears the [N, cout] keys the scatter epilogues reduce into.
template <typename T, int SPLIT = 0, bool MAX = false>
__global__ void k_node_prep(const float* __restrict__ x, const float* __restrict__ root, const float* __restrict__ bias,
                            int64_t N, float* __restrict__ out, int g_out, const int* __restrict__ src_nodes, int S, int cin,
                            int cin_p, int cout, const float* __restrict__ B3, T* __restrict__ Xc, float* __restrict__ cvec,
                            float* __restrict__ xs, int* __restrict__ flags, int flags_stride, int n_batches,
                            unsigned node_flags, unsigned long long* __restrict__ keys) {
  extern __shared__ float sx[];
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int64_t gid = static_cast<int64_t>(blockIdx.x) * (blockDim.x * blockDim.y) + tid;
  const int64_t n_threads = static_cast<int64_t>(gridDim.x) * (blockDim.x * blockDim.y);
  for (int64_t i = gid; i < n_batches; i += n_threads) {
#pragma unroll
    for (int j = 0; j < 5; ++j) flags[j * flags_stride + i] = 0;
  }
  if constexpr (MAX) {
    for (int64_t i = gid; i < N * cout; i += n_threads) keys[i] = 0ull;
  }
  if (static_cast<int>(blockIdx.x) < g_out)
    out_init_rows(x, root, bias, N, cin, cout, out, node_flags, blockIdx.x, sx);
  else
    src_prep_rows<T, SPLIT>(x, src_nodes, S, cin, cin_p, cout, B3, Xc, cvec, xs, node_flags,
                            static_cast<int>(blockIdx.x) - g_out, sx);
}

// ------------------------------------------------------------------------------------------------
// fp32 NT GEMM, 64x64x16 tiles, 256 threads, 4x4 register blocking.   C = A[M,K] * B[N,K]^T
// ------------------------------------------------------------------------------------------------
// EPI_BIAS_ACT + ACT: bias and another hidden activation (act.cuh) where EPI_BIAS_RELU applies the ReLU
enum { EPI_STORE = 0, EPI_BIAS_RELU = 1, EPI_SCATTER = 2, EPI_SCATTER_MAX = 3, EPI_BIAS_ACT = 8 };

struct SgemmArgs {
  const float* A;
  int64_t lda;
  const float* B;
  int64_t ldb;
  float* C;
  int64_t ldc;
  int M, N, K;
  const float* bias;   // EPI_BIAS_RELU, EPI_BIAS_ACT + ACT
  // EPI_SCATTER (grid.x = tile): A rows = h rows of the tile, B = Y of the tile's source
  const int *tile_c, *tile_e0, *tile_cnt, *dst_sorted;
  const float *inv_deg, *cvec;
  int tile_begin, c0;
  int64_t y_stride;    // elements between consecutive sources in Y
  // EPI_SCATTER_MAX (aggr = max): the rows reduce keys (common.cuh max_key) into keys [N, ldc] instead of adding to C
  unsigned long long* keys;
  const int* perm;
  ActParams act_p;     // EPI_BIAS_ACT + ACT
};

template <int EPI>
__global__ void __launch_bounds__(256) k_sgemm_nt(SgemmArgs a) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const float* A = a.A;
  const float* B = a.B;
  int M = a.M;
  int n0 = blockIdx.y * 64;
  int c = 0, e0 = 0;
  int m_base = 0;
  if (EPI == EPI_SCATTER || EPI == EPI_SCATTER_MAX) {
    int t = a.tile_begin + blockIdx.x / 2;
    c = a.tile_c[t];
    e0 = a.tile_e0[t];
    M = a.tile_cnt[t];
    m_base = (blockIdx.x % 2) * 64;
    if (m_base >= M) return;
    A = a.A + static_cast<int64_t>(e0) * a.lda;
    B = a.B + static_cast<int64_t>(c - a.c0) * a.y_stride;
  } else {
    m_base = blockIdx.x * 64;
  }
  float acc[4][4] = {};
  for (int k0 = 0; k0 < a.K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      int r = i / 16, kk = i % 16;
      int gm = m_base + r, gn = n0 + r, gk = k0 + kk;
      As[kk][r] = (gm < M && gk < a.K) ? A[static_cast<int64_t>(gm) * a.lda + gk] : 0.f;
      Bs[kk][r] = (gn < a.N && gk < a.K) ? B[static_cast<int64_t>(gn) * a.ldb + gk] : 0.f;
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
    int gm = m_base + ty * 4 + i;
    if (gm >= M) continue;
    if (EPI == EPI_SCATTER_MAX) {
      const int d = a.dst_sorted[e0 + gm];
      const uint32_t ce = caller_edge(a.perm, e0 + gm);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gn = n0 + tx * 4 + j;
        if (gn < a.N)
          atomicMax(&a.keys[static_cast<int64_t>(d) * a.ldc + gn],
                    max_key(acc[i][j] + a.cvec[static_cast<int64_t>(c) * a.N + gn], ce));
      }
    } else if (EPI == EPI_SCATTER) {
      int d = a.dst_sorted[e0 + gm];
      float sc = a.inv_deg ? a.inv_deg[d] : 1.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int gn = n0 + tx * 4 + j;
        if (gn < a.N) {
          float v = (acc[i][j] + a.cvec[static_cast<int64_t>(c) * a.N + gn]) * sc;
          atomicAdd(&a.C[static_cast<int64_t>(d) * a.ldc + gn], v);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int gn = n0 + tx * 4 + j;
        if (gn < a.N) {
          float v = acc[i][j];
          if (EPI == EPI_BIAS_RELU) v = fmaxf(v + a.bias[gn], 0.f);
          if constexpr (EPI > EPI_BIAS_ACT) v = act_fwd<EPI - EPI_BIAS_ACT>(v + a.bias[gn], a.act_p);
          a.C[static_cast<int64_t>(gm) * a.ldc + gn] = v;
        }
      }
    }
  }
}

// ---- formulation B application: one warp per edge, out[dst_e, :] += (x_src . K_e) / deg.
// K_e is [cin, cout] 16-bit row-major (8 KB at 64 x 64): for a fixed input channel i the 32 lanes read one
// contiguous row of cout 16-bit values (lane -> 2 columns), so the pass streams Kmat at full sector efficiency.
template <typename T2>
__device__ __forceinline__ float2 cvt2(T2 v);
template <>
__device__ __forceinline__ float2 cvt2<__half2>(__half2 v) { return __half22float2(v); }
template <>
__device__ __forceinline__ float2 cvt2<__nv_bfloat162>(__nv_bfloat162 v) { return __bfloat1622float2(v); }

template <typename T2>
__global__ void __launch_bounds__(256)
k_apply_edge(const T2* __restrict__ Kmat, const float* __restrict__ x, const int* __restrict__ src_nodes,
             const int* __restrict__ group_ptr, const int* __restrict__ dst_sorted, const float* __restrict__ inv_deg,
             int S, int64_t E, int cin, int cout, float* __restrict__ out, unsigned node_flags) {
  // one warp per EDGE (sorted position p): parallelism = E warps whatever the degree distribution is (one warp per
  // source serialises the 18-55 edges of MGKN's coarse levels)
  extern __shared__ float sxe[];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int64_t p = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + warp;
  if (p >= E) return;
  // compact source of this edge: the last c with group_ptr[c] <= p (all lanes search together: broadcast loads)
  int lo = 0, hi = S;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(group_ptr + mid) <= p) lo = mid; else hi = mid;
  }
  float* sx = sxe + warp * cin;
  const int n = __ldg(src_nodes + lo);
  const bool relu_in = (node_flags & 1u) != 0;     // x is a pre-activation (see k_out_init)
  for (int i = lane; i < cin; i += 32) {
    const float v = __ldg(x + static_cast<int64_t>(n) * cin + i);
    sx[i] = relu_in ? fmaxf(v, 0.f) : v;
  }
  __syncwarp();
  const int half_cout = cout / 2;
  const T2* Kp = Kmat + p * cin * half_cout;
  const int d = __ldg(dst_sorted + p);
  const float sc = inv_deg ? __ldg(inv_deg + d) : 1.f;
  for (int o2 = lane; o2 < half_cout; o2 += 32) {
    float ax = 0.f, ay = 0.f;
#pragma unroll 16
    for (int i = 0; i < cin; ++i) {
      const float2 k = cvt2<T2>(Kp[i * half_cout + o2]);
      ax = fmaf(sx[i], k.x, ax);
      ay = fmaf(sx[i], k.y, ay);
    }
    float* o = out + static_cast<int64_t>(d) * cout + 2 * o2;
    atomicAdd(o, ax * sc);
    atomicAdd(o + 1, ay * sc);
  }
}

// variant for very low out-degree (E <= 8 S, the 1-D multipole stencils): one warp per SOURCE loads x_src once and walks
// its 2-4 edges -- no per-edge source search
template <typename T2>
__global__ void __launch_bounds__(128)
k_apply_edge_src(const T2* __restrict__ Kmat, const float* __restrict__ x, const int* __restrict__ src_nodes,
                 const int* __restrict__ group_ptr, const int* __restrict__ dst_sorted, const float* __restrict__ inv_deg,
                 int S, int cin, int cout, float* __restrict__ out, unsigned node_flags) {
  extern __shared__ float sxe[];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int c = blockIdx.x * 4 + warp;
  if (c >= S) return;
  float* sx = sxe + warp * cin;
  const int n = src_nodes[c];
  const bool relu_in = (node_flags & 1u) != 0;
  for (int i = lane; i < cin; i += 32) {
    const float v = x[static_cast<int64_t>(n) * cin + i];
    sx[i] = relu_in ? fmaxf(v, 0.f) : v;
  }
  __syncwarp();
  const int e0 = group_ptr[c], e1 = group_ptr[c + 1];
  const int half_cout = cout / 2;
  for (int p = e0; p < e1; ++p) {
    const T2* Kp = Kmat + static_cast<int64_t>(p) * cin * half_cout;
    const int d = dst_sorted[p];
    const float sc = inv_deg ? inv_deg[d] : 1.f;
    for (int o2 = lane; o2 < half_cout; o2 += 32) {
      float ax = 0.f, ay = 0.f;
#pragma unroll 8
      for (int i = 0; i < cin; ++i) {
        const float2 k = cvt2<T2>(Kp[i * half_cout + o2]);
        ax = fmaf(sx[i], k.x, ax);
        ay = fmaf(sx[i], k.y, ay);
      }
      float* o = out + static_cast<int64_t>(d) * cout + 2 * o2;
      atomicAdd(o, ax * sc);
      atomicAdd(o + 1, ay * sc);
    }
  }
}

// ---- 16-byte-load variants of the two kernels above for the shapes the reference's scripts use (in = out = 64 or 32).
// A K_e row of COUT 16-bit values is LPR = COUT/8 lanes wide, so ONE warp-wide load instruction covers RPI = 256/COUT
// input channels and an edge needs only CIN/RPI (= 16 at 64 x 64) independent loads per lane, all issued back to back
// BEFORE the source search / x staging they do not depend on.  The scalar kernels issue 64 dependent-looking 4-byte
// loads per lane and are latency bound.
__device__ __forceinline__ void red_add_v4f(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <int CIN, int COUT>
struct EdgeVec {
  static constexpr int LPR = COUT / 8;     // lanes per K_e row
  static constexpr int RPI = 32 / LPR;     // input channels per warp-wide load
  static constexpr int NIT = CIN / RPI;    // loads per lane and edge
  static_assert(COUT % 8 == 0 && 32 % LPR == 0 && CIN % RPI == 0 && RPI >= 2, "unsupported K_e shape");

  template <typename T2>
  static __device__ __forceinline__ void load(const T2* __restrict__ Kp, int lane, uint4 (&kv)[NIT]) {
    const uint4* src = reinterpret_cast<const uint4*>(Kp) + lane;     // row lane / LPR, 16-byte piece lane % LPR
#pragma unroll
    for (int it = 0; it < NIT; ++it) kv[it] = __ldg(src + it * 32);   // RPI rows further = 32 pieces further
  }

  // out row += sc * (x . K_e): every lane accumulates its 8 columns over its rows, the RPI row groups are summed with
  // shuffles, and lane groups 0 / 1 each add one 16-byte piece of the lane's 8 columns.
  template <typename T2>
  static __device__ __forceinline__ void fma_scatter(const uint4 (&kv)[NIT], const float* sx, int lane, float sc,
                                                     float* __restrict__ orow) {
    const int r = lane / LPR, q = lane % LPR;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      const float xv = sx[it * RPI + r];
      const T2* h = reinterpret_cast<const T2*>(&kv[it]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 k = cvt2<T2>(h[j]);
        acc[2 * j] = fmaf(xv, k.x, acc[2 * j]);
        acc[2 * j + 1] = fmaf(xv, k.y, acc[2 * j + 1]);
      }
    }
#pragma unroll
    for (int m = LPR; m < 32; m <<= 1) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], m);
    }
    if (r < 2) {
      const float a0 = r ? acc[4] : acc[0], a1 = r ? acc[5] : acc[1], a2 = r ? acc[6] : acc[2], a3 = r ? acc[7] : acc[3];
      red_add_v4f(orow + q * 8 + 4 * r, a0 * sc, a1 * sc, a2 * sc, a3 * sc);
    }
  }
};

template <typename T2, int CIN, int COUT>
__global__ void __launch_bounds__(256)
k_apply_edge_v(const T2* __restrict__ Kmat, const float* __restrict__ x, const int* __restrict__ src_nodes,
               const int* __restrict__ group_ptr, const int* __restrict__ dst_sorted, const float* __restrict__ inv_deg,
               int S, int64_t E, float* __restrict__ out, unsigned node_flags) {
  using V = EdgeVec<CIN, COUT>;
  __shared__ float sxe[8 * CIN];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int64_t p = static_cast<int64_t>(blockIdx.x) * 8 + warp;
  if (p >= E) return;
  uint4 kv[V::NIT];
  V::template load<T2>(Kmat + p * (CIN * COUT / 2), lane, kv);
  int lo = 0, hi = S;                       // compact source of edge p: the last c with group_ptr[c] <= p
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(group_ptr + mid) <= p) lo = mid; else hi = mid;
  }
  float* sx = sxe + warp * CIN;
  const int n = __ldg(src_nodes + lo);
  const bool relu_in = (node_flags & 1u) != 0;
  for (int i = lane; i < CIN; i += 32) {
    const float v = __ldg(x + static_cast<int64_t>(n) * CIN + i);
    sx[i] = relu_in ? fmaxf(v, 0.f) : v;
  }
  __syncwarp();
  const int d = __ldg(dst_sorted + p);
  const float sc = inv_deg ? __ldg(inv_deg + d) : 1.f;
  V::template fma_scatter<T2>(kv, sx, lane, sc, out + static_cast<int64_t>(d) * COUT);
}

template <typename T2, int CIN, int COUT>
__global__ void __launch_bounds__(128)
k_apply_edge_src_v(const T2* __restrict__ Kmat, const float* __restrict__ x, const int* __restrict__ src_nodes,
                   const int* __restrict__ group_ptr, const int* __restrict__ dst_sorted, const float* __restrict__ inv_deg,
                   int S, float* __restrict__ out, unsigned node_flags) {
  using V = EdgeVec<CIN, COUT>;
  __shared__ float sxe[4 * CIN];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int c = blockIdx.x * 4 + warp;
  if (c >= S) return;
  const int e0 = group_ptr[c], e1 = group_ptr[c + 1];
  uint4 kv[V::NIT];
  if (e0 < e1) V::template load<T2>(Kmat + static_cast<int64_t>(e0) * (CIN * COUT / 2), lane, kv);
  float* sx = sxe + warp * CIN;
  const int n = src_nodes[c];
  const bool relu_in = (node_flags & 1u) != 0;
  for (int i = lane; i < CIN; i += 32) {
    const float v = x[static_cast<int64_t>(n) * CIN + i];
    sx[i] = relu_in ? fmaxf(v, 0.f) : v;
  }
  __syncwarp();
  for (int p = e0; p < e1; ++p) {
    const int d = dst_sorted[p];
    const float sc = inv_deg ? inv_deg[d] : 1.f;
    uint4 cur[V::NIT];
#pragma unroll
    for (int it = 0; it < V::NIT; ++it) cur[it] = kv[it];
    if (p + 1 < e1) V::template load<T2>(Kmat + static_cast<int64_t>(p + 1) * (CIN * COUT / 2), lane, kv);   // next edge in flight
    V::template fma_scatter<T2>(cur, sx, lane, sc, out + static_cast<int64_t>(d) * COUT);
  }
}

template <typename T>
int launch_pad_convert_t(const float* src, int R, int C, void* dst, int Rp, int Cp, cudaStream_t st) {
  int64_t total = static_cast<int64_t>(Rp) * Cp;
  if (total == 0) return NNCONV_OK;
  k_pad_convert<T><<<(unsigned)ceil_div64(total, 256), 256, 0, st>>>(src, R, C, static_cast<T*>(dst), Rp, Cp);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

}  // namespace

int launch_pad_convert(int prec, const float* src, int R, int C, void* dst, int Rp, int Cp, cudaStream_t st) {
  if (prec == PREC_F16X2) {
    const int64_t total = static_cast<int64_t>(Rp) * 3 * Cp;
    if (total == 0) return NNCONV_OK;
    k_pad_convert_split3<<<(unsigned)ceil_div64(total, 256), 256, 0, st>>>(src, R, C, static_cast<__half*>(dst), Rp, Cp,
                                                                           nullptr);
    NNC_CHECK_LAUNCH();
    return NNCONV_OK;
  }
  if (prec == PREC_FP32) return launch_pad_convert_t<float>(src, R, C, dst, Rp, Cp, st);
  if (prec == PREC_F16) return launch_pad_convert_t<__half>(src, R, C, dst, Rp, Cp, st);
  return launch_pad_convert_t<__nv_bfloat16>(src, R, C, dst, Rp, Cp, st);
}

int launch_pad_convert_split3(const float* src, int R, int C, void* dst, int Rp, int Cp, const float* scale, cudaStream_t st) {
  const int64_t total = static_cast<int64_t>(Rp) * 3 * Cp;
  if (total == 0) return NNCONV_OK;
  k_pad_convert_split3<<<(unsigned)ceil_div64(total, 256), 256, 0, st>>>(src, R, C, static_cast<__half*>(dst), Rp, Cp, scale);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_pow2_scale(const float* src, int64_t n, float* scale2, cudaStream_t st) {
  NNC_CHECK_CUDA(cudaMemsetAsync(scale2, 0, 2 * sizeof(float), st));
  if (n > 0) {
    int g = static_cast<int>(ceil_div64(n, 1024));
    if (g > 592) g = 592;
    k_absmax_bits<<<g, 256, 0, st>>>(src, n, reinterpret_cast<unsigned int*>(scale2));
    NNC_CHECK_LAUNCH();
  }
  k_pow2_from_max<<<1, 1, 0, st>>>(scale2);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_overflow_accumulate(const int* counter, int* sticky, cudaStream_t st) {
  k_overflow_accumulate<<<1, 1, 0, st>>>(counter, sticky);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_w3p(int prec, const float* WL, int cin, int cout, int K, int Kp, int cin_p, void* dst, cudaStream_t st,
               const float* scale) {
  int64_t total = static_cast<int64_t>(cout) * Kp * cin_p;
  if (prec == PREC_F16X2) {
    k_w3p_split3<<<(unsigned)ceil_div64(3 * total, 256), 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, static_cast<__half*>(dst),
                                                                       scale);
    NNC_CHECK_LAUNCH();
    return NNCONV_OK;
  }
  unsigned g = (unsigned)ceil_div64(total, 256);
  if (prec == PREC_FP32) k_w3p<float><<<g, 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, static_cast<float*>(dst));
  else if (prec == PREC_F16) k_w3p<__half><<<g, 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, static_cast<__half*>(dst));
  else k_w3p<__nv_bfloat16><<<g, 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, static_cast<__nv_bfloat16*>(dst));
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_w3q(int prec, const float* WL, int cin, int cout, int K, int Kp, int cin_p, int transposed, void* dst,
               cudaStream_t st, const float* scale) {
  const int64_t total = static_cast<int64_t>(cout) * Kp * cin_p;
  const unsigned g = (unsigned)ceil_div64(total, 256);
  if (prec == PREC_F16X2) {
    NNC_REQUIRE(scale != nullptr, NNCONV_ERR_ARG, "w3q: split images need their power-of-two scale");
    k_w3q_split3<<<(unsigned)ceil_div64(3 * total, 256), 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, transposed,
                                                                       static_cast<__half*>(dst), scale);
    NNC_CHECK_LAUNCH();
    return NNCONV_OK;
  }
  if (prec == PREC_F16) k_w3q<__half><<<g, 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, transposed, static_cast<__half*>(dst));
  else k_w3q<__nv_bfloat16><<<g, 256, 0, st>>>(WL, cin, cout, K, Kp, cin_p, transposed, static_cast<__nv_bfloat16*>(dst));
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_transpose_pad(int prec, const float* src, int R, int C, void* dst, int Rp, int Cp, cudaStream_t st,
                         const float* scale) {
  const int64_t total = static_cast<int64_t>(Rp) * Cp;
  const unsigned g = (unsigned)ceil_div64(total, 256);
  if (prec == PREC_F16X2) {
    NNC_REQUIRE(scale != nullptr, NNCONV_ERR_ARG, "transpose_pad: split images need their power-of-two scale");
    k_transpose_pad_split3<<<(unsigned)ceil_div64(3 * total, 256), 256, 0, st>>>(src, R, C, static_cast<__half*>(dst), Rp,
                                                                                 Cp, scale);
    NNC_CHECK_LAUNCH();
    return NNCONV_OK;
  }
  if (prec == PREC_F16) k_transpose_pad<__half><<<g, 256, 0, st>>>(src, R, C, static_cast<__half*>(dst), Rp, Cp);
  else k_transpose_pad<__nv_bfloat16><<<g, 256, 0, st>>>(src, R, C, static_cast<__nv_bfloat16*>(dst), Rp, Cp);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_edge_layer1(int prec, const float* edge_attr, const int* perm, int64_t e_begin, int64_t e_count, int k_in,
                       const float* W1, const float* b1, int kp1, int identity, void* out, cudaStream_t st,
                       int64_t chunk_rows_pad, int64_t out_row0, int* overflow, Act act) {
  if (e_count <= 0) return NNCONV_OK;
  unsigned g = (unsigned)ceil_div64(e_count, kL1Edges);
  size_t sm = sizeof(float) * kL1Edges * k_in;
  if (!identity && act.kind != ACT_RELU) {
    act_dispatch(act.kind, [&](auto k) {
      constexpr int A = decltype(k)::value;
      if (prec == PREC_FP32)
        k_edge_layer1_act<A, float><<<g, 256, sm, st>>>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1,
                                                         static_cast<float*>(out), chunk_rows_pad, out_row0, nullptr,
                                                         act.p);
      else if (prec == PREC_F16 || prec == PREC_F16X2)
        k_edge_layer1_act<A, __half><<<g, 256, sm, st>>>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1,
                                                          static_cast<__half*>(out), chunk_rows_pad, out_row0, overflow,
                                                          act.p);
      else
        k_edge_layer1_act<A, __nv_bfloat16><<<g, 256, sm, st>>>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1,
                                                                 static_cast<__nv_bfloat16*>(out), chunk_rows_pad,
                                                                 out_row0, nullptr, act.p);
    });
  } else if (prec == PREC_FP32)
    k_edge_layer1<float><<<g, 256, sm, st>>>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1, identity,
                                             static_cast<float*>(out), chunk_rows_pad, out_row0, nullptr);
  else if (prec == PREC_F16 || prec == PREC_F16X2)
    k_edge_layer1<__half><<<g, 256, sm, st>>>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1, identity,
                                              static_cast<__half*>(out), chunk_rows_pad, out_row0, overflow);
  else
    k_edge_layer1<__nv_bfloat16><<<g, 256, sm, st>>>(edge_attr, perm, e_begin, e_count, k_in, W1, b1, kp1, identity,
                                                     static_cast<__nv_bfloat16*>(out), chunk_rows_pad, out_row0, nullptr);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_build_a1(int prec, const float* edge_attr, const int* perm, int64_t e_begin, int64_t e_count, int k_in,
                    void* A1, cudaStream_t st) {
  if (e_count <= 0) return NNCONV_OK;
  unsigned g = (unsigned)ceil_div64(e_count * 8, 256);
  if (prec == PREC_F16 || prec == PREC_F16X2)
    k_build_a1<__half><<<g, 256, 0, st>>>(edge_attr, perm, e_begin, e_count, k_in, static_cast<__half*>(A1));
  else
    k_build_a1<__nv_bfloat16><<<g, 256, 0, st>>>(edge_attr, perm, e_begin, e_count, k_in,
                                                 static_cast<__nv_bfloat16*>(A1));
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_w1aug(int prec, const float* W1, const float* b1, int k1, int kp1, int k_in, void* dst, cudaStream_t st) {
  unsigned g = (unsigned)ceil_div(kp1 * 64, 256);
  if (prec == PREC_F16 || prec == PREC_F16X2) k_w1aug<__half><<<g, 256, 0, st>>>(W1, b1, k1, kp1, k_in, static_cast<__half*>(dst));
  else k_w1aug<__nv_bfloat16><<<g, 256, 0, st>>>(W1, b1, k1, kp1, k_in, static_cast<__nv_bfloat16*>(dst));
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_out_init(const float* x, const float* root, const float* bias, int64_t N, int cin, int cout, float* out,
                    cudaStream_t st, unsigned node_flags) {
  dim3 b(64, 4);
  unsigned g = (unsigned)ceil_div64(N, b.y);
  k_out_init<<<g, b, sizeof(float) * b.y * cin, st>>>(x, root, bias, N, cin, cout, out, node_flags);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int root_term(const float* x, const float* root, const float* bias, int64_t N, int cin, int cout, float* out,
              cudaStream_t st) {
  if (N <= 0 || (root == nullptr && bias == nullptr)) return NNCONV_OK;
  dim3 b(64, 4);
  unsigned g = (unsigned)ceil_div64(N, b.y);
  k_root_add<<<g, b, root ? sizeof(float) * b.y * cin : 0, st>>>(x, root, bias, N, cin, cout, out);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_src_prep(int prec, const float* x, const int* src_nodes, int S, int cin, int cin_p, int cout,
                    const float* B3, void* Xc, float* cvec, float* xs, cudaStream_t st, unsigned node_flags) {
  if (S <= 0) return NNCONV_OK;
  dim3 b(64, 4);
  unsigned g = (unsigned)ceil_div(S, (int)b.y);
  size_t sm = sizeof(float) * b.y * cin;
  if (prec == PREC_FP32)
    k_src_prep<float><<<g, b, sm, st>>>(x, src_nodes, S, cin, cin_p, cout, B3, static_cast<float*>(Xc), cvec, nullptr,
                                        node_flags);
  else if (prec == PREC_F16)
    k_src_prep<__half><<<g, b, sm, st>>>(x, src_nodes, S, cin, cin_p, cout, B3, static_cast<__half*>(Xc), cvec, xs,
                                         node_flags);
  else if (prec == PREC_F16X2)
    k_src_prep<__half, 1><<<g, b, sm, st>>>(x, src_nodes, S, cin, cin_p, cout, B3, static_cast<__half*>(Xc), cvec, xs,
                                            node_flags);
  else
    k_src_prep<__nv_bfloat16><<<g, b, sm, st>>>(x, src_nodes, S, cin, cin_p, cout, B3,
                                                static_cast<__nv_bfloat16*>(Xc), cvec, xs, node_flags);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

// out_init + src_prep + the flag reset of one application as ONE launch (16-bit precisions)
int launch_node_prep(int prec, const float* x, const float* root, const float* bias, int64_t N, float* out,
                     const int* src_nodes, int S, int cin, int cin_p, int cout, const float* B3, void* Xc, float* cvec,
                     float* xs, int* flags, int flags_stride, int n_batches, cudaStream_t st, unsigned node_flags,
                     unsigned long long* max_keys) {
  dim3 b(64, 4);
  const int g_out = static_cast<int>(ceil_div64(N, b.y));
  const int g_src = ceil_div(S, (int)b.y);
  const unsigned g = static_cast<unsigned>(g_out + g_src);
  size_t sm = sizeof(float) * b.y * cin;
  auto go = [&](auto t, auto split, auto mx) {
    using T = decltype(t);
    k_node_prep<T, decltype(split)::value, decltype(mx)::value><<<g, b, sm, st>>>(
        x, root, bias, N, out, g_out, src_nodes, S, cin, cin_p, cout, B3, static_cast<T*>(Xc), cvec, xs, flags,
        flags_stride, n_batches, node_flags, max_keys);
  };
  auto by_max = [&](auto t, auto split) {
    if (max_keys != nullptr) go(t, split, std::true_type());
    else go(t, split, std::false_type());
  };
  if (prec == PREC_F16)
    by_max(__half(), std::integral_constant<int, 0>());
  else if (prec == PREC_F16X2)
    by_max(__half(), std::integral_constant<int, 1>());
  else if (prec == PREC_BF16)
    by_max(__nv_bfloat16(), std::integral_constant<int, 0>());
  else
    return NNCONV_ERR_UNSUPPORTED;
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

namespace {
template <typename T2>
int launch_apply_edge_t(const Plan* P, const Weights* W, const void* Kmat_, const float* x, const float* inv_deg, float* out,
                        cudaStream_t st, unsigned node_flags) {
  const T2* Kmat = static_cast<const T2*>(Kmat_);
  const int S = P->n_src;
  // warp per SOURCE only when there are enough sources to fill the machine with warps (the 1-D multipole stencils: 8192
  // ... 2048 sources with 2-4 edges each); a coarse MGKN level (100 sources x 6 edges) runs warp per EDGE
  const bool per_source = P->E <= 8 * static_cast<int64_t>(S) && S >= 2048;
  const bool v64 = W->cin == 64 && W->cout == 64, v32 = W->cin == 32 && W->cout == 32;
  if (per_source) {
    const unsigned g = (unsigned)ceil_div(S, 4);
    if (v64)
      k_apply_edge_src_v<T2, 64, 64><<<g, 128, 0, st>>>(Kmat, x, P->src_nodes, P->group_ptr, P->dst_sorted, inv_deg, S, out,
                                                        node_flags);
    else if (v32)
      k_apply_edge_src_v<T2, 32, 32><<<g, 128, 0, st>>>(Kmat, x, P->src_nodes, P->group_ptr, P->dst_sorted, inv_deg, S, out,
                                                        node_flags);
    else
      k_apply_edge_src<T2><<<g, 128, sizeof(float) * 4 * W->cin, st>>>(Kmat, x, P->src_nodes, P->group_ptr, P->dst_sorted,
                                                                       inv_deg, S, W->cin, W->cout, out, node_flags);
  } else {
    const unsigned g = (unsigned)ceil_div64(P->E, 8);
    if (v64)
      k_apply_edge_v<T2, 64, 64><<<g, 256, 0, st>>>(Kmat, x, P->src_nodes, P->group_ptr, P->dst_sorted, inv_deg, S, P->E, out,
                                                    node_flags);
    else if (v32)
      k_apply_edge_v<T2, 32, 32><<<g, 256, 0, st>>>(Kmat, x, P->src_nodes, P->group_ptr, P->dst_sorted, inv_deg, S, P->E, out,
                                                    node_flags);
    else
      k_apply_edge<T2><<<g, 256, sizeof(float) * 8 * W->cin, st>>>(Kmat, x, P->src_nodes, P->group_ptr, P->dst_sorted, inv_deg,
                                                                   S, P->E, W->cin, W->cout, out, node_flags);
  }
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}
}  // namespace

int launch_apply_edge(int prec, const Plan* P, const Weights* W, const void* Kmat, const float* x, int aggr_mean, float* out,
                      cudaStream_t st, unsigned node_flags) {
  if (P->n_src <= 0 || P->E <= 0) return NNCONV_OK;
  const float* inv_deg = aggr_mean ? P->inv_deg : nullptr;
  if (prec == PREC_BF16) return launch_apply_edge_t<__nv_bfloat162>(P, W, Kmat, x, inv_deg, out, st, node_flags);
  return launch_apply_edge_t<__half2>(P, W, Kmat, x, inv_deg, out, st, node_flags);
}

int launch_sgemm_store(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M, int N,
                       int K, const float* bias_relu, cudaStream_t st, Act act) {
  if (M <= 0 || N <= 0) return NNCONV_OK;
  SgemmArgs a{};
  a.A = A; a.lda = lda; a.B = B; a.ldb = ldb; a.C = C; a.ldc = ldc; a.M = M; a.N = N; a.K = K; a.bias = bias_relu;
  a.act_p = act.p;
  dim3 g(ceil_div(M, 64), ceil_div(N, 64));
  if (bias_relu && act.kind != ACT_RELU)
    act_dispatch(act.kind, [&](auto k) { k_sgemm_nt<EPI_BIAS_ACT + decltype(k)::value><<<g, 256, 0, st>>>(a); });
  else if (bias_relu) k_sgemm_nt<EPI_BIAS_RELU><<<g, 256, 0, st>>>(a);
  else k_sgemm_nt<EPI_STORE><<<g, 256, 0, st>>>(a);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

int launch_sgemm_scatter(const Plan* P, const float* h, int Kp, const float* Y, int cout, int tile_begin, int tile_end,
                         int c0, const float* cvec, int aggr_mean, float* out, cudaStream_t st,
                         unsigned long long* max_keys) {
  int nt = tile_end - tile_begin;
  if (nt <= 0) return NNCONV_OK;
  SgemmArgs a{};
  a.A = h; a.lda = Kp; a.B = Y; a.ldb = Kp; a.C = out; a.ldc = cout; a.M = 0; a.N = cout; a.K = Kp;
  a.tile_c = P->tile_c; a.tile_e0 = P->tile_e0; a.tile_cnt = P->tile_cnt; a.dst_sorted = P->dst_sorted;
  a.inv_deg = aggr_mean ? P->inv_deg : nullptr; a.cvec = cvec; a.tile_begin = tile_begin; a.c0 = c0;
  a.y_stride = static_cast<int64_t>(cout) * Kp;
  a.keys = max_keys; a.perm = P->perm;
  dim3 g(nt * 2, ceil_div(cout, 64));
  if (max_keys != nullptr) k_sgemm_nt<EPI_SCATTER_MAX><<<g, 256, 0, st>>>(a);
  else k_sgemm_nt<EPI_SCATTER><<<g, 256, 0, st>>>(a);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

// aggr = max, after the last contraction of an application: out += the max the key encodes (nothing for key 0, the
// empty neighbourhood), argmax = the winning caller edge index (-1 when empty)
__global__ void k_max_finalize(const unsigned long long* __restrict__ keys, int64_t n, float* __restrict__ out,
                               int* __restrict__ argmax) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == 0ull) {
      argmax[i] = -1;
      continue;
    }
    const uint32_t hi = static_cast<uint32_t>(k >> 32);
    const uint32_t u = (hi & 0x80000000u) ? (hi ^ 0x80000000u) : ~hi;
    out[i] += __uint_as_float(u);
    argmax[i] = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(k));
  }
}

int launch_max_finalize(const unsigned long long* keys, int64_t n, float* out, int* argmax, cudaStream_t st) {
  if (n <= 0) return NNCONV_OK;
  const int64_t blocks = ceil_div64(n, 256);
  k_max_finalize<<<static_cast<unsigned>(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(keys, n, out, argmax);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

}  // namespace nnc
