// Fused per-edge contraction + scatter of NNConv (graph-neural-operator/nn_conv.py:273-275 + PyG
// propagate/scatter_mean), reassociated around the per-SOURCE matrix Y_src:
//
//     m_e[o]  = sum_i x[src_e, i] * K_e[i, o],        K_e = (W_L h_e + b_L).view(in, out)
//             = sum_k h_e[k] * Y_src[o, k] + c_src[o] (Y_src[o,k] = sum_i x[src,i] W_L[i*out+o, k],
//                                                      c_src = x[src] @ b_L.view(in,out))
//     out[dst_e, :] += m_e / max(deg_in(dst_e), 1)
//
// Edges arrive grouped by source (np.where order of the reference's ball graphs), so for one source all
// its edges form a dense GEMM  M[cnt, out] = H[cnt, Kp] * Y_src[out, Kp]^T  with the SAME B operand.
//
// Work decomposition
//   tile  = <= 128 consecutive edges of one source (one warpgroup, two m64 wgmma halves)
//   unit  = <= kTU consecutive tiles of one source; tile ti of a unit is accumulated (in registers) and scattered
//           by consumer warpgroup ti
//   pass  = a slice of nb_slots K-chunks (64 columns each) of Y_src that is resident in shared memory.
//           For Kp = 1024, out = 64 the whole Y_src (128 KB) would leave room for only one CTA per SM;
//           splitting K in two passes (64 KB resident) lets TWO CTAs share an SM, so that consecutive
//           kernels of one application (launched with programmatic stream serialization) overlap their
//           ramp-up / drain and the Y GEMM of the next batch runs beside the contraction of this one.
//   per unit: for pass p: for tile ti: for slot s: D[ti] += A(tile ti, chunk p*nb+s) * B(slot s)
// Data movement
//   * A (h rows, chunk-major panels [Kp/64][E_pad][64]): one contiguous TMA box per (tile, chunk), rows
//     rounded up to 16 -- this stream is the kernel's HBM roofline (Kp * 2 bytes per edge-application);
//   * B slots: TMA from the L2-resident per-batch Y buffer, one full/empty mbarrier pair per slot, so the
//     next pass / next source is fetched slot by slot as soon as the last tile has consumed it;
//   * epilogue (the tile's warpgroup): registers -> per-warp transpose (thread = edge row) -> + c_src, * 1/deg(dst)
//     -> red.global.add.v4.f32 into out[dst] (fp32, L2 resident).
// Persistent: each CTA owns a contiguous range of tiles.
#include <cstdlib>
#include <type_traits>

#include "kernels.h"
#include "options.h"
#include "tc05.cuh"
#include "tmap.h"

namespace nnc {

int tc_num_sms();

namespace {

using namespace tc05;

constexpr int kMaxSlots = 16;
constexpr int kMaxAStages = 8;
constexpr int kTU = 2;                     // tiles per unit = consumer warpgroups
constexpr int kThreads = 32 * (4 * kTU + 1);   // consumer warpgroups, then the TMA producer warp
constexpr int kScratchBytes = 4 * kTU * acc_scratch_bytes<16>();
constexpr int kATileBytes = 128 * 64 * 2;
constexpr int kSmemTwoPerSm = 115200;      // dynamic smem per CTA that still lets two CTAs share one SM

struct ConvTcArgs {
  const int* tile_c;
  const int* tile_e0;
  const int* tile_cnt;
  const int* dst_sorted;
  const float* inv_deg;   // nullptr -> aggr = add
  const float* cvec;      // [S, cout]
  const float* xs;        // [S] power-of-two row scale of the Y operand (see k_src_prep)
  float* out;             // [N, cout]
  int tile_begin, tile_end;
  int c0;                 // compact source index of Y row block 0
  int nb_slots;           // resident K chunks per pass
  int passes;             // nb_slots * passes == Kp / 64
  int a_stages;
  int e_pad;              // rows per 64-column panel of the chunk-major h
  int e_base;             // sorted edge of h row 0 (0 unless h is a chunk of the edges)
  int debug;              // NNCONV_DEBUG bit0: skip the scatter (measurement experiments only)
  // cross-kernel pipelining (tc05.cuh): Y of this batch must be complete; raise done when all reds are out;
  // the last kernel of an application also joins every earlier kernel of the chain before it exits
  const int* wait_ok;
  int* done_cnt;
  int* done_ok;
  const int* join_ok;
  int join_n;
  TraceBuf trace;
  unsigned int trace_seq;
  // aggr = max (the MAX instantiation only): [N, cout] keys (common.cuh max_key) and the plan's perm (nullable)
  unsigned long long* keys;
  const int* perm;
};

// tmH.m[i] has a box of 16*(i+1) rows: the last tile of a source group only fetches the rows it owns
// (rounded up to 16) instead of a full 128-row box that would re-read the next group's rows from HBM.
struct HMaps {
  CUtensorMap m[8];
};

struct Unit {
  int t, u, c;
};
__device__ __forceinline__ bool next_unit(const ConvTcArgs& a, int t1, int& t, Unit& un) {
  if (t >= t1) return false;
  un.t = t;
  un.c = a.tile_c[t];
  un.u = 1;
  while (un.u < kTU && t + un.u < t1 && a.tile_c[t + un.u] == un.c) ++un.u;
  t += un.u;
  return true;
}

// The kernel body, shared by k_conv_tc (aggr add / mean) and k_conv_tc_max.  MAX: aggr = max -- the epilogue reduces
// one key per (edge row, channel) with red.global.max.u64 into a.keys.
template <int FMT, int NC, bool MAX>
__device__ __forceinline__ void conv_tc_body(const HMaps& tmH, const CUtensorMap& tmY, const ConvTcArgs& a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();            // SWIZZLE_128B tiles need 1024 B alignment
  const int b_chunk_bytes = NC * 128;                 // [cout rows x 64 k] 16-bit
  const int b_stride = (b_chunk_bytes + 1023) & ~1023;
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem + a.nb_slots * b_stride;
  float* scratch = reinterpret_cast<float*>(smem_a + a.a_stages * kATileBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + a.a_stages * kATileBytes + kScratchBytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + kMaxAStages;
  uint64_t* b_full = bars + 2 * kMaxAStages;
  uint64_t* b_empty = b_full + kMaxSlots;

  // shfl: warp-uniform role index (wgmma under a branch the compiler cannot prove uniform is serialised)
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x / 32), 0), lane = threadIdx.x % 32;
  const int total = a.tile_end - a.tile_begin;
  const int t0 = a.tile_begin + static_cast<int>((static_cast<int64_t>(total) * blockIdx.x) / gridDim.x);
  const int t1 = a.tile_begin + static_cast<int>((static_cast<int64_t>(total) * (blockIdx.x + 1)) / gridDim.x);
  constexpr int kProducer = 4 * kTU;

  if (warp == kProducer && lane == 0) {
    for (int i = 0; i < 8; ++i) prefetch_tmap(&tmH.m[i]);
    prefetch_tmap(&tmY);
    for (int s = 0; s < a.a_stages; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 4);                // the 4 warps of the tile's warpgroup
    }
    for (int j = 0; j < a.nb_slots; ++j) {
      mbar_init(&b_full[j], 1);
      mbar_init(&b_empty[j], 4 * kTU);          // every consumer warp
    }
    fence_barrier_init();
  }
  const unsigned long long tr0 = a.trace.rec ? gtime() : 0ull;
  pdl_launch_dependents();
  if (a.wait_ok != nullptr && threadIdx.x == 0) flag_wait(a.wait_ok);
  const unsigned long long tr1 = a.trace.rec ? gtime() : 0ull;
  __syncthreads();

  if (warp == kProducer) {
    if (lane == 0) {
      // ------------------------------------------------------------ TMA producer
      ARing ring[kTU];
      for (int ti = 0; ti < kTU; ++ti) ring[ti].init(ti, a.a_stages);
      int prev_c = -1;
      uint32_t ld = 0;                              // B load events so far
      int t = t0;
      Unit un;
      while (next_unit(a, t1, t, un)) {
        for (int p = 0; p < a.passes; ++p) {
          const bool need = a.passes > 1 || un.c != prev_c;
          for (int ti = 0; ti < un.u; ++ti) {
            const int e0 = a.tile_e0[un.t + ti];
            const int box = (a.tile_cnt[un.t + ti] + 15) >> 4;            // 1..8 -> rows = 16 * box
            const CUtensorMap* mh = &tmH.m[box - 1];
            const uint32_t a_bytes = static_cast<uint32_t>(box) * 16u * 128u;
            for (int s = 0; s < a.nb_slots; ++s) {
              const int j = p * a.nb_slots + s;
              if (need && ti == 0) {
                mbar_wait(&b_empty[s], (ld & 1u) ^ 1u);
                mbar_arrive_expect_tx(&b_full[s], b_chunk_bytes);
                tma_load_2d(smem_b + s * b_stride, &tmY, &b_full[s], j * 64, (un.c - a.c0) * NC, kEvictLast);
              }
              const int stage = ring[ti].stage;
              mbar_wait(&a_empty[stage], ring[ti].phase ^ 1u);
              mbar_arrive_expect_tx(&a_full[stage], a_bytes);
              tma_load_2d(smem_a + stage * kATileBytes, mh, &a_full[stage], 0, j * a.e_pad + e0 - a.e_base, kEvictFirst);
              ring[ti].next();
            }
          }
          if (need) ++ld;
        }
        prev_c = un.c;
      }
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroup g = tile g of every unit
    const int g = warp / 4, quarter = warp % 4;
    float* wb = scratch + warp * (acc_scratch_bytes<16>() / 4);
    Acc<NC> acc;
    ARing ring;
    ring.init(g, a.a_stages);
    int prev_c = -1;
    uint32_t ld = 0;
    int t = t0;
    Unit un;
    while (next_unit(a, t1, t, un)) {
      un.u = __shfl_sync(0xffffffffu, un.u, 0);       // warp-uniform (see above)
      un.c = __shfl_sync(0xffffffffu, un.c, 0);
      const bool has_next = t < t1;
      const bool next_same = has_next && a.tile_c[t] == un.c;
      for (int p = 0; p < a.passes; ++p) {
        const bool need = a.passes > 1 || un.c != prev_c;
        if (need) ++ld;
        // the resident slots are released (for re-filling) iff the next (unit, pass) loads B again
        const bool release = (p + 1 < a.passes) || !has_next || a.passes > 1 || !next_same;
        for (int ti = 0; ti < un.u; ++ti) {
          for (int s = 0; s < a.nb_slots; ++s) {
            if (ti == g) {
              mbar_wait(&b_full[s], (ld - 1) & 1u);
              mbar_wait(&a_full[ring.stage], ring.phase);
              const uint64_t adesc = smem_desc_sw128(smem_u32(smem_a + ring.stage * kATileBytes));
              const uint64_t bdesc = smem_desc_sw128(smem_u32(smem_b + s * b_stride));
              mma_block<NC, FMT>(acc, adesc, bdesc, 512, 2, 4, (p | s) != 0);
              wgmma_wait<0>();
              __syncwarp();
              if (lane == 0) mbar_arrive(&a_empty[ring.stage]);
              ring.next();
            }
          }
        }
        if (release) {
          // every consumer warp releases the slots, after the load it releases has landed (never a phase ahead)
          for (int s = 0; s < a.nb_slots; ++s) {
            mbar_wait(&b_full[s], (ld - 1) & 1u);
            __syncwarp();
            if (lane == 0) mbar_arrive(&b_empty[s]);
          }
        }
      }
      prev_c = un.c;
      if (g >= un.u) continue;
      // ---- epilogue of tile g
      const int r = acc_row(quarter, lane);
      const bool ok = r < a.tile_cnt[un.t + g];
      int d = 0;
      float sc = 1.f;
      if (ok) {
        d = __ldg(a.dst_sorted + a.tile_e0[un.t + g] + r);
        if (a.inv_deg) sc = __ldg(a.inv_deg + d);
      }
      const float* cv = a.cvec + static_cast<int64_t>(un.c) * NC;
      const float xsc = __ldg(a.xs + un.c);
      float* orow = a.out + static_cast<int64_t>(d) * NC;
      const uint32_t ce = MAX && ok ? caller_edge(a.perm, a.tile_e0[un.t + g] + r) : 0u;
#pragma unroll
      for (int cc = 0; cc < NC; cc += 16) {
        uint32_t v[16];
        acc_rows<NC, 16>(acc, cc, wb, v);
        if constexpr (MAX) {
          if (ok) {
            unsigned long long* krow = a.keys + static_cast<int64_t>(d) * NC + cc;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float4 cq = __ldg(reinterpret_cast<const float4*>(cv + cc) + q);
              atomicMax(krow + 4 * q + 0, max_key(fmaf(__uint_as_float(v[4 * q + 0]), xsc, cq.x), ce));
              atomicMax(krow + 4 * q + 1, max_key(fmaf(__uint_as_float(v[4 * q + 1]), xsc, cq.y), ce));
              atomicMax(krow + 4 * q + 2, max_key(fmaf(__uint_as_float(v[4 * q + 2]), xsc, cq.z), ce));
              atomicMax(krow + 4 * q + 3, max_key(fmaf(__uint_as_float(v[4 * q + 3]), xsc, cq.w), ce));
            }
          }
        } else if (ok && !(a.debug & 1)) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 cq = __ldg(reinterpret_cast<const float4*>(cv + cc) + q);
            red_add_v4(orow + cc + 4 * q, fmaf(__uint_as_float(v[4 * q + 0]), xsc, cq.x) * sc,
                       fmaf(__uint_as_float(v[4 * q + 1]), xsc, cq.y) * sc,
                       fmaf(__uint_as_float(v[4 * q + 2]), xsc, cq.z) * sc,
                       fmaf(__uint_as_float(v[4 * q + 3]), xsc, cq.w) * sc);
          }
        }
      }
    }
  }
  if (a.done_cnt != nullptr) signal_done(a.done_cnt, a.done_ok);   // includes __syncthreads
  else __syncthreads();
  if (threadIdx.x == 0) trace_write(a.trace, 200u | (a.trace_seq << 12), tr0, tr1, a.trace.rec ? gtime() : 0ull);
  if (a.join_ok != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
    for (int i = 0; i < a.join_n; ++i) flag_wait(a.join_ok + i);
  }
}

template <int FMT, int NC>
__global__ void __launch_bounds__(kThreads, NC <= 64 ? 2 : 1)
k_conv_tc(const __grid_constant__ HMaps tmH, const __grid_constant__ CUtensorMap tmY, ConvTcArgs a) {
  conv_tc_body<FMT, NC, false>(tmH, tmY, a);
}

template <int FMT, int NC>
__global__ void __launch_bounds__(kThreads, NC <= 64 ? 2 : 1)
k_conv_tc_max(const __grid_constant__ HMaps tmH, const __grid_constant__ CUtensorMap tmY, ConvTcArgs a) {
  conv_tc_body<FMT, NC, true>(tmH, tmY, a);
}

struct ConvShape {
  int nb_slots, passes, a_stages, smem_bytes, ctas_per_sm;
};

// Choose the K split: prefer a configuration in which two CTAs fit one SM (smem <= kSmemTwoPerSm and
// out <= 64, i.e. <= 64 accumulator registers per thread) with >= 3 A stages; otherwise one CTA per SM with
// everything resident.  out <= 128: a warpgroup holds its [128 x out] fp32 tile in registers.
bool conv_shape(int cout, int Kp, ConvShape* cs) {
  if (cout % 16 != 0 || cout < 16 || cout > 128 || Kp % 64 != 0) return false;
  const int num_kc = Kp / 64;
  const int b_stride = (cout * 128 + 1023) & ~1023;
  const int bar_bytes = 512 + kScratchBytes;
  const bool one_per_sm = options().conv_one_per_sm != 0;   // measurement knob
  for (int two = one_per_sm ? 0 : 1; two >= 0; --two) {
    if (two && cout > 64) continue;
    const int budget = two ? kSmemTwoPerSm : 227 * 1024;
    for (int passes = 1; passes <= num_kc; ++passes) {
      if (num_kc % passes) continue;
      const int nb = num_kc / passes;
      if (nb > kMaxSlots) continue;
      int stages = (budget - bar_bytes - nb * b_stride) / kATileBytes;
      if (stages > kMaxAStages) stages = kMaxAStages;
      if (stages >= 3) {
        cs->nb_slots = nb;
        cs->passes = passes;
        cs->a_stages = stages;
        cs->smem_bytes = nb * b_stride + stages * kATileBytes + bar_bytes;
        cs->ctas_per_sm = two ? 2 : 1;
        return true;
      }
    }
  }
  return false;
}

}  // namespace

bool tc_shapes_supported(const Weights* W) {
  if (W->prec != PREC_F16 && W->prec != PREC_BF16 && W->prec != PREC_F16X2) return false;
  if (W->split) return apply_fused_supported(W);   // split precision exists in the fused kernel only
  ConvShape cs;
  return conv_shape(W->cout, W->Kp, &cs);
}

int launch_conv_tc(int prec, const Plan* P, const void* h, int Kp, const void* Y, int64_t y_nodes, int cout,
                   int tile_begin, int tile_end, int c0, const float* cvec, const float* xs, int aggr_mean, float* out,
                   cudaStream_t st, const PipeFlags* pf, int64_t e_base, int64_t h_rows, unsigned long long* max_keys) {
  if (tile_end <= tile_begin) return NNCONV_OK;
  int s = tc_init();
  if (s != NNCONV_OK) return s;
  const int bf = prec == PREC_BF16;
  const int64_t e_pad = h_rows > 0 ? h_rows : round_up64(P->E, 128);
  ConvShape cs;
  NNC_REQUIRE(conv_shape(cout, Kp, &cs), NNCONV_ERR_UNSUPPORTED,
              "conv_tc: shape not supported by the tensor-core contraction (cout=%d Kp=%d)", cout, Kp);
  HMaps tmH;
  CUtensorMap tmY;
  for (int i = 0; i < 8; ++i) {
    // chunk-major h: [Kp/64 panels][E_pad rows][64 cols] viewed as a 2-D tensor of 64-column rows
    s = make_tmap_2d_16b(&tmH.m[i], bf, h, static_cast<uint64_t>(Kp / 64) * e_pad, 64, 16 * (i + 1));
    if (s != NNCONV_OK) return s;
  }
  s = make_tmap_2d_16b(&tmY, bf, Y, static_cast<uint64_t>(y_nodes) * cout, static_cast<uint64_t>(Kp), cout);
  if (s != NNCONV_OK) return s;
  ConvTcArgs a{};
  a.e_pad = static_cast<int>(e_pad);
  a.e_base = static_cast<int>(e_base);
  a.tile_c = P->tile_c; a.tile_e0 = P->tile_e0; a.tile_cnt = P->tile_cnt; a.dst_sorted = P->dst_sorted;
  a.inv_deg = aggr_mean ? P->inv_deg : nullptr; a.cvec = cvec; a.xs = xs; a.out = out;
  a.tile_begin = tile_begin; a.tile_end = tile_end; a.c0 = c0;
  a.nb_slots = cs.nb_slots; a.passes = cs.passes; a.a_stages = cs.a_stages;
  { const int v = options().conv_stages; if (v >= 2 && v < a.a_stages) a.a_stages = v; }
  a.debug = options().conv_debug;
  {
    TraceHandle th = trace_get();
    static unsigned int launch_seq = 0;
    a.trace = TraceBuf{th.rec, th.count, th.cap};
    a.trace_seq = launch_seq++;
  }
  a.wait_ok = pf ? pf->wait_ok : nullptr;
  a.done_cnt = pf ? pf->done_cnt : nullptr;
  a.done_ok = pf ? pf->done_ok : nullptr;
  a.join_ok = pf ? pf->join_ok : nullptr;
  a.join_n = pf ? pf->join_n : 0;
  a.keys = max_keys;
  a.perm = P->perm;
  const int tiles = tile_end - tile_begin;
  const int max_ctas = tc_num_sms() * cs.ctas_per_sm;
  const int grid = tiles < max_ctas ? tiles : max_ctas;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = cs.smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pf && pf->pdl) ? 1 : 0;
  auto go_v = [&](auto fmt, auto nc, auto mx) -> int {
    constexpr int F = decltype(fmt)::value, C = decltype(nc)::value;
    constexpr bool M = decltype(mx)::value;
    constexpr auto kern = M ? k_conv_tc_max<F, C> : k_conv_tc<F, C>;
    static bool attr_set = false;
    if (!attr_set) {
      NNC_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_set = true;
    }
    NNC_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, tmH, tmY, a));
    return NNCONV_OK;
  };
  auto go = [&](auto fmt, auto nc) -> int {
    if (max_keys != nullptr) return go_v(fmt, nc, std::true_type());
    return go_v(fmt, nc, std::false_type());
  };
  auto by_cout = [&](auto fmt) -> int {
    switch (cout) {
      case 16: return go(fmt, std::integral_constant<int, 16>());
      case 32: return go(fmt, std::integral_constant<int, 32>());
      case 48: return go(fmt, std::integral_constant<int, 48>());
      case 64: return go(fmt, std::integral_constant<int, 64>());
      case 80: return go(fmt, std::integral_constant<int, 80>());
      case 96: return go(fmt, std::integral_constant<int, 96>());
      case 112: return go(fmt, std::integral_constant<int, 112>());
      default: return go(fmt, std::integral_constant<int, 128>());
    }
  };
  return bf ? by_cout(std::integral_constant<int, 1>()) : by_cout(std::integral_constant<int, 0>());
}

}  // namespace nnc
