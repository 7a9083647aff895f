// One persistent kernel per NNConv application (tensor-core path): the per-source Y GEMM and the per-edge
// contraction + scatter run CONCURRENTLY inside every CTA as two independent warp-specialised pipelines,
// coupled only through completion flags in global memory and a ring of Y batches that lives in L2.
//
// Why: with one launch per batch of sources (the batch must be small for
// Y to stay L2 resident) every CTA streamed only ~3 tiles per launch and spent as long ramping up / draining
// as streaming; PDL overlapped the launches but not the per-CTA ramps.  Here a CTA never drains: its
// contraction pipeline walks batch after batch (its share of each batch's tiles), while its Y pipeline
// produces the batches ahead.
//
//   roles (14 warps):  0-3 / 4-7 conv warpgroups (tile 0 / tile 1 of every unit: wgmma into registers, scatter)
//                      8-11 Y warpgroup (wgmma into registers, fp16 stores) | 12 conv TMA producer | 13 Y TMA producer
//   flags per batch b: okY[b]  raised when all 4*grid Y warps finished batch b                (conv waits)
//                      okC[b]  raised when all grid CTAs consumed batch b                 (Y waits okC[b-ring])
//
// Math and data movement of the two pipelines are those of conv_tc.cu and gemm_tc.cu.
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
constexpr int kMaxAStages = 10;
constexpr int kTU = 2;
constexpr int kATileBytes = 128 * 64 * 2;
constexpr int kYStages = 2;
constexpr int kThreads = 14 * 32;
constexpr int kConvProducer = 12, kYProducer = 13;
constexpr int kQueue = 8;                  // unit queue between the scheduler and the conv warpgroups
constexpr int kScatterPitch = 272;         // bytes per staged edge row (64 fp32 + 16 B)
constexpr int kScatterBytes = 8 * 32 * kScatterPitch;
constexpr int kYScratchBytes = 4 * acc_scratch_bytes<16>();

struct ApplyArgs {
  // plan
  const int* tile_c;
  const int* tile_e0;
  const int* tile_cnt;
  const int* tile_ptr;    // device [S+1]
  const int* unit_ptr;    // device [S+1]
  const int* unit_t;      // [U]
  const int* unit_u;      // [U]
  const int* dst_sorted;
  const float* inv_deg;   // nullptr -> aggr = add
  const float* cvec;      // [S, cout]
  const float* xs;        // [S] power-of-two row scale of the Y operand (see k_src_prep)
  float* out;             // [N, cout]
  int n_src, nb, n_batches, ring;
  int nb_slots, passes, a_stages, e_pad;
  // PREC_F16X2 (plan.h): split_nk = Kp/64 > 0 -> h holds 2*split_nk chunk panels [hi | lo], a Y ring row is
  // [cout][hi(Kp) | lo(Kp)], and contraction step j = 3q + r pairs (A, B) = (hi_q, Yhi_q), (hi_q, Ylo_q), (lo_q, Yhi_q)
  int split_nk;
  int Kp;
  const float* y_scale;   // PREC_F16X2: inverse of the power-of-two scale of the stored W3p (device scalar), or nullptr
  // Y GEMM
  int NY;                 // cout * Kp
  int num_kx;             // cin_p / 64
  void* Yring;            // [ring * nb, NY] 16-bit
  int* cntY;
  int* okY;
  int* cntC;
  int* okC;
  int* cntU;              // units handed out so far (one counter per application)
  unsigned long long y_store_policy;   // L2 eviction-priority hint of the Y ring stores
  unsigned long long a_policy;         // ... of the h stream loads
  int scatter_mode;                    // 1: rows staged in shared memory + cp.reduce.async.bulk (see options.h)
  int debug_scatter;      // timing experiments only (NNCONV_DEBUG_SCATTER): 1 = drop the scatter, 2 = plain stores
  TraceBuf trace;
};

struct HMaps {
  CUtensorMap m[8];
};

__device__ __forceinline__ void raise_when_all(int* cnt, int* ok, int target) {
  const int prev = atomicAdd(cnt, 1);
  if (prev == target - 1) {
    __threadfence();
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(ok), "r"(1) : "memory");
  }
}

template <int FMT, int kYBlockN, int NC>
__global__ void __launch_bounds__(kThreads, 1)
k_apply_tc(const __grid_constant__ HMaps tmH, const __grid_constant__ CUtensorMap tmY,
           const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, ApplyArgs a) {
  constexpr int kYStageBytes = kATileBytes + kYBlockN * 64 * 2;   // Xc tile + W3p tile
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const int b_chunk_bytes = NC * 128;
  const int b_stride = (b_chunk_bytes + 1023) & ~1023;
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem_b + a.nb_slots * b_stride;
  uint8_t* smem_y = smem_a + a.a_stages * kATileBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_y + kYStages * kYStageBytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kMaxAStages;
  uint64_t* b_full = a_empty + kMaxAStages;
  uint64_t* b_empty = b_full + kMaxSlots;
  uint64_t* y_full = b_empty + kMaxSlots;
  uint64_t* y_empty = y_full + kYStages;
  uint64_t* q_full = y_empty + kYStages;   // [kQueue] 1 arrival (scheduler)
  uint64_t* q_empty = q_full + kQueue;   // [kQueue] 8 arrivals (the conv warps)
  int4* q_ent = reinterpret_cast<int4*>(q_empty + kQueue);
  // Y transposes (4 warps), then the scatter staging (scatter_mode 1: 8 conv warps x 32 rows x kScatterPitch bytes),
  // after the 1 KB barrier block
  float* y_scratch = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 1024);
  uint8_t* smem_sc = reinterpret_cast<uint8_t*>(bars) + 1024 + kYScratchBytes;

  // shfl: the warp index is warp-uniform for the compiler (see tc05::elect_one)
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x / 32), 0), lane = threadIdx.x % 32;
  const unsigned long long tr0 = a.trace.rec ? gtime() : 0ull;

  if (warp == kConvProducer && lane == 0) {
    for (int i = 0; i < 8; ++i) prefetch_tmap(&tmH.m[i]);
    prefetch_tmap(&tmY);
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW);
    for (int s = 0; s < a.a_stages; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 4);          // the 4 warps of the tile's warpgroup
    }
    for (int j = 0; j < a.nb_slots; ++j) {
      mbar_init(&b_full[j], 1);
      mbar_init(&b_empty[j], 8);          // both conv warpgroups
    }
    for (int s = 0; s < kYStages; ++s) {
      mbar_init(&y_full[s], 1);
      mbar_init(&y_empty[s], 4);
    }
    for (int s = 0; s < kQueue; ++s) {
      mbar_init(&q_full[s], 1);
      mbar_init(&q_empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // ---- contraction work distribution: units (<= 2 tiles of one source) of batch b are handed out
  // dynamically (atomic counter per batch) to whichever CTA is ready, so that the period of a batch is not set by
  // its slowest CTA (as with a static equal split).
  // The producer thread grabs units and publishes them to the conv warpgroups through a small
  // shared-memory queue: entry = {first tile, #tiles (0 = end of this CTA's share of batch b, -1 = done), c, b}.
  if (warp == kConvProducer) {
    // ============================================================== contraction: TMA producer + scheduler
    // (whole warp runs the loops; the elected lane issues -- see tc05::elect_one)
    ARing ring[kTU];
#pragma unroll
    for (int ti = 0; ti < kTU; ++ti) ring[ti].init(ti, a.a_stages);
    int bs = 0;               // B slot ring (one slot per K chunk of the current unit's Y slice)
    uint32_t bph = 0;
    const int num_kc = a.passes * a.nb_slots;
    int qi = 0;
    uint32_t qph = 0;
    auto publish = [&](int t, int u, int c, int b) {
      mbar_wait(&q_empty[qi], qph ^ 1u);
      if (elect_one()) {
        q_ent[qi] = make_int4(t, u, c, b);
        mbar_arrive(&q_full[qi]);                         // release: entry visible to the waiters
      }
      __syncwarp();
      if (++qi == kQueue) { qi = 0; qph ^= 1u; }
    };
    // ONE unit counter for the whole application: units are globally ordered by source, so the batch of
    // a unit follows from its source (b = c / nb); the grab of the next unit is always in flight while the
    // current one streams (no exposed atomic round trip at batch boundaries).
    auto grab = [&]() {
      int v = 0;
      if (lane == 0) v = atomicAdd(a.cntU, 1);
      return __shfl_sync(0xffffffffu, v, 0);
    };
    const int n_units = __ldg(a.unit_ptr + a.n_src);
    int nxt = grab();
    int cur_b = -1;
    while (nxt < n_units) {
      const int ui = nxt;
      nxt = grab();                                       // grab the NEXT unit now
      const int ut = __shfl_sync(0xffffffffu, __ldg(a.unit_t + ui), 0);
      const int uu = __shfl_sync(0xffffffffu, __ldg(a.unit_u + ui), 0);
      const int uc = __shfl_sync(0xffffffffu, __ldg(a.tile_c + ut), 0);
      const int b = uc / a.nb;
      if (b != cur_b) {
        const unsigned long long tw0 = a.trace.rec ? gtime() : 0ull;
        if (lane == 0) flag_wait(a.okY + b);              // Y of this batch is complete (and visible to TMA)
        __syncwarp();
        asm volatile("fence.proxy.async.global;" ::: "memory");
        if (a.trace.rec && lane == 0 && (blockIdx.x % 37) == 0)
          trace_write(a.trace, 301u | (static_cast<unsigned>(b) << 12), tw0, gtime(), 0ull);
        cur_b = b;
      }
      const int ring_row0 = (b % a.ring) * a.nb - b * a.nb;
      publish(ut, uu, uc, b);
      int te0[kTU], tbox[kTU];
#pragma unroll
      for (int ti = 0; ti < kTU; ++ti) {
        te0[ti] = ti < uu ? __shfl_sync(0xffffffffu, __ldg(a.tile_e0 + ut + ti), 0) : 0;
        tbox[ti] = ti < uu ? (__shfl_sync(0xffffffffu, __ldg(a.tile_cnt + ut + ti), 0) + 15) >> 4 : 1;
      }
      // K chunk outer, tile inner: the B slot of chunk j is released after the unit's LAST tile and needed again
      // only nb_slots chunks later, i.e. 2*nb_slots - 1 MMA blocks for a 2-tile unit (a pass-major order leaves only
      // nb_slots - 1)
      for (int j = 0; j < num_kc; ++j) {
        int ja = j, jb = j;
        if (a.split_nk > 0) {
          const int q = j / 3, r = j - 3 * q;
          ja = r == 2 ? a.split_nk + q : q;
          jb = r == 1 ? a.split_nk + q : q;
        }
        mbar_wait(&b_empty[bs], bph ^ 1u);
        if (elect_one()) {
          mbar_arrive_expect_tx(&b_full[bs], b_chunk_bytes);
          tma_load_2d(smem_b + bs * b_stride, &tmY, &b_full[bs], jb * 64, (ring_row0 + uc) * NC, kEvictLast);
        }
        __syncwarp();
        if (++bs == a.nb_slots) { bs = 0; bph ^= 1u; }
#pragma unroll
        for (int ti = 0; ti < kTU; ++ti) {
          if (ti < uu) {
            const CUtensorMap* mh = &tmH.m[tbox[ti] - 1];
            const uint32_t a_bytes = static_cast<uint32_t>(tbox[ti]) * 16u * 128u;
            const int stage = ring[ti].stage;
            mbar_wait(&a_empty[stage], ring[ti].phase ^ 1u);
            if (elect_one()) {
              mbar_arrive_expect_tx(&a_full[stage], a_bytes);
              tma_load_2d(smem_a + stage * kATileBytes, mh, &a_full[stage], 0, ja * a.e_pad + te0[ti], a.a_policy);
            }
            __syncwarp();
            ring[ti].next();
          }
        }
      }
    }
    publish(0, -1, 0, 0);
  } else if (warp < 8) {
    // ============================================================== contraction: warpgroup g = tile g of every unit
    const int g = warp / 4, quarter = warp % 4;
    Acc<NC> acc;
    ARing ring;
    ring.init(g, a.a_stages);
    int bs = 0;
    uint32_t bph = 0;
    const int num_kc = a.passes * a.nb_slots;
    int qi = 0;
    uint32_t qph = 0;
    // fragment rows of this thread (acc_row numbering: lane L of the warp stands for row acc_row(quarter, L))
    const int fr = lane >> 2, fc = (lane & 3) * 2;
    const uint32_t my_rows = smem_u32(smem_sc) + static_cast<uint32_t>(warp * 32 * kScatterPitch);
    for (;;) {
      mbar_wait(&q_full[qi], qph);
      int4 en = q_ent[qi];
      en.y = __shfl_sync(0xffffffffu, en.y, 0);          // warp-uniform: wgmma sits under `g < en.y`
      __syncwarp();
      if (lane == 0) mbar_arrive(&q_empty[qi]);
      if (++qi == kQueue) { qi = 0; qph ^= 1u; }
      if (en.y < 0) break;
      if (en.y == 0) continue;
      for (int j = 0; j < num_kc; ++j) {
        mbar_wait(&b_full[bs], bph);
        const uint64_t bdesc = smem_desc_sw128(smem_u32(smem_b + bs * b_stride));
        if (g < en.y) {
          mbar_wait(&a_full[ring.stage], ring.phase);
          const uint64_t adesc = smem_desc_sw128(smem_u32(smem_a + ring.stage * kATileBytes));
          mma_block<NC, FMT>(acc, adesc, bdesc, 512, 2, 4, j != 0);
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_empty[ring.stage]);
          ring.next();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[bs]);          // B is re-loaded for every unit
        if (++bs == a.nb_slots) { bs = 0; bph ^= 1u; }
      }
      // every MMA that read this unit's Y slice has completed: count the unit; the last unit of batch b frees the
      // ring slot for the Y pipeline
      named_bar_sync(1, 256);
      if (warp == 0 && lane == 0) {
        const int c0 = en.w * a.nb;
        const int target = __ldg(a.unit_ptr + min(c0 + a.nb, a.n_src)) - __ldg(a.unit_ptr + c0);
        raise_when_all(a.cntC + en.w, a.okC + en.w, target);
      }
      if (g >= en.y) continue;
      // ---- scatter of tile g straight from the accumulator fragments: thread (lane) holds rows
      // L = fr, fr + 8 (first m64 half) and 16 + fr, 24 + fr (second half) of the warp, columns 8 jj + fc, + 1
      const int r = acc_row(quarter, lane);
      const bool ok = r < a.tile_cnt[en.x + g];
      int d = 0;
      float sc = 1.f;
      if (ok) {
        d = __ldg(a.dst_sorted + a.tile_e0[en.x + g] + r);
        if (a.inv_deg) sc = __ldg(a.inv_deg + d);
      }
      const float* cv = a.cvec + static_cast<int64_t>(en.z) * NC;
      const float xsc = __ldg(a.xs + en.z);
      float* orow = a.out + static_cast<int64_t>(d) * NC;
      int fd[4];
      float fsc[4];
      bool fok[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int L = fr + 8 * i;
        fd[i] = __shfl_sync(0xffffffffu, d, L);
        fsc[i] = __shfl_sync(0xffffffffu, sc, L);
        fok[i] = __shfl_sync(0xffffffffu, ok ? 1 : 0, L) != 0;
      }
      if (a.scatter_mode == 1) {
        // rows staged in shared memory, then one bulk reduction per row (its lane issues it)
        bulk_wait_read0();                                 // this lane's previous row has left its staging slot
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < NC / 8; ++jj) {
          const float2 cq = __ldg(reinterpret_cast<const float2*>(cv + 8 * jj + fc));
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float* dv = acc.d[i >> 1] + 4 * jj + 2 * (i & 1);
            const uint32_t addr = my_rows + static_cast<uint32_t>((fr + 8 * i) * kScatterPitch + (8 * jj + fc) * 4);
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(fmaf(dv[0], xsc, cq.x) * fsc[i]),
                         "f"(fmaf(dv[1], xsc, cq.y) * fsc[i])
                         : "memory");
          }
        }
        fence_proxy_async_smem();                         // generic-proxy writes of the warp -> async proxy
        __syncwarp();
        if (ok) bulk_reduce_add_f32(orow, my_rows + static_cast<uint32_t>(lane * kScatterPitch), static_cast<uint32_t>(NC) * 4u);
        bulk_commit();
      } else if (a.debug_scatter != 1) {
#pragma unroll
        for (int jj = 0; jj < NC / 8; ++jj) {
          const float2 cq = __ldg(reinterpret_cast<const float2*>(cv + 8 * jj + fc));
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (!fok[i]) continue;
            const float* dv = acc.d[i >> 1] + 4 * jj + 2 * (i & 1);
            float* dst = a.out + static_cast<int64_t>(fd[i]) * NC + 8 * jj + fc;
            if (a.debug_scatter == 2) {
              *reinterpret_cast<float2*>(dst) = make_float2(dv[0], dv[1]);
            } else {
              asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(fmaf(dv[0], xsc, cq.x) * fsc[i]),
                           "f"(fmaf(dv[1], xsc, cq.y) * fsc[i])
                           : "memory");
            }
          }
        }
      }
    }
    if (a.scatter_mode == 1) bulk_wait0();                  // every row has been added before the CTA retires
  } else if (warp == kYProducer) {
    // ============================================================== Y GEMM: TMA producer (whole warp, elected lane)
    const int n_blocks = a.NY / kYBlockN;
    int stage = 0;
    uint32_t phase = 0;
    for (int b = 0; b < a.n_batches; ++b) {
      const int c0 = b * a.nb;
      const int rows = min(a.nb, a.n_src - c0);
      const int tiles = ((rows + 127) / 128) * n_blocks;
      for (int i = static_cast<int>((blockIdx.x + 7u * b) % gridDim.x); i < tiles; i += gridDim.x) {
        const int mb = i / n_blocks, nbk = i % n_blocks;
        for (int kx = 0; kx < a.num_kx; ++kx) {
          mbar_wait(&y_empty[stage], phase ^ 1u);
          if (elect_one()) {
            mbar_arrive_expect_tx(&y_full[stage], kYStageBytes);
            uint8_t* st = smem_y + stage * kYStageBytes;
            tma_load_2d(st, &tmX, &y_full[stage], kx * 64, c0 + mb * 128, kEvictLast);
            tma_load_2d(st + kATileBytes, &tmW, &y_full[stage], kx * 64, nbk * kYBlockN, kEvictLast);
          }
          __syncwarp();
          if (++stage == kYStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ================================================================ Y GEMM: warpgroup of warps 8..11
    const int quarter = warp % 4;
    const int n_blocks = a.NY / kYBlockN;
    float* wb = y_scratch + quarter * (acc_scratch_bytes<16>() / 4);
    Acc<kYBlockN> acc;
    int stage = 0;
    uint32_t phase = 0;
    for (int b = 0; b < a.n_batches; ++b) {
      const int c0 = b * a.nb;
      const int rows = min(a.nb, a.n_src - c0);
      const int tiles = ((rows + 127) / 128) * n_blocks;
      const unsigned long long ty0 = a.trace.rec ? gtime() : 0ull;
      if (b >= a.ring) {                         // the ring slot must have been consumed by every CTA
        // ONE slow poller per CTA (the Y pipeline runs ring-1 batches ahead, so this wait is long and never
        // urgent); the other three warps of the Y warpgroup park on a named barrier
        if (warp == 8 && lane == 0) flag_wait(a.okC + (b - a.ring), 500);
        named_bar_sync(2, 128);
      }
      const unsigned long long ty1 = a.trace.rec ? gtime() : 0ull;
      const int ymul = a.split_nk > 0 ? 2 : 1;
      const float ysc = a.y_scale != nullptr ? __ldg(a.y_scale) : 1.f;
      uint16_t* ybase = reinterpret_cast<uint16_t*>(a.Yring) + static_cast<int64_t>(b % a.ring) * a.nb * a.NY * ymul;
      for (int i = static_cast<int>((blockIdx.x + 7u * b) % gridDim.x); i < tiles; i += gridDim.x) {
        const int mb = i / n_blocks, nbk = i % n_blocks;
        for (int kx = 0; kx < a.num_kx; ++kx) {
          mbar_wait(&y_full[stage], phase);
          uint8_t* st = smem_y + stage * kYStageBytes;
          mma_block<kYBlockN, FMT>(acc, smem_desc_sw128(smem_u32(st)), smem_desc_sw128(smem_u32(st + kATileBytes)), 512, 2,
                                   4, kx != 0);
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&y_empty[stage]);
          if (++stage == kYStages) { stage = 0; phase ^= 1u; }
        }
        const int row = mb * 128 + acc_row(quarter, lane);
        const bool row_ok = row < rows;
        // column n = o * Kp + k of the source's matrix; with split rows of 2*Kp: offset n + o * Kp
        const int n0 = nbk * kYBlockN;
        uint16_t* yrow0 = ybase + static_cast<int64_t>(row) * a.NY * ymul;
#pragma unroll
        for (int cc = 0; cc < kYBlockN / 16; ++cc) {
          uint32_t vv[16];
          acc_rows<kYBlockN, 16>(acc, cc * 16, wb, vv);
          if (row_ok) {
            uint32_t packed[8], packed_lo[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float f0 = __uint_as_float(vv[2 * j]), f1 = __uint_as_float(vv[2 * j + 1]);
              if (FMT == 0 && a.split_nk > 0) { f0 *= ysc; f1 *= ysc; }
              if (FMT == 0) {
                __half2 hh = __floats2half2_rn(f0, f1);
                packed[j] = *reinterpret_cast<uint32_t*>(&hh);
                if (a.split_nk > 0) {
                  const float2 hf = __half22float2(hh);
                  __half2 ll = __floats2half2_rn(f0 - hf.x, f1 - hf.y);
                  packed_lo[j] = *reinterpret_cast<uint32_t*>(&ll);
                }
              } else {
                __nv_bfloat162 hh = __floats2bfloat162_rn(f0, f1);
                packed[j] = *reinterpret_cast<uint32_t*>(&hh);
              }
            }
            const int n = n0 + cc * 16;
            uint16_t* yrow = yrow0 + n + (a.split_nk > 0 ? (n / a.Kp) * a.Kp : 0);
            st_global_32b_hint(yrow, packed, a.y_store_policy);
            if (FMT == 0 && a.split_nk > 0) st_global_32b_hint(yrow + a.Kp, packed_lo, a.y_store_policy);
          }
        }
      }
      // this warp's stores of batch b are out: 4 warps x grid arrivals complete the batch
      __threadfence();
      __syncwarp();
      if (lane == 0) raise_when_all(a.cntY + b, a.okY + b, 4 * static_cast<int>(gridDim.x));
      if (a.trace.rec && warp == 8 && lane == 0 && (blockIdx.x % 37) == 0)
        trace_write(a.trace, 302u | (static_cast<unsigned>(b) << 12), ty0, ty1, gtime());
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) trace_write(a.trace, 300u, tr0, tr0, a.trace.rec ? gtime() : 0ull);
}

struct ApplyShape {
  int nb_slots, passes, a_stages, smem_bytes;
};

bool apply_shape(int cout, int Kp, int ybn, ApplyShape* as) {
  const int kYStageBytes = kATileBytes + ybn * 64 * 2;
  if (cout % 16 != 0 || cout < 16 || cout > 64 || Kp % 64 != 0) return false;
  const int num_kc = Kp / 64;
  const int b_stride = (cout * 128 + 1023) & ~1023;
  const int bar_bytes = 1024 + kYScratchBytes + (options().scatter_mode == 1 ? kScatterBytes : 0);
  const int budget = 227 * 1024 - bar_bytes - kYStages * kYStageBytes;
  // fewest passes that leave >= 7 A stages (the h stream needs the bytes in flight), else >= 5, else >= 3
  const int forced = options().apply_passes;
  for (int min_stages = 7; min_stages >= 3; min_stages -= 2) {
    for (int passes = 1; passes <= num_kc; ++passes) {
      if (num_kc % passes) continue;
      if (forced > 0 && passes != forced && num_kc % forced == 0) continue;
      const int nb = num_kc / passes;
      if (nb > kMaxSlots) continue;
      if (passes > 1 && nb < 4) continue;   // too little time between a slot's release and its next use
      int stages = (budget - nb * b_stride) / kATileBytes;
      if (stages > kMaxAStages) stages = kMaxAStages;
      if (stages >= min_stages) {
        as->nb_slots = nb;
        as->passes = passes;
        as->a_stages = stages;
        as->smem_bytes = nb * b_stride + stages * kATileBytes + kYStages * kYStageBytes + bar_bytes;
        return true;
      }
    }
  }
  return false;
}

}  // namespace

// N tile of the Y pipeline: 64 columns = 64 accumulator registers per thread of the Y warpgroup, which shares the SM's
// register file with the two conv warpgroups (a 128-column tile spills and serialises its wgmma on sm_90)
constexpr int kYBN = 64;

static int eff_kp(const Weights* W) { return W->split ? 3 * W->Kp : W->Kp; }

bool apply_fused_supported(const Weights* W) {
  if (W->prec != PREC_F16 && W->prec != PREC_BF16 && W->prec != PREC_F16X2) return false;
  if ((W->cout * W->Kp) % 128 != 0) return false;
  ApplyShape as;
  return apply_shape(W->cout, eff_kp(W), kYBN, &as);
}

namespace {
template <int FMT, int YBN, int NC>
int launch_variant(int grid, int smem_bytes, bool coop, cudaStream_t st, const HMaps& tmH, const CUtensorMap& tmY,
                   const CUtensorMap& tmX, const CUtensorMap& tmW, const ApplyArgs& a) {
  static bool attr_set = false;
  static int blocks_per_sm = -1;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_apply_tc<FMT, YBN, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  if (blocks_per_sm < 0)
    NNC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k_apply_tc<FMT, YBN, NC>, kThreads,
                                                                 smem_bytes));
  NNC_REQUIRE(blocks_per_sm >= 1, NNCONV_ERR_UNSUPPORTED, "apply_tc: the persistent kernel does not fit one SM");
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  // The CTAs of this kernel wait for each other (okY / okC flags), so ALL of them must be resident at the same
  // time.  A cooperative launch makes the driver guarantee exactly that: it only starts the grid once every CTA
  // can be co-scheduled, whatever else (an overlapped NCCL kernel, a second stream, MPS) holds SMs right now,
  // and fails with cudaErrorCooperativeLaunchTooLarge when that can never happen -- the caller then falls back
  // to the per-batch kernels, which need no co-residency.
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = coop ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, k_apply_tc<FMT, YBN, NC>, tmH, tmY, tmX, tmW, a);
  if (e == cudaErrorCooperativeLaunchTooLarge) {
    cudaGetLastError();
    return kApplyCannotCoSchedule;   // handled by apply(): per-batch kernels instead
  }
  NNC_CHECK_CUDA(e);
  return NNCONV_OK;
}
}  // namespace

int launch_apply_tc(int prec, const Plan* P, const Weights* W, const void* h, const void* Xc, void* Yring, int nb,
                    int ring, const float* cvec, const float* xs, int aggr_mean, float* out, int* flags,
                    int flags_stride, cudaStream_t st) {
  int s = tc_init();
  if (s != NNCONV_OK) return s;
  const Options& opt = options();
  const int bf = prec == PREC_BF16;
  const int split = W->split ? 1 : 0;
  const int ybn = kYBN;
  ApplyShape as;
  NNC_REQUIRE(apply_shape(W->cout, eff_kp(W), ybn, &as), NNCONV_ERR_UNSUPPORTED, "apply_tc: unsupported shape");
  if (opt.apply_stages >= 2 && opt.apply_stages < as.a_stages) as.a_stages = opt.apply_stages;
  const int64_t e_pad = round_up64(P->E, 128);
  const int NY = W->cout * W->Kp;
  const int kmul = split ? 2 : 1;      // [hi | lo] activations / Y rows
  const int xmul = split ? 3 : 1;      // [hi | hi | lo] x [hi | lo | hi] operands of the Y GEMM
  const int n_batches = ceil_div(P->n_src, nb);
  NNC_REQUIRE(n_batches <= flags_stride, NNCONV_ERR_WORKSPACE, "apply_tc: too many source batches (%d)", n_batches);
  NNC_REQUIRE(static_cast<uint64_t>(kmul * W->Kp / 64) * e_pad < (1ull << 31), NNCONV_ERR_UNSUPPORTED,
              "apply_tc: edge-feature tensor exceeds 2^31 rows of 64 columns");
  HMaps tmH;
  CUtensorMap tmY, tmX, tmW;
  for (int i = 0; i < 8; ++i) {
    s = make_tmap_2d_16b(&tmH.m[i], bf, h, static_cast<uint64_t>(kmul * W->Kp / 64) * e_pad, 64, 16 * (i + 1));
    if (s != NNCONV_OK) return s;
  }
  s = make_tmap_2d_16b(&tmY, bf, Yring, static_cast<uint64_t>(ring) * nb * W->cout, static_cast<uint64_t>(kmul) * W->Kp,
                       W->cout);
  if (s != NNCONV_OK) return s;
  s = make_tmap_2d_16b(&tmX, bf, Xc, static_cast<uint64_t>(P->n_src), static_cast<uint64_t>(xmul) * W->cin_p, 128);
  if (s != NNCONV_OK) return s;
  s = make_tmap_2d_16b(&tmW, bf, W->W3p, static_cast<uint64_t>(NY), static_cast<uint64_t>(xmul) * W->cin_p, ybn);
  if (s != NNCONV_OK) return s;
  ApplyArgs a;
  a.tile_c = P->tile_c; a.tile_e0 = P->tile_e0; a.tile_cnt = P->tile_cnt; a.tile_ptr = P->tile_ptr;
  a.unit_ptr = P->unit_ptr; a.unit_t = P->unit_t; a.unit_u = P->unit_u;
  a.dst_sorted = P->dst_sorted; a.inv_deg = aggr_mean ? P->inv_deg : nullptr; a.cvec = cvec; a.xs = xs; a.out = out;
  a.n_src = P->n_src; a.nb = nb; a.n_batches = n_batches; a.ring = ring;
  a.nb_slots = as.nb_slots; a.passes = as.passes; a.a_stages = as.a_stages;
  a.e_pad = static_cast<int>(e_pad);
  a.split_nk = split ? W->Kp / 64 : 0;
  a.Kp = W->Kp;
  a.y_scale = (split && W->wscale) ? W->wscale + 2 * W->n_layers + 1 : nullptr;
  a.NY = NY; a.num_kx = xmul * W->cin_p / 64; a.Yring = Yring;
  a.y_store_policy = opt.y_store_policy == 1 ? kEvictLast : opt.y_store_policy == 2 ? kEvictFirst : kEvictNormal;
  a.a_policy = opt.apply_a_policy == 1 ? kEvictNormal : kEvictFirst;
  a.scatter_mode = (opt.scatter_mode == 1 && W->cout <= 64) ? 1 : 0;
  a.debug_scatter = opt.debug_scatter;   // wrong results, timing only
  a.cntY = flags; a.cntC = flags + flags_stride; a.okY = flags + 2 * flags_stride; a.okC = flags + 3 * flags_stride;
  a.cntU = flags + 4 * flags_stride;
  {
    TraceHandle th = trace_get();
    a.trace = TraceBuf{th.rec, th.count, th.cap};
  }
  // Optional (l2_persist option): pin the Y ring in L2 with an access-policy window on the caller's stream
  // for the duration of this launch (persisting hits for the ring, everything else streaming).
  bool window_set = false;
  if (opt.l2_persist > 0) {
    static int max_persist = -1;
    if (max_persist < 0) {
      int dev = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev);
      if (opt.l2_persist > 1 && (static_cast<size_t>(opt.l2_persist) << 20) < static_cast<size_t>(max_persist))
        max_persist = opt.l2_persist << 20;
      if (max_persist > 0) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, static_cast<size_t>(max_persist));
    }
    const size_t ring_bytes = static_cast<size_t>(ring) * nb * NY * 2 * kmul;
    if (max_persist > 0) {
      cudaStreamAttrValue v{};
      v.accessPolicyWindow.base_ptr = Yring;
      v.accessPolicyWindow.num_bytes = ring_bytes;
      v.accessPolicyWindow.hitRatio = ring_bytes <= static_cast<size_t>(max_persist)
                                          ? 1.0f
                                          : static_cast<float>(max_persist) / static_cast<float>(ring_bytes);
      v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      window_set = cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v) == cudaSuccess;
    }
  }
  // exactly one CTA per SM, never more than #SMs (see launch_variant about co-residency)
  const int grid = tc_num_sms();
  const bool coop = opt.no_coop == 0;
  auto go = [&](auto fmt, auto nc) -> int {
    return launch_variant<decltype(fmt)::value, kYBN, decltype(nc)::value>(grid, as.smem_bytes, coop, st,
                                                                                           tmH, tmY, tmX, tmW, a);
  };
  auto by_cout = [&](auto fmt) -> int {
    switch (W->cout) {
      case 16: return go(fmt, std::integral_constant<int, 16>());
      case 32: return go(fmt, std::integral_constant<int, 32>());
      case 48: return go(fmt, std::integral_constant<int, 48>());
      default: return go(fmt, std::integral_constant<int, 64>());
    }
  };
  s = bf ? by_cout(std::integral_constant<int, 1>()) : by_cout(std::integral_constant<int, 0>());
  if (window_set) {
    cudaStreamAttrValue v{};
    v.accessPolicyWindow.num_bytes = 0;
    cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v);
  }
  return s;
}

}  // namespace nnc
