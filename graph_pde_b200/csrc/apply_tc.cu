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
constexpr int kScatterRows = 16;           // staged rows per conv warp: its 32 rows go out as two halves
constexpr int kScatterBytes = 8 * kScatterRows * kScatterPitch;
// aggr = max: a staged row holds NC 8-byte keys (512 B at NC = 64); a warp's 32 rows go out in four trips of 8 rows
// through the same staging slots
constexpr int kKeyPitch = 64 * 8 + 16;
constexpr int kKeyRows = 8;
static_assert(kKeyRows * kKeyPitch <= kScatterRows * kScatterPitch, "key rows exceed a warp's scatter staging");
constexpr int kMaxXBytes = 3 * kATileBytes;   // largest Xc tile (num_kx boxes) the Y GEMM keeps resident
constexpr int kYStagingBytes = 4 * 32 * 128;   // Y epilogue: per Y warp, its 32 rows x 64 16-bit columns

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
  // the launch contracts units [u_begin, u_end) of sources [c_begin, c_end); its Y batches are numbered from c_begin
  // (batch b = sources c_begin + b*nb ..), and h holds the rows of sorted edges [e_base, e_base + e_pad) only
  int u_begin, u_end, c_begin, c_end, e_base;
  int nb, n_batches, ring;
  int nb_slots, passes, a_stages, e_pad;
  int x_resident;         // Y GEMM: the Xc tile of a (batch, m-block) stays in shared memory while its n-blocks stream
  int y_bytes;            // shared memory of the Y GEMM (resident Xc tile and / or its stages)
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
  // aggr = max (the MAX instantiation only): [N, cout] keys (common.cuh max_key) and the plan's perm (nullable)
  unsigned long long* keys;
  const int* perm;
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

// The kernel body, shared by k_apply_tc (aggr add / mean) and k_apply_tc_max.  MAX: aggr = max -- the epilogue
// reduces each edge row's keys into a.keys with one bulk max.u64 request (DESIGN 4.1).
template <int FMT, int kYBlockN, int NC, bool MAX>
__device__ __forceinline__ void apply_tc_body(const HMaps& tmH, const CUtensorMap& tmY, const CUtensorMap& tmX,
                                              const CUtensorMap& tmW, const ApplyArgs& a) {
  constexpr int kWBytes = kYBlockN * 64 * 2;   // one W3p box
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  const int b_chunk_bytes = NC * 128;
  const int b_stride = (b_chunk_bytes + 1023) & ~1023;
  uint8_t* smem_b = smem;
  uint8_t* smem_a = smem_b + a.nb_slots * b_stride;
  // Y GEMM: [Xc tile: num_kx boxes, if resident][kYStages x (W3p box, preceded by its Xc box if not resident)]
  const int y_stage_bytes = a.x_resident ? kWBytes : kATileBytes + kWBytes;
  uint8_t* smem_x = smem_a + a.a_stages * kATileBytes;
  uint8_t* smem_y = smem_x + (a.x_resident ? a.num_kx * kATileBytes : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_a + a.a_stages * kATileBytes + a.y_bytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kMaxAStages;
  uint64_t* b_full = a_empty + kMaxAStages;
  uint64_t* b_empty = b_full + kMaxSlots;
  uint64_t* y_full = b_empty + kMaxSlots;
  uint64_t* y_empty = y_full + kYStages;
  uint64_t* q_full = y_empty + kYStages;   // [kQueue] 1 arrival (scheduler)
  uint64_t* q_empty = q_full + kQueue;   // [kQueue] 8 arrivals (the conv warps)
  uint64_t* x_full = q_empty + kQueue;     // resident Xc tile: 1 arrival (+ tx)
  uint64_t* x_empty = x_full + 1;          // 4 arrivals (the Y warps, when they move on to the next tile)
  int4* q_ent = reinterpret_cast<int4*>(x_empty + 1);
  // Y epilogue staging (4 warps), then the scatter staging (scatter_mode 1: 8 conv warps x kScatterRows x
  // kScatterPitch bytes), after the 1 KB barrier block
  uint8_t* y_staging = reinterpret_cast<uint8_t*>(bars) + 1024;
  uint8_t* smem_sc = reinterpret_cast<uint8_t*>(bars) + 1024 + kYStagingBytes;

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
    mbar_init(x_full, 1);
    mbar_init(x_empty, 4);
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
      if (lane == 0) v = a.u_begin + atomicAdd(a.cntU, 1);
      return __shfl_sync(0xffffffffu, v, 0);
    };
    const int n_units = a.u_end;
    int nxt = grab();
    int cur_b = -1;
    while (nxt < n_units) {
      const int ui = nxt;
      nxt = grab();                                       // grab the NEXT unit now
      const int ut = __shfl_sync(0xffffffffu, __ldg(a.unit_t + ui), 0);
      const int uu = __shfl_sync(0xffffffffu, __ldg(a.unit_u + ui), 0);
      const int uc = __shfl_sync(0xffffffffu, __ldg(a.tile_c + ut), 0);
      const int b = (uc - a.c_begin) / a.nb;
      if (b != cur_b) {
        const unsigned long long tw0 = a.trace.rec ? gtime() : 0ull;
        if (lane == 0) flag_wait(a.okY + b);              // Y of this batch is complete (and visible to TMA)
        __syncwarp();
        asm volatile("fence.proxy.async.global;" ::: "memory");
        if (a.trace.rec && lane == 0 && (blockIdx.x % 37) == 0)
          trace_write(a.trace, 301u | (static_cast<unsigned>(b) << 12), tw0, gtime(), 0ull);
        cur_b = b;
      }
      const int ring_row0 = (b % a.ring) * a.nb - b * a.nb - a.c_begin;
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
              tma_load_2d(smem_a + stage * kATileBytes, mh, &a_full[stage], 0, ja * a.e_pad + te0[ti] - a.e_base,
                          a.a_policy);
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
    const uint32_t my_rows = smem_u32(smem_sc) + static_cast<uint32_t>(warp * kScatterRows * kScatterPitch);
    for (;;) {
      mbar_wait(&q_full[qi], qph);
      int4 en = q_ent[qi];
      en.y = __shfl_sync(0xffffffffu, en.y, 0);          // warp-uniform: wgmma sits under `g < en.y`
      __syncwarp();
      if (lane == 0) mbar_arrive(&q_empty[qi]);
      if (++qi == kQueue) { qi = 0; qph ^= 1u; }
      if (en.y < 0) break;
      if (en.y == 0) continue;
      // a block's A stage and B slot are released as soon as its MMAs retire: keeping one block in flight (as
      // k_gemm_tc does) holds every stage and B slot one block longer, which measured slower here (DESIGN 4.3)
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
        const int c0 = a.c_begin + en.w * a.nb;
        const int target = min(__ldg(a.unit_ptr + min(c0 + a.nb, a.c_end)), a.u_end) - max(__ldg(a.unit_ptr + c0), a.u_begin);
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
      if constexpr (MAX) {
        // the keys of the message add scatters (no degree scale), rows staged in shared memory, then ONE bulk
        // .max.u64 reduction of NC * 8 bytes per row (its lane issues it); the warp's 32 rows go out in four trips of
        // 8 -- rows 8 h + r (fragment i = h) in trip h -- through its scatter staging slots
        const uint32_t ce = ok ? caller_edge(a.perm, a.tile_e0[en.x + g] + r) : 0u;
        unsigned long long* krow = a.keys + static_cast<int64_t>(d) * NC;
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const uint32_t ceh = __shfl_sync(0xffffffffu, ce, fr + 8 * h);
          bulk_wait_read0();                               // this lane's previous row has left its staging slot
          __syncwarp();
#pragma unroll
          for (int jj = 0; jj < NC / 8; ++jj) {
            const float2 cq = __ldg(reinterpret_cast<const float2*>(cv + 8 * jj + fc));
            const float* dv = acc.d[h >> 1] + 4 * jj + 2 * (h & 1);
            const unsigned long long k0 = max_key(fmaf(dv[0], xsc, cq.x), ceh);
            const unsigned long long k1 = max_key(fmaf(dv[1], xsc, cq.y), ceh);
            const uint32_t addr = my_rows + static_cast<uint32_t>(fr * kKeyPitch + (8 * jj + fc) * 8);
            asm volatile("st.shared.v2.u64 [%0], {%1, %2};" ::"r"(addr), "l"(k0), "l"(k1) : "memory");
          }
          fence_proxy_async_smem();                       // generic-proxy writes of the warp -> async proxy
          __syncwarp();
          if (ok && (lane >> 3) == h)
            bulk_reduce_max_u64(krow, my_rows + static_cast<uint32_t>((lane & 7) * kKeyPitch), static_cast<uint32_t>(NC) * 8u);
          bulk_commit();
        }
      } else if (a.scatter_mode == 1) {
        // rows staged in shared memory, then one bulk reduction per row (its lane issues it); the warp's 32 rows go
        // out as two halves of 16 through the same staging slots: rows 16 h + r (fragment i = 2 h, 2 h + 1) in half h
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          bulk_wait_read0();                               // this lane's previous row has left its staging slot
          __syncwarp();
#pragma unroll
          for (int jj = 0; jj < NC / 8; ++jj) {
            const float2 cq = __ldg(reinterpret_cast<const float2*>(cv + 8 * jj + fc));
#pragma unroll
            for (int i = 2 * h; i < 2 * h + 2; ++i) {
              const float* dv = acc.d[i >> 1] + 4 * jj + 2 * (i & 1);
              const uint32_t addr = my_rows + static_cast<uint32_t>((fr + 8 * (i & 1)) * kScatterPitch + (8 * jj + fc) * 4);
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(fmaf(dv[0], xsc, cq.x) * fsc[i]),
                           "f"(fmaf(dv[1], xsc, cq.y) * fsc[i])
                           : "memory");
            }
          }
          fence_proxy_async_smem();                       // generic-proxy writes of the warp -> async proxy
          __syncwarp();
          if (ok && (lane >> 4) == h)
            bulk_reduce_add_f32(orow, my_rows + static_cast<uint32_t>((lane & 15) * kScatterPitch), static_cast<uint32_t>(NC) * 4u);
          bulk_commit();
        }
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
    if (MAX || a.scatter_mode == 1) bulk_wait0();           // every row has been reduced before the CTA retires
  } else if (warp == kYProducer) {
    // ============================================================== Y GEMM: TMA producer (whole warp, elected lane)
    const int n_blocks = a.NY / kYBlockN;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t xph = 0;
    int x_b = -1, x_mb = -1;   // (batch, m-block) of the resident Xc tile
    for (int b = 0; b < a.n_batches; ++b) {
      const int c0 = a.c_begin + b * a.nb;
      const int rows = min(a.nb, a.c_end - c0);
      const int tiles = ((rows + 127) / 128) * n_blocks;
      // a contiguous range of the batch's tiles per CTA (rotated by batch), so that the resident Xc tile changes at
      // most once per n_blocks tiles
      const int64_t rot = (blockIdx.x + 7u * b) % gridDim.x;
      const int t_end = static_cast<int>(tiles * (rot + 1) / gridDim.x);
      for (int i = static_cast<int>(tiles * rot / gridDim.x); i < t_end; ++i) {
        const int mb = i / n_blocks, nbk = i % n_blocks;
        if (a.x_resident && (b != x_b || mb != x_mb)) {
          mbar_wait(x_empty, xph ^ 1u);                    // the Y warps are done with the previous tile
          if (elect_one()) {
            mbar_arrive_expect_tx(x_full, a.num_kx * kATileBytes);
            for (int kx = 0; kx < a.num_kx; ++kx)
              tma_load_2d(smem_x + kx * kATileBytes, &tmX, x_full, kx * 64, c0 + mb * 128, kEvictLast);
          }
          __syncwarp();
          xph ^= 1u;
          x_b = b;
          x_mb = mb;
        }
        for (int kx = 0; kx < a.num_kx; ++kx) {
          mbar_wait(&y_empty[stage], phase ^ 1u);
          if (elect_one()) {
            mbar_arrive_expect_tx(&y_full[stage], y_stage_bytes);
            uint8_t* st = smem_y + stage * y_stage_bytes;
            if (!a.x_resident) tma_load_2d(st + kWBytes, &tmX, &y_full[stage], kx * 64, c0 + mb * 128, kEvictLast);
            tma_load_2d(st, &tmW, &y_full[stage], kx * 64, nbk * kYBlockN, kEvictLast);
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
    const uint32_t stg = smem_u32(y_staging) + static_cast<uint32_t>(quarter * 32 * 128);
    const int fr = lane >> 2, fc = (lane & 3) * 2;
    Acc<kYBlockN> acc;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t xph = 0;
    int x_b = -1, x_mb = -1;
    for (int b = 0; b < a.n_batches; ++b) {
      const int c0 = a.c_begin + b * a.nb;
      const int rows = min(a.nb, a.c_end - c0);
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
      // a contiguous range of the batch's tiles per CTA (rotated by batch), so that the resident Xc tile changes at
      // most once per n_blocks tiles
      const int64_t rot = (blockIdx.x + 7u * b) % gridDim.x;
      const int t_end = static_cast<int>(tiles * (rot + 1) / gridDim.x);
      for (int i = static_cast<int>(tiles * rot / gridDim.x); i < t_end; ++i) {
        const int mb = i / n_blocks, nbk = i % n_blocks;
        if (a.x_resident && (b != x_b || mb != x_mb)) {
          if (x_b >= 0) {                                  // every MMA on the previous tile has retired (wait<0> below)
            __syncwarp();
            if (lane == 0) mbar_arrive(x_empty);
          }
          mbar_wait(x_full, xph);
          xph ^= 1u;
          x_b = b;
          x_mb = mb;
        }
        for (int kx = 0; kx < a.num_kx; ++kx) {
          mbar_wait(&y_full[stage], phase);
          uint8_t* st = smem_y + stage * y_stage_bytes;
          const uint8_t* xt = a.x_resident ? smem_x + kx * kATileBytes : st + kWBytes;
          mma_block<kYBlockN, FMT>(acc, smem_desc_sw128(smem_u32(xt)), smem_desc_sw128(smem_u32(st)), 512, 2, 4, kx != 0);
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&y_empty[stage]);
          if (++stage == kYStages) { stage = 0; phase ^= 1u; }
        }
        // epilogue: the warp converts its 32 rows x 64 columns to 16 bits into its staging tile (128-byte rows, 16-byte
        // chunks XOR-swizzled by row: conflict-free both ways), then stores whole 128-byte row segments, 8 lanes per
        // row and 4 rows per instruction (storing lane = row splits every 128-byte line into eight 16-byte writes).
        // Column n = o * Kp + k of the source's matrix; with split rows of 2 * Kp ([hi | lo] per o): n + o * Kp, and
        // the lo half (part 1) another Kp further.
        const int n0 = nbk * kYBlockN;
        const int ncol = n0 + (a.split_nk > 0 ? (n0 / a.Kp) * a.Kp : 0);
        const int n_parts = (FMT == 0 && a.split_nk > 0) ? 2 : 1;
        if (FMT == 0 && a.split_nk > 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < kYBlockN / 2; ++k) acc.d[h][k] *= ysc;
        }
#pragma unroll 1
        for (int part = 0; part < n_parts; ++part) {
          __syncwarp();                                    // the previous part's reads of the staging tile are done
#pragma unroll
          for (int j = 0; j < kYBlockN / 8; ++j) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {                  // m64 half q / 2, rows fr (+ 8 for odd q) of the warp
              const int R = 16 * (q >> 1) + fr + 8 * (q & 1);
              float f0 = acc.d[q >> 1][4 * j + 2 * (q & 1)], f1 = acc.d[q >> 1][4 * j + 2 * (q & 1) + 1];
              uint32_t p;
              if (FMT == 0) {
                __half2 hh = __floats2half2_rn(f0, f1);
                if (part == 1) {
                  const float2 hf = __half22float2(hh);
                  hh = __floats2half2_rn(f0 - hf.x, f1 - hf.y);
                }
                p = *reinterpret_cast<uint32_t*>(&hh);
              } else {
                __nv_bfloat162 hh = __floats2bfloat162_rn(f0, f1);
                p = *reinterpret_cast<uint32_t*>(&hh);
              }
              const uint32_t addr = stg + static_cast<uint32_t>(R * 128 + ((j ^ (R & 7)) << 4) + fc * 2);
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(p) : "memory");
            }
          }
          __syncwarp();
          uint16_t* ytile = ybase + ncol + part * a.Kp;
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int R = 4 * it + (lane >> 3), ch = lane & 7;
            const int row = mb * 128 + acc_row(quarter, R);
            uint32_t v[4];
            const uint32_t addr = stg + static_cast<uint32_t>(R * 128 + ((ch ^ (R & 7)) << 4));
            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr)
                         : "memory");
            if (row < rows) {
              uint16_t* dst = ytile + static_cast<int64_t>(row) * a.NY * ymul + ch * 8;
              asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(dst), "r"(v[0]), "r"(v[1]),
                           "r"(v[2]), "r"(v[3]), "l"(a.y_store_policy)
                           : "memory");
            }
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

template <int FMT, int kYBlockN, int NC>
__global__ void __launch_bounds__(kThreads, 1)
k_apply_tc(const __grid_constant__ HMaps tmH, const __grid_constant__ CUtensorMap tmY,
           const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, ApplyArgs a) {
  apply_tc_body<FMT, kYBlockN, NC, false>(tmH, tmY, tmX, tmW, a);
}

template <int FMT, int kYBlockN, int NC>
__global__ void __launch_bounds__(kThreads, 1)
k_apply_tc_max(const __grid_constant__ HMaps tmH, const __grid_constant__ CUtensorMap tmY,
               const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, ApplyArgs a) {
  apply_tc_body<FMT, kYBlockN, NC, true>(tmH, tmY, tmX, tmW, a);
}

template <int FMT, int YBN, int NC, bool MAX>
struct ApplyKernel {
  static constexpr auto fn = MAX ? k_apply_tc_max<FMT, YBN, NC> : k_apply_tc<FMT, YBN, NC>;
};

struct ApplyShape {
  int nb_slots, passes, a_stages, x_resident, y_bytes, smem_bytes;
};

// num_kx: 64-column boxes of the Y GEMM's K (the Xc tile of a 128-source m-block is num_kx * 16 KiB)
// staging: the scatter staging is needed whatever scatter_mode says (aggr = max stages its key rows there)
// forced: the only pass count to consider (0 = any)
static bool apply_shape_passes(int cout, int Kp, int ybn, int num_kx, ApplyShape* as, bool staging, int forced) {
  const int w_bytes = ybn * 64 * 2;
  if (cout % 16 != 0 || cout < 16 || cout > 64 || Kp % 64 != 0) return false;
  const int num_kc = Kp / 64;
  const int b_stride = (cout * 128 + 1023) & ~1023;
  const int bar_bytes = 1024 + kYStagingBytes + (options().scatter_mode == 1 || staging ? kScatterBytes : 0);
  // fewest passes that leave >= 7 A stages (the h stream needs the bytes in flight), else >= 5, else >= 3; at each
  // level a resident Xc tile (loaded once per m-block instead of once per n-block) first, where it fits
  for (int min_stages = 7; min_stages >= 3; min_stages -= 2) {
    for (int xres = num_kx * kATileBytes <= kMaxXBytes ? 1 : 0; xres >= 0; --xres) {
      const int y_bytes = xres ? num_kx * kATileBytes + kYStages * w_bytes : kYStages * (kATileBytes + w_bytes);
      const int budget = 227 * 1024 - bar_bytes - y_bytes;
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
          as->x_resident = xres;
          as->y_bytes = y_bytes;
          as->smem_bytes = nb * b_stride + stages * kATileBytes + y_bytes + bar_bytes;
          return true;
        }
      }
    }
  }
  return false;
}

// The apply_passes option forces the pass count where that count has a shape.  A count that leaves none (fewer than
// 4 B slots per pass, or too few A stages) is ignored like one that does not divide Kp / 64: the option never makes a
// shape unsupported, so it cannot turn the fused kernel into the per-batch one or refuse precision f16x2.
bool apply_shape(int cout, int Kp, int ybn, int num_kx, ApplyShape* as, bool staging = false) {
  const int forced = options().apply_passes;
  if (forced > 0 && apply_shape_passes(cout, Kp, ybn, num_kx, as, staging, forced)) return true;
  return apply_shape_passes(cout, Kp, ybn, num_kx, as, staging, 0);
}

}  // namespace

// N tile of the Y pipeline: 64 columns = 64 accumulator registers per thread of the Y warpgroup, which shares the SM's
// register file with the two conv warpgroups (a 128-column tile spills and serialises its wgmma on sm_90)
constexpr int kYBN = 64;

static int eff_kp(const Weights* W) { return W->split ? 3 * W->Kp : W->Kp; }
static int y_num_kx(const Weights* W) { return (W->split ? 3 : 1) * W->cin_p / 64; }

bool apply_fused_supported(const Weights* W) {
  if (W->prec != PREC_F16 && W->prec != PREC_BF16 && W->prec != PREC_F16X2) return false;
  if ((W->cout * W->Kp) % 128 != 0) return false;
  ApplyShape as;
  return apply_shape(W->cout, eff_kp(W), kYBN, y_num_kx(W), &as);
}

namespace {
template <int FMT, int YBN, int NC, bool MAX>
int launch_variant(int grid, int smem_bytes, bool coop, cudaStream_t st, const HMaps& tmH, const CUtensorMap& tmY,
                   const CUtensorMap& tmX, const CUtensorMap& tmW, const ApplyArgs& a) {
  static bool attr_set = false;
  static int blocks_per_sm = -1;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(ApplyKernel<FMT, YBN, NC, MAX>::fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  if (blocks_per_sm < 0)
    NNC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, ApplyKernel<FMT, YBN, NC, MAX>::fn, kThreads,
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
  cudaError_t e = cudaLaunchKernelEx(&cfg, ApplyKernel<FMT, YBN, NC, MAX>::fn, tmH, tmY, tmX, tmW, a);
  if (e == cudaErrorCooperativeLaunchTooLarge) {
    cudaGetLastError();
    return kApplyCannotCoSchedule;   // handled by the application driver (api.cu): per-batch kernels instead
  }
  NNC_CHECK_CUDA(e);
  return NNCONV_OK;
}
}  // namespace

int launch_apply_tc(int prec, const Plan* P, const Weights* W, const void* h, const void* Xc, void* Yring, int nb,
                    int ring, const float* cvec, const float* xs, int aggr_mean, float* out, int* flags,
                    int flags_stride, cudaStream_t st, const UnitRange& R, unsigned long long* max_keys) {
  int s = tc_init();
  if (s != NNCONV_OK) return s;
  const Options& opt = options();
  const int bf = prec == PREC_BF16;
  const int split = W->split ? 1 : 0;
  const int ybn = kYBN;
  ApplyShape as;
  NNC_REQUIRE(apply_shape(W->cout, eff_kp(W), ybn, y_num_kx(W), &as, max_keys != nullptr), NNCONV_ERR_UNSUPPORTED,
              "apply_tc: unsupported shape");
  if (opt.apply_stages >= 2 && opt.apply_stages < as.a_stages) as.a_stages = opt.apply_stages;
  const int64_t e_pad = R.h_rows;
  const int NY = W->cout * W->Kp;
  const int kmul = split ? 2 : 1;      // [hi | lo] activations / Y rows
  const int xmul = split ? 3 : 1;      // [hi | hi | lo] x [hi | lo | hi] operands of the Y GEMM
  const int n_batches = ceil_div(R.c_end - R.c_begin, nb);
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
  a.u_begin = R.u_begin; a.u_end = R.u_end; a.c_begin = R.c_begin; a.c_end = R.c_end;
  a.e_base = static_cast<int>(R.e_base);
  a.nb = nb; a.n_batches = n_batches; a.ring = ring;
  a.nb_slots = as.nb_slots; a.passes = as.passes; a.a_stages = as.a_stages;
  a.x_resident = as.x_resident; a.y_bytes = as.y_bytes;
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
  a.keys = max_keys;
  a.perm = P->perm;
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
    if (max_keys != nullptr)
      return launch_variant<decltype(fmt)::value, kYBN, decltype(nc)::value, true>(grid, as.smem_bytes, coop, st, tmH, tmY,
                                                                                  tmX, tmW, a);
    return launch_variant<decltype(fmt)::value, kYBN, decltype(nc)::value, false>(grid, as.smem_bytes, coop, st,
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
