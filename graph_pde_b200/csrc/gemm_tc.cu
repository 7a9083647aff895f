// wgmma GEMM for the dense stages of the NNConv path (sm_90a):
//     C[M, N] (fp16/bf16) = act( A[M, K] * B[N, K]^T + bias )          fp32 accumulation in registers
// used for (a) the hidden layers of the edge MLP (graph-neural-operator/utilities.py:223-227,
// Linear + ReLU) over a chunk of edges and (b) the per-source matrices
// Y[c, (o,k)] = sum_i x[c, i] * W_L[i*out + o, k]  (the last Linear reassociated, nn_conv.py:274-275).
//
// Structure: persistent CTAs (grid = #SMs), 12 warps: warps 0..7 = two consumer warpgroups, each owning half of
// the BLOCK_N columns of the tile (wgmma into registers, then the epilogue: bias/ReLU -> 16-bit on the accumulator
// fragments -> stmatrix into a per-warp swizzled smem piece -> TMA store; direct 32-byte stores of the staged rows for
// pipelined / small launches), warps 8..11 = the TMA
// producer warpgroup (warp 8 loops, one elected lane issues).  The producer gives its registers to the consumers
// (setmaxnreg), so a [128 x 128] fp32 accumulator per warpgroup and the epilogue fit without spilling.  The SMALL
// configuration keeps a single producer warp (9 warps) so that two CTAs share an SM.  Operands are K-major
// 128B-swizzled tiles [128 x 64] / [BLOCK_N x 64] staged by TMA in a ring of kStages, so the producer runs ahead
// into the next tile while the warpgroups run the epilogue of this one.
#include "act.cuh"
#include "kernels.h"
#include "options.h"
#include "tc05.cuh"
#include "tmap.h"

namespace nnc {

namespace {

using namespace tc05;

struct GemmTcArgs {
  int M, N, K;
  int a_row0;          // first row of A inside the tensor map
  const float* bias;   // [N] or nullptr
  int relu;
  void* C;
  int64_t ldc;         // elements
  // chunk-major output (the layout the contraction kernel streams): element (row, col) lives at
  // ((col / 64) * chunk_rows_pad + c_row0 + row) * 64 + col % 64, i.e. one contiguous [rows, 64] panel per
  // 64-column K chunk, so a TMA box of consecutive rows is ONE contiguous block of DRAM.  0 = row-major.
  int64_t chunk_rows_pad;
  int64_t c_row0;
  // optional cross-kernel pipelining (see tc05.cuh): wait for *wait_ok before touching C, raise *done_ok
  const int* wait_ok;
  int* done_cnt;
  int* done_ok;
  // 1: every epilogue warp stages its [32 rows x 32 cols] piece in its own double-buffered 2 KB of shared
  // memory (64-byte swizzle) and one lane writes it with TMA (tmC, two [16 x 32] panels): no global stores on the
  // LSU data pipe, no block-level barrier, and the store of piece i drains while piece i+1 is converted.
  int tma_store;
  int bias_v4;         // bias is 16-byte aligned: vector loads
  // PREC_F16X2 (see plan.h): a_split_nk = K/3/64 > 0 -> A holds [hi | lo] (2K/3 columns) and K block kb reads
  // A chunk (kb < nk ? kb : kb - nk), i.e. [hi | hi | lo] against B = [hi | lo | hi]; c_split -> the fp32 result is
  // written as the pair hi = fp16(v) at column c and lo = fp16(v - hi) at column c + N (row-major, ldc = 2N) or at
  // chunk (c / 64) + N / 64 (chunk-major).
  int a_split_nk;
  int c_split;
  const float* acc_scale;     // optional device scalar multiplied into the fp32 accumulator before bias (exact power of two)
  unsigned long long b_policy;   // L2 eviction hint of the B (weight) tiles
  int64_t a_chunk_rows_pad;   // > 0: A is chunk-major [K/64][a_chunk_rows_pad][64] (the edge-feature layout): K block kb of
                              // row r is the box at (0, kb * a_chunk_rows_pad + r) of the [K/64 * rows_pad, 64] view
  int* overflow;       // counts [32 x 32] warp pieces holding a value beyond the fp16 range (fp16 outputs only), or nullptr
  // backward epilogues: mask != nullptr -> C[r, c] = mask16[r * mask_ld + c] > 0 ? acc : 0 (ReLU derivative taken
  // from the stored 16-bit activation); out_f32 -> C is fp32 [M, ldc], plain stores, no conversion.
  const uint16_t* mask;
  int64_t mask_ld;
  int out_f32;
  TraceBuf trace;
  unsigned int trace_seq;
  ActParams act_p;     // parameter block of the activation epi_act(EPI)
};

// EPI selects the epilogue at COMPILE time (runtime flags inside the 32-column inner loop cut it into dozens of
// tiny basic blocks, and the K = 64 first-layer GEMM is epilogue bound):
//   EPI_PLAIN bias / ReLU / 16-bit store     EPI_SPLIT the same, written as (hi, lo) fp16 pairs (PREC_F16X2)
//   EPI_MASK  ReLU-derivative mask from a stored activation (backward)     EPI_F32 fp32 output, plain stores
//   EPI_NOCHECK = EPI_PLAIN without the fp16 range tracking (bf16 outputs, option overflow_check = 0, test hooks)
//   EPI_MASK_SPLIT = EPI_MASK with acc_scale, written as (hi, lo) pairs (PREC_F16X2 backward; the mask is the hi half)
// The hidden activation (act.cuh) rides in the bits above: EPI = base | ACT << 3.  ReLU is ACT 0, so the ReLU
// instantiations keep their names and code; for the other activations the forward epilogues apply act_fwd<ACT> where
// ReLU applies the max, and the mask epilogues multiply by act_grad<ACT>(y) of the stored activation y (the split
// form reads y = hi + lo, the lo half at column c + N of the mask row).  For CLAMP the forward epilogues also apply the
// store rule of act.cuh (act_store16, act_split_lo), so that no interior entry is stored on a bound's image.
// The forward epilogues (PLAIN, NOCHECK, SPLIT) work on the accumulator fragments and write the 16-bit staging with
// stmatrix; the backward ones first transpose the fragments through a per-warp fp32 scratch (acc_rows: lane = row),
// because their mask is read and their fp32 output written a row at a time.
enum { EPI_PLAIN = 0, EPI_SPLIT = 1, EPI_MASK = 2, EPI_F32 = 3, EPI_NOCHECK = 4, EPI_MASK_SPLIT = 5 };
constexpr int epi_base(int epi) { return epi & 7; }
constexpr int epi_act(int epi) { return epi >> 3; }
constexpr int epi_with_act(int epi, int act) { return epi | act << 3; }
constexpr bool epi_uses_rows(int epi) {
  return epi_base(epi) == EPI_MASK || epi_base(epi) == EPI_MASK_SPLIT || epi_base(epi) == EPI_F32;
}

// SMALL = 1: a 2-stage, BLOCK_N = 128, 288-thread footprint (~100 KB smem) that can share an SM with a
// contraction CTA or a second GEMM CTA -- used for the per-source Y GEMM, which is store bound and runs
// concurrently with the contraction of the previous batch.
template <int BLOCK_N, int SMALL = 0, int EPI = EPI_PLAIN>
struct GemmCfg {
  static constexpr int kThreads = SMALL ? 288 : 384;
  // setmaxnreg budgets of the 384-thread CTA: (40 + 2 * 232) * 128 = 64512 <= 65536 registers, the launch-time
  // allocation of 168 per thread (65536 / 384 rounded down to a multiple of 8)
  static constexpr uint32_t kProducerRegs = 40;
  static constexpr uint32_t kConsumerRegs = 232;
  static constexpr int kBlockM = 128;
  static constexpr int kBlockK = 64;
  static constexpr int kABytes = kBlockM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // output staging of the epilogue: 8 warps x 2 buffers x [32 x 32] 16-bit pieces
  static constexpr int kStoreBytes = 8 * 2 * 2048;
  static constexpr int kScratchBytes = epi_uses_rows(EPI) ? 8 * acc_scratch_bytes<32>() : 0;   // per-warp transposes
  static constexpr int kFixedBytes = kStoreBytes + kScratchBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  // as many stages as the 227 KB an SM gives one CTA hold (less 256 B for the static trace words), at most 8;
  // 256-column tiles: 4 x 48 KB for the forward epilogues, 3 for the ones with the fp32 scratch
  static constexpr int kFitStages = (232448 - 256 - kFixedBytes) / kStageBytes;
  static constexpr int kStages = SMALL ? 2 : (kFitStages > 8 ? 8 : kFitStages);
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixedBytes;
  static_assert(SMALL || kStages >= 3, "gemm_tc: ring too shallow");
};

template <int BLOCK_N, int FMT, int SMALL, int EPI>
__global__ void __launch_bounds__(GemmCfg<BLOCK_N, SMALL, EPI>::kThreads, SMALL ? 2 : 1)
k_gemm_tc(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
          const __grid_constant__ CUtensorMap tmC, GemmTcArgs a) {
  using Cfg = GemmCfg<BLOCK_N, SMALL, EPI>;
  constexpr int kEpi = epi_base(EPI), kAct = epi_act(EPI);
  constexpr bool kSplitOut = kEpi == EPI_SPLIT || kEpi == EPI_MASK_SPLIT;
  constexpr bool kMask = kEpi == EPI_MASK || kEpi == EPI_MASK_SPLIT;
  constexpr bool kRows = epi_uses_rows(EPI);
  constexpr bool kRangeCheck = FMT == 0 && (kEpi == EPI_PLAIN || kEpi == EPI_SPLIT);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  uint8_t* smem_c = smem + Cfg::kStages * Cfg::kStageBytes;     // 1024-aligned (stage sizes are multiples of 8 KB)
  float* scratch = reinterpret_cast<float*>(smem_c + Cfg::kStoreBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_c + Cfg::kStoreBytes + Cfg::kScratchBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::kStages;

  // shfl: the warp index is warp-uniform for the compiler (role branches converge, operands stay in uniform registers)
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x / 32), 0), lane = threadIdx.x % 32;
  const int m_blocks = ceil_div(a.M, Cfg::kBlockM);
  const int n_blocks = ceil_div(a.N, BLOCK_N);
  const int num_tiles = m_blocks * n_blocks;
  const int num_kb = a.K / Cfg::kBlockK;

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (a.tma_store) prefetch_tmap(&tmC);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  // trace times of thread 0 (which writes the record), kept in shared memory rather than in registers that would
  // stay live through the mainloop and the epilogue
  __shared__ unsigned long long trace_t[2];
  if (threadIdx.x == 0 && a.trace.rec) trace_t[0] = gtime();
  pdl_launch_dependents();
  if (a.wait_ok != nullptr && threadIdx.x == 0) flag_wait(a.wait_ok);
  if (threadIdx.x == 0 && a.trace.rec) trace_t[1] = gtime();
  __syncthreads();

  if (warp >= 8) {
    // -------------------------------------------------------------- TMA producer (warp 8 loops, elected lane issues)
    if (!SMALL) warpgroup_reg_dealloc<Cfg::kProducerRegs>();
    if (warp == 8) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int mb = t / n_blocks, nb = t % n_blocks;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u);
          if (elect_one()) {
            mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
            const int ka = (a.a_split_nk > 0 && kb >= a.a_split_nk) ? kb - a.a_split_nk : kb;
            if (a.a_chunk_rows_pad > 0)
              tma_load_2d(smem_a + stage * Cfg::kABytes, &tmA, &full[stage], 0,
                          static_cast<int>(ka * a.a_chunk_rows_pad) + a.a_row0 + mb * Cfg::kBlockM, kEvictNormal);
            else
              tma_load_2d(smem_a + stage * Cfg::kABytes, &tmA, &full[stage], ka * Cfg::kBlockK,
                          a.a_row0 + mb * Cfg::kBlockM, kEvictNormal);
            tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmB, &full[stage], kb * Cfg::kBlockK, nb * BLOCK_N,
                        a.b_policy);
          }
          __syncwarp();
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroups (warps 0..7)
    // warpgroup `half` computes columns [half * BLOCK_N / 2, (half + 1) * BLOCK_N / 2) of the tile, then stores them;
    // warp `quarter` of it owns tile rows acc_row(quarter, lane) in the epilogue
    if (!SMALL) warpgroup_reg_alloc<Cfg::kConsumerRegs>();
    const int quarter = warp % 4;
    const int half = warp / 4;
    constexpr int kChunks = BLOCK_N / 64;          // 32-column chunks per half
    float* wb = kRows ? scratch + warp * (acc_scratch_bytes<32>() / 4) : nullptr;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t piece = 0;   // pieces staged by this warp (selects the staging buffer)
    Acc<BLOCK_N / 2> acc;
    const bool use_tma = a.tma_store != 0;
    // this warp's staging: 2 buffers of 32 rows x 64 B, row i = tile row acc_row(quarter, i); 16-byte unit u of row i
    // sits at (u ^ ((i >> 1) & 3)) (SWIZZLE_64B of tmC) -- conflict-free for the 8-lane phases of whole-row v4 shared
    // accesses and for the 8 rows of one stmatrix matrix alike
    const uint32_t stage0 = smem_u32(smem_c) + warp * 4096;
    const uint32_t sw = static_cast<uint32_t>((lane >> 1) & 3);
    // stmatrix x4: lane l gives the address of row (l & 7) of matrix l >> 3; matrix m covers staging rows
    // 8 (m & 1) .. + 7 (of a 16-row half) and the (m >> 1)-th of a pair of 16-byte units
    const uint32_t sm_row = 8 * ((lane >> 3) & 1) + (lane & 7);
    const uint32_t sm_sw = (sm_row >> 1) & 3, sm_u = static_cast<uint32_t>(lane >> 4);
    // accumulator fragment of the lane: rows (lane >> 2) and + 8 of the warp's 16-row runs, columns fc, fc + 1 of every 8
    const int fr = lane >> 2, fc = 2 * (lane & 3);
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int mb = t / n_blocks, nb = t % n_blocks;
      int prev = stage;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = smem_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes));
        const uint64_t bdesc = smem_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes + half * (BLOCK_N / 2) * 128));
        mma_block<BLOCK_N / 2, FMT>(acc, adesc, bdesc, 512, 2, Cfg::kBlockK / 16, kb != 0);
        // keep this block's MMAs in flight while the next stage is awaited: wait for the PREVIOUS block only and
        // free its slot (this warp's MMAs have read it)
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0 && kb > 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      const int row = mb * Cfg::kBlockM + acc_row(quarter, lane);
      const bool row_ok = row < a.M;
      const float accs = (kSplitOut && a.acc_scale != nullptr) ? __ldg(a.acc_scale) : 1.f;
      const bool issuer = elect_one();    // same lane every time: bulk groups are per thread
      // a piece's staging buffer, once the TMA store issued two pieces ago has finished reading it
      auto begin_piece = [&]() {
        const uint32_t buf = stage0 + (piece & 1) * 2048;
        if (use_tma && issuer) bulk_wait_read1();
        __syncwarp();
        return buf;
      };
      // the staged [32 rows x 32 cols] piece at column colx of the (possibly doubled) output: two [16 x 32] TMA panels
      // (staging rows 0..15 and 16..31 are two 16-row runs of the tile), or every lane writes its row directly
      auto end_piece = [&](uint32_t buf, int colx) {
        if (use_tma) {
          fence_proxy_async_smem();
          __syncwarp();
          if (issuer) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int r0 = mb * Cfg::kBlockM + 64 * hh + 16 * quarter;
              if (a.chunk_rows_pad > 0)
                tma_store_2d(&tmC, buf + hh * 1024, colx & 63,
                             static_cast<int>((colx >> 6) * a.chunk_rows_pad + a.c_row0 + r0));
              else
                tma_store_2d(&tmC, buf + hh * 1024, colx, r0);
            }
            bulk_commit();
          }
        } else {
          __syncwarp();
          if (row_ok) {
            uint32_t pk[16];
#pragma unroll
            for (int u = 0; u < 4; ++u) ld_shared_v4(buf + lane * 64 + ((static_cast<uint32_t>(u) ^ sw) << 4), pk + 4 * u);
            uint16_t* dst = a.chunk_rows_pad > 0
                                ? reinterpret_cast<uint16_t*>(a.C) +
                                      (static_cast<int64_t>(colx >> 6) * a.chunk_rows_pad + a.c_row0 + row) * 64 + (colx & 63)
                                : reinterpret_cast<uint16_t*>(a.C) + static_cast<int64_t>(row) * a.ldc + colx;
            st_global_32b(dst, pk);            // 2 x 32 B: full sectors (16 B stores were half-used
            st_global_32b(dst + 16, pk + 8);   // sectors)
          }
        }
        ++piece;
      };
#pragma unroll
      for (int cc = 0; cc < kChunks; ++cc) {
        const int col0 = nb * BLOCK_N + half * (BLOCK_N / 2) + cc * 32;
        if (col0 >= a.N) continue;
        if constexpr (!kRows) {
          // ---- forward epilogues, on the fragments: value (h, g, j) of the lane = tile row 64 h + 16 quarter + 8 g + fr,
          // columns col0 + 8 j + fc and + 1 (accumulator registers 4 (4 cc + j) + 2 g and + 1 of half h)
          float2 bj[4];
          if (a.bias) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              bj[j] = a.bias_v4 ? __ldg(reinterpret_cast<const float2*>(a.bias + col0 + 8 * j + fc))
                                : make_float2(__ldg(a.bias + col0 + 8 * j + fc), __ldg(a.bias + col0 + 8 * j + fc + 1));
          }
          uint32_t hi[2][2][4], lo[2][2][4];
          float vmax[2] = {0.f, 0.f};   // two independent max chains
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int g = 0; g < 2; ++g) {
              const bool ok = mb * Cfg::kBlockM + 64 * h + 16 * quarter + 8 * g + fr < a.M;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                float f0 = acc.d[h][4 * (4 * cc + j) + 2 * g], f1 = acc.d[h][4 * (4 * cc + j) + 2 * g + 1];
                if (kSplitOut) { f0 *= accs; f1 *= accs; }
                if (a.bias) { f0 += bj[j].x; f1 += bj[j].y; }
                if (kAct == ACT_RELU) {
                  if (a.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
                  if (kRangeCheck && ok) vmax[j & 1] = fmaxf(vmax[j & 1], fmaxf(fabsf(f0), fabsf(f1)));
                } else {
                  float r0 = fabsf(f0), r1 = fabsf(f1);
                  if (a.relu) {
                    const float y0 = act_fwd<kAct>(f0, a.act_p);
                    const float y1 = act_fwd<kAct>(f1, a.act_p);
                    r0 = act_range<kAct>(f0, y0);
                    r1 = act_range<kAct>(f1, y1);
                    f0 = kSplitOut ? y0 : act_store16<kAct, FMT>(y0, a.act_p);
                    f1 = kSplitOut ? y1 : act_store16<kAct, FMT>(y1, a.act_p);
                  }
                  if (kRangeCheck && ok) vmax[j & 1] = fmaxf(vmax[j & 1], fmaxf(r0, r1));
                }
                if (FMT == 0) {
                  const __half2 hv = __floats2half2_rn(f0, f1);
                  hi[h][g][j] = *reinterpret_cast<const uint32_t*>(&hv);
                  if (kSplitOut) {
                    const float2 hf = __half22float2(hv);
                    __half2 lv = __floats2half2_rn(f0 - hf.x, f1 - hf.y);
                    if (kAct == ACT_CLAMP && a.relu) {
                      lv.x = act_split_lo<kAct>(f0, hv.x, lv.x, a.act_p);
                      lv.y = act_split_lo<kAct>(f1, hv.y, lv.y, a.act_p);
                    }
                    lo[h][g][j] = *reinterpret_cast<const uint32_t*>(&lv);
                  }
                } else {
                  const __nv_bfloat162 hv = __floats2bfloat162_rn(f0, f1);
                  hi[h][g][j] = *reinterpret_cast<const uint32_t*>(&hv);
                }
              }
            }
          }
          // one count per warp and piece holding a value beyond the fp16 range in a row inside M
          if (kRangeCheck && a.overflow != nullptr) {
            const bool bad = __any_sync(0xffffffffu, !(fmaxf(vmax[0], vmax[1]) <= 65504.f));
            if (bad && issuer) atomicAdd(a.overflow, 1);
          }
          auto stage_frags = [&](const uint32_t (&pk)[2][2][4], int colx) {
            const uint32_t buf = begin_piece();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
              for (int jp = 0; jp < 2; ++jp)
                stmatrix_x4(buf + (16 * h + sm_row) * 64 + (((2 * jp + sm_u) ^ sm_sw) << 4), pk[h][0][2 * jp],
                            pk[h][1][2 * jp], pk[h][0][2 * jp + 1], pk[h][1][2 * jp + 1]);
            }
            end_piece(buf, colx);
          };
          stage_frags(hi, col0);
          if (FMT == 0 && kSplitOut) stage_frags(lo, col0 + a.N);
        } else {
          // ---- backward epilogues, a row per lane
          uint32_t v[32];
          acc_rows<BLOCK_N / 2, 32>(acc, cc * 32, wb, v);
          uint32_t packed[16], packed_lo[kSplitOut ? 16 : 1];
          // EPI_MASK: the row's 32 stored activations (64 B), one 16-byte load per 8 columns
          const uint4* mp = reinterpret_cast<const uint4*>(a.mask + static_cast<int64_t>(row) * a.mask_ld + col0);
          uint4 mkw = make_uint4(0u, 0u, 0u, 0u);
          uint4 mkl = make_uint4(0u, 0u, 0u, 0u);   // split form, other activations: the lo half of the same columns
#pragma unroll
          for (int j4 = 0; j4 < 8; ++j4) {
            float f[4] = {__uint_as_float(v[4 * j4]), __uint_as_float(v[4 * j4 + 1]),
                          __uint_as_float(v[4 * j4 + 2]), __uint_as_float(v[4 * j4 + 3])};
            if (kSplitOut) {
#pragma unroll
              for (int q = 0; q < 4; ++q) f[q] *= accs;
            }
            if (a.bias) {
              if (a.bias_v4) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.bias + col0) + j4);
                f[0] += b4.x; f[1] += b4.y; f[2] += b4.z; f[3] += b4.w;
              } else {
#pragma unroll
                for (int q = 0; q < 4; ++q) f[q] += __ldg(a.bias + col0 + 4 * j4 + q);
              }
            }
            if (a.relu) {
#pragma unroll
              for (int q = 0; q < 4; ++q) f[q] = act_fwd<kAct>(f[q], a.act_p);
            }
            if (kMask && kAct != ACT_RELU) {
              // f'(y) from the stored activation: y = hi (+ lo at column c + N for the split form)
              if (row_ok) {
                if (j4 % 2 == 0) {
                  mkw = __ldg(mp + j4 / 2);
                  if (kSplitOut) mkl = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(mp) + a.N) + j4 / 2);
                }
                const uint32_t mw[2] = {j4 % 2 ? mkw.z : mkw.x, j4 % 2 ? mkw.w : mkw.y};
                const uint32_t lw[2] = {j4 % 2 ? mkl.z : mkl.x, j4 % 2 ? mkl.w : mkl.y};
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                  float2 y = unpack2<FMT>(mw[q]);
                  if (kSplitOut) {
                    const float2 yl = unpack2<FMT>(lw[q]);
                    y.x += yl.x;
                    y.y += yl.y;
                  }
                  f[2 * q] *= act_grad<kAct>(y.x, a.act_p);
                  f[2 * q + 1] *= act_grad<kAct>(y.y, a.act_p);
                }
              }
            } else if (kMask) {
              if (row_ok) {
                if (j4 % 2 == 0) mkw = __ldg(mp + j4 / 2);
                const uint32_t mx = j4 % 2 ? mkw.z : mkw.x, my = j4 % 2 ? mkw.w : mkw.y;
                if ((mx & 0x7FFFu) == 0u) f[0] = 0.f;
                if ((mx & 0x7FFF0000u) == 0u) f[1] = 0.f;
                if ((my & 0x7FFFu) == 0u) f[2] = 0.f;
                if ((my & 0x7FFF0000u) == 0u) f[3] = 0.f;
              }
            }
            if (kEpi == EPI_F32) {
              if (row_ok)
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(a.C) + static_cast<int64_t>(row) * a.ldc + col0 + 4 * j4) =
                    make_float4(f[0], f[1], f[2], f[3]);
            } else {
#pragma unroll
              for (int q = 0; q < 2; ++q) {
                if (FMT == 0) {
                  __half2 h = __floats2half2_rn(f[2 * q], f[2 * q + 1]);
                  packed[2 * j4 + q] = *reinterpret_cast<uint32_t*>(&h);
                  if (kSplitOut) {
                    const float2 hf = __half22float2(h);
                    __half2 l = __floats2half2_rn(f[2 * q] - hf.x, f[2 * q + 1] - hf.y);
                    packed_lo[2 * j4 + q] = *reinterpret_cast<uint32_t*>(&l);
                  }
                } else {
                  __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
                  packed[2 * j4 + q] = *reinterpret_cast<uint32_t*>(&h);
                }
              }
            }
          }
          auto stage_row = [&](const uint32_t* pk, int colx) {
            const uint32_t buf = begin_piece();
#pragma unroll
            for (int u = 0; u < 4; ++u)
              st_shared_v4(buf + lane * 64 + ((static_cast<uint32_t>(u) ^ sw) << 4), pk[4 * u], pk[4 * u + 1],
                           pk[4 * u + 2], pk[4 * u + 3]);
            end_piece(buf, colx);
          };
          if (kEpi != EPI_F32) {
            stage_row(packed, col0);
            if (FMT == 0 && kSplitOut) stage_row(packed_lo, col0 + a.N);
          }
        }
      }
    }
  }
  if (a.tma_store && warp < 8 && elect_one()) bulk_wait0();
  if (a.done_cnt != nullptr) signal_done(a.done_cnt, a.done_ok);   // includes __syncthreads
  else __syncthreads();
  if (threadIdx.x == 0) trace_write(a.trace, (100u + (a.K > 64 ? 1u : 0u)) | (a.trace_seq << 12), trace_t[0], trace_t[1], a.trace.rec ? gtime() : 0ull);
}

int g_num_sms = 0;

template <int BLOCK_N, int FMT, int SMALL, int EPI = EPI_PLAIN>
int launch_gemm_cfg(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmTcArgs& a,
                    cudaStream_t st, bool pdl) {
  using Cfg = GemmCfg<BLOCK_N, SMALL, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_gemm_tc<BLOCK_N, FMT, SMALL, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::kSmemBytes));
    attr_set = true;
  }
  const int tiles = ceil_div(a.M, 128) * ceil_div(a.N, BLOCK_N);
  const int max_ctas = SMALL ? 2 * g_num_sms : g_num_sms;
  const int grid = tiles < max_ctas ? tiles : max_ctas;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(Cfg::kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  NNC_CHECK_CUDA(cudaLaunchKernelEx(&cfg, k_gemm_tc<BLOCK_N, FMT, SMALL, EPI>, tmA, tmB, tmC, a));
  return NNCONV_OK;
}

// the launch of launch_gemm_tc's configuration with the hidden activation ACT (ACT_RELU: the original instantiations)
template <int ACT>
int dispatch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmTcArgs& a,
                  cudaStream_t st, bool pdl, int BN, int bf, bool small, int out_f32, bool mask_split, bool has_mask,
                  bool c_split) {
  // backward / split epilogues (never pipelined, never the small-footprint configuration)
#define NNC_GEMM_EPI(E)                                                                                              \
  do {                                                                                                               \
    if (BN == 256) return bf ? launch_gemm_cfg<256, 1, 0, E>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<256, 0, 0, E>(tmA, tmB, tmC, a, st, pdl); \
    if (BN == 128) return bf ? launch_gemm_cfg<128, 1, 0, E>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<128, 0, 0, E>(tmA, tmB, tmC, a, st, pdl); \
    return bf ? launch_gemm_cfg<64, 1, 0, E>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<64, 0, 0, E>(tmA, tmB, tmC, a, st, pdl); \
  } while (0)
  if constexpr (ACT == ACT_RELU) {    // fp32 output and the small footprint never apply the activation
    if (out_f32) { NNC_REQUIRE(!small && !c_split && !has_mask, NNCONV_ERR_ARG, "gemm_tc: fp32 output excludes split / mask"); NNC_GEMM_EPI(EPI_F32); }
  }
  if (mask_split) {
    NNC_REQUIRE(!small && !bf, NNCONV_ERR_ARG, "gemm_tc: split mask epilogue is fp16 only");
    if (BN == 128) return launch_gemm_cfg<128, 0, 0, epi_with_act(EPI_MASK_SPLIT, ACT)>(tmA, tmB, tmC, a, st, pdl);
    return launch_gemm_cfg<64, 0, 0, epi_with_act(EPI_MASK_SPLIT, ACT)>(tmA, tmB, tmC, a, st, pdl);
  }
  if (has_mask) { NNC_REQUIRE(!small, NNCONV_ERR_ARG, "gemm_tc: mask excludes the small-footprint configuration"); NNC_GEMM_EPI(epi_with_act(EPI_MASK, ACT)); }
  if (c_split) {
    NNC_REQUIRE(!small, NNCONV_ERR_ARG, "gemm_tc: split output excludes the small-footprint configuration");
    if (BN == 256) return launch_gemm_cfg<256, 0, 0, epi_with_act(EPI_SPLIT, ACT)>(tmA, tmB, tmC, a, st, pdl);
    if (BN == 128) return launch_gemm_cfg<128, 0, 0, epi_with_act(EPI_SPLIT, ACT)>(tmA, tmB, tmC, a, st, pdl);
    return launch_gemm_cfg<64, 0, 0, epi_with_act(EPI_SPLIT, ACT)>(tmA, tmB, tmC, a, st, pdl);
  }
#undef NNC_GEMM_EPI
  if (!bf && !small && a.overflow == nullptr) {      // fp16 output nobody wants range-checked
    if (BN == 256) return launch_gemm_cfg<256, 0, 0, epi_with_act(EPI_NOCHECK, ACT)>(tmA, tmB, tmC, a, st, pdl);
    if (BN == 128) return launch_gemm_cfg<128, 0, 0, epi_with_act(EPI_NOCHECK, ACT)>(tmA, tmB, tmC, a, st, pdl);
    return launch_gemm_cfg<64, 0, 0, epi_with_act(EPI_NOCHECK, ACT)>(tmA, tmB, tmC, a, st, pdl);
  }
  if constexpr (ACT == ACT_RELU) {
    if (small) return bf ? launch_gemm_cfg<128, 1, 1>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<128, 0, 1>(tmA, tmB, tmC, a, st, pdl);
  }
  if (BN == 256) return bf ? launch_gemm_cfg<256, 1, 0, epi_with_act(EPI_PLAIN, ACT)>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<256, 0, 0, epi_with_act(EPI_PLAIN, ACT)>(tmA, tmB, tmC, a, st, pdl);
  if (BN == 128) return bf ? launch_gemm_cfg<128, 1, 0, epi_with_act(EPI_PLAIN, ACT)>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<128, 0, 0, epi_with_act(EPI_PLAIN, ACT)>(tmA, tmB, tmC, a, st, pdl);
  return bf ? launch_gemm_cfg<64, 1, 0, epi_with_act(EPI_PLAIN, ACT)>(tmA, tmB, tmC, a, st, pdl) : launch_gemm_cfg<64, 0, 0, epi_with_act(EPI_PLAIN, ACT)>(tmA, tmB, tmC, a, st, pdl);
}

}  // namespace

int tc_init() {
  if (g_num_sms > 0) return NNCONV_OK;
  int dev = 0;
  NNC_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  NNC_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  NNC_REQUIRE(prop.major == 9 && prop.minor == 0, NNCONV_ERR_UNSUPPORTED,
              "libnnconv_b200 needs an sm_90 GPU (found sm_%d%d)", prop.major, prop.minor);
  int s = tmap_init();
  if (s != NNCONV_OK) return s;
  g_num_sms = prop.multiProcessorCount;
  return NNCONV_OK;
}

int tc_num_sms() { return g_num_sms; }

int launch_gemm_tc(int prec, const void* A_base, int64_t a_rows_total, int64_t a_row0, int M, int K, const void* B,
                   int N, const float* bias, int relu, void* C, int64_t ldc, cudaStream_t st, const PipeFlags* pf,
                   int64_t chunk_rows_pad, int64_t c_row0, int split_flags, int* overflow, const void* mask,
                   int64_t mask_ld, int out_f32, int64_t a_chunk_rows_pad, const float* acc_scale, Act act) {
  if (M <= 0 || N <= 0) return NNCONV_OK;
  int s = tc_init();
  if (s != NNCONV_OK) return s;
  NNC_REQUIRE(prec == PREC_F16 || prec == PREC_BF16 || prec == PREC_F16X2, NNCONV_ERR_ARG, "gemm_tc: 16-bit precisions only");
  const bool a_split = (split_flags & GEMM_A_SPLIT) != 0, c_split = (split_flags & GEMM_C_SPLIT) != 0;
  NNC_REQUIRE(!a_split || K % 192 == 0, NNCONV_ERR_ARG, "gemm_tc: split A needs K = 3 x a multiple of 64");
  NNC_REQUIRE(!(a_split || c_split) || prec != PREC_BF16, NNCONV_ERR_ARG, "gemm_tc: split operands are fp16 only");
  const int nmul = c_split ? 2 : 1;
  NNC_REQUIRE(K % 64 == 0 && N % 64 == 0 && K >= 64, NNCONV_ERR_ARG, "gemm_tc: K=%d N=%d must be multiples of 64", K, N);
  NNC_REQUIRE((ldc % 16 == 0 || (out_f32 && ldc % 4 == 0)) && (reinterpret_cast<uintptr_t>(C) & 31) == 0, NNCONV_ERR_ARG,
              "gemm_tc: C must be 32-byte aligned with ldc a multiple of 16 elements");
  const int bf = prec == PREC_BF16;
  const bool small = pf && pf->small_footprint && N >= 128;
  // the split mask epilogue (two output pieces plus the mask words per 32 columns) runs at half width
  const bool mask_split = mask != nullptr && c_split;
  const int BN = small ? 128
                 : mask_split ? ((N % 128 == 0 || N > 128) ? 128 : 64)
                 : (N % 256 == 0 || N > 256) ? 256 : (N % 128 == 0 || N > 128) ? 128 : 64;
  CUtensorMap tmA, tmB;
  if (a_chunk_rows_pad > 0) {
    NNC_REQUIRE(!a_split && static_cast<int64_t>(K / 64) * a_chunk_rows_pad < (int64_t(1) << 31), NNCONV_ERR_ARG,
                "gemm_tc: chunk-major A too large / not splittable");
    s = make_tmap_2d_16b(&tmA, bf, A_base, static_cast<uint64_t>(K / 64) * static_cast<uint64_t>(a_chunk_rows_pad), 64, 128);
  } else {
    s = make_tmap_2d_16b(&tmA, bf, A_base, static_cast<uint64_t>(a_rows_total),
                         static_cast<uint64_t>(a_split ? K / 3 * 2 : K), 128);
  }
  if (s != NNCONV_OK) return s;
  s = make_tmap_2d_16b(&tmB, bf, B, static_cast<uint64_t>(N), static_cast<uint64_t>(K), BN);
  if (s != NNCONV_OK) return s;
  GemmTcArgs a;
  a.M = M; a.N = N; a.K = K; a.a_row0 = static_cast<int>(a_row0); a.bias = bias; a.relu = relu; a.C = C; a.ldc = ldc;
  a.chunk_rows_pad = chunk_rows_pad;
  a.c_row0 = c_row0;
  a.a_chunk_rows_pad = a_chunk_rows_pad;
  a.b_policy = options().gemm_b_policy ? kEvictLast : kEvictNormal;
  a.acc_scale = acc_scale;
  a.a_split_nk = a_split ? K / 192 : 0;
  a.c_split = c_split ? 1 : 0;
  a.overflow = (overflow != nullptr && !bf) ? overflow : nullptr;
  a.mask = static_cast<const uint16_t*>(mask);
  a.mask_ld = mask_ld;
  a.out_f32 = out_f32;
  NNC_REQUIRE(mask == nullptr || (mask_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(mask) & 15) == 0), NNCONV_ERR_ARG,
              "gemm_tc: mask must be 16-byte aligned with mask_ld a multiple of 8");
  {
    TraceHandle th = trace_get();
    static unsigned int launch_seq = 0;
    a.trace = TraceBuf{th.rec, th.count, th.cap};
    a.trace_seq = launch_seq++;
  }
  // TMA-store epilogue: [16 x 32] panels; rows past M are clipped by the tensor bounds (row-major) or land in
  // the row padding of each chunk panel (chunk-major, chunk_rows_pad >= round_up(c_row0 + M, 32))
  const bool no_tma_store = options().gemm_direct_store != 0;
  a.tma_store = 0;
  a.bias_v4 = bias != nullptr && (reinterpret_cast<uintptr_t>(bias) & 15) == 0;
  CUtensorMap tmC = tmA;
  const bool panel_ok = chunk_rows_pad > 0
                            ? ((c_row0 + M + 31) / 32 * 32 <= chunk_rows_pad &&
                               static_cast<int64_t>(nmul * N / 64) * chunk_rows_pad < (int64_t(1) << 31))
                            : ldc == static_cast<int64_t>(nmul) * N;
  if (!no_tma_store && pf == nullptr && panel_ok && !out_f32) {
    if (chunk_rows_pad > 0) {
      s = make_tmap_store_16b(&tmC, bf, C, static_cast<uint64_t>(nmul * N / 64) * static_cast<uint64_t>(chunk_rows_pad), 64);
    } else {
      s = make_tmap_store_16b(&tmC, bf, C, static_cast<uint64_t>(M), static_cast<uint64_t>(nmul) * N);
    }
    if (s != NNCONV_OK) return s;
    a.tma_store = 1;
  }
  a.wait_ok = pf ? pf->wait_ok : nullptr;
  a.done_cnt = pf ? pf->done_cnt : nullptr;
  a.done_ok = pf ? pf->done_ok : nullptr;
  const bool pdl = pf && pf->pdl;
  // the activation matters only where it is applied (relu) or differentiated (mask); every other launch is the ReLU
  // instantiation, as it always was
  a.act_p = act.p;
  if (act.kind == ACT_RELU || (!relu && mask == nullptr)) return dispatch_gemm<ACT_RELU>(tmA, tmB, tmC, a, st, pdl, BN, bf, small, out_f32, mask_split, mask != nullptr, c_split);
  NNC_REQUIRE(!out_f32 && !small, NNCONV_ERR_ARG, "gemm_tc: the activation excludes fp32 output / the small-footprint configuration");
  return act_dispatch(act.kind, [&](auto k) {
    return dispatch_gemm<decltype(k)::value>(tmA, tmB, tmC, a, st, pdl, BN, bf, small, out_f32, mask_split, mask != nullptr, c_split);
  });
}

}  // namespace nnc
