// wgmma "TN" GEMM: a reduction over ROWS (edges / sources), the shape every parameter gradient of the
// NNConv path has (SURVEY Appendix A: dW_l = sum_e dz_l[e] (x) h_{l-1}[e]; dW_L = sum_c x_c (x) dY_c):
//
//     C[M, N] (fp32)  (+)=  alpha * sum_{r < R} A[r, m] * B[r, n]        A: [R, lda], B: [R, ldb] 16-bit row-major
//
// Both operands are "MN-major" for the tensor core (contiguous along M / N, strided along the reduction):
// a TMA box of [64 rows x 64 columns] with SWIZZLE_128B lands in shared memory exactly in the canonical
// MN-major SW128 layout (8 rows of 128 B per swizzle atom; atoms 1024 B apart along K = SBO; the next 64
// columns of M / N are the next box = LBO), so the rows are used as they lie in HBM -- no transposed copy
// of the 2 KB/edge activations is ever written.  The wgmma transpose flags select MN-major A / B.
//
// Work split: tiles of 128 x BLOCK_N of C times `ksplit` row ranges; each CTA accumulates its range in the registers
// of two warpgroups (BLOCK_N / 2 columns each) and adds the tile to C with red.global.add.v4.f32 (C is a
// zero-initialised fp32 accumulator owned by the caller).
// Rows past R are zero-filled by TMA, so R needs no padding.
#include "kernels.h"
#include "tc05.cuh"
#include "tmap.h"

namespace nnc {

int tc_num_sms();

namespace {

using namespace tc05;

struct GemmTnArgs {
  int M, N, R;
  int kb_per_split;        // 64-row blocks per CTA along the reduction
  int a_col0, b_col0;      // first column of A / B inside their tensor maps
  float* C;
  int64_t ldc;
  float alpha;
  const float* alpha_dev;  // optional device scalar multiplied into alpha
};

template <int BLOCK_N>
struct TnCfg {
  static constexpr int kRowsK = 64;                       // reduction rows per stage
  static constexpr int kBoxBytes = kRowsK * 128;          // one [64 x 64] 16-bit box
  static constexpr int kABytes = 2 * kBoxBytes;           // M = 128: two boxes
  static constexpr int kBBytes = (BLOCK_N / 64) * kBoxBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kScratchBytes = 8 * acc_scratch_bytes<32>();
  static constexpr int kStages = (180 * 1024 / kStageBytes) > 6 ? 6 : (180 * 1024 / kStageBytes);
  static constexpr int kSmemBytes = kStages * kStageBytes + kScratchBytes + 1024 + 256;
};

template <int BLOCK_N, int FMT>
__global__ void __launch_bounds__(288, 1)
k_gemm_tn(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmTnArgs a) {
  using Cfg = TnCfg<BLOCK_N>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
  float* scratch = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes + Cfg::kScratchBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::kStages;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x / 32), 0), lane = threadIdx.x % 32;
  const int n_blocks = ceil_div(a.N, BLOCK_N);
  const int tile = blockIdx.x, split = blockIdx.y;
  const int mb = tile / n_blocks, nb = tile % n_blocks;
  const int total_kb = ceil_div(a.R, Cfg::kRowsK);
  const int kb0 = split * a.kb_per_split;
  const int kb1 = min(total_kb, kb0 + a.kb_per_split);
  const int num_kb = kb1 - kb0;
  if (num_kb <= 0) return;     // uniform per CTA, before any barrier

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ---------------------------------------------------------------- TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&empty[stage], phase ^ 1u);
      if (elect_one()) {
        uint8_t* st = smem + stage * Cfg::kStageBytes;
        mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
        const int r0 = kb * Cfg::kRowsK;
#pragma unroll
        for (int i = 0; i < 2; ++i)
          tma_load_2d(st + i * Cfg::kBoxBytes, &tmA, &full[stage], a.a_col0 + mb * 128 + i * 64, r0, kEvictFirst);
#pragma unroll
        for (int i = 0; i < BLOCK_N / 64; ++i)
          tma_load_2d(st + Cfg::kABytes + i * Cfg::kBoxBytes, &tmB, &full[stage], a.b_col0 + nb * BLOCK_N + i * 64, r0,
                      kEvictFirst);
      }
      __syncwarp();
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
    }
  } else {
    // ---------------------------------------------------------------- consumer warpgroups: columns [half * BLOCK_N / 2, ...)
    constexpr int NH = BLOCK_N / 2;                 // whole 64-column boxes of B
    const int quarter = warp % 4, half = warp / 4;
    const int n_base = nb * BLOCK_N + half * NH;
    const bool live = n_base < a.N;                 // N <= BLOCK_N / 2: the second warpgroup only drains the ring
    float* wb = scratch + warp * (acc_scratch_bytes<32>() / 4);
    Acc<NH> acc;
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      if (live) {
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint64_t adesc = smem_desc_mn_sw128(sa, Cfg::kBoxBytes);
        const uint64_t bdesc = smem_desc_mn_sw128(sa + Cfg::kABytes + half * (NH / 64) * Cfg::kBoxBytes, Cfg::kBoxBytes);
        // the second m64 half of A is the next [64 x 64] box; 16 reduction rows = two 8-row groups of 1024 B
        mma_block<NH, FMT, 1, 1>(acc, adesc, bdesc, Cfg::kBoxBytes >> 4, 128, Cfg::kRowsK / 16, kb != 0);
        wgmma_wait<0>();
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
    }
    if (live) {
      // ---- epilogue: C += alpha * D
      float alpha = a.alpha;
      if (a.alpha_dev != nullptr) alpha *= __ldg(a.alpha_dev);
      const int m = mb * 128 + acc_row(quarter, lane);
      float* crow = a.C + static_cast<int64_t>(m) * a.ldc + n_base;
#pragma unroll
      for (int cc = 0; cc < NH; cc += 32) {
        uint32_t v[32];
        acc_rows<NH, 32>(acc, cc, wb, v);
        if (m < a.M) {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int n = n_base + cc + 4 * q;
            if (n + 3 < a.N) {
              red_add_v4(crow + cc + 4 * q, alpha * __uint_as_float(v[4 * q]), alpha * __uint_as_float(v[4 * q + 1]),
                         alpha * __uint_as_float(v[4 * q + 2]), alpha * __uint_as_float(v[4 * q + 3]));
            } else {
              for (int j = 0; j < 4; ++j)
                if (n + j < a.N) atomicAdd(crow + cc + 4 * q + j, alpha * __uint_as_float(v[4 * q + j]));
            }
          }
        }
      }
    }
  }
}

template <int BLOCK_N, int FMT>
int launch_tn_cfg(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmTnArgs& a, dim3 grid, cudaStream_t st) {
  using Cfg = TnCfg<BLOCK_N>;
  static bool attr_set = false;
  if (!attr_set) {
    NNC_CHECK_CUDA(cudaFuncSetAttribute(k_gemm_tn<BLOCK_N, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        Cfg::kSmemBytes));
    attr_set = true;
  }
  k_gemm_tn<BLOCK_N, FMT><<<grid, 288, Cfg::kSmemBytes, st>>>(tmA, tmB, a);
  NNC_CHECK_LAUNCH();
  return NNCONV_OK;
}

}  // namespace

int launch_gemm_tn(int prec, const void* A, int64_t lda, int a_col0, const void* B, int64_t ldb, int b_col0, int64_t R,
                   int M, int N, float* C, int64_t ldc, float alpha, const float* alpha_dev, cudaStream_t st) {
  if (M <= 0 || N <= 0 || R <= 0) return NNCONV_OK;
  int s = tc_init();
  if (s != NNCONV_OK) return s;
  NNC_REQUIRE(prec == PREC_F16 || prec == PREC_BF16, NNCONV_ERR_ARG, "gemm_tn: 16-bit operands only");
  NNC_REQUIRE(lda % 64 == 0 && ldb % 64 == 0 && a_col0 % 64 == 0 && b_col0 % 64 == 0 && R < (int64_t(1) << 31),
              NNCONV_ERR_ARG, "gemm_tn: leading dimensions / column offsets must be multiples of 64");
  NNC_REQUIRE(ldc % 4 == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0, NNCONV_ERR_ARG,
              "gemm_tn: C must be 16-byte aligned with ldc a multiple of 4");
  const int bf = prec == PREC_BF16;
  const int BN = N > 128 ? 256 : 128;
  CUtensorMap tmA, tmB;
  s = make_tmap_2d_16b(&tmA, bf, A, static_cast<uint64_t>(R), static_cast<uint64_t>(lda), 64);
  if (s != NNCONV_OK) return s;
  s = make_tmap_2d_16b(&tmB, bf, B, static_cast<uint64_t>(R), static_cast<uint64_t>(ldb), 64);
  if (s != NNCONV_OK) return s;
  GemmTnArgs a;
  a.M = M; a.N = N; a.R = static_cast<int>(R); a.a_col0 = a_col0; a.b_col0 = b_col0;
  a.C = C; a.ldc = ldc; a.alpha = alpha; a.alpha_dev = alpha_dev;
  const int tiles = ceil_div(M, 128) * ceil_div(N, BN);
  const int total_kb = static_cast<int>(ceil_div64(R, 64));
  // split the reduction so that about two waves of CTAs cover the machine, but keep >= 8 row blocks per CTA
  // (the fp32 atomics of a tile cost about as much as 2-4 blocks of MMAs)
  int ksplit = (2 * tc_num_sms() + tiles - 1) / tiles;
  if (ksplit > total_kb / 8) ksplit = total_kb / 8;
  if (ksplit < 1) ksplit = 1;
  if (ksplit > 65535) ksplit = 65535;
  a.kb_per_split = ceil_div(total_kb, ksplit);
  ksplit = ceil_div(total_kb, a.kb_per_split);
  dim3 grid(tiles, ksplit);
  if (BN == 256) return bf ? launch_tn_cfg<256, 1>(tmA, tmB, a, grid, st) : launch_tn_cfg<256, 0>(tmA, tmB, a, grid, st);
  return bf ? launch_tn_cfg<128, 1>(tmA, tmB, a, grid, st) : launch_tn_cfg<128, 0>(tmA, tmB, a, grid, st);
}

}  // namespace nnc
