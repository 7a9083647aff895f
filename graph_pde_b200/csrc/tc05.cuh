// sm_90a building blocks: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA, fp32 accumulators in registers).
// Thin inline-PTX wrappers only; no CUTLASS dependency.  All waits are bounded (trap instead of
// hanging the GPU if a pipeline is mis-programmed).
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>

namespace tc05 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: ~seconds of polling, then trap (a trapped kernel returns an error; a hung one costs
// the whole GPU lease).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#pragma unroll 1
  for (uint32_t i = 0; i < (1u << 24); ++i) {
    if (mbar_try_wait(bar, parity)) return;
  }
  __trap();
}

// ---------------------------------------------------------------- TMA
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
// 2-D tile load: coordinates (c0 = innermost/column element index, c1 = row index).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// 2-D tile store smem -> global through the async proxy (bulk group completion).  The smem tile uses the tensor
// map's swizzle; rows/columns outside the tensor are clipped by the hardware.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(m), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed groups have finished READING shared memory (the buffer may be overwritten)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... all but the most recent one
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
// all committed groups are complete (global writes performed)
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Register reallocation between warpgroups (setmaxnreg): every warp of the warpgroup executes it; R is a multiple
// of 8 in [24, 256].  A producer warpgroup hands registers back so the consumer warpgroups can hold their
// accumulators and run the epilogue without spilling.
template <uint32_t R>
__device__ __forceinline__ void warpgroup_reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <uint32_t R>
__device__ __forceinline__ void warpgroup_reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void ld_shared_v4(uint32_t addr, uint32_t* v) {
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr)
               : "memory");
}
// Four 8x8 16-bit matrices from registers in the mma / wgmma accumulator layout (register i of lane l: row l / 4,
// columns 2 (l % 4), + 1 of matrix i, two 16-bit values) to shared memory; lanes 8i .. 8i + 7 give the addresses of
// the eight 16-byte rows of matrix i.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}

// One lane of a CONVERGED warp (elect.sync).  Role loops run on all 32 lanes and only issue through the elected
// lane: operands computed in converged code are warp-uniform for the compiler (uniform registers), whereas
// inside an `if (lane == 0)` region every TMA / mbarrier instruction is wrapped in an
// ELECT / R2UR / BRA.U.ANY waterfall loop (~45 cycles each).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n .reg .pred p;\n elect.sync _|p, 0xffffffff;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- wgmma
// A 128-row tile is computed by ONE warpgroup (4 warps) as two m64 halves; the fp32 accumulators stay in the
// registers of that warpgroup, which also runs the tile's epilogue.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N]; FMT 0 = fp16, 1 = bf16 operands; TA / TB = 1: MN-major A / B.
template <int N, int FMT>
struct Wgmma;
// operand lists shared by the fp16 / bf16 forms of one width
#define TC05_WG_TAIL_16 "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n}"
#define TC05_WG_OUT_16 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
#define TC05_WG_TAIL_32 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n}"
#define TC05_WG_OUT_32 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define TC05_WG_TAIL_64 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n}"
#define TC05_WG_OUT_64 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define TC05_WG_TAIL_128 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n}"
#define TC05_WG_OUT_128 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define TC05_WG_DEF(N, SC) \
  template <int FMT> \
  struct Wgmma<N, FMT> { \
    template <int TA, int TB> \
    static __device__ __forceinline__ void run(float* d, uint64_t a, uint64_t b, int scale_d) { \
      if constexpr (FMT == 0) \
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #SC ", 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " TC05_WG_TAIL_##N \
                     : TC05_WG_OUT_##N : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)); \
      else \
        asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #SC ", 0;\n" \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 " TC05_WG_TAIL_##N \
                     : TC05_WG_OUT_##N : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)); \
    } \
  };
TC05_WG_DEF(16, 10)
TC05_WG_DEF(32, 18)
TC05_WG_DEF(64, 34)
TC05_WG_DEF(128, 66)

template <int N, int FMT, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma(float* d, uint64_t a, uint64_t b, int scale_d) {
  if constexpr (N == 16 || N == 32 || N == 64 || N == 128) {
    Wgmma<N, FMT>::template run<TA, TB>(d, a, b, scale_d);
  } else {
    // other widths as 64 / 32 / 16-column pieces: a K-major B sub-tile of P rows starts P * 128 B (P * 8 descriptor
    // units, a whole number of 8-row swizzle atoms) further; its accumulators are the next P / 2 registers
    static_assert(N % 16 == 0 && N < 128 && TB == 0, "wgmma: unsupported width");
    constexpr int P = N > 64 ? 64 : N > 32 ? 32 : 16;
    Wgmma<P, FMT>::template run<TA, TB>(d, a, b, scale_d);
    wgmma<N - P, FMT, TA, TB>(d + P / 2, a, b + P * 8, scale_d);
  }
}

// Accumulator of a [128 x N] tile held by one warpgroup: d[0] rows 0..63, d[1] rows 64..127.
template <int N>
struct Acc {
  float d[2][N / 2];
};

// One K block of a 128-row tile: `ksteps` k16 steps, the two m64 halves `a_half` descriptor units apart, every step
// advancing both descriptors by `kstep` units (16-byte units of the shared-memory start address).
template <int N, int FMT, int TA = 0, int TB = 0>
__device__ __forceinline__ void mma_block(Acc<N>& acc, uint64_t adesc, uint64_t bdesc, uint32_t a_half, uint32_t kstep,
                                          int ksteps, bool accumulate) {
  wgmma_fence();
#pragma unroll 1
  for (int k = 0; k < ksteps; ++k) {
    const int sd = (accumulate || k != 0) ? 1 : 0;
    wgmma<N, FMT, TA, TB>(acc.d[0], adesc + kstep * k, bdesc + kstep * k, sd);
    wgmma<N, FMT, TA, TB>(acc.d[1], adesc + a_half + kstep * k, bdesc + kstep * k, sd);
  }
  wgmma_commit();
}

// Row of the 128-row tile that lane `lane` of warp `w` (0..3 inside its warpgroup) stands for in the epilogue: a
// warp's accumulator fragments cover rows 16w..16w+15 of both m64 halves, so its 32 lanes take exactly those rows.
__device__ __forceinline__ int acc_row(int w, int lane) { return lane < 16 ? 16 * w + lane : 48 + 16 * w + lane; }

// Columns [c0, c0 + NC) of the lane's row (acc_row) into v[0..NC): the warp transposes its fragments through `wb`,
// a private [32 x (NC + 4)] fp32 shared-memory scratch.  Call from fully unrolled loops only (c0 must fold to a
// constant, or the accumulator is demoted to local memory).
template <int NC>
constexpr int acc_scratch_bytes() { return 32 * (NC + 4) * 4; }
template <int N, int NC>
__device__ __forceinline__ void acc_rows(const Acc<N>& acc, int c0, float* wb, uint32_t* v) {
  constexpr int P = NC + 4;
  const int lane = threadIdx.x & 31;
  const int r = lane >> 2, c = (lane & 3) * 2;
  __syncwarp();
#pragma unroll
  for (int jj = 0; jj < NC / 8; ++jj) {
    const int j = c0 / 8 + jj;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      *reinterpret_cast<float2*>(wb + (16 * h + r) * P + 8 * jj + c) = make_float2(acc.d[h][4 * j], acc.d[h][4 * j + 1]);
      *reinterpret_cast<float2*>(wb + (16 * h + r + 8) * P + 8 * jj + c) =
          make_float2(acc.d[h][4 * j + 2], acc.d[h][4 * j + 3]);
    }
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < NC / 4; ++q) {
    const float4 f = *reinterpret_cast<const float4*>(wb + lane * P + 4 * q);
    v[4 * q] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y);
    v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
  }
}

// ---------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor, K-major operand tile stored as rows of 128 bytes with the 128B swizzle
// (what a TMA box {64 x 16-bit, rows} with CU_TENSOR_MAP_SWIZZLE_128B writes): 8-row groups are 1024 B apart (SBO),
// LBO unused for swizzled K-major, layout type 1 (SWIZZLE_128B).  A k16 step is +32 B (+2 units), the second m64
// half of a 128-row tile +8 KB (+512 units).
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;             // LBO (ignored)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;     // SBO
  d |= static_cast<uint64_t>(1) << 62;             // SWIZZLE_128B
  return d;
}
// MN-major SW128 operand: start address, LBO = bytes between consecutive 64-element blocks along M / N,
// SBO = 1024 B between consecutive 8-row groups along K.  A k16 step is two 8-row groups (+2048 B, +128 units).
__device__ __forceinline__ uint64_t smem_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;             // SWIZZLE_128B
  return d;
}

// red.global.add.v4.f32 (sm_90+): four fp32 atomics to 16 contiguous, 16B-aligned bytes in one request.
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}

// Bulk reduction smem -> global through the async proxy (TMA engine): global[0..bytes) += smem[0..bytes) as fp32 adds.
// bytes multiple of 16, both addresses 16-byte aligned; completion through the issuing thread's bulk groups.
__device__ __forceinline__ void bulk_reduce_add_f32(float* gdst, uint32_t smem_src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
               ::"l"(gdst), "r"(smem_src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_reduce_max_u64(unsigned long long* gdst, uint32_t smem_src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.max.u64 [%0], [%1], %2;"
               ::"l"(gdst), "r"(smem_src), "r"(bytes)
               : "memory");
}

// 32 bytes (one full sector) per thread as two 16-byte stores
__device__ __forceinline__ void st_global_32b(void* addr, const uint32_t* v) {
  uint4* p = reinterpret_cast<uint4*>(addr);
  p[0] = make_uint4(v[0], v[1], v[2], v[3]);
  p[1] = make_uint4(v[4], v[5], v[6], v[7]);
}

// same with an L2 eviction-priority hint (Y ring: keep resident against the evict-first h stream)
__device__ __forceinline__ void st_global_32b_hint(void* addr, const uint32_t* v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]),
               "r"(v[3]), "l"(policy)
               : "memory");
  asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(static_cast<char*>(addr) + 16), "r"(v[4]),
               "r"(v[5]), "r"(v[6]), "r"(v[7]), "l"(policy)
               : "memory");
}

// ---------------------------------------------------------------- A-tile rings of the two-warpgroup contractions
// The A stages are split into one ring per tile slot of a unit (ring 0: stages [0, r0), ring 1: [r0, a_stages),
// r0 = ceil(a_stages / 2)): each ring has exactly one consumer warpgroup, which therefore never waits on a stage more
// than one phase ahead of it (a stage shared by both warpgroups could be two phases ahead and pass a parity wait
// on a stale phase).
struct ARing {
  int stage, end, begin;
  uint32_t phase;
  __device__ void init(int ti, int a_stages) {
    const int r0 = (a_stages + 1) / 2;
    begin = ti == 0 ? 0 : r0;
    end = ti == 0 ? r0 : a_stages;
    stage = begin;
    phase = 0;
  }
  __device__ void next() {
    if (++stage == end) { stage = begin; phase ^= 1u; }
  }
};

// ---------------------------------------------------------------- cross-kernel pipelining (PDL + flags)
// Kernels of one NNConv application are launched with programmatic stream serialization: a kernel may
// start as soon as every CTA of its predecessor has executed launch_dependents, i.e. CTAs of kernel k+1
// fill SMs as CTAs of kernel k retire (no grid-wide drain between the many small launches).  Real data
// dependencies are carried by completion flags in global memory (release/acquire at gpu scope).
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// one thread: wait until *ok != 0 (bounded), then order later async-proxy (TMA) reads after it
// `sleep_ns`: pause between polls.  Every poll is an L2 round trip to ONE line; hundreds of threads polling it
// back to back saturate that L2 slice and delay every tile load that has
// a sector behind it -- long expected waits must poll slowly.
__device__ __forceinline__ void flag_wait(const int* ok, uint32_t sleep_ns = 64) {
#pragma unroll 1
  for (uint32_t i = 0; i < (1u << 26); ++i) {
    if (ld_acquire(ok) != 0) {
      // order the acquire (generic proxy) before the TMA reads (async proxy) of GLOBAL memory only: the
      // unqualified fence also covers shared memory and would drain the producer's in-flight TMA loads at every
      // batch boundary
      asm volatile("fence.proxy.async.global;" ::: "memory");
      return;
    }
    __nanosleep(sleep_ns);
  }
  __trap();
}
// call with ALL threads of the CTA after its last global write: the last CTA of the grid raises *ok
__device__ __forceinline__ void signal_done(int* cnt, int* ok) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(cnt, 1);
    if (prev == static_cast<int>(gridDim.x) - 1) {
      __threadfence();
      asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(ok), "r"(1) : "memory");
    }
  }
}

// ---------------------------------------------------------------- optional CTA timeline tracing
// (NNCONV_TRACE=1, measurement only): one record per CTA = {kernel tag, blockIdx, smid, start, ready, end}
// in nanoseconds of %globaltimer; `ready` = after the cross-kernel flag wait.
struct TraceBuf {
  unsigned long long* rec;   // [cap][6]
  unsigned int* count;
  unsigned int cap;
};
__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned int smid() {
  unsigned int r;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void trace_write(const TraceBuf& tb, unsigned int tag, unsigned long long t0,
                                            unsigned long long t1, unsigned long long t2) {
  if (tb.rec == nullptr) return;
  const unsigned int i = atomicAdd(tb.count, 1u);
  if (i >= tb.cap) return;
  unsigned long long* r = tb.rec + static_cast<size_t>(i) * 6;
  r[0] = tag;
  r[1] = blockIdx.x;
  r[2] = smid();
  r[3] = t0;
  r[4] = t1;
  r[5] = t2;
}

}  // namespace tc05
