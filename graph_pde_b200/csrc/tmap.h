// Host-side TMA descriptor (CUtensorMap) construction without linking libcuda: the driver entry point
// is resolved through the runtime (cudaGetDriverEntryPoint).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace nnc {

int tmap_init();
// 2-D row-major tensor of 16-bit elements [rows, cols] (cols contiguous), box = [box_rows, 64 cols],
// 128-byte swizzle (the layout wgmma K-major SW128 descriptors expect).
int make_tmap_2d_16b(CUtensorMap* out, int is_bf16, const void* base, uint64_t rows, uint64_t cols,
                     uint32_t box_rows);
// same tensor, described for the GEMM epilogue's TMA stores: box = [32 rows, 32 cols], 64-byte swizzle
// (one warp's 32 x 32 output piece, 2 KB of shared memory).
int make_tmap_store_16b(CUtensorMap* out, int is_bf16, const void* base, uint64_t rows, uint64_t cols);

}  // namespace nnc
