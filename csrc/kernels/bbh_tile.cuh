// BBH64 tile product on the tensor cores, shared by bb_xfer (xfer_fused.cu) and bb_xfer_fp8 (xfer_mxfp8.cu).
//
// One warpgroup hashes a landed 16 KiB tile in place: D[128x16] = A[128x128] * W[128x16] is two M=64 halves of four
// `wgmma.mma_async.m64n16k32.s32.u8.u8` each, both operands read straight from shared memory through no-swizzle
// K-major descriptors (the tile layout of tchash_def.h).  The 16 s32 accumulators per thread then become the
// position-dependent row hashes; each warp returns the sum over its 32 rows, the four warps cover all 128 rows.
#pragma once
#include <cstdint>

#include "common/tchash_def.h"
#include "kernels/ptx.cuh"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {

// Thread `tid` of `nthreads` writes its share of the 2 KiB BBH64 weight matrix W[k][n] as the wgmma B operand (N = 16
// rows, K-major, no swizzle); the caller fences it for the async proxy and synchronises.
__device__ __forceinline__ void bbh_load_weights(uint8_t* w, uint32_t tid, uint32_t nthreads) {
  for (uint32_t o = tid; o < 2048; o += nthreads) w[o] = static_cast<uint8_t>(tchash::weight(tchash::off_to_k(o), tchash::off_to_row(o)));
}

// d[8h + i] (h = M half) follows the wgmma_m64n16k32_u8 fragment layout, with rows offset by 64 h.
// Every thread of the warpgroup must call this (the MMAs are warpgroup-wide).
__device__ __forceinline__ void bbh_tile_mma(uint32_t a_addr, uint32_t w_addr, uint32_t (&d)[16]) {
  uint32_t (&lo)[8] = *reinterpret_cast<uint32_t(*)[8]>(&d[0]);
  uint32_t (&hi)[8] = *reinterpret_cast<uint32_t(*)[8]>(&d[8]);
  ptx::wgmma_fence();
#pragma unroll
  for (uint32_t j = 0; j < tchash::kK / 32; ++j) {
    // each MMA consumes K = 32 bytes = two 16-byte K chunks (LBO 128 B apart); 8-row groups are 1024 B apart
    const uint64_t db = ptx::gmma_desc_kmajor_noswizzle(w_addr + j * 256, 128, 1024);
    ptx::wgmma_m64n16k32_u8(lo, ptx::gmma_desc_kmajor_noswizzle(a_addr + j * 256, 128, 1024), db, j > 0 ? 1u : 0u);
    ptx::wgmma_m64n16k32_u8(hi, ptx::gmma_desc_kmajor_noswizzle(a_addr + 8192 + j * 256, 128, 1024), db, j > 0 ? 1u : 0u);
  }
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
}

// Tile row / column of accumulator d[k] held by lane `lane` of warp `q` (0..3) of the warpgroup.
__device__ __forceinline__ uint32_t bbh_acc_row(uint32_t k, uint32_t q, uint32_t lane) {
  return 64u * (k >> 3) + 16u * q + (lane >> 2) + 8u * ((k >> 1) & 1u);
}
__device__ __forceinline__ uint32_t bbh_acc_col(uint32_t k, uint32_t lane) { return 2u * (lane & 3u) + (k & 1u) + 8u * ((k >> 2) & 1u); }

// Sum over this warp's 32 rows of row_contrib(r(m), tile_index * 128 + m), returned in every lane.  A row's 16 columns
// are spread over the 4 lanes of a quad; the quad reduce-scatters its 4 rows so that each lane finishes one of them.
__device__ __forceinline__ uint64_t bbh_tile_rows(const uint32_t (&d)[16], const uint64_t* col_mul, uint32_t tile_index, uint32_t q,
                                                  uint32_t lane) {
  uint64_t part[4] = {0, 0, 0, 0};  // rows bbh_acc_row(k) for k = 0, 2, 8, 10
#pragma unroll
  for (uint32_t k = 0; k < 16; ++k) part[2 * (k >> 3) + ((k >> 1) & 1u)] += static_cast<uint64_t>(d[k]) * col_mul[bbh_acc_col(k, lane)];
  const bool b1 = (lane >> 1) & 1u, b0 = lane & 1u;
  const uint64_t k0 = (b1 ? part[2] : part[0]) + shfl_xor_u64(b1 ? part[0] : part[2], 2);  // M half b1
  const uint64_t k1 = (b1 ? part[3] : part[1]) + shfl_xor_u64(b1 ? part[1] : part[3], 2);
  const uint64_t r = (b0 ? k1 : k0) + shfl_xor_u64(b0 ? k0 : k1, 1);                        // row offset 8 b0
  const uint32_t row = 64u * b1 + 16u * q + (lane >> 2) + 8u * b0;
  uint64_t v = tchash::row_contrib(r, static_cast<uint64_t>(tile_index) * tchash::kRows + row);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += shfl_xor_u64(v, o);
  return v;
}

}  // namespace bb::gpu
