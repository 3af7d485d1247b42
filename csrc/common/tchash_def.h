// BBH64 ("tensor-core hash") — definition shared by the CPU reference and the sm_90a kernels.
//
// The reference computes no checksum at all (error_codes.h:62-63 defines CHECKSUM_MISMATCH /
// DATA_CORRUPTION but nothing produces them, SURVEY K11).  BBH64 is the checksum designed for
// the GPU data plane: the 16 KiB tile that TMA lands in shared memory is consumed *in place* as
// the A operand of `wgmma.mma_async...s32.u8.u8` (u8 x u8 -> s32) against a fixed pseudo-random
// weight matrix, so the payload bytes never pass through registers and hashing overlaps the copy.
//
//   tile   = 16384 bytes, viewed as A[128 rows][128 k] in the wgmma K-major no-swizzle
//            canonical layout: linear offset o -> row m = (o/1024)*8 + (o%128)/16,
//                                                k     = ((o%1024)/128)*16 + o%16
//            (8-row x 16-byte core matrices; LBO = 128 B between K chunks, SBO = 1024 B
//             between 8-row groups).  Short tiles are zero padded.
//   D[m][n] = sum_k A[m][k] * W[k][n]            (u8*u8 accumulated in 32 bits; N = 16)
//   r(m)    = sum_n D[m][n] * KN[n]              (mod 2^64)
//   c(g)    = mix64(r(m) + (g+1)*GOLD),  g = tile_index*128 + m   (position dependent)
//   digest  = mix64( (sum_g c(g) mod 2^64) ^ (nbytes * LENMUL) )
//
// The outer sum is commutative, so tiles may complete in any order on any SM.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define BB_HD __host__ __device__ __forceinline__
#else
#define BB_HD inline
#endif

namespace bb::tchash {

constexpr uint32_t kTileBytes = 16384;
constexpr uint32_t kRows = 128;   // tile rows (two wgmma M=64 halves)
constexpr uint32_t kK = 128;      // bytes per row (4 MMAs of K=32)
constexpr uint32_t kN = 16;       // wgmma N (hash columns)
constexpr uint64_t kGold = 0x9E3779B97F4A7C15ull;
constexpr uint64_t kLenMul = 0xD6E8FEB86659FD93ull;

BB_HD uint32_t weight(uint32_t k, uint32_t n) {
  uint32_t h = (k * kN + n + 1u) * 0x9E3779B1u;
  h ^= h >> 15;
  h *= 0x85EBCA77u;
  h ^= h >> 13;
  return ((h >> 8) & 0xFFu) | 1u;  // odd, 1..255
}

BB_HD uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

BB_HD uint64_t col_mul(uint32_t n) { return splitmix64(n + 1u) | 1ull; }

BB_HD uint64_t mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

BB_HD uint64_t row_contrib(uint64_t r, uint64_t global_row) { return mix64(r + (global_row + 1ull) * kGold); }
BB_HD uint64_t finalize(uint64_t sum, uint64_t nbytes) { return mix64(sum ^ (nbytes * kLenMul)); }

// tile-linear offset -> (row, k)
BB_HD uint32_t off_to_row(uint32_t o) { return (o >> 10) * 8u + ((o & 127u) >> 4); }
BB_HD uint32_t off_to_k(uint32_t o) { return (((o & 1023u) >> 7) << 4) + (o & 15u); }
// (row, k) -> tile-linear offset
BB_HD uint32_t rk_to_off(uint32_t m, uint32_t k) { return (m >> 3) * 1024u + (k >> 4) * 128u + (m & 7u) * 16u + (k & 15u); }

}  // namespace bb::tchash
