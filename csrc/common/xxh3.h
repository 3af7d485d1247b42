// XXH3-64 of one 16 KiB tile -- the standard digest of the data plane (`ChecksumAlgo::XXH3`).
//
// BASELINE.json / SURVEY K11 name "CRC32/xxhash" as the checksums to fuse into put / get; the reference only declares the
// error codes (include/blackbird/common/error/error_codes.h:62-63) and computes nothing.  XXH3-64 (Yann Collet's xxHash
// 0.8 specification, default secret, seed 0) over a whole object is a serial recurrence (the 8-lane accumulator is
// scrambled after every 1 KiB block), so it cannot be evaluated tile-parallel by 132 SMs whose tiles finish in any order.
// The object digest therefore is
//
//   digest = mix64( ( sum over tiles t of  mix64( XXH3_64(tile_t) + (t + 1) * GOLD ) )  ^  nbytes * LENMUL )
//
// where tile_t is the t-th 16 KiB of the object, the last one zero padded, and XXH3_64 is the *unmodified* standard
// function (any xxHash library reproduces the per-tile values: tests/test_common.py checks against python-xxhash); the
// outer combine is the position-keyed commutative sum BBH64 uses (tchash_def.h), so tiles may complete in any order on
// any SM, byte ranges can be hashed as slices and summed (XFER_RAW_SUM), and host tiers stream it chunk by chunk.
//
// For a 16384-byte input XXH3_64 is always the "long input" path: 15 blocks of 16 stripes with a scramble after each, a
// 16th block of 15 stripes, the last stripe with the secret at offset 121, then the merge.  Only that path is
// implemented (tiles are always padded to 16 KiB).
//
// GPU mapping (xfer_fused.cu, ALGO_XXH3): the per-block stripe sums do not depend on the accumulator, so the 4 epilogue
// warps compute all 16 x 8 (block, lane) sums of a tile in parallel (one thread each, 16 stripes of 8 bytes) straight from
// the shared-memory tile; the 15-step scramble chain and the merge run on 8 lanes of the finalizer warp.
#pragma once
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define BB_XHD __host__ __device__ __forceinline__
#else
#define BB_XHD inline
#endif

namespace bb::xxh3 {

constexpr uint32_t kTileBytes = 16384;
constexpr uint64_t P32_1 = 0x9E3779B1ull, P32_2 = 0x85EBCA77ull, P32_3 = 0xC2B2AE3Dull;
constexpr uint64_t P64_1 = 0x9E3779B185EBCA87ull, P64_2 = 0xC2B2AE3D27D4EB4Full, P64_3 = 0x165667B19E3779F9ull,
                   P64_4 = 0x85EBCA77C2B2AE63ull, P64_5 = 0x27D4EB2F165667C5ull, PMX1 = 0x165667919E3779F9ull;
constexpr uint32_t kSecretSize = 192, kStripe = 64, kStripesPerBlock = 16, kBlock = 1024;
constexpr uint32_t kLastAccStart = 7, kMergeStart = 11;

// The default secret of the specification (XXH3_kSecret).
constexpr uint8_t kSecret[kSecretSize] = {
    0xb8, 0xfe, 0x6c, 0x39, 0x23, 0xa4, 0x4b, 0xbe, 0x7c, 0x01, 0x81, 0x2c, 0xf7, 0x21, 0xad, 0x1c, 0xde, 0xd4, 0x6d, 0xe9, 0x83, 0x90, 0x97, 0xdb,
    0x72, 0x40, 0xa4, 0xa4, 0xb7, 0xb3, 0x67, 0x1f, 0xcb, 0x79, 0xe6, 0x4e, 0xcc, 0xc0, 0xe5, 0x78, 0x82, 0x5a, 0xd0, 0x7d, 0xcc, 0xff, 0x72, 0x21,
    0xb8, 0x08, 0x46, 0x74, 0xf7, 0x43, 0x24, 0x8e, 0xe0, 0x35, 0x90, 0xe6, 0x81, 0x3a, 0x26, 0x4c, 0x3c, 0x28, 0x52, 0xbb, 0x91, 0xc3, 0x00, 0xcb,
    0x88, 0xd0, 0x65, 0x8b, 0x1b, 0x53, 0x2e, 0xa3, 0x71, 0x64, 0x48, 0x97, 0xa2, 0x0d, 0xf9, 0x4e, 0x38, 0x19, 0xef, 0x46, 0xa9, 0xde, 0xac, 0xd8,
    0xa8, 0xfa, 0x76, 0x3f, 0xe3, 0x9c, 0x34, 0x3f, 0xf9, 0xdc, 0xbb, 0xc7, 0xc7, 0x0b, 0x4f, 0x1d, 0x8a, 0x51, 0xe0, 0x4b, 0xcd, 0xb4, 0x59, 0x31,
    0xc8, 0x9f, 0x7e, 0xc9, 0xd9, 0x78, 0x73, 0x64, 0xea, 0xc5, 0xac, 0x83, 0x34, 0xd3, 0xeb, 0xc3, 0xc5, 0x81, 0xa0, 0xff, 0xfa, 0x13, 0x63, 0xeb,
    0x17, 0x0d, 0xdd, 0x51, 0xb7, 0xf0, 0xda, 0x49, 0xd3, 0x16, 0x55, 0x26, 0x29, 0xd4, 0x68, 0x9e, 0x2b, 0x16, 0xbe, 0x58, 0x7d, 0x47, 0xa1, 0xfc,
    0x8f, 0xf8, 0xb8, 0xd1, 0x7a, 0xd0, 0x31, 0xce, 0x45, 0xcb, 0x3a, 0x8f, 0x95, 0x16, 0x04, 0x28, 0xaf, 0xd7, 0xfb, 0xca, 0xbb, 0x4b, 0x40, 0x7e,
};

constexpr uint64_t secret64(uint32_t off) {  // little-endian 64-bit read of the secret at any byte offset
  uint64_t v = 0;
  for (int i = 7; i >= 0; --i) v = (v << 8) | kSecret[off + static_cast<uint32_t>(i)];
  return v;
}

BB_XHD uint64_t init_acc(uint32_t lane) {
  switch (lane) {
    case 0: return P32_3;
    case 1: return P64_1;
    case 2: return P64_2;
    case 3: return P64_3;
    case 4: return P64_4;
    case 5: return P32_2;
    case 6: return P64_5;
    default: return P32_1;
  }
}
BB_XHD uint64_t scramble(uint64_t acc, uint64_t key) { return ((acc ^ (acc >> 47)) ^ key) * P32_1; }
BB_XHD uint64_t avalanche(uint64_t h) {
  h ^= h >> 37;
  h *= PMX1;
  return h ^ (h >> 32);
}
BB_XHD uint64_t mul128_fold64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return (a * b) ^ __umul64hi(a, b);
#else
  const unsigned __int128 p = static_cast<unsigned __int128>(a) * b;
  return static_cast<uint64_t>(p) ^ static_cast<uint64_t>(p >> 64);
#endif
}
// secret words in the order the kernel wants them
constexpr uint64_t stripe_key(uint32_t stripe, uint32_t lane) { return secret64(stripe * 8 + lane * 8); }           // accumulate
constexpr uint64_t last_key(uint32_t lane) { return secret64(kSecretSize - kStripe - kLastAccStart + lane * 8); }    // last stripe
constexpr uint64_t scramble_key(uint32_t lane) { return secret64(kSecretSize - kStripe + lane * 8); }
constexpr uint64_t merge_key(uint32_t i) { return secret64(kMergeStart + i * 8); }  // i = 0..7

#if !defined(__CUDA_ARCH__)
// Reference implementation: XXH3_64bits(tile, 16384) with the default secret and seed 0.
inline uint64_t tile_hash(const uint8_t* p) {
  uint64_t acc[8];
  for (uint32_t l = 0; l < 8; ++l) acc[l] = init_acc(l);
  auto accumulate = [&](const uint8_t* stripe, uint32_t secret_off) {
    for (uint32_t i = 0; i < 8; ++i) {
      uint64_t dv;
      std::memcpy(&dv, stripe + 8 * i, 8);
      const uint64_t dk = dv ^ secret64(secret_off + 8 * i);
      acc[i ^ 1] += dv;
      acc[i] += static_cast<uint64_t>(static_cast<uint32_t>(dk)) * (dk >> 32);
    }
  };
  constexpr uint32_t nblocks = (kTileBytes - 1) / kBlock;  // 15 full blocks, each followed by a scramble
  for (uint32_t b = 0; b < nblocks; ++b) {
    for (uint32_t s = 0; s < kStripesPerBlock; ++s) accumulate(p + b * kBlock + s * kStripe, s * 8);
    for (uint32_t l = 0; l < 8; ++l) acc[l] = scramble(acc[l], scramble_key(l));
  }
  constexpr uint32_t nstripes = ((kTileBytes - 1) - kBlock * nblocks) / kStripe;  // 15
  for (uint32_t s = 0; s < nstripes; ++s) accumulate(p + nblocks * kBlock + s * kStripe, s * 8);
  accumulate(p + kTileBytes - kStripe, kSecretSize - kStripe - kLastAccStart);
  uint64_t r = static_cast<uint64_t>(kTileBytes) * P64_1;
  for (uint32_t i = 0; i < 4; ++i) r += mul128_fold64(acc[2 * i] ^ merge_key(2 * i), acc[2 * i + 1] ^ merge_key(2 * i + 1));
  return avalanche(r);
}
#endif

}  // namespace bb::xxh3
