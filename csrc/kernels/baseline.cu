// Comparator / utility kernels: the "unfused" baseline the fused kernel must beat
// (BASELINE.md §4: unfused copy kernel + separate CRC32C kernel), L2 flush and synthetic data.
// Reference analogue: examples/benchmark_ucx_transports.cpp:83-103 times a plain memcpy.
#include <cuda_runtime.h>

#include <cstdint>

#include "common/checksum.h"
#include "kernels/ptx.cuh"
#include "kernels/xfer.h"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {
namespace {

using namespace bb::ptx;

__global__ void __launch_bounds__(256) copy_simt_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src,
                                                        uint64_t n16, uint8_t* dst_tail, const uint8_t* src_tail,
                                                        uint32_t tail) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  // 4 independent 16-byte loads in flight per thread
  for (; i + 3 * stride < n16; i += 4 * stride) {
    uint4 a = ld_nc_v4(src + i), b = ld_nc_v4(src + i + stride), c = ld_nc_v4(src + i + 2 * stride),
          d = ld_nc_v4(src + i + 3 * stride);
    st_na_v4(dst + i, a);
    st_na_v4(dst + i + stride, b);
    st_na_v4(dst + i + 2 * stride, c);
    st_na_v4(dst + i + 3 * stride, d);
  }
  for (; i < n16; i += stride) st_na_v4(dst + i, ld_nc_v4(src + i));
  if (blockIdx.x == 0 && threadIdx.x < tail) dst_tail[threadIdx.x] = src_tail[threadIdx.x];
}

__global__ void __launch_bounds__(256) fill_kernel(uint4* dst, uint64_t n16, uint32_t v) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n16; i += stride)
    dst[i] = make_uint4(v, v, v, v);
}

__device__ __forceinline__ uint64_t sm64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__global__ void __launch_bounds__(256) random_fill_kernel(uint8_t* dst, uint64_t nbytes, uint64_t seed) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t n8 = nbytes / 8;
  uint64_t* d8 = reinterpret_cast<uint64_t*>(dst);
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride)
    d8[i] = sm64(seed ^ (i * 0xD1B54A32D192ED03ull));
  if (blockIdx.x == 0 && threadIdx.x < (nbytes & 7))
    dst[n8 * 8 + threadIdx.x] = static_cast<uint8_t>(sm64(seed + threadIdx.x + 12345) & 0xFF);
}

// ---------------------------------------------------------------- stand-alone CRC32C
constexpr uint32_t kCrcChunk = 512;  // bytes per thread chunk; chunks are aligned from the END so
                                     // that the (virtually zero-prefixed) first chunk keeps the raw
                                     // remainder unchanged and every tree level has one constant.
struct CrcConsts {
  uint32_t level_xp[40];  // x^(8 * kCrcChunk * 2^L) mod P
  uint32_t init_term;     // 0xFFFFFFFF * x^(8 n) mod P
};

__constant__ uint32_t c_crc_table[4][256];  // slice-by-4 byte tables for the standard byte step

__device__ __forceinline__ uint32_t gf2_mulmod_simt(uint32_t a, uint32_t b) {
  uint32_t p = 0;
#pragma unroll 1
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = (b & 1u) ? (b >> 1) ^ 0x82F63B78u : b >> 1;
  }
  return p;
}

__global__ void __launch_bounds__(256) crc_chunks_kernel(const uint8_t* __restrict__ data, uint64_t n,
                                                         uint64_t nchunks, uint32_t* __restrict__ arr) {
  __shared__ uint32_t T[4][256];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) T[i >> 8][i & 255] = c_crc_table[i >> 8][i & 255];
  __syncthreads();
  const uint64_t pad = nchunks * kCrcChunk - n;  // virtual zero prefix
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t c = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; c < nchunks; c += stride) {
    uint32_t reg = 0;
    if (c == 0 && pad) {
      for (uint64_t b = 0; b < kCrcChunk - pad; ++b) reg = T[0][(reg ^ data[b]) & 0xFF] ^ (reg >> 8);
    } else {
      const uint8_t* p = data + c * kCrcChunk - pad;
      if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
        const uint4* q = reinterpret_cast<const uint4*>(p);
#pragma unroll 4
        for (uint32_t j = 0; j < kCrcChunk / 16; ++j) {
          const uint4 v = __ldg(q + j);
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint32_t x = reg ^ w[k];
            reg = T[3][x & 0xFF] ^ T[2][(x >> 8) & 0xFF] ^ T[1][(x >> 16) & 0xFF] ^ T[0][x >> 24];
          }
        }
      } else {
        for (uint32_t b = 0; b < kCrcChunk; ++b) reg = T[0][(reg ^ p[b]) & 0xFF] ^ (reg >> 8);
      }
    }
    arr[nchunks - 1 - c] = reg;  // reverse index: j = chunks after this one
  }
}

__global__ void __launch_bounds__(1024) crc_combine_kernel(uint32_t* arr, uint64_t nchunks, CrcConsts k, uint32_t* out) {
  // arr[j] (j = distance from the end); parent = lo ^ hi * x^(8*chunk*2^L)
  uint32_t L = 0;
  for (uint64_t s = 1; s < nchunks; s <<= 1, ++L) {
    for (uint64_t lo = static_cast<uint64_t>(threadIdx.x) * 2 * s; lo + s < nchunks; lo += static_cast<uint64_t>(blockDim.x) * 2 * s)
      arr[lo] ^= gf2_mulmod_simt(arr[lo + s], k.level_xp[L]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = arr[0] ^ k.init_term ^ 0xFFFFFFFFu;
}

PerDeviceOnce g_crc_table_once;  // c_crc_table upload

}  // namespace

int launch_copy_simt(void* dst, const void* src, uint64_t nbytes, void* stream) {
  if (nbytes == 0) return 0;
  if ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) return static_cast<int>(cudaErrorMisalignedAddress);
  const uint64_t n16 = nbytes / 16;
  const uint32_t tail = static_cast<uint32_t>(nbytes & 15);
  copy_simt_kernel<<<grid_for(n16 / 4 + 1, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint4*>(dst), static_cast<const uint4*>(src), n16, static_cast<uint8_t*>(dst) + n16 * 16,
      static_cast<const uint8_t*>(src) + n16 * 16, tail);
  return static_cast<int>(cudaGetLastError());
}

int launch_fill(void* dst, uint64_t nbytes, uint32_t value, void* stream) {
  if (nbytes < 16) return 0;
  fill_kernel<<<grid_for(nbytes / 16, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<uint4*>(dst),
                                                                                           nbytes / 16, value);
  return static_cast<int>(cudaGetLastError());
}

int launch_random_fill(void* dst, uint64_t nbytes, uint64_t seed, void* stream) {
  if (nbytes == 0) return 0;
  random_fill_kernel<<<grid_for(nbytes / 8 + 1, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<uint8_t*>(dst), nbytes, seed);
  return static_cast<int>(cudaGetLastError());
}

int launch_crc32c_simt(const void* data, uint64_t nbytes, uint32_t* out, uint32_t* scratch, void* stream) {
  int dev = 0;
  if (const cudaError_t e = current_device(&dev); e != cudaSuccess) return static_cast<int>(e);
  const cudaError_t e = g_crc_table_once.run(dev, [] {
    uint32_t t[4][256];
    // byte-step tables: T[k][b] = remainder of byte b followed by k zero bytes
    for (uint32_t b = 0; b < 256; ++b) {
      uint32_t c = b;
      for (int i = 0; i < 8; ++i) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      t[0][b] = c;
    }
    for (uint32_t b = 0; b < 256; ++b)
      for (int k = 1; k < 4; ++k) t[k][b] = (t[k - 1][b] >> 8) ^ t[0][t[k - 1][b] & 0xFF];
    return cudaMemcpyToSymbol(c_crc_table, t, sizeof t);
  });
  if (e != cudaSuccess) return static_cast<int>(e);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (nbytes == 0) {
    const uint32_t zero = 0;
    return static_cast<int>(cudaMemcpyAsync(out, &zero, 4, cudaMemcpyHostToDevice, st));
  }
  const uint64_t nchunks = (nbytes + kCrcChunk - 1) / kCrcChunk;
  CrcConsts k;
  uint64_t span = kCrcChunk;
  for (int L = 0; L < 40; ++L, span <<= 1) k.level_xp[L] = gf2_xpow_bytes(span);
  k.init_term = gf2_mulmod(0xFFFFFFFFu, gf2_xpow_bytes(nbytes));
  crc_chunks_kernel<<<grid_for(nchunks, 256, 8), 256, 0, st>>>(static_cast<const uint8_t*>(data), nbytes, nchunks, scratch);
  crc_combine_kernel<<<1, 1024, 0, st>>>(scratch, nchunks, k, out);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace bb::gpu
