// MXFP8 pack / unpack kernels (sm_90a): bf16 / fp16 / fp32 <-> [E4M3 payload | E8M0 block scales].
// Memory-bound grid-stride loops over the chunk codec of mxfp8.cuh (the one the fused transfer uses): one chunk of 8 elements
// (one 16-byte load, two for fp32) per thread, 4 lanes share a 32-element block, 8-byte payload store per thread.
// Destination / source may be peer-mapped slab memory, so the pack can write straight across NVLink.
#include <cuda_runtime.h>

#include <cstdint>

#include "common/mxfp8.h"
#include "kernels/mxfp8.cuh"
#include "kernels/ptx.cuh"
#include "kernels/xfer.h"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {
namespace {

// W is the wide type (mxfp8::Wide): a chunk is 8 elements, one 16-byte word of bf16 / fp16 or two of fp32.
template <mxfp8::Wide W>
__global__ void __launch_bounds__(256) mxfp8_pack_kernel(const uint4* __restrict__ src, uint64_t nblocks, uint2* __restrict__ payload,
                                                         uint8_t* __restrict__ scales) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t nchunks = nblocks * 4;
  // the trip count is padded to whole warps: pack_chunk's block max is a full-warp shuffle
  for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < ((nchunks + 31) / 32) * 32; t += stride) {
    const bool active = t < nchunks;
    uint2 pay;
    uint8_t scale;
    if constexpr (W == mxfp8::Wide::BF16) {
      const uint4 v = active ? ptx::ld_nc_v4(src + t) : make_uint4(0, 0, 0, 0);
      pack_chunk(v, &pay, &scale, true);
    } else {
      float2 f[4];
      if constexpr (W == mxfp8::Wide::F16) {
        load_f16_chunk(active ? ptx::ld_nc_v4(src + t) : make_uint4(0, 0, 0, 0), f);
      } else {
        load_f32_chunk(active ? ptx::ld_nc_v4(src + 2 * t) : make_uint4(0, 0, 0, 0),
                       active ? ptx::ld_nc_v4(src + 2 * t + 1) : make_uint4(0, 0, 0, 0), f);
      }
      pack_chunk_f32(f, &pay, &scale, true);
    }
    if (active) {
      payload[t] = pay;
      if ((t & 3) == 0) scales[t >> 2] = scale;
    }
  }
}

template <mxfp8::Wide W>
__global__ void __launch_bounds__(256) mxfp8_unpack_kernel(const uint2* __restrict__ payload, const uint8_t* __restrict__ scales,
                                                           uint64_t nblocks, uint4* __restrict__ dst) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t nchunks = nblocks * 4;
  for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < nchunks; t += stride) {
    if constexpr (W == mxfp8::Wide::BF16) dst[t] = unpack_chunk(payload[t], scales[t >> 2]);
    else unpack_wide_chunk<mxfp8::wide_bytes(W)>(payload[t], scales[t >> 2], W == mxfp8::Wide::F16, dst + mxfp8::wide_bytes(W) / 2 * t, 0);
  }
}

}  // namespace

int launch_mxfp8_pack(const void* src_wide, uint64_t n_elems, void* dst_packed, void* stream, mxfp8::Wide wide) {
  if (n_elems == 0) return 0;
  if (n_elems % 32) return static_cast<int>(cudaErrorInvalidValue);
  if ((reinterpret_cast<uintptr_t>(src_wide) & 15) || (reinterpret_cast<uintptr_t>(dst_packed) & 7)) return static_cast<int>(cudaErrorMisalignedAddress);
  const uint64_t nblocks = n_elems / 32;
  const auto* src = static_cast<const uint4*>(src_wide);
  auto* pay = static_cast<uint2*>(dst_packed);
  auto* sc = static_cast<uint8_t*>(dst_packed) + n_elems;
  const int grid = grid_for(nblocks * 4, 256, 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (wide) {
    case mxfp8::Wide::BF16: mxfp8_pack_kernel<mxfp8::Wide::BF16><<<grid, 256, 0, st>>>(src, nblocks, pay, sc); break;
    case mxfp8::Wide::F16: mxfp8_pack_kernel<mxfp8::Wide::F16><<<grid, 256, 0, st>>>(src, nblocks, pay, sc); break;
    case mxfp8::Wide::F32: mxfp8_pack_kernel<mxfp8::Wide::F32><<<grid, 256, 0, st>>>(src, nblocks, pay, sc); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  return static_cast<int>(cudaGetLastError());
}

int launch_mxfp8_unpack(const void* src_packed, uint64_t n_elems, void* dst_wide, void* stream, mxfp8::Wide wide) {
  if (n_elems == 0) return 0;
  if (n_elems % 32) return static_cast<int>(cudaErrorInvalidValue);
  if ((reinterpret_cast<uintptr_t>(dst_wide) & 15) || (reinterpret_cast<uintptr_t>(src_packed) & 7)) return static_cast<int>(cudaErrorMisalignedAddress);
  const uint64_t nblocks = n_elems / 32;
  const auto* pay = static_cast<const uint2*>(src_packed);
  const auto* sc = static_cast<const uint8_t*>(src_packed) + n_elems;
  auto* dst = static_cast<uint4*>(dst_wide);
  const int grid = grid_for(nblocks * 4, 256, 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (wide) {
    case mxfp8::Wide::BF16: mxfp8_unpack_kernel<mxfp8::Wide::BF16><<<grid, 256, 0, st>>>(pay, sc, nblocks, dst); break;
    case mxfp8::Wide::F16: mxfp8_unpack_kernel<mxfp8::Wide::F16><<<grid, 256, 0, st>>>(pay, sc, nblocks, dst); break;
    case mxfp8::Wide::F32: mxfp8_unpack_kernel<mxfp8::Wide::F32><<<grid, 256, 0, st>>>(pay, sc, nblocks, dst); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  return static_cast<int>(cudaGetLastError());
}

}  // namespace bb::gpu
