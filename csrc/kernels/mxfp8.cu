// MXFP8 pack / unpack kernels (sm_90a): bf16 <-> [E4M3 payload | E8M0 block scales].
// Memory-bound grid-stride loops over the chunk codec of mxfp8.cuh (the one the fused transfer uses): one 16-byte load
// (8 bf16) per thread, 4 lanes share a 32-element block, 8-byte payload store per thread.  Destination / source may be
// peer-mapped slab memory, so the pack can write straight across NVLink.
#include <cuda_runtime.h>

#include <cstdint>

#include "kernels/mxfp8.cuh"
#include "kernels/ptx.cuh"
#include "kernels/xfer.h"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {
namespace {

__global__ void __launch_bounds__(256) mxfp8_pack_kernel(const uint4* __restrict__ src, uint64_t nblocks, uint2* __restrict__ payload,
                                                         uint8_t* __restrict__ scales) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t nchunks = nblocks * 4;
  // the trip count is padded to whole warps: pack_chunk's block max is a full-warp shuffle
  for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < ((nchunks + 31) / 32) * 32; t += stride) {
    const bool active = t < nchunks;
    const uint4 v = active ? ptx::ld_nc_v4(src + t) : make_uint4(0, 0, 0, 0);
    uint2 pay;
    uint8_t scale;
    pack_chunk(v, &pay, &scale, true);
    if (active) {
      payload[t] = pay;
      if ((t & 3) == 0) scales[t >> 2] = scale;
    }
  }
}

__global__ void __launch_bounds__(256) mxfp8_unpack_kernel(const uint2* __restrict__ payload, const uint8_t* __restrict__ scales,
                                                           uint64_t nblocks, uint4* __restrict__ dst) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t nchunks = nblocks * 4;
  for (uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < nchunks; t += stride)
    dst[t] = unpack_chunk(payload[t], scales[t >> 2]);
}

}  // namespace

int launch_mxfp8_pack(const void* src_bf16, uint64_t n_elems, void* dst_packed, void* stream) {
  if (n_elems == 0) return 0;
  if (n_elems % 32) return static_cast<int>(cudaErrorInvalidValue);
  if ((reinterpret_cast<uintptr_t>(src_bf16) & 15) || (reinterpret_cast<uintptr_t>(dst_packed) & 7)) return static_cast<int>(cudaErrorMisalignedAddress);
  const uint64_t nblocks = n_elems / 32;
  mxfp8_pack_kernel<<<grid_for(nblocks * 4, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(src_bf16), nblocks, static_cast<uint2*>(dst_packed), static_cast<uint8_t*>(dst_packed) + n_elems);
  return static_cast<int>(cudaGetLastError());
}

int launch_mxfp8_unpack(const void* src_packed, uint64_t n_elems, void* dst_bf16, void* stream) {
  if (n_elems == 0) return 0;
  if (n_elems % 32) return static_cast<int>(cudaErrorInvalidValue);
  if ((reinterpret_cast<uintptr_t>(dst_bf16) & 15) || (reinterpret_cast<uintptr_t>(src_packed) & 7)) return static_cast<int>(cudaErrorMisalignedAddress);
  const uint64_t nblocks = n_elems / 32;
  mxfp8_unpack_kernel<<<grid_for(nblocks * 4, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint2*>(src_packed), static_cast<const uint8_t*>(src_packed) + n_elems, nblocks, static_cast<uint4*>(dst_bf16));
  return static_cast<int>(cudaGetLastError());
}

}  // namespace bb::gpu
