// Page tables from device-resident block ids: the device half of SourceBlocks (common/store_window.h), whose host
// resolve() is the reference.  The transfer engine launches it on the caller's stream after the copy of the descriptor
// table and before the transfer kernel, so it reads the ids after whatever work the caller queued to produce them, and
// the transfer kernel reads the entries it writes.
#include <cuda_runtime.h>

#include <cstdint>

#include "kernels/xfer.h"

namespace bb::gpu {
namespace {

constexpr int kResolveThreads = 512;
constexpr uint32_t kBitmapWords = static_cast<uint32_t>(kBlocksMaxDistinct / 32);  // 32 KiB of shared memory

__device__ __forceinline__ int64_t id_at(const void* p, uint32_t bytes, uint64_t k) {
  return bytes == 8 ? static_cast<const int64_t*>(p)[k] : static_cast<const int32_t*>(p)[k];
}

// Whether n values at p are pairwise distinct, all known to lie in [0, bound): one bit per value in shared memory.
// Called by the whole CTA; returns the same answer to every thread.
__device__ bool all_distinct(const void* p, uint32_t bytes, uint64_t n, uint64_t bound, uint32_t* bits, uint32_t* flag) {
  const uint32_t words = static_cast<uint32_t>((bound + 31) / 32);
  for (uint32_t w = threadIdx.x; w < words; w += blockDim.x) bits[w] = 0;
  if (threadIdx.x == 0) *flag = 0;
  __syncthreads();
  for (uint64_t k = threadIdx.x; k < n; k += blockDim.x) {
    const uint64_t x = static_cast<uint64_t>(id_at(p, bytes, k));
    const uint32_t bit = 1u << (x & 31);
    if (atomicOr(&bits[x >> 5], bit) & bit) *flag = 1;
  }
  __syncthreads();
  const bool ok = *flag == 0;
  __syncthreads();  // *flag is reused by the next call
  return ok;
}

__global__ void __launch_bounds__(kResolveThreads) bb_resolve_blocks_kernel(const BlocksJob* __restrict__ jobs) {
  __shared__ uint32_t bits[kBitmapWords];
  __shared__ uint32_t bad, flag;
  const BlocksJob j = jobs[blockIdx.x];
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (uint64_t k = threadIdx.x; k < j.n_ids; k += blockDim.x) {
    const int64_t x = id_at(j.ids, j.id_bytes, k);
    bool out = x < 0 || static_cast<uint64_t>(x) >= j.n_blocks;
    if (j.sel) {
      const int64_t s = id_at(j.sel, j.id_bytes, k);
      out = out || s < 0 || static_cast<uint64_t>(s) >= j.n_stored;
    }
    if (out) bad = 1;
  }
  __syncthreads();
  uint32_t verdict = bad ? kBlocksOutOfRange : kBlocksOk;
  if (verdict == kBlocksOk && j.get &&
      (!all_distinct(j.ids, j.id_bytes, j.n_ids, j.n_blocks, bits, &flag) ||
       (j.sel && !all_distinct(j.sel, j.id_bytes, j.n_ids, j.n_stored, bits, &flag))))
    verdict = kBlocksDuplicate;
  if (threadIdx.x == 0) *j.verdict = verdict;

  const uint64_t per = j.sel ? j.n_stored : j.n_ids;
  for (uint64_t t = threadIdx.x; t < j.count; t += blockDim.x) {
    const uint64_t r = j.first + t, q = r / per;
    uint64_t e = 0;
    if (verdict != kBlocksOk) e = j.get ? 0 : j.outer[q];
    else if (!j.sel) e = j.outer[q] + static_cast<uint64_t>(id_at(j.ids, j.id_bytes, r % per)) * j.stride;
    j.entries[t] = e;
  }
  if (verdict != kBlocksOk || !j.sel) return;
  __syncthreads();  // the null entries above are written before the selected ones below
  for (uint64_t i = threadIdx.x; i < j.n_outer * j.n_ids; i += blockDim.x) {
    const uint64_t q = i / j.n_ids, m = i % j.n_ids;
    const uint64_t r = q * j.n_stored + static_cast<uint64_t>(id_at(j.sel, j.id_bytes, m));
    if (r >= j.first && r - j.first < j.count)
      j.entries[r - j.first] = j.outer[q] + static_cast<uint64_t>(id_at(j.ids, j.id_bytes, m)) * j.stride;
  }
}

}  // namespace

int launch_resolve_blocks(const BlocksJob* jobs, uint32_t njobs, void* stream) {
  if (njobs == 0) return 0;
  bb_resolve_blocks_kernel<<<njobs, kResolveThreads, 0, static_cast<cudaStream_t>(stream)>>>(jobs);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace bb::gpu
