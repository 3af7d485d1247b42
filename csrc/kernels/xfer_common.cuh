// What the data-plane kernels share: reading the XferDesc table, the split of a batch's tiles over the CTAs, 64-bit warp
// shuffles, the GF(2) multiply of the CRC32C combine, and the per-device state of the host launchers.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <mutex>

#include "kernels/ptx.cuh"
#include "kernels/xfer.h"

namespace bb::gpu {

// ---------------------------------------------------------------- descriptor table
// The 32- / 64-bit field at byte offset OFF of a descriptor read as four 16-byte words.
template <size_t OFF>
__device__ __forceinline__ uint32_t desc_u32(const uint4 (&w)[4]) {
  static_assert(OFF % 4 == 0 && OFF + 4 <= sizeof(XferDesc));
  return reinterpret_cast<const uint32_t*>(w)[OFF / 4];
}
template <size_t OFF>
__device__ __forceinline__ uint64_t desc_u64(const uint4 (&w)[4]) {
  static_assert(OFF % 8 == 0);
  return (static_cast<uint64_t>(desc_u32<OFF + 4>(w)) << 32) | desc_u32<OFF>(w);
}

// A descriptor read as words; the field positions come from XferDesc itself.
__device__ __forceinline__ XferDesc desc_from_words(const uint4 (&w)[4]) {
  static_assert(sizeof(XferDesc) == sizeof(w) && kMaxDst == 3 && sizeof(void*) == 8 && sizeof(XferDesc::nbytes) == 8);
  XferDesc d;
  d.src = reinterpret_cast<const void*>(desc_u64<offsetof(XferDesc, src)>(w));
  d.dst[0] = reinterpret_cast<void*>(desc_u64<offsetof(XferDesc, dst) + 0 * sizeof(void*)>(w));
  d.dst[1] = reinterpret_cast<void*>(desc_u64<offsetof(XferDesc, dst) + 1 * sizeof(void*)>(w));
  d.dst[2] = reinterpret_cast<void*>(desc_u64<offsetof(XferDesc, dst) + 2 * sizeof(void*)>(w));
  d.nbytes = desc_u64<offsetof(XferDesc, nbytes)>(w);
  d.first_tile = desc_u32<offsetof(XferDesc, first_tile)>(w);
  d.ndst = desc_u32<offsetof(XferDesc, ndst)>(w);
  d.expect = desc_u64<offsetof(XferDesc, expect)>(w);
  d.flags = desc_u32<offsetof(XferDesc, flags)>(w);
  d.reserved = desc_u32<offsetof(XferDesc, reserved)>(w);
  return d;
}

// The descriptor table of a launch, as a copy in the kernel parameters (PARAM: plain loads, ld.global.nc is illegal on
// the parameter space) or in device memory (read-only path).  tile_start[i] is the first tile of descriptor i and
// tile_start[ndesc] the batch's tile count; kernels that do not split objects into tiles leave it null.
template <bool PARAM>
struct DescTable {
  const XferDesc* descs;
  const uint32_t* tile_start;
  uint32_t ndesc;

  __device__ __forceinline__ uint32_t start(uint32_t i) const { return PARAM ? tile_start[i] : __ldg(&tile_start[i]); }

  // Descriptor i as four 16-byte words, for desc_from_words.
  __device__ __forceinline__ void load(uint32_t i, uint4 (&w)[4]) const {
    const uint4* q = reinterpret_cast<const uint4*>(&descs[i]);
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = PARAM ? q[k] : __ldg(q + k);
  }
  __device__ __forceinline__ XferDesc operator[](uint32_t i) const {
    uint4 w[4];
    load(i, w);
    return desc_from_words(w);
  }

  // The descriptor holding tile t: start(i) <= t < start(i + 1).
  __device__ __forceinline__ uint32_t desc_of_tile(uint32_t t) const {
    uint32_t lo = 0, hi = ndesc;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (start(mid) <= t) lo = mid; else hi = mid;
    }
    return lo;
  }
};

// (t0, n): this CTA's contiguous run of tiles [t0, t0 + n) when a batch of total_tiles is split evenly over the grid.
__device__ __forceinline__ uint2 cta_tile_run(uint32_t total_tiles) {
  const uint32_t tpc = (total_tiles + gridDim.x - 1) / gridDim.x;
  const uint32_t t0 = blockIdx.x * tpc;
  return make_uint2(t0, t0 < total_tiles ? min(tpc, total_tiles - t0) : 0);
}

// ---------------------------------------------------------------- store window
// The part of one tile a store warp writes: object bytes [off, off + bytes) of the tile, cut to the store window [lo, hi)
// (object offsets) when `windowed`.  [x0, x1) is that span, tile-relative (x0 == x1: nothing to store); its 16-byte
// aligned middle [a0, a1) goes out by TMA; the head [x0, h1) and the tail [tb, x1) are under 16 bytes each and are
// stored byte-wise by lanes 0-15 and 16-31.  Without a window x0 = 0, so there is no head.
struct TileSpan {
  uint32_t x0, x1, a0, a1, h1, tb;
};
// The parts of the tile-relative span [x0, x1): aligned middle, head and tail as above.
__device__ __forceinline__ TileSpan span_parts(uint32_t x0, uint32_t x1) {
  const uint32_t a0 = (x0 + 15u) & ~15u, a1 = max(x1 & ~15u, a0);
  const uint32_t h1 = min(a0, x1), tb = max(a1, h1);
  return {x0, x1, a0, a1, h1, tb};
}
__device__ __forceinline__ TileSpan tile_span(uint64_t off, uint32_t bytes, bool windowed, uint64_t lo, uint64_t hi) {
  uint32_t x0 = 0, x1 = bytes;
  if (windowed) {
    x0 = static_cast<uint32_t>(min(max(lo, off) - off, static_cast<uint64_t>(bytes)));
    x1 = static_cast<uint32_t>(max(min(hi, off + bytes), off) - off);
    x1 = max(x1, x0);
  }
  return span_parts(x0, x1);
}

// Strided window (XFER_STRIDED, pattern `st`): the span [x0, x1) of a tile at object offset `off` (from tile_span) holds
// rows first_row(...) .. + row_count(...) - 1 of the pattern, in part or whole.  Row r's segment is the tile-relative span
// segment_span(...) of it, stored at row_dst(...) + o for tile byte o; with co-aligned rows that address is congruent to o
// mod 16, so the segment splits into TMA middle, head and tail exactly like a window span.
__device__ __forceinline__ uint64_t first_row(uint64_t off, uint32_t x0, const XferStride& st) {
  return (off + x0 + st.phase) / st.pitch;
}
__device__ __forceinline__ uint32_t row_count(uint64_t off, uint32_t x0, uint32_t x1, const XferStride& st) {
  return x1 > x0 ? static_cast<uint32_t>((off + x1 - 1u + st.phase) / st.pitch - first_row(off, x0, st) + 1u) : 0u;
}
__device__ __forceinline__ TileSpan segment_span(uint64_t off, uint32_t x0, uint32_t x1, uint64_t r, const XferStride& st) {
  const int64_t s = static_cast<int64_t>(r * st.pitch) - static_cast<int64_t>(off + st.phase);  // row start, tile-relative
  const uint32_t s0 = static_cast<uint32_t>(min(max(s, static_cast<int64_t>(x0)), static_cast<int64_t>(x1)));
  const uint32_t s1 = static_cast<uint32_t>(min(max(s + static_cast<int64_t>(st.width), static_cast<int64_t>(s0)), static_cast<int64_t>(x1)));
  return span_parts(s0, s1);
}
// dst[0] + r * width + (off + o + phase - r * pitch): where tile byte o of row r lands, less o.
__device__ __forceinline__ uint64_t row_dst(uint64_t dst0, uint64_t off, uint64_t r, const XferStride& st) {
  return dst0 + off + st.phase - r * (st.pitch - st.width);
}
// Calls f(r, g) for every row r of pattern `st` that the span [x0, x1) of a tile at object offset `off` holds, in part or
// whole, g being that row's segment (segment_span); one row per lane (a tile can hold thousands of short rows).
template <class F>
__device__ __forceinline__ void for_row_segments(uint64_t off, uint32_t x0, uint32_t x1, const XferStride& st, uint32_t lane, F&& f) {
  const uint64_t r0 = first_row(off, x0, st);
  const uint32_t nrow = row_count(off, x0, x1, st);
  for (uint32_t k = lane; k < nrow; k += 32) {
    const uint64_t r = r0 + k;
    f(r, segment_span(off, x0, x1, r, st));
  }
}
// Stores the tile bytes of segment g at d + o for tile byte o (d + o congruent to o mod 16): the TMA middle, then the head
// and tail byte-wise.  The calling lane still has to commit its bulk group and wait on it.
__device__ __forceinline__ void store_segment(uint8_t* d, const uint8_t* tile, const TileSpan& g) {
  if (g.a1 > g.a0) ptx::bulk_s2g(d + g.a0, tile + g.a0, g.a1 - g.a0);
  for (uint32_t o = g.x0; o < g.h1; ++o) d[o] = tile[o];
  for (uint32_t o = g.tb; o < g.x1; ++o) d[o] = tile[o];
}
// The store warp's part of a strided tile: the row segments of the span [x0, x1) of `tile` (shared memory, object bytes
// [off, off + ...)), one per lane, each as a TMA middle plus a byte-wise head and tail.  dst0 is the descriptor's dst[0].
__device__ __forceinline__ void store_row_segments(const uint8_t* tile, uint64_t dst0, uint64_t off, uint32_t x0, uint32_t x1,
                                                   const XferStride& st, uint32_t lane) {
  for_row_segments(off, x0, x1, st, lane, [&](uint64_t r, const TileSpan& g) {
    store_segment(reinterpret_cast<uint8_t*>(row_dst(dst0, off, r, st)), tile, g);
  });
}
// Gathering load (XFER_GATHER, source rows `st`), the mirror of the strided store: a tile at object offset `off` of `bytes`
// bytes holds rows first_row(...) .. + row_count(...) - 1 of the object's own dense layout {width, width, phase}, and tile
// byte o of row r is read from row_src(...) + o.  With co-aligned rows that address is congruent to o mod 16, so each row
// segment splits into TMA middle, head and tail exactly like a store segment.  The scattering store (XFER_SCATTER) is the
// same map with the rows on the destination side: tile byte o of row r is stored at row_src(dst0, ...) + o.
__device__ __forceinline__ uint64_t row_src(uint64_t src, uint64_t off, uint64_t r, const XferStride& st) {
  return src + off + st.phase + r * (st.pitch - st.width);
}
// The same for a paged descriptor (XFER_PAGED, entry {pages, page, phase}): row r of the dense layout is page r, which
// starts at pages[r], so tile byte o of it sits at pages[r] + off + phase - r * page + o.  `base` is ignored.
template <bool PAGED>
__device__ __forceinline__ uint64_t row_addr(uint64_t base, uint64_t off, uint64_t r, const XferStride& st) {
  if constexpr (PAGED) return __ldg(reinterpret_cast<const unsigned long long*>(st.pages) + r) + off + st.phase - r * st.width;
  else return row_src(base, off, r, st);
}
// The producer's part of a gathered tile: the row segments of the tile, one per lane, the middle bulk-loaded into `tile`
// with completion on `bar`, head and tail by plain loads and shared stores.  Returns the bytes this lane's bulk loads
// deliver; the caller sums them over the warp for the stage's expect_tx, and the calling lane still has to fence its
// shared stores for the async proxy.  PAGED: the rows are the pages of an XFER_PAGED descriptor (row_addr).
template <bool PAGED = false>
__device__ __forceinline__ uint32_t gather_row_segments(uint8_t* tile, uint64_t* bar, uint64_t src, uint64_t off, uint32_t bytes,
                                                        const XferStride& st, uint32_t lane) {
  uint32_t tx = 0;
  for_row_segments(off, 0, bytes, XferStride{{st.width}, st.width, st.phase}, lane, [&](uint64_t r, const TileSpan& g) {
    const uint8_t* s = reinterpret_cast<const uint8_t*>(row_addr<PAGED>(src, off, r, st));
    if (g.a1 > g.a0) {
      ptx::bulk_g2s(tile + g.a0, s + g.a0, g.a1 - g.a0, bar);
      tx += g.a1 - g.a0;
    }
    for (uint32_t o = g.x0; o < g.h1; ++o) tile[o] = s[o];
    for (uint32_t o = g.tb; o < g.x1; ++o) tile[o] = s[o];
  });
  return tx;
}
// The store warp's part of a scattered tile (XFER_SCATTER, destination rows `st`), the mirror of gather_row_segments: the
// tile's `bytes` object bytes from `off`, in the object's dense layout {width, width, phase}, one row segment per lane,
// each stored at row_src(dst0, ...) as a TMA middle plus a byte-wise head and tail.  dst0 is the descriptor's dst[0], where
// the pattern's row 0 starts.  The calling lane still has to commit its bulk group and wait on it.  PAGED: the rows are
// the pages of an XFER_PAGED descriptor (row_addr), dst0 is not read.
template <bool PAGED = false>
__device__ __forceinline__ void scatter_row_segments(const uint8_t* tile, uint64_t dst0, uint64_t off, uint32_t bytes,
                                                     const XferStride& st, uint32_t lane) {
  for_row_segments(off, 0, bytes, XferStride{{st.width}, st.width, st.phase}, lane, [&](uint64_t r, const TileSpan& g) {
    store_segment(reinterpret_cast<uint8_t*>(row_addr<PAGED>(dst0, off, r, st)), tile, g);
  });
}
// The row pattern of descriptor `i` from a device table (read-only path).
__device__ __forceinline__ XferStride load_stride(const XferStride* table, uint32_t i) {
  const uint64_t* e = reinterpret_cast<const uint64_t*>(&table[i]);
  return {__ldg(e), __ldg(e + 1), __ldg(e + 2)};
}

// ---------------------------------------------------------------- warp helpers
__device__ __forceinline__ uint64_t shfl_xor_u64(uint64_t v, int m) {
  const uint32_t lo = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(v), m);
  const uint32_t hi = __shfl_xor_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), m);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
  const uint32_t lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v), src);
  const uint32_t hi = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), src);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

// a * b mod P in the reflected CRC32C representation (0x80000000 == 1).
__device__ __forceinline__ uint32_t gf2_mulmod_dev(uint32_t a, uint32_t b) {
  uint32_t p = 0;
#pragma unroll 4
  for (int i = 31; i >= 0; --i) {
    p ^= ((a >> i) & 1u) ? b : 0u;
    b = (b >> 1) ^ ((b & 1u) ? 0x82F63B78u : 0u);
  }
  return p;
}

// ---------------------------------------------------------------- host: per-device launcher state
constexpr int kMaxDevices = 16;  // launchers keep their per-device state in arrays of this size

// The calling thread's current device; cudaErrorInvalidDevice if it has no slot in those arrays.
inline cudaError_t current_device(int* dev) {
  const cudaError_t e = cudaGetDevice(dev);
  if (e != cudaSuccess) return e;
  return *dev >= 0 && *dev < kMaxDevices ? cudaSuccess : cudaErrorInvalidDevice;
}

// Multiprocessor count of the current device, queried once per device; 132 (an H100 SXM) if the query fails.
inline int current_sm_count() {
  static std::atomic<int> cache[kMaxDevices];
  int dev = 0;
  if (current_device(&dev) != cudaSuccess) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// Grid of a grid-stride kernel: enough blocks of `threads` for `work_items`, at most `per_sm` per SM.
inline int grid_for(uint64_t work_items, int threads, int per_sm) {
  const uint64_t need = (work_items + threads - 1) / threads, cap = static_cast<uint64_t>(current_sm_count()) * per_sm;
  return static_cast<int>(need < 1 ? 1 : (need > cap ? cap : need));
}

// Raises KERNEL's dynamic shared-memory limit to `bytes` on device `dev`, once (a repeated call is harmless).
template <auto KERNEL>
cudaError_t set_max_dynamic_smem_once(int dev, int bytes) {
  static std::atomic<bool> done[kMaxDevices];
  if (done[dev].load(std::memory_order_acquire)) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done[dev].store(true, std::memory_order_release);
  return e;
}

// Runs a launcher's per-device set-up (its own __constant__ uploads and tables: without relocatable device code every
// translation unit has its own copy of its constants) once per device, serialised; a failed set-up returns its error
// and runs again on the next call.
class PerDeviceOnce {
 public:
  template <class F>
  cudaError_t run(int dev, F&& init) {
    std::lock_guard<std::mutex> lk(mu_);
    if (done_[dev]) return cudaSuccess;
    const cudaError_t e = init();
    if (e == cudaSuccess) done_[dev] = true;
    return e;
  }

 private:
  std::mutex mu_;
  bool done_[kMaxDevices] = {};
};

}  // namespace bb::gpu
