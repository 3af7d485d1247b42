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
// starts at pages[r], so tile byte o of it sits at pages[r] + off + phase - r * page + o.  `base` is ignored.  ROWS
// (XFER_PAGE_ROWS): the dense layout's rows are the row_width-byte in-page rows instead, n = page / row_width per page,
// row r being in-page row r % n of page r / n: tile byte o of it sits at
// pages[r / n] + (r % n) * row_pitch + off + phase - r * row_width + o.
__device__ __forceinline__ uint64_t page_entry(const XferStride& st, uint64_t r) {
  return __ldg(reinterpret_cast<const unsigned long long*>(st.pages) + r);
}
template <bool PAGED, bool ROWS = false>
__device__ __forceinline__ uint64_t row_addr(uint64_t base, uint64_t off, uint64_t r, const XferStride& st) {
  if constexpr (PAGED && ROWS) {
    const uint64_t n = st.width / st.row_width;
    return page_entry(st, r / n) + (r % n) * st.row_pitch + off + st.phase - r * st.row_width;
  } else if constexpr (PAGED) {
    return page_entry(st, r) + off + st.phase - r * st.width;
  } else {
    return row_src(base, off, r, st);
  }
}
// The width of the dense layout's rows whose segments the gathering load and scattering store move: a page, or with
// ROWS an in-page row.
template <bool PAGED, bool ROWS>
__device__ __forceinline__ uint64_t dense_row(const XferStride& st) {
  return PAGED && ROWS ? st.row_width : st.width;
}
// Segments (XFER_SEGMENTS, entry {segs, nseg, phase}): entry k of the table is the 16-byte {start, addr} of segment k,
// entry nseg's start ends the last one.
__device__ __forceinline__ uint64_t seg_start(const XferStride& st, uint64_t k) {
  return __ldg(reinterpret_cast<const unsigned long long*>(st.pages) + 2 * k);
}
// Calls f(a, g, null) for every segment of the segment table `st` that the tile of `bytes` bytes at descriptor offset
// `off` overlaps: g is its tile-relative span, tile byte o of it lives at a + o (a = addr - start + phase + off), and
// `null` marks a null segment (address 0).  The warp finds the segment holding the tile's first byte by a 32-way search (each lane loads one
// start per step, a ballot picks the last one at or before the byte), then takes the overlapping segments one per lane,
// so that a tile of thousands of short segments keeps every lane busy; a segment over many tiles is one span per tile.
// The whole warp calls it.
template <class F>
__device__ __forceinline__ void for_table_segments(uint64_t off, uint32_t bytes, const XferStride& st, uint32_t lane, F&& f) {
  constexpr uint32_t kAll = 0xffffffffu;
  const uint64_t g0 = st.phase + off, g1 = g0 + bytes;
  uint64_t k0 = 0, cnt = st.width;  // segment entries [k0, k0 + cnt) hold g0, the first at or before it
  while (cnt > 1) {
    const uint64_t step = (cnt + 31) / 32, k = k0 + lane * step;
    const uint32_t le = __ballot_sync(kAll, k < k0 + cnt && seg_start(st, k) <= g0);
    const uint32_t j = 31 - __clz(le);  // lane 0's entry always starts at or before g0
    k0 += j * step;
    cnt = min(step, cnt - j * step);
  }
  for (uint64_t b = k0;; b += 32) {
    const uint64_t k = b + lane;
    uint64_t s0 = 0;
    const bool in = k < st.width && (s0 = seg_start(st, k)) < g1;
    if (in) {
      const uint4 e = __ldg(reinterpret_cast<const uint4*>(st.pages) + k);
      const uint64_t addr = (static_cast<uint64_t>(e.w) << 32) | e.z, s1 = seg_start(st, k + 1);
      const uint32_t x0 = s0 > g0 ? static_cast<uint32_t>(s0 - g0) : 0u;
      const uint32_t x1 = static_cast<uint32_t>(min(s1, g1) - g0);
      f(addr - s0 + g0, span_parts(x0, x1), addr == 0);
    }
    if (__ballot_sync(kAll, in) != kAll) break;
  }
}
// The producer's part of a gathered tile: the row segments of the tile, one per lane, the middle bulk-loaded into `tile`
// with completion on `bar`, head and tail by plain loads and shared stores.  Returns the bytes this lane's bulk loads
// deliver; the caller sums them over the warp for the stage's expect_tx, and the calling lane still has to fence its
// shared stores for the async proxy.  PAGED: the rows are the pages of an XFER_PAGED descriptor (row_addr), or with ROWS
// their in-page rows.  SEGS: the segments of an XFER_SEGMENTS descriptor (for_table_segments) instead of rows.
template <bool PAGED = false, bool ROWS = false, bool SEGS = false>
__device__ __forceinline__ uint32_t gather_row_segments(uint8_t* tile, uint64_t* bar, uint64_t src, uint64_t off, uint32_t bytes,
                                                        const XferStride& st, uint32_t lane) {
  uint32_t tx = 0;
  auto load = [&](const uint8_t* s, const TileSpan& g) {
    if (g.a1 > g.a0) {
      ptx::bulk_g2s(tile + g.a0, s + g.a0, g.a1 - g.a0, bar);
      tx += g.a1 - g.a0;
    }
    for (uint32_t o = g.x0; o < g.h1; ++o) tile[o] = s[o];
    for (uint32_t o = g.tb; o < g.x1; ++o) tile[o] = s[o];
  };
  if constexpr (SEGS) {
    for_table_segments(off, bytes, st, lane, [&](uint64_t a, const TileSpan& g, bool) { load(reinterpret_cast<const uint8_t*>(a), g); });
  } else {
    const uint64_t w = dense_row<PAGED, ROWS>(st);
    for_row_segments(off, 0, bytes, XferStride{{w}, w, st.phase}, lane, [&](uint64_t r, const TileSpan& g) {
      load(reinterpret_cast<const uint8_t*>(row_addr<PAGED, ROWS>(src, off, r, st)), g);
    });
  }
  return tx;
}
// The store warp's part of a scattered tile (XFER_SCATTER, destination rows `st`), the mirror of gather_row_segments: the
// tile's `bytes` object bytes from `off`, in the object's dense layout {width, width, phase}, one row segment per lane,
// each stored at row_src(dst0, ...) as a TMA middle plus a byte-wise head and tail.  dst0 is the descriptor's dst[0], where
// the pattern's row 0 starts.  The calling lane still has to commit its bulk group and wait on it.  PAGED: the rows are
// the pages of an XFER_PAGED descriptor (row_addr), dst0 is not read, and a page whose entry is 0 is not stored (the null
// page of SourcePages): its lane stores nothing and still commits its empty bulk group.  ROWS: the segments are the
// pages' in-page rows, and row r's page is r / (page / row_width).  SEGS: the segments of an XFER_SEGMENTS descriptor
// (for_table_segments), a null segment's lane storing nothing as a null page's.
template <bool PAGED = false, bool ROWS = false, bool SEGS = false>
__device__ __forceinline__ void scatter_row_segments(const uint8_t* tile, uint64_t dst0, uint64_t off, uint32_t bytes,
                                                     const XferStride& st, uint32_t lane) {
  if constexpr (SEGS) {
    for_table_segments(off, bytes, st, lane, [&](uint64_t a, const TileSpan& g, bool null) {
      if (!null) store_segment(reinterpret_cast<uint8_t*>(a), tile, g);
    });
    return;
  }
  const uint64_t w = dense_row<PAGED, ROWS>(st);
  for_row_segments(off, 0, bytes, XferStride{{w}, w, st.phase}, lane, [&](uint64_t r, const TileSpan& g) {
    if (PAGED && page_entry(st, ROWS ? r / (st.width / st.row_width) : r) == 0) return;
    store_segment(reinterpret_cast<uint8_t*>(row_addr<PAGED, ROWS>(dst0, off, r, st)), tile, g);
  });
}
// The row pattern of descriptor `i` from a device table (read-only path); `rows`: with the in-page row pattern of an
// XFER_PAGE_ROWS descriptor or the destination rows of an XFER_WINDOW_ROWS one, else without (those words are not read).
__device__ __forceinline__ XferStride load_stride(const XferStride* table, uint32_t i, bool rows = false) {
  const uint64_t* e = reinterpret_cast<const uint64_t*>(&table[i]);
  if (rows) return {__ldg(e), __ldg(e + 1), __ldg(e + 2), __ldg(e + 3), __ldg(e + 4), __ldg(e + 5)};
  return {__ldg(e), __ldg(e + 1), __ldg(e + 2)};
}
// The store warp's part of a windowed scattering store (XFER_WINDOW_ROWS, entry `st`): the window's segments of the tile
// at object offset `off` -- the span [x0, x1) of a range window whose lower bound is `lo`, or with `strided` the row
// segments of the window pattern -- each cut at the destination rows (row_width / row_pitch / row_phase) and stored as a
// TMA middle plus a byte-wise head and tail.  Tile byte o of a segment has the dense index poff + o (poff = off - lo, or
// row_dst(0, ...) of its window row), and lands in destination row j = (poff + o + row_phase) / row_width at
// row_src(dst0, poff, j, rows) + o.  Every piece (a segment's part in one destination row) goes to its own lane: a range
// window's pieces directly, a strided window's through a warp prefix sum of its segments' piece counts, 32 segments at
// a time, so that neither many short window rows nor a few window rows cut into many destination rows leave lanes idle.
// The calling lane still has to commit its bulk group and wait on it.
__device__ __forceinline__ void store_window_rows(const uint8_t* tile, uint64_t dst0, uint64_t off, uint32_t x0, uint32_t x1, uint64_t lo,
                                                  bool strided, const XferStride& st, uint32_t lane) {
  const XferStride rows{{st.row_pitch}, st.row_width, st.row_phase};
  const XferStride dense{{st.row_width}, st.row_width, st.row_phase};
  if (!strided) {
    const uint64_t poff = off - lo;
    for_row_segments(poff, x0, x1, dense, lane, [&](uint64_t j, const TileSpan& g) {
      store_segment(reinterpret_cast<uint8_t*>(row_src(dst0, poff, j, rows)), tile, g);
    });
    return;
  }
  constexpr uint32_t kAll = 0xffffffffu;
  auto shfl64 = [](uint64_t v, uint32_t src) {
    return (static_cast<uint64_t>(__shfl_sync(kAll, static_cast<uint32_t>(v >> 32), src)) << 32) | __shfl_sync(kAll, static_cast<uint32_t>(v), src);
  };
  const uint64_t r0 = first_row(off, x0, st);
  const uint32_t nseg = row_count(off, x0, x1, st);
  for (uint32_t base = 0; base < nseg; base += 32) {
    // lane k describes segment base + k: its span, dense offset, first destination row and piece count
    uint32_t s0 = 0, s1 = 0, cnt = 0;
    uint64_t poff = 0, j0 = 0;
    if (base + lane < nseg) {
      const uint64_t r = r0 + base + lane;
      const TileSpan g = segment_span(off, x0, x1, r, st);
      s0 = g.x0, s1 = g.x1, poff = row_dst(0, off, r, st);
      cnt = row_count(poff, s0, s1, dense);
      j0 = first_row(poff, s0, dense);
    }
    uint32_t incl = cnt;  // inclusive prefix sum of the piece counts
    for (uint32_t d = 1; d < 32; d <<= 1) {
      const uint32_t v = __shfl_up_sync(kAll, incl, d);
      if (lane >= d) incl += v;
    }
    const uint32_t total = __shfl_sync(kAll, incl, 31), excl = incl - cnt;
    for (uint32_t t0 = 0; t0 < total; t0 += 32) {
      const uint32_t t = t0 + lane;
      uint32_t k = 0;  // the segment of piece t: how many segments end at or before it
      for (uint32_t b = 16; b; b >>= 1)
        if (__shfl_sync(kAll, incl, k + b - 1) <= t) k += b;
      const uint32_t ks0 = __shfl_sync(kAll, s0, k), ks1 = __shfl_sync(kAll, s1, k), before = __shfl_sync(kAll, excl, k);
      const uint64_t kpoff = shfl64(poff, k), kj0 = shfl64(j0, k);
      if (t < total) {
        const uint64_t j = kj0 + (t - before);
        store_segment(reinterpret_cast<uint8_t*>(row_src(dst0, kpoff, j, rows)), tile, segment_span(kpoff, ks0, ks1, j, dense));
      }
    }
  }
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
