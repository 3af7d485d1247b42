// StoreWindow: which units of an object a device get stores, and where each one lands.  This is the one statement of the
// rule; the transfer engine (XferItem, Fp8Item), the fabric's ops (DeviceShardOp, DeviceFp8Op), the client, the host
// loopback transport and the kernels' XFER_WINDOW / XFER_STRIDED descriptors (kernels/xfer.h) all follow it.  A unit is a
// byte of an object or shard, or an element of an MXFP8-packed tensor (to_wide_bytes() turns elements into bytes of its
// wide side: bf16, fp16 or fp32).
//
// Unit x in [lo, hi) is stored iff pitch == 0 or c = (x + phase) % pitch < width.  Relative to the base the window goes
// with, it lands at
//   x                                          contiguous (pitch == 0): the base is the virtual base, where unit 0 would land;
//   (row + (x + phase) / pitch) * width + c    strided: the base is where the result's row 0 lands, so the rows land densely
//                                              and pattern row 0 is result row `row` (negative when the window starts later).
// The default window, [0, UINT64_MAX) without a pattern, is the whole object.
//
// SourceRows, below, maps a dense object onto strided memory instead: where a put reads each byte from, or where a get into
// a sliced destination stores it.  SourcePages maps it onto pages at arbitrary addresses.
#pragma once
#include <algorithm>
#include <cstdint>

#include "common/error.h"

namespace bb {

struct StoreWindow {
  uint64_t lo = 0, hi = UINT64_MAX;          // units stored: [lo, hi)
  uint64_t pitch = 0, width = 0, phase = 0;  // all 0: contiguous
  int64_t row = 0;                           // strided: the result row that pattern row 0 is

  bool strided() const { return (pitch | width | phase) != 0; }
  bool whole() const { return lo == 0 && hi == UINT64_MAX && !strided(); }
  bool empty() const { return lo >= hi; }
  // Whether every unit of an object of n units is stored in place: a whole-object get, which needs no window.
  bool covers(uint64_t n) const { return lo == 0 && hi >= n && !strided(); }

  // The window of `rows` rows of `width` units every `pitch` units from `offset`, in an object of `size` units: one range
  // when there is one row or the rows touch, else a pattern whose result row 0 is the first row.  INVALID_ARGUMENT for
  // several rows wider than the pitch; VALUE_OUT_OF_RANGE when the last row passes `size` or the arithmetic overflows; OK
  // with an empty window when there is nothing to read (no rows, or rows of zero width).
  static ErrorCode from_rows(uint64_t offset, uint64_t width, uint64_t pitch, uint64_t rows, uint64_t size, StoreWindow* out) {
    uint64_t extent = width;
    if (rows != 1) {
      if (rows > 1 && width > pitch) return ErrorCode::INVALID_ARGUMENT;
      if (rows == 0 || width == 0) {
        *out = {offset, offset};
        return ErrorCode::OK;
      }
      if (__builtin_mul_overflow(rows - 1, pitch, &extent) || __builtin_add_overflow(extent, width, &extent)) return ErrorCode::VALUE_OUT_OF_RANGE;
    }
    if (offset + extent < offset || offset + extent > size) return ErrorCode::VALUE_OUT_OF_RANGE;
    *out = {offset, offset + extent};
    if (rows > 1 && width < pitch) {  // gaps between the rows: the phase puts pattern rows at the rows' starts
      out->pitch = pitch, out->width = width, out->phase = (pitch - offset % pitch) % pitch;
      out->row = -static_cast<int64_t>((offset + out->phase) / pitch);
    }
    return ErrorCode::OK;
  }

  // The window over an object of n units: the default bounds [0, UINT64_MAX) stand for [0, n).
  StoreWindow over(uint64_t n) const {
    StoreWindow w = *this;
    if (lo == 0 && hi == UINT64_MAX) w.hi = n;
    return w;
  }
  // The INVALID_ARGUMENT rules against an object of n units: lo <= hi <= n, and for a pattern 0 < width <= pitch and
  // phase < pitch.
  bool valid(uint64_t n) const { return lo <= hi && hi <= n && (!strided() || (width != 0 && width <= pitch && phase < pitch)); }

  // The window of an MXFP8 get in bytes of the unpacked object, whose elements are `b` bytes (2 or 4).  False for a pitch
  // of 2^63 / b elements or more, whose byte arithmetic could overflow.  The default bounds [0, UINT64_MAX) stay the whole
  // object only through over() first.
  bool to_wide_bytes(uint64_t b, StoreWindow* out) const {
    if (pitch > (UINT64_MAX >> 1) / b) return false;
    *out = {b * lo, b * hi, b * pitch, b * width, b * phase, row};
    return true;
  }

  // The window seen from unit `off` (off <= hi), clipped to [off, off + len): unit x of the result is unit off + x here and
  // lands at the same address once the base has moved by base_shift(off).
  StoreWindow rebase(uint64_t off, uint64_t len = UINT64_MAX) const {
    StoreWindow w = *this;
    w.lo = std::max(lo, off) - off;
    w.hi = std::min(hi - off, len);
    if (strided()) w.phase = (phase + off) % pitch, w.row = row + static_cast<int64_t>((phase + off) / pitch);
    return w;
  }
  // How far the base moves with the origin: a contiguous window's units land relative to the origin, a strided window's
  // relative to the result's row 0, which stays where it is.
  uint64_t base_shift(uint64_t off) const { return strided() ? 0 : off; }
  // Where pattern row 0 lands relative to the base: the descriptor base of the kernels, which know no `row`.
  uint64_t origin() const { return static_cast<uint64_t>(row) * width; }

  // Whether the window stores a unit of [off, off + len).  A whole window reads every unit, and every empty span too.
  bool touches(uint64_t off, uint64_t len) const {
    if (whole()) return true;
    if (!(off < hi && off + len > lo)) return false;
    if (!strided()) return true;
    const uint64_t x = std::max(off, lo), c = (x + phase) % pitch;  // in a row, or the next row starts inside the span
    return c < width || x + (pitch - c) < std::min(off + len, hi);
  }

  // Whether every row a strided window (in bytes) touches is co-aligned with the tiles, so that the kernels only
  // bulk-store 16-byte congruent spans: byte x of pattern row r lands at base + origin() + phase - r * (pitch - width) + x,
  // so that address offset must be 16-byte aligned for the window's first row, and the gap a multiple of 16 when the
  // window touches more than one row.
  bool coaligned(uintptr_t base) const {
    const uint64_t gap = pitch - width;
    const uint64_t r_lo = (lo + phase) / pitch;
    const uint64_t r_hi = hi > lo ? (hi - 1 + phase) / pitch : r_lo;
    if (r_hi > r_lo && gap % 16) return false;
    return (base + origin() + phase - r_lo * gap) % 16 == 0;
  }

  // The client's rule for whether a device get of this window (in bytes; an MXFP8 get's after to_wide_bytes()) into `ptr`,
  // where its first stored unit lands, may take the fused path as far as the shard [off, off + len) of a copy goes; the
  // get is fused only if every shard of every copy passes (an MXFP8 object is one shard, [0, 2 * n_elems)).  The kernels
  // store 16-byte aligned spans only, so the virtual base ptr - lo must be 16-byte aligned at the shard's start: at every
  // shard for a contiguous window, at the shards it touches for a strided one.  A strided window also needs a gap that is
  // a multiple of 16 bytes, even where each shard it touches holds a single row and coaligned() would pass it: so whether
  // a strided get is fused depends on its own shape and pointer, as the API documents it, not on where the placement
  // happened to cut the object.
  bool fused_get_aligned(uintptr_t ptr, uint64_t off, uint64_t len) const {
    if (strided()) {
      if ((pitch - width) % 16) return false;
      if (!touches(off, len)) return true;
    }
    return (ptr - lo + off) % 16 == 0;
  }

  // Calls f(x, at, n) for every run of n stored units from unit x of an object of n_units, landing at `at` relative to
  // the base, in order.
  template <class F>
  void for_each_run(uint64_t n_units, F&& f) const {
    const uint64_t end = std::min(hi, n_units);
    if (!strided()) {
      if (end > lo) f(lo, lo, end - lo);
      return;
    }
    for (uint64_t x = lo; x < end;) {
      const uint64_t y = x + phase, c = y % pitch;
      if (c >= width) {  // in the gap: on to the next row
        x += pitch - c;
        continue;
      }
      const uint64_t n = std::min(width - c, end - x);
      f(x, (static_cast<uint64_t>(row) + y / pitch) * width + c, n);
      x += n;
    }
  }
};

// SourceRows: where each byte of a dense object sits in strided memory, rows of `width` bytes every `pitch` bytes (a slice
// of a larger tensor), on either side of a transfer: the source a device put reads from, or the destination a device get
// stores into.  It is the inverse of a strided StoreWindow, which maps a strided object onto a dense destination: here the
// object is dense and the memory strided.  This is the one statement of the rule; the transfer engine (XferItem, Fp8Item),
// the fabric's ops (DeviceShardOp, DeviceFp8Op), the client, the host loopback transport and the kernels' XFER_GATHER and
// XFER_SCATTER descriptors (kernels/xfer.h) all follow it.  The unit is a byte, or for an MXFP8 transfer an element of the
// wide side (to_wide_bytes() turns elements into bytes of the wide type).
//
// With `src` where the pattern's row 0 starts, object byte x is read from (put) or stored at (get)
//   src + ((x + phase) / width) * pitch + (x + phase) % width
// so the rows are read or written back to back and the object holds no gaps.  pitch == 0 (the default) is contiguous
// memory: byte x at src + x.
struct SourceRows {
  uint64_t pitch = 0, width = 0, phase = 0;

  bool strided() const { return pitch != 0; }
  // 0 < width <= pitch and phase < width for a pattern.
  bool valid() const { return !strided() || (width != 0 && width <= pitch && phase < width); }

  // The rows of an MXFP8 transfer's wide side, given in elements, in bytes of elements of `b` bytes (2 or 4).  False for a
  // pitch of 2^63 / b elements or more, whose byte arithmetic could overflow (as StoreWindow::to_wide_bytes).
  bool to_wide_bytes(uint64_t b, SourceRows* out) const {
    if (pitch > (UINT64_MAX >> 1) / b) return false;
    *out = {b * pitch, b * width, b * phase};
    return true;
  }

  // The source of `rows` rows of `width` bytes every `pitch` bytes: an object of *size = rows * width bytes spread over
  // *extent = (rows - 1) * pitch + width source bytes.  INVALID_ARGUMENT for several rows wider than the pitch;
  // VALUE_OUT_OF_RANGE when either product overflows.  One row, rows that touch, no rows and rows of zero width are a
  // contiguous source (no pattern).
  static ErrorCode from_rows(uint64_t width, uint64_t pitch, uint64_t rows, SourceRows* out, uint64_t* size, uint64_t* extent) {
    *out = {};
    if (rows > 1 && width > pitch) return ErrorCode::INVALID_ARGUMENT;
    if (rows == 0 || width == 0) {
      *size = *extent = 0;
      return ErrorCode::OK;
    }
    if (__builtin_mul_overflow(rows, width, size) || __builtin_mul_overflow(rows - 1, pitch, extent) ||
        __builtin_add_overflow(*extent, width, extent))
      return ErrorCode::VALUE_OUT_OF_RANGE;
    if (rows > 1 && width < pitch) out->pitch = pitch, out->width = width;
    return ErrorCode::OK;
  }

  // The pattern seen from object byte `off`: byte x of the result is byte off + x here, read relative to a source that
  // has moved by *shift bytes (where the new pattern's row 0 starts).
  SourceRows rebase(uint64_t off, uint64_t* shift) const {
    if (!strided()) {
      *shift = off;
      return *this;
    }
    *shift = (phase + off) / width * pitch;
    return {pitch, width, (phase + off) % width};
  }

  // Source bytes from where the pattern's row 0 starts to the last byte object bytes [0, n) are read from.
  uint64_t extent(uint64_t n) const {
    if (!strided() || n == 0) return n;
    const uint64_t last = n - 1 + phase;
    return last / width * pitch + last % width + 1;
  }

  // Whether object bytes [0, len) read from `src` are co-aligned with the tiles, so that the kernel only bulk-loads 16-byte
  // congruent spans: byte x of row r is read from src + phase + r * (pitch - width) + x, so src + phase must be 16-byte
  // aligned, and the gap a multiple of 16 when the span covers more than one row.
  bool coaligned(uintptr_t src, uint64_t len) const {
    if (!strided()) return src % 16 == 0;
    if (len > 0 && (len - 1 + phase) / width > 0 && (pitch - width) % 16) return false;
    return (src + phase) % 16 == 0;
  }

  // The client's rule for whether a device get into these rows (in bytes; an MXFP8 get's after to_wide_bytes()), row 0 at
  // `dst`, may take the fused path as far as the shard [off, off + len) of a copy goes; the get is fused only if every shard
  // of every copy passes.  The shard's rows must be co-aligned from where it starts, and the gap a multiple of 16 bytes
  // even where the shard holds a single row, so that whether a get is fused depends on its own shape and pointer, not on
  // where the placement happened to cut the object (as StoreWindow::fused_get_aligned).
  bool fused_get_aligned(uintptr_t dst, uint64_t off, uint64_t len) const {
    if (strided() && (pitch - width) % 16) return false;
    uint64_t at = 0;
    const SourceRows r = rebase(off, &at);
    return r.coaligned(dst + at, len);
  }

  // Calls f(x, at, n) for every run of n contiguous source bytes of object bytes [0, len): object bytes [x, x + n) are read
  // from src + at, in order.
  template <class F>
  void for_each_run(uint64_t len, F&& f) const {
    if (!strided()) {
      if (len) f(0, 0, len);
      return;
    }
    for (uint64_t x = 0; x < len;) {
      const uint64_t y = x + phase, c = y % width, n = std::min(width - c, len - x);
      f(x, y / width * pitch + c, n);
      x += n;
    }
  }
};

// SourcePages: a dense object cut into equal pages of `page` bytes that sit at arbitrary addresses (the blocks of a paged
// KV cache), on either side of a transfer: the source a device put reads from, or the destination a device get stores
// into.  Object byte x lives at
//   addrs[(x + phase) / page] + (x + phase) % page
// `addrs` is a host array of npages page addresses owned by the caller.  SourceRows is the special case
// addrs[k] = src + k * pitch (with page = width).  This is the one statement of the rule; the transfer engine (XferItem),
// the fabric's ops (DeviceShardOp), the client, the host loopback transport and the kernel's XFER_PAGED descriptors
// (kernels/xfer.h) all follow it.  page == 0 (the default) is no table.
struct SourcePages {
  const uint64_t* addrs = nullptr;
  uint64_t npages = 0, page = 0, phase = 0;

  bool paged() const { return page != 0; }
  // Pages that object bytes [0, len) touch.
  uint64_t pages_for(uint64_t len) const { return len == 0 || !paged() ? 0 : (len - 1 + phase) / page + 1; }
  // Whether the table holds every page of an object of `len` bytes, with phase < page.
  bool valid(uint64_t len) const { return paged() && phase < page && pages_for(len) <= npages; }

  // The table of `npages` pages of `page` bytes at addrs: an object of *size = npages * page bytes.  INVALID_ARGUMENT for
  // page == 0 with pages; VALUE_OUT_OF_RANGE when the product overflows.  No pages is a zero-byte object (no table).
  static ErrorCode from_pages(uint64_t npages, uint64_t page, const uint64_t* addrs, SourcePages* out, uint64_t* size) {
    *out = {};
    *size = 0;
    if (npages == 0) return ErrorCode::OK;
    if (page == 0) return ErrorCode::INVALID_ARGUMENT;
    if (__builtin_mul_overflow(npages, page, size)) return ErrorCode::VALUE_OUT_OF_RANGE;
    *out = {addrs, npages, page, 0};
    return ErrorCode::OK;
  }

  // The table seen from object byte `off`: byte x of the result is byte off + x here.  Shards of a striped object may
  // start mid-page, which the new phase records.
  SourcePages rebase(uint64_t off) const {
    if (!paged()) return *this;
    const uint64_t k = (phase + off) / page;
    return {addrs + std::min(k, npages), npages - std::min(k, npages), page, (phase + off) % page};
  }

  // Whether object bytes [0, len) are co-aligned with the tiles, so that the kernel only moves 16-byte congruent spans by
  // TMA: byte x of page k lives at addrs[k] + phase - k * page + x, so addrs[k] + phase must be 16-byte aligned for every
  // page touched, and the page a multiple of 16 bytes when more than one page is touched.  (With phase % 16 == 0, as for
  // a table cut at 16-byte shard starts, that is every page 16-byte aligned.)
  bool coaligned(uint64_t len) const {
    const uint64_t n = pages_for(len);
    if (n > 1 && page % 16) return false;
    for (uint64_t k = 0; k < n; ++k)
      if ((addrs[k] + phase) % 16) return false;
    return true;
  }

  // The client's rule for whether a device get into these pages may take the fused path as far as the shard
  // [off, off + len) of a copy goes; the get is fused only if every shard of every copy passes.  The page must be a
  // multiple of 16 bytes whenever the table has more than one page, even where a shard touches a single page, so that
  // whether a get is fused depends on the call, not on where the placement cut the object (as
  // SourceRows::fused_get_aligned).
  bool fused_get_aligned(uint64_t off, uint64_t len) const {
    if (npages > 1 && page % 16) return false;
    return rebase(off).coaligned(len);
  }

  // Calls f(x, addr, n) for every run of n contiguous bytes of object bytes [0, len): object bytes [x, x + n) live at
  // [addr, addr + n), in order.  Pages that follow one another in memory make one run.
  template <class F>
  void for_each_run(uint64_t len, F&& f) const {
    uint64_t x = 0, run_x = 0, run_at = 0, run_n = 0;
    for (uint64_t k = 0; x < len; ++k) {
      const uint64_t c = k == 0 ? phase : 0, n = std::min(page - c, len - x), at = addrs[k] + c;
      if (run_n && run_at + run_n == at) {
        run_n += n;
      } else {
        if (run_n) f(run_x, run_at, run_n);
        run_x = x, run_at = at, run_n = n;
      }
      x += n;
    }
    if (run_n) f(run_x, run_at, run_n);
  }
};

}  // namespace bb
