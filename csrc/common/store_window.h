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
// a sliced destination stores it.  SourcePages maps it onto pages at arbitrary addresses, SourceBlocks onto pages named
// by block ids in device memory, SourceSegments onto a list of segments of any sizes.  DeviceLayout, at the end, is the
// one type the other layers hold for any of them.
#pragma once
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

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

// WindowRows: a store window whose result lands in rows of a larger tensor the caller owns (a slice of a stored tensor
// read into a slice of a live one).  The units `win` selects keep their dense result index p, the position the window's
// own get gives them in a contiguous result:
//   p = x - lo                                              contiguous window
//   p = (row + (x + phase) / pitch) * width + (x + phase) % pitch   strided window
// and unit p lands at
//   dst + ((p + rows.phase) / rows.width) * rows.pitch + (p + rows.phase) % rows.width
// which is SourceRows applied to the result.  Without a pattern in `rows` the result is contiguous at dst: the window's
// own get.  This is the one statement of the rule; the transfer engine (XferItem, Fp8Item with a WINDOW_ROWS layout),
// the fabric's ops, the client, the host loopback transport and the kernels' XFER_WINDOW_ROWS descriptors
// (kernels/xfer.h) all follow it.  The unit is a byte, or for an MXFP8 get an element of the wide side until
// to_wide_bytes().
struct WindowRows {
  StoreWindow win;
  SourceRows rows;

  // The INVALID_ARGUMENT rules against an object of n units: StoreWindow::valid and SourceRows::valid.
  bool valid(uint64_t n) const { return win.valid(n) && rows.valid(); }

  // The dense result index of stored unit x.
  uint64_t index(uint64_t x) const {
    if (!win.strided()) return x - win.lo;
    const uint64_t y = x + win.phase;
    return (static_cast<uint64_t>(win.row) + y / win.pitch) * win.width + y % win.pitch;
  }
  // Where result unit p lands relative to dst.
  uint64_t at(uint64_t p) const {
    if (!rows.strided()) return p;
    const uint64_t q = p + rows.phase;
    return q / rows.width * rows.pitch + q % rows.width;
  }
  // The first and the last stored unit of an object of n units; false when the window stores none.
  bool stored_bounds(uint64_t n, uint64_t* first, uint64_t* last) const {
    const uint64_t hi = std::min(win.hi, n);
    if (win.lo >= hi) return false;
    uint64_t a = win.lo, b = hi - 1;
    if (win.strided()) {
      const uint64_t ca = (a + win.phase) % win.pitch, cb = (b + win.phase) % win.pitch;
      if (ca >= win.width) a += win.pitch - ca;
      if (cb >= win.width) {
        if (b < cb - win.width + 1) return false;
        b -= cb - win.width + 1;
      }
      if (a > b || a >= hi) return false;
    }
    *first = a, *last = b;
    return true;
  }

  // Whether every stored unit of an object of n units (in bytes) lands at an address congruent mod 16 to its object
  // offset, so that the kernels only bulk-store 16-byte congruent spans, a TMA middle plus a byte-wise head and tail per
  // segment.  The closed form: the first stored byte congruent; the gap between window rows a multiple of 16 when the
  // stored bytes span more than one window row, and the gap between destination rows when they span more than one
  // destination row.  With both gaps multiples of 16 that is exact; otherwise it may refuse a shape whose rows happen to
  // line up, which then takes the host-staged path.
  bool coaligned(uintptr_t dst, uint64_t n) const {
    uint64_t a = 0, b = 0;
    if (!stored_bounds(n, &a, &b)) return true;
    if (win.strided() && (a + win.phase) / win.pitch != (b + win.phase) / win.pitch && (win.pitch - win.width) % 16) return false;
    const uint64_t pa = index(a), pb = index(b);
    if (rows.strided() && (pa + rows.phase) / rows.width != (pb + rows.phase) / rows.width && (rows.pitch - rows.width) % 16)
      return false;
    return (dst + at(pa) - a) % 16 == 0;
  }

  // The window seen from unit `off` (off <= win.hi), clipped to [off, off + len), with its rows: unit x of the result is
  // unit off + x here and lands at the same address once dst has moved by *shift.  A contiguous window's dense index
  // starts again at the shard's first stored unit, so the rows move on by the units stored before it; a strided
  // window's index does not change.
  WindowRows rebase(uint64_t off, uint64_t len, uint64_t* shift) const {
    const uint64_t d = win.strided() ? 0 : std::min(std::max(win.lo, off), win.hi) - win.lo;
    WindowRows r{win.rebase(off, len), rows};
    r.rows = rows.rebase(d, shift);
    return r;
  }

  // The client's rule for whether a device get of this window into these rows at dst (in bytes; an MXFP8 get's after
  // to_wide_bytes()) may take the fused path as far as the shard [off, off + len) of a copy goes; the get is fused only
  // if every shard of every copy passes.  Both gaps must be multiples of 16 bytes whatever the shard holds, so that
  // whether a get is fused depends on the call's own shape and pointer, not on where the placement cut the object (as
  // StoreWindow::fused_get_aligned); then the shard must be coaligned().
  bool fused_get_aligned(uintptr_t dst, uint64_t off, uint64_t len) const {
    if ((win.strided() && (win.pitch - win.width) % 16) || (rows.strided() && (rows.pitch - rows.width) % 16)) return false;
    if (!win.touches(off, len)) return true;
    uint64_t shift = 0;
    const WindowRows r = rebase(off, len, &shift);
    return r.coaligned(dst + shift, len);
  }

  // Calls f(x, at, n) for every run of n stored units from unit x of an object of n_units that land contiguously at
  // dst + at, in order: the window's runs cut at the destination rows.
  template <class F>
  void for_each_run(uint64_t n_units, F&& f) const {
    win.for_each_run(n_units, [&](uint64_t x, uint64_t a, uint64_t n) {
      uint64_t p = win.strided() ? a : a - win.lo;
      while (n) {
        const uint64_t k = rows.strided() ? std::min(n, rows.width - (p + rows.phase) % rows.width) : n;
        f(x, at(p), k);
        x += k, p += k, n -= k;
      }
    });
  }

  // The rule in bytes of elements of `b` bytes (an MXFP8 get's wide side); false when the arithmetic could overflow.
  bool to_wide_bytes(uint64_t b, WindowRows* out) const { return win.to_wide_bytes(b, &out->win) && rows.to_wide_bytes(b, &out->rows); }

  // The rows as the kernels see them: their dense index of a strided window counts from pattern row 0, which is result
  // row `row`, so the rows move back by row * width units; *shift receives how far dst moves (modulo 2^64: the kernels
  // never dereference an address outside the rows).
  SourceRows kernel_rows(uint64_t* shift) const {
    *shift = 0;
    if (!win.strided() || !rows.strided()) return rows;
    const int64_t k = win.row * static_cast<int64_t>(win.width) + static_cast<int64_t>(rows.phase);
    const int64_t w = static_cast<int64_t>(rows.width);
    const int64_t j = k >= 0 ? k / w : -((-k + w - 1) / w);  // floor(k / w)
    *shift = static_cast<uint64_t>(j) * rows.pitch;
    return {rows.pitch, rows.width, static_cast<uint64_t>(k - j * w)};
  }
};

// SourcePages: a dense object cut into equal pages of `page` bytes that sit at arbitrary addresses (the blocks of a paged
// KV cache), on either side of a transfer: the source a device put reads from, or the destination a device get stores
// into.  A page may itself be rows inside its block (a head slice of a KV block): `row_width` bytes every `row_pitch`
// bytes, n = page / row_width rows per page.  With k = (x + phase) / page and c = (x + phase) % page, object byte x lives at
//   addrs[k] + c                                            row_width == 0 (one row per page, the default)
//   addrs[k] + (c / row_width) * row_pitch + c % row_width  an in-page row pattern
// `addrs` is a host array of npages page addresses owned by the caller.  SourceRows is the special case
// addrs[k] = src + k * pitch (with page = width).  This is the one statement of the rule; the transfer engine (XferItem,
// Fp8Item), the fabric's ops (DeviceShardOp, DeviceFp8Op), the client, the host loopback transport and the kernels'
// XFER_PAGED descriptors (kernels/xfer.h) all follow it.  page == 0 (the default) is no table.  The unit of `page`,
// `phase`, `row_width` and `row_pitch` is a byte, or for an MXFP8 transfer an element of the wide side (to_wide_bytes()
// turns elements into bytes); the addresses are byte addresses either way.  `page` stays the dense bytes of a page, so
// the pattern changes neither the object's size nor where its shards are cut.  A pattern is 0 < row_width < row_pitch
// with page % row_width == 0 and more than one row per page; from_pages() drops one whose rows touch or that has one row
// per page, which is the same memory as no pattern.
//
// An address of 0 is a null page: on the get side, the object bytes that fall in it are not stored (a partial restore
// into some of a cache's blocks).  No CUDA allocation or host buffer lives at address 0, so the marker cannot collide
// with a real page.  Null pages start and extend no run (for_each_run) and are exempt from the alignment rules
// (coaligned, fused_get_aligned); the table still covers the whole object.  A put must read every byte, so its table may
// hold no null page (has_null, DeviceLayout::valid_source).
struct SourcePages {
  const uint64_t* addrs = nullptr;
  uint64_t npages = 0, page = 0, phase = 0;
  uint64_t row_width = 0, row_pitch = 0;  // in-page row pattern; 0 / 0: one row per page

  bool paged() const { return page != 0; }
  bool has_rows() const { return row_width != 0; }
  // The in-page pattern of pages of `page` units, checked and normalised: INVALID_ARGUMENT when exactly one of *width and
  // *pitch is 0, *width > *pitch or page % *width != 0; VALUE_OUT_OF_RANGE when a page's extent,
  // (page / *width - 1) * *pitch + *width, overflows.  A pattern with one row per page or rows that touch becomes 0 / 0.  SourceBlocks::from_blocks applies it too.
  static ErrorCode page_rows(uint64_t page, uint64_t* width, uint64_t* pitch) {
    if ((*width == 0) != (*pitch == 0)) return ErrorCode::INVALID_ARGUMENT;
    if (*width == 0) return ErrorCode::OK;
    if (*width > *pitch || page % *width) return ErrorCode::INVALID_ARGUMENT;
    uint64_t e = 0;
    if (__builtin_mul_overflow(page / *width - 1, *pitch, &e) || __builtin_add_overflow(e, *width, &e)) return ErrorCode::VALUE_OUT_OF_RANGE;
    if (*width == page || *width == *pitch) *width = *pitch = 0;
    return ErrorCode::OK;
  }
  // Where in-page unit c of a page lies from the page's address.
  uint64_t in_page(uint64_t c) const { return has_rows() ? c / row_width * row_pitch + c % row_width : c; }
  // The table of an MXFP8 transfer's wide side, given in elements, in bytes of elements of `b` bytes (2 or 4): page,
  // phase and the row pattern times b, the same addresses.  False when a product overflows.
  bool to_wide_bytes(uint64_t b, SourcePages* out) const {
    *out = *this;
    return !__builtin_mul_overflow(page, b, &out->page) && !__builtin_mul_overflow(phase, b, &out->phase) &&
           !__builtin_mul_overflow(row_width, b, &out->row_width) && !__builtin_mul_overflow(row_pitch, b, &out->row_pitch);
  }
  // Pages that object bytes [0, len) touch.
  uint64_t pages_for(uint64_t len) const { return len == 0 || !paged() ? 0 : (len - 1 + phase) / page + 1; }
  // Whether the table holds every page of an object of `len` bytes, with phase < page, and its pattern is one
  // page_rows() keeps.
  bool valid(uint64_t len) const {
    return paged() && phase < page && pages_for(len) <= npages && rows_valid(page, row_width, row_pitch);
  }
  // Whether (width, pitch) is a pattern page_rows() keeps for pages of `page` units: 0 / 0, or more than one row per page
  // with gaps between them.
  static bool rows_valid(uint64_t page, uint64_t width, uint64_t pitch) {
    return width == 0 ? pitch == 0 : width < pitch && width < page && page % width == 0;
  }
  // Whether a page that object bytes [0, len) touch is null.
  bool has_null(uint64_t len) const {
    const uint64_t n = pages_for(len);
    for (uint64_t k = 0; k < n; ++k)
      if (addrs[k] == 0) return true;
    return false;
  }

  // The table of `npages` pages of `page` bytes at addrs, each page rows of row_width bytes every row_pitch bytes (0 / 0:
  // one row): an object of *size = npages * page bytes.  INVALID_ARGUMENT for page == 0 with pages and for a pattern
  // page_rows() refuses; VALUE_OUT_OF_RANGE when the product or a page's extent overflows.  No pages is a zero-byte object
  // (no table).
  static ErrorCode from_pages(uint64_t npages, uint64_t page, const uint64_t* addrs, SourcePages* out, uint64_t* size,
                              uint64_t row_width = 0, uint64_t row_pitch = 0) {
    *out = {};
    *size = 0;
    if (npages == 0) return ErrorCode::OK;
    if (page == 0) return ErrorCode::INVALID_ARGUMENT;
    if (const ErrorCode ec = page_rows(page, &row_width, &row_pitch); ec != ErrorCode::OK) return ec;
    if (__builtin_mul_overflow(npages, page, size)) return ErrorCode::VALUE_OUT_OF_RANGE;
    *out = {addrs, npages, page, 0, row_width, row_pitch};
    return ErrorCode::OK;
  }

  // The table seen from object byte `off`: byte x of the result is byte off + x here.  Shards of a striped object may
  // start mid-page, which the new phase records.
  SourcePages rebase(uint64_t off) const {
    if (!paged()) return *this;
    const uint64_t k = (phase + off) / page;
    return {addrs + std::min(k, npages), npages - std::min(k, npages), page, (phase + off) % page, row_width, row_pitch};
  }

  // Whether object bytes [0, len) are co-aligned with the tiles, so that the kernel only moves 16-byte congruent spans by
  // TMA: byte x of in-page row j of page k lives at addrs[k] + phase - k * page + j * (row_pitch - row_width) + x, so
  // addrs[k] + phase must be 16-byte aligned for every non-null page touched, the page a multiple of 16 bytes when more
  // than one page is touched, and with a pattern the gap between rows a multiple of 16 (decided by the pattern, not by
  // how many rows the span touches, as SourceRows::fused_get_aligned).  (With phase % 16 == 0, as for a table cut at
  // 16-byte shard starts, that is every page 16-byte aligned.)
  bool coaligned(uint64_t len) const {
    const uint64_t n = pages_for(len);
    if ((n > 1 && page % 16) || (n > 0 && has_rows() && (row_pitch - row_width) % 16)) return false;
    for (uint64_t k = 0; k < n; ++k)
      if (addrs[k] != 0 && (addrs[k] + phase) % 16) return false;
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
  // [addr, addr + n), in order.  One segment per page, or per in-page row with a pattern; segments that follow one
  // another in memory make one run; null pages make none and end the run before them.
  template <class F>
  void for_each_run(uint64_t len, F&& f) const {
    const uint64_t w = has_rows() ? row_width : page;
    uint64_t x = 0, run_x = 0, run_at = 0, run_n = 0;
    for (uint64_t k = 0; x < len; ++k) {
      for (uint64_t c = k == 0 ? phase : 0; c < page && x < len;) {
        const uint64_t n = std::min(w - c % w, len - x), at = addrs[k] + in_page(c);
        if (addrs[k] == 0) {
          if (run_n) f(run_x, run_at, run_n);
          run_n = 0;
        } else if (run_n && run_at + run_n == at) {
          run_n += n;
        } else {
          if (run_n) f(run_x, run_at, run_n);
          run_x = x, run_at = at, run_n = n;
        }
        x += n, c += n;
      }
    }
    if (run_n) f(run_x, run_at, run_n);
  }
};

// SourceBlocks: the pages of a paged KV cache picked by block ids that stay in device memory, on either side of a
// transfer.  The cache is n_outer outer slices (for one tensor per layer: layer-major, then each layer's outer index),
// slice q starting at the byte address outer[q]; block b of a slice lies `stride` bytes after block b - 1.  Without a
// selection the object has n_outer * n_ids pages, page r = q * n_ids + k at
//   outer[q] + ids[k] * stride
// With a selection `sel` (a partial restore, gets only) it has n_outer * n_stored pages: page q * n_stored + sel[m] is at
// outer[q] + ids[m] * stride and every other page is a null page (not stored, as SourcePages').  Object bytes then map
// onto the pages exactly as SourcePages maps them, with `page`, `phase` and the in-page row pattern (row_width,
// row_pitch: a head slice of each block) in its units; `first` is the table's first page after rebase().  `outer` is a small host array, one entry per slice; `ids` and `sel` are n_ids integers of id_bytes (4
// or 8, signed) that the host never reads on the device route: the transfer engine's resolve kernel builds the page
// table on the device (kernels/resolve_blocks.cu) and the host loopback transport calls resolve() below, the reference.
//
// The ids decide the verdict: every id in [0, n_blocks) or VALUE_OUT_OF_RANGE; for a get, ids pairwise distinct or
// INVALID_ARGUMENT; a selection's entries in [0, n_stored) and pairwise distinct, under the same two codes.  A refused
// table never leads a transfer outside the caller's cache: a get's entries are all null (nothing is stored) and a put's
// are all block 0 of their slice, outer[q] (the put is then cancelled).  Co-alignment needs no id: every address is
// outer[q] + a multiple of the stride, so coaligned() is a closed form over outer[], stride, page and the pattern.
struct SourceBlocks {
  const uint64_t* outer = nullptr;
  uint64_t n_outer = 0;
  const void* ids = nullptr;
  uint64_t n_ids = 0;
  const void* sel = nullptr;  // null: no selection
  uint64_t n_stored = 0;
  uint32_t id_bytes = 4;
  uint64_t n_blocks = 0, stride = 0, page = 0, phase = 0, first = 0;
  uint64_t row_width = 0, row_pitch = 0;  // in-page row pattern, as SourcePages'

  // Gets check duplicates in a bitmap of this many bits over n_blocks (and n_stored) in the resolve kernel's shared
  // memory; a larger bound is NOT_IMPLEMENTED on the device route.
  static constexpr uint64_t kMaxDistinct = uint64_t{1} << 18;

  bool paged() const { return page != 0; }
  uint64_t per_outer() const { return sel ? n_stored : n_ids; }
  uint64_t npages() const { return n_outer * per_outer(); }
  uint64_t pages_for(uint64_t len) const { return len == 0 || !paged() ? 0 : (len - 1 + phase) / page + 1; }
  // Whether the table holds every page of an object of `len` units from page `first`, with phase < page, and its pattern
  // is one SourcePages::page_rows keeps.
  bool valid(uint64_t len) const {
    return paged() && phase < page && (id_bytes == 4 || id_bytes == 8) && first + pages_for(len) <= npages() &&
           (n_ids == 0 || (ids && n_blocks != 0)) && (n_outer == 0 || outer) && SourcePages::rows_valid(page, row_width, row_pitch);
  }
  // A put reads every unit: no selection, whose pages may be null.
  bool has_null() const { return sel != nullptr; }
  // Whether the device route can check a get's ids for duplicates (kMaxDistinct).
  bool distinct_checkable() const { return n_blocks <= kMaxDistinct && (!sel || n_stored <= kMaxDistinct); }

  // The table of ids.size() blocks of every slice in outer[], pages of `page` units: an object of *size = n_outer *
  // per_outer() * page units.  INVALID_ARGUMENT for page == 0 with pages, a selection without stored blocks, ids of
  // another width than 4 or 8 bytes or a pattern SourcePages::page_rows refuses (which also normalises it);
  // VALUE_OUT_OF_RANGE when the size or a page's extent overflows.  No pages is a zero-unit object.
  static ErrorCode from_blocks(const SourceBlocks& b, SourceBlocks* out, uint64_t* size) {
    *out = b;
    out->first = 0, out->phase = 0;
    *size = 0;
    if ((b.id_bytes != 4 && b.id_bytes != 8) || (b.sel && b.n_stored == 0)) return ErrorCode::INVALID_ARGUMENT;
    uint64_t pages = 0;
    if (__builtin_mul_overflow(b.n_outer, out->per_outer(), &pages)) return ErrorCode::VALUE_OUT_OF_RANGE;
    if (pages == 0) return ErrorCode::OK;
    if (b.page == 0) return ErrorCode::INVALID_ARGUMENT;
    if (const ErrorCode ec = SourcePages::page_rows(b.page, &out->row_width, &out->row_pitch); ec != ErrorCode::OK) return ec;
    if (__builtin_mul_overflow(pages, b.page, size)) return ErrorCode::VALUE_OUT_OF_RANGE;
    return ErrorCode::OK;
  }
  bool has_rows() const { return row_width != 0; }

  // The table in bytes of elements of `b` bytes (an MXFP8 transfer's wide side): page, phase and the row pattern times b,
  // the same addresses and stride.  False when a product overflows.
  bool to_wide_bytes(uint64_t b, SourceBlocks* out) const {
    *out = *this;
    return !__builtin_mul_overflow(page, b, &out->page) && !__builtin_mul_overflow(phase, b, &out->phase) &&
           !__builtin_mul_overflow(row_width, b, &out->row_width) && !__builtin_mul_overflow(row_pitch, b, &out->row_pitch);
  }
  // The table seen from object unit `off`: unit x of the result is unit off + x here (as SourcePages::rebase).
  SourceBlocks rebase(uint64_t off) const {
    SourceBlocks r = *this;
    if (!paged()) return r;
    r.first = first + (phase + off) / page;
    r.phase = (phase + off) % page;
    return r;
  }
  // SourcePages::coaligned for every table the ids could make: the stride a multiple of 16 bytes, every outer[q] + phase
  // 16-byte aligned, the page a multiple of 16 when object units [0, len) touch more than one page, and with a pattern
  // the gap between rows a multiple of 16.
  bool coaligned(uint64_t len) const {
    const uint64_t n = pages_for(len);
    if (n == 0) return true;
    if ((n > 1 && page % 16) || stride % 16 || (has_rows() && (row_pitch - row_width) % 16)) return false;
    for (uint64_t q = 0; q < n_outer; ++q)
      if ((outer[q] + phase) % 16) return false;
    return true;
  }
  // The client's fused-get rule, as SourcePages::fused_get_aligned: the page a multiple of 16 whenever the object has
  // more than one page, and the shard [off, off + len) co-aligned.
  bool fused_get_aligned(uint64_t off, uint64_t len) const {
    if (npages() > 1 && page % 16) return false;
    return rebase(off).coaligned(len);
  }

  int64_t id_at(const void* p, uint64_t k) const {
    return id_bytes == 8 ? static_cast<const int64_t*>(p)[k] : static_cast<const int32_t*>(p)[k];
  }
  // The reference resolve, with ids and sel in host memory: writes the `count` page entries from page `first` into
  // table[0, count) and returns the verdict (OK, VALUE_OUT_OF_RANGE or INVALID_ARGUMENT, see above).  `get` refuses
  // duplicate ids.  Every id is checked, not only those of the pages written, so every shard of an object reaches the
  // same verdict.
  ErrorCode verdict(bool get) const {
    auto in_range = [&](const void* p, uint64_t bound) {
      for (uint64_t k = 0; k < n_ids; ++k)
        if (id_at(p, k) < 0 || static_cast<uint64_t>(id_at(p, k)) >= bound) return false;
      return true;
    };
    auto distinct = [&](const void* p, uint64_t bound) {
      std::vector<bool> seen(bound);
      for (uint64_t k = 0; k < n_ids; ++k) {
        if (seen[id_at(p, k)]) return false;
        seen[id_at(p, k)] = true;
      }
      return true;
    };
    if (!in_range(ids, n_blocks) || (sel && !in_range(sel, n_stored))) return ErrorCode::VALUE_OUT_OF_RANGE;
    if (get && (!distinct(ids, n_blocks) || (sel && !distinct(sel, n_stored)))) return ErrorCode::INVALID_ARGUMENT;
    return ErrorCode::OK;
  }
  ErrorCode resolve(uint64_t* table, uint64_t count, bool get) const {
    const ErrorCode v = verdict(get);
    const uint64_t per = per_outer();
    for (uint64_t t = 0; t < count; ++t) {
      const uint64_t r = first + t, q = r / per;
      table[t] = v != ErrorCode::OK ? (get ? 0 : outer[q]) : sel ? 0 : outer[q] + static_cast<uint64_t>(id_at(ids, r % per)) * stride;
    }
    if (v == ErrorCode::OK && sel)
      for (uint64_t q = 0; q < n_outer; ++q)
        for (uint64_t m = 0; m < n_ids; ++m) {
          const uint64_t r = q * n_stored + static_cast<uint64_t>(id_at(sel, m));
          if (r >= first && r - first < count) table[r - first] = outer[q] + static_cast<uint64_t>(id_at(ids, m)) * stride;
        }
    return v;
  }
};

// One segment of a SourceSegments table as the kernels load it, 16 bytes: the object offset of its first byte and its
// address.
struct SegmentEntry {
  uint64_t start, addr;
};
static_assert(sizeof(SegmentEntry) == 16, "one uint4 load per segment entry");

// SourceSegments: an object that is the concatenation of a list of segments of any sizes at arbitrary addresses (the
// tensors of a state_dict, a request's KV pages and SSM state), on either side of a transfer: the source a device put
// reads from, or the destination a device get stores into.  Segment k is (addr[k], len[k]) and holds object bytes
// [start[k], start[k] + len[k]), start being the exclusive prefix sum of the lengths, so object byte x lives at
//   addr[k] + (x - start[k])    for the k with start[k] <= x < start[k + 1]
// The table is `nseg` SegmentEntry {start, addr} followed by the end sentinel {total, 0}, so that entry k + 1 gives the
// end of segment k; from_segments() builds it (zero-length segments dropped, starts strictly increasing).  `phase` is
// the object byte offset of byte 0 as the holder sees it (rebase()): byte x of a rebased table is object byte phase + x.
// This is the one statement of the rule; the transfer engine (XferItem, Fp8Item), the fabric's ops (DeviceShardOp,
// DeviceFp8Op), the client, the host loopback transport and the kernels' XFER_SEGMENTS descriptors (kernels/xfer.h) all
// follow it.
//
// Units.  The table (start, phase, total()) is always in bytes.  `unit` is the bytes per unit of its callers' lengths and
// offsets: 1 for the byte calls, whose segments are (address, bytes), and b for an MXFP8 transfer, whose segments are
// (address, elements) of its wide type of b bytes (2: bf16 / fp16, 4: fp32).  from_segments() scales the lengths once;
// valid, rebase, has_null, segments_for, coaligned, fused_get_aligned and for_each_run take units; to_wide_bytes(b) is
// the same table with unit 1, no copy.  So a packed segment transfer's wide bytes are co-aligned when
// addr[k] = b * start_elem[k] (mod 16) for every non-null segment k, start_elem being its first element's object index.
//
// An address of 0 is a null segment, as SourcePages' null page: on the get side its bytes are read and verified but not
// stored (a partial restore of some tensors of a bundle); a put refuses it (has_null, DeviceLayout::valid_source).  Null
// segments start and extend no run and are exempt from the alignment rules.
struct SourceSegments {
  using Segment = std::pair<uint64_t, uint64_t>;  // (address, units)

  const SegmentEntry* entries = nullptr;  // nseg entries, then the sentinel
  uint64_t nseg = 0, phase = 0;
  uint64_t unit = 1;  // bytes per unit of the callers' lengths and offsets

  bool segmented() const { return entries != nullptr; }
  // The object's size in bytes: the sentinel's start.
  uint64_t total() const { return entries ? entries[nseg].start : 0; }

  // The table of the `count` segments at segs, each (address, units of `unit` bytes), into *table (which the result points
  // into): an object of *size units.  Zero-length segments are dropped.  VALUE_OUT_OF_RANGE when a segment's or the
  // total's bytes overflow.  No segment (or only empty ones) is a zero-unit object, with no table.
  static ErrorCode from_segments(const Segment* segs, uint64_t count, std::vector<SegmentEntry>* table, SourceSegments* out, uint64_t* size,
                                 uint64_t unit = 1) {
    *out = {};
    *size = 0;
    table->clear();
    uint64_t total = 0, bytes = 0;
    for (uint64_t k = 0; k < count; ++k) {
      if (segs[k].second == 0) continue;
      table->push_back({total, segs[k].first});
      if (__builtin_mul_overflow(segs[k].second, unit, &bytes) || __builtin_add_overflow(total, bytes, &total)) {
        table->clear();
        return ErrorCode::VALUE_OUT_OF_RANGE;
      }
    }
    if (table->empty()) return ErrorCode::OK;
    const uint64_t n = table->size();
    table->push_back({total, 0});
    *out = {table->data(), n, 0, unit};
    *size = total / unit;
    return ErrorCode::OK;
  }

  // The layout of an MXFP8 transfer's wide side, in bytes of elements of `b` bytes: the same table with unit 1.  False
  // unless its unit is b (a table of bytes, or of another wide type).
  bool to_wide_bytes(uint64_t b, SourceSegments* out) const {
    *out = *this;
    out->unit = 1;
    return unit == b;
  }

  // The segment holding unit x (x < units left): the last entry starting at or before byte phase + unit * x.
  uint64_t seg_of(uint64_t x) const {
    const uint64_t g = phase + unit * x;
    const SegmentEntry* e = std::upper_bound(entries, entries + nseg, g, [](uint64_t v, const SegmentEntry& s) { return v < s.start; });
    return e == entries ? 0 : static_cast<uint64_t>(e - entries) - 1;
  }
  // Whether the table holds units [0, len) with its entry 0 holding unit 0, the form from_segments() and rebase() keep
  // (start[0] <= phase < start[1], or phase == total() for a table rebased to its end): the kernels search from entry 0
  // and the engine copies the entries from there.
  bool valid(uint64_t len) const {
    if (!segmented() || entries[0].start > phase || phase > total() || len > (total() - phase) / unit) return false;
    return nseg == 0 ? phase == total() : phase < entries[1].start;
  }
  // Calls f(k) for every segment that units [0, len) touch, in order.
  template <class F>
  void for_each_touched(uint64_t len, F&& f) const {
    if (len == 0 || !segmented()) return;
    for (uint64_t k = seg_of(0); k < nseg && entries[k].start < phase + unit * len; ++k) f(k);
  }
  // Segments that units [0, len) touch, the first being entry 0 of a rebased table.
  uint64_t segments_for(uint64_t len) const {
    uint64_t n = 0;
    for_each_touched(len, [&](uint64_t) { ++n; });
    return n;
  }
  // Whether a segment that units [0, len) touch is null.
  bool has_null(uint64_t len) const {
    bool null = false;
    for_each_touched(len, [&](uint64_t k) { null = null || entries[k].addr == 0; });
    return null;
  }

  // The table seen from unit `off` (off <= units left): unit x of the result is unit off + x here.  Shards of a striped
  // object may start inside a segment, which the new phase records; entry 0 of the result holds its unit 0.
  SourceSegments rebase(uint64_t off) const {
    if (!segmented()) return *this;
    const uint64_t g = phase + unit * off;
    const uint64_t k = g < total() ? seg_of(off) : nseg;
    return {entries + k, nseg - k, g, unit};
  }

  // Whether units [0, len) are co-aligned with the tiles, so that the kernel only moves 16-byte congruent spans by TMA:
  // byte x of segment k lives at addr[k] - start[k] + phase + x, so addr[k] + phase - start[k] must be 16-byte aligned
  // for every non-null segment touched.  (For a shard cut at a multiple of 16 bytes that is addr[k] = start[k] mod 16.)
  bool coaligned(uint64_t len) const {
    bool ok = true;
    for_each_touched(len, [&](uint64_t k) { ok = ok && (entries[k].addr == 0 || (entries[k].addr + phase - entries[k].start) % 16 == 0); });
    return ok;
  }
  // The client's rule for whether a device get into these segments may take the fused path as far as the shard
  // [off, off + len) of a copy goes; the get is fused only if every shard of every copy passes.  As for pages, the verdict
  // is the segments' own, addr[k] = start[k] mod 16 where the object is cut at 16-byte multiples.
  bool fused_get_aligned(uint64_t off, uint64_t len) const { return rebase(off).coaligned(len); }

  // Calls f(x, addr, n) for every run of n contiguous units of units [0, len): units [x, x + n) live at bytes
  // [addr, addr + unit * n), in order.  Segments that follow one another in memory make one run; null segments make none
  // and end the run before them.
  template <class F>
  void for_each_run(uint64_t len, F&& f) const {
    uint64_t run_x = 0, run_at = 0, run_n = 0;
    auto emit = [&] {
      if (run_n) f(run_x / unit, run_at, run_n / unit);
    };
    for_each_touched(len, [&](uint64_t k) {
      const uint64_t a = std::max(entries[k].start, phase), b = std::min(entries[k + 1].start, phase + unit * len);
      const uint64_t x = a - phase, n = b - a, at = entries[k].addr + (a - entries[k].start);
      if (entries[k].addr == 0) {
        emit();
        run_n = 0;
      } else if (run_n && run_at + run_n == at) {
        run_n += n;
      } else {
        emit();
        run_x = x, run_at = at, run_n = n;
      }
    });
    emit();
  }
};

// DeviceLayout: where the caller's units of one object sit on the device side of a transfer, relative to a base address:
// contiguous (unit x at base + x, the default), in rows (SourceRows, with row 0 at the base), in pages (SourcePages,
// whose addresses are absolute: the base is not used), in blocks picked by device-resident ids (SourceBlocks, absolute
// too) or in segments of any sizes (SourceSegments, absolute too).  It is the source of a put and the destination of a
// get, in bytes, or for an MXFP8 transfer in elements of the wide side until to_wide_bytes().  This is the one place
// that knows the kinds; the transfer engine (XferItem, Fp8Item), the fabric's ops (DeviceShardOp, DeviceFp8Op), the client and the transports all hold one of these.  A
// StoreWindow goes with a contiguous layout, or with WINDOW_ROWS: rows of the window's dense result (WindowRows), which
// only a get's destination has and only the calls that take both a window and destination rows build (window_rows()).
// Its rows() are the WindowRows' rows, and the functions below that have no window treat it as the rows of a whole-object
// get (the window [0, n) without a pattern, where p = x).  A BLOCKS layout has no host copy runs (for_each_run does
// nothing for it) until resolved() has turned it into pages.
class DeviceLayout {
 public:
  enum Kind { CONTIGUOUS, ROWS, PAGES, BLOCKS, WINDOW_ROWS, SEGMENTS };

  DeviceLayout() = default;
  // Rows without a pattern, and a table without pages, are contiguous.
  explicit DeviceLayout(const SourceRows& r) : kind_(r.strided() ? ROWS : CONTIGUOUS), rows_(r) {}
  explicit DeviceLayout(const SourcePages& p) : kind_(p.paged() ? PAGES : CONTIGUOUS), pages_(p) {}
  explicit DeviceLayout(const SourceBlocks& b) : kind_(b.paged() ? BLOCKS : CONTIGUOUS), blocks_(b) {}
  explicit DeviceLayout(const SourceSegments& s) : kind_(s.segmented() ? SEGMENTS : CONTIGUOUS), segments_(s) {}
  // Rows of a windowed get's result; rows without a pattern are contiguous (the window's own get).
  static DeviceLayout window_rows(const SourceRows& r) {
    DeviceLayout l(r);
    if (r.strided()) l.kind_ = WINDOW_ROWS;
    return l;
  }
  // The same rows as the destination of a whole object, where the result index is the object offset.
  DeviceLayout as_rows() const { return kind_ == WINDOW_ROWS ? DeviceLayout(rows_) : *this; }

  // The layouts of SourceRows::from_rows and SourcePages::from_pages, with their object size and error rules.
  static ErrorCode from_rows(uint64_t width, uint64_t pitch, uint64_t rows, DeviceLayout* out, uint64_t* size, uint64_t* extent) {
    SourceRows r;
    const ErrorCode ec = SourceRows::from_rows(width, pitch, rows, &r, size, extent);
    *out = DeviceLayout(r);
    return ec;
  }
  static ErrorCode from_pages(uint64_t npages, uint64_t page, const uint64_t* addrs, DeviceLayout* out, uint64_t* size,
                              uint64_t row_width = 0, uint64_t row_pitch = 0) {
    SourcePages p;
    const ErrorCode ec = SourcePages::from_pages(npages, page, addrs, &p, size, row_width, row_pitch);
    *out = DeviceLayout(p);
    return ec;
  }

  Kind kind() const { return kind_; }
  bool contiguous() const { return kind_ == CONTIGUOUS; }
  const SourceRows& rows() const { return rows_; }     // the pattern of a ROWS or WINDOW_ROWS layout
  const SourcePages& pages() const { return pages_; }  // the table of a PAGES layout
  const SourceBlocks& blocks() const { return blocks_; }  // the description of a BLOCKS layout
  const SourceSegments& segments() const { return segments_; }  // the table of a SEGMENTS layout

  // The INVALID_ARGUMENT rules against an object of len units: a valid pattern, or a table that holds every page.
  bool valid(uint64_t len) const {
    return kind_ == ROWS || kind_ == WINDOW_ROWS ? rows_.valid()
           : kind_ == PAGES                      ? pages_.valid(len)
           : kind_ == BLOCKS                     ? blocks_.valid(len)
           : kind_ == SEGMENTS                   ? segments_.valid(len)
                                                 : true;
  }
  // The same for a put's source, which must read every unit: valid(len), no null page or segment (nor a selection of
  // blocks), and not the rows of a get's result.
  bool valid_source(uint64_t len) const {
    return valid(len) && kind_ != WINDOW_ROWS && !(kind_ == PAGES && pages_.has_null(len)) && !(kind_ == BLOCKS && blocks_.has_null()) &&
           !(kind_ == SEGMENTS && segments_.has_null(len));
  }

  // The layout of an MXFP8 transfer's wide side, given in elements, in bytes of elements of `b` bytes (2 or 4).  False
  // when the byte arithmetic could overflow, and for segments whose unit is not b.
  bool to_wide_bytes(uint64_t b, DeviceLayout* out) const {
    *out = *this;
    return kind_ == ROWS || kind_ == WINDOW_ROWS ? rows_.to_wide_bytes(b, &out->rows_)
           : kind_ == PAGES    ? pages_.to_wide_bytes(b, &out->pages_)
           : kind_ == BLOCKS   ? blocks_.to_wide_bytes(b, &out->blocks_)
           : kind_ == SEGMENTS ? segments_.to_wide_bytes(b, &out->segments_)
                               : true;
  }

  // The layout seen from object unit `off`: unit x of the result is unit off + x here, relative to a base that has moved
  // by *shift (off when contiguous, to where the new pattern's row 0 starts for rows, 0 for pages, blocks and segments).
  DeviceLayout rebase(uint64_t off, uint64_t* shift) const {
    DeviceLayout l = *this;
    *shift = off;
    if (kind_ == ROWS || kind_ == WINDOW_ROWS) l.rows_ = rows_.rebase(off, shift);
    if (kind_ == PAGES) l.pages_ = pages_.rebase(off), *shift = 0;
    if (kind_ == BLOCKS) l.blocks_ = blocks_.rebase(off), *shift = 0;
    if (kind_ == SEGMENTS) l.segments_ = segments_.rebase(off), *shift = 0;
    return l;
  }

  // Whether object bytes [0, len) at `base` are co-aligned with the tiles, so that the kernels only move 16-byte congruent
  // spans: the base 16-byte aligned when contiguous, else SourceRows::coaligned, SourcePages::coaligned,
  // SourceBlocks::coaligned or SourceSegments::coaligned.
  bool coaligned(uintptr_t base, uint64_t len) const {
    return kind_ == ROWS || kind_ == WINDOW_ROWS ? rows_.coaligned(base, len)
           : kind_ == PAGES    ? pages_.coaligned(len)
           : kind_ == BLOCKS   ? blocks_.coaligned(len)
           : kind_ == SEGMENTS ? segments_.coaligned(len)
                               : base % 16 == 0;
  }

  // The client's rule for whether a device get into this layout at `base` may take the fused path as far as the shard
  // [off, off + len) of a copy goes: a contiguous get by its store window (StoreWindow::fused_get_aligned; the default is
  // the whole object), rows, pages and segments by their own fused_get_aligned, rows of the window's result by
  // WindowRows::fused_get_aligned.
  bool fused_get_aligned(uintptr_t base, uint64_t off, uint64_t len, const StoreWindow& win = {}) const {
    if (kind_ == WINDOW_ROWS) return WindowRows{win, rows_}.fused_get_aligned(base, off, len);
    if (kind_ == ROWS) return rows_.fused_get_aligned(base, off, len);
    if (kind_ == PAGES) return pages_.fused_get_aligned(off, len);
    if (kind_ == BLOCKS) return blocks_.fused_get_aligned(off, len);
    if (kind_ == SEGMENTS) return segments_.fused_get_aligned(off, len);
    return win.fused_get_aligned(base, off, len);
  }

  // Calls f(x, addr, n) for every run of n contiguous bytes of object bytes [0, len) at `base`: object bytes [x, x + n)
  // live at [addr, addr + n), in order.
  template <class F>
  void for_each_run(uintptr_t base, uint64_t len, F&& f) const {
    if (kind_ == ROWS || kind_ == WINDOW_ROWS) rows_.for_each_run(len, [&](uint64_t x, uint64_t at, uint64_t n) { f(x, base + at, n); });
    else if (kind_ == PAGES) pages_.for_each_run(len, f);
    else if (kind_ == SEGMENTS) segments_.for_each_run(len, f);
    else if (len && kind_ == CONTIGUOUS) f(uint64_t{0}, static_cast<uint64_t>(base), len);
  }

  // The layout with host-resident ids resolved (SourceBlocks::resolve) into pages over *table, for object units
  // [0, len) of a get or a put; *verdict receives the verdict.  Other kinds come back as they are, with OK.
  DeviceLayout resolved(uint64_t len, bool get, std::vector<uint64_t>* table, ErrorCode* verdict) const {
    *verdict = ErrorCode::OK;
    if (kind_ != BLOCKS) return *this;
    table->assign(blocks_.pages_for(len), 0);
    *verdict = blocks_.resolve(table->data(), table->size(), get);
    return DeviceLayout(SourcePages{table->data(), table->size(), blocks_.page, blocks_.phase, blocks_.row_width, blocks_.row_pitch});
  }

 private:
  Kind kind_ = CONTIGUOUS;
  SourceRows rows_;
  SourcePages pages_;
  SourceBlocks blocks_;
  SourceSegments segments_;
};

}  // namespace bb
