// StoreWindow: which units of an object a device get stores, and where each one lands.  This is the one statement of the
// rule; the transfer engine (XferItem, Fp8Item), the fabric's ops (DeviceShardOp, DeviceFp8Op), the client, the host
// loopback transport and the kernels' XFER_WINDOW / XFER_STRIDED descriptors (kernels/xfer.h) all follow it.  A unit is a
// byte of an object or shard, or an element of an MXFP8-packed tensor (to_bf16_bytes() turns elements into bf16 bytes).
//
// Unit x in [lo, hi) is stored iff pitch == 0 or c = (x + phase) % pitch < width.  Relative to the base the window goes
// with, it lands at
//   x                                          contiguous (pitch == 0): the base is the virtual base, where unit 0 would land;
//   (row + (x + phase) / pitch) * width + c    strided: the base is where the result's row 0 lands, so the rows land densely
//                                              and pattern row 0 is result row `row` (negative when the window starts later).
// The default window, [0, UINT64_MAX) without a pattern, is the whole object.
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

  // The window of an MXFP8 get in bf16 bytes of the unpacked object.  False for a pitch of 2^62 elements or more, whose
  // byte arithmetic could overflow.
  bool to_bf16_bytes(StoreWindow* out) const {
    if (pitch > (UINT64_MAX >> 2)) return false;
    *out = {2 * lo, 2 * hi, 2 * pitch, 2 * width, 2 * phase, row};
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

}  // namespace bb
