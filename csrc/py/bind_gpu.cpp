// Bindings for the sm_90a data plane: XferEngine (fused batched transfer), comparators and
// device helpers.  Pointers cross the boundary as integers (tensor.data_ptr()), streams as
// integers (torch.cuda.current_stream().cuda_stream).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <deque>

#include "client/blackbird_client.h"
#include "fabric/gpu_fabric.h"
#include "fabric/xfer_engine.h"
#include "kernels/xfer.h"
#include "py/py_blocks.h"

namespace py = pybind11;
using namespace bb;
using namespace bb::gpu;

namespace {
void check(ErrorCode ec, const char* what) {
  if (ec != ErrorCode::OK) throw std::runtime_error(std::string(what) + ": " + std::string(to_string(ec)));
}
void check_cuda(int rc, const char* what) {
  if (rc != 0) throw std::runtime_error(std::string(what) + ": CUDA error " + std::to_string(rc) + " " + cuda_error_string(rc));
}
// Pointers given as one integer or a list of up to kMaxDst integers; returns how many.
uint32_t to_ptrs(const py::handle& h, void* (&out)[kMaxDst]) {
  if (py::isinstance<py::int_>(h)) {
    out[0] = reinterpret_cast<void*>(h.cast<uintptr_t>());
    return 1;
  }
  auto v = h.cast<std::vector<uintptr_t>>();
  if (v.size() > kMaxDst) throw py::value_error("at most 3 destinations");
  for (size_t i = 0; i < v.size(); ++i) out[i] = reinterpret_cast<void*>(v[i]);
  return static_cast<uint32_t>(v.size());
}
// A store window (common/store_window.h) given as (lo, hi) or (lo, hi, pitch, width, phase); returns whether it has the
// pattern's three numbers.
bool to_window(const py::handle& h, StoreWindow* win) {
  auto w = h.cast<std::vector<uint64_t>>();
  if (w.size() != 2 && w.size() != 5) throw py::value_error("window = (lo, hi) or (lo, hi, pitch, width, phase)");
  win->lo = w[0];
  win->hi = w[1];
  if (w.size() == 2) return false;
  win->pitch = w[2];
  win->width = w[3];
  win->phase = w[4];
  return true;
}
// What a batch's layouts point into until it has been submitted: page addresses and segment tables.
struct Keep {
  std::deque<std::vector<uint64_t>> pages;
  std::deque<std::vector<SegmentEntry>> segments;
};
// The layout slots of an item tuple (common/store_window.h), first to last: gather rows, scatter rows, source pages,
// destination pages, source blocks, destination blocks, source segments and destination segments.  Rows are given as
// (pitch, width, phase), pages as (addrs, page, phase), whose addresses are kept in `keep` until the batch has been
// submitted, blocks as a DeviceBlocks, segments as (segments, off[, unit]): the (address, units) pairs of the whole
// object in units of `unit` bytes (1 unless given; an MXFP8 transfer's are elements of its wide type), seen from object
// unit off (SourceSegments::from_segments and rebase, the table kept in `keep`).  Returns the slot set, -1 for none
// (even: the source side); an item takes one layout, so a second slot is the engine's INVALID_ARGUMENT, raised as `what`.
int to_layout(const py::tuple& t, const size_t (&slots)[8], Keep& keep, DeviceLayout* out, const char* what) {
  int set = -1;
  for (int k = 0; k < 8; ++k) {
    if (t.size() <= slots[k] || t[slots[k]].is_none()) continue;
    if (set >= 0) check(ErrorCode::INVALID_ARGUMENT, what);
    set = k;
    if (k >= 6) {
      auto g = py::cast<py::tuple>(t[slots[k]]);
      if (g.size() != 2 && g.size() != 3) throw py::value_error("segments = ([(addr, units), ...], off[, unit])");
      const uint64_t unit = g.size() == 3 ? g[2].cast<uint64_t>() : 1;
      if (unit == 0) throw py::value_error("segments: unit must be positive");
      const auto pairs = g[0].cast<std::vector<std::pair<uint64_t, uint64_t>>>();
      keep.segments.emplace_back();
      SourceSegments seg;
      uint64_t size = 0;
      check(SourceSegments::from_segments(pairs.data(), pairs.size(), &keep.segments.back(), &seg, &size, unit), what);
      *out = DeviceLayout(seg.rebase(std::min(g[1].cast<uint64_t>(), size)));
    } else if (k < 2) {
      auto g = t[slots[k]].cast<std::vector<uint64_t>>();
      if (g.size() != 3) throw py::value_error("gather / scatter = (pitch, width, phase)");
      *out = DeviceLayout(SourceRows{g[0], g[1], g[2]});
    } else if (k >= 4) {
      *out = DeviceLayout(t[slots[k]].cast<PyBlocks>().b);  // the outer array lives in the Python object until the call returns
    } else {
      auto p = py::cast<py::tuple>(t[slots[k]]);
      if (p.size() != 3 && p.size() != 5) throw py::value_error("pages = (addrs, page, phase[, row_width, row_pitch])");
      keep.pages.push_back(p[0].cast<std::vector<uint64_t>>());
      *out = DeviceLayout(SourcePages{keep.pages.back().data(), keep.pages.back().size(), p[1].cast<uint64_t>(), p[2].cast<uint64_t>(),
                                      p.size() == 5 ? p[3].cast<uint64_t>() : 0, p.size() == 5 ? p[4].cast<uint64_t>() : 0});
    }
  }
  return set;
}
// The fourteenth (run) or thirteenth (run_fp8) slot of an item tuple: the rows (pitch, width, phase) that a windowed
// get's dense result lands in, a WINDOW_ROWS layout (WindowRows).  An item takes one layout: with another one (k >= 0) it
// is INVALID_ARGUMENT.  Returns whether the slot is set.
bool to_window_rows(const py::tuple& t, size_t slot, int k, DeviceLayout* out) {
  if (t.size() <= slot || t[slot].is_none()) return false;
  if (k >= 0) check(ErrorCode::INVALID_ARGUMENT, "XferEngine: one layout per item");
  auto g = t[slot].cast<std::vector<uint64_t>>();
  if (g.size() != 3) throw py::value_error("window rows = (pitch, width, phase)");
  *out = DeviceLayout::window_rows(SourceRows{g[0], g[1], g[2]});
  return true;
}
// item tuple: (src, dst | [dst...], nbytes, expect=0, flags=0, tile_base=0, window=None, gather=None, scatter=None,
// source pages=None, destination pages=None, source blocks=None, destination blocks=None, window rows=None, source
// segments=None, destination segments=None).  An empty destination list makes a hash-only XFER_RAW_SUM descriptor (the engine rejects
// it without that flag).  A window sets XFER_WINDOW, and one with a pattern XFER_STRIDED as well.  A gather pattern
// (pitch, width, phase) sets XFER_GATHER, with src = row 0; a scatter pattern XFER_SCATTER, with dst = row 0.  Source
// pages (addrs, page, phase[, row_width, row_pitch]) set XFER_GATHER | XFER_PAGED, destination pages
// XFER_SCATTER | XFER_PAGED (with an in-page row pattern also XFER_PAGE_ROWS).  Source segments set XFER_GATHER,
// destination segments XFER_SCATTER (the engine adds XFER_SEGMENTS).  At most one layout.
XferItem to_item(const py::handle& h, Keep& keep) {
  py::tuple t = py::cast<py::tuple>(h);
  if (t.size() < 3 || t.size() > 16)
    throw py::value_error(
        "xfer item = (src, dst|[dst..], nbytes[, expect[, flags[, tile_base[, (lo, hi)[, gather (pitch, width, phase)[, scatter "
        "(pitch, width, phase)[, src pages (addrs, page, phase)[, dst pages (addrs, page, phase)]]]]]]]])");
  XferItem it;
  it.src = reinterpret_cast<const void*>(t[0].cast<uintptr_t>());
  it.ndst = to_ptrs(t[1], it.dst);
  it.nbytes = t[2].cast<uint64_t>();
  if (t.size() > 3) it.expect = t[3].cast<uint64_t>();
  if (t.size() > 4) it.flags = t[4].cast<uint32_t>();
  if (t.size() > 5) it.tile_base = t[5].cast<uint32_t>();
  if (t.size() > 6 && !t[6].is_none()) it.flags |= to_window(t[6], &it.win) ? XFER_WINDOW | XFER_STRIDED : XFER_WINDOW;
  static const uint32_t side[8] = {XFER_GATHER, XFER_SCATTER, XFER_GATHER | XFER_PAGED, XFER_SCATTER | XFER_PAGED,
                                   XFER_GATHER | XFER_PAGED, XFER_SCATTER | XFER_PAGED, XFER_GATHER, XFER_SCATTER};
  const int k = to_layout(t, {7, 8, 9, 10, 11, 12, 14, 15}, keep, &it.mem, "XferEngine.submit");
  if (k >= 0) it.flags |= side[k];
  if (to_window_rows(t, 13, k, &it.mem)) it.flags |= XFER_SCATTER;
  return it;
}
// (digests, status, device_ms), with the verdicts behind them when an item is laid out in blocks.
template <class Item>
py::tuple results(const std::vector<Item>& items, const XferResult& res) {
  for (const Item& it : items)
    if (it.mem.kind() == DeviceLayout::BLOCKS) return py::make_tuple(res.digest, res.status, res.device_ms, res.verdict);
  return py::make_tuple(res.digest, res.status, res.device_ms);
}
}  // namespace

void bind_gpu(py::module_& m) {
  m.attr("TILE_BYTES") = kTileBytes;
  m.attr("XFER_VERIFY") = static_cast<uint32_t>(XFER_VERIFY);
  m.attr("XFER_MULTIMEM") = static_cast<uint32_t>(XFER_MULTIMEM);
  m.attr("XFER_RAW_SUM") = static_cast<uint32_t>(XFER_RAW_SUM);
  m.attr("XFER_WINDOW") = static_cast<uint32_t>(XFER_WINDOW);
  m.attr("XFER_STRIDED") = static_cast<uint32_t>(XFER_STRIDED);
  m.attr("XFER_GATHER") = static_cast<uint32_t>(XFER_GATHER);
  m.attr("XFER_SCATTER") = static_cast<uint32_t>(XFER_SCATTER);
  m.attr("XFER_PAGED") = static_cast<uint32_t>(XFER_PAGED);
  m.attr("XFER_PAGE_ROWS") = static_cast<uint32_t>(XFER_PAGE_ROWS);
  m.attr("XFER_WINDOW_ROWS") = static_cast<uint32_t>(XFER_WINDOW_ROWS);
  m.attr("XFER_SEGMENTS") = static_cast<uint32_t>(XFER_SEGMENTS);
  m.def("cuda_device_count", [] {
    int n = 0;
    device_count(&n);
    return n;
  });

  py::class_<XferEngine>(m, "XferEngine")
      .def(py::init([](int device, uint32_t max_items, int slots) {
             auto r = XferEngine::create(device, max_items, slots);
             if (!r.ok()) throw std::runtime_error("XferEngine.create: " + std::string(to_string(r.error())));
             return std::move(r.value());
           }),
           py::arg("device") = 0, py::arg("max_items") = 1u << 16, py::arg("slots") = 4)
      .def("run",
           [](XferEngine& e, const py::list& items, ChecksumAlgo algo, uintptr_t stream, bool debug) {
             std::vector<XferItem> v;
             Keep keep;
             v.reserve(items.size());
             for (auto h : items) v.push_back(to_item(h, keep));
             XferResult res;
             {
               py::gil_scoped_release rel;
               auto t = e.submit(v, algo, reinterpret_cast<void*>(stream), debug);
               if (!t.ok()) check(t.error(), "XferEngine.submit");
               check(e.wait(t.value(), &res), "XferEngine.wait");
             }
             return results(v, res);
           },
           py::arg("items"), py::arg("algo") = ChecksumAlgo::BBH64, py::arg("stream") = 0, py::arg("debug") = false,
           "Runs one fused batch; items = (src, dst | [dst, ...], nbytes[, expect[, flags[, tile_base[, (lo, hi)]]]]), where [] "
           "destinations with XFER_RAW_SUM hash a slice whose first tile is tile `tile_base` of its object (digest = the "
           "unfinalised tile sum), and a window (lo, hi) sets XFER_WINDOW: the whole object is read and verified but only "
           "bytes [lo, hi) are stored, object byte x at dst + x (pass dst = buffer - lo; one destination; with "
           "ChecksumAlgo.NONE only the window's 16-byte aligned span is read).  A window (lo, hi, pitch, width, phase) also "
           "sets XFER_STRIDED: of [lo, hi), byte x is stored iff c = (x + phase) % pitch < width, at dst + ((x + phase) // "
           "pitch) * width + c.  A gather pattern (pitch, width, phase) as the eighth element sets XFER_GATHER: object byte x "
           "is read from src + ((x + phase) // width) * pitch + (x + phase) % width.  A scatter pattern (pitch, width, phase) "
           "as the ninth element (the slots before it may be None) sets XFER_SCATTER: object byte x is stored at dst + ((x + "
           "phase) // width) * pitch + (x + phase) % width.  Source pages (addrs, page, phase) as the tenth element set "
           "XFER_GATHER | XFER_PAGED: object byte x is read from addrs[(x + phase) // page] + (x + phase) % page (src is "
           "not read); destination pages as the eleventh set XFER_SCATTER | XFER_PAGED and store by the same rule (dst is "
           "not read); pages (addrs, page, phase, row_width, row_pitch) are in-page rows (SourcePages), c = (x + phase) % "
           "page at addrs[...] + (c // row_width) * row_pitch + c % row_width; source blocks (a DeviceBlocks, ids on the device) as the twelfth and destination blocks as the "
           "thirteenth do the same with a page table the resolve kernel builds on the stream.  Window rows (pitch, width, "
           "phase) as the fourteenth element, with a window, set XFER_SCATTER with a WINDOW_ROWS layout: the window's dense "
           "result (p = x - lo, or the strided window's result index) lands at dst + ((p + phase) // width) * pitch + (p + "
           "phase) % width, which the engine marks XFER_WINDOW_ROWS; returns (digests, status, "
           "device_ms), and for a batch with blocks also the verdicts, one ErrorCode per item (VALUE_OUT_OF_RANGE or "
           "INVALID_ARGUMENT for refused ids).  Source segments (pairs, off) as the fifteenth element set XFER_GATHER: "
           "the object is the (address, bytes) pairs concatenated, seen from object byte off, and object byte x is read "
           "from the segment holding off + x (src is not read); destination segments as the sixteenth set XFER_SCATTER "
           "and store by the same rule, a segment at address 0 not stored (dst is not read).  The engine marks both "
           "XFER_SEGMENTS.")
      .def("run_fp8",
           [](XferEngine& e, const py::list& items, bool unpack, uintptr_t stream, mxfp8::Wide wide) {
             std::vector<gpu::Fp8Item> v;
             Keep keep;
             for (auto h : items) {
               auto t = h.cast<py::tuple>();
               gpu::Fp8Item it;
               it.wide = reinterpret_cast<void*>(t[0].cast<uintptr_t>());
               it.wide_type = wide;
               void* packed[kMaxDst] = {nullptr, nullptr, nullptr};
               it.nreplicas = to_ptrs(t[1], packed);
               if (it.nreplicas == 0) throw py::value_error("1..3 packed objects");
               it.packed = packed[0];
               it.more_packed[0] = packed[1];
               it.more_packed[1] = packed[2];
               it.n_elems = t[2].cast<uint64_t>();
               if (t.size() < 3 || t.size() > 15)
                 throw py::value_error(
                     "fp8 item = (bf16_ptr, packed_ptr|[packed..], n_elems[, expect[, window[, gather (pitch, width, phase)[, "
                     "scatter (pitch, width, phase)[, wide[, src pages (addrs, page, phase)[, dst pages (addrs, page, phase)[, src "
                     "blocks[, dst blocks[, window rows[, src segments ([(addr, elems)], off, elem_bytes)[, dst segments]]]]]]]]]]]])");
               if (t.size() > 3 && !t[3].is_none()) it.expect = t[3].cast<uint64_t>(), it.verify = true;
               if (t.size() > 4 && !t[4].is_none()) to_window(t[4], &it.win);
               if (t.size() > 7 && !t[7].is_none()) it.wide_type = t[7].cast<mxfp8::Wide>();
               // the gather slots are a pack's, the scatter slots an unpack's
               const int k = to_layout(t, {5, 6, 8, 9, 10, 11, 13, 14}, keep, &it.mem, "XferEngine.run_fp8");
               if (k >= 0 && (k % 2 == 1) != unpack) check(ErrorCode::INVALID_ARGUMENT, "XferEngine.run_fp8");
               to_window_rows(t, 12, k, &it.mem);
               v.push_back(it);
             }
             XferResult res;
             {
               py::gil_scoped_release rel;
               check(e.run_fp8(v, unpack, reinterpret_cast<void*>(stream), &res), "XferEngine.run_fp8");
             }
             return results(v, res);
           },
           py::arg("items"), py::arg("unpack"), py::arg("stream") = 0, py::arg("wide") = mxfp8::Wide::BF16,
           "`wide` (MxWide) is the element type of every item's wide side: bf16, fp16 or fp32, unless an item gives its own as "
           "the eighth element (a batch mixing 2- and 4-byte types is INVALID_ARGUMENT); below, '2' bytes per element "
           "and '% 8' elements are those of bf16 and fp16, 4 and % 4 for fp32.  Fused MXFP8 put (unpack=False: bf16 -> packed slab object) or get (unpack=True); items = (bf16_ptr, packed_ptr "
           "| [packed_ptr, ...], n_elems[, expected_digest[, (lo, hi)]]), where a put writes every packed replica in the list "
           "(1..3) and a get reads the first.  A get with a window (lo, hi) reads and verifies the whole packed object but "
           "stores only elements [lo, hi), element x at bf16_ptr + 2x (pass bf16_ptr = buffer - 2 * lo, 16-byte aligned); a "
           "window on a put, lo > hi or hi > n_elems is INVALID_ARGUMENT.  A window (lo, hi, pitch, width, phase), in "
           "elements, is strided: of [lo, hi), element x is stored iff c = (x + phase) % pitch < width, at bf16_ptr + 2 * "
           "((x + phase) // pitch * width + c); INVALID_ARGUMENT for width == 0, width > pitch or phase >= pitch, "
           "INVALID_ADDRESS unless every row the window touches is co-aligned in bf16 bytes (the address of its first "
           "element congruent to twice that element's index mod 16).  A put's gather pattern (pitch, width, phase), in "
           "elements, as the sixth element (expected_digest and window may be None) reads the bf16 source in rows: element x "
           "is read from bf16_ptr + 2 * ((x + phase) // width * pitch + (x + phase) % width), bf16_ptr being where the "
           "pattern's row 0 starts, and the packed object and its digest are those of the compacted rows; INVALID_ARGUMENT "
           "for a pattern on a get, width == 0, width > pitch, phase >= width or pitch >= 2^62, INVALID_ADDRESS unless "
           "bf16_ptr + 2 * phase is 16-byte aligned and, when the object spans more than one row, (pitch - width) % 8 == 0.  "
           "A get's scatter pattern (pitch, width, phase), in elements, as the seventh element stores into rows by the same "
           "rule, element x at bf16_ptr + 2 * ((x + phase) // width * pitch + (x + phase) % width), under the same rules; "
           "INVALID_ARGUMENT on a put or with a window.  A put's source pages (addrs, page, phase), page and phase in "
           "elements, as the ninth element read element x from addrs[(x + phase) // page] + 2 * ((x + phase) % page) "
           "(bf16_ptr is not read); a get's destination pages as the tenth store by the same rule.  INVALID_ARGUMENT for "
           "pages on the wrong side, with rows or a window, phase >= page or a table too short; INVALID_ADDRESS unless "
           "every page touched is co-aligned in wide bytes and, for several pages, page % 8 == 0.  A put's source blocks "
           "(DeviceBlocks, page in elements) as the eleventh element and a get's destination blocks as the twelfth take a "
           "page table the resolve kernel builds on the stream.  A get's window rows (pitch, width, phase), in elements, as the "
           "thirteenth element store the window's dense result into rows by the rule of WindowRows.  A put's source segments "
           "(pairs, off, elem_bytes) as the fourteenth element read the (address, elements) pairs concatenated, seen from "
           "element off: element x from the segment holding off + x (bf16_ptr is not read); a get's destination segments "
           "as the fifteenth store by the same rule, a segment at address 0 not stored.  INVALID_ARGUMENT for segments on "
           "the wrong side, with a window, null on a put, or whose unit is not the item's element size (elem_bytes 2 for "
           "bf16 / fp16, 4 for fp32; (pairs, off) is a table of bytes, as run's); INVALID_ADDRESS unless every non-null "
           "segment's address is congruent to elem_bytes times its first element's index mod 16.  Returns (digests of the packed objects, "
           "status, device_ms), and for a batch with blocks also the verdicts, one ErrorCode per item.")
      .def_static("fp8_eligible", &XferEngine::fp8_eligible)
      .def("submit",
           [](XferEngine& e, const py::list& items, ChecksumAlgo algo, uintptr_t stream) {
             std::vector<XferItem> v;
             Keep keep;
             v.reserve(items.size());
             for (auto h : items) v.push_back(to_item(h, keep));
             auto t = e.submit(v, algo, reinterpret_cast<void*>(stream));
             if (!t.ok()) check(t.error(), "XferEngine.submit");
             return t.value();
           },
           py::arg("items"), py::arg("algo") = ChecksumAlgo::BBH64, py::arg("stream") = 0)
      .def("wait",
           [](XferEngine& e, uint64_t ticket) {
             XferResult res;
             {
               py::gil_scoped_release rel;
               check(e.wait(ticket, &res), "XferEngine.wait");
             }
             return py::make_tuple(res.digest, res.status, res.device_ms);
           })
      .def("debug_accumulators", [](XferEngine& e) { return e.debug_accumulators(); })
      .def("set_max_ctas", &XferEngine::set_max_ctas)
      .def("set_small_path", &XferEngine::set_small_path)
      .def("set_flag_completion", &XferEngine::set_flag_completion)
      .def("set_mailbox", &XferEngine::set_mailbox)
      .def_property_readonly("mailbox_requests", &XferEngine::mailbox_requests)
      .def_property_readonly("mailbox_launches", &XferEngine::mailbox_launches)
      .def_property_readonly("small_launches", &XferEngine::small_launches)
      .def("set_tile_trace", &XferEngine::set_tile_trace)
      .def("tile_trace", [](XferEngine& e) { return e.tile_trace(); }, "[tile][4] globaltimer ns: load issued, landed, store issued, slot released")
      .def_property_readonly("launches", &XferEngine::launches)
      .def_property_readonly("slots", &XferEngine::slots, "allocated slots: create()'s, plus those added for concurrent callers")
      .def_property_readonly("device", &XferEngine::device);

  m.def("copy_simt", [](uintptr_t dst, uintptr_t src, uint64_t n, uintptr_t stream) {
    check_cuda(launch_copy_simt(reinterpret_cast<void*>(dst), reinterpret_cast<const void*>(src), n,
                                reinterpret_cast<void*>(stream)), "copy_simt");
  }, py::arg("dst"), py::arg("src"), py::arg("nbytes"), py::arg("stream") = 0);
  m.def("crc32c_device", [](uintptr_t data, uint64_t n, uintptr_t out, uintptr_t scratch, uintptr_t stream) {
    check_cuda(launch_crc32c_simt(reinterpret_cast<const void*>(data), n, reinterpret_cast<uint32_t*>(out),
                                  reinterpret_cast<uint32_t*>(scratch), reinterpret_cast<void*>(stream)), "crc32c_device");
  }, py::arg("data"), py::arg("nbytes"), py::arg("out"), py::arg("scratch"), py::arg("stream") = 0,
     "Stand-alone CRC32C; scratch needs 4*ceil(nbytes/512) bytes.");
  m.def("fill", [](uintptr_t dst, uint64_t n, uint32_t v, uintptr_t stream) {
    check_cuda(launch_fill(reinterpret_cast<void*>(dst), n, v, reinterpret_cast<void*>(stream)), "fill");
  }, py::arg("dst"), py::arg("nbytes"), py::arg("value") = 0, py::arg("stream") = 0);
  m.def("random_fill", [](uintptr_t dst, uint64_t n, uint64_t seed, uintptr_t stream) {
    check_cuda(launch_random_fill(reinterpret_cast<void*>(dst), n, seed, reinterpret_cast<void*>(stream)), "random_fill");
  }, py::arg("dst"), py::arg("nbytes"), py::arg("seed") = 1, py::arg("stream") = 0);
  m.def("memcpy_peer_async", [](uintptr_t dst, int dst_dev, uintptr_t src, int src_dev, uint64_t n, uintptr_t stream) {
    check_cuda(device_memcpy_peer_async(reinterpret_cast<void*>(dst), dst_dev, reinterpret_cast<const void*>(src), src_dev, n,
                                        reinterpret_cast<void*>(stream)), "memcpy_peer_async");
  }, py::arg("dst"), py::arg("dst_device"), py::arg("src"), py::arg("src_device"), py::arg("nbytes"), py::arg("stream") = 0,
     "cudaMemcpyPeerAsync (copy engines): the naive P2P comparator of BASELINE.md section 4.");
  m.def("enable_peer_access", [](int device, int peer) { check_cuda(device_enable_peer_access(device, peer), "enable_peer_access"); });
  m.def("xfer_smem_bytes", [] { return xfer_smem_bytes(ALGO_BBH64); });
  m.def(
      "xfer_geometry",
      [](ChecksumAlgo algo, uint32_t total_tiles, int max_ctas) {
        const int a = algo == ChecksumAlgo::BBH64 ? ALGO_BBH64 : algo == ChecksumAlgo::CRC32C ? ALGO_CRC32C : algo == ChecksumAlgo::XXH3 ? ALGO_XXH3 : ALGO_NONE;
        const XferGeometry g = xfer_geometry(a, total_tiles, max_ctas);
        const int resident = xfer_resident_ctas(a);
        if (resident < 0) throw std::runtime_error("xfer_geometry: the occupancy query failed");
        py::dict d;
        d["grid"] = g.grid;
        d["stages"] = g.stages;
        d["smem_bytes"] = g.smem_bytes;
        d["resident_ctas_per_sm"] = resident;
        return d;
      },
      py::arg("algo"), py::arg("total_tiles"), py::arg("max_ctas") = 0,
      "Launch geometry of the fused kernel on the current device for a batch of total_tiles 16 KiB tiles: grid, stages, "
      "smem_bytes per CTA and resident_ctas_per_sm (occupancy query); max_ctas as XferEngine.set_max_ctas.");
  m.def("mxfp8_pack", [](uintptr_t src, uint64_t n, uintptr_t dst, uintptr_t stream, mxfp8::Wide wide) {
    check_cuda(launch_mxfp8_pack(reinterpret_cast<const void*>(src), n, reinterpret_cast<void*>(dst), reinterpret_cast<void*>(stream), wide), "mxfp8_pack");
  }, py::arg("src_bf16"), py::arg("n_elems"), py::arg("dst_packed"), py::arg("stream") = 0, py::arg("wide") = mxfp8::Wide::BF16,
     "n_elems elements of type `wide` (bf16 / fp16 / fp32, 16-byte aligned) -> [E4M3 payload | E8M0 scales]");
  m.def("mxfp8_unpack", [](uintptr_t src, uint64_t n, uintptr_t dst, uintptr_t stream, mxfp8::Wide wide) {
    check_cuda(launch_mxfp8_unpack(reinterpret_cast<const void*>(src), n, reinterpret_cast<void*>(dst), reinterpret_cast<void*>(stream), wide), "mxfp8_unpack");
  }, py::arg("src_packed"), py::arg("n_elems"), py::arg("dst_bf16"), py::arg("stream") = 0, py::arg("wide") = mxfp8::Wide::BF16,
     "packed object of n_elems elements -> n_elems elements of type `wide` (16-byte aligned)");
  m.def("xfer_fp8_smem_bytes", [](mxfp8::Wide wide) { return xfer_fp8_smem_bytes(mxfp8::wide_bytes(wide)); }, py::arg("wide") = mxfp8::Wide::BF16,
        "Dynamic shared memory per CTA of the fused MXFP8 kernel instantiation for `wide`");

  // ---- fabric: GPU tier + device transport of the client SDK
  m.def("install_gpu_backend_factory", &install_gpu_backend_factory,
        "Registers the RAM_GPU storage tier (cudaMalloc slab + CUDA IPC export) with the worker.");
  py::class_<GpuFabric, std::shared_ptr<GpuFabric>>(m, "GpuFabric")
      .def(py::init([](int device, std::shared_ptr<rpc::KeystoneApi> ks) {
             auto f = GpuFabric::create(device, std::move(ks));
             if (!f.ok()) throw std::runtime_error("GpuFabric.create: " + std::string(to_string(f.error())));
             return f.value();
           }),
           py::arg("device"), py::arg("keystone"))
      .def("refresh_pools", &GpuFabric::refresh_pools, py::call_guard<py::gil_scoped_release>())
      .def("mapped_pools", &GpuFabric::mapped_pools)
      .def("mapped_host_pools", &GpuFabric::mapped_host_pools)
      .def_property_readonly("remaps", &GpuFabric::remaps)
      .def("metrics_text", &GpuFabric::metrics_text)
      .def("path_bytes", &GpuFabric::path_bytes, py::arg("put"), py::arg("path"), "path: 0 hbm, 1 nvlink, 2 pcie, 3 nvlink multicast")
      .def_property_readonly("launches", &GpuFabric::launches)
      .def_property_readonly("last_device_ms", &GpuFabric::last_device_ms)
      .def_property_readonly("total_device_ms", &GpuFabric::total_device_ms)
      .def("set_max_ctas", [](GpuFabric& f, int n) { f.engine().set_max_ctas(n); })
      .def("set_small_path", [](GpuFabric& f, bool on) { f.engine().set_small_path(on); })
      .def("set_flag_completion", [](GpuFabric& f, bool on) { f.engine().set_flag_completion(on); })
      .def("set_mailbox", [](GpuFabric& f, bool on) { f.engine().set_mailbox(on); })
      .def_property_readonly("mailbox_requests", [](GpuFabric& f) { return f.engine().mailbox_requests(); })
      .def_property_readonly("mailbox_launches", [](GpuFabric& f) { return f.engine().mailbox_launches(); })
      .def_property_readonly("small_launches", [](GpuFabric& f) { return f.engine().small_launches(); })
      .def("set_tile_trace", [](GpuFabric& f, bool on) { f.engine().set_tile_trace(on); })
      .def("tile_trace", [](GpuFabric& f) { return f.engine().tile_trace(); })
      .def("set_arena", &GpuFabric::set_arena)
      .def_property_readonly("multicast_puts", &GpuFabric::multicast_puts);
  py::class_<NvlsArena, std::shared_ptr<NvlsArena>>(m, "NvlsArena")
      .def(py::init<int, int, int, std::string, std::vector<std::vector<int>>, uint64_t>(), py::arg("device"), py::arg("rank"), py::arg("world"),
           py::arg("tag"), py::arg("groups"), py::arg("arena_bytes"))
      .def_static("supported", &NvlsArena::supported)
      .def("phase1_create", &NvlsArena::phase1_create, py::call_guard<py::gil_scoped_release>())
      .def("phase2_join", &NvlsArena::phase2_join, py::call_guard<py::gil_scoped_release>())
      .def("phase3_bind", &NvlsArena::phase3_bind, py::call_guard<py::gil_scoped_release>())
      .def("phase4_map_peers", &NvlsArena::phase4_map_peers, py::call_guard<py::gil_scoped_release>())
      .def("num_groups", &NvlsArena::num_groups)
      .def("members", &NvlsArena::members)
      .def("member_of", &NvlsArena::member_of)
      .def_property_readonly("arena_bytes", &NvlsArena::arena_bytes)
      .def("mc_ptr", [](NvlsArena& a, size_t g) { return reinterpret_cast<uintptr_t>(a.mc_ptr(g)); })
      .def("peer_ptr", [](NvlsArena& a, size_t g, int r) { return reinterpret_cast<uintptr_t>(a.peer_ptr(g, r)); })
      .def_static("pool_id", &NvlsArena::pool_id)
      .def_static("domain", &NvlsArena::domain)
      .def_property_readonly("last_error", &NvlsArena::last_error);
  m.def("attach_fabric", [](client::BlackbirdClient& c, std::shared_ptr<GpuFabric> f) { c.set_device_transport(std::move(f)); });
}
