#include "fabric/xfer_engine.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>

#include "common/log.h"
#include "common/result.h"
#include "common/tchash_def.h"

namespace bb::gpu {

// Logs a failed CUDA call and returns FABRIC_ERROR.  Inside XferEngine's members `cuda_failed` is the member, which also
// keeps the code for last_cuda_error(); in the free helpers below it is the namespace-level function.
#define BB_CUDA(expr)                                                        \
  do {                                                                       \
    const cudaError_t _e = (expr);                                           \
    if (_e != cudaSuccess) return cuda_failed(static_cast<int>(_e), #expr);  \
  } while (0)

static ErrorCode cuda_failed(int code, const char* what) {
  BB_LOG(ERROR) << "CUDA error " << cudaGetErrorString(static_cast<cudaError_t>(code)) << " (" << code << ") at " << what;
  return ErrorCode::FABRIC_ERROR;
}

ErrorCode XferEngine::cuda_failed(int code, const char* what) {
  last_cuda_error_.store(code, std::memory_order_relaxed);
  return gpu::cuda_failed(code, what);
}

namespace {
// A slot's table of nd descriptors is [descs | tile_start (nd + 1) | strides (nd), only for batches with strided items |
// page entries, SEGMENTS items' segment entries and BLOCKS items' slice addresses, only for batches with paged or
// segmented items | resolve jobs, only for batches with BLOCKS items], and in the device copy only, behind it, the BLOCKS
// items' page entries, which the resolve kernel writes: the host neither fills nor copies them.  The page entries start
// 16-byte aligned, so that the kernels load a segment entry as one uint4.
size_t stride_table_offset(size_t nd) { return (nd * sizeof(XferDesc) + (nd + 1) * 4 + 7) & ~size_t{7}; }
size_t page_table_offset(size_t nd) { return (stride_table_offset(nd) + nd * sizeof(XferStride) + 15) & ~size_t{15}; }
}  // namespace

struct XferEngine::Slot {
  // How wait() learns that the batch has finished (chosen in submit()).
  enum class Completion {
    EVENTS,   // CUDA events: timing events around the launch, a completion event after the result copies
    FLAG,     // the kernel's status words in pinned memory; no event on the stream (small-object latency path)
    MAILBOX,  // served by the resident mailbox warp: results arrive in the mailbox's result ring
  };
  // host (pinned): [descs | tile_start | strides | pages | jobs], tab_bytes
  uint8_t* h_tab = nullptr;
  // device: the same, then the BLOCKS items' page entries, dtab_bytes
  uint8_t* d_tab = nullptr;
  size_t tab_bytes = 0, dtab_bytes = 0;
  uint64_t* d_sum = nullptr;
  uint32_t* d_done = nullptr;
  uint64_t* d_digest = nullptr;
  uint32_t* d_status = nullptr;
  // host (pinned) results: [digest | status | verdict], max_items each
  uint8_t* h_res = nullptr;
  uint32_t* d_debug = nullptr;
  size_t d_debug_bytes = 0;
  uint64_t* d_trace = nullptr;
  size_t d_trace_bytes = 0;
  bool traced = false;
  Completion completion = Completion::EVENTS;
  uint32_t mail_first = 0;  // MAILBOX: first sequence number of this batch in the mailbox
  void* stream = nullptr;   // FLAG: stream of the batch (fallback sync)
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_done = nullptr;
  uint64_t ticket = 0;  // 0 = free
  uint32_t nitems = 0;
  uint32_t ndesc = 0;
  uint32_t total_tiles = 0;
  bool debug = false;
  bool hashed = true;
  bool crc = false;
  uint64_t empty_digest = 0;
  std::vector<int32_t> item_to_desc;  // -1 for zero-size items
  // per descriptor up to the last XFER_STRIDED, XFER_GATHER or XFER_SCATTER one; empty when the batch has none
  std::vector<XferStride> strides;
  void set_stride(uint32_t k, const XferStride& e) {
    if (strides.size() <= k) strides.resize(k + 1, XferStride{1, 1, 0});
    strides[k] = e;
  }
  void set_stride(uint32_t k, const StoreWindow& w) { set_stride(k, XferStride{w.pitch, w.width, w.phase}); }
  // Writes the stride table behind tile_start when the batch has a strided descriptor, and returns the bytes of the
  // table to copy to the device: [descs | tile_start | strides], or without the strides.
  size_t write_strides(uint32_t nd) {
    if (strides.empty()) return static_cast<size_t>(nd) * sizeof(XferDesc) + (static_cast<size_t>(nd) + 1) * 4;
    strides.resize(nd, XferStride{1, 1, 0});
    std::memcpy(h_tab + stride_table_offset(nd), strides.data(), static_cast<size_t>(nd) * sizeof(XferStride));
    return stride_table_offset(nd) + static_cast<size_t>(nd) * sizeof(XferStride);
  }
  // The page entries of the batch's XFER_PAGED descriptors and the segment entries of its XFER_SEGMENTS ones (two words
  // each, at an even index), back to back; each one's stride entry holds the index of its first entry here until
  // write_pages() turns it into a device address.
  std::vector<uint64_t> pages;
  std::vector<uint32_t> paged_descs;
  // The resolve jobs of the batch's BLOCKS descriptors; their outer pointers hold indices into `pages`, their entries
  // (like the stride entries of blocks_descs) indices into the `reserved` device-only entries, and their verdict pointers
  // descriptor indices, until write_pages() turns them into addresses.
  std::vector<BlocksJob> jobs;
  std::vector<uint32_t> blocks_descs;
  uint64_t reserved = 0;
  void clear_layouts() {
    strides.clear();
    pages.clear();
    paged_descs.clear();
    jobs.clear();
    blocks_descs.clear();
    reserved = 0;
  }
  // The table entry of descriptor k's gathered or scattered layout (in bytes, over nbytes): its pattern, or its page
  // entries, or for blocks room for them and a resolve job (`get`: the scattering side), with the in-page row pattern of
  // either, or the segment entries its bytes touch and the sentinel after them.  Returns the XFER_PAGED flag for pages
  // and blocks (and XFER_PAGE_ROWS with a pattern), XFER_SEGMENTS for segments, 0 for rows.  O(segments), not O(tiles).
  uint32_t set_layout(uint32_t k, const DeviceLayout& m, uint64_t nbytes, bool get) {
    if (m.kind() == DeviceLayout::ROWS) {
      set_stride(k, XferStride{m.rows().pitch, m.rows().width, m.rows().phase});
      return 0;
    }
    if (m.kind() == DeviceLayout::SEGMENTS) {
      const SourceSegments& g = m.segments();  // rebased: entry 0 holds byte 0
      const uint64_t n = g.segments_for(nbytes);
      if (pages.size() % 2) pages.push_back(0);
      paged_descs.push_back(k);
      set_stride(k, XferStride{{pages.size()}, n, g.phase});
      for (uint64_t j = 0; j <= n; ++j) pages.push_back(g.entries[j].start), pages.push_back(g.entries[j].addr);
      return XFER_SEGMENTS;
    }
    if (m.kind() == DeviceLayout::PAGES) {
      const SourcePages& p = m.pages();
      paged_descs.push_back(k);
      set_stride(k, XferStride{{pages.size()}, p.page, p.phase, p.row_width, p.row_pitch});
      pages.insert(pages.end(), p.addrs, p.addrs + p.pages_for(nbytes));
      return p.has_rows() ? XFER_PAGED | XFER_PAGE_ROWS : XFER_PAGED;
    }
    const SourceBlocks& b = m.blocks();
    BlocksJob j{};
    blocks_descs.push_back(k);
    set_stride(k, XferStride{{reserved}, b.page, b.phase, b.row_width, b.row_pitch});
    j.entries = reinterpret_cast<uint64_t*>(reserved);
    j.count = b.pages_for(nbytes);
    reserved += j.count;
    j.outer = reinterpret_cast<const uint64_t*>(pages.size());
    pages.insert(pages.end(), b.outer, b.outer + b.n_outer);
    j.ids = b.ids, j.sel = b.sel;
    j.n_outer = b.n_outer, j.n_ids = b.n_ids, j.n_stored = b.n_stored, j.n_blocks = b.n_blocks;
    j.stride = b.stride, j.first = b.first, j.id_bytes = b.id_bytes, j.get = get;
    j.verdict = reinterpret_cast<uint32_t*>(static_cast<uintptr_t>(k));
    jobs.push_back(j);
    return b.has_rows() ? XFER_PAGED | XFER_PAGE_ROWS : XFER_PAGED;
  }
  // The table entry of descriptor k whose window's result lands in rows (WindowRows, in bytes; the descriptor's byte 0
  // is unit `trim`): the window pattern, if any, then the rows as the kernels count them.  *base receives the
  // descriptor's dst[0], from the rows' base `dst`.  Returns XFER_WINDOW_ROWS.
  uint32_t set_window_rows(uint32_t k, const WindowRows& wr, uint64_t trim, uintptr_t dst, void** base) {
    uint64_t shift = 0, kshift = 0;
    const WindowRows r = wr.rebase(trim, UINT64_MAX, &shift);
    const SourceRows kr = r.kernel_rows(&kshift);
    const StoreWindow& w = r.win;
    set_stride(k, XferStride{{w.strided() ? w.pitch : 1}, w.strided() ? w.width : 1, w.phase, kr.width, kr.pitch, kr.phase});
    *base = reinterpret_cast<void*>(dst + shift + kshift);
    return XFER_WINDOW_ROWS;
  }
  // Zero-size items get no descriptor: wait() reports their digest and checks their `expect` itself.
  struct Empty {
    uint32_t item;
    uint32_t flags;
    uint64_t expect;
  };
  std::vector<Empty> empties;

  ~Slot() {
    if (ev_done) cudaEventSynchronize(ev_done);
    cudaFreeHost(h_tab);
    cudaFreeHost(h_res);
    cudaFree(d_tab);
    cudaFree(d_sum);
    cudaFree(d_done);
    cudaFree(d_digest);
    cudaFree(d_status);
    if (d_debug) cudaFree(d_debug);
    if (d_trace) cudaFree(d_trace);
    if (ev_start) cudaEventDestroy(ev_start);
    if (ev_stop) cudaEventDestroy(ev_stop);
    if (ev_done) cudaEventDestroy(ev_done);
  }
};

// Releases a claimed slot when the call that holds it returns, whichever way it returns, unless the slot was kept (a
// submitted batch holds it until wait()).  Work the call queued on a stream before it failed is finished first, so
// that the next batch in the slot, maybe another thread's on another stream, cannot race it for the slot's tables.
class XferEngine::SlotHold {
 public:
  SlotHold(XferEngine* e, Slot* s) : e_(e), s_(s) {}
  ~SlotHold() {
    if (!s_) return;
    if (queued_) cudaStreamSynchronize(stream_);
    e_->release_slot(s_);
  }
  SlotHold(const SlotHold&) = delete;
  SlotHold& operator=(const SlotHold&) = delete;
  void queued(cudaStream_t st) {
    queued_ = true;
    stream_ = st;
  }
  void settled() { queued_ = false; }
  void keep() { s_ = nullptr; }

 private:
  XferEngine* e_;
  Slot* s_;
  bool queued_ = false;
  cudaStream_t stream_ = nullptr;
};

// Allocates one slot for batches of up to `max_items` objects on the current device.  Its digest workspace is zeroed
// on a stream of its own that does not synchronise with the legacy default stream: a slot added for a concurrent caller
// must not wait for other threads' batches.
Result<std::unique_ptr<XferEngine::Slot>> XferEngine::new_slot(uint32_t max_items) {
  const size_t tab_bytes = stride_table_offset(max_items) + static_cast<size_t>(max_items) * sizeof(XferStride);
  const size_t res_bytes = static_cast<size_t>(max_items) * 16;
  auto s = std::make_unique<Slot>();
  cudaStream_t zero = nullptr;
  bool ok = cudaMallocHost(reinterpret_cast<void**>(&s->h_tab), tab_bytes) == cudaSuccess;
  ok = ok && cudaMallocHost(reinterpret_cast<void**>(&s->h_res), res_bytes) == cudaSuccess;
  ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_tab), tab_bytes) == cudaSuccess;
  s->tab_bytes = s->dtab_bytes = tab_bytes;
  ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_sum), static_cast<size_t>(max_items) * 8) == cudaSuccess;
  ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_done), static_cast<size_t>(max_items) * 4) == cudaSuccess;
  ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_digest), static_cast<size_t>(max_items) * 8) == cudaSuccess;
  ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_status), static_cast<size_t>(max_items) * 4) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&zero, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaMemsetAsync(s->d_sum, 0, static_cast<size_t>(max_items) * 8, zero) == cudaSuccess;
  ok = ok && cudaMemsetAsync(s->d_done, 0, static_cast<size_t>(max_items) * 4, zero) == cudaSuccess;
  ok = ok && cudaStreamSynchronize(zero) == cudaSuccess;
  if (zero) cudaStreamDestroy(zero);
  ok = ok && cudaEventCreate(&s->ev_start) == cudaSuccess;
  ok = ok && cudaEventCreate(&s->ev_stop) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&s->ev_done, cudaEventDisableTiming) == cudaSuccess;
  if (!ok) {
    BB_LOG(ERROR) << "XferEngine: device allocation failed: " << cudaGetErrorString(cudaGetLastError());
    return ErrorCode::OUT_OF_MEMORY;  // the slot's destructor frees what was allocated
  }
  return s;
}

Result<std::unique_ptr<XferEngine>> XferEngine::create(int device, uint32_t max_items, int slots) {
  std::unique_ptr<XferEngine> e(new XferEngine());
  e->device_ = device;
  e->max_items_ = max_items;
  if (slots < 1 || slots > kMaxSlots) return ErrorCode::INVALID_ARGUMENT;
  int prev = 0;
  if (cudaGetDevice(&prev) != cudaSuccess) return ErrorCode::FABRIC_ERROR;
  if (cudaSetDevice(device) != cudaSuccess) return ErrorCode::FABRIC_ERROR;
  ErrorCode ec = ErrorCode::OK;
  for (int i = 0; i < slots && ec == ErrorCode::OK; ++i) {
    auto s = new_slot(max_items);
    if (s.ok()) e->slots_.push_back(std::move(s).value());
    else ec = s.error();
  }
  cudaSetDevice(prev);
  if (ec != ErrorCode::OK) return ec;
  return e;
}

XferEngine::~XferEngine() {
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(device_);
  slots_.clear();
  cudaSetDevice(prev);
}

struct XferEngine::Mailbox {
  MailSlot* slots = nullptr;      // pinned host
  MailResult* results = nullptr;  // pinned host
  MailCtl* ctl = nullptr;         // pinned host
  cudaStream_t stream = nullptr;  // non-blocking: never synchronises with the legacy default stream
  uint32_t next_seq = 1;          // next sequence number to hand out
  uint32_t epoch = 0;             // incarnation counter (0 = never launched)
  uint32_t outstanding = 0;       // posted requests whose results have not been collected
  uint64_t linger_ns = 200000, max_ns = 50000000;
  ~Mailbox() {
    if (stream) {
      cudaStreamSynchronize(stream);  // the resident warp leaves by itself after linger_ns
      cudaStreamDestroy(stream);
    }
    if (slots) cudaFreeHost(slots);
    if (results) cudaFreeHost(results);
    if (ctl) cudaFreeHost(ctl);
  }
};

bool XferEngine::mailbox_enabled() {
  static const bool on = [] {
    const char* e = std::getenv("BB_XFER_MAILBOX");
    return !(e && e[0] == '0');
  }();
  return on && mailbox_on_;
}

ErrorCode XferEngine::mailbox_launch_locked(uint32_t first_seq) {
  Mailbox& m = *mb_;
  ++m.epoch;
  const int rc = launch_mailbox(m.slots, m.results, m.ctl, first_seq, m.epoch, m.linger_ns, m.max_ns, m.stream);
  if (rc != 0) return cuda_failed(rc, "launch_mailbox");
  mailbox_launches_.fetch_add(1, std::memory_order_relaxed);
  launches_.fetch_add(1, std::memory_order_relaxed);
  return ErrorCode::OK;
}

// Hands `nd` small single-destination descriptors to the resident warp.  Slot layout and ordering: the 64-byte slot is
// written field by field, the sequence number last (x86 stores stay in order); the warp reads the whole line in one PCIe
// request and acts only when the sequence number is the one it expects.
ErrorCode XferEngine::mailbox_post(Slot* s, const XferDesc* descs, uint32_t nd, int algo) {
  if (!mb_) {
    auto m = std::make_unique<Mailbox>();
    BB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->slots), sizeof(MailSlot) * kMailSlots));
    BB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->results), sizeof(MailResult) * kMailSlots));
    BB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->ctl), sizeof(MailCtl)));
    std::memset(m->slots, 0, sizeof(MailSlot) * kMailSlots);
    std::memset(m->results, 0, sizeof(MailResult) * kMailSlots);
    std::memset(m->ctl, 0, sizeof(MailCtl));
    BB_CUDA(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    if (const char* e = std::getenv("BB_MAILBOX_LINGER_US")) m->linger_ns = static_cast<uint64_t>(std::max(1, std::atoi(e))) * 1000ull;
    mb_ = std::move(m);
  }
  Mailbox& m = *mb_;
  s->mail_first = m.next_seq;
  for (uint32_t i = 0; i < nd; ++i) {
    const uint32_t seq = m.next_seq++;
    MailSlot& q = m.slots[seq % kMailSlots];
    q.src = reinterpret_cast<uint64_t>(descs[i].src);
    q.dst = reinterpret_cast<uint64_t>(descs[i].dst[0]);
    q.expect = descs[i].expect;
    q.nbytes = static_cast<uint32_t>(descs[i].nbytes);
    q.flags = descs[i].flags;
    q.algo = static_cast<uint32_t>(algo);
    q.reserved = descs[i].reserved;
    std::atomic_thread_fence(std::memory_order_release);
    *reinterpret_cast<volatile uint32_t*>(&q.seq) = seq;
  }
  m.outstanding += nd;
  mailbox_requests_.fetch_add(nd, std::memory_order_relaxed);
  // is anybody polling?  (exit_epoch == epoch: the last incarnation has announced its exit; epoch 0: never launched)
  if (m.epoch == 0 || *reinterpret_cast<volatile uint32_t*>(&m.ctl->exit_epoch) == m.epoch) {
    const uint32_t first = m.epoch == 0 ? s->mail_first : *reinterpret_cast<volatile uint32_t*>(&m.ctl->next_seq);
    return mailbox_launch_locked(first);
  }
  return ErrorCode::OK;
}

ErrorCode XferEngine::mailbox_wait(Slot* s) {
  Mailbox& m = *mb_;
  const uint32_t nd = s->ndesc;
  auto* dg = reinterpret_cast<uint64_t*>(s->h_res);
  auto* stt = reinterpret_cast<uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 8);
  const auto t0 = std::chrono::steady_clock::now();
  for (uint32_t i = 0; i < nd; ++i) {
    const uint32_t seq = s->mail_first + i;
    const volatile MailResult* r = &m.results[seq % kMailSlots];
    uint32_t spins = 0;
    while (r->seq != seq) {
      if ((++spins & 0x3Fu) != 0) continue;
      std::lock_guard<std::mutex> lk(mu_);
      // the warp may have left just before our request landed (it lingers only so long): start the next incarnation
      if (*reinterpret_cast<volatile uint32_t*>(&m.ctl->exit_epoch) == m.epoch && r->seq != seq) {
        BB_CUDA(cudaSetDevice(device_));
        const ErrorCode ec = mailbox_launch_locked(*reinterpret_cast<volatile uint32_t*>(&m.ctl->next_seq));
        if (ec != ErrorCode::OK) return ec;
      }
      if ((spins & 0xFFFFu) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(2)) {
        BB_LOG(ERROR) << "XferEngine: the mailbox warp did not answer request " << seq;
        m.outstanding -= std::min(m.outstanding, nd - i);
        return ErrorCode::FABRIC_ERROR;
      }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    dg[i] = r->digest;
    stt[i] = r->status;
  }
  std::lock_guard<std::mutex> lk(mu_);
  m.outstanding -= std::min(m.outstanding, nd);
  return ErrorCode::OK;
}

bool XferEngine::flag_completion_enabled() {
  static const bool on = [] {
    const char* e = std::getenv("BB_XFER_FLAG_COMPLETION");
    return !(e && e[0] == '0');
  }();
  return on && flag_completion_;
}

bool XferEngine::small_path_enabled() {
  static const bool on = [] {
    const char* e = std::getenv("BB_XFER_SMALL");
    return !(e && e[0] == '0');
  }();
  return on && small_path_;
}

Result<XferEngine::Slot*> XferEngine::claim_slot() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (auto& c : slots_)
      if (c->ticket == 0) {
        c->ticket = next_ticket_++;
        return c.get();
      }
    if (static_cast<int>(slots_.size()) + growing_ >= kMaxSlots) return ErrorCode::RESOURCE_EXHAUSTED;
    ++growing_;
  }
  // Every slot is held by a batch of another thread, or of this one: a pipelined caller, or run_fp8 asking for its
  // scales batch, holds one slot while it asks for the next, so waiting for a free one could wait forever.
  auto fresh = new_slot(max_items_);
  std::lock_guard<std::mutex> lk(mu_);
  --growing_;
  if (!fresh.ok()) return fresh.error();
  Slot* s = fresh.value().get();
  s->ticket = next_ticket_++;
  slots_.push_back(std::move(fresh).value());
  return s;
}

void XferEngine::release_slot(Slot* s) {
  std::lock_guard<std::mutex> lk(mu_);
  s->ticket = 0;
}

// Completes the slot's pinned table for the `nd` descriptors at its start, [descs | tile_start]: every descriptor's
// first_tile and the nd + 1 tile_start prefix sums behind the descriptors.
ErrorCode XferEngine::write_tile_table(Slot* s, uint32_t nd) {
  auto* descs = reinterpret_cast<XferDesc*>(s->h_tab);
  auto* tile_start = reinterpret_cast<uint32_t*>(s->h_tab + static_cast<size_t>(nd) * sizeof(XferDesc));
  uint64_t tiles = 0;
  for (uint32_t i = 0; i < nd; ++i) {
    descs[i].first_tile = tile_start[i] = static_cast<uint32_t>(tiles);
    tiles += (descs[i].nbytes + kTileBytes - 1) / kTileBytes;
    if (tiles > 0xFFFFFFF0ull) return ErrorCode::VALUE_OUT_OF_RANGE;
  }
  tile_start[nd] = static_cast<uint32_t>(tiles);
  s->ndesc = nd;
  s->total_tiles = static_cast<uint32_t>(tiles);
  return ErrorCode::OK;
}

// Appends the batch's page entries, slice addresses and resolve jobs to the slot's table of `nd` descriptors (written up
// to tile_start), growing the table first when it is too small (the slot is idle: nothing reads it), and points every
// paged descriptor's stride entry at its first entry in the device copy.  The device copy also holds the BLOCKS items'
// page entries behind the jobs, which only the resolve kernel writes.  *tab: the bytes of the table to copy to the
// device.
ErrorCode XferEngine::write_pages(Slot* s, uint32_t nd, size_t* tab) {
  const size_t off = page_table_offset(nd), filled = jobs_offset(s, nd) + s->jobs.size() * sizeof(BlocksJob);
  const size_t need = filled + s->reserved * sizeof(uint64_t);
  if (filled > s->tab_bytes || need > s->dtab_bytes) {
    // the new buffers first: on a failure the slot keeps its old, still valid pair
    uint8_t *h = nullptr, *d = nullptr;
    cudaError_t e = filled > s->tab_bytes ? cudaMallocHost(reinterpret_cast<void**>(&h), filled) : cudaSuccess;
    if (e == cudaSuccess && need > s->dtab_bytes) e = cudaMalloc(reinterpret_cast<void**>(&d), need);
    if (e != cudaSuccess) {
      if (h) cudaFreeHost(h);
      cudaGetLastError();
      BB_LOG(ERROR) << "XferEngine: growing a descriptor table to " << need << " bytes failed: " << cudaGetErrorString(e);
      return ErrorCode::OUT_OF_MEMORY;
    }
    if (h) {
      std::memcpy(h, s->h_tab, stride_table_offset(nd));
      cudaFreeHost(s->h_tab);
      s->h_tab = h;
      s->tab_bytes = filled;
    }
    if (d) {
      cudaFree(s->d_tab);
      s->d_tab = d;
      s->dtab_bytes = need;
    }
  }
  const auto d_pages = reinterpret_cast<uint64_t>(s->d_tab + off);
  const auto d_reserved = reinterpret_cast<uint64_t>(s->d_tab + filled);
  for (uint32_t k : s->paged_descs) s->strides[k].pages = d_pages + s->strides[k].pages * sizeof(uint64_t);
  for (uint32_t k : s->blocks_descs) s->strides[k].pages = d_reserved + s->strides[k].pages * sizeof(uint64_t);
  s->write_strides(nd);
  std::memcpy(s->h_tab + off, s->pages.data(), s->pages.size() * sizeof(uint64_t));
  // read_verdicts() reads the word of every descriptor of a batch with jobs: a descriptor without one must not report
  // the verdict a refused BLOCKS item left at its index in an earlier batch of this slot
  auto* verdicts = reinterpret_cast<uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 12);
  if (!s->jobs.empty()) std::fill(verdicts, verdicts + nd, kBlocksOk);
  for (BlocksJob& j : s->jobs) {
    j.entries = reinterpret_cast<uint64_t*>(d_reserved + reinterpret_cast<uintptr_t>(j.entries) * sizeof(uint64_t));
    j.outer = reinterpret_cast<const uint64_t*>(d_pages + reinterpret_cast<uintptr_t>(j.outer) * sizeof(uint64_t));
    j.verdict = verdicts + reinterpret_cast<uintptr_t>(j.verdict);
  }
  std::memcpy(s->h_tab + jobs_offset(s, nd), s->jobs.data(), s->jobs.size() * sizeof(BlocksJob));
  *tab = filled;
  return ErrorCode::OK;
}

// Queues the resolve kernel of the batch's BLOCKS descriptors on stream `st`, after the copy of the table it reads.
ErrorCode XferEngine::launch_resolve(Slot* s, uint32_t nd, void* st) {
  if (s->jobs.empty()) return ErrorCode::OK;
  const int rc = launch_resolve_blocks(reinterpret_cast<const BlocksJob*>(s->d_tab + jobs_offset(s, nd)), static_cast<uint32_t>(s->jobs.size()), st);
  if (rc != 0) return cuda_failed(rc, "launch_resolve_blocks");
  launches_.fetch_add(1, std::memory_order_relaxed);
  return ErrorCode::OK;
}

size_t XferEngine::jobs_offset(const Slot* s, uint32_t nd) {
  return page_table_offset(nd) + s->pages.size() * sizeof(uint64_t);
}

// The verdict of every item of the slot's last batch: OK, or the resolve kernel's for a BLOCKS item (read once the
// batch has finished).
void XferEngine::read_verdicts(const Slot* s, uint32_t nitems, const std::vector<int32_t>& item_to_desc, std::vector<ErrorCode>* out) const {
  out->assign(nitems, ErrorCode::OK);
  if (s->jobs.empty()) return;
  const auto* v = reinterpret_cast<const volatile uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 12);
  for (uint32_t i = 0; i < nitems; ++i) {
    const int32_t d = item_to_desc[i];
    if (d < 0) continue;
    (*out)[i] = v[d] == kBlocksOutOfRange ? ErrorCode::VALUE_OUT_OF_RANGE : v[d] == kBlocksDuplicate ? ErrorCode::INVALID_ARGUMENT : ErrorCode::OK;
  }
}

Result<uint64_t> XferEngine::submit(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream,
                                    bool capture_debug) {
  if (items.size() > max_items_) return ErrorCode::RESOURCE_EXHAUSTED;
  BB_CUDA(cudaSetDevice(device_));
  auto claimed = claim_slot();
  if (!claimed.ok()) return claimed.error();
  Slot* s = claimed.value();
  const uint64_t ticket = s->ticket;
  SlotHold hold(this, s);
  auto* descs = reinterpret_cast<XferDesc*>(s->h_tab);
  s->item_to_desc.assign(items.size(), -1);
  s->empties.clear();
  s->clear_layouts();
  uint32_t nd = 0;
  bool all_small = small_path_enabled();
  for (size_t i = 0; i < items.size(); ++i) {
    const XferItem& it = items[i];
    const bool win = it.flags & XFER_WINDOW;
    const bool strided = it.flags & XFER_STRIDED;
    const bool gather = it.flags & XFER_GATHER;
    const bool scatter = it.flags & XFER_SCATTER;
    if ((strided && !win) || (win && (strided != it.win.strided() || !it.win.valid(it.nbytes) || it.ndst != 1 ||
                                      (it.flags & (XFER_MULTIMEM | XFER_RAW_SUM)))))
      return ErrorCode::INVALID_ARGUMENT;
    // a layout is the gathering load's source or the scattering store's destination, the side its flag names
    const bool blocks = it.mem.kind() == DeviceLayout::BLOCKS;
    // XFER_PAGE_ROWS, XFER_WINDOW_ROWS and XFER_SEGMENTS are the engine's to set, from the layout (set_layout, and a
    // WINDOW_ROWS layout below): a caller's flag would send a descriptor without its table down the in-page row walk, the
    // windowed store or the segment walk
    if (it.flags & (XFER_PAGE_ROWS | XFER_WINDOW_ROWS | XFER_SEGMENTS)) return ErrorCode::INVALID_ARGUMENT;
    // The one scattering store with a window: into rows of the window's result (WindowRows).  Without a window those are
    // the object's own rows.
    const bool wrows = scatter && win && it.mem.kind() == DeviceLayout::WINDOW_ROWS;
    const DeviceLayout mem = scatter && !win ? it.mem.as_rows() : it.mem;
    const uint32_t scatter_excl = (wrows ? 0u : XFER_WINDOW | XFER_STRIDED) | XFER_GATHER | XFER_MULTIMEM | XFER_RAW_SUM;
    if ((gather || scatter) == mem.contiguous() || ((it.flags & XFER_PAGED) && mem.kind() != DeviceLayout::PAGES && !blocks) ||
        !(gather ? mem.valid_source(it.nbytes) : mem.valid(it.nbytes)) || (gather && (it.flags & (XFER_WINDOW | XFER_STRIDED | XFER_RAW_SUM))) ||
        (mem.kind() == DeviceLayout::SEGMENTS && mem.segments().unit != 1) ||
        (scatter && (it.ndst != 1 || (it.flags & scatter_excl))))
      return ErrorCode::INVALID_ARGUMENT;
    if (blocks && scatter && !it.mem.blocks().distinct_checkable()) return ErrorCode::NOT_IMPLEMENTED;
    // Without a checksum nothing outside the window has to be read: the descriptor starts at the 16-byte boundary at or
    // below the window and ends with it (an empty window reads nothing).  A verified window reads the whole object.
    const uint64_t nbytes = window_read_bytes(it, algo);
    const uint64_t trim = win && algo == ChecksumAlgo::NONE ? it.win.lo & ~uint64_t{15} : 0;
    if (nbytes == 0) {
      s->empties.push_back({static_cast<uint32_t>(i), it.flags, it.expect});
      continue;
    }
    // windowed items (strided ones included), gathered and scattered ones always take bb_xfer: neither the warp-per-object
    // kernel nor the mailbox has a store window, a gathering load or a scattering store
    all_small = all_small && nbytes <= kSmallBytes && !(it.flags & (XFER_RAW_SUM | XFER_WINDOW | XFER_GATHER | XFER_SCATTER)) && it.ndst >= 1;
    if (it.ndst > kMaxDst || (it.ndst == 0 && !(it.flags & XFER_RAW_SUM))) return ErrorCode::INVALID_ARGUMENT;
    uintptr_t al = gather ? 0 : reinterpret_cast<uintptr_t>(it.src);  // gathered: the source layout instead
    // strided: the window instead; scattered: the destination layout instead
    for (uint32_t r = strided || scatter ? 1 : 0; r < it.ndst; ++r) al |= reinterpret_cast<uintptr_t>(it.dst[r]);
    const auto dst0 = reinterpret_cast<uintptr_t>(it.dst[0]);
    const WindowRows wr{it.win, mem.rows()};
    if ((al & 15) || (strided && !wrows && !it.win.coaligned(dst0)) || (wrows && !wr.coaligned(dst0, it.nbytes)) ||
        ((gather || scatter) && !wrows && !mem.coaligned(reinterpret_cast<uintptr_t>(gather ? it.src : it.dst[0]), it.nbytes)))
      return ErrorCode::INVALID_ADDRESS;
    if ((it.flags & XFER_MULTIMEM) && (it.nbytes & 15)) return ErrorCode::INVALID_ARGUMENT;
    XferDesc& d = descs[nd];
    d.src = static_cast<const uint8_t*>(it.src) + trim;
    for (uint32_t r = 0; r < kMaxDst; ++r) d.dst[r] = r < it.ndst ? it.dst[r] : nullptr;
    if (win) {  // the descriptor's byte 0 is object byte `trim`
      const StoreWindow w = it.win.rebase(trim);
      d.win.base = reinterpret_cast<void*>(dst0 + w.base_shift(trim) + w.origin());
      d.win.lo = w.lo;
      d.win.hi = w.hi;
      if (strided && !wrows) s->set_stride(nd, w);
    }
    d.nbytes = nbytes;
    d.ndst = it.ndst;
    d.expect = it.expect;
    d.flags = it.flags;
    if (wrows) d.flags = (d.flags & ~XFER_SCATTER) | s->set_window_rows(nd, wr, trim, dst0, &d.win.base);
    else if (gather || scatter) d.flags |= s->set_layout(nd, mem, nbytes, scatter);
    d.reserved = (it.flags & XFER_RAW_SUM) ? it.tile_base : 0;
    if (algo == ChecksumAlgo::CRC32C) {
      d.expect = (static_cast<uint64_t>(crc_init_term_for(nbytes)) << 32) | (it.expect & 0xFFFFFFFFull);
      d.reserved = crc_unpad_for(nbytes);
    }
    s->item_to_desc[i] = static_cast<int32_t>(nd++);
  }
  BB_TRY(write_tile_table(s, nd));
  const bool any_strided = !s->strides.empty();
  size_t tab = 0;
  if (s->pages.empty()) tab = s->write_strides(nd);
  else BB_TRY(write_pages(s, nd, &tab));
  descs = reinterpret_cast<XferDesc*>(s->h_tab);  // write_pages may have moved the table
  s->nitems = static_cast<uint32_t>(items.size());
  s->debug = capture_debug;
  s->traced = tile_trace_;
  s->hashed = algo != ChecksumAlgo::NONE;
  s->crc = algo == ChecksumAlgo::CRC32C;
  s->empty_digest = is_tile_sum(algo) ? tchash::finalize(0, 0) : 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int xalgo = algo == ChecksumAlgo::BBH64 ? ALGO_BBH64 : algo == ChecksumAlgo::CRC32C ? ALGO_CRC32C : algo == ChecksumAlgo::XXH3 ? ALGO_XXH3 : ALGO_NONE;
  // Small batches: the finalizer warp writes digests / status straight into the pinned result block (UVA).
  const bool direct = nd <= kDirectResults;

  // Completion mode.  A small batch without diagnostics whose results land in pinned memory needs no CUDA event (each
  // costs about as much GPU time as the kernel): the resident mailbox warp serves it without any launch, or else it
  // completes by flag and the launch is the ONLY stream operation.  The mailbox request bypasses `stream`, so
  // everything already queued there must have finished (the caller's source data is ready), and only one mailed batch
  // is in flight at a time (across all threads: checked again under mu_ where the batch is posted).
  using Completion = Slot::Completion;
  s->completion = Completion::EVENTS;
  if (nd && all_small && direct && !capture_debug && !tile_trace_) {
    bool mail = nd <= kMailSlots / 2 && mailbox_enabled();
    if (mail) {
      std::lock_guard<std::mutex> lk(mu_);
      mail = !mb_ || mb_->outstanding == 0;
    }
    if (mail) {
      bool simple = true;
      for (uint32_t i = 0; i < nd; ++i) simple = simple && descs[i].ndst == 1 && !(descs[i].flags & (XFER_MULTIMEM | XFER_WINDOW));
      mail = simple && cudaStreamQuery(st) == cudaSuccess;
      if (!mail) cudaGetLastError();  // cudaErrorNotReady is not sticky, but keep the error state clean
    }
    if (mail) {
      std::lock_guard<std::mutex> lk(mu_);
      if (!mb_ || mb_->outstanding == 0) {
        s->completion = Completion::MAILBOX;
        BB_TRY(mailbox_post(s, descs, nd, xalgo));
        hold.keep();
        return ticket;
      }
    }
    if (flag_completion_enabled()) s->completion = Completion::FLAG;
  }

  if (nd) {
    const bool inline_tab = nd <= kInlineDescs && s->pages.empty();  // page entries live in the device table only
    hold.queued(st);
    if (!inline_tab) BB_CUDA(cudaMemcpyAsync(s->d_tab, s->h_tab, tab, cudaMemcpyHostToDevice, st));
    BB_TRY(launch_resolve(s, nd, st));
    if (capture_debug) {
      const size_t need = static_cast<size_t>(s->total_tiles) * tchash::kRows * tchash::kN * 4;
      if (need > s->d_debug_bytes) {
        if (s->d_debug) cudaFree(s->d_debug);
        BB_CUDA(cudaMalloc(reinterpret_cast<void**>(&s->d_debug), need));
        s->d_debug_bytes = need;
      }
    }
    XferLaunch l;
    l.descs = reinterpret_cast<const XferDesc*>(s->d_tab);
    l.tile_start = reinterpret_cast<const uint32_t*>(s->d_tab + static_cast<size_t>(nd) * sizeof(XferDesc));
    l.ndesc = nd;
    l.total_tiles = s->total_tiles;
    l.sum_ws = s->d_sum;
    l.done_ws = s->d_done;
    l.digest_out = direct ? reinterpret_cast<uint64_t*>(s->h_res) : s->d_digest;
    l.status_out = direct ? reinterpret_cast<uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 8) : s->d_status;
    if (inline_tab) {
      l.host_descs = descs;
      l.host_tile_start = reinterpret_cast<const uint32_t*>(s->h_tab + static_cast<size_t>(nd) * sizeof(XferDesc));
    }
    if (any_strided) {
      l.strides = reinterpret_cast<const XferStride*>(s->d_tab + stride_table_offset(nd));
      if (inline_tab) l.host_strides = reinterpret_cast<const XferStride*>(s->h_tab + stride_table_offset(nd));
    }
    l.debug_d = capture_debug ? s->d_debug : nullptr;
    if (tile_trace_) {
      const size_t need = static_cast<size_t>(s->total_tiles) * 4 * sizeof(uint64_t);
      if (need > s->d_trace_bytes) {
        if (s->d_trace) cudaFree(s->d_trace);
        BB_CUDA(cudaMalloc(reinterpret_cast<void**>(&s->d_trace), need));
        s->d_trace_bytes = need;
      }
      BB_CUDA(cudaMemsetAsync(s->d_trace, 0, need, st));
      l.trace_d = s->d_trace;
    }
    l.algo = xalgo;
    l.max_ctas = max_ctas_;
    l.stream = stream;
    l.small_path = all_small;
    if (s->completion == Completion::FLAG) {
      auto* stt = reinterpret_cast<volatile uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 8);
      for (uint32_t i = 0; i < nd; ++i) stt[i] = kSmallPending;
      l.flag_completion = true;
      s->stream = stream;
    } else {
      BB_CUDA(cudaEventRecord(s->ev_start, st));
    }
    const int rc = launch_xfer(l);
    if (rc != 0) return cuda_failed(rc, "launch_xfer");
    launches_.fetch_add(1, std::memory_order_relaxed);
    if (all_small && !capture_debug && !tile_trace_) small_launches_.fetch_add(1, std::memory_order_relaxed);
    if (s->completion == Completion::EVENTS) {
      BB_CUDA(cudaEventRecord(s->ev_stop, st));
      if (algo != ChecksumAlgo::NONE && !direct) {
        BB_CUDA(cudaMemcpyAsync(s->h_res, s->d_digest, static_cast<size_t>(nd) * 8, cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaMemcpyAsync(s->h_res + static_cast<size_t>(max_items_) * 8, s->d_status, static_cast<size_t>(nd) * 4,
                                cudaMemcpyDeviceToHost, st));
      }
    }
  }
  if (s->completion == Completion::EVENTS) BB_CUDA(cudaEventRecord(s->ev_done, st));
  hold.keep();
  return ticket;
}

ErrorCode XferEngine::wait(uint64_t ticket, XferResult* out) {
  Slot* s = nullptr;
  {
    std::lock_guard<std::mutex> lk(mu_);
    for (auto& c : slots_)
      if (ticket != 0 && c->ticket == ticket) { s = c.get(); break; }
  }
  if (!s) return ErrorCode::NOT_FOUND;
  SlotHold release(this, s);
  const uint32_t nd = s->ndesc;
  switch (s->completion) {
    case Slot::Completion::MAILBOX:
      BB_TRY(mailbox_wait(s));
      break;
    case Slot::Completion::FLAG: {
      // spin on the status words the kernel writes last (pinned memory); fall back to a stream sync if they do not show
      // up within a generous bound, so that a launch failure surfaces as an error instead of a hang
      const auto* stt = reinterpret_cast<const volatile uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 8);
      const auto t0 = std::chrono::steady_clock::now();
      uint32_t done = 0, spins = 0;
      while (done < nd) {
        if (stt[done] != kSmallPending) {
          ++done;
          continue;
        }
        if ((++spins & 0x3FFu) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(200)) {
          BB_CUDA(cudaSetDevice(device_));
          BB_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(s->stream)));
          if (stt[done] == kSmallPending) {
            BB_LOG(ERROR) << "XferEngine: small-object kernel finished without publishing its results";
            return ErrorCode::FABRIC_ERROR;
          }
        }
      }
      std::atomic_thread_fence(std::memory_order_acquire);
      break;
    }
    case Slot::Completion::EVENTS:
      BB_CUDA(cudaEventSynchronize(s->ev_done));
      break;
  }
  const bool no_hash = !s->hashed;
  if (out) {
    out->digest.assign(s->nitems, no_hash ? 0 : s->empty_digest);
    out->status.assign(s->nitems, 0);
    const auto* dg = reinterpret_cast<const uint64_t*>(s->h_res);
    const auto* stt = reinterpret_cast<const uint32_t*>(s->h_res + static_cast<size_t>(max_items_) * 8);
    if (!no_hash) {
      for (uint32_t i = 0; i < s->nitems; ++i) {
        const int32_t d = s->item_to_desc[i];
        if (d >= 0) {
          out->digest[i] = dg[d];
          out->status[i] = stt[d];
        }
      }
      // The digest of an empty object (a RAW_SUM slice of no tiles sums to 0); verified as the kernels verify: CRC32C
      // compares the low 32 bits of `expect`.
      for (const Slot::Empty& e : s->empties) {
        const uint64_t digest = (e.flags & XFER_RAW_SUM) ? 0 : s->empty_digest;
        const uint64_t want = s->crc ? (e.expect & 0xFFFFFFFFull) : e.expect;
        out->digest[e.item] = digest;
        out->status[e.item] = ((e.flags & XFER_VERIFY) && digest != want) ? 1u : 0u;
      }
    }
    read_verdicts(s, s->nitems, s->item_to_desc, &out->verdict);
    out->device_ms = 0.f;
    if (nd && s->completion == Slot::Completion::EVENTS) cudaEventElapsedTime(&out->device_ms, s->ev_start, s->ev_stop);
  }
  if (s->debug && nd) {
    std::vector<uint32_t> acc(static_cast<size_t>(s->total_tiles) * tchash::kRows * tchash::kN);
    BB_CUDA(cudaMemcpy(acc.data(), s->d_debug, acc.size() * 4, cudaMemcpyDeviceToHost));
    std::lock_guard<std::mutex> lk(mu_);
    debug_host_ = std::move(acc);
  }
  if (s->traced && nd) {
    std::vector<uint64_t> trace(static_cast<size_t>(s->total_tiles) * 4);
    BB_CUDA(cudaMemcpy(trace.data(), s->d_trace, trace.size() * 8, cudaMemcpyDeviceToHost));
    std::lock_guard<std::mutex> lk(mu_);
    trace_host_ = std::move(trace);
  }
  return ErrorCode::OK;
}

ErrorCode XferEngine::run_fp8(const std::vector<Fp8Item>& items, bool unpack, void* stream, XferResult* out) {
  const uint32_t n = static_cast<uint32_t>(items.size());
  if (n == 0) return ErrorCode::OK;
  if (n > max_items_) return ErrorCode::RESOURCE_EXHAUSTED;
  BB_CUDA(cudaSetDevice(device_));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // The fused kernel's batch holds this slot for the whole call; the scales batch below takes a second one.  The slot's
  // d_digest collects the payload sums (d_sum must stay zero between batches for bb_xfer).
  auto claimed = claim_slot();
  if (!claimed.ok()) return claimed.error();
  Slot* s = claimed.value();
  SlotHold release(this, s);
  auto* descs = reinterpret_cast<XferDesc*>(s->h_tab);
  std::vector<XferItem> scale_items(n);  // scales region of every object, hashed as a RAW_SUM slice by bb_xfer
  // as submit() does: nothing of the slot's last batch (a paged bb_xfer batch's page entries included) carries over
  s->clear_layouts();
  // one kernel instantiation per launch: bf16 and fp16 items share the 2-byte one, fp32 items take the 4-byte one
  const uint32_t eb = mxfp8::wide_bytes(items[0].wide_type);
  for (uint32_t i = 0; i < n; ++i) {
    const Fp8Item& it = items[i];
    const bool strided = it.win.strided();
    // an unpack into rows of the window's result (WindowRows); with a window that stores the whole object in place those
    // are the object's own rows
    const bool wrows = unpack && it.mem.kind() == DeviceLayout::WINDOW_ROWS && !it.win.covers(it.n_elems);
    const DeviceLayout lay = wrows ? DeviceLayout{} : unpack ? it.mem.as_rows() : it.mem;
    const bool shaped = !lay.contiguous();
    // the window a shaped layout may go with: none, or for rows of a window's result one that stores the whole object
    const bool in_place = it.win.whole() || (unpack && it.mem.kind() == DeviceLayout::WINDOW_ROWS && it.win.covers(it.n_elems));
    if (!fp8_eligible(it.n_elems)) return ErrorCode::INVALID_ARGUMENT;
    if (it.wide_type != mxfp8::Wide::BF16 && it.wide_type != mxfp8::Wide::F16 && it.wide_type != mxfp8::Wide::F32)
      return ErrorCode::INVALID_ARGUMENT;
    if (mxfp8::wide_bytes(it.wide_type) != eb) return ErrorCode::INVALID_ARGUMENT;  // mixes 2- and 4-byte wide types
    DeviceLayout mem;  // a gathered put's source, or a scattered get's destination, in wide bytes; never with a window
    if (shaped && (!in_place || !(unpack ? lay.valid(it.n_elems) : lay.valid_source(it.n_elems)) || !lay.to_wide_bytes(eb, &mem)))
      return ErrorCode::INVALID_ARGUMENT;
    if (unpack && mem.kind() == DeviceLayout::BLOCKS && !mem.blocks().distinct_checkable()) return ErrorCode::NOT_IMPLEMENTED;
    // a strided window's rows need not start at `wide` (row 0 of the pattern may lie before the window, or the object's
    // first element after row 0's start): the window is checked instead, below
    if ((reinterpret_cast<uintptr_t>(it.packed) & 15) || (!strided && !wrows && !mem.coaligned(reinterpret_cast<uintptr_t>(it.wide), eb * it.n_elems)))
      return ErrorCode::INVALID_ADDRESS;
    const uint32_t nrep = unpack ? 1u : it.nreplicas;
    if (nrep < 1 || nrep > kMaxDst) return ErrorCode::INVALID_ARGUMENT;
    // a put stores the whole object; from here on the window is in wide bytes
    StoreWindow w = it.win.over(it.n_elems);
    if ((!unpack && !it.win.whole()) || !w.valid(it.n_elems) || !w.to_wide_bytes(eb, &w)) return ErrorCode::INVALID_ARGUMENT;
    for (uint32_t r = 1; r < nrep; ++r)
      if (!it.more_packed[r - 1] || (reinterpret_cast<uintptr_t>(it.more_packed[r - 1]) & 15)) return ErrorCode::INVALID_ADDRESS;
    auto* payload = static_cast<uint8_t*>(it.packed);
    XferDesc& d = descs[i];
    d.src = unpack ? static_cast<const void*>(payload) : it.wide;
    d.dst[0] = unpack ? it.wide : static_cast<void*>(payload);  // pack: base of the packed object in every replica
    d.dst[1] = nrep > 1 ? it.more_packed[0] : nullptr;
    d.dst[2] = nrep > 2 ? it.more_packed[1] : nullptr;
    d.nbytes = it.n_elems;  // payload tiles, the last one possibly partial
    d.ndst = nrep;
    d.expect = 0;
    d.flags = it.wide_type == mxfp8::Wide::F16 ? XFER_WIDE_F16 : 0u;
    d.reserved = 0;
    // whole-object gets keep exactly the descriptors they had; a strided item always carries its window
    if (unpack && !it.win.covers(it.n_elems)) {
      d.flags |= XFER_WINDOW;
      d.win.lo = w.lo;
      d.win.hi = w.hi;
    }
    if (wrows) {  // held to the rule submit() applies to an XferItem with a WINDOW_ROWS layout, in wide bytes
      WindowRows wr{w, it.mem.rows()};
      if (!it.mem.rows().valid() || !it.mem.rows().to_wide_bytes(eb, &wr.rows)) return ErrorCode::INVALID_ARGUMENT;
      if (!wr.coaligned(reinterpret_cast<uintptr_t>(it.wide), eb * it.n_elems)) return ErrorCode::INVALID_ADDRESS;
      if (strided) d.flags |= XFER_STRIDED;
      d.flags |= s->set_window_rows(i, wr, 0, reinterpret_cast<uintptr_t>(it.wide), &d.win.base);
    } else if (strided) {  // held to the rule submit() applies to a strided XferItem
      if (!w.coaligned(reinterpret_cast<uintptr_t>(it.wide))) return ErrorCode::INVALID_ADDRESS;
      d.win.base = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(it.wide) + w.origin());
      d.flags |= XFER_STRIDED;
      s->set_stride(i, w);
    }
    if (shaped)  // d.src (gather) or d.dst[0] (scatter) is the layout's base
      d.flags |= (unpack ? XFER_SCATTER : XFER_GATHER) | s->set_layout(i, mem, eb * it.n_elems, unpack);
    // the fused kernel hashes the whole payload tiles; everything past them (payload tail + scales) is hashed from the
    // stored bytes as a slice
    const uint64_t nt_full = it.n_elems / kTileBytes;
    XferItem& sc = scale_items[i];
    sc.src = payload + nt_full * kTileBytes;
    sc.ndst = 0;
    sc.nbytes = (it.n_elems - nt_full * kTileBytes) + it.n_elems / 32;
    sc.flags = XFER_RAW_SUM;
    sc.tile_base = static_cast<uint32_t>(nt_full);
  }
  BB_TRY(write_tile_table(s, n));
  const bool any_strided = !s->strides.empty();
  size_t tab = 0;
  if (s->pages.empty()) tab = s->write_strides(n);
  else BB_TRY(write_pages(s, n, &tab));  // may move the table: the launch's pointers are taken below
  release.queued(st);
  BB_CUDA(cudaMemcpyAsync(s->d_tab, s->h_tab, tab, cudaMemcpyHostToDevice, st));
  BB_TRY(launch_resolve(s, n, st));
  BB_CUDA(cudaMemsetAsync(s->d_digest, 0, static_cast<size_t>(n) * 8, st));
  XferLaunch l;
  l.descs = reinterpret_cast<const XferDesc*>(s->d_tab);
  l.tile_start = reinterpret_cast<const uint32_t*>(s->d_tab + static_cast<size_t>(n) * sizeof(XferDesc));
  l.ndesc = n;
  l.total_tiles = s->total_tiles;
  if (any_strided) l.strides = reinterpret_cast<const XferStride*>(s->d_tab + stride_table_offset(n));
  l.sum_ws = s->d_digest;
  l.max_ctas = max_ctas_;
  l.stream = stream;
  BB_CUDA(cudaEventRecord(s->ev_start, st));
  const int rc = launch_xfer_fp8(l, unpack, eb);
  if (rc != 0) return cuda_failed(rc, "launch_xfer_fp8");
  launches_.fetch_add(1, std::memory_order_relaxed);
  BB_CUDA(cudaEventRecord(s->ev_stop, st));
  BB_CUDA(cudaMemcpyAsync(s->h_res, s->d_digest, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost, st));
  // scales: for a put they were just written by the kernel above (same stream), for a get they are read twice
  XferResult sres;
  BB_TRY(run(scale_items, ChecksumAlgo::BBH64, stream, &sres));  // waits for the stream up to here
  BB_CUDA(cudaStreamSynchronize(st));
  release.settled();
  if (out) {
    const auto* sums = reinterpret_cast<const uint64_t*>(s->h_res);
    out->digest.assign(n, 0);
    out->status.assign(n, 0);
    for (uint32_t i = 0; i < n; ++i) {
      const uint64_t total = items[i].n_elems + items[i].n_elems / 32;
      out->digest[i] = tchash::finalize(sums[i] + sres.digest[i], total);
      if (items[i].verify && out->digest[i] != items[i].expect) out->status[i] = 1;
    }
    std::vector<int32_t> ident(n);
    for (uint32_t i = 0; i < n; ++i) ident[i] = static_cast<int32_t>(i);
    read_verdicts(s, n, ident, &out->verdict);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, s->ev_start, s->ev_stop);
    out->device_ms = ms + sres.device_ms;
  }
  return ErrorCode::OK;
}

ErrorCode XferEngine::run(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream, XferResult* out) {
  auto t = submit(items, algo, stream);
  if (!t.ok()) return t.error();
  return wait(t.value(), out);
}

// ---------------------------------------------------------------- helpers
ErrorCode device_count(int* n) {
  *n = 0;
  cudaError_t e = cudaGetDeviceCount(n);
  if (e != cudaSuccess) {
    *n = 0;
    cudaGetLastError();
  }
  return ErrorCode::OK;
}
ErrorCode device_malloc(int device, uint64_t bytes, void** out) {
  BB_CUDA(cudaSetDevice(device));
  cudaError_t e = cudaMalloc(out, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return ErrorCode::OUT_OF_MEMORY;
  }
  return ErrorCode::OK;
}
ErrorCode device_free(int device, void* p) {
  BB_CUDA(cudaSetDevice(device));
  BB_CUDA(cudaFree(p));
  return ErrorCode::OK;
}
ErrorCode host_alloc_pinned(uint64_t bytes, void** out) {
  cudaError_t e = cudaMallocHost(out, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return ErrorCode::OUT_OF_MEMORY;
  }
  return ErrorCode::OK;
}
ErrorCode host_free_pinned(void* p) {
  BB_CUDA(cudaFreeHost(p));
  return ErrorCode::OK;
}
ErrorCode stream_synchronize(void* stream) {
  BB_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return ErrorCode::OK;
}
ErrorCode device_synchronize(int device) {
  BB_CUDA(cudaSetDevice(device));
  BB_CUDA(cudaDeviceSynchronize());
  return ErrorCode::OK;
}
int device_memcpy_peer_async(void* dst, int dst_device, const void* src, int src_device, uint64_t nbytes, void* stream) {
  return static_cast<int>(cudaMemcpyPeerAsync(dst, dst_device, src, src_device, nbytes, static_cast<cudaStream_t>(stream)));
}
int device_enable_peer_access(int device, int peer) {
  int prev = 0;
  cudaGetDevice(&prev);
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) {
    e = cudaDeviceEnablePeerAccess(peer, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) {
      cudaGetLastError();
      e = cudaSuccess;
    }
  }
  cudaSetDevice(prev);
  return static_cast<int>(e);
}

const char* cuda_error_string(int code) { return cudaGetErrorString(static_cast<cudaError_t>(code)); }

}  // namespace bb::gpu
