#include "fabric/xfer_engine.h"

#include <cuda_runtime.h>

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
  last_cuda_error_ = code;
  return gpu::cuda_failed(code, what);
}

namespace {
// Frees a slot when the call that holds it returns, whichever way it returns.
struct SlotRelease {
  uint64_t& ticket;
  ~SlotRelease() { ticket = 0; }
};

// A slot's table of nd descriptors is [descs | tile_start (nd + 1) | strides (nd), only for batches with strided items |
// page entries, only for batches with paged items].
size_t stride_table_offset(size_t nd) { return (nd * sizeof(XferDesc) + (nd + 1) * 4 + 7) & ~size_t{7}; }
size_t page_table_offset(size_t nd) { return stride_table_offset(nd) + nd * sizeof(XferStride); }
}  // namespace

struct XferEngine::Slot {
  // How wait() learns that the batch has finished (chosen in submit()).
  enum class Completion {
    EVENTS,   // CUDA events: timing events around the launch, a completion event after the result copies
    FLAG,     // the kernel's status words in pinned memory; no event on the stream (small-object latency path)
    MAILBOX,  // served by the resident mailbox warp: results arrive in the mailbox's result ring
  };
  // host (pinned): [descs | tile_start | strides | pages], tab_bytes each way
  uint8_t* h_tab = nullptr;
  // device
  uint8_t* d_tab = nullptr;
  size_t tab_bytes = 0;
  uint64_t* d_sum = nullptr;
  uint32_t* d_done = nullptr;
  uint64_t* d_digest = nullptr;
  uint32_t* d_status = nullptr;
  // host (pinned) results: [digest | status]
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
  void set_stride(uint32_t k, const SourceRows& r) { set_stride(k, XferStride{r.pitch, r.width, r.phase}); }
  // Writes the stride table behind tile_start when the batch has a strided descriptor, and returns the bytes of the
  // table to copy to the device: [descs | tile_start | strides], or without the strides.
  size_t write_strides(uint32_t nd) {
    if (strides.empty()) return static_cast<size_t>(nd) * sizeof(XferDesc) + (static_cast<size_t>(nd) + 1) * 4;
    strides.resize(nd, XferStride{1, 1, 0});
    std::memcpy(h_tab + stride_table_offset(nd), strides.data(), static_cast<size_t>(nd) * sizeof(XferStride));
    return stride_table_offset(nd) + static_cast<size_t>(nd) * sizeof(XferStride);
  }
  // The page entries of the batch's XFER_PAGED descriptors, back to back; each one's stride entry holds the index of its
  // first entry here until write_pages() turns it into a device address.
  std::vector<uint64_t> pages;
  std::vector<uint32_t> paged_descs;
  void add_pages(uint32_t k, const SourcePages& p, uint64_t nbytes) {
    set_stride(k, XferStride{{pages.size()}, p.page, p.phase});
    paged_descs.push_back(k);
    pages.insert(pages.end(), p.addrs, p.addrs + p.pages_for(nbytes));
  }
  // Zero-size items get no descriptor: wait() reports their digest and checks their `expect` itself.
  struct Empty {
    uint32_t item;
    uint32_t flags;
    uint64_t expect;
  };
  std::vector<Empty> empties;
};

Result<std::unique_ptr<XferEngine>> XferEngine::create(int device, uint32_t max_items, int slots) {
  std::unique_ptr<XferEngine> e(new XferEngine());
  e->device_ = device;
  e->max_items_ = max_items;
  int prev = 0;
  if (cudaGetDevice(&prev) != cudaSuccess) return ErrorCode::FABRIC_ERROR;
  if (cudaSetDevice(device) != cudaSuccess) return ErrorCode::FABRIC_ERROR;
  const size_t tab_bytes = stride_table_offset(max_items) + static_cast<size_t>(max_items) * sizeof(XferStride);
  const size_t res_bytes = static_cast<size_t>(max_items) * 12;
  bool ok = true;
  for (int i = 0; i < slots && ok; ++i) {
    auto s = std::make_unique<Slot>();
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&s->h_tab), tab_bytes) == cudaSuccess;
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&s->h_res), res_bytes) == cudaSuccess;
    ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_tab), tab_bytes) == cudaSuccess;
    s->tab_bytes = tab_bytes;
    ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_sum), static_cast<size_t>(max_items) * 8) == cudaSuccess;
    ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_done), static_cast<size_t>(max_items) * 4) == cudaSuccess;
    ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_digest), static_cast<size_t>(max_items) * 8) == cudaSuccess;
    ok = ok && cudaMalloc(reinterpret_cast<void**>(&s->d_status), static_cast<size_t>(max_items) * 4) == cudaSuccess;
    ok = ok && cudaMemset(s->d_sum, 0, static_cast<size_t>(max_items) * 8) == cudaSuccess;
    ok = ok && cudaMemset(s->d_done, 0, static_cast<size_t>(max_items) * 4) == cudaSuccess;
    ok = ok && cudaEventCreate(&s->ev_start) == cudaSuccess;
    ok = ok && cudaEventCreate(&s->ev_stop) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&s->ev_done, cudaEventDisableTiming) == cudaSuccess;
    e->slots_.push_back(std::move(s));
  }
  ok = ok && cudaDeviceSynchronize() == cudaSuccess;
  cudaSetDevice(prev);
  if (!ok) {
    BB_LOG(ERROR) << "XferEngine: device allocation failed: " << cudaGetErrorString(cudaGetLastError());
    return ErrorCode::OUT_OF_MEMORY;
  }
  return e;
}

XferEngine::~XferEngine() {
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(device_);
  for (auto& s : slots_) {
    if (s->ev_done) cudaEventSynchronize(s->ev_done);
    cudaFreeHost(s->h_tab);
    cudaFreeHost(s->h_res);
    cudaFree(s->d_tab);
    cudaFree(s->d_sum);
    cudaFree(s->d_done);
    cudaFree(s->d_digest);
    cudaFree(s->d_status);
    if (s->d_debug) cudaFree(s->d_debug);
    if (s->d_trace) cudaFree(s->d_trace);
    if (s->ev_start) cudaEventDestroy(s->ev_start);
    if (s->ev_stop) cudaEventDestroy(s->ev_stop);
    if (s->ev_done) cudaEventDestroy(s->ev_done);
  }
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
  ++mailbox_launches_;
  ++launches_;
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
  mailbox_requests_ += nd;
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

XferEngine::Slot* XferEngine::free_slot() {
  for (auto& c : slots_)
    if (c->ticket == 0) return c.get();
  return nullptr;
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

// Appends the batch's page entries to the slot's table of `nd` descriptors (written up to tile_start), growing both
// copies of the table first when they are too small (the slot is idle: nothing reads them), and points every paged
// descriptor's stride entry at its first entry in the device copy.  *tab: the bytes of the table to copy to the device.
ErrorCode XferEngine::write_pages(Slot* s, uint32_t nd, size_t* tab) {
  const size_t off = page_table_offset(nd), need = off + s->pages.size() * sizeof(uint64_t);
  if (need > s->tab_bytes) {
    // both new buffers first: on a failure the slot keeps its old, still valid pair
    uint8_t *h = nullptr, *d = nullptr;
    const cudaError_t eh = cudaMallocHost(reinterpret_cast<void**>(&h), need);
    const cudaError_t ed = eh == cudaSuccess ? cudaMalloc(reinterpret_cast<void**>(&d), need) : eh;
    if (ed != cudaSuccess) {
      if (h) cudaFreeHost(h);
      cudaGetLastError();
      BB_LOG(ERROR) << "XferEngine: growing a descriptor table to " << need << " bytes failed: " << cudaGetErrorString(ed);
      return ErrorCode::OUT_OF_MEMORY;
    }
    std::memcpy(h, s->h_tab, stride_table_offset(nd));
    cudaFreeHost(s->h_tab);
    cudaFree(s->d_tab);
    s->h_tab = h;
    s->d_tab = d;
    s->tab_bytes = need;
  }
  const auto d_pages = reinterpret_cast<uint64_t>(s->d_tab + off);
  for (uint32_t k : s->paged_descs) s->strides[k].pages = d_pages + s->strides[k].pages * sizeof(uint64_t);
  s->write_strides(nd);
  std::memcpy(s->h_tab + off, s->pages.data(), s->pages.size() * sizeof(uint64_t));
  *tab = need;
  return ErrorCode::OK;
}

Result<uint64_t> XferEngine::submit(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream,
                                    bool capture_debug) {
  if (items.size() > max_items_) return ErrorCode::RESOURCE_EXHAUSTED;
  Slot* s = free_slot();
  if (!s) return ErrorCode::RESOURCE_EXHAUSTED;  // caller must wait() on outstanding tickets
  BB_CUDA(cudaSetDevice(device_));
  auto* descs = reinterpret_cast<XferDesc*>(s->h_tab);
  s->item_to_desc.assign(items.size(), -1);
  s->empties.clear();
  s->strides.clear();
  s->pages.clear();
  s->paged_descs.clear();
  uint32_t nd = 0;
  bool all_small = small_path_enabled();
  for (size_t i = 0; i < items.size(); ++i) {
    const XferItem& it = items[i];
    const bool win = it.flags & XFER_WINDOW;
    const bool strided = it.flags & XFER_STRIDED;
    const bool gather = it.flags & XFER_GATHER;
    const bool scatter = it.flags & XFER_SCATTER;
    const bool src_paged = it.pages.paged(), dst_paged = it.dst_pages.paged();
    if ((strided && !win) || (win && (strided != it.win.strided() || !it.win.valid(it.nbytes) || it.ndst != 1 ||
                                      (it.flags & (XFER_MULTIMEM | XFER_RAW_SUM)))))
      return ErrorCode::INVALID_ARGUMENT;
    // pages are the gathering load's source or the scattering store's destination, instead of rows on the same side
    if (static_cast<bool>(it.flags & XFER_PAGED) != (src_paged || dst_paged) || (src_paged && (dst_paged || it.rows.strided())) ||
        (dst_paged && it.dst_rows.strided()) || (src_paged && !it.pages.valid(it.nbytes)) ||
        (dst_paged && !it.dst_pages.valid(it.nbytes)))
      return ErrorCode::INVALID_ARGUMENT;
    if (gather != (it.rows.strided() || src_paged) ||
        (gather && ((!src_paged && !it.rows.valid()) || (it.flags & (XFER_WINDOW | XFER_STRIDED | XFER_RAW_SUM)))))
      return ErrorCode::INVALID_ARGUMENT;
    if (scatter != (it.dst_rows.strided() || dst_paged) ||
        (scatter && ((!dst_paged && !it.dst_rows.valid()) || it.ndst != 1 ||
                     (it.flags & (XFER_WINDOW | XFER_STRIDED | XFER_GATHER | XFER_MULTIMEM | XFER_RAW_SUM)))))
      return ErrorCode::INVALID_ARGUMENT;
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
    uintptr_t al = gather ? 0 : reinterpret_cast<uintptr_t>(it.src);  // gathered: source rows instead
    // strided and scattered: rows instead
    for (uint32_t r = strided || scatter ? 1 : 0; r < it.ndst; ++r) al |= reinterpret_cast<uintptr_t>(it.dst[r]);
    if ((al & 15) || (strided && !it.win.coaligned(reinterpret_cast<uintptr_t>(it.dst[0]))) ||
        (gather && !(src_paged ? it.pages.coaligned(it.nbytes) : it.rows.coaligned(reinterpret_cast<uintptr_t>(it.src), it.nbytes))) ||
        (scatter && !(dst_paged ? it.dst_pages.coaligned(it.nbytes) : it.dst_rows.coaligned(reinterpret_cast<uintptr_t>(it.dst[0]), it.nbytes))))
      return ErrorCode::INVALID_ADDRESS;
    if ((it.flags & XFER_MULTIMEM) && (it.nbytes & 15)) return ErrorCode::INVALID_ARGUMENT;
    XferDesc& d = descs[nd];
    d.src = static_cast<const uint8_t*>(it.src) + trim;
    for (uint32_t r = 0; r < kMaxDst; ++r) d.dst[r] = r < it.ndst ? it.dst[r] : nullptr;
    if (win) {  // the descriptor's byte 0 is object byte `trim`
      const StoreWindow w = it.win.rebase(trim);
      d.win.base = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(it.dst[0]) + w.base_shift(trim) + w.origin());
      d.win.lo = w.lo;
      d.win.hi = w.hi;
      if (strided) s->set_stride(nd, w);
    }
    if (src_paged) s->add_pages(nd, it.pages, nbytes);
    else if (dst_paged) s->add_pages(nd, it.dst_pages, nbytes);
    else if (gather) s->set_stride(nd, it.rows);
    else if (scatter) s->set_stride(nd, it.dst_rows);
    d.nbytes = nbytes;
    d.ndst = it.ndst;
    d.expect = it.expect;
    d.flags = it.flags;
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
  // is in flight at a time.
  using Completion = Slot::Completion;
  s->completion = Completion::EVENTS;
  if (nd && all_small && direct && !capture_debug && !tile_trace_) {
    if (nd <= kMailSlots / 2 && mailbox_enabled() && (!mb_ || mb_->outstanding == 0)) {
      bool simple = true;
      for (uint32_t i = 0; i < nd; ++i) simple = simple && descs[i].ndst == 1 && !(descs[i].flags & (XFER_MULTIMEM | XFER_WINDOW));
      if (simple && cudaStreamQuery(st) == cudaSuccess)
        s->completion = Completion::MAILBOX;
      else
        cudaGetLastError();  // cudaErrorNotReady is not sticky, but keep the error state clean
    }
    if (s->completion == Completion::EVENTS && flag_completion_enabled()) s->completion = Completion::FLAG;
  }

  if (s->completion == Completion::MAILBOX) {
    BB_TRY(mailbox_post(s, descs, nd, xalgo));
    s->ticket = next_ticket_++;
    return s->ticket;
  }
  if (nd) {
    const bool inline_tab = nd <= kInlineDescs && s->pages.empty();  // page entries live in the device table only
    if (!inline_tab) BB_CUDA(cudaMemcpyAsync(s->d_tab, s->h_tab, tab, cudaMemcpyHostToDevice, st));
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
    ++launches_;
    if (all_small && !capture_debug && !tile_trace_) ++small_launches_;
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
  s->ticket = next_ticket_++;
  return s->ticket;
}

ErrorCode XferEngine::wait(uint64_t ticket, XferResult* out) {
  Slot* s = nullptr;
  for (auto& c : slots_)
    if (c->ticket == ticket) { s = c.get(); break; }
  if (!s) return ErrorCode::NOT_FOUND;
  SlotRelease release{s->ticket};
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
    out->device_ms = 0.f;
    if (nd && s->completion == Slot::Completion::EVENTS) cudaEventElapsedTime(&out->device_ms, s->ev_start, s->ev_stop);
  }
  if (s->debug && nd) {
    debug_host_.resize(static_cast<size_t>(s->total_tiles) * tchash::kRows * tchash::kN);
    BB_CUDA(cudaMemcpy(debug_host_.data(), s->d_debug, debug_host_.size() * 4, cudaMemcpyDeviceToHost));
  }
  if (s->traced && nd) {
    trace_host_.resize(static_cast<size_t>(s->total_tiles) * 4);
    BB_CUDA(cudaMemcpy(trace_host_.data(), s->d_trace, trace_host_.size() * 8, cudaMemcpyDeviceToHost));
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
  Slot* s = free_slot();
  if (!s) return ErrorCode::RESOURCE_EXHAUSTED;
  s->ticket = next_ticket_++;
  SlotRelease release{s->ticket};
  auto* descs = reinterpret_cast<XferDesc*>(s->h_tab);
  std::vector<XferItem> scale_items(n);  // scales region of every object, hashed as a RAW_SUM slice by bb_xfer
  s->strides.clear();
  // one kernel instantiation per launch: bf16 and fp16 items share the 2-byte one, fp32 items take the 4-byte one
  const uint32_t eb = mxfp8::wide_bytes(items[0].wide_type);
  for (uint32_t i = 0; i < n; ++i) {
    const Fp8Item& it = items[i];
    const bool strided = it.win.strided();
    const bool gather = it.rows.strided();
    const bool scatter = it.dst_rows.strided();
    if (!fp8_eligible(it.n_elems)) return ErrorCode::INVALID_ARGUMENT;
    if (it.wide_type != mxfp8::Wide::BF16 && it.wide_type != mxfp8::Wide::F16 && it.wide_type != mxfp8::Wide::F32)
      return ErrorCode::INVALID_ARGUMENT;
    if (mxfp8::wide_bytes(it.wide_type) != eb) return ErrorCode::INVALID_ARGUMENT;  // mixes 2- and 4-byte wide types
    SourceRows rows;  // a gathered put's source rows, or a scattered get's destination rows, in wide bytes
    if (gather && (unpack || !it.rows.valid() || !it.rows.to_wide_bytes(eb, &rows))) return ErrorCode::INVALID_ARGUMENT;
    if (scatter && (!unpack || gather || !it.win.whole() || !it.dst_rows.valid() || !it.dst_rows.to_wide_bytes(eb, &rows)))
      return ErrorCode::INVALID_ARGUMENT;
    // a strided item's rows need not start at `wide` (row 0 of the pattern may lie before the window, or the object's
    // first element after row 0's start): the rows are checked instead
    if (((strided || gather || scatter ? 0 : reinterpret_cast<uintptr_t>(it.wide)) | reinterpret_cast<uintptr_t>(it.packed)) & 15 ||
        ((gather || scatter) && !rows.coaligned(reinterpret_cast<uintptr_t>(it.wide), eb * it.n_elems)))
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
    if (strided) {  // held to the rule submit() applies to a strided XferItem
      if (!w.coaligned(reinterpret_cast<uintptr_t>(it.wide))) return ErrorCode::INVALID_ADDRESS;
      d.win.base = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(it.wide) + w.origin());
      d.flags |= XFER_STRIDED;
      s->set_stride(i, w);
    }
    if (gather || scatter) {  // d.src (gather) or d.dst[0] (scatter) is the pattern's row 0
      d.flags |= gather ? XFER_GATHER : XFER_SCATTER;
      s->set_stride(i, rows);
    }
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
  const size_t tab = s->write_strides(n);
  BB_CUDA(cudaMemcpyAsync(s->d_tab, s->h_tab, tab, cudaMemcpyHostToDevice, st));
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
  ++launches_;
  BB_CUDA(cudaEventRecord(s->ev_stop, st));
  BB_CUDA(cudaMemcpyAsync(s->h_res, s->d_digest, static_cast<size_t>(n) * 8, cudaMemcpyDeviceToHost, st));
  // scales: for a put they were just written by the kernel above (same stream), for a get they are read twice
  XferResult sres;
  BB_TRY(run(scale_items, ChecksumAlgo::BBH64, stream, &sres));  // waits for the stream up to here
  BB_CUDA(cudaStreamSynchronize(st));
  if (out) {
    const auto* sums = reinterpret_cast<const uint64_t*>(s->h_res);
    out->digest.assign(n, 0);
    out->status.assign(n, 0);
    for (uint32_t i = 0; i < n; ++i) {
      const uint64_t total = items[i].n_elems + items[i].n_elems / 32;
      out->digest[i] = tchash::finalize(sums[i] + sres.digest[i], total);
      if (items[i].verify && out->digest[i] != items[i].expect) out->status[i] = 1;
    }
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
