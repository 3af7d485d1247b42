// XferEngine: host-side driver of the fused transfer kernel.
//
// Owns per-device descriptor rings (pinned host staging + device tables + self-cleaning digest
// workspace) so that a batched put/get costs: one small H2D copy of the descriptor table, ONE
// kernel launch, one small D2H copy of digests/status.  This is what replaces the reference
// client's per-shard `UcxContext` + endpoint create/destroy + `ucp_put_nbx` + busy-poll
// (blackbird_client.cpp:204-274, 276-351): zero per-object setup, zero per-object launches.
#pragma once
#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <vector>

#include "common/checksum.h"
#include "common/error.h"
#include "common/result.h"
#include "common/store_window.h"
#include "kernels/xfer.h"

namespace bb::gpu {

struct XferItem {
  const void* src = nullptr;
  void* dst[kMaxDst] = {nullptr, nullptr, nullptr};
  uint32_t ndst = 1;
  uint64_t nbytes = 0;
  uint64_t expect = 0;   // expected digest when flags & XFER_VERIFY
  uint32_t flags = 0;
  uint32_t tile_base = 0;  // XFER_RAW_SUM: index of this slice's first tile inside the hashed object
  // XFER_WINDOW: only the object bytes `win` selects are stored (common/store_window.h), relative to dst[0]; XFER_STRIDED
  // exactly when it has a pattern.  INVALID_ARGUMENT unless win.valid(nbytes); INVALID_ADDRESS unless a strided window is
  // win.coaligned(dst[0]).  The whole object is still read and hashed, except with ChecksumAlgo::NONE, where the engine
  // reads only the 16-byte aligned span of the window (see window_read_bytes).
  StoreWindow win;
  // Rows or pages (common/store_window.h) on one side of the transfer, which its flag names: a put's source with
  // XFER_GATHER (src is the layout's base), or a get's destination with XFER_SCATTER (dst[0] is).  A page table's base is
  // not read, and its entries are copied into the batch's device table by submit(), so the host array need only live
  // until submit() returns; submit() sets XFER_PAGED for it, and XFER_PAGE_ROWS when its pages are in-page rows (the
  // pattern is checked by mem.valid and mem.coaligned); XFER_PAGE_ROWS among the caller's flags is INVALID_ARGUMENT.
  // INVALID_ARGUMENT for a side flag without a layout or a
  // layout without one, XFER_PAGED without pages, !mem.valid(nbytes), XFER_GATHER with a null page
  // (!mem.valid_source(nbytes)), with XFER_WINDOW, XFER_STRIDED or XFER_RAW_SUM, and XFER_SCATTER with those, XFER_GATHER,
  // XFER_MULTIMEM or ndst != 1.  A scattering store's table may hold null pages: the bytes that fall in them are read and
  // hashed but not stored.  INVALID_ADDRESS unless mem.coaligned(base, nbytes), which replaces the 16-byte alignment check
  // of the base.  Blocks (SourceBlocks) take XFER_PAGED too: their ids stay on the device, the resolve kernel builds the
  // page entries on `stream` before the transfer kernel, and its verdict comes back in XferResult::verdict; a
  // scattering store's n_blocks (and n_stored) beyond SourceBlocks::kMaxDistinct is NOT_IMPLEMENTED.  The ids must be
  // ready on `stream` (stream order), and the outer array need only live until submit() returns.  Segments
  // (SourceSegments) take XFER_SEGMENTS, which submit() sets (among the caller's flags it is INVALID_ARGUMENT): the entries
  // the item's bytes touch are copied into the batch's device table like page entries, a get's null segments are read and
  // hashed but not stored, a put's are INVALID_ARGUMENT, and so is a table whose unit is not a byte.
  DeviceLayout mem;
};

// Bytes the kernel reads for `it` under `algo`: nbytes, or for a windowed item without a checksum the trimmed span
// [win.lo & ~15, win.hi) (nothing for an empty window).
inline uint64_t window_read_bytes(const XferItem& it, ChecksumAlgo algo) {
  if (!(it.flags & XFER_WINDOW) || algo != ChecksumAlgo::NONE) return it.nbytes;
  return it.win.hi > it.win.lo ? it.win.hi - (it.win.lo & ~uint64_t{15}) : 0;
}

// One object of a fused MXFP8 transfer: `wide` is the caller's tensor, of element type `wide_type` (bf16, fp16 or fp32),
// `packed` the slab location of the stored object ([E4M3 payload n_elems][E8M0 scales n_elems / 32]).  Below, "bf16
// bytes" are bytes of the wide type.
struct Fp8Item {
  void* wide = nullptr;
  // run_fp8 returns INVALID_ARGUMENT for a batch that mixes 2-byte (bf16, fp16) and 4-byte (fp32) types: each is one
  // launch of its own kernel instantiation.
  mxfp8::Wide wide_type = mxfp8::Wide::BF16;
  void* packed = nullptr;            // replica 0 (the copy a get reads)
  void* more_packed[kMaxDst - 1] = {nullptr, nullptr};  // put: further replicas written by the same tile pass
  uint32_t nreplicas = 1;            // put: 1..kMaxDst
  uint64_t n_elems = 0;   // multiple of 32 (whole MX blocks)
  uint64_t expect = 0;    // unpack + verify: digest recorded at put time
  bool verify = false;
  // Unpack only: the elements of the object that are stored (common/store_window.h), relative to `wide`; the default is
  // the whole object.  The whole packed object is still read and verified.  INVALID_ARGUMENT unless valid against
  // n_elems; INVALID_ADDRESS unless a strided window is co-aligned in bf16 bytes, as XferItem's.
  StoreWindow win;
  // The wide side's rows, pages or segments in elements, the addresses in bytes (common/store_window.h), `wide` being the
  // layout's base (not read for pages and segments): a pack's source or an unpack's destination.  The default is
  // contiguous.  run_fp8 sets XFER_GATHER or XFER_SCATTER for it, with XFER_PAGED for pages whose entries it copies into
  // the batch's device table (and XFER_PAGE_ROWS for in-page rows), or XFER_SEGMENTS for segments (a table whose unit is
  // the wide type's bytes), whose entries it copies likewise, so the host array need only live until run_fp8 returns.  An
  // MX block may straddle two pages, two in-page rows or two segments.  An unpack's table may hold null pages or
  // segments, whose elements are not stored; a pack's may not.
  // INVALID_ARGUMENT with a window, unless mem.valid(n_elems) (a pack: mem.valid_source(n_elems)), or when its wide-byte
  // arithmetic overflows;
  // INVALID_ADDRESS unless it is co-aligned in wide bytes (DeviceLayout::coaligned of b * n_elems), which replaces the
  // 16-byte alignment check of `wide`.  Blocks as XferItem's, the verdict in XferResult::verdict.  Segments whose unit is
  // not the wide type's bytes are INVALID_ARGUMENT.
  DeviceLayout mem;
};

struct XferResult {
  std::vector<uint64_t> digest;  // per item
  std::vector<uint32_t> status;  // per item: 0 ok, 1 checksum mismatch
  float device_ms = 0.f;         // kernel time (CUDA events) of the batch
  // per item: OK, or for an item laid out in blocks the resolve kernel's verdict on its ids (SourceBlocks):
  // VALUE_OUT_OF_RANGE or INVALID_ARGUMENT.  A refused item moved nothing outside the caller's tensors: a get stored
  // nothing, a put read block 0 of every slice instead of the blocks named (its digest must not be recorded).
  std::vector<ErrorCode> verdict;
};

// One engine may be shared by many host threads: submit, wait, run and run_fp8 may be called concurrently, each thread
// with its own stream.  A batch holds one slot (pinned and device descriptor table, digest workspace) from submit() to
// wait(); the setters below are configuration, to be called before the engine is shared.
class XferEngine {
 public:
  // `device` is the CUDA ordinal the kernels run on; `max_items` bounds one batch.  `slots` are allocated up front; when
  // concurrent callers hold all of them, a batch adds one more, up to kMaxSlots.
  static Result<std::unique_ptr<XferEngine>> create(int device, uint32_t max_items = 1u << 16, int slots = 4);
  static constexpr int kMaxSlots = 64;
  ~XferEngine();
  XferEngine(const XferEngine&) = delete;
  XferEngine& operator=(const XferEngine&) = delete;

  // Enqueues the whole batch on `stream` (cudaStream_t, nullptr = legacy default stream) and returns a ticket.  Does not
  // block.  RESOURCE_EXHAUSTED when kMaxSlots batches are in flight.
  Result<uint64_t> submit(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream,
                          bool capture_debug = false);
  // Blocks until the ticket's batch has finished on the device and fills `out`.
  ErrorCode wait(uint64_t ticket, XferResult* out);
  // Convenience: submit + wait.
  ErrorCode run(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream, XferResult* out);
  // Fused MXFP8 put (pack = wide -> slab) or get (unpack = slab -> wide): the wide side is read / written once, the
  // E4M3 payload is hashed on the tensor cores while it sits in shared memory, and the digest returned is the
  // BBH64 of the stored packed object (identical to hashing the output of mxfp8_pack).  Synchronous; holds two slots
  // (the fused kernel's batch and the batch that hashes the scales).
  ErrorCode run_fp8(const std::vector<Fp8Item>& items, bool unpack, void* stream, XferResult* out);
  static bool fp8_eligible(uint64_t n_elems) { return n_elems != 0 && n_elems % 32 == 0; }  // whole MX blocks

  // Raw accumulators of the last capture_debug batch: [total_tiles][128][16] (tests only; not to be read while another
  // thread waits for a capture_debug or traced batch).
  const std::vector<uint32_t>& debug_accumulators() const { return debug_host_; }
  // Diagnostics: when on, every batch records per-tile pipeline timestamps (globaltimer ns):
  // [tile][4] = load issued, landed in shared memory, store issued, slot released.  Read after wait().
  void set_tile_trace(bool on) { tile_trace_ = on; }
  const std::vector<uint64_t>& tile_trace() const { return trace_host_; }

  int device() const { return device_; }
  uint64_t launches() const { return launches_.load(std::memory_order_relaxed); }  // kernels launched so far
  // of which warp-per-object launches (xfer_small.cu)
  uint64_t small_launches() const { return small_launches_.load(std::memory_order_relaxed); }
  size_t slots() const {  // allocated slots: create()'s, plus those added for concurrent callers
    std::lock_guard<std::mutex> lk(mu_);
    return slots_.size();
  }
  // Batches made only of objects <= kSmallBytes take the warp-per-object kernel (default on; BB_XFER_SMALL=0 disables).
  void set_small_path(bool on) { small_path_ = on; }
  // Small batches (<= kDirectResults objects on the warp path) complete by a flag in pinned memory instead of CUDA
  // events (default on; BB_XFER_FLAG_COMPLETION=0 disables).  Their XferResult::device_ms is 0 (not measured).
  void set_flag_completion(bool on) { flag_completion_ = on; }
  // Batches of <= 8 single-destination small objects whose stream has nothing pending are handed to the resident mailbox
  // warp (xfer_small.cu) instead of being launched: no cudaLaunchKernel in the steady state.  Default on;
  // BB_XFER_MAILBOX=0 disables; BB_MAILBOX_LINGER_US (default 200) = how long the warp waits for the next request.
  void set_mailbox(bool on) { mailbox_on_ = on; }
  // objects served by the resident warp
  uint64_t mailbox_requests() const { return mailbox_requests_.load(std::memory_order_relaxed); }
  // incarnations of the mailbox kernel
  uint64_t mailbox_launches() const { return mailbox_launches_.load(std::memory_order_relaxed); }
  void set_max_ctas(int n) { max_ctas_ = n; }
  int last_cuda_error() const { return last_cuda_error_.load(std::memory_order_relaxed); }

 private:
  struct Slot;
  class SlotHold;
  XferEngine() = default;
  static Result<std::unique_ptr<Slot>> new_slot(uint32_t max_items);
  // Takes a free slot, or adds one, and gives it a fresh ticket: from here on no other batch can take it.
  Result<Slot*> claim_slot();
  void release_slot(Slot* s);
  ErrorCode write_tile_table(Slot* s, uint32_t nd);
  ErrorCode write_pages(Slot* s, uint32_t nd, size_t* tab);
  ErrorCode launch_resolve(Slot* s, uint32_t nd, void* stream);
  static size_t jobs_offset(const Slot* s, uint32_t nd);
  void read_verdicts(const Slot* s, uint32_t nitems, const std::vector<int32_t>& item_to_desc, std::vector<ErrorCode>* out) const;
  ErrorCode cuda_failed(int code, const char* what);
  int device_ = 0;
  uint32_t max_items_ = 0;
  // Guards the slot table (slots_, every slot's ticket), next_ticket_, the mailbox (mb_) and debug_host_ / trace_host_.
  // Held only for that bookkeeping (and the mailbox kernel's launch): never across a descriptor-table write, a batch's
  // launch or a wait.  A claimed slot's other fields belong to the thread that claimed it.
  mutable std::mutex mu_;
  std::vector<std::unique_ptr<Slot>> slots_;
  int growing_ = 0;  // slots being allocated outside mu_, counted against kMaxSlots
  uint64_t next_ticket_ = 1;
  std::atomic<uint64_t> launches_{0};
  std::atomic<uint64_t> small_launches_{0};
  bool small_path_ = true;
  bool flag_completion_ = true;
  bool mailbox_on_ = true;
  bool mailbox_enabled();
  struct Mailbox;
  std::unique_ptr<Mailbox> mb_;
  // mailbox_post and mailbox_launch_locked are called with mu_ held
  ErrorCode mailbox_post(Slot* s, const XferDesc* descs, uint32_t nd, int algo);
  ErrorCode mailbox_wait(Slot* s);
  ErrorCode mailbox_launch_locked(uint32_t first_seq);
  std::atomic<uint64_t> mailbox_requests_{0}, mailbox_launches_{0};
  bool small_path_enabled();
  bool flag_completion_enabled();
  int max_ctas_ = 0;
  std::atomic<int> last_cuda_error_{0};
  std::vector<uint32_t> debug_host_;
  bool tile_trace_ = false;
  std::vector<uint64_t> trace_host_;
};

// Device helpers used by bindings, the worker and benchmarks (all return ErrorCode).
ErrorCode device_count(int* n);
ErrorCode device_malloc(int device, uint64_t bytes, void** out);
ErrorCode device_free(int device, void* p);
ErrorCode host_alloc_pinned(uint64_t bytes, void** out);
ErrorCode host_free_pinned(void* p);
ErrorCode stream_synchronize(void* stream);
ErrorCode device_synchronize(int device);
const char* cuda_error_string(int code);
// Comparator helpers (return a cudaError_t value).
int device_memcpy_peer_async(void* dst, int dst_device, const void* src, int src_device, uint64_t nbytes, void* stream);
int device_enable_peer_access(int device, int peer);

}  // namespace bb::gpu
