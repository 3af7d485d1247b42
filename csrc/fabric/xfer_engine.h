// XferEngine: host-side driver of the fused transfer kernel.
//
// Owns per-device descriptor rings (pinned host staging + device tables + self-cleaning digest
// workspace) so that a batched put/get costs: one small H2D copy of the descriptor table, ONE
// kernel launch, one small D2H copy of digests/status.  This is what replaces the reference
// client's per-shard `UcxContext` + endpoint create/destroy + `ucp_put_nbx` + busy-poll
// (blackbird_client.cpp:204-274, 276-351): zero per-object setup, zero per-object launches.
#pragma once
#include <cstdint>
#include <memory>
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
  // Put of a strided source (common/store_window.h): src is where the pattern's row 0 starts; XFER_GATHER exactly when it
  // has a pattern.  INVALID_ARGUMENT for an invalid pattern, or one with XFER_WINDOW, XFER_STRIDED or XFER_RAW_SUM;
  // INVALID_ADDRESS unless rows.coaligned(src, nbytes), which replaces the 16-byte alignment check of src.
  SourceRows rows;
  // Get into a strided destination, the same rule on the other side: dst[0] is where the pattern's row 0 starts;
  // XFER_SCATTER exactly when it has a pattern.  INVALID_ARGUMENT for an invalid pattern, or one with XFER_WINDOW,
  // XFER_STRIDED, XFER_GATHER, XFER_MULTIMEM, XFER_RAW_SUM or ndst != 1; INVALID_ADDRESS unless
  // dst_rows.coaligned(dst[0], nbytes), which replaces the 16-byte alignment check of dst[0].
  SourceRows dst_rows;
  // Paged put source (with XFER_GATHER) or paged get destination (with XFER_SCATTER), XFER_PAGED exactly when one of them
  // is set (common/store_window.h): object byte x at addrs[(x + phase) / page] + (x + phase) % page; src, or dst[0], is
  // not read.  The page entries are copied into the batch's device table by submit(), so the host array need only live
  // until submit() returns.  INVALID_ARGUMENT for both at once, a table too short for nbytes or phase >= page, pages
  // together with a SourceRows pattern on the same side, or XFER_PAGED without its XFER_GATHER / XFER_SCATTER, with
  // XFER_WINDOW, XFER_STRIDED or XFER_RAW_SUM; the destination rules are those of rows / dst_rows.  INVALID_ADDRESS
  // unless the pages are coaligned(nbytes).
  SourcePages pages;
  SourcePages dst_pages;
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
  // Put only: the source rows in elements (common/store_window.h), `wide` being where the pattern's row 0 starts; the
  // default is a contiguous source.  run_fp8 sets XFER_GATHER exactly when it has a pattern.  INVALID_ARGUMENT for a
  // pattern on an unpack, an invalid one, or one whose bf16 byte count overflows; INVALID_ADDRESS unless it is co-aligned
  // in bf16 bytes, which replaces the 16-byte alignment check of `wide`.
  SourceRows rows;
  // Unpack only: the destination rows in elements, `wide` being where the pattern's row 0 starts; the default is a
  // contiguous destination.  run_fp8 sets XFER_SCATTER exactly when it has a pattern.  INVALID_ARGUMENT for a pattern on a
  // pack, with a window, an invalid one, or one whose bf16 byte count overflows; INVALID_ADDRESS unless it is co-aligned in
  // bf16 bytes, which replaces the 16-byte alignment check of `wide`.
  SourceRows dst_rows;
};

struct XferResult {
  std::vector<uint64_t> digest;  // per item
  std::vector<uint32_t> status;  // per item: 0 ok, 1 checksum mismatch
  float device_ms = 0.f;         // kernel time (CUDA events) of the batch
};

class XferEngine {
 public:
  // `device` is the CUDA ordinal the kernels run on; `max_items` bounds one batch.
  static Result<std::unique_ptr<XferEngine>> create(int device, uint32_t max_items = 1u << 16, int slots = 4);
  ~XferEngine();
  XferEngine(const XferEngine&) = delete;
  XferEngine& operator=(const XferEngine&) = delete;

  // Enqueues the whole batch on `stream` (cudaStream_t, nullptr = legacy default stream) and
  // returns a ticket.  Does not block (unless all slots are in flight).
  Result<uint64_t> submit(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream,
                          bool capture_debug = false);
  // Blocks until the ticket's batch has finished on the device and fills `out`.
  ErrorCode wait(uint64_t ticket, XferResult* out);
  // Convenience: submit + wait.
  ErrorCode run(const std::vector<XferItem>& items, ChecksumAlgo algo, void* stream, XferResult* out);
  // Fused MXFP8 put (pack = wide -> slab) or get (unpack = slab -> wide): the wide side is read / written once, the
  // E4M3 payload is hashed on the tensor cores while it sits in shared memory, and the digest returned is the
  // BBH64 of the stored packed object (identical to hashing the output of mxfp8_pack).  Synchronous; needs two free
  // slots (the fused kernel's batch and the batch that hashes the scales).
  ErrorCode run_fp8(const std::vector<Fp8Item>& items, bool unpack, void* stream, XferResult* out);
  static bool fp8_eligible(uint64_t n_elems) { return n_elems != 0 && n_elems % 32 == 0; }  // whole MX blocks

  // Raw accumulators of the last capture_debug batch: [total_tiles][128][16] (tests only).
  const std::vector<uint32_t>& debug_accumulators() const { return debug_host_; }
  // Diagnostics: when on, every batch records per-tile pipeline timestamps (globaltimer ns):
  // [tile][4] = load issued, landed in shared memory, store issued, slot released.  Read after wait().
  void set_tile_trace(bool on) { tile_trace_ = on; }
  const std::vector<uint64_t>& tile_trace() const { return trace_host_; }

  int device() const { return device_; }
  uint64_t launches() const { return launches_; }  // kernels launched so far
  uint64_t small_launches() const { return small_launches_; }  // of which warp-per-object launches (xfer_small.cu)
  // Batches made only of objects <= kSmallBytes take the warp-per-object kernel (default on; BB_XFER_SMALL=0 disables).
  void set_small_path(bool on) { small_path_ = on; }
  // Small batches (<= kDirectResults objects on the warp path) complete by a flag in pinned memory instead of CUDA
  // events (default on; BB_XFER_FLAG_COMPLETION=0 disables).  Their XferResult::device_ms is 0 (not measured).
  void set_flag_completion(bool on) { flag_completion_ = on; }
  // Batches of <= 8 single-destination small objects whose stream has nothing pending are handed to the resident mailbox
  // warp (xfer_small.cu) instead of being launched: no cudaLaunchKernel in the steady state.  Default on;
  // BB_XFER_MAILBOX=0 disables; BB_MAILBOX_LINGER_US (default 200) = how long the warp waits for the next request.
  void set_mailbox(bool on) { mailbox_on_ = on; }
  uint64_t mailbox_requests() const { return mailbox_requests_; }   // objects served by the resident warp
  uint64_t mailbox_launches() const { return mailbox_launches_; }   // incarnations of the mailbox kernel
  void set_max_ctas(int n) { max_ctas_ = n; }
  int last_cuda_error() const { return last_cuda_error_; }

 private:
  struct Slot;
  XferEngine() = default;
  Slot* free_slot();
  ErrorCode write_tile_table(Slot* s, uint32_t nd);
  ErrorCode write_pages(Slot* s, uint32_t nd, size_t* tab);
  ErrorCode cuda_failed(int code, const char* what);
  int device_ = 0;
  uint32_t max_items_ = 0;
  std::vector<std::unique_ptr<Slot>> slots_;
  uint64_t next_ticket_ = 1;
  uint64_t launches_ = 0;
  uint64_t small_launches_ = 0;
  bool small_path_ = true;
  bool flag_completion_ = true;
  bool mailbox_on_ = true;
  bool mailbox_enabled();
  struct Mailbox;
  std::unique_ptr<Mailbox> mb_;
  ErrorCode mailbox_post(Slot* s, const XferDesc* descs, uint32_t nd, int algo);
  ErrorCode mailbox_wait(Slot* s);
  ErrorCode mailbox_launch_locked(uint32_t first_seq);
  uint64_t mailbox_requests_ = 0, mailbox_launches_ = 0;
  bool small_path_enabled();
  bool flag_completion_enabled();
  int max_ctas_ = 0;
  int last_cuda_error_ = 0;
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
