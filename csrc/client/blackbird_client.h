// BlackbirdClient: the SDK (SURVEY C19).
//
// Parity: reference include/blackbird/client/blackbird_client.h:22-139 — BlackbirdClientOptions
// (keystone_host/port, rpc_timeout, io_parallelism), connect, object_exists, get_workers,
// get(key) -> bytes, put(key, ptr, size, cfg), put(key, vector, cfg), remove.
// New surface required by BASELINE.json: batch_put / batch_get for host buffers and for device
// pointers (the fused NVLink kernel path, installed by fabric/gpu_fabric.h as a DeviceTransport).
//
// Behavioural fixes over the reference: rpc_timeout and io_parallelism are honoured (:204-205
// ignores them); the source pointer of a shard is `data + running offset` (not `data +
// remote_addr`, bug #8); connections to workers are cached instead of re-created per call;
// every shard is checksummed and verified; reads fail over to the next replica; a failed put is
// cancelled.
#pragma once
#include <atomic>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <utility>
#include <vector>

#include "common/metrics.h"
#include "common/mxfp8.h"
#include "common/store_window.h"
#include "net/tcp.h"
#include "rpc/rpc_service.h"

namespace bb::client {

// The in-page row pattern of one paged object, (row_width, row_pitch) in its units (SourcePages); (0, 0): one row per page.
using PageRows = std::pair<uint64_t, uint64_t>;

struct BlackbirdClientOptions {
  std::string keystone_host = "127.0.0.1";
  uint16_t keystone_port = 9090;
  // HA deployments: every keystone ("host:port"); when set it replaces keystone_host/port and the control connection
  // follows the elected leader (KeystoneRpcClient::connect_any).
  std::vector<std::string> keystone_endpoints;
  int rpc_timeout_ms = 30000;
  size_t io_parallelism = 4;
  std::string node_id;        // where this client runs (locality-aware placement)
  bool register_session = false;
  // Same-host fast path: DRAM pools that their worker backs with a memfd (`shared_memory: true`) are mapped into this
  // process and shards are moved with memcpy instead of the TCP data server (the role UCX's shared-memory transports
  // play for the reference's intra-node RMA).  BB_DISABLE_SHM=1 in the environment also turns it off.
  bool enable_shm = true;
  std::string auth_token;  // shared cluster token (net/tcp.h); empty = BB_AUTH_TOKEN / open cluster
  bool encrypt_transport = false;  // secure mode of the RPC protocol (net/tcp.h); also BB_ENCRYPT_TRANSPORT=1
  std::string auth_token_ro;       // read-only membership: set this INSTEAD of auth_token (net/tcp.h); also BB_AUTH_TOKEN_RO
  // Tenant identity (common/tenant.h): set these INSTEAD of a member token.  The servers then know who is calling: keys
  // outside the tenant's grants are ACCESS_DENIED, puts beyond its budget QUOTA_EXCEEDED.  Also BB_TENANT / BB_TENANT_SECRET.
  std::string tenant, tenant_secret;
};

// One device-side transfer request of a batch (a shard).
struct DeviceShardOp {
  size_t item = 0;            // index of the object in the batch
  size_t copy = 0, shard = 0;
  const ShardPlacement* placement = nullptr;
  std::vector<const ShardPlacement*> replicas;  // same shard on the other copies (put fan-out)
  // Get: the shard bytes that are stored (common/store_window.h); the whole shard is still read and verified.  An op whose
  // window covers the shard, the default included, is a whole-shard op.
  StoreWindow win;
  // Where the shard's bytes sit in the caller's memory (common/store_window.h): a put's source or a get's destination,
  // the object's layout rebased to the shard's first byte, with its base mem_at bytes from dev_ptrs[item].  Never
  // together with a window unless contiguous or WINDOW_ROWS (the rows of the window's result, WindowRows::rebase).
  DeviceLayout mem;
  uint64_t mem_at = 0;
  // The base of `mem` given the object's; a get's also the base `win` goes with (a strided window's base is where the
  // result's row 0 lands, which does not move with the shard, unless the result lands in rows).
  const void* src(const void* obj_base) const { return static_cast<const uint8_t*>(obj_base) + mem_at; }
  void* dst(void* obj_base) const {
    return static_cast<uint8_t*>(obj_base) + (mem.kind() == DeviceLayout::WINDOW_ROWS ? mem_at : win.base_shift(mem_at));
  }
};

// One object of a fused MXFP8 transfer: the whole packed object ([E4M3 payload][E8M0 scales]) is a single shard.
struct DeviceFp8Op {
  const ShardPlacement* placement = nullptr;
  void* wide = nullptr;     // client's tensor (source of a put, destination of a get: the base of `win`)
  uint64_t n_elems = 0;
  std::vector<const ShardPlacement*> replicas;  // put: the other copies (<= 2), written by the same tile pass
  // Get: the elements that are stored (common/store_window.h); the whole packed object is still read and verified.  The
  // default is the whole object.
  StoreWindow win;
  // The wide side's layout in elements (common/store_window.h) at `wide`: a put's source or a get's destination, never
  // together with a window unless contiguous.  The packed object is one shard, so the layout is the object's own.
  DeviceLayout mem;
  // The element type of `wide`: bf16, fp16 or fp32 (common/mxfp8.h).  Ops of one call share its size (2 or 4 bytes).
  mxfp8::Wide wide_type = mxfp8::Wide::BF16;
};

// What a device batch did, one entry per op in every field.
struct DeviceBatchResult {
  std::vector<uint64_t> digests;   // put: the digest of the op's shard (MXFP8: BBH64 of the stored packed object)
  std::vector<uint32_t> status;    // get: 0 = the shard verified against its placement's digest, else a mismatch
  // OK, or the refusal of the block ids of a BLOCKS layout (SourceBlocks in common/store_window.h).  A refused op's
  // transfer touched nothing outside the caller's memory, and its digest or status means nothing.
  std::vector<ErrorCode> verdicts;
};

// Implemented by the GPU fabric: moves shards between client device buffers and worker slabs
// with the fused kernels.  Returns per-op digests (put) or verifies them (get).
class DeviceTransport {
 public:
  virtual ~DeviceTransport() = default;
  virtual bool can_reach(const ShardPlacement& s) const = 0;
  virtual uint64_t launches() const = 0;
  // submit_* enqueues a batch and returns a ticket, so the caller can overlap control-plane round trips of the next chunk
  // with this one's transfer; wait() blocks until it is done and fills its result.  dev_ptrs[item] is the device buffer of
  // object `item`.  A put digests every op; a get verifies each shard with its placement's algorithm.
  virtual Result<uint64_t> submit_put(const std::vector<DeviceShardOp>& ops, const std::vector<const void*>& dev_ptrs, ChecksumAlgo algo,
                                      void* stream) = 0;
  virtual Result<uint64_t> submit_get(const std::vector<DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, void* stream) = 0;
  virtual ErrorCode wait(uint64_t ticket, DeviceBatchResult* res) = 0;
  // True when the shard lives in this client's own device memory (a get from it never leaves the GPU).
  virtual bool is_local(const ShardPlacement& s) const { return false; }
  virtual size_t max_in_flight() const { return 1; }
  // Prometheus lines of the transport's own counters (bytes per path, launches, ...); appended to the client's metrics.
  virtual std::string metrics_text() const { return {}; }
  virtual bool fp8_eligible(uint64_t n_elems) const { return false; }
  // Fused MXFP8 put (pack inside the transfer kernel) or, with `unpack`, get, synchronous.  Objects must satisfy
  // fp8_eligible().
  virtual ErrorCode run_fp8(const std::vector<DeviceFp8Op>& ops, bool unpack, void* stream, DeviceBatchResult* res) {
    return ErrorCode::NOT_IMPLEMENTED;
  }
  // Staging copies for objects (or shards) that live on host tiers, synchronous: object bytes [0, n) laid out by `layout`
  // at `base` (common/store_window.h) from / to n bytes packed back to back at `host`.  copy_to_device skips null pages;
  // copy_from_device refuses them (INVALID_ARGUMENT).  A BLOCKS layout is NOT_IMPLEMENTED on a GPU: the host cannot read
  // its ids without synchronising.
  virtual ErrorCode copy_from_device(void* host, const void* base, const DeviceLayout& layout, size_t n, void* stream) {
    return ErrorCode::NOT_IMPLEMENTED;
  }
  virtual ErrorCode copy_to_device(void* base, const DeviceLayout& layout, const void* host, size_t n, void* stream) {
    return ErrorCode::NOT_IMPLEMENTED;
  }
};

class HostLoopbackTransport;

class BlackbirdClient {
 public:
  explicit BlackbirdClient(BlackbirdClientOptions opts = {});
  // In-process deployment: talk to a KeystoneApi directly (no TCP to the control plane).
  BlackbirdClient(std::shared_ptr<rpc::KeystoneApi> keystone, BlackbirdClientOptions opts = {});
  ~BlackbirdClient();

  ErrorCode connect();
  bool connected() const { return keystone_ != nullptr; }
  const std::string& session_id() const { return session_id_; }

  // ---- reference API
  Result<bool> object_exists(const ObjectKey& key);
  Result<std::vector<CopyPlacement>> get_workers(const ObjectKey& key);
  Result<std::vector<uint8_t>> get(const ObjectKey& key);
  ErrorCode get_into(const ObjectKey& key, void* buf, size_t capacity, size_t* out_size);
  ErrorCode put(const ObjectKey& key, const uint8_t* data, size_t size, const WorkerConfig& cfg = {});
  ErrorCode put(const ObjectKey& key, const std::vector<uint8_t>& data, const WorkerConfig& cfg = {}) {
    return put(key, data.data(), data.size(), cfg);
  }
  ErrorCode remove(const ObjectKey& key);
  // bf16 tensors stored as MXFP8 (common/mxfp8.h layout) with the pack fused into the put kernel and the unpack
  // into the get kernel.  n_elems[i] must be a multiple of 32 (whole MX blocks; pad + mxfp8_pack otherwise); up to 3 copies
  // (written by one tile pass: converted once, stored to every replica; gets fail over between them), one
  // shard per object.  The stored object is identical to packing first and putting the packed bytes.
  //
  // Every fp8 call takes a trailing `wide`: the element type of the tensors on the device side, bf16 (the default), fp16
  // or fp32, the same for the whole call.  The packed format does not depend on it (common/mxfp8.h): a bf16-representable
  // tensor packs to the same bytes from any type, and any packed object can be read into any type.  Below, "2 * x"
  // bytes and "% 8" elements are stated for 2-byte types: with b = wide_bytes(wide) they are b * x bytes and
  // % (16 / b) elements (4 for fp32).  The *_bytes_total metrics count wide bytes.
  std::vector<ErrorCode> batch_put_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                              const std::vector<uint64_t>& n_elems, const WorkerConfig& cfg, void* stream,
                                              mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Packed puts of sliced bf16 tensors (`kv[:, h0:h1, :]`, `W[:, k0:k1]`, `t[::k]`): object i holds the rows[i] *
  // elem_widths[i] elements of rows[i] rows of elem_widths[i] elements, row r read from bf16_ptrs[i] + 2 * r *
  // elem_pitches[i] (SourceRows in common/store_window.h, in elements).  The put kernel gathers the rows while it packs, so
  // no contiguous copy is made; the stored packed object and its digest are byte for byte those of batch_put_device_fp8
  // of the compacted rows, so every fp8 get reads it.  Placement, replica fan-out and errors are batch_put_device_fp8's.
  // Per object, the shaped calls' admission (shaped_put) of SourceRows::from_rows: INVALID_ARGUMENT for elem_widths[i] >
  // elem_pitches[i] with rows[i] > 1; co-aligned means bf16_ptrs[i] 16-byte aligned and, for rows[i] > 1,
  // (elem_pitches[i] - elem_widths[i]) % 8 == 0.  rows[i] == 1 or elem_widths[i] == elem_pitches[i] is exactly
  // batch_put_device_fp8 of one contiguous tensor.
  std::vector<ErrorCode> batch_put_device_fp8_strided(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                                      const std::vector<uint64_t>& elem_widths, const std::vector<uint64_t>& elem_pitches,
                                                      const std::vector<uint64_t>& rows, const WorkerConfig& cfg, void* stream,
                                                      mxfp8::Wide wide = mxfp8::Wide::BF16);
  std::vector<ErrorCode> batch_get_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                              const std::vector<uint64_t>& n_elems, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Element-range gets of packed tensors: elements [elem_offsets[i], elem_offsets[i] + elem_counts[i]) of the n_elems[i]-element
  // object i, unpacked to bf16, land at bf16_ptrs[i].  The whole packed object is read and verified against its digest (a
  // corrupt byte outside the range still fails that copy over to the next replica); only the range is unpacked and stored,
  // and no byte outside it is ever written.  Per object: VALUE_OUT_OF_RANGE when the range passes n_elems or overflows; a
  // zero count is OK and moves nothing; NOT_IMPLEMENTED when the object is not fusable (as batch_get_device_fp8) or when
  // the virtual base bf16_ptrs[i] - 2 * elem_offsets[i] is not 16-byte aligned -- the rest of the batch still takes the
  // fused launch.  On CHECKSUM_MISMATCH the range's contents are unspecified.
  std::vector<ErrorCode> batch_get_device_fp8_range(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                    const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_offsets,
                                                    const std::vector<uint64_t>& elem_counts, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Strided gets of packed tensors (a slice along an inner dimension): rows[i] rows of elem_widths[i] elements, row r being
  // elements [elem_offsets[i] + r * elem_pitches[i], + elem_widths[i]) of the n_elems[i]-element object i, unpacked to bf16,
  // land densely at bf16_ptrs[i] + 2 * r * elem_widths[i].  The whole packed object is read and verified (a corrupt byte
  // in a gap between rows still fails that copy over to the next replica); only the rows are unpacked and stored, and no
  // byte outside them is ever written.  Per object: INVALID_ARGUMENT for elem_widths[i] > elem_pitches[i] with rows[i] > 1;
  // VALUE_OUT_OF_RANGE when the last row passes n_elems or the arithmetic overflows; OK with nothing read for rows[i] == 0
  // or elem_widths[i] == 0; Keystone errors as before; NOT_IMPLEMENTED when the object is not fusable (as
  // batch_get_device_fp8), or when the virtual base bf16_ptrs[i] - 2 * elem_offsets[i] is not 16-byte aligned or, for
  // rows[i] > 1, (elem_pitches[i] - elem_widths[i]) % 8 != 0 -- the rest of the batch still takes the fused launch.
  // rows[i] == 1, and rows that touch, are batch_get_device_fp8_range.
  std::vector<ErrorCode> batch_get_device_fp8_strided(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                      const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_offsets,
                                                      const std::vector<uint64_t>& elem_widths, const std::vector<uint64_t>& elem_pitches,
                                                      const std::vector<uint64_t>& rows, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Gets of packed tensors into sliced bf16 tensors the caller owns: object i (n_elems[i] elements) is unpacked into rows[i]
  // rows of elem_widths[i] elements, row r at bf16_ptrs[i] + 2 * r * elem_pitches[i] (SourceRows in common/store_window.h,
  // in elements), by the scattering store of the fused unpack.  No element outside the rows is ever written.  Fail-over
  // and the placement refresh are batch_get_device_fp8's.  Per object, the shaped calls' admission (shaped_get) of
  // SourceRows::from_rows: INVALID_ARGUMENT for elem_widths[i] > elem_pitches[i] with rows[i] > 1 or unless rows[i] *
  // elem_widths[i] == n_elems[i].  Then NOT_IMPLEMENTED when the object is not fusable (as batch_get_device_fp8), or
  // unless bf16_ptrs[i] is 16-byte aligned and, for rows[i] > 1, (elem_pitches[i] - elem_widths[i]) % 8 == 0 -- there is
  // no host-staged path; the rest of the batch keeps the fused launch.  rows[i] == 1 or elem_widths[i] ==
  // elem_pitches[i] is batch_get_device_fp8.
  // Strided or range gets of packed tensors into slices of tensors the caller owns (a TP rank's shard of a stored weight
  // into its place in a fused parameter): the window of batch_get_device_fp8_strided (rows[i] rows of elem_widths[i]
  // elements every elem_pitches[i] from elem_offsets[i]; a range is one row), whose dense result lands in rows of
  // dst_widths[i] elements every dst_pitches[i] elements from bf16_ptrs[i] (WindowRows in common/store_window.h, in
  // elements): result element p at bf16_ptrs[i] + 2 * ((p / dst_widths[i]) * dst_pitches[i] + p % dst_widths[i]).  The
  // whole packed object is read and verified, only the window is unpacked into the rows, and no element outside them is
  // ever written.  Per object, the window's errors as batch_get_device_fp8_strided; INVALID_ARGUMENT for dst_widths[i]
  // == 0 with a non-empty result or dst_widths[i] > dst_pitches[i] when the result spans several rows; NOT_IMPLEMENTED
  // when the object is not fusable or the item fails WindowRows::fused_get_aligned in wide bytes (the first stored
  // element's destination congruent to twice its index mod 16, and (pitches - widths) % 8 == 0 for both patterns) --
  // there is no host-staged path; the rest of the batch keeps the fused launch.  dst_widths[i] == dst_pitches[i] is
  // batch_get_device_fp8_strided.
  std::vector<ErrorCode> batch_get_device_fp8_strided_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                              const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_offsets,
                                                              const std::vector<uint64_t>& elem_widths, const std::vector<uint64_t>& elem_pitches,
                                                              const std::vector<uint64_t>& rows, const std::vector<uint64_t>& dst_widths,
                                                              const std::vector<uint64_t>& dst_pitches, void* stream,
                                                              mxfp8::Wide wide = mxfp8::Wide::BF16);
  std::vector<ErrorCode> batch_get_device_fp8_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                      const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_widths,
                                                      const std::vector<uint64_t>& elem_pitches, const std::vector<uint64_t>& rows,
                                                      void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Packed puts of paged tensors (the blocks of a paged KV cache, one object for a whole request): object i is the
  // concatenation of the pages[i].size() pages of page_elems[i] elements at the device addresses pages[i], in list order
  // (SourcePages in common/store_window.h, page size in elements, addresses in bytes).  The pack kernel reads each page in
  // place; an MX block may straddle two pages.  The stored packed object and its digest are byte for byte those of
  // batch_put_device_fp8 of the concatenation, so every fp8 get reads it.  Placement, replica fan-out and errors are
  // batch_put_device_fp8's.  Per object, the shaped calls' admission (shaped_put) of SourcePages::from_pages:
  // INVALID_ARGUMENT for page_elems[i] == 0 with pages; co-aligned means every page 16-byte aligned and, for several
  // pages, page_elems[i] % 8 == 0.
  std::vector<ErrorCode> batch_put_device_fp8_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                    const std::vector<uint64_t>& page_elems, const WorkerConfig& cfg, void* stream,
                                                    mxfp8::Wide wide = mxfp8::Wide::BF16, const std::vector<PageRows>& page_rows = {});
  // Gets of packed tensors into pages, the mirror: object i is unpacked into the pages pages[i] of page_elems[i] elements,
  // element x in page x / page_elems[i] at element x % page_elems[i], by the paged scattering store of the fused unpack.
  // Only the object's elements are written; pages of one get must not overlap (not checked).  A zero page address is a
  // page that is not stored (SourcePages' null page): a partial restore names only the pages it wants and leaves the
  // others 0.  The table still covers the whole object, which is still read whole and verified, so a corrupt copy fails
  // over even when no page is stored.  Fail-over and the placement refresh are batch_get_device_fp8's.  Per object, the
  // shaped calls' admission (shaped_get) of SourcePages::from_pages: INVALID_ARGUMENT for page_elems[i] == 0 with pages.
  // Then INVALID_ARGUMENT unless the stored object holds exactly pages[i].size() * page_elems[i] elements;
  // NOT_IMPLEMENTED when the object is not fusable (as batch_get_device_fp8) or the pages fail
  // SourcePages::fused_get_aligned in wide bytes -- there is no host-staged path; the rest of the batch keeps the fused
  // launch.
  std::vector<ErrorCode> batch_get_device_fp8_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                    const std::vector<uint64_t>& page_elems, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16,
                                                    const std::vector<PageRows>& page_rows = {});
  // Packed puts and gets from block ids that stay on the device: batch_put_device_blocks and batch_get_device_blocks for
  // packed tensors, `page` counted in elements of `wide` (the stride and slice addresses in bytes), with the rules of
  // batch_put_device_fp8_paged and batch_get_device_fp8_paged.  Per object, the shaped calls' admission (shaped_put,
  // shaped_get) of SourceBlocks::from_blocks, whose shape errors are the byte calls'.  Then, on a get, INVALID_ARGUMENT
  // unless the element count is exactly the stored object's, and NOT_IMPLEMENTED when the object is not fusable or the
  // table fails SourceBlocks::fused_get_aligned in wide bytes -- there is no host-staged path.  After the transfer the
  // device's verdict on the ids answers the object as for the byte calls: a refused put is cancelled, a refused get
  // stores nothing and is not retried.
  std::vector<ErrorCode> batch_put_device_fp8_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks,
                                                     const WorkerConfig& cfg, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
  std::vector<ErrorCode> batch_get_device_fp8_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks, void* stream,
                                                     mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Packed segment-list puts (a list of bf16, fp16 or fp32 tensors as one packed object): object i is the concatenation of
  // the segments segments[i], each a (device address, elements of `wide`) pair, in list order (SourceSegments with the
  // unit of the wide type, common/store_window.h).  The pack kernel reads each segment in place; an MX block may straddle
  // two segments.  The stored packed object and its digest are byte for byte those of batch_put_device_fp8 of the
  // concatenation, so every fp8 get reads it.  Placement, replica fan-out and errors are batch_put_device_fp8's.  Per
  // object, the shaped calls' admission (shaped_put) of SourceSegments::from_segments: zero-length segments are dropped,
  // VALUE_OUT_OF_RANGE when the total's bytes overflow, INVALID_ARGUMENT for a segment at address 0 and for an element
  // total that is 0 or not a multiple of 32, NOT_IMPLEMENTED unless co-aligned in wide bytes (address = b * element
  // offset mod 16 for every segment) -- there is no host-staged packed put.
  std::vector<ErrorCode> batch_put_device_fp8_segments(const std::vector<ObjectKey>& keys,
                                                       const std::vector<std::vector<SourceSegments::Segment>>& segments, const WorkerConfig& cfg,
                                                       void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
  // Gets of packed objects into segments, the mirror: object i is unpacked into the segments segments[i] in list order,
  // by the segmented scattering store of the fused unpack; out_sizes[i] receives its elements.  A segment at address 0
  // is not stored (a null segment): its elements are still read, unpacked and verified, so a partial restore names only
  // the segments it wants.  Fail-over and the placement refresh are batch_get_device_fp8's.  Admission as
  // batch_put_device_fp8_segments', null segments allowed and co-alignment not checked there.  Then INVALID_ARGUMENT
  // unless the stored object holds exactly the segments' element total, null segments counted; NOT_IMPLEMENTED when the
  // object is not fusable (as batch_get_device_fp8) or the segments fail SourceSegments::fused_get_aligned in wide bytes
  // -- there is no host-staged path; the rest of the batch keeps the fused launch.
  std::vector<ErrorCode> batch_get_device_fp8_segments(const std::vector<ObjectKey>& keys,
                                                       const std::vector<std::vector<SourceSegments::Segment>>& segments, void* stream,
                                                       std::vector<size_t>* out_sizes, mxfp8::Wide wide = mxfp8::Wide::BF16);
  bool device_fp8_eligible(uint64_t n_elems) const { return device_ && device_->fp8_eligible(n_elems); }
  // Moves every copy of the object to `target` (promotion to the GPU tier, demotion to DRAM / NVMe ...).
  ErrorCode migrate(const ObjectKey& key, StorageClass target);

  // ---- batched host-memory API
  std::vector<ErrorCode> batch_put(const std::vector<ObjectKey>& keys, const std::vector<const uint8_t*>& data,
                                   const std::vector<size_t>& sizes, const WorkerConfig& cfg = {});
  std::vector<Result<std::vector<uint8_t>>> batch_get(const std::vector<ObjectKey>& keys);
  std::vector<ErrorCode> batch_remove(const std::vector<ObjectKey>& keys);
  std::vector<Result<bool>> batch_exists(const std::vector<ObjectKey>& keys);

  // ---- batched device-memory API (fused kernels; requires a DeviceTransport)
  void set_device_transport(std::shared_ptr<DeviceTransport> t) { device_ = std::move(t); }
  std::vector<ErrorCode> batch_put_device(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs,
                                          const std::vector<size_t>& sizes, const WorkerConfig& cfg, void* stream);
  // Puts of strided sources (a slice of a larger tensor along an inner dimension): object i is the rows[i] * widths[i]
  // bytes of rows[i] rows of widths[i] bytes, row r read from dev_ptrs[i] + r * pitches[i] (SourceRows in
  // common/store_window.h).  The stored object and its digests are those of batch_put_device of the compacted rows, so
  // every get reads it.  The fused path gathers the rows in the put kernel; it needs dev_ptrs[i] 16-byte aligned, for
  // rows[i] > 1 (pitches[i] - widths[i]) % 16 == 0, and every shard start 16-byte aligned.  Any other item, and every
  // placement the fabric cannot reach, is staged through the host (one copy of the source extent, rows compacted there)
  // while the rest of the batch keeps the fused launch.  Per object, the shaped calls' admission (shaped_put) of
  // SourceRows::from_rows: INVALID_ARGUMENT for widths[i] > pitches[i] with rows[i] > 1.  rows[i] == 1 or widths[i] ==
  // pitches[i] is exactly batch_put_device of one contiguous block, rows[i] == 0 or widths[i] == 0 that of a zero-byte
  // object.
  std::vector<ErrorCode> batch_put_device_strided(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs,
                                                  const std::vector<uint64_t>& widths, const std::vector<uint64_t>& pitches,
                                                  const std::vector<uint64_t>& rows, const WorkerConfig& cfg, void* stream);
  // out_sizes[i] receives the object size; buffers must be large enough (capacity[i]).
  std::vector<ErrorCode> batch_get_device(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                          const std::vector<size_t>& capacity, void* stream, std::vector<size_t>* out_sizes);
  // Byte-range gets: bytes [offsets[i], offsets[i] + lengths[i]) of object i land at dev_ptrs[i].  Every shard that overlaps
  // a range is read whole and verified against its digest (a corrupt byte outside the range still fails that copy over to
  // the next replica); shards outside the range are not touched.  A range whose virtual base dev_ptrs[i] - offsets[i] is
  // not 16-byte aligned at the start of every shard of every copy is staged through the host, like a misaligned
  // batch_get_device (StoreWindow::fused_get_aligned).  Per-object VALUE_OUT_OF_RANGE when the range passes the end of the
  // object.
  std::vector<ErrorCode> batch_get_device_range(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                const std::vector<uint64_t>& offsets, const std::vector<uint64_t>& lengths, void* stream);
  // Strided gets (a slice along an inner dimension): rows[i] rows of widths[i] bytes, row r being object bytes
  // [offsets[i] + r * pitches[i], + widths[i]), land densely at dev_ptrs[i] + r * widths[i].  Every shard that holds a stored
  // byte is read whole and verified; shards that hold none (outside the rows, or wholly inside a gap between them) are not
  // touched.  The fused path needs the virtual base dev_ptrs[i] - offsets[i] 16-byte aligned at the start of every shard
  // it reads and, for rows[i] > 1, (pitches[i] - widths[i]) % 16 == 0; any other item is staged through the host (its rows
  // compacted there, one H2D copy) while the rest of the batch keeps the fused launch.  Per object: INVALID_ARGUMENT for
  // widths[i] > pitches[i] with rows[i] > 1; VALUE_OUT_OF_RANGE when the last row passes the end of the object or the
  // arithmetic overflows; OK with nothing read for rows[i] == 0 or widths[i] == 0; Keystone errors as for
  // batch_get_device_range.  rows[i] == 1 is batch_get_device_range of (offsets[i], widths[i]).
  std::vector<ErrorCode> batch_get_device_strided(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                  const std::vector<uint64_t>& offsets, const std::vector<uint64_t>& widths,
                                                  const std::vector<uint64_t>& pitches, const std::vector<uint64_t>& rows, void* stream);
  // Gets into strided destinations (a slice of a tensor the caller owns, `cache[layer, :, slot]`, `W[:, k0:k1]`): object i
  // lands in rows[i] rows of widths[i] bytes, row r at dev_ptrs[i] + r * pitches[i] (SourceRows in common/store_window.h),
  // object byte x at row x / widths[i], column x % widths[i].  The capacity is rows[i] * widths[i]: a larger object is
  // BUFFER_OVERFLOW, a shorter one fills its bytes in row order; out_sizes[i] receives the size.  No byte outside the
  // object's bytes of the rows is ever written.  Every shard is read whole and verified, with fail-over and the placement
  // refresh of batch_get_device.  The fused path scatters the rows in the get kernel; it needs dev_ptrs[i] 16-byte aligned,
  // for rows[i] > 1 (pitches[i] - widths[i]) % 16 == 0, and every shard start 16-byte aligned.  Any other item, and every
  // placement the fabric cannot reach, is staged through the host (one 2-D H2D copy of the rows) while the rest of the
  // batch keeps the fused launch.  Per object, the shaped calls' admission (shaped_get) of SourceRows::from_rows:
  // INVALID_ARGUMENT for widths[i] > pitches[i] with rows[i] > 1.  rows[i] == 1 or widths[i] == pitches[i] is exactly
  // batch_get_device with capacity rows[i] * widths[i].
  // Strided or range gets into slices of tensors the caller owns (`out[:, h0:h1, :]`, a TP shard into a fused
  // parameter): the window of batch_get_device_strided (rows[i] rows of widths[i] bytes every pitches[i] from
  // offsets[i]; a range is one row), whose dense result lands in rows of dst_widths[i] bytes every dst_pitches[i] bytes
  // from dev_ptrs[i] (WindowRows in common/store_window.h): result byte p at dev_ptrs[i] + (p / dst_widths[i]) *
  // dst_pitches[i] + p % dst_widths[i].  Shards are read and verified as for batch_get_device_strided, with its
  // fail-over and placement refresh, and no byte outside the destination rows is ever written.  The fused path stores
  // the window's pieces in the get kernel; it needs WindowRows::fused_get_aligned for every shard of every copy (both
  // gaps multiples of 16 bytes, each shard's first stored byte at an address congruent to its offset mod 16).  Any other
  // item, and every placement the fabric cannot reach, is staged through the host (the window compacted there, one 2-D
  // H2D copy into the rows).  Per object, the window's errors as batch_get_device_strided; INVALID_ARGUMENT for
  // dst_widths[i] == 0 with a non-empty result or dst_widths[i] > dst_pitches[i] when the result spans several rows.
  // dst_widths[i] == dst_pitches[i] is batch_get_device_strided.
  std::vector<ErrorCode> batch_get_device_strided_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                          const std::vector<uint64_t>& offsets, const std::vector<uint64_t>& widths,
                                                          const std::vector<uint64_t>& pitches, const std::vector<uint64_t>& rows,
                                                          const std::vector<uint64_t>& dst_widths, const std::vector<uint64_t>& dst_pitches,
                                                          void* stream);
  std::vector<ErrorCode> batch_get_device_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                  const std::vector<uint64_t>& widths, const std::vector<uint64_t>& pitches,
                                                  const std::vector<uint64_t>& rows, void* stream, std::vector<size_t>* out_sizes);
  // Paged puts (the blocks of a paged KV cache, one object for a whole request): object i is the concatenation of the
  // pages[i].size() pages of page_bytes[i] bytes at the device addresses pages[i], in list order (SourcePages in
  // common/store_window.h); one object, one metadata record.  A page may repeat.  The stored object and its digests are
  // those of batch_put_device of the concatenation, so every get reads it.  The fused path reads each page in place in
  // the put kernel; it needs every shard of every copy co-aligned (SourcePages::coaligned: 16-byte aligned pages and shard starts and, for
  // several pages, page_bytes[i] % 16 == 0).  Any other item, and every placement the fabric cannot reach, is staged
  // through the host (one D2H copy per run of pages) while the rest of the batch keeps the fused launch.  Per object, the
  // shaped calls' admission (shaped_put) of SourcePages::from_pages: INVALID_ARGUMENT for page_bytes[i] == 0 with pages.
  // No pages is a zero-byte object.  page_rows (PageRows), empty or one per object, makes every page of object i rows of
  // page_rows[i].first bytes every page_rows[i].second bytes inside its block (a head slice of a KV block; (0, 0): one
  // row), under the from_pages rules of the pattern; co-aligned then also needs a gap between rows that is a multiple
  // of 16 bytes.  The four paged calls, byte and MXFP8, take it alike (MXFP8 in elements); SourceBlocks carries its own.
  std::vector<ErrorCode> batch_put_device_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                const std::vector<uint64_t>& page_bytes, const WorkerConfig& cfg, void* stream,
                                                const std::vector<PageRows>& page_rows = {});
  // Paged gets, the mirror: object i lands in the pages pages[i] of page_bytes[i] bytes, object byte x in page
  // x / page_bytes[i] at offset x % page_bytes[i].  The capacity is pages[i].size() * page_bytes[i]: a larger object is
  // BUFFER_OVERFLOW, a shorter one fills its bytes in page order; out_sizes[i] receives the size.  Only the object's bytes
  // are written.  Pages of one get must not overlap (not checked).  A zero page address is a page that is not stored
  // (SourcePages' null page): a partial restore names only the pages it wants and leaves the others 0; the capacity and
  // out_sizes rules do not change.  Every shard is read whole and verified, stored pages or not, with the
  // fail-over and placement refresh of batch_get_device.  The fused path scatters the pages in the get kernel; it needs
  // SourcePages::fused_get_aligned for every shard of every copy.  Any other item, and every placement the fabric cannot
  // reach, is staged through the host (one H2D copy per run of pages).  Per object, the shaped calls' admission
  // (shaped_get) of SourcePages::from_pages: INVALID_ARGUMENT for page_bytes[i] == 0 with pages.
  std::vector<ErrorCode> batch_get_device_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                const std::vector<uint64_t>& page_bytes, void* stream, std::vector<size_t>* out_sizes,
                                                const std::vector<PageRows>& page_rows = {});
  // Paged puts from block ids that stay on the device: object i is the pages of blocks[i] (SourceBlocks in
  // common/store_window.h: outer slice q, block ids[k], page r = q * n_ids + k at outer[q] + ids[k] * stride), in page
  // order, as batch_put_device_paged of that table would store it.  The ids are read on `stream` by the transfer
  // engine's resolve kernel, after the work queued there before the call; the host never reads them, and no host work
  // depends on their number beyond the small outer array.  Placement, replica fan-out and digests are
  // batch_put_device_paged's.  Per object, the shaped calls' admission (shaped_put) of SourceBlocks::from_blocks:
  // INVALID_ARGUMENT for page == 0 with pages or ids other than 4 or 8 bytes.  After the transfer, from the device:
  // VALUE_OUT_OF_RANGE for an id outside [0, n_blocks); the put is then cancelled, nothing is stored and the rest of the
  // batch carries on.  NOT_IMPLEMENTED when the table is not co-aligned (SourceBlocks::coaligned) or a placement is not on
  // the GPU fabric: there is no host-staged path; the put is cancelled.
  std::vector<ErrorCode> batch_put_device_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks,
                                                 const WorkerConfig& cfg, void* stream);
  // Paged gets into blocks named by device-resident ids, the mirror: object i lands in the pages of blocks[i], with a
  // selection (sel, n_stored) as a partial restore: only the pages of the stored blocks sel[m] land, in block ids[m], and
  // the others are not stored.  The capacity is the table's size; out_sizes[i] receives the object's size.  Every shard
  // is read whole and verified, with the fail-over and placement refresh of batch_get_device.  Per object, the shaped
  // calls' admission (shaped_get) of SourceBlocks::from_blocks: INVALID_ARGUMENT for page == 0 with pages or ids other
  // than 4 or 8 bytes.  Then BUFFER_OVERFLOW for a larger object; NOT_IMPLEMENTED when the table fails
  // SourceBlocks::fused_get_aligned or no copy is on the GPU fabric.  After the transfer, from the device:
  // VALUE_OUT_OF_RANGE for an id (or selection entry) out of range, INVALID_ARGUMENT for a repeated one; then nothing
  // of the object is stored, it is not retried on another replica, and the rest of the batch carries on.
  std::vector<ErrorCode> batch_get_device_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks, void* stream,
                                                 std::vector<size_t>* out_sizes);
  // Segment-list puts (the tensors of a state_dict, a request's per-layer state of several sizes, as one object):
  // object i is the concatenation of the segments segments[i], each a (device address, bytes) pair, in list order
  // (SourceSegments in common/store_window.h); one object, one metadata record, one digest set, one placement.  The stored
  // object and its digests are those of batch_put_device of the concatenation, so every get reads it.  The fused path
  // reads each segment in place in the put kernel; it needs every shard of every copy co-aligned (SourceSegments::
  // coaligned: address = object offset mod 16 for every segment, with shards cut at 16-byte multiples).  Any other item,
  // and every placement the fabric cannot reach, is staged through the host (one D2H copy per run of segments) while the
  // rest of the batch keeps the fused launch.  Per object, the shaped calls' admission (shaped_put) of
  // SourceSegments::from_segments: zero-length segments are dropped, VALUE_OUT_OF_RANGE when the total overflows,
  // INVALID_ARGUMENT for a segment at address 0.  No segments is a zero-byte object.
  std::vector<ErrorCode> batch_put_device_segments(const std::vector<ObjectKey>& keys, const std::vector<std::vector<SourceSegments::Segment>>& segments,
                                                   const WorkerConfig& cfg, void* stream);
  // Segment-list gets, the mirror: object i lands in the segments segments[i] in list order.  The capacity is the sum of
  // the lengths, null segments included: a larger object is BUFFER_OVERFLOW, a shorter one fills its bytes in list order;
  // out_sizes[i] receives the size.  A segment at address 0 is not stored (a null segment): a partial restore names only
  // the segments it wants.  Every shard is read whole and verified, with the fail-over and placement refresh of
  // batch_get_device.  The fused path scatters the segments in the get kernel; it needs SourceSegments::fused_get_aligned
  // for every shard of every copy.  Any other item, and every placement the fabric cannot reach, is staged through the
  // host (one H2D copy per run of segments).  Admission as batch_put_device_segments', null segments allowed.
  std::vector<ErrorCode> batch_get_device_segments(const std::vector<ObjectKey>& keys, const std::vector<std::vector<SourceSegments::Segment>>& segments,
                                                   void* stream, std::vector<size_t>* out_sizes);

  Result<ClusterStats> cluster_stats();
  rpc::KeystoneApi& keystone() { return *keystone_; }
  std::string metrics_text() const { return metrics_.render("bb_client_") + (device_ ? device_->metrics_text() : std::string()); }
  // Device batches are split into `chunks` pipelined launches; 0 = decide from the measured RPC latency.
  void set_device_pipeline_chunks(size_t chunks) { pipeline_chunks_ = chunks; }
  std::map<std::string, std::vector<double>> phase_summary() const { return metrics_.histogram_summary(); }

 private:
  friend class HostLoopbackTransport;
  struct WorkerConn;
  std::shared_ptr<net::RpcClient> acquire(const std::string& endpoint);
  void release(const std::string& endpoint, std::shared_ptr<net::RpcClient> c);
  ErrorCode write_shard(const ShardPlacement& s, const uint8_t* src, uint64_t* digest, ChecksumAlgo algo);
  ErrorCode read_shard(const ShardPlacement& s, uint8_t* dst, ChecksumAlgo algo);
  ErrorCode put_once(const ObjectKey& key, const uint8_t* data, size_t size, const WorkerConfig& cfg);
  ErrorCode transfer_put(const std::vector<CopyPlacement>& copies, const uint8_t* data, ChecksumAlgo algo,
                         keystone::ShardChecksums* sums);
  // Reads the object into dst[0, size) from the first copy that verifies: every shard, or with a window only those that
  // hold a byte it stores (whole, and verified).  The other bytes of dst are left as they are.
  ErrorCode transfer_get(const std::vector<CopyPlacement>& copies, uint8_t* dst, size_t size, const StoreWindow& win = {});
  // batch_get_device, batch_get_device_range, batch_get_device_strided, batch_get_device_scatter and
  // batch_get_device_paged: `ranges` null = whole objects into buffers of `capacity`, else object i's rows into dev_ptrs[i]
  // (capacity[i] = rows * length, for the chunk plan).  A range is the single row `rows == 1`.  `mem` null = contiguous
  // buffers, else object i lands by (*mem)[i] at dev_ptrs[i]: with `ranges` only a WINDOW_ROWS layout (the rows of the
  // range's result) or a contiguous one.
  struct ByteRange {
    uint64_t offset = 0, length = 0;
    uint64_t pitch = 0, rows = 1;  // row r = bytes [offset + r * pitch, + length)
  };
  // batch_put_device, batch_put_device_strided and batch_put_device_paged: `mem` null = contiguous sources, else object i
  // is read by (*mem)[i] at dev_ptrs[i].
  std::vector<ErrorCode> put_device(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs, const std::vector<size_t>& sizes,
                                    const std::vector<DeviceLayout>* mem, const WorkerConfig& cfg, void* stream);
  std::vector<ErrorCode> get_device(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs, const std::vector<size_t>& capacity,
                                    const std::vector<ByteRange>* ranges, const std::vector<DeviceLayout>* mem, void* stream,
                                    std::vector<size_t>* out_sizes);
  // batch_put_device_fp8, batch_put_device_fp8_strided and batch_put_device_fp8_paged: `mem` null = contiguous tensors,
  // else object i is read by (*mem)[i] at bf16_ptrs[i], in elements.
  std::vector<ErrorCode> put_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                        const std::vector<uint64_t>& n_elems, const std::vector<DeviceLayout>* mem, const WorkerConfig& cfg,
                                        void* stream, mxfp8::Wide wide);
  // batch_get_device_fp8, batch_get_device_fp8_range, batch_get_device_fp8_strided, batch_get_device_fp8_scatter and
  // batch_get_device_fp8_paged: `ranges` null = whole tensors, else object i's rows (offset, length and pitch in elements)
  // into bf16_ptrs[i]; `mem` (whole tensors only) null = contiguous destinations, else object i lands by (*mem)[i] at
  // bf16_ptrs[i], in elements.  An object laid out in pages must hold exactly n_elems[i] elements.
  std::vector<ErrorCode> get_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                        const std::vector<uint64_t>& n_elems, const std::vector<ByteRange>* ranges,
                                        const std::vector<DeviceLayout>* mem, void* stream, mxfp8::Wide wide);
  // The shaped batch_*_device_* calls over the four above, and the placement refresh of get_device and get_device_fp8.
  template <class Shape, class Run>
  std::vector<ErrorCode> shaped_batch(std::string_view name, bool admit, size_t n, bool arity_ok, Shape&& shape, Run&& run);
  // The strided, scatter, paged and blocks puts and gets, bytes and MXFP8 (`fp8`: the wide type).  build(i, &item) makes
  // item i's layout and size from the call's own arguments, in bytes or elements of the wide type:
  // SourceRows::from_rows, SourcePages::from_pages or SourceBlocks::from_blocks, with their errors (INVALID_ARGUMENT for
  // a shape, VALUE_OUT_OF_RANGE for an overflow).  Then one admission rule, in this order:
  //   - MXFP8 from a page table (pages, blocks): INVALID_ARGUMENT unless a positive whole number of MX blocks.  Rows
  //     are left to put_device_fp8 and get_device_fp8, which answer for a count that is not fusable;
  //   - a put: INVALID_ARGUMENT for a null page or a selection of blocks (a put reads every unit);
  //   - VALUE_OUT_OF_RANGE when the size does not fit in size_t, or for MXFP8 when the source extent or the layout
  //     overflows in wide bytes;
  //   - an MXFP8 put: NOT_IMPLEMENTED unless the layout at ptrs[i] is co-aligned in wide bytes (DeviceLayout::coaligned),
  //     as there is no host-staged path for packed puts;
  //   - a get: NOT_IMPLEMENTED when n_blocks or n_stored exceeds SourceBlocks::kMaxDistinct.
  // A refused put item never reaches the Keystone and a refused get item is not looked up; the rest of the batch goes on
  // through put_device, get_device, put_device_fp8 or get_device_fp8 (dev_ptrs[i] = ptrs[i]), whose own rules follow.
  // out_sizes, when given, is the get's, 0 for a refused item; the metrics are shaped_batch's, in wide bytes for MXFP8.
  template <class Build>
  std::vector<ErrorCode> shaped_put(std::string_view name, const std::vector<ObjectKey>& keys, const std::vector<const void*>& ptrs,
                                    bool arity_ok, std::optional<mxfp8::Wide> fp8, Build&& build, const WorkerConfig& cfg, void* stream);
  template <class Build>
  std::vector<ErrorCode> shaped_get(std::string_view name, const std::vector<ObjectKey>& keys, const std::vector<void*>& ptrs,
                                    bool arity_ok, std::optional<mxfp8::Wide> fp8, Build&& build, void* stream, std::vector<size_t>* out_sizes);
  template <class Reissue>
  void refresh_placements(const std::vector<ObjectKey>& keys, const std::vector<Result<std::vector<CopyPlacement>>>& placed,
                          std::vector<ErrorCode>& out, Reissue&& reissue);
  ErrorCode get_with_refresh(const ObjectKey& key, uint8_t* (*alloc)(void*, size_t), void* ctx, size_t capacity, size_t* out_size);
  static uint64_t shard_offset(const ShardPlacement& s);
  static ChecksumAlgo algo_of(const std::vector<CopyPlacement>& copies, ChecksumAlgo hint);
  // [begin, end) index ranges that split a batch so that transfers of one chunk overlap the
  // control-plane round trips of its neighbours (large batches only).
  std::vector<std::pair<size_t, size_t>> plan_chunks(const std::vector<size_t>& sizes, double rpc_us_per_object) const;

  // Mapped shared DRAM pools (same-host fast path); a mapping is dropped when the pool re-registers under a new key.
  struct ShmPool {
    uint8_t* base = nullptr;
    uint64_t size = 0;
    uint64_t remote_base = 0;
    std::vector<uint8_t> key;
  };
  uint8_t* shm_resolve(const ShardPlacement& s);
  std::mutex shm_mu_;
  std::map<std::string, ShmPool> shm_pools_;
  std::map<std::string, std::vector<uint8_t>> shm_unreachable_;  // pool -> key that could not be mapped

  BlackbirdClientOptions opts_;
  std::shared_ptr<rpc::KeystoneApi> keystone_;
  std::shared_ptr<DeviceTransport> device_;
  size_t pipeline_chunks_ = 0;  // 0 = adaptive (from the measured control-plane latency)
  std::atomic<double> put_rpc_us_per_obj_{0}, get_rpc_us_per_obj_{0};
  std::string session_id_;
  std::mutex conn_mu_;
  std::map<std::string, std::vector<std::shared_ptr<net::RpcClient>>> idle_conns_;
  mutable Metrics metrics_;
};

// A DeviceTransport without a GPU: "device pointers" are host pointers and shards move over the host data paths of a
// second (I/O) client.  It exists so that the device-side client logic -- chunk planning and pipelining, fan-out
// descriptors, replica choice and fail-over, host-staged fall-backs, placement refresh -- is testable on CPU-only
// machines (the reference has no fake transport at all, SURVEY section 4); the GPU fabric replaces it in production.
class HostLoopbackTransport : public DeviceTransport {
 public:
  // `io` moves the bytes (its own connections / shared-memory mappings); it must outlive the transport.
  explicit HostLoopbackTransport(std::shared_ptr<BlackbirdClient> io, bool reach_disk_tiers = false)
      : io_(std::move(io)), reach_disk_(reach_disk_tiers) {}
  // Synchronous: submit_* moves the shards and keeps the result under the ticket it returns.
  Result<uint64_t> submit_put(const std::vector<DeviceShardOp>& ops, const std::vector<const void*>& dev_ptrs, ChecksumAlgo algo,
                              void* stream) override;
  Result<uint64_t> submit_get(const std::vector<DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, void* stream) override;
  ErrorCode wait(uint64_t ticket, DeviceBatchResult* res) override;
  bool can_reach(const ShardPlacement& s) const override;
  uint64_t launches() const override { return launches_; }
  // A BLOCKS layout is resolved on the host (SourceBlocks::resolve): here the "device" ids are host memory.
  ErrorCode copy_from_device(void* host, const void* base, const DeviceLayout& layout, size_t n, void*) override {
    if (!layout.valid_source(n)) return ErrorCode::INVALID_ARGUMENT;
    std::vector<uint64_t> table;
    ErrorCode v;
    layout.resolved(n, false, &table, &v).for_each_run(reinterpret_cast<uintptr_t>(base), n, [&](uint64_t x, uint64_t addr, uint64_t len) {
      std::memcpy(static_cast<uint8_t*>(host) + x, reinterpret_cast<const void*>(addr), len);
    });
    return ErrorCode::OK;
  }
  ErrorCode copy_to_device(void* base, const DeviceLayout& layout, const void* host, size_t n, void*) override {
    std::vector<uint64_t> table;
    ErrorCode v;
    layout.resolved(n, true, &table, &v).for_each_run(reinterpret_cast<uintptr_t>(base), n, [&](uint64_t x, uint64_t addr, uint64_t len) {
      std::memcpy(reinterpret_cast<void*>(addr), static_cast<const uint8_t*>(host) + x, len);
    });
    return ErrorCode::OK;
  }
  size_t max_in_flight() const override { return 2; }
  // MXFP8 through the CPU reference codec (common/mxfp8.h): the stored object and its digest are the ones the fused
  // kernels produce, so the fp8 client logic (replica fan-out, fail-over between replicas) is testable on CPU too.
  bool fp8_eligible(uint64_t n_elems) const override { return n_elems != 0 && n_elems % 32 == 0; }
  ErrorCode run_fp8(const std::vector<DeviceFp8Op>& ops, bool unpack, void* stream, DeviceBatchResult* res) override;

 private:
  std::shared_ptr<BlackbirdClient> io_;
  bool reach_disk_;
  std::atomic<uint64_t> launches_{0};
  std::mutex done_mu_;
  uint64_t next_ticket_ = 1;
  std::map<uint64_t, DeviceBatchResult> done_;
};

}  // namespace bb::client
