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
#include <string>
#include <vector>

#include "common/metrics.h"
#include "common/mxfp8.h"
#include "common/store_window.h"
#include "net/tcp.h"
#include "rpc/rpc_service.h"

namespace bb::client {

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
  uint64_t obj_offset = 0;    // byte offset of this shard inside the object
  // Get: the shard bytes that are stored (common/store_window.h); the whole shard is still read and verified.  An op whose
  // window covers the shard, the default included, is a whole-shard op.
  StoreWindow win;
  // The base `win` goes with, given the object's: dev_ptrs[item] is where object byte 0 lands, or for a strided get where
  // the result's row 0 lands.
  void* dst(void* obj_base) const { return static_cast<uint8_t*>(obj_base) + win.base_shift(obj_offset); }
  // Where the shard's bytes sit in the caller's strided memory (common/store_window.h): a put's source rows, or a get's
  // destination rows (a get into a sliced tensor), the object's rows rebased to obj_offset; rows_at is where the shard's
  // pattern row 0 starts relative to dev_ptrs[item].  The default is contiguous memory.  A get op never has both a
  // pattern and a window.
  SourceRows rows;
  uint64_t rows_at = 0;
  // A put's source pages or a get's destination pages (common/store_window.h), the object's table rebased to obj_offset;
  // dev_ptrs[item] is not used then.  Never together with rows or a window.
  SourcePages pages;
  const void* src(const void* obj_base) const {
    return static_cast<const uint8_t*>(obj_base) + (rows.strided() ? rows_at : obj_offset);
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
  // The wide side's rows in elements (common/store_window.h), `wide` being where the pattern's row 0 starts: a put's source
  // rows, or a get's destination rows (never together with a window).  The packed object is one shard, so the pattern is
  // the object's own.  The default is contiguous memory.
  SourceRows rows;
  // The element type of `wide`: bf16, fp16 or fp32 (common/mxfp8.h).  Ops of one call share its size (2 or 4 bytes).
  mxfp8::Wide wide_type = mxfp8::Wide::BF16;
};

// Implemented by the GPU fabric: moves shards between client device buffers and worker slabs
// with the fused kernels.  Returns per-op digests (put) or verifies them (get).
class DeviceTransport {
 public:
  virtual ~DeviceTransport() = default;
  virtual bool can_reach(const ShardPlacement& s) const = 0;
  virtual uint64_t launches() const = 0;
  // submit_* enqueues a batch and returns a ticket, so the caller can overlap control-plane round trips of the next chunk
  // with this one's transfer; wait_* blocks until it is done.  dev_ptrs[item] is the device buffer of object `item`.  A
  // put returns one digest per op; a get verifies each shard with its placement's algorithm (status per op, 0 = ok).
  virtual Result<uint64_t> submit_put(const std::vector<DeviceShardOp>& ops, const std::vector<const void*>& dev_ptrs, ChecksumAlgo algo,
                                      void* stream) = 0;
  virtual ErrorCode wait_put(uint64_t ticket, std::vector<uint64_t>* digests) = 0;
  virtual Result<uint64_t> submit_get(const std::vector<DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, void* stream) = 0;
  virtual ErrorCode wait_get(uint64_t ticket, std::vector<uint32_t>* status) = 0;
  // True when the shard lives in this client's own device memory (a get from it never leaves the GPU).
  virtual bool is_local(const ShardPlacement& s) const { return false; }
  virtual size_t max_in_flight() const { return 1; }
  // Prometheus lines of the transport's own counters (bytes per path, launches, ...); appended to the client's metrics.
  virtual std::string metrics_text() const { return {}; }
  virtual bool fp8_eligible(uint64_t n_elems) const { return false; }
  // Fused MXFP8 put / get (pack / unpack inside the transfer kernel).  digests[i] = BBH64 of the stored packed
  // object; status[i] != 0 = digest mismatch on get.  Objects must satisfy fp8_eligible().
  virtual ErrorCode put_fp8(const std::vector<DeviceFp8Op>& ops, void* stream, std::vector<uint64_t>* digests) { return ErrorCode::NOT_IMPLEMENTED; }
  virtual ErrorCode get_fp8(const std::vector<DeviceFp8Op>& ops, void* stream, std::vector<uint32_t>* status) { return ErrorCode::NOT_IMPLEMENTED; }
  // Staging copies for objects (or shards) that live on host tiers: device <-> host buffer, synchronous.
  virtual ErrorCode copy_h2d(void* dev, const void* host, size_t n, void* stream) { return ErrorCode::NOT_IMPLEMENTED; }
  // `rows` rows of `width` bytes, packed back to back at `host`, into row r = dev + r * pitch: one copy however many rows.
  virtual ErrorCode copy_h2d_rows(void* dev, size_t pitch, const void* host, size_t width, size_t rows, void* stream) {
    return ErrorCode::NOT_IMPLEMENTED;
  }
  virtual ErrorCode copy_d2h(void* host, const void* dev, size_t n, void* stream) { return ErrorCode::NOT_IMPLEMENTED; }
  // Object bytes [0, n) of `pages` (common/store_window.h) from / to n bytes packed back to back at `host`: one copy per
  // run of pages (SourcePages::for_each_run), synchronous.
  virtual ErrorCode copy_d2h_pages(void* host, const SourcePages& pages, size_t n, void* stream) { return ErrorCode::NOT_IMPLEMENTED; }
  virtual ErrorCode copy_h2d_pages(const SourcePages& pages, const void* host, size_t n, void* stream) { return ErrorCode::NOT_IMPLEMENTED; }
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
  // Per object, before anything is allocated: INVALID_ARGUMENT for elem_widths[i] > elem_pitches[i] with rows[i] > 1;
  // VALUE_OUT_OF_RANGE when the element count or the source extent overflows; NOT_IMPLEMENTED unless bf16_ptrs[i] is
  // 16-byte aligned and, for rows[i] > 1, (elem_pitches[i] - elem_widths[i]) % 8 == 0 -- there is no host-staged path;
  // the rest of the batch keeps its single launch.  rows[i] == 1 or elem_widths[i] == elem_pitches[i] is exactly
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
  // and the placement refresh are batch_get_device_fp8's.  Per object: INVALID_ARGUMENT unless rows[i] * elem_widths[i] ==
  // n_elems[i], or for elem_widths[i] > elem_pitches[i] with rows[i] > 1; VALUE_OUT_OF_RANGE when a product overflows;
  // NOT_IMPLEMENTED when the object is not fusable (as batch_get_device_fp8), or unless bf16_ptrs[i] is 16-byte aligned
  // and, for rows[i] > 1, (elem_pitches[i] - elem_widths[i]) % 8 == 0 -- there is no host-staged path; the rest of the
  // batch keeps the fused launch.  rows[i] == 1 or elem_widths[i] == elem_pitches[i] is batch_get_device_fp8.
  std::vector<ErrorCode> batch_get_device_fp8_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                      const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_widths,
                                                      const std::vector<uint64_t>& elem_pitches, const std::vector<uint64_t>& rows,
                                                      void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
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
  // while the rest of the batch keeps the fused launch.  Per object, before anything is allocated: INVALID_ARGUMENT for
  // widths[i] > pitches[i] with rows[i] > 1; VALUE_OUT_OF_RANGE when the size or the extent overflows.  rows[i] == 1 or
  // widths[i] == pitches[i] is exactly batch_put_device of one contiguous block, rows[i] == 0 or widths[i] == 0 that of a
  // zero-byte object.
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
  // batch keeps the fused launch.  Per object, before anything is read: INVALID_ARGUMENT for widths[i] > pitches[i] with
  // rows[i] > 1; VALUE_OUT_OF_RANGE when the size or the extent overflows.  rows[i] == 1 or widths[i] == pitches[i] is
  // exactly batch_get_device with capacity rows[i] * widths[i].
  std::vector<ErrorCode> batch_get_device_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                  const std::vector<uint64_t>& widths, const std::vector<uint64_t>& pitches,
                                                  const std::vector<uint64_t>& rows, void* stream, std::vector<size_t>* out_sizes);
  // Paged puts (the blocks of a paged KV cache, one object for a whole request): object i is the concatenation of the
  // pages[i].size() pages of page_bytes[i] bytes at the device addresses pages[i], in list order (SourcePages in
  // common/store_window.h); one object, one metadata record.  A page may repeat.  The stored object and its digests are
  // those of batch_put_device of the concatenation, so every get reads it.  The fused path reads each page in place in
  // the put kernel; it needs every shard of every copy co-aligned (SourcePages::coaligned: 16-byte aligned pages and shard starts and, for
  // several pages, page_bytes[i] % 16 == 0).  Any other item, and every placement the fabric cannot reach, is staged
  // through the host (one D2H copy per run of pages) while the rest of the batch keeps the fused launch.  Per object,
  // before anything is allocated: INVALID_ARGUMENT for page_bytes[i] == 0 with pages; VALUE_OUT_OF_RANGE when the size
  // overflows.  No pages is a zero-byte object.
  std::vector<ErrorCode> batch_put_device_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                const std::vector<uint64_t>& page_bytes, const WorkerConfig& cfg, void* stream);
  // Paged gets, the mirror: object i lands in the pages pages[i] of page_bytes[i] bytes, object byte x in page
  // x / page_bytes[i] at offset x % page_bytes[i].  The capacity is pages[i].size() * page_bytes[i]: a larger object is
  // BUFFER_OVERFLOW, a shorter one fills its bytes in page order; out_sizes[i] receives the size.  Only the object's bytes
  // are written.  Pages of one get must not overlap (not checked).  Every shard is read whole and verified, with the
  // fail-over and placement refresh of batch_get_device.  The fused path scatters the pages in the get kernel; it needs
  // SourcePages::fused_get_aligned for every shard of every copy.  Any other item, and every placement the fabric cannot
  // reach, is staged through the host (one H2D copy per run of pages).  Per object: INVALID_ARGUMENT for
  // page_bytes[i] == 0 with pages; VALUE_OUT_OF_RANGE when the capacity overflows.
  std::vector<ErrorCode> batch_get_device_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                const std::vector<uint64_t>& page_bytes, void* stream, std::vector<size_t>* out_sizes);

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
  // batch_get_device, batch_get_device_range, batch_get_device_strided and batch_get_device_scatter: `ranges` null = whole
  // objects into buffers of `capacity`, else object i's rows into dev_ptrs[i] (capacity[i] = rows * length, for the chunk
  // plan).  A range is the single row `rows == 1`.  `rows` (whole objects only) null = contiguous buffers, else object i
  // lands in (*rows)[i], row 0 at dev_ptrs[i].
  struct ByteRange {
    uint64_t offset = 0, length = 0;
    uint64_t pitch = 0, rows = 1;  // row r = bytes [offset + r * pitch, + length)
  };
  // batch_put_device, batch_put_device_strided and batch_put_device_paged: `rows` null = contiguous sources, else object i
  // is read by (*rows)[i]; `pages` non-null = object i is read from the pages (*pages)[i] wherever they are paged (dev_ptrs
  // are then not read).
  std::vector<ErrorCode> put_device(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs, const std::vector<size_t>& sizes,
                                    const std::vector<SourceRows>* rows, const WorkerConfig& cfg, void* stream,
                                    const std::vector<SourcePages>* pages = nullptr);
  // `pages` (whole objects only, never with `rows`) non-null = object i lands in the pages (*pages)[i] wherever they are
  // paged.
  std::vector<ErrorCode> get_device(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs, const std::vector<size_t>& capacity,
                                    const std::vector<ByteRange>* ranges, const std::vector<SourceRows>* rows, void* stream,
                                    std::vector<size_t>* out_sizes, const std::vector<SourcePages>* pages = nullptr);
  // batch_put_device_fp8 and batch_put_device_fp8_strided: `rows` null = contiguous tensors, else object i is read by
  // (*rows)[i], in elements.
  std::vector<ErrorCode> put_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                        const std::vector<uint64_t>& n_elems, const std::vector<SourceRows>* rows, const WorkerConfig& cfg,
                                        void* stream, mxfp8::Wide wide);
  // batch_get_device_fp8, batch_get_device_fp8_range, batch_get_device_fp8_strided and batch_get_device_fp8_scatter:
  // `ranges` null = whole tensors, else object i's rows (offset, length and pitch in elements) into bf16_ptrs[i]; `rows`
  // (whole tensors only) null = contiguous destinations, else object i lands in (*rows)[i], in elements.
  std::vector<ErrorCode> get_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                        const std::vector<uint64_t>& n_elems, const std::vector<ByteRange>* ranges,
                                        const std::vector<SourceRows>* rows, void* stream, mxfp8::Wide wide);
  // The eight shaped batch_*_device_* calls over the four above, and the placement refresh of get_device and get_device_fp8.
  template <class Shape, class Run>
  std::vector<ErrorCode> shaped_batch(std::string_view name, bool admit, size_t n, bool arity_ok, Shape&& shape, Run&& run);
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
  ErrorCode wait_put(uint64_t ticket, std::vector<uint64_t>* digests) override;
  Result<uint64_t> submit_get(const std::vector<DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, void* stream) override;
  ErrorCode wait_get(uint64_t ticket, std::vector<uint32_t>* status) override;
  bool can_reach(const ShardPlacement& s) const override;
  uint64_t launches() const override { return launches_; }
  ErrorCode copy_h2d(void* dev, const void* host, size_t n, void*) override {
    std::memcpy(dev, host, n);
    return ErrorCode::OK;
  }
  ErrorCode copy_h2d_rows(void* dev, size_t pitch, const void* host, size_t width, size_t rows, void*) override {
    for (size_t r = 0; r < rows; ++r) std::memcpy(static_cast<uint8_t*>(dev) + r * pitch, static_cast<const uint8_t*>(host) + r * width, width);
    return ErrorCode::OK;
  }
  ErrorCode copy_d2h(void* host, const void* dev, size_t n, void*) override {
    std::memcpy(host, dev, n);
    return ErrorCode::OK;
  }
  ErrorCode copy_d2h_pages(void* host, const SourcePages& pages, size_t n, void*) override {
    pages.for_each_run(n, [&](uint64_t x, uint64_t at, uint64_t len) {
      std::memcpy(static_cast<uint8_t*>(host) + x, reinterpret_cast<const void*>(at), len);
    });
    return ErrorCode::OK;
  }
  ErrorCode copy_h2d_pages(const SourcePages& pages, const void* host, size_t n, void*) override {
    pages.for_each_run(n, [&](uint64_t x, uint64_t at, uint64_t len) {
      std::memcpy(reinterpret_cast<void*>(at), static_cast<const uint8_t*>(host) + x, len);
    });
    return ErrorCode::OK;
  }
  size_t max_in_flight() const override { return 2; }
  // MXFP8 through the CPU reference codec (common/mxfp8.h): the stored object and its digest are the ones the fused
  // kernels produce, so the fp8 client logic (replica fan-out, fail-over between replicas) is testable on CPU too.
  bool fp8_eligible(uint64_t n_elems) const override { return n_elems != 0 && n_elems % 32 == 0; }
  ErrorCode put_fp8(const std::vector<DeviceFp8Op>& ops, void* stream, std::vector<uint64_t>* digests) override;
  ErrorCode get_fp8(const std::vector<DeviceFp8Op>& ops, void* stream, std::vector<uint32_t>* status) override;

 private:
  std::shared_ptr<BlackbirdClient> io_;
  bool reach_disk_;
  std::atomic<uint64_t> launches_{0};
  std::mutex done_mu_;
  uint64_t next_ticket_ = 1;
  std::map<uint64_t, std::pair<std::vector<uint64_t>, std::vector<uint32_t>>> done_;  // ticket -> (put digests, get status)
};

}  // namespace bb::client
