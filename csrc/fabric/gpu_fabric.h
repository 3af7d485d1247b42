// GPU fabric: the GPU-native replacement of the reference's UcxEngine (SURVEY C11, §2.5).
//
//   reference (src/transport/ucx_engine.cpp)            here
//   ucp_mem_map + ucp_rkey_pack of a malloc'd pool  ->  cudaMalloc'd HBM slab + cudaIpcGetMemHandle
//   rkey hex advertised through etcd pool JSON      ->  IPC handle hex in the same JSON field
//   client ucp_ep_create + ucp_ep_rkey_unpack/call  ->  one-time cudaIpcOpenMemHandle per peer slab
//   ucp_put_nbx / ucp_get_nbx per shard + busy poll ->  one fused kernel launch per *batch* issuing
//                                                       TMA loads/stores on the peer-mapped pointers
//
// GpuSlabBackend is the RAM_GPU storage tier (`malloc` + "Does not work" in the reference,
// ram_backend.cpp:188, worker_service.cpp:196).  GpuFabric implements client::DeviceTransport.
#pragma once
#include <atomic>
#include <map>
#include <set>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "client/blackbird_client.h"
#include "fabric/nvls.h"
#include "fabric/xfer_engine.h"
#include "worker/storage_backend.h"

namespace bb::gpu {

class GpuSlabBackend : public worker::StorageBackend {
 public:
  GpuSlabBackend(uint64_t capacity, worker::BackendOptions opts);
  ~GpuSlabBackend() override;
  StorageClass get_storage_class() const override { return StorageClass::RAM_GPU; }
  uint64_t get_total_capacity() const override { return capacity_; }
  uint64_t get_base_address() const override { return reinterpret_cast<uint64_t>(base_); }
  uint64_t get_rkey() const override { return rkey_; }
  ErrorCode initialize() override;
  void shutdown() override;
  // Slow path (host tiers, TCP clients, tier demotion): staged cudaMemcpy.
  ErrorCode write(uint64_t offset, const void* data, uint64_t len) override;
  ErrorCode read(uint64_t offset, void* data, uint64_t len) override;
  void* direct_ptr(uint64_t offset) override { return base_ ? base_ + offset : nullptr; }
  bool cuda_accessible() const override { return base_ != nullptr; }
  // Tier move through the fused kernel (GPU slab <-> another slab or a pinned DRAM pool): one launch,
  // digest from the tensor-core hash / fused CRC.
  ErrorCode device_copy(worker::StorageBackend& peer, bool to_peer, uint64_t my_off, uint64_t peer_off, uint64_t len, ChecksumAlgo algo,
                        uint64_t* digest) override;
  ErrorCode pull_from_peer(const std::vector<uint8_t>& peer_key, uint64_t peer_off, uint64_t my_off, uint64_t len, ChecksumAlgo algo,
                           uint64_t* digest) override;
  int device() const { return opts_.gpu_device_id; }
  void* device_ptr() const { return base_; }
  // 64-byte cudaIpcMemHandle_t as 128 hex chars: the "rkey" peers open the slab with.
  std::string ipc_handle_hex() const { return handle_hex_; }
  std::string registration_key_hex() const override { return handle_hex_; }

 private:
  ErrorCode move_shard(const void* src, void* dst, uint64_t len, ChecksumAlgo algo, uint64_t* digest, std::atomic<uint64_t>& moved);
  uint8_t* base_ = nullptr;
  uint64_t rkey_ = 0;
  std::string handle_hex_;
  void* stream_ = nullptr;
  std::mutex move_mu_;
  std::unique_ptr<XferEngine> move_engine_;  // created on the first tier move
};

// Registers the GPU tier with worker::create_storage_backend (call once at start-up).
void install_gpu_backend_factory();

class GpuFabric : public client::DeviceTransport {
 public:
  // `device`: CUDA ordinal the client's kernels run on.
  static Result<std::shared_ptr<GpuFabric>> create(int device, std::shared_ptr<rpc::KeystoneApi> keystone);
  ~GpuFabric() override;

  bool can_reach(const ShardPlacement& s) const override;
  bool is_local(const ShardPlacement& s) const override;
  uint64_t launches() const override { return engine_->launches(); }
  Result<uint64_t> submit_put(const std::vector<client::DeviceShardOp>& ops, const std::vector<const void*>& dev_ptrs, ChecksumAlgo algo,
                              void* stream) override;
  // One engine batch per checksum algorithm in `ops` (normally exactly one).  A batch that mixes algorithms runs all
  // groups but the last to completion before returning, so it never holds more than one engine slot.
  Result<uint64_t> submit_get(const std::vector<client::DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, void* stream) override;
  ErrorCode wait(uint64_t ticket, client::DeviceBatchResult* res) override;
  size_t max_in_flight() const override { return 3; }
  bool fp8_eligible(uint64_t n_elems) const override { return XferEngine::fp8_eligible(n_elems); }
  ErrorCode run_fp8(const std::vector<client::DeviceFp8Op>& ops, bool unpack, void* stream, client::DeviceBatchResult* res) override;
  // One async copy per call (rows: the extent from the device, compacted on the host, or one 2-D copy of the whole rows
  // to it; pages: one per run of pages), then one synchronise.
  ErrorCode copy_from_device(void* host, const void* base, const DeviceLayout& layout, size_t n, void* stream) override;
  ErrorCode copy_to_device(void* base, const DeviceLayout& layout, const void* host, size_t n, void* stream) override;

  // Re-reads the pool registry from the keystone and maps any new GPU slab.
  ErrorCode refresh_pools();
  size_t mapped_pools() const;
  size_t mapped_host_pools() const;  // shared / pinned DRAM pools reachable by the fused kernels
  // NVLS replica arenas: pools named mc<g>@gpu<r> resolve through the arena; a put whose replica set is
  // exactly one multicast group (same offset everywhere) becomes ONE multimem.st stream.
  void set_arena(std::shared_ptr<NvlsArena> a) { arena_ = std::move(a); }
  uint64_t multicast_puts() const { return multicast_puts_.load(std::memory_order_relaxed); }
  uint64_t remaps() const { return remaps_; }
  // Payload bytes moved by the fused kernels, by direction and path: "hbm" (slab on this client's own GPU), "nvlink"
  // (peer slab over NVSwitch; multicast puts count one egress stream), "pcie" (pinned / shared DRAM pool).
  std::string metrics_text() const override;
  uint64_t path_bytes(bool put, int path) const { return bytes_[put ? 0 : 1][path].load(std::memory_order_relaxed); }  // mappings dropped because their pool was re-registered under a new key
  XferEngine& engine() { return *engine_; }
  float last_device_ms() const {
    std::lock_guard<std::mutex> lk(mu_);
    return last_ms_;
  }
  double total_device_ms() const {  // sum of kernel times of all finished batches
    std::lock_guard<std::mutex> lk(mu_);
    return total_ms_;
  }

 private:
  GpuFabric() = default;
  struct Mapping {
    uint8_t* base = nullptr;
    uint64_t size = 0;
    int device = -1;
    bool ipc_opened = false;
    bool host = false;           // pinned host memory (a worker's shared DRAM pool): reached over PCIe
    bool host_mapped = false;    // mapped + registered by this fabric (unmapped in the destructor)
    uint64_t remote_base = 0;    // host pools: the address MemoryLocation::remote_addr is relative to
    std::vector<uint8_t> key;    // registration key the mapping was made from (IPC handle / "file:<path>")
  };
  // A placement carries its pool's current registration key (TransportEndpoint::worker_key): a mapping made from a
  // different key belongs to a previous incarnation of the pool (worker restarted with the same pool id) and is dropped.
  void drop_if_stale(const ShardPlacement& s);
  struct HostCandidate {         // DRAM pool seen in the registry; mapped lazily on first use
    uint64_t size = 0;
    uint64_t remote_base = 0;
    std::string key_hex;
  };
  bool ensure_host_pool(const std::string& pool_id);
  Result<void*> resolve(const ShardPlacement& s);
  ErrorCode build_put_items(const std::vector<client::DeviceShardOp>& ops, const std::vector<const void*>& dev_ptrs,
                            std::vector<XferItem>* items, std::vector<size_t>* op_of_item);
  ErrorCode build_get_items(const std::vector<client::DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, ChecksumAlgo algo,
                            std::vector<XferItem>* items, std::vector<size_t>* op_of_item);
  struct InFlight {
    size_t nops = 0;
    std::vector<size_t> op_of_item;  // item -> op
    client::DeviceBatchResult done;  // get: per op, from the groups of a mixed batch that finished in submit_get
  };
  ErrorCode finish(uint64_t ticket, InFlight* fl, XferResult* res);
  void note_device_ms(float ms) {
    std::lock_guard<std::mutex> lk(mu_);
    last_ms_ = ms;
    total_ms_ += ms;
  }
  std::map<uint64_t, InFlight> inflight_;  // engine ticket -> bookkeeping
  int device_ = 0;
  std::shared_ptr<rpc::KeystoneApi> keystone_;
  std::unique_ptr<XferEngine> engine_;
  mutable std::mutex mu_;
  std::map<std::string, Mapping> pools_;
  std::map<std::string, HostCandidate> host_candidates_;
  std::set<std::string> host_unreachable_;
  std::shared_ptr<NvlsArena> arena_;
  std::atomic<uint64_t> multicast_puts_{0};
  std::atomic<uint64_t> remaps_{0};
  enum Path : int { PATH_HBM = 0, PATH_NVLINK = 1, PATH_PCIE = 2, PATH_MULTICAST = 3, kNumPaths = 4 };
  Path classify(const ShardPlacement& s) const;
  void count(bool put, Path p, uint64_t bytes) { bytes_[put ? 0 : 1][p].fetch_add(bytes, std::memory_order_relaxed); }
  std::atomic<uint64_t> bytes_[2][kNumPaths] = {};
  float last_ms_ = 0.f;    // guarded by mu_
  double total_ms_ = 0.0;  // guarded by mu_
};

// Process-local slab registry (in-process workers + clients share pointers directly; CUDA IPC
// cannot open a handle inside the process that exported it).
void register_local_slab(const std::string& pool_id, int device, void* base, uint64_t size);
void unregister_local_slab(const std::string& pool_id);

}  // namespace bb::gpu
