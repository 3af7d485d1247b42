#include "common/trace.h"
#include "client/blackbird_client.h"

#include "common/tenant.h"
#include "common/mxfp8.h"
#include "common/tchash_def.h"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <future>
#include <map>
#include <thread>

#include "common/log.h"
#include "rpc/wire.h"
#include "worker/worker_service.h"

namespace bb::client {

using keystone::PutStartItem;
using keystone::ShardChecksums;

namespace {
double us_since(TimePoint t0) { return std::chrono::duration<double, std::micro>(Clock::now() - t0).count(); }

// Runs fn(i) for i in [0, n) on up to `par` threads; returns the first error.
template <typename F>
ErrorCode parallel_for(size_t n, size_t par, F&& fn) {
  if (n == 0) return ErrorCode::OK;
  par = std::max<size_t>(1, std::min(par, n));
  if (par == 1) {
    for (size_t i = 0; i < n; ++i) {
      ErrorCode ec = fn(i);
      if (ec != ErrorCode::OK) return ec;
    }
    return ErrorCode::OK;
  }
  std::atomic<size_t> next{0};
  std::atomic<uint32_t> first_err{0};
  std::vector<std::thread> th;
  for (size_t t = 0; t < par; ++t)
    th.emplace_back([&] {
      while (first_err.load() == 0) {
        const size_t i = next.fetch_add(1);
        if (i >= n) break;
        ErrorCode ec = fn(i);
        if (ec != ErrorCode::OK) {
          uint32_t z = 0;
          first_err.compare_exchange_strong(z, static_cast<uint32_t>(ec));
        }
      }
    });
  for (auto& t : th) t.join();
  return static_cast<ErrorCode>(first_err.load());
}
}  // namespace

BlackbirdClient::BlackbirdClient(BlackbirdClientOptions opts) : opts_(std::move(opts)) {}
BlackbirdClient::BlackbirdClient(std::shared_ptr<rpc::KeystoneApi> keystone, BlackbirdClientOptions opts)
    : opts_(std::move(opts)), keystone_(std::move(keystone)) {
  if (keystone_) keystone_->set_identity(session_id_, opts_.node_id);
}
BlackbirdClient::~BlackbirdClient() {
  std::lock_guard<std::mutex> lk(shm_mu_);
  for (auto& [id, p] : shm_pools_) worker::unmap_shared_pool(p.base, p.size);
  shm_pools_.clear();
}

ErrorCode BlackbirdClient::connect() {
  if (!opts_.auth_token.empty()) net::set_cluster_token(opts_.auth_token);
  if (opts_.encrypt_transport) net::set_transport_encryption(true);
  if (!opts_.auth_token_ro.empty()) net::set_cluster_token_ro(opts_.auth_token_ro);
  if (!opts_.tenant.empty()) set_client_tenant(opts_.tenant, opts_.tenant_secret);
  if (!keystone_) {
    auto c = std::make_shared<rpc::KeystoneRpcClient>();
    c->set_timeout_ms(opts_.rpc_timeout_ms);
    const int connect_ms = std::min(opts_.rpc_timeout_ms, 5000);
    ErrorCode ec = opts_.keystone_endpoints.empty() ? c->connect(opts_.keystone_host, opts_.keystone_port, connect_ms)
                                                    : c->connect_any(opts_.keystone_endpoints, connect_ms);
    if (ec != ErrorCode::OK) return ec;
    keystone_ = c;
  }
  if (opts_.register_session) {
    auto s = keystone_->client_register(opts_.node_id);
    if (!s.ok()) return s.error();
    session_id_ = s.value();
  }
  keystone_->set_identity(session_id_, opts_.node_id);
  return ErrorCode::OK;
}

// ================================================================ worker connections
std::shared_ptr<net::RpcClient> BlackbirdClient::acquire(const std::string& endpoint) {
  {
    std::lock_guard<std::mutex> lk(conn_mu_);
    auto& v = idle_conns_[endpoint];
    if (!v.empty()) {
      auto c = v.back();
      v.pop_back();
      return c;
    }
  }
  auto hp = split_host_port(endpoint);
  if (!hp) return nullptr;
  auto c = std::make_shared<net::RpcClient>();
  if (c->connect(hp->first, static_cast<uint16_t>(hp->second), std::min(opts_.rpc_timeout_ms, 5000)) != ErrorCode::OK) return nullptr;
  c->set_bulk_buffers();
  return c;
}

void BlackbirdClient::release(const std::string& endpoint, std::shared_ptr<net::RpcClient> c) {
  if (!c || !c->connected()) return;
  std::lock_guard<std::mutex> lk(conn_mu_);
  auto& v = idle_conns_[endpoint];
  if (v.size() < 16) v.push_back(std::move(c));
}

uint64_t BlackbirdClient::shard_offset(const ShardPlacement& s) {
  if (auto* g = std::get_if<GpuSlabLocation>(&s.location)) return g->offset;
  if (auto* f = std::get_if<FileLocation>(&s.location)) return f->file_offset;
  if (auto* c = std::get_if<CxlMemoryLocation>(&s.location)) return c->offset;
  return 0;
}

namespace {
constexpr uint64_t kDataChunk = 8ull << 20;     // one D_WRITE / D_READ request
constexpr uint64_t kStreamMin = 4ull << 20;     // a shard is split over several connections from 2x this size

// Splits [0, len) into up to `par` ranges whose boundaries are multiples of the BBH64 tile (so per-range digests
// combine) and runs fn(range_begin, range_len, range_index) on one thread each.
template <typename F>
ErrorCode for_each_stream(uint64_t len, size_t par, F&& fn) {
  size_t n = static_cast<size_t>(std::min<uint64_t>(std::max<size_t>(par, 1), len / kStreamMin));
  if (n <= 1) return fn(0, len, 0);
  const uint64_t tiles = (len + tchash::kTileBytes - 1) / tchash::kTileBytes;
  const uint64_t per = (tiles + n - 1) / n * tchash::kTileBytes;
  n = static_cast<size_t>((len + per - 1) / per);
  std::vector<ErrorCode> ecs(n, ErrorCode::OK);
  std::vector<std::thread> th;
  for (size_t i = 1; i < n; ++i)
    th.emplace_back([&, i] { ecs[i] = fn(i * per, std::min<uint64_t>(per, len - i * per), i); });
  ecs[0] = fn(0, std::min<uint64_t>(per, len), 0);
  for (auto& t : th) t.join();
  for (ErrorCode ec : ecs)
    if (ec != ErrorCode::OK) return ec;
  return ErrorCode::OK;
}
// Hashes a byte range on its own thread while the transfer loop moves it: the loop publishes how far the bytes are
// valid (a put has them all from the start, a get as the chunks arrive) and collects the range digest at the end.
class RangeHasher {
 public:
  RangeHasher(ChecksumAlgo algo, const uint8_t* base, uint64_t shard_len, uint64_t begin, uint64_t len, bool all_valid)
      : algo_(algo), base_(base), shard_len_(shard_len), begin_(begin), len_(len), valid_(all_valid ? len : 0) {
    if (algo_ != ChecksumAlgo::NONE && len_ >= (1u << 20)) th_ = std::thread([this] { run(); });
    else inline_ = true;
  }
  ~RangeHasher() {
    abort_.store(true);
    if (th_.joinable()) th_.join();
  }
  void advance(uint64_t valid_len) { valid_.store(valid_len, std::memory_order_release); }
  // crc: CRC32C of the range (standard init / final xor, combinable with crc32c_combine); bbh: unfinalised tile sum
  void finish(uint32_t* crc, uint64_t* bbh) {
    valid_.store(len_, std::memory_order_release);
    if (inline_) run();
    else if (th_.joinable()) th_.join();
    *crc = crc_;
    *bbh = bbh_;
  }

 private:
  void run() {
    constexpr uint64_t kStep = 1ull << 20;  // multiple of the BBH64 tile
    uint64_t done = 0;
    while (done < len_) {
      uint64_t v = valid_.load(std::memory_order_acquire);
      if (v <= done) {
        if (abort_.load()) return;
        std::this_thread::yield();
        continue;
      }
      v = v == len_ ? len_ : v / kStep * kStep;  // whole steps (tile aligned) until the tail
      if (v <= done) {
        if (abort_.load()) return;
        std::this_thread::yield();
        continue;
      }
      const uint64_t n = std::min(kStep, v - done);
      if (algo_ == ChecksumAlgo::CRC32C) crc_ = crc32c(base_ + begin_ + done, n, crc_);
      else if (is_tile_sum(algo_))
        bbh_ += tile_sum_partial(algo_, base_, shard_len_, (begin_ + done) / tchash::kTileBytes, (n + tchash::kTileBytes - 1) / tchash::kTileBytes);
      done += n;
    }
  }
  ChecksumAlgo algo_;
  const uint8_t* base_;
  uint64_t shard_len_, begin_, len_;
  std::atomic<uint64_t> valid_;
  std::atomic<bool> abort_{false};
  bool inline_ = false;
  uint32_t crc_ = 0;
  uint64_t bbh_ = 0;
  std::thread th_;
};
}  // namespace

uint8_t* BlackbirdClient::shm_resolve(const ShardPlacement& s) {
  static const bool env_off = [] { const char* e = std::getenv("BB_DISABLE_SHM"); return e && *e && *e != '0'; }();
  if (!opts_.enable_shm || env_off || s.storage_class != StorageClass::RAM_CPU) return nullptr;
  const auto* loc = std::get_if<MemoryLocation>(&s.location);
  const auto& key = s.endpoint.worker_key;
  if (!loc || key.size() <= 5 || std::memcmp(key.data(), "file:", 5) != 0) return nullptr;
  {
    std::lock_guard<std::mutex> lk(shm_mu_);
    auto it = shm_pools_.find(s.pool_id);
    if (it != shm_pools_.end()) {
      if (it->second.key == key) {
        const ShmPool& p = it->second;
        if (loc->remote_addr < p.remote_base || loc->remote_addr - p.remote_base + s.length > p.size) return nullptr;
        return p.base + (loc->remote_addr - p.remote_base);
      }
      worker::unmap_shared_pool(it->second.base, it->second.size);  // the worker restarted: new memfd, new key
      shm_pools_.erase(it);
    }
    auto un = shm_unreachable_.find(s.pool_id);
    if (un != shm_unreachable_.end() && un->second == key) return nullptr;
  }
  // first shard in this pool: learn its geometry from the registry, then map it
  ShmPool p;
  auto pools = keystone_->get_memory_pools();
  if (pools.ok())
    for (const auto& mp : pools.value())
      if (mp.id == s.pool_id) {
        p.size = mp.size;
        p.remote_base = mp.ucx_remote_addr ? mp.ucx_remote_addr : mp.base_addr;
      }
  if (p.size) p.base = static_cast<uint8_t*>(worker::map_shared_pool(key, p.size));
  std::lock_guard<std::mutex> lk(shm_mu_);
  if (!p.base) {  // other host / pid namespace / user: stay on the data server
    shm_unreachable_[s.pool_id] = key;
    return nullptr;
  }
  p.key = key;
  auto [it, fresh] = shm_pools_.emplace(s.pool_id, p);
  if (!fresh) worker::unmap_shared_pool(p.base, p.size);  // another thread mapped it first
  else metrics_.inc("shm_pools_mapped_total");
  const ShmPool& q = it->second;
  if (loc->remote_addr < q.remote_base || loc->remote_addr - q.remote_base + s.length > q.size) return nullptr;
  return q.base + (loc->remote_addr - q.remote_base);
}

namespace {
// memcpy of a shard as up to `par` tile-aligned ranges on their own threads, each hashed while it is hot in cache.
struct ShmPart {
  uint32_t crc = 0;
  uint64_t len = 0;
  uint64_t bbh = 0;
};
uint64_t shm_copy(uint8_t* dst, const uint8_t* src, const uint8_t* hash_base, uint64_t len, size_t par, ChecksumAlgo algo) {
  if (algo == ChecksumAlgo::NONE) par = 1;  // a bare memcpy already runs at memory speed; threads only help the hashing
  std::vector<ShmPart> parts(std::max<size_t>(1, par));
  for_each_stream(len, par, [&](uint64_t begin, uint64_t n, size_t idx) -> ErrorCode {
    ShmPart& part = parts[idx];
    part.len = n;
    constexpr uint64_t kStep = 1ull << 20;  // copy + hash in cache-sized steps (multiple of the BBH64 tile)
    for (uint64_t o = begin; o < begin + n; o += kStep) {
      const uint64_t m = std::min(kStep, begin + n - o);
      std::memcpy(dst + o, src + o, m);
      if (algo == ChecksumAlgo::CRC32C) part.crc = crc32c(hash_base + o, m, part.crc);
      else if (is_tile_sum(algo))
        part.bbh += tile_sum_partial(algo, hash_base, len, o / tchash::kTileBytes, (m + tchash::kTileBytes - 1) / tchash::kTileBytes);
    }
    return ErrorCode::OK;
  });
  if (algo == ChecksumAlgo::CRC32C) {
    uint32_t crc = 0;
    bool first = true;
    for (const ShmPart& p : parts) {
      if (p.len == 0 && !first) continue;
      crc = first ? p.crc : crc32c_combine(crc, p.crc, p.len);
      first = false;
    }
    return crc;
  }
  if (is_tile_sum(algo)) {
    uint64_t sum = 0;
    for (const ShmPart& p : parts) sum += p.bbh;
    return tile_sum_finalize(sum, len);
  }
  return 0;
}
}  // namespace

ErrorCode BlackbirdClient::write_shard(const ShardPlacement& s, const uint8_t* src, uint64_t* digest, ChecksumAlgo algo) {
  if (uint8_t* mapped = shm_resolve(s)) {  // same host: one-sided write into the worker's pool
    const uint64_t d = shm_copy(mapped, src, src, s.length, opts_.io_parallelism, algo);
    if (digest) *digest = d;
    metrics_.inc("shm_put_shards_total");
    metrics_.inc("shm_put_bytes_total", s.length);
    return ErrorCode::OK;
  }
  const std::string ep = s.endpoint.ip + ":" + std::to_string(s.endpoint.port);
  uint64_t base_off = shard_offset(s);
  bool absolute = false;
  if (auto* m = std::get_if<MemoryLocation>(&s.location)) {
    base_off = m->remote_addr;  // absolute address; the worker subtracts its base
    absolute = true;
  }
  // Large shards go out as several streams (one connection + one thread each); every stream sends its range in
  // kDataChunk requests with a gathered write (header + bytes straight from the caller's buffer) and hashes it while the
  // worker stores the previous chunk.  Per-stream digests combine: CRC32C by shift algebra, BBH64 by addition.
  struct Part {
    uint32_t crc = 0;
    uint64_t len = 0;
    uint64_t bbh = 0;
  };
  std::vector<Part> parts(std::max<size_t>(1, opts_.io_parallelism));
  ErrorCode ec = for_each_stream(s.length, opts_.io_parallelism, [&](uint64_t begin, uint64_t len, size_t idx) -> ErrorCode {
    auto conn = acquire(ep);
    if (!conn) return ErrorCode::CONNECTION_FAILED;
    Part& part = parts[idx];
    part.len = len;
    RangeHasher hasher(algo, src, s.length, begin, len, /*all_valid=*/true);
    for (uint64_t pos = begin; pos < begin + len || (s.length == 0 && pos == 0); pos += kDataChunk) {
      const uint32_t n = static_cast<uint32_t>(std::min<uint64_t>(kDataChunk, begin + len - pos));
      wire::Writer w;
      w.str(s.pool_id);
      w.u64((base_off + pos) | (absolute ? (1ull << 63) : 0));
      w.u32(n);
      auto r = conn->call_gather(worker::D_WRITE, w.data(), src + pos, n, opts_.rpc_timeout_ms);
      if (!r.ok()) return ErrorCode::TRANSFER_FAILED;
      wire::Reader rd(r.value());
      const ErrorCode wec = rd.ec();
      if (wec != ErrorCode::OK) {
        release(ep, conn);
        return wec;
      }
      if (s.length == 0) break;
    }
    hasher.finish(&part.crc, &part.bbh);
    release(ep, conn);
    return ErrorCode::OK;
  });
  if (ec != ErrorCode::OK) return ec;
  if (digest) {
    if (algo == ChecksumAlgo::CRC32C) {
      uint32_t crc = 0;
      bool first = true;
      for (const Part& p : parts) {
        if (p.len == 0 && !first) continue;
        crc = first ? p.crc : crc32c_combine(crc, p.crc, p.len);
        first = false;
      }
      *digest = crc;
    } else if (is_tile_sum(algo)) {
      uint64_t sum = 0;
      for (const Part& p : parts) sum += p.bbh;
      *digest = tile_sum_finalize(sum, s.length);
    } else {
      *digest = 0;
    }
  }
  return ErrorCode::OK;
}

ErrorCode BlackbirdClient::read_shard(const ShardPlacement& s, uint8_t* dst, ChecksumAlgo algo) {
  if (const uint8_t* mapped = shm_resolve(s)) {  // same host: one-sided read out of the worker's pool
    const bool check = algo != ChecksumAlgo::NONE && s.checksum_algo == algo;
    const uint64_t got = shm_copy(dst, mapped, dst, s.length, opts_.io_parallelism, check ? algo : ChecksumAlgo::NONE);
    metrics_.inc("shm_get_shards_total");
    metrics_.inc("shm_get_bytes_total", s.length);
    if (check && got != s.checksum) {
      metrics_.inc("checksum_mismatch_total");
      return ErrorCode::CHECKSUM_MISMATCH;
    }
    return ErrorCode::OK;
  }
  const std::string ep = s.endpoint.ip + ":" + std::to_string(s.endpoint.port);
  uint64_t base_off = shard_offset(s);
  bool absolute = false;
  if (auto* m = std::get_if<MemoryLocation>(&s.location)) {
    base_off = m->remote_addr;
    absolute = true;
  }
  const bool verify = algo != ChecksumAlgo::NONE && s.checksum_algo == algo;
  struct Part {
    uint32_t crc = 0;
    uint64_t len = 0;
    uint64_t bbh = 0;
  };
  std::vector<Part> parts(std::max<size_t>(1, opts_.io_parallelism));
  // Same streams as write_shard; the response payload is received straight into the caller's buffer.
  ErrorCode ec = for_each_stream(s.length, opts_.io_parallelism, [&](uint64_t begin, uint64_t len, size_t idx) -> ErrorCode {
    auto conn = acquire(ep);
    if (!conn) return ErrorCode::CONNECTION_FAILED;
    Part& part = parts[idx];
    part.len = len;
    RangeHasher hasher(verify ? algo : ChecksumAlgo::NONE, dst, s.length, begin, len, /*all_valid=*/false);
    for (uint64_t pos = begin; pos < begin + len; pos += kDataChunk) {
      const uint32_t n = static_cast<uint32_t>(std::min<uint64_t>(kDataChunk, begin + len - pos));
      wire::Writer w;
      w.str(s.pool_id);
      w.u64((base_off + pos) | (absolute ? (1ull << 63) : 0));
      w.u32(n);
      size_t got = 0;
      auto r = conn->call_scatter(worker::D_READ, w.data(), 4, dst + pos, n, &got, opts_.rpc_timeout_ms);
      if (!r.ok()) return ErrorCode::TRANSFER_FAILED;
      if (r.value().size() < 4) return ErrorCode::TRANSFER_FAILED;
      uint32_t e;
      std::memcpy(&e, r.value().data(), 4);
      if (e != 0) {
        release(ep, conn);
        return static_cast<ErrorCode>(e);
      }
      if (got != n) return ErrorCode::TRANSFER_FAILED;
      hasher.advance(pos + n - begin);
    }
    hasher.finish(&part.crc, &part.bbh);
    release(ep, conn);
    return ErrorCode::OK;
  });
  if (ec != ErrorCode::OK) return ec;
  if (verify) {
    uint64_t got = 0;
    if (algo == ChecksumAlgo::CRC32C) {
      uint32_t crc = 0;
      bool first = true;
      for (const Part& p : parts) {
        if (p.len == 0 && !first) continue;
        crc = first ? p.crc : crc32c_combine(crc, p.crc, p.len);
        first = false;
      }
      got = crc;
    } else {
      uint64_t sum = 0;
      for (const Part& p : parts) sum += p.bbh;
      got = bbh64_finalize(sum, s.length);
    }
    if (got != s.checksum) {
      metrics_.inc("checksum_mismatch_total");
      return ErrorCode::CHECKSUM_MISMATCH;
    }
  }
  return ErrorCode::OK;
}

ErrorCode BlackbirdClient::transfer_put(const std::vector<CopyPlacement>& copies, const uint8_t* data, ChecksumAlgo algo,
                                        ShardChecksums* sums) {
  struct Job {
    size_t c, s;
    uint64_t off;
  };
  std::vector<Job> jobs;
  sums->assign(copies.size(), {});
  for (size_t c = 0; c < copies.size(); ++c) {
    uint64_t off = 0;
    (*sums)[c].assign(copies[c].shards.size(), 0);
    for (size_t s = 0; s < copies[c].shards.size(); ++s) {
      jobs.push_back({c, s, off});
      off += copies[c].shards[s].length;  // the source offset is the running shard offset (bug #8)
    }
  }
  return parallel_for(jobs.size(), opts_.io_parallelism, [&](size_t i) {
    const Job& j = jobs[i];
    return write_shard(copies[j.c].shards[j.s], data + j.off, &(*sums)[j.c][j.s], algo);
  });
}

ErrorCode BlackbirdClient::transfer_get(const std::vector<CopyPlacement>& copies, uint8_t* dst, size_t size, const StoreWindow& win) {
  ErrorCode last = ErrorCode::NO_COMPLETE_WORKER;
  for (const auto& copy : copies) {  // replica fail-over (reference reads copy 0 only, :283-287)
    uint64_t total = 0;
    for (const auto& s : copy.shards) total += s.length;
    if (total != size) {
      last = ErrorCode::DATA_CORRUPTION;
      continue;
    }
    std::vector<uint64_t> offs(copy.shards.size());
    uint64_t off = 0;
    for (size_t s = 0; s < copy.shards.size(); ++s) {
      offs[s] = off;
      off += copy.shards[s].length;
    }
    last = parallel_for(copy.shards.size(), opts_.io_parallelism, [&](size_t s) {
      if (!win.touches(offs[s], copy.shards[s].length)) return ErrorCode::OK;  // nothing to store
      return read_shard(copy.shards[s], dst + offs[s], copy.shards[s].checksum_algo);
    });
    if (last == ErrorCode::OK) return ErrorCode::OK;
    metrics_.inc("replica_failover_total");
    BB_LOG(WARNING) << "get: copy " << copy.copy_index << " failed with " << to_string(last) << ", trying next replica";
  }
  return last;
}

// ================================================================ reference API
Result<bool> BlackbirdClient::object_exists(const ObjectKey& key) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  return keystone_->object_exists(key);
}

Result<std::vector<CopyPlacement>> BlackbirdClient::get_workers(const ObjectKey& key) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  return keystone_->get_workers(key);
}

ErrorCode BlackbirdClient::put(const ObjectKey& key, const uint8_t* data, size_t size, const WorkerConfig& cfg) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  if (!data && size) return ErrorCode::INVALID_PARAMETERS;
  auto* ha = dynamic_cast<rpc::KeystoneRpcClient*>(keystone_.get());
  const uint64_t failovers = ha ? ha->failovers() : 0;
  ErrorCode ec = put_once(key, data, size, cfg);
  // The keystone failed over in the middle of this put: only completed objects are in the metadata log, so the new
  // leader has never heard of our pending one and put_complete comes back OBJECT_NOT_FOUND.  The bytes are still in
  // hand -- start over against the new leader instead of handing the caller an error that is not theirs.
  if (ec == ErrorCode::OBJECT_NOT_FOUND && ha && ha->failovers() != failovers) {
    metrics_.inc("put_restarted_after_failover_total");
    ec = put_once(key, data, size, cfg);
  }
  return ec;
}

ErrorCode BlackbirdClient::put_once(const ObjectKey& key, const uint8_t* data, size_t size, const WorkerConfig& cfg) {
  const TimePoint t0 = Clock::now();
  BB_TRACE_SPAN("client.put", size);
  auto placed = keystone_->put_start(key, size, cfg);
  if (!placed.ok()) return placed.error();
  ShardChecksums sums;
  ErrorCode ec = transfer_put(placed.value(), data, cfg.checksum, &sums);
  if (ec != ErrorCode::OK) {
    keystone_->put_cancel(key);
    metrics_.inc("put_failed_total");
    return ec;
  }
  ec = keystone_->put_complete(key, sums);
  if (ec == ErrorCode::OK) {
    metrics_.inc("put_total");
    metrics_.inc("put_bytes_total", size);
    metrics_.observe("put_latency_us", us_since(t0));
  }
  return ec;
}

// A transfer can lose a race with the Keystone moving the object (tier demotion / promotion, migrate_object, pool
// compaction, repair): the placements it holds were swapped and their extents re-used, which shows up as a digest
// mismatch or a failed read.  Fresh placements that differ from the ones just tried are worth one more attempt.
ErrorCode BlackbirdClient::get_with_refresh(const ObjectKey& key, uint8_t* (*alloc)(void*, size_t), void* ctx, size_t capacity, size_t* out_size) {
  Result<std::vector<CopyPlacement>> copies = keystone_->get_workers(key);
  ErrorCode ec = ErrorCode::OK;
  bool reread_same = false;
  for (int attempt = 0; attempt < 3; ++attempt) {
    if (!copies.ok()) return copies.error();
    if (copies.value().empty()) return ErrorCode::NO_COMPLETE_WORKER;
    size_t size = 0;
    for (const auto& s : copies.value().front().shards) size += s.length;
    if (out_size) *out_size = size;
    if (size > capacity) return ErrorCode::BUFFER_OVERFLOW;
    uint8_t* dst = alloc(ctx, size);
    ec = transfer_get(copies.value(), dst, size);
    if (ec == ErrorCode::OK) return ec;
    auto again = keystone_->get_workers(key);
    if (!again.ok()) return again.error();              // removed (or being re-written) meanwhile: that is the answer
    if (again.value() == copies.value()) {
      // Same placements.  A digest mismatch can still be a race -- the key was removed and re-put onto the very same
      // extent (first fit) and we read it half-written -- so that gets one more read; anything else is real.
      if (ec != ErrorCode::CHECKSUM_MISMATCH || reread_same) return ec;
      reread_same = true;
    }
    metrics_.inc("get_placement_refresh_total");
    copies = std::move(again);
  }
  return ec;
}

Result<std::vector<uint8_t>> BlackbirdClient::get(const ObjectKey& key) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  const TimePoint t0 = Clock::now();
  BB_TRACE_SPAN("client.get");
  std::vector<uint8_t> buf;
  size_t size = 0;
  ErrorCode ec = get_with_refresh(key, [](void* c, size_t n) {
    auto* v = static_cast<std::vector<uint8_t>*>(c);
    v->resize(n);
    return v->data();
  }, &buf, ~size_t{0}, &size);
  if (ec != ErrorCode::OK) return ec;
  metrics_.inc("get_total");
  metrics_.inc("get_bytes_total", size);
  metrics_.observe("get_latency_us", us_since(t0));
  return buf;
}

ErrorCode BlackbirdClient::get_into(const ObjectKey& key, void* buf, size_t capacity, size_t* out_size) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  return get_with_refresh(key, [](void* c, size_t) { return static_cast<uint8_t*>(c); }, buf, capacity, out_size);
}

ErrorCode BlackbirdClient::remove(const ObjectKey& key) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  return keystone_->remove_object(key);
}

// ================================================================ shared by the device calls
template <class T>
static std::vector<T> pick(const std::vector<T>& v, const std::vector<size_t>& idx) {
  std::vector<T> out;
  out.reserve(idx.size());
  for (size_t i : idx) out.push_back(v[i]);
  return out;
}

// The shaped calls over put_device, put_device_fp8, get_device and get_device_fp8.  Unless `arity_ok`, every item is
// INVALID_PARAMETERS (CLIENT_DISCONNECTED without a Keystone).  Then shape(i, &bytes) records item i's shape and returns
// its error.  For a put (`admit`) an item with an error fails here, before the Keystone allocates anything for it, and
// run(idx) puts the others as one batch, or nothing runs when there are none.  A get runs run(idx) for the others, an
// empty batch included.  <name>_total and <name>_bytes_total count the OK items and their `bytes`.
template <class Shape, class Run>
std::vector<ErrorCode> BlackbirdClient::shaped_batch(std::string_view name, bool admit, size_t n, bool arity_ok, Shape&& shape, Run&& run) {
  if (!arity_ok) return std::vector<ErrorCode>(n, keystone_ ? ErrorCode::INVALID_PARAMETERS : ErrorCode::CLIENT_DISCONNECTED);
  std::vector<ErrorCode> out(n, ErrorCode::OK);
  std::vector<uint64_t> bytes(n, 0);
  std::vector<size_t> idx;
  idx.reserve(n);
  for (size_t i = 0; i < n; ++i) {
    out[i] = shape(i, &bytes[i]);
    if (out[i] == ErrorCode::OK) idx.push_back(i);
  }
  if (admit && idx.empty()) return out;
  const std::vector<ErrorCode> ecs = run(idx);
  uint64_t done = 0, total = 0;
  for (size_t j = 0; j < idx.size(); ++j) {
    out[idx[j]] = ecs[j];
    if (ecs[j] == ErrorCode::OK) ++done, total += bytes[idx[j]];
  }
  metrics_.inc(std::string(name) + "_total", done);
  metrics_.inc(std::string(name) + "_bytes_total", total);
  return out;
}

// What the builder of a shaped put or get makes of item i: the layout of the caller's side and the object's size, in
// bytes or, for MXFP8, in elements of the wide side.  `table`: the size is that of a table (pages, blocks or segments),
// not of rows.
struct ShapedItem {
  DeviceLayout mem;
  uint64_t units = 0;
  bool table = false;
  std::vector<SegmentEntry> segments;  // the table a SEGMENTS layout points into
};

static ErrorCode rows_item(uint64_t width, uint64_t pitch, uint64_t rows, ShapedItem* it) {
  uint64_t extent = 0;  // admit_shaped has it from the layout
  return DeviceLayout::from_rows(width, pitch, rows, &it->mem, &it->units, &extent);
}

// Item i of a paged call: its pages, with the in-page row pattern page_rows[i] when the call has one ((0, 0): none).
static ErrorCode pages_item(const std::vector<uint64_t>& pages, uint64_t page, const std::vector<PageRows>& page_rows, size_t i,
                            ShapedItem* it) {
  it->table = true;
  const PageRows r = page_rows.empty() ? PageRows{} : page_rows[i];
  return DeviceLayout::from_pages(pages.size(), page, pages.data(), &it->mem, &it->units, r.first, r.second);
}

static ErrorCode blocks_item(const SourceBlocks& blocks, ShapedItem* it) {
  SourceBlocks b;
  const ErrorCode ec = SourceBlocks::from_blocks(blocks, &b, &it->units);
  it->mem = DeviceLayout(b);
  it->table = true;
  return ec;
}

// Item i of a segment call, its segments in units of `unit` bytes (1, or for MXFP8 the wide type's).
static ErrorCode segments_item(const std::vector<SourceSegments::Segment>& segs, uint64_t unit, ShapedItem* it) {
  SourceSegments g;
  const ErrorCode ec = SourceSegments::from_segments(segs.data(), segs.size(), &it->segments, &g, &it->units, unit);
  it->mem = DeviceLayout(g);
  it->table = true;
  return ec;
}

// The admission rule of the shaped calls (blackbird_client.h), in this order: an item of a put or a get of units of b
// bytes (`packed`: MXFP8 elements), its layout at `base`.
static ErrorCode admit_shaped(const ShapedItem& it, bool put, uint64_t b, bool packed, const void* base) {
  const DeviceLayout& m = it.mem;
  const uint64_t u = it.units;
  if (packed && it.table && (u == 0 || u % 32)) return ErrorCode::INVALID_ARGUMENT;  // no packed object has that many elements
  if (put && (m.pages().has_null(u) || m.blocks().has_null() || m.segments().has_null(u))) return ErrorCode::INVALID_ARGUMENT;  // a put reads every unit
  if (u > SIZE_MAX) return ErrorCode::VALUE_OUT_OF_RANGE;
  DeviceLayout bytes;
  const uint64_t extent = m.kind() == DeviceLayout::ROWS ? m.rows().extent(u) : u;
  if (packed && (extent > UINT64_MAX / b || !m.to_wide_bytes(b, &bytes))) return ErrorCode::VALUE_OUT_OF_RANGE;
  // the engine's rule for a gathering pack, checked once: there is no host-staged path for packed puts
  if (packed && put && !bytes.coaligned(reinterpret_cast<uintptr_t>(base), b * u)) return ErrorCode::NOT_IMPLEMENTED;
  // the resolve kernel checks a get's ids for duplicates in a bitmap of bounded size: larger caches are the caller's
  if (!put && !m.blocks().distinct_checkable()) return ErrorCode::NOT_IMPLEMENTED;
  return ErrorCode::OK;
}

template <class Build>
std::vector<ErrorCode> BlackbirdClient::shaped_put(std::string_view name, const std::vector<ObjectKey>& keys, const std::vector<const void*>& ptrs,
                                                   bool arity_ok, std::optional<mxfp8::Wide> fp8, Build&& build, const WorkerConfig& cfg,
                                                   void* stream) {
  const uint64_t b = fp8 ? mxfp8::wide_bytes(*fp8) : 1;
  std::vector<ShapedItem> items(keys.size());
  return shaped_batch(
      name, true, keys.size(), arity_ok,
      [&](size_t i, uint64_t* bytes) {
        ErrorCode ec = build(i, &items[i]);
        if (ec == ErrorCode::OK) ec = admit_shaped(items[i], true, b, fp8.has_value(), ptrs[i]);
        *bytes = b * items[i].units;
        return ec;
      },
      [&](const std::vector<size_t>& idx) {
        std::vector<DeviceLayout> mems;
        std::vector<uint64_t> units;
        for (size_t i : idx) mems.push_back(items[i].mem), units.push_back(items[i].units);
        if (fp8) return put_device_fp8(pick(keys, idx), pick(ptrs, idx), units, &mems, cfg, stream, *fp8);
        return put_device(pick(keys, idx), pick(ptrs, idx), std::vector<size_t>(units.begin(), units.end()), &mems, cfg, stream);
      });
}

template <class Build>
std::vector<ErrorCode> BlackbirdClient::shaped_get(std::string_view name, const std::vector<ObjectKey>& keys, const std::vector<void*>& ptrs,
                                                   bool arity_ok, std::optional<mxfp8::Wide> fp8, Build&& build, void* stream,
                                                   std::vector<size_t>* out_sizes) {
  const uint64_t b = fp8 ? mxfp8::wide_bytes(*fp8) : 1;
  std::vector<ShapedItem> items(keys.size());
  if (out_sizes) out_sizes->assign(keys.size(), 0);
  return shaped_batch(
      name, false, keys.size(), arity_ok,
      [&](size_t i, uint64_t* bytes) {
        ErrorCode ec = build(i, &items[i]);
        if (ec == ErrorCode::OK) ec = admit_shaped(items[i], false, b, fp8.has_value(), ptrs[i]);
        *bytes = b * items[i].units;
        return ec;
      },
      [&](const std::vector<size_t>& idx) {
        std::vector<DeviceLayout> mems;
        std::vector<uint64_t> units;
        for (size_t i : idx) mems.push_back(items[i].mem), units.push_back(items[i].units);
        if (fp8) {  // a fused get stores exactly the units its layout holds
          auto ecs = get_device_fp8(pick(keys, idx), pick(ptrs, idx), units, nullptr, &mems, stream, *fp8);
          for (size_t k = 0; out_sizes && k < idx.size(); ++k) (*out_sizes)[idx[k]] = ecs[k] == ErrorCode::OK ? units[k] : 0;
          return ecs;
        }
        std::vector<size_t> sizes;
        auto ecs = get_device(pick(keys, idx), pick(ptrs, idx), std::vector<size_t>(units.begin(), units.end()), nullptr, &mems, stream, &sizes);
        for (size_t k = 0; out_sizes && k < idx.size() && k < sizes.size(); ++k) (*out_sizes)[idx[k]] = sizes[k];
        return ecs;
      });
}

// A digest mismatch on every replica can also mean that the Keystone moved the object under us (tier move, compaction,
// repair): the extents we read were freed and re-used.  Items whose placements changed since we fetched them get one
// more pass, reissue(idx) being the same get of items idx; so do unchanged ones once, at the outermost call, because a
// remove + re-put can land on the very same extent (first fit) and be read half-written.  Passes nest at most twice.
static thread_local int refresh_depth = 0;

template <class Reissue>
void BlackbirdClient::refresh_placements(const std::vector<ObjectKey>& keys, const std::vector<Result<std::vector<CopyPlacement>>>& placed,
                                         std::vector<ErrorCode>& out, Reissue&& reissue) {
  if (refresh_depth >= 2) return;
  std::vector<size_t> bad;
  for (size_t i = 0; i < keys.size(); ++i)
    if (out[i] == ErrorCode::CHECKSUM_MISMATCH && placed[i].ok()) bad.push_back(i);
  if (bad.empty()) return;
  const auto again = keystone_->batch_get_workers(pick(keys, bad));
  std::vector<size_t> redo;
  for (size_t k = 0; k < bad.size(); ++k) {
    const size_t i = bad[k];
    if (!again[k].ok()) out[i] = again[k].error();  // removed (or being re-written) meanwhile: that is the answer
    else if (!(again[k].value() == placed[i].value()) || refresh_depth == 0) redo.push_back(i);
  }
  if (redo.empty()) return;
  metrics_.inc("get_placement_refresh_total", redo.size());
  ++refresh_depth;
  const std::vector<ErrorCode> recs = reissue(redo);
  --refresh_depth;
  for (size_t k = 0; k < redo.size(); ++k) out[redo[k]] = recs[k];
}

// ================================================================ fused MXFP8 device API
std::vector<ErrorCode> BlackbirdClient::batch_put_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                                             const std::vector<uint64_t>& n_elems, const WorkerConfig& cfg, void* stream,
                                                             mxfp8::Wide wide) {
  return put_device_fp8(keys, bf16_ptrs, n_elems, nullptr, cfg, stream, wide);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_fp8_strided(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                                                     const std::vector<uint64_t>& elem_widths,
                                                                     const std::vector<uint64_t>& elem_pitches,
                                                                     const std::vector<uint64_t>& rows, const WorkerConfig& cfg, void* stream,
                                                                     mxfp8::Wide wide) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_fp8_strided", keys, bf16_ptrs,
      bf16_ptrs.size() == n && elem_widths.size() == n && elem_pitches.size() == n && rows.size() == n, wide,
      [&](size_t i, ShapedItem* it) { return rows_item(elem_widths[i], elem_pitches[i], rows[i], it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_fp8_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                                   const std::vector<uint64_t>& page_elems, const WorkerConfig& cfg, void* stream,
                                                                   mxfp8::Wide wide, const std::vector<PageRows>& page_rows) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_fp8_paged", keys, std::vector<const void*>(n), pages.size() == n && page_elems.size() == n && (page_rows.empty() || page_rows.size() == n), wide,
      [&](size_t i, ShapedItem* it) { return pages_item(pages[i], page_elems[i], page_rows, i, it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::put_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<const void*>& bf16_ptrs,
                                                       const std::vector<uint64_t>& n_elems, const std::vector<DeviceLayout>* mem,
                                                       const WorkerConfig& cfg, void* stream, mxfp8::Wide wide) {
  std::vector<ErrorCode> out(keys.size(), ErrorCode::INVALID_PARAMETERS);
  if (!keystone_) return std::vector<ErrorCode>(keys.size(), ErrorCode::CLIENT_DISCONNECTED);
  if (!device_) return std::vector<ErrorCode>(keys.size(), ErrorCode::NOT_IMPLEMENTED);
  if (bf16_ptrs.size() != keys.size() || n_elems.size() != keys.size() || (mem && mem->size() != keys.size())) return out;
  BB_TRACE_SPAN("batch_put_device_fp8", keys.size());
  WorkerConfig c = cfg;
  c.replication_factor = std::max<size_t>(1, std::min<size_t>(cfg.replication_factor, 3));  // one tile pass fans out to <= 3 copies
  c.max_workers_per_copy = 1;    // payload + scales of an object stay in one shard
  c.checksum = ChecksumAlgo::BBH64;
  c.pack_fp8 = true;
  if (c.preferred_classes.empty()) c.preferred_classes = {StorageClass::RAM_GPU};
  std::vector<PutStartItem> items;
  for (size_t i = 0; i < keys.size(); ++i) {
    if (!device_->fp8_eligible(n_elems[i])) return out;
    items.push_back(PutStartItem{keys[i], static_cast<size_t>(n_elems[i] + n_elems[i] / 32), c});
  }
  auto placed = keystone_->batch_put_start(items);
  std::vector<DeviceFp8Op> ops;
  std::vector<size_t> idx;
  for (size_t i = 0; i < keys.size(); ++i) {
    if (!placed[i].ok()) {
      out[i] = placed[i].error();
      continue;
    }
    const auto& copies = placed[i].value();
    bool fits = !copies.empty() && copies.size() <= 3;
    for (const auto& cp : copies) fits = fits && cp.shards.size() == 1 && device_->can_reach(cp.shards[0]);
    if (!fits) {
      keystone_->put_cancel(keys[i]);
      out[i] = ErrorCode::NOT_IMPLEMENTED;  // a copy is not a single GPU-fabric shard: caller packs + puts instead
      continue;
    }
    DeviceFp8Op op{&copies[0].shards[0], const_cast<void*>(bf16_ptrs[i]), n_elems[i], {}};
    if (mem) op.mem = (*mem)[i];
    op.wide_type = wide;
    for (size_t cidx = 1; cidx < copies.size(); ++cidx) op.replicas.push_back(&copies[cidx].shards[0]);
    ops.push_back(std::move(op));
    idx.push_back(i);
  }
  DeviceBatchResult res;
  ErrorCode ec = ops.empty() ? ErrorCode::OK : device_->run_fp8(ops, false, stream, &res);
  std::vector<ObjectKey> done;
  std::vector<ShardChecksums> sums;
  for (size_t k = 0; k < idx.size(); ++k) {
    const ErrorCode v = ec != ErrorCode::OK ? ec : res.verdicts[k];  // refused ids: the answer, and no digest
    if (v != ErrorCode::OK || res.digests.size() != idx.size()) {
      keystone_->put_cancel(keys[idx[k]]);
      out[idx[k]] = v != ErrorCode::OK ? v : ErrorCode::INTERNAL_ERROR;
      continue;
    }
    done.push_back(keys[idx[k]]);
    sums.push_back(ShardChecksums(placed[idx[k]].value().size(), std::vector<uint64_t>{res.digests[k]}));  // same bytes in every copy
  }
  if (!done.empty()) {
    auto r = keystone_->batch_put_complete(done, sums);
    size_t j = 0;
    for (size_t k = 0; k < idx.size(); ++k)
      if (out[idx[k]] == ErrorCode::INVALID_PARAMETERS) out[idx[k]] = r[j++];
  }
  metrics_.inc("device_put_fp8_batches_total");
  return out;
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                             const std::vector<uint64_t>& n_elems, void* stream, mxfp8::Wide wide) {
  return get_device_fp8(keys, bf16_ptrs, n_elems, nullptr, nullptr, stream, wide);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                                     const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_widths,
                                                                     const std::vector<uint64_t>& elem_pitches, const std::vector<uint64_t>& rows,
                                                                     void* stream, mxfp8::Wide wide) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_fp8_scatter", keys, bf16_ptrs,
      bf16_ptrs.size() == n && n_elems.size() == n && elem_widths.size() == n && elem_pitches.size() == n && rows.size() == n, wide,
      [&](size_t i, ShapedItem* it) {
        const ErrorCode ec = rows_item(elem_widths[i], elem_pitches[i], rows[i], it);
        return ec != ErrorCode::OK || it->units == n_elems[i] ? ec : ErrorCode::INVALID_ARGUMENT;
      },
      stream, nullptr);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_range(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                                   const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_offsets,
                                                                   const std::vector<uint64_t>& elem_counts, void* stream, mxfp8::Wide wide) {
  const size_t n = keys.size();
  const uint64_t b = mxfp8::wide_bytes(wide);
  std::vector<ByteRange> ranges(n);
  return shaped_batch(
      "device_get_fp8_range", false, n, elem_offsets.size() == n && elem_counts.size() == n,
      [&](size_t i, uint64_t* bytes) {
        ranges[i] = {elem_offsets[i], elem_counts[i]};
        *bytes = b * elem_counts[i];
        return ErrorCode::OK;
      },
      [&](const std::vector<size_t>&) { return get_device_fp8(keys, bf16_ptrs, n_elems, &ranges, nullptr, stream, wide); });
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_strided(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                                     const std::vector<uint64_t>& n_elems, const std::vector<uint64_t>& elem_offsets,
                                                                     const std::vector<uint64_t>& elem_widths, const std::vector<uint64_t>& elem_pitches,
                                                                     const std::vector<uint64_t>& rows, void* stream, mxfp8::Wide wide) {
  const size_t n = keys.size();
  const uint64_t b = mxfp8::wide_bytes(wide);
  std::vector<ByteRange> ranges(n);
  return shaped_batch(
      "device_get_fp8_strided", false, n, elem_offsets.size() == n && elem_widths.size() == n && elem_pitches.size() == n && rows.size() == n,
      [&](size_t i, uint64_t* bytes) {
        ranges[i] = {elem_offsets[i], elem_widths[i], elem_pitches[i], rows[i]};
        *bytes = b * rows[i] * elem_widths[i];  // counted for OK items only, whose rows lie inside the object
        return ErrorCode::OK;
      },
      [&](const std::vector<size_t>&) { return get_device_fp8(keys, bf16_ptrs, n_elems, &ranges, nullptr, stream, wide); });
}

// The destination of a slice get's result of `units` units: rows of dst_width units every dst_pitch units, as many as the
// result fills (the last one possibly in part), with SourceRows::from_rows' errors; INVALID_ARGUMENT for a zero width with
// a result.
static ErrorCode result_rows(uint64_t units, uint64_t dst_width, uint64_t dst_pitch, DeviceLayout* out) {
  *out = {};
  if (units == 0) return ErrorCode::OK;
  if (dst_width == 0) return ErrorCode::INVALID_ARGUMENT;
  SourceRows r;
  uint64_t size = 0, extent = 0;
  const ErrorCode ec = SourceRows::from_rows(dst_width, dst_pitch, (units - 1) / dst_width + 1, &r, &size, &extent);
  *out = DeviceLayout::window_rows(r);
  return ec;
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_strided_scatter(
    const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs, const std::vector<uint64_t>& n_elems,
    const std::vector<uint64_t>& elem_offsets, const std::vector<uint64_t>& elem_widths, const std::vector<uint64_t>& elem_pitches,
    const std::vector<uint64_t>& rows, const std::vector<uint64_t>& dst_widths, const std::vector<uint64_t>& dst_pitches, void* stream,
    mxfp8::Wide wide) {
  const size_t n = keys.size();
  const uint64_t b = mxfp8::wide_bytes(wide);
  std::vector<ByteRange> ranges(n);
  std::vector<DeviceLayout> mem(n);
  return shaped_batch(
      "device_get_fp8_strided_scatter", false, n,
      bf16_ptrs.size() == n && n_elems.size() == n && elem_offsets.size() == n && elem_widths.size() == n && elem_pitches.size() == n &&
          rows.size() == n && dst_widths.size() == n && dst_pitches.size() == n,
      [&](size_t i, uint64_t* bytes) {
        ranges[i] = {elem_offsets[i], elem_widths[i], elem_pitches[i], rows[i]};
        uint64_t total = 0;
        if (__builtin_mul_overflow(rows[i], elem_widths[i], &total)) return ErrorCode::VALUE_OUT_OF_RANGE;
        *bytes = b * total;  // counted for OK items only, whose rows lie inside the object
        return result_rows(total, dst_widths[i], dst_pitches[i], &mem[i]);
      },
      [&](const std::vector<size_t>& idx) {
        const auto rr = pick(ranges, idx);
        const auto rm = pick(mem, idx);
        return get_device_fp8(pick(keys, idx), pick(bf16_ptrs, idx), pick(n_elems, idx), &rr, &rm, stream, wide);
      });
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                                   const std::vector<uint64_t>& page_elems, void* stream, mxfp8::Wide wide,
                                                                   const std::vector<PageRows>& page_rows) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_fp8_paged", keys, std::vector<void*>(n), pages.size() == n && page_elems.size() == n && (page_rows.empty() || page_rows.size() == n), wide,
      [&](size_t i, ShapedItem* it) { return pages_item(pages[i], page_elems[i], page_rows, i, it); }, stream, nullptr);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_fp8_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks,
                                                                    const WorkerConfig& cfg, void* stream, mxfp8::Wide wide) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_fp8_blocks", keys, std::vector<const void*>(n), blocks.size() == n, wide,
      [&](size_t i, ShapedItem* it) { return blocks_item(blocks[i], it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks,
                                                                    void* stream, mxfp8::Wide wide) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_fp8_blocks", keys, std::vector<void*>(n), blocks.size() == n, wide,
      [&](size_t i, ShapedItem* it) { return blocks_item(blocks[i], it); }, stream, nullptr);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_fp8_segments(const std::vector<ObjectKey>& keys,
                                                                      const std::vector<std::vector<SourceSegments::Segment>>& segments,
                                                                      const WorkerConfig& cfg, void* stream, mxfp8::Wide wide) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_fp8_segments", keys, std::vector<const void*>(n), segments.size() == n, wide,
      [&](size_t i, ShapedItem* it) { return segments_item(segments[i], mxfp8::wide_bytes(wide), it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_fp8_segments(const std::vector<ObjectKey>& keys,
                                                                      const std::vector<std::vector<SourceSegments::Segment>>& segments,
                                                                      void* stream, std::vector<size_t>* out_sizes, mxfp8::Wide wide) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_fp8_segments", keys, std::vector<void*>(n), segments.size() == n, wide,
      [&](size_t i, ShapedItem* it) { return segments_item(segments[i], mxfp8::wide_bytes(wide), it); }, stream, out_sizes);
}

std::vector<ErrorCode> BlackbirdClient::get_device_fp8(const std::vector<ObjectKey>& keys, const std::vector<void*>& bf16_ptrs,
                                                       const std::vector<uint64_t>& n_elems, const std::vector<ByteRange>* ranges,
                                                       const std::vector<DeviceLayout>* mem, void* stream, mxfp8::Wide wide) {
  std::vector<ErrorCode> out(keys.size(), ErrorCode::INVALID_PARAMETERS);
  const uint64_t b = mxfp8::wide_bytes(wide);
  if (!keystone_) return std::vector<ErrorCode>(keys.size(), ErrorCode::CLIENT_DISCONNECTED);
  if (!device_) return std::vector<ErrorCode>(keys.size(), ErrorCode::NOT_IMPLEMENTED);
  if (bf16_ptrs.size() != keys.size() || n_elems.size() != keys.size() || (ranges && ranges->size() != keys.size()) ||
      (mem && mem->size() != keys.size()))
    return out;
  auto mem_of = [&](size_t i) { return mem ? (*mem)[i] : DeviceLayout{}; };
  BB_TRACE_SPAN("batch_get_device_fp8", keys.size());
  auto placed = keystone_->batch_get_workers(keys);
  std::vector<std::vector<size_t>> candidates(keys.size());
  std::vector<size_t> idx;
  // The elements each get stores, and the base they land relative to: the caller's pointer, less the window's offset for
  // a range get (the virtual base; the kernel never touches an address outside the range).
  std::vector<StoreWindow> wins(keys.size());
  std::vector<void*> bases = bf16_ptrs;
  for (size_t i = 0; i < keys.size(); ++i) {
    if (!placed[i].ok()) {
      out[i] = placed[i].error();
      continue;
    }
    StoreWindow& w = wins[i];
    if (ranges) {
      const ByteRange& r = (*ranges)[i];
      const ErrorCode ec = StoreWindow::from_rows(r.offset, r.length, r.pitch, r.rows, n_elems[i], &w);
      if (ec != ErrorCode::OK || w.empty()) {  // an error, or nothing to read or store
        out[i] = ec;
        continue;
      }
      // rows of the result (WINDOW_ROWS) start at the caller's pointer
      if (mem_of(i).kind() != DeviceLayout::WINDOW_ROWS)
        bases[i] = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(bf16_ptrs[i]) - b * w.base_shift(w.lo));
    }
    const auto& copies = placed[i].value();
    const uint64_t packed = n_elems[i] + n_elems[i] / 32;
    const DeviceLayout::Kind kind = mem_of(i).kind();
    // the pages or segments must hold exactly the stored object's elements
    if ((kind == DeviceLayout::PAGES || kind == DeviceLayout::BLOCKS || kind == DeviceLayout::SEGMENTS) && !copies.empty()) {
      uint64_t stored = 0;
      for (const auto& sh : copies[0].shards) stored += sh.length;
      if (stored != packed) {
        out[i] = ErrorCode::INVALID_ARGUMENT;
        continue;
      }
    }
    // usable copies: single GPU-fabric shard holding the whole packed object with a BBH64 digest; a copy in this
    // client's own HBM first, the others in hashed order (readers spread over the replicas)
    std::vector<size_t> order;
    const size_t start = copies.empty() ? 0 : std::hash<std::string>{}(opts_.node_id + keys[i]) % copies.size();
    for (int pass = 0; pass < 2; ++pass)
      for (size_t k = 0; k < copies.size(); ++k) {
        const size_t cidx = (start + k) % copies.size();
        const auto& cp = copies[cidx];
        if (cp.shards.size() != 1 || cp.shards[0].length != packed || cp.shards[0].checksum_algo != ChecksumAlgo::BBH64) continue;
        if (!device_->can_reach(cp.shards[0]) || device_->is_local(cp.shards[0]) != (pass == 0)) continue;
        order.push_back(cidx);
      }
    if (!device_->fp8_eligible(n_elems[i]) || order.empty()) {
      out[i] = ErrorCode::NOT_IMPLEMENTED;  // demoted to a host tier, striped, other digest: caller gets + unpacks instead
      continue;
    }
    // a range or a layout the kernel cannot store into (DeviceLayout::fused_get_aligned) fails alone, so that the rest of
    // the batch still takes the fused launch; the caller reads it whole and slices instead.  A whole tensor of a plain get
    // is left to the engine.
    StoreWindow bytes;
    DeviceLayout dst_bytes;
    if ((ranges || mem) &&
        (!w.to_wide_bytes(b, &bytes) || !mem_of(i).to_wide_bytes(b, &dst_bytes) ||
         !dst_bytes.fused_get_aligned(reinterpret_cast<uintptr_t>(bf16_ptrs[i]), 0, b * n_elems[i], bytes))) {
      out[i] = ErrorCode::NOT_IMPLEMENTED;
      continue;
    }
    candidates[i] = std::move(order);
    idx.push_back(i);
  }
  // one fused launch per attempt; objects whose digest did not verify are retried on their next replica
  std::vector<size_t> todo = idx;
  for (size_t attempt = 0; !todo.empty(); ++attempt) {
    std::vector<DeviceFp8Op> ops;
    std::vector<size_t> cur;
    for (size_t i : todo) {
      if (attempt >= candidates[i].size()) {
        out[i] = ErrorCode::CHECKSUM_MISMATCH;
        continue;
      }
      ops.push_back({&placed[i].value()[candidates[i][attempt]].shards[0], bases[i], n_elems[i], {}, wins[i], mem_of(i), wide});
      cur.push_back(i);
    }
    if (ops.empty()) break;
    if (attempt > 0) metrics_.inc("replica_failover_total");
    DeviceBatchResult res;
    ErrorCode ec = device_->run_fp8(ops, true, stream, &res);
    todo.clear();
    for (size_t k = 0; k < cur.size(); ++k) {
      if (ec != ErrorCode::OK || res.status.size() != cur.size()) out[cur[k]] = ec != ErrorCode::OK ? ec : ErrorCode::INTERNAL_ERROR;
      else if (res.verdicts[k] != ErrorCode::OK) out[cur[k]] = res.verdicts[k];  // its ids, not its copy: no fail-over
      else if (res.status[k]) todo.push_back(cur[k]);
      else out[cur[k]] = ErrorCode::OK;
    }
  }
  // a key that moved to a non-fusable placement comes back NOT_IMPLEMENTED from the refresh, i.e. "get + unpack instead"
  refresh_placements(keys, placed, out, [&](const std::vector<size_t>& r) {
    const auto rranges = ranges ? pick(*ranges, r) : std::vector<ByteRange>();
    const auto rmem = mem ? pick(*mem, r) : std::vector<DeviceLayout>();
    return get_device_fp8(pick(keys, r), pick(bf16_ptrs, r), pick(n_elems, r), ranges ? &rranges : nullptr, mem ? &rmem : nullptr, stream,
                          wide);
  });
  metrics_.inc("device_get_fp8_batches_total");
  return out;
}

ErrorCode BlackbirdClient::migrate(const ObjectKey& key, StorageClass target) {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  return keystone_->migrate_object(key, target);
}

Result<ClusterStats> BlackbirdClient::cluster_stats() {
  if (!keystone_) return ErrorCode::CLIENT_DISCONNECTED;
  return keystone_->get_cluster_stats();
}

// ================================================================ batched host API
std::vector<ErrorCode> BlackbirdClient::batch_put(const std::vector<ObjectKey>& keys, const std::vector<const uint8_t*>& data,
                                                  const std::vector<size_t>& sizes, const WorkerConfig& cfg) {
  std::vector<ErrorCode> out(keys.size(), ErrorCode::INVALID_PARAMETERS);
  if (!keystone_) return std::vector<ErrorCode>(keys.size(), ErrorCode::CLIENT_DISCONNECTED);
  if (data.size() != keys.size() || sizes.size() != keys.size()) return out;
  std::vector<PutStartItem> items(keys.size());
  for (size_t i = 0; i < keys.size(); ++i) items[i] = PutStartItem{keys[i], sizes[i], cfg};
  auto placed = keystone_->batch_put_start(items);  // ONE control-plane round trip for the batch
  std::vector<ShardChecksums> sums(keys.size());
  std::vector<ObjectKey> done_keys, cancel_keys;
  std::vector<ShardChecksums> done_sums;
  std::vector<size_t> done_idx;
  parallel_for(keys.size(), opts_.io_parallelism, [&](size_t i) {
    if (!placed[i].ok()) {
      out[i] = placed[i].error();
      return ErrorCode::OK;
    }
    out[i] = transfer_put(placed[i].value(), data[i], cfg.checksum, &sums[i]);
    return ErrorCode::OK;
  });
  for (size_t i = 0; i < keys.size(); ++i) {
    if (!placed[i].ok()) continue;
    if (out[i] == ErrorCode::OK) {
      done_keys.push_back(keys[i]);
      done_sums.push_back(std::move(sums[i]));
      done_idx.push_back(i);
    } else {
      cancel_keys.push_back(keys[i]);
    }
  }
  if (!cancel_keys.empty()) keystone_->batch_put_cancel(cancel_keys);
  if (!done_keys.empty()) {
    auto ecs = keystone_->batch_put_complete(done_keys, done_sums);
    for (size_t k = 0; k < done_idx.size(); ++k) out[done_idx[k]] = ecs[k];
  }
  return out;
}

std::vector<Result<std::vector<uint8_t>>> BlackbirdClient::batch_get(const std::vector<ObjectKey>& keys) {
  std::vector<Result<std::vector<uint8_t>>> out(keys.size(), Result<std::vector<uint8_t>>(ErrorCode::CLIENT_DISCONNECTED));
  if (!keystone_) return out;
  auto placed = keystone_->batch_get_workers(keys);
  parallel_for(keys.size(), opts_.io_parallelism, [&](size_t i) {
    if (!placed[i].ok()) {
      out[i] = placed[i].error();
      return ErrorCode::OK;
    }
    if (placed[i].value().empty()) {
      out[i] = ErrorCode::NO_COMPLETE_WORKER;
      return ErrorCode::OK;
    }
    size_t size = 0;
    for (const auto& s : placed[i].value().front().shards) size += s.length;
    std::vector<uint8_t> buf(size);
    ErrorCode ec = transfer_get(placed[i].value(), buf.data(), size);
    if (ec == ErrorCode::OK) out[i] = std::move(buf);
    else out[i] = ec;
    return ErrorCode::OK;
  });
  return out;
}

std::vector<ErrorCode> BlackbirdClient::batch_remove(const std::vector<ObjectKey>& keys) {
  if (!keystone_) return std::vector<ErrorCode>(keys.size(), ErrorCode::CLIENT_DISCONNECTED);
  const TimePoint t0 = Clock::now();
  auto r = keystone_->batch_remove_object(keys);
  metrics_.observe("phase_remove_us", us_since(t0));
  return r;
}

std::vector<Result<bool>> BlackbirdClient::batch_exists(const std::vector<ObjectKey>& keys) {
  if (!keystone_) return std::vector<Result<bool>>(keys.size(), Result<bool>(ErrorCode::CLIENT_DISCONNECTED));
  return keystone_->batch_object_exists(keys);
}

// ================================================================ batched device API
std::vector<std::pair<size_t, size_t>> BlackbirdClient::plan_chunks(const std::vector<size_t>& sizes, double rpc_us_per_object) const {
  std::vector<std::pair<size_t, size_t>> chunks;
  uint64_t total = 0;
  for (size_t s : sizes) total += s;
  constexpr uint64_t kMinChunk = 256ull << 20;  // below this a chunk's kernel is too short to hide an RPC
  constexpr double kLaunchPenaltyUs = 120.0;    // measured: ramp + tail + launch gap + result read-back of one more fused launch
  const size_t depth = device_ ? device_->max_in_flight() : 1;
  size_t want = 1;
  if (depth >= 2 && sizes.size() >= 2 && total >= 2 * kMinChunk) {
    if (pipeline_chunks_ > 0) {
      want = pipeline_chunks_;
    } else {
      // Splitting hides (1 - 1/c) of the control-plane time behind kernels and costs (c - 1) launch penalties.
      // An in-process Keystone (tens of us per batch) is not worth a split; a remote one (100s of us) is.
      const double rpc_us = rpc_us_per_object * static_cast<double>(sizes.size());
      double best = 0;
      for (size_t c : {size_t{2}, size_t{4}}) {
        const double gain = rpc_us * (1.0 - 1.0 / static_cast<double>(c)) - static_cast<double>(c - 1) * kLaunchPenaltyUs;
        if (gain > best) best = gain, want = c;
      }
    }
    want = std::min<size_t>({want, static_cast<size_t>(total / kMinChunk), sizes.size()});
  }
  if (want <= 1) {
    chunks.emplace_back(0, sizes.size());
    return chunks;
  }
  const uint64_t target = total / want;
  size_t begin = 0;
  uint64_t acc = 0;
  for (size_t i = 0; i < sizes.size(); ++i) {
    acc += sizes[i];
    if (acc >= target && i + 1 < sizes.size() && chunks.size() + 1 < want) {
      chunks.emplace_back(begin, i + 1);
      begin = i + 1;
      acc = 0;
    }
  }
  chunks.emplace_back(begin, sizes.size());
  return chunks;
}

static void ewma_update(std::atomic<double>& v, double sample) {
  const double old = v.load(std::memory_order_relaxed);
  v.store(old == 0 ? sample : 0.75 * old + 0.25 * sample, std::memory_order_relaxed);
}

// The fused kernels move 16-byte aligned buffers only (XferEngine::submit refuses a whole batch otherwise).  An object
// whose caller buffer is not aligned with one of its shards is staged through host memory instead, so that it does not
// fail its neighbours: a put's source by DeviceLayout::coaligned from every shard's start, a get's destination by
// DeviceLayout::fused_get_aligned.  Whether ok(off, len) holds for the shard [off, off + len) of every copy.
template <class F>
static bool fabric_aligned(const std::vector<CopyPlacement>& copies, F&& ok) {
  for (const auto& c : copies) {
    uint64_t off = 0;
    for (const auto& sh : c.shards) {
      if (!ok(off, sh.length)) return false;
      off += sh.length;
    }
  }
  return true;
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs,
                                                         const std::vector<size_t>& sizes, const WorkerConfig& cfg, void* stream) {
  return put_device(keys, dev_ptrs, sizes, nullptr, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_strided(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs,
                                                                 const std::vector<uint64_t>& widths, const std::vector<uint64_t>& pitches,
                                                                 const std::vector<uint64_t>& rows, const WorkerConfig& cfg, void* stream) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_strided", keys, dev_ptrs, dev_ptrs.size() == n && widths.size() == n && pitches.size() == n && rows.size() == n,
      std::nullopt, [&](size_t i, ShapedItem* it) { return rows_item(widths[i], pitches[i], rows[i], it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                               const std::vector<uint64_t>& page_bytes, const WorkerConfig& cfg, void* stream,
                                                               const std::vector<PageRows>& page_rows) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_paged", keys, std::vector<const void*>(n), pages.size() == n && page_bytes.size() == n && (page_rows.empty() || page_rows.size() == n), std::nullopt,
      [&](size_t i, ShapedItem* it) { return pages_item(pages[i], page_bytes[i], page_rows, i, it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_segments(const std::vector<ObjectKey>& keys,
                                                                  const std::vector<std::vector<SourceSegments::Segment>>& segments,
                                                                  const WorkerConfig& cfg, void* stream) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_segments", keys, std::vector<const void*>(n), segments.size() == n, std::nullopt,
      [&](size_t i, ShapedItem* it) { return segments_item(segments[i], 1, it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::put_device(const std::vector<ObjectKey>& keys, const std::vector<const void*>& dev_ptrs,
                                                   const std::vector<size_t>& sizes, const std::vector<DeviceLayout>* mem,
                                                   const WorkerConfig& cfg, void* stream) {
  std::vector<ErrorCode> out(keys.size(), ErrorCode::INVALID_PARAMETERS);
  if (!keystone_) return std::vector<ErrorCode>(keys.size(), ErrorCode::CLIENT_DISCONNECTED);
  if (!device_) return std::vector<ErrorCode>(keys.size(), ErrorCode::NOT_IMPLEMENTED);
  if (dev_ptrs.size() != keys.size() || sizes.size() != keys.size() || (mem && mem->size() != keys.size())) return out;
  auto mem_of = [&](size_t i) { return mem ? (*mem)[i] : DeviceLayout{}; };
  const TimePoint t_all = Clock::now();
  BB_TRACE_SPAN("batch_put_device", keys.size());

  struct Chunk {
    size_t begin = 0, end = 0;
    std::vector<Result<std::vector<CopyPlacement>>> placed;
    std::vector<DeviceShardOp> ops;
    uint64_t ticket = 0;
    bool submitted = false;
    ErrorCode submit_error = ErrorCode::OK;
  };
  const auto plan = plan_chunks(sizes, put_rpc_us_per_obj_.load(std::memory_order_relaxed));
  double rpc_us_total = 0;
  std::vector<Chunk> chunks(plan.size());
  std::vector<size_t> host_put;                      // objects whose placement is not on the GPU fabric
  std::map<size_t, std::vector<CopyPlacement>> host_placed;
  std::vector<bool> refused(keys.size(), false);     // blocks off the fabric (no host-staged path), or refused ids

  std::string reach_pool;
  bool reach_answer = false;
  auto start_chunk = [&](Chunk& ch) {
    const TimePoint t0 = Clock::now();
    BB_TRACE_SPAN("put.start_chunk", ch.end - ch.begin);
    std::vector<PutStartItem> items;
    items.reserve(ch.end - ch.begin);
    for (size_t i = ch.begin; i < ch.end; ++i) items.push_back(PutStartItem{keys[i], sizes[i], cfg});
    ch.placed = keystone_->batch_put_start(items);  // one control-plane round trip per chunk
    rpc_us_total += us_since(t0);
    metrics_.observe("phase_put_start_us", us_since(t0));
    // One descriptor per (object, shard): copy 0's placement plus the same shard of every other
    // copy as extra destinations, so the kernel reads the source once and fans out.
    for (size_t i = ch.begin; i < ch.end; ++i) {
      const auto& pr = ch.placed[i - ch.begin];
      if (!pr.ok()) {
        out[i] = pr.error();
        continue;
      }
      out[i] = ErrorCode::OK;
      const auto& copies = pr.value();
      if (copies.empty()) continue;
      // placements on host tiers (DRAM / CXL / NVMe) and unaligned caller buffers: stage through host memory and use the
      // data servers
      const DeviceLayout m = mem_of(i);
      const auto src = reinterpret_cast<uintptr_t>(dev_ptrs[i]);
      bool on_fabric = fabric_aligned(copies, [&](uint64_t off, uint64_t len) {
        uint64_t at = 0;
        return m.rebase(off, &at).coaligned(src + at, len);
      });
      for (const auto& c : copies)
        for (const auto& sh : c.shards) {
          // a batch lands on a handful of pools: ask the transport once per run of shards on the same pool
          if (reach_pool.empty() || reach_pool != sh.pool_id || !reach_answer) {
            reach_answer = device_->can_reach(sh);
            reach_pool = sh.pool_id;
          }
          on_fabric &= reach_answer;
        }
      if (!on_fabric && m.kind() == DeviceLayout::BLOCKS) {  // the host cannot read the ids without a sync
        out[i] = ErrorCode::NOT_IMPLEMENTED;
        refused[i] = true;
        continue;
      }
      if (!on_fabric) {
        host_put.push_back(i);
        host_placed[i] = copies;
        continue;
      }
      // copies striped differently cannot share a descriptor: then every shard of every copy is an op of its own
      bool same_layout = true;
      for (const auto& c : copies) same_layout &= c.shards.size() == copies[0].shards.size();
      for (size_t c = 0; c < (same_layout ? 1 : copies.size()); ++c) {
        uint64_t off = 0;
        for (size_t s = 0; s < copies[c].shards.size(); ++s) {
          DeviceShardOp op;
          op.item = i;
          op.copy = c;
          op.shard = s;
          op.placement = &copies[c].shards[s];
          op.mem = m.rebase(off, &op.mem_at);
          for (size_t r = 1; same_layout && r < copies.size(); ++r) op.replicas.push_back(&copies[r].shards[s]);
          ch.ops.push_back(std::move(op));
          off += copies[c].shards[s].length;
        }
      }
    }
    const TimePoint t1 = Clock::now();
    auto t = device_->submit_put(ch.ops, dev_ptrs, cfg.checksum, stream);
    metrics_.observe("phase_put_submit_us", us_since(t1));
    if (t.ok()) {
      ch.ticket = t.value();
      ch.submitted = true;
    } else {
      ch.submit_error = t.error();
    }
  };

  auto finish_chunk = [&](Chunk& ch) {
    BB_TRACE_SPAN("finish_chunk", ch.end - ch.begin);
    DeviceBatchResult res;
    ErrorCode ec = ch.submit_error;
    const TimePoint t1 = Clock::now();
    if (ch.submitted) ec = device_->wait(ch.ticket, &res);
    for (size_t k = 0; ec == ErrorCode::OK && k < ch.ops.size(); ++k)  // refused ids: the item's answer, and no digest
      if (res.verdicts[k] != ErrorCode::OK && !refused[ch.ops[k].item]) out[ch.ops[k].item] = res.verdicts[k], refused[ch.ops[k].item] = true;
    metrics_.observe("phase_put_wait_us", us_since(t1));
    const TimePoint t2 = Clock::now();
    std::vector<ObjectKey> done_keys, cancel_keys;
    std::vector<ShardChecksums> done_sums;
    std::vector<size_t> done_idx;
    if (ec != ErrorCode::OK) {
      for (size_t i = ch.begin; i < ch.end; ++i)
        if (ch.placed[i - ch.begin].ok()) {
          if (!refused[i]) out[i] = ec;
          cancel_keys.push_back(keys[i]);
        }
    } else {
      for (size_t i = ch.begin; i < ch.end; ++i)
        if (refused[i]) cancel_keys.push_back(keys[i]);
      std::vector<ShardChecksums> sums(ch.end - ch.begin);
      for (size_t i = ch.begin; i < ch.end; ++i) {
        const auto& pr = ch.placed[i - ch.begin];
        if (!pr.ok()) continue;
        auto& sm = sums[i - ch.begin];
        sm.resize(pr.value().size());
        for (size_t c = 0; c < sm.size(); ++c) sm[c].assign(pr.value()[c].shards.size(), 0);
      }
      for (size_t k = 0; k < ch.ops.size(); ++k) {
        const auto& op = ch.ops[k];
        auto& sm = sums[op.item - ch.begin];
        sm[op.copy][op.shard] = res.digests[k];
        for (size_t r = 0; r < op.replicas.size(); ++r) sm[r + 1][op.shard] = res.digests[k];
      }
      for (size_t i = ch.begin; i < ch.end; ++i)
        if (ch.placed[i - ch.begin].ok() && !host_placed.count(i) && !refused[i]) {
          done_keys.push_back(keys[i]);
          done_sums.push_back(std::move(sums[i - ch.begin]));
          done_idx.push_back(i);
        }
    }
    if (!cancel_keys.empty()) keystone_->batch_put_cancel(cancel_keys);
    if (!done_keys.empty()) {
      auto ecs = keystone_->batch_put_complete(done_keys, done_sums);
      for (size_t k = 0; k < done_idx.size(); ++k) out[done_idx[k]] = ecs[k];
    }
    rpc_us_total += us_since(t2);
    metrics_.observe("phase_put_complete_us", us_since(t2));
  };

  const size_t depth = std::max<size_t>(1, std::min<size_t>(2, device_->max_in_flight()));
  size_t finished = 0;
  for (size_t c = 0; c < chunks.size(); ++c) {
    while (c - finished >= depth) finish_chunk(chunks[finished++]);  // at most `depth` chunks in flight
    chunks[c].begin = plan[c].first;
    chunks[c].end = plan[c].second;
    start_chunk(chunks[c]);
  }
  while (finished < chunks.size()) finish_chunk(chunks[finished++]);
  // host-tier placements: D2H into a staging buffer, then the TCP data path (checksums on the CPU)
  for (size_t i : host_put) {
    std::vector<uint8_t> stage(sizes[i]);
    ErrorCode ec = device_->copy_from_device(stage.data(), dev_ptrs[i], mem_of(i), sizes[i], stream);
    ShardChecksums sums;
    if (ec == ErrorCode::OK) ec = transfer_put(host_placed[i], stage.data(), cfg.checksum, &sums);
    if (ec == ErrorCode::OK) ec = keystone_->put_complete(keys[i], sums);
    else keystone_->put_cancel(keys[i]);
    out[i] = ec;
    metrics_.inc("device_put_host_staged_total");
  }
  if (!keys.empty()) ewma_update(put_rpc_us_per_obj_, rpc_us_total / static_cast<double>(keys.size()));
  metrics_.inc("device_put_batches_total");
  metrics_.observe("device_put_batch_latency_us", us_since(t_all));
  return out;
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                         const std::vector<size_t>& capacity, void* stream,
                                                         std::vector<size_t>* out_sizes) {
  return get_device(keys, dev_ptrs, capacity, nullptr, nullptr, stream, out_sizes);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                                 const std::vector<uint64_t>& widths, const std::vector<uint64_t>& pitches,
                                                                 const std::vector<uint64_t>& rows, void* stream, std::vector<size_t>* out_sizes) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_scatter", keys, dev_ptrs, dev_ptrs.size() == n && widths.size() == n && pitches.size() == n && rows.size() == n,
      std::nullopt, [&](size_t i, ShapedItem* it) { return rows_item(widths[i], pitches[i], rows[i], it); }, stream, out_sizes);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_paged(const std::vector<ObjectKey>& keys, const std::vector<std::vector<uint64_t>>& pages,
                                                               const std::vector<uint64_t>& page_bytes, void* stream, std::vector<size_t>* out_sizes,
                                                               const std::vector<PageRows>& page_rows) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_paged", keys, std::vector<void*>(n), pages.size() == n && page_bytes.size() == n && (page_rows.empty() || page_rows.size() == n), std::nullopt,
      [&](size_t i, ShapedItem* it) { return pages_item(pages[i], page_bytes[i], page_rows, i, it); }, stream, out_sizes);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_segments(const std::vector<ObjectKey>& keys,
                                                                  const std::vector<std::vector<SourceSegments::Segment>>& segments, void* stream,
                                                                  std::vector<size_t>* out_sizes) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_segments", keys, std::vector<void*>(n), segments.size() == n, std::nullopt,
      [&](size_t i, ShapedItem* it) { return segments_item(segments[i], 1, it); }, stream, out_sizes);
}

std::vector<ErrorCode> BlackbirdClient::batch_put_device_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks,
                                                                const WorkerConfig& cfg, void* stream) {
  const size_t n = keys.size();
  return shaped_put(
      "device_put_blocks", keys, std::vector<const void*>(n), blocks.size() == n, std::nullopt,
      [&](size_t i, ShapedItem* it) { return blocks_item(blocks[i], it); }, cfg, stream);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_blocks(const std::vector<ObjectKey>& keys, const std::vector<SourceBlocks>& blocks,
                                                                void* stream, std::vector<size_t>* out_sizes) {
  const size_t n = keys.size();
  return shaped_get(
      "device_get_blocks", keys, std::vector<void*>(n), blocks.size() == n, std::nullopt,
      [&](size_t i, ShapedItem* it) { return blocks_item(blocks[i], it); }, stream, out_sizes);
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_range(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                               const std::vector<uint64_t>& offsets, const std::vector<uint64_t>& lengths,
                                                               void* stream) {
  const size_t n = keys.size();
  std::vector<ByteRange> ranges(n);
  std::vector<size_t> lens(n);
  return shaped_batch(
      "device_get_range", false, n, offsets.size() == n && lengths.size() == n,
      [&](size_t i, uint64_t* bytes) {
        ranges[i] = {offsets[i], lengths[i]};
        lens[i] = static_cast<size_t>(lengths[i]);
        *bytes = lengths[i];
        return ErrorCode::OK;
      },
      [&](const std::vector<size_t>&) { return get_device(keys, dev_ptrs, lens, &ranges, nullptr, stream, nullptr); });
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_strided(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                                 const std::vector<uint64_t>& offsets, const std::vector<uint64_t>& widths,
                                                                 const std::vector<uint64_t>& pitches, const std::vector<uint64_t>& rows,
                                                                 void* stream) {
  const size_t n = keys.size();
  std::vector<ByteRange> ranges(n);
  std::vector<size_t> lens(n);
  return shaped_batch(
      "device_get_strided", false, n, offsets.size() == n && widths.size() == n && pitches.size() == n && rows.size() == n,
      [&](size_t i, uint64_t* bytes) {
        ranges[i] = {offsets[i], widths[i], pitches[i], rows[i]};
        uint64_t total = 0;
        lens[i] = __builtin_mul_overflow(rows[i], widths[i], &total) ? SIZE_MAX : static_cast<size_t>(total);
        *bytes = lens[i];
        return ErrorCode::OK;
      },
      [&](const std::vector<size_t>&) { return get_device(keys, dev_ptrs, lens, &ranges, nullptr, stream, nullptr); });
}

std::vector<ErrorCode> BlackbirdClient::batch_get_device_strided_scatter(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                                         const std::vector<uint64_t>& offsets, const std::vector<uint64_t>& widths,
                                                                         const std::vector<uint64_t>& pitches, const std::vector<uint64_t>& rows,
                                                                         const std::vector<uint64_t>& dst_widths,
                                                                         const std::vector<uint64_t>& dst_pitches, void* stream) {
  const size_t n = keys.size();
  std::vector<ByteRange> ranges(n);
  std::vector<DeviceLayout> mem(n);
  std::vector<size_t> lens(n);
  return shaped_batch(
      "device_get_strided_scatter", false, n,
      dev_ptrs.size() == n && offsets.size() == n && widths.size() == n && pitches.size() == n && rows.size() == n &&
          dst_widths.size() == n && dst_pitches.size() == n,
      [&](size_t i, uint64_t* bytes) {
        ranges[i] = {offsets[i], widths[i], pitches[i], rows[i]};
        uint64_t total = 0;
        if (__builtin_mul_overflow(rows[i], widths[i], &total) || total > SIZE_MAX) return ErrorCode::VALUE_OUT_OF_RANGE;
        lens[i] = static_cast<size_t>(total);
        *bytes = total;
        return result_rows(total, dst_widths[i], dst_pitches[i], &mem[i]);
      },
      [&](const std::vector<size_t>& idx) {
        const auto rr = pick(ranges, idx);
        const auto rm = pick(mem, idx);
        return get_device(pick(keys, idx), pick(dev_ptrs, idx), pick(lens, idx), &rr, &rm, stream, nullptr);
      });
}

std::vector<ErrorCode> BlackbirdClient::get_device(const std::vector<ObjectKey>& keys, const std::vector<void*>& dev_ptrs,
                                                   const std::vector<size_t>& capacity, const std::vector<ByteRange>* ranges,
                                                   const std::vector<DeviceLayout>* mem, void* stream, std::vector<size_t>* out_sizes) {
  std::vector<ErrorCode> out(keys.size(), ErrorCode::INVALID_PARAMETERS);
  if (!keystone_) return std::vector<ErrorCode>(keys.size(), ErrorCode::CLIENT_DISCONNECTED);
  if (!device_) return std::vector<ErrorCode>(keys.size(), ErrorCode::NOT_IMPLEMENTED);
  if (dev_ptrs.size() != keys.size() || capacity.size() != keys.size() || (ranges && ranges->size() != keys.size()) ||
      (mem && mem->size() != keys.size()))
    return out;
  auto mem_of = [&](size_t i) { return mem ? (*mem)[i] : DeviceLayout{}; };
  const TimePoint t_all = Clock::now();
  BB_TRACE_SPAN("batch_get_device", keys.size());
  if (out_sizes) out_sizes->assign(keys.size(), 0);
  std::vector<Result<std::vector<CopyPlacement>>> placed(keys.size(), Result<std::vector<CopyPlacement>>(ErrorCode::INTERNAL_ERROR));
  std::vector<size_t> copy_choice(keys.size(), 0);
  std::vector<bool> pending(keys.size(), false);
  // The object bytes each get stores (every shard of a whole-object get is read, zero-length ones included), and the base
  // they land relative to: the caller's pointer, less the window's offset for a range get (the virtual base; the fabric
  // never touches an address outside the range).
  std::vector<StoreWindow> span(keys.size());
  std::vector<void*> range_bases;
  if (ranges) range_bases.resize(keys.size());
  const std::vector<void*>& bases = ranges ? range_bases : dev_ptrs;

  auto build_ops = [&](size_t begin, size_t end, std::vector<DeviceShardOp>& ops) {
    for (size_t i = begin; i < end; ++i) {
      if (!pending[i]) continue;
      const auto& copies = placed[i].value();
      const auto& copy = copies[copy_choice[i] % copies.size()];
      const StoreWindow& sp = span[i];
      const bool whole = sp.whole();
      uint64_t off = 0;
      for (size_t s = 0; s < copy.shards.size(); ++s) {
        const uint64_t len = copy.shards[s].length;
        if (whole || sp.touches(off, len)) {
          DeviceShardOp op;
          op.item = i;
          op.copy = copy_choice[i] % copies.size();
          op.shard = s;
          op.placement = &copy.shards[s];
          const DeviceLayout m = mem_of(i);
          if (!whole) op.win = sp.rebase(off, len);
          if (m.kind() == DeviceLayout::WINDOW_ROWS)  // the rows move on with the shard's first stored unit
            op.mem = DeviceLayout::window_rows(WindowRows{sp, m.rows()}.rebase(off, len, &op.mem_at).rows);
          else
            op.mem = m.rebase(off, &op.mem_at);
          ops.push_back(std::move(op));
        }
        off += len;
      }
    }
  };
  // A verdict on an item's block ids answers it, ahead of its digests: its ids, not its copy, are wrong.
  auto apply_status = [&](const std::vector<DeviceShardOp>& ops, const DeviceBatchResult& res, std::vector<size_t>* retry) {
    std::vector<bool> bad(keys.size(), false), seen(keys.size(), false);
    for (size_t k = 0; k < ops.size(); ++k) {
      seen[ops[k].item] = true;
      if (res.status[k] != 0) bad[ops[k].item] = true;
      if (res.verdicts[k] != ErrorCode::OK && pending[ops[k].item]) {
        out[ops[k].item] = res.verdicts[k];
        pending[ops[k].item] = false;
      }
    }
    for (size_t i = 0; i < keys.size(); ++i) {
      if (!seen[i] || !pending[i]) continue;
      if (!bad[i]) {
        out[i] = ErrorCode::OK;
        pending[i] = false;
      } else {
        metrics_.inc("checksum_mismatch_total");
        ++copy_choice[i];  // fail over to the next replica
        if (retry) retry->push_back(i);
      }
    }
  };

  // ---- first attempt: chunks pipelined against the get_workers round trips
  struct Chunk {
    size_t begin = 0, end = 0;
    std::vector<DeviceShardOp> ops;
    uint64_t ticket = 0;
    bool submitted = false;
    ErrorCode err = ErrorCode::OK;
  };
  const auto plan = plan_chunks(capacity, get_rpc_us_per_obj_.load(std::memory_order_relaxed));
  double rpc_us_total = 0;
  std::vector<Chunk> chunks(plan.size());
  std::vector<size_t> retry;
  // A batch mostly reads from a handful of pools: remember the transport's answer for the last pool asked about instead of
  // taking its lock and looking the pool id up once per shard, and count per-object events locally (a named counter is a
  // map lookup under a mutex).
  const std::string* local_pool = nullptr;
  bool local_answer = false;
  auto pool_is_local = [&](const ShardPlacement& sh) {
    if (!local_pool || *local_pool != sh.pool_id) {
      local_answer = device_->is_local(sh);
      local_pool = &sh.pool_id;
    }
    return local_answer;
  };
  std::string reach_pool;
  bool reach_answer = false;
  auto pool_reachable = [&](const ShardPlacement& sh) {
    if (reach_pool.empty() || reach_pool != sh.pool_id || !reach_answer) {
      reach_answer = device_->can_reach(sh);
      reach_pool = sh.pool_id;
    }
    return reach_answer;
  };
  uint64_t n_local = 0, n_dram_direct = 0;
  auto start_chunk = [&](Chunk& ch) {
    const TimePoint t0 = Clock::now();
    local_pool = nullptr;  // the cached pointer refers into the previous chunk's placements
    const bool whole = ch.begin == 0 && ch.end == keys.size();
    std::vector<ObjectKey> part;
    if (!whole) part.assign(keys.begin() + static_cast<std::ptrdiff_t>(ch.begin), keys.begin() + static_cast<std::ptrdiff_t>(ch.end));
    const std::vector<ObjectKey>& ck = whole ? keys : part;
    auto res = keystone_->batch_get_workers(ck);
    rpc_us_total += us_since(t0);
    metrics_.observe("phase_get_workers_us", us_since(t0));
    for (size_t i = ch.begin; i < ch.end; ++i) {
      placed[i] = std::move(res[i - ch.begin]);
      if (!placed[i].ok()) {
        out[i] = placed[i].error();
        continue;
      }
      if (placed[i].value().empty()) {
        out[i] = ErrorCode::NO_COMPLETE_WORKER;
        continue;
      }
      size_t size = 0;
      for (const auto& s : placed[i].value()[0].shards) size += s.length;
      if (out_sizes) (*out_sizes)[i] = size;
      StoreWindow& sp = span[i];
      if (ranges) {
        const ByteRange& r = (*ranges)[i];
        const ErrorCode ec = StoreWindow::from_rows(r.offset, r.length, r.pitch, r.rows, size, &sp);
        if (ec != ErrorCode::OK || sp.empty()) {  // an error, or nothing to read or store
          out[i] = ec;
          continue;
        }
        // rows of the result (WINDOW_ROWS) start at the caller's pointer
        range_bases[i] = mem_of(i).kind() == DeviceLayout::WINDOW_ROWS
                             ? dev_ptrs[i]
                             : reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(dev_ptrs[i]) - sp.base_shift(sp.lo));
      } else if (size > capacity[i]) {
        out[i] = ErrorCode::BUFFER_OVERFLOW;
        continue;
      }
      // replica choice: one that lives on this client's own GPU (HBM speed, no NVLink), else a replica that is
      // fully reachable over the GPU fabric (readers spread over the replicas), else stage through the host.  Only the
      // shards a get reads count: a range get ignores the shards outside its range.
      const auto& copies = placed[i].value();
      auto for_read_shards = [&](const CopyPlacement& c, auto&& f) {  // returns how many shards the get reads
        size_t n = 0;
        uint64_t off = 0;
        for (const auto& sh : c.shards) {
          if (sp.touches(off, sh.length)) f(sh), ++n;
          off += sh.length;
        }
        return n;
      };
      // (the spread over replicas only matters when there is more than one; thousands of single-copy objects skip the hash)
      const size_t start = copies.size() > 1 ? std::hash<std::string>{}(opts_.node_id + keys[i]) % copies.size() : 0;
      // an unaligned caller buffer is staged through the host whatever the replicas (see fabric_aligned)
      const auto dst = reinterpret_cast<uintptr_t>(dev_ptrs[i]);
      const DeviceLayout m = mem_of(i);
      const bool aligned = fabric_aligned(copies, [&](uint64_t off, uint64_t len) { return m.fused_get_aligned(dst, off, len, sp); });
      bool found = false;
      for (size_t k = 0; aligned && k < copies.size() && !found; ++k) {
        bool local = true;
        local = for_read_shards(copies[k], [&](const ShardPlacement& sh) { local &= pool_is_local(sh); }) > 0 && local;
        if (local) {
          copy_choice[i] = k;
          found = true;
          ++n_local;
        }
      }
      // HBM replicas first (NVLink), then replicas in mapped DRAM pools (PCIe)
      for (int pass = 0; aligned && pass < 2 && !found; ++pass) {
        for (size_t k = 0; k < copies.size() && !found; ++k) {
          bool ok = true;
          ok = for_read_shards(copies[(start + k) % copies.size()], [&](const ShardPlacement& sh) {
                 ok = ok && (pass == 1 || sh.storage_class == StorageClass::RAM_GPU) && pool_reachable(sh);
               }) > 0 && ok;
          if (ok) {
            copy_choice[i] = (start + k) % copies.size();
            found = true;
            if (pass == 1) ++n_dram_direct;
          }
        }
      }
      if (!found && m.kind() == DeviceLayout::BLOCKS) {  // no host-staged path: the host cannot read the ids without a sync
        out[i] = ErrorCode::NOT_IMPLEMENTED;
        continue;
      }
      if (!found) {
        std::vector<uint8_t> stage(size);
        // data servers + CPU checksum + replica fail-over, over the shards the get reads
        ErrorCode ec = transfer_get(copies, stage.data(), size, sp);
        // compact the rows on the host: one H2D copy of rows * width bytes, into the result's rows for WINDOW_ROWS
        if (ec == ErrorCode::OK && sp.strided()) {
          std::vector<uint8_t> dense(capacity[i]);
          sp.for_each_run(size, [&](uint64_t x, uint64_t at, uint64_t n) { std::memcpy(dense.data() + at, stage.data() + x, n); });
          ec = device_->copy_to_device(dev_ptrs[i], m.kind() == DeviceLayout::WINDOW_ROWS ? m.as_rows() : DeviceLayout{}, dense.data(),
                                       dense.size(), stream);
        } else if (ec == ErrorCode::OK) {  // the range, or the whole object into its layout
          ec = device_->copy_to_device(dev_ptrs[i], m.as_rows(), stage.data() + sp.lo, std::min<uint64_t>(sp.hi, size) - sp.lo, stream);
        }
        out[i] = ec;
        metrics_.inc("device_get_host_staged_total");
        continue;
      }
      pending[i] = true;
    }
    build_ops(ch.begin, ch.end, ch.ops);
    if (ch.ops.empty()) return;
    const TimePoint t1 = Clock::now();
    auto t = device_->submit_get(ch.ops, bases, stream);
    metrics_.observe("phase_get_submit_us", us_since(t1));
    if (t.ok()) {
      ch.ticket = t.value();
      ch.submitted = true;
    } else {
      ch.err = t.error();
    }
  };
  auto finish_chunk = [&](Chunk& ch) {
    BB_TRACE_SPAN("finish_chunk", ch.end - ch.begin);
    if (ch.ops.empty()) return;
    DeviceBatchResult res;
    ErrorCode ec = ch.err;
    const TimePoint t1 = Clock::now();
    if (ch.submitted) ec = device_->wait(ch.ticket, &res);
    metrics_.observe("phase_get_wait_us", us_since(t1));
    if (ec != ErrorCode::OK) {
      for (size_t i = ch.begin; i < ch.end; ++i)
        if (pending[i]) {
          out[i] = ec;
          pending[i] = false;
        }
      return;
    }
    apply_status(ch.ops, res, &retry);
  };
  const size_t depth = std::max<size_t>(1, std::min<size_t>(2, device_->max_in_flight()));
  size_t finished = 0;
  for (size_t c = 0; c < chunks.size(); ++c) {
    while (c - finished >= depth) finish_chunk(chunks[finished++]);  // at most `depth` chunks in flight
    chunks[c].begin = plan[c].first;
    chunks[c].end = plan[c].second;
    start_chunk(chunks[c]);
  }
  while (finished < chunks.size()) finish_chunk(chunks[finished++]);

  // ---- replica fail-over for objects whose digest did not verify
  for (size_t attempt = 1; attempt < 4 && !retry.empty(); ++attempt) {
    std::vector<size_t> still;
    std::vector<DeviceShardOp> ops;
    for (size_t i : retry) {
      if (attempt >= placed[i].value().size()) {
        out[i] = ErrorCode::CHECKSUM_MISMATCH;
        pending[i] = false;
      }
    }
    build_ops(0, keys.size(), ops);
    if (ops.empty()) break;
    metrics_.inc("replica_failover_total");
    DeviceBatchResult res;
    auto t = device_->submit_get(ops, bases, stream);
    ErrorCode ec = t.ok() ? device_->wait(t.value(), &res) : t.error();
    if (ec != ErrorCode::OK) {
      for (size_t i = 0; i < keys.size(); ++i)
        if (pending[i]) {
          out[i] = ec;
          pending[i] = false;
        }
      break;
    }
    apply_status(ops, res, &still);
    retry.swap(still);
  }
  for (size_t i = 0; i < keys.size(); ++i)
    if (pending[i]) out[i] = ErrorCode::CHECKSUM_MISMATCH;
  if (n_local) metrics_.inc("device_get_local_replica_total", n_local);
  if (n_dram_direct) metrics_.inc("device_get_dram_direct_total", n_dram_direct);
  refresh_placements(keys, placed, out, [&](const std::vector<size_t>& r) {
    const auto rranges = ranges ? pick(*ranges, r) : std::vector<ByteRange>();
    const auto rmem = mem ? pick(*mem, r) : std::vector<DeviceLayout>();
    std::vector<size_t> rsizes;
    auto recs = get_device(pick(keys, r), pick(dev_ptrs, r), pick(capacity, r), ranges ? &rranges : nullptr, mem ? &rmem : nullptr,
                           stream, &rsizes);
    for (size_t k = 0; out_sizes && k < r.size() && k < rsizes.size(); ++k) (*out_sizes)[r[k]] = rsizes[k];
    return recs;
  });
  if (!keys.empty()) ewma_update(get_rpc_us_per_obj_, rpc_us_total / static_cast<double>(keys.size()));
  metrics_.inc("device_get_batches_total");
  metrics_.observe("device_get_batch_latency_us", us_since(t_all));
  return out;
}

// ================================================================ HostLoopbackTransport (CPU stand-in for the GPU fabric)
bool HostLoopbackTransport::can_reach(const ShardPlacement& s) const {
  if (s.storage_class == StorageClass::RAM_GPU) return false;
  return reach_disk_ || !is_disk_class(s.storage_class);
}

Result<uint64_t> HostLoopbackTransport::submit_put(const std::vector<DeviceShardOp>& ops, const std::vector<const void*>& dev_ptrs,
                                                   ChecksumAlgo algo, void*) {
  ++launches_;  // one "launch" per batch, like the fused kernel
  std::vector<uint64_t> digests(ops.size(), 0);
  std::vector<ErrorCode> verdicts(ops.size(), ErrorCode::OK);
  for (size_t k = 0; k < ops.size(); ++k) {
    const DeviceShardOp& op = ops[k];
    const auto* src = static_cast<const uint8_t*>(op.src(dev_ptrs[op.item]));
    std::vector<uint8_t> dense;
    if (!op.mem.contiguous()) {  // as the kernel's gathering load: the shard's bytes, compacted from its rows or pages
      if (!op.mem.valid_source(op.placement->length)) return ErrorCode::INVALID_ARGUMENT;
      if (op.mem.kind() == DeviceLayout::BLOCKS && !op.mem.coaligned(0, op.placement->length)) return ErrorCode::INVALID_ADDRESS;
      std::vector<uint64_t> table;  // blocks: as the resolve kernel, a refused table reads block 0 of every slice
      const DeviceLayout m = op.mem.resolved(op.placement->length, false, &table, &verdicts[k]);
      dense.resize(op.placement->length);
      copy_from_device(dense.data(), src, m, dense.size(), nullptr);
      src = dense.data();
    }
    ErrorCode ec = io_->write_shard(*op.placement, src, &digests[k], algo);
    for (size_t r = 0; r < op.replicas.size() && ec == ErrorCode::OK; ++r) ec = io_->write_shard(*op.replicas[r], src, nullptr, ChecksumAlgo::NONE);
    if (ec != ErrorCode::OK) return ec;
  }
  std::lock_guard<std::mutex> lk(done_mu_);
  done_[next_ticket_] = {std::move(digests), std::vector<uint32_t>(ops.size(), 0), std::move(verdicts)};
  return next_ticket_++;
}

Result<uint64_t> HostLoopbackTransport::submit_get(const std::vector<DeviceShardOp>& ops, const std::vector<void*>& dev_ptrs, void*) {
  ++launches_;
  std::vector<uint32_t> status(ops.size(), 0);
  std::vector<ErrorCode> verdicts(ops.size(), ErrorCode::OK);
  for (size_t k = 0; k < ops.size(); ++k) {
    const DeviceShardOp& op = ops[k];
    ErrorCode ec;
    auto* dst = static_cast<uint8_t*>(op.dst(dev_ptrs[op.item]));
    const uint64_t len = op.placement->length;
    if (op.mem.kind() == DeviceLayout::WINDOW_ROWS && !op.win.covers(len)) {
      // as the kernel's windowed scattering store: the whole shard read and verified, the window's units stored into the
      // rows of its result
      const WindowRows wr{op.win, op.mem.rows()};
      if (!wr.valid(len)) return ErrorCode::INVALID_ARGUMENT;
      std::vector<uint8_t> whole(len);
      ec = io_->read_shard(*op.placement, whole.data(), op.placement->checksum_algo);
      if (ec == ErrorCode::OK) wr.for_each_run(len, [&](uint64_t x, uint64_t at, uint64_t n) { std::memcpy(dst + at, whole.data() + x, n); });
    } else if (!op.mem.contiguous()) {  // as the kernel's scattering store: the whole shard, read and verified, stored into its rows or pages
      if (!op.mem.valid(op.placement->length) || (!op.win.whole() && op.mem.kind() != DeviceLayout::WINDOW_ROWS)) return ErrorCode::INVALID_ARGUMENT;
      if (op.mem.kind() == DeviceLayout::BLOCKS && !op.mem.blocks().distinct_checkable()) return ErrorCode::NOT_IMPLEMENTED;  // as the engine
      if (op.mem.kind() == DeviceLayout::BLOCKS && !op.mem.coaligned(0, op.placement->length)) return ErrorCode::INVALID_ADDRESS;
      std::vector<uint64_t> table;  // blocks: as the resolve kernel, a refused table is all null pages
      const DeviceLayout m = op.mem.as_rows().resolved(op.placement->length, true, &table, &verdicts[k]);
      std::vector<uint8_t> whole(op.placement->length);
      ec = io_->read_shard(*op.placement, whole.data(), op.placement->checksum_algo);
      if (ec == ErrorCode::OK) copy_to_device(dst, m, whole.data(), whole.size(), nullptr);
    } else if (op.win.covers(op.placement->length)) {
      ec = io_->read_shard(*op.placement, dst, op.placement->checksum_algo);
    } else {  // as the kernel does: read and verify the whole shard, store only the window (only it is real memory)
      std::vector<uint8_t> whole(op.placement->length);
      ec = io_->read_shard(*op.placement, whole.data(), op.placement->checksum_algo);
      if (ec == ErrorCode::OK)
        op.win.for_each_run(whole.size(), [&](uint64_t x, uint64_t at, uint64_t n) { std::memcpy(dst + at, whole.data() + x, n); });
    }
    if (ec == ErrorCode::CHECKSUM_MISMATCH) {
      status[k] = 1;  // reported per shard, like the kernel's verify flag
    } else if (ec != ErrorCode::OK) {
      return ec;
    }
  }
  std::lock_guard<std::mutex> lk(done_mu_);
  done_[next_ticket_] = {std::vector<uint64_t>(ops.size(), 0), std::move(status), std::move(verdicts)};
  return next_ticket_++;
}

ErrorCode HostLoopbackTransport::wait(uint64_t ticket, DeviceBatchResult* res) {
  std::lock_guard<std::mutex> lk(done_mu_);
  auto it = done_.find(ticket);
  if (it == done_.end()) return ErrorCode::NOT_FOUND;
  *res = std::move(it->second);
  done_.erase(it);
  return ErrorCode::OK;
}

ErrorCode HostLoopbackTransport::run_fp8(const std::vector<DeviceFp8Op>& ops, bool unpack, void*, DeviceBatchResult* res) {
  ++launches_;
  *res = {std::vector<uint64_t>(ops.size(), 0), std::vector<uint32_t>(ops.size(), 0), std::vector<ErrorCode>(ops.size(), ErrorCode::OK)};
  for (size_t k = 0; k < ops.size(); ++k) {
    const DeviceFp8Op& op = ops[k];
    const uint64_t eb = mxfp8::wide_bytes(op.wide_type);
    if (eb != mxfp8::wide_bytes(ops[0].wide_type)) return ErrorCode::INVALID_ARGUMENT;  // as the engine: one element size
    if (!unpack) {
      const auto* src = static_cast<const uint8_t*>(op.wide);
      std::vector<uint8_t> dense;
      if (!op.mem.contiguous()) {  // as the engine and the kernel's gathering load: the elements, compacted from their rows or pages
        DeviceLayout b;
        if (!op.win.whole() || !op.mem.valid_source(op.n_elems) || !op.mem.to_wide_bytes(eb, &b)) return ErrorCode::INVALID_ARGUMENT;
        if (!b.coaligned(reinterpret_cast<uintptr_t>(op.wide), eb * op.n_elems)) return ErrorCode::INVALID_ADDRESS;
        std::vector<uint64_t> table;  // blocks: as the resolve kernel, a refused table reads block 0 of every slice
        b = b.resolved(eb * op.n_elems, false, &table, &res->verdicts[k]);
        dense.resize(eb * op.n_elems);
        copy_from_device(dense.data(), op.wide, b, dense.size(), nullptr);
        src = dense.data();
      }
      std::vector<uint8_t> packed(mxfp8::packed_bytes(op.n_elems));
      mxfp8::pack(src, op.wide_type, op.n_elems, packed.data());
      ErrorCode ec = io_->write_shard(*op.placement, packed.data(), &res->digests[k], ChecksumAlgo::BBH64);
      for (size_t r = 0; r < op.replicas.size() && ec == ErrorCode::OK; ++r) ec = io_->write_shard(*op.replicas[r], packed.data(), nullptr, ChecksumAlgo::NONE);
      if (ec != ErrorCode::OK) return ec;
      continue;
    }
    if (!op.win.over(op.n_elems).valid(op.n_elems)) return ErrorCode::INVALID_ARGUMENT;  // as the engine
    // as the engine: rows of the window's result (WindowRows), co-aligned in wide bytes, unless the window stores the
    // whole object in place, where they are the object's own rows
    const bool wrows = op.mem.kind() == DeviceLayout::WINDOW_ROWS && !op.win.covers(op.n_elems);
    const WindowRows wr{op.win.over(op.n_elems), op.mem.rows()};
    if (wrows) {
      WindowRows wb;
      if (!op.mem.rows().valid() || !wr.to_wide_bytes(eb, &wb)) return ErrorCode::INVALID_ARGUMENT;
      if (!wb.coaligned(reinterpret_cast<uintptr_t>(op.wide), eb * op.n_elems)) return ErrorCode::INVALID_ADDRESS;
    }
    const DeviceLayout lay = wrows ? DeviceLayout{} : op.mem.as_rows();
    DeviceLayout b;
    if (!lay.contiguous()) {  // as the engine: destination rows or pages, never with a window, co-aligned in wide bytes
      // with rows of a window's result, the window stores the whole object in place (wrows is false)
      if ((!op.win.whole() && op.mem.kind() != DeviceLayout::WINDOW_ROWS) || !lay.valid(op.n_elems) || !lay.to_wide_bytes(eb, &b))
        return ErrorCode::INVALID_ARGUMENT;
      if (!b.coaligned(reinterpret_cast<uintptr_t>(op.wide), eb * op.n_elems)) return ErrorCode::INVALID_ADDRESS;
      if (b.kind() == DeviceLayout::BLOCKS && !b.blocks().distinct_checkable()) return ErrorCode::NOT_IMPLEMENTED;  // as the engine
    }
    std::vector<uint64_t> table;  // blocks: as the resolve kernel, a refused table is all null pages
    b = b.resolved(eb * op.n_elems, true, &table, &res->verdicts[k]);
    std::vector<uint8_t> packed(mxfp8::packed_bytes(op.n_elems));
    const ErrorCode ec = io_->read_shard(*op.placement, packed.data(), ChecksumAlgo::BBH64);
    if (ec == ErrorCode::CHECKSUM_MISMATCH) {
      res->status[k] = 1;
      continue;
    }
    if (ec != ErrorCode::OK) return ec;
    auto* dst = static_cast<uint8_t*>(op.wide);
    if (op.win.whole() && lay.contiguous()) {
      mxfp8::unpack(packed.data(), op.n_elems, op.wide_type, dst);
      continue;
    }
    std::vector<uint8_t> wide(eb * op.n_elems);
    mxfp8::unpack(packed.data(), op.n_elems, op.wide_type, wide.data());
    if (!lay.contiguous()) {  // as the kernel's scattering store: the unpacked object into its rows or pages
      copy_to_device(dst, b, wide.data(), wide.size(), nullptr);
      continue;
    }
    if (wrows) {  // as the kernel's windowed scattering store: the window's elements into the rows of its result
      wr.for_each_run(op.n_elems, [&](uint64_t x, uint64_t at, uint64_t n) { std::memcpy(dst + eb * at, wide.data() + eb * x, eb * n); });
      continue;
    }
    // as the kernel does: the whole object read and verified, only the window stored
    op.win.for_each_run(op.n_elems, [&](uint64_t x, uint64_t at, uint64_t n) { std::memcpy(dst + eb * at, wide.data() + eb * x, eb * n); });
  }
  return ErrorCode::OK;
}

}  // namespace bb::client
