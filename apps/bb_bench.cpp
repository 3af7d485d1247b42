// bb-bench: native benchmark client (reference clients/benchmark_client.cpp: per-iteration put +
// get of `--size` bytes, avg latency and MiB/s; examples/benchmark_disk_backends.cpp: reserve /
// commit / free ops/s on a disk backend).
//   bb-bench client  --keystone host:port --size 1048576 --iterations 50 [--replicas 1] [--max-workers 1] [--batch 1]
//   bb-bench backend --class NVME --path /tmp/x --ops 50 --size 4096
//   bb-bench gpu --keystone host:port [--device 0] [--objects 64] [--size 67108864] [--iterations 20] [--node gpu1]
//              (device-resident batched put + get through the fused kernels: no Python, no torch)
//   bb-bench devclient [--batch 4096] [--size 4096] [--iterations 20]   (client-level cost of the device batch API, transfers free)
//   bb-bench control [--threads 4] [--batch 4096] [--iterations 20] [--pools 8] [--rpc]   (keystone metadata ops/s)
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <random>

#include "apps/cli_util.h"
#include "net/tcp.h"
#include "common/tenant.h"
#include <thread>

#include "client/blackbird_client.h"
#include "fabric/gpu_fabric.h"
#include "fabric/xfer_engine.h"
#include "keystone/keystone_service.h"
#include "rpc/rpc_service.h"
#include "worker/storage_backend.h"

using namespace bb;
using Clk = std::chrono::steady_clock;

namespace {
double ms(Clk::time_point a, Clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }
double pct(std::vector<double> v, double q) {
  if (v.empty()) return 0;
  std::sort(v.begin(), v.end());
  return v[std::min(v.size() - 1, static_cast<size_t>(q * static_cast<double>(v.size())))];
}
}  // namespace

int main(int argc, char** argv) {
  auto args = bbapp::parse_args(argc, argv);
  if (args.has("auth-token")) bb::net::set_cluster_token(args.get("auth-token"));  // else BB_AUTH_TOKEN / config
  if (args.has("encrypt-transport")) bb::net::set_transport_encryption(true);  // else BB_ENCRYPT_TRANSPORT / config
  if (args.has("auth-token-ro")) bb::net::set_cluster_token_ro(args.get("auth-token-ro"));  // else BB_AUTH_TOKEN_RO / config
  if (args.has("tenant")) bb::set_client_tenant(args.get("tenant"), args.get("tenant-secret"));  // else BB_TENANT / BB_TENANT_SECRET (common/tenant.h)
  const std::string mode = args.positional.empty() ? "client" : args.positional[0];
  if (args.has("help")) {
    std::printf("usage: bb-bench client|backend|control|devclient|gpu [options]\n");
    return 0;
  }
  if (mode == "backend") {
    auto sc = parse_storage_class(args.get("class", "NVME"));
    if (!sc) return 2;
    worker::BackendOptions o;
    o.mount_path = args.get("path", "/tmp/bb_bench_backend");
    auto b = worker::create_storage_backend(*sc, static_cast<uint64_t>(args.num("capacity", 100ll << 20)), o);
    if (!b || b->initialize() != ErrorCode::OK) {
      std::fprintf(stderr, "backend init failed\n");
      return 1;
    }
    const int ops = static_cast<int>(args.num("ops", 50));
    const uint64_t size = static_cast<uint64_t>(args.num("size", 4096));
    std::vector<uint8_t> buf(size, 0xA5);
    std::vector<double> t_res, t_wr, t_com, t_free;
    for (int i = 0; i < ops; ++i) {
      auto a = Clk::now();
      auto tok = b->reserve_shard(size);
      auto c = Clk::now();
      if (!tok.ok()) break;
      b->write(tok.value().remote_addr - b->get_base_address(), buf.data(), size);
      auto d = Clk::now();
      b->commit_shard(tok.value());
      auto e = Clk::now();
      b->free_shard(tok.value().remote_addr, size);
      auto f = Clk::now();
      t_res.push_back(ms(a, c));
      t_wr.push_back(ms(c, d));
      t_com.push_back(ms(d, e));
      t_free.push_back(ms(e, f));
    }
    auto avg = [](const std::vector<double>& v) { return v.empty() ? 0.0 : std::accumulate(v.begin(), v.end(), 0.0) / static_cast<double>(v.size()); };
    const size_t done = t_res.size();  // never divide by a zero iteration count (reference bug #15)
    std::printf("%s backend, %zu ops x %llu B: reserve %.4f ms | write %.4f ms | commit %.4f ms | free %.4f ms | %.0f lifecycle ops/s\n",
                args.get("class", "NVME").c_str(), done, static_cast<unsigned long long>(size), avg(t_res), avg(t_wr), avg(t_com), avg(t_free),
                done ? 1000.0 / (avg(t_res) + avg(t_wr) + avg(t_com) + avg(t_free)) : 0.0);
    return 0;
  }
  if (mode == "gpu") {
    // Native device-path benchmark: this process is a client with its own GPU; objects live in device memory and
    // move to the GPU-tier workers' slabs (bb-worker with a RAM_GPU pool, same box) through the fused kernels.
    auto khp = split_host_port(args.get("keystone", "127.0.0.1:9090"));
    if (!khp) return 2;
    const int device = static_cast<int>(args.num("device", 0));
    const size_t nobj = static_cast<size_t>(args.num("objects", 64));
    const size_t osz = static_cast<size_t>(args.num("size", 64ll << 20)) / 256 * 256;
    const int iters = std::max(1, static_cast<int>(args.num("iterations", 20)));
    int ndev = 0;
    gpu::device_count(&ndev);
    if (ndev <= device) {
      std::fprintf(stderr, "bb-bench gpu: CUDA device %d not present (%d devices)\n", device, ndev);
      return 3;
    }
    auto api = std::make_shared<rpc::KeystoneRpcClient>();
    if (api->connect(khp->first, static_cast<uint16_t>(khp->second), 10000) != ErrorCode::OK) {
      std::fprintf(stderr, "bb-bench gpu: cannot reach keystone %s\n", args.get("keystone", "127.0.0.1:9090").c_str());
      return 1;
    }
    client::BlackbirdClientOptions o;
    o.keystone_host = khp->first;
    o.keystone_port = static_cast<uint16_t>(khp->second);
    o.node_id = args.get("client-node", "bench-gpu" + std::to_string(device));
    client::BlackbirdClient cl(api, o);
    if (cl.connect() != ErrorCode::OK) return 1;
    auto fab = gpu::GpuFabric::create(device, api);
    if (!fab.ok()) {
      std::fprintf(stderr, "bb-bench gpu: fabric init failed: %s\n", std::string(to_string(fab.error())).c_str());
      return 1;
    }
    cl.set_device_transport(fab.value());
    void *src = nullptr, *dst = nullptr;
    if (gpu::device_malloc(device, nobj * osz, &src) != ErrorCode::OK || gpu::device_malloc(device, nobj * osz, &dst) != ErrorCode::OK) return 1;
    gpu::launch_random_fill(src, nobj * osz, 0xB200, nullptr);
    gpu::device_synchronize(device);
    WorkerConfig cfg;
    cfg.replication_factor = static_cast<size_t>(args.num("replicas", 1));
    cfg.max_workers_per_copy = static_cast<size_t>(args.num("max-workers", 1));
    cfg.ttl_ms = 0;
    cfg.preferred_classes = {StorageClass::RAM_GPU};
    cfg.preferred_node = args.get("node", "");
    if (args.get("checksum") == "crc32c") cfg.checksum = ChecksumAlgo::CRC32C;
    if (args.get("checksum") == "xxh3") cfg.checksum = ChecksumAlgo::XXH3;
    if (args.get("checksum") == "none") cfg.checksum = ChecksumAlgo::NONE;
    std::vector<const void*> sp;
    std::vector<void*> dp;
    std::vector<size_t> sizes(nobj, osz);
    for (size_t i = 0; i < nobj; ++i) {
      sp.push_back(static_cast<uint8_t*>(src) + i * osz);
      dp.push_back(static_cast<uint8_t*>(dst) + i * osz);
    }
    std::vector<double> put_ms, get_ms;
    int failures = 0;
    const double dev0 = fab.value()->total_device_ms();
    for (int it = -2; it < iters; ++it) {  // two warm-up rounds
      std::vector<ObjectKey> keys;
      for (size_t i = 0; i < nobj; ++i) keys.push_back("gpubench/" + std::to_string(it + 2) + "/" + std::to_string(i));
      auto a = Clk::now();
      auto pe = cl.batch_put_device(keys, sp, sizes, cfg, nullptr);
      auto b = Clk::now();
      std::vector<size_t> got;
      auto ge = cl.batch_get_device(keys, dp, sizes, nullptr, &got);
      auto c = Clk::now();
      const bool ok = std::all_of(pe.begin(), pe.end(), [](ErrorCode e) { return e == ErrorCode::OK; }) &&
                      std::all_of(ge.begin(), ge.end(), [](ErrorCode e) { return e == ErrorCode::OK; });
      if (!ok) ++failures;
      cl.batch_remove(keys);
      if (it >= 0 && ok) put_ms.push_back(ms(a, b)), get_ms.push_back(ms(b, c));
    }
    // spot check: first and last 64 KiB of the read-back equal the source
    std::vector<uint8_t> h1(65536), h2(65536);
    bool same = true;
    for (size_t off : {size_t{0}, nobj * osz - 65536}) {
      fab.value()->copy_from_device(h1.data(), static_cast<uint8_t*>(src) + off, {}, 65536, nullptr);
      fab.value()->copy_from_device(h2.data(), static_cast<uint8_t*>(dst) + off, {}, 65536, nullptr);
      same &= h1 == h2;
    }
    auto avg = [](const std::vector<double>& v) { return v.empty() ? 0.0 : std::accumulate(v.begin(), v.end(), 0.0) / static_cast<double>(v.size()); };
    const double gb = static_cast<double>(nobj * osz) / 1e9;
    std::printf("{\"mode\": \"gpu\", \"device\": %d, \"objects\": %zu, \"size\": %zu, \"iterations\": %zu, \"failures\": %d, \"verified\": %s, "
                "\"put_ms_p50\": %.3f, \"get_ms_p50\": %.3f, \"put_GBps\": %.1f, \"get_GBps\": %.1f, \"kernel_ms_total\": %.2f, \"launches\": %llu}\n",
                device, nobj, osz, put_ms.size(), failures, same ? "true" : "false", pct(put_ms, 0.5), pct(get_ms, 0.5),
                put_ms.empty() ? 0.0 : gb / (avg(put_ms) * 1e-3), get_ms.empty() ? 0.0 : gb / (avg(get_ms) * 1e-3),
                fab.value()->total_device_ms() - dev0, static_cast<unsigned long long>(fab.value()->launches()));
    gpu::device_free(device, src);
    gpu::device_free(device, dst);
    return failures || !same ? 1 : 0;
  }
  if (mode == "devclient") {
    // Client-level cost of the device batch API without a GPU: an in-process keystone behind the real RPC server (the client
    // reaches it over the same-host shared-memory channel), synthetic GPU pools, and a transport whose transfers are free.
    // What is left is exactly what bounds batches of small objects: Keystone round trips + the client's own per-object work.
    struct NullTransport : client::DeviceTransport {
      // ticket = launch number; the batch's op count is all wait needs
      Result<uint64_t> submit_put(const std::vector<client::DeviceShardOp>& ops, const std::vector<const void*>&, ChecksumAlgo,
                                  void*) override {
        return submit(ops.size());
      }
      Result<uint64_t> submit_get(const std::vector<client::DeviceShardOp>& ops, const std::vector<void*>&, void*) override {
        return submit(ops.size());
      }
      ErrorCode wait(uint64_t ticket, client::DeviceBatchResult* res) override {
        const size_t nops = nops_of[ticket];
        nops_of.erase(ticket);
        *res = {std::vector<uint64_t>(nops, 0x1234), std::vector<uint32_t>(nops, 0), std::vector<ErrorCode>(nops, ErrorCode::OK)};
        return ErrorCode::OK;
      }
      bool can_reach(const ShardPlacement&) const override { return true; }
      uint64_t launches() const override { return n; }
      uint64_t submit(size_t nops) {
        nops_of[++n] = nops;
        return n;
      }
      uint64_t n = 0;
      std::map<uint64_t, size_t> nops_of;
    };
    const int batch = std::max(1, static_cast<int>(args.num("batch", 4096)));
    const int iters = std::max(1, static_cast<int>(args.num("iterations", 20)));
    const size_t size = static_cast<size_t>(args.num("size", 4096));
    KeystoneConfig kc;
    kc.cluster_id = "bench";
    kc.listen_address = "127.0.0.1:0";
    kc.http_metrics_port = "off";
    kc.enable_gc = false;
    auto ks = std::make_shared<keystone::KeystoneService>(kc, nullptr);
    if (ks->initialize() != ErrorCode::OK || ks->start() != ErrorCode::OK) return 1;
    rpc::RpcService rpc(ks, kc);
    if (rpc.start() != ErrorCode::OK) return 1;
    for (int p = 0; p < 8; ++p) {
      MemoryPool mp;
      mp.id = "hbm" + std::to_string(p);
      mp.node_id = "gpu" + std::to_string(p);
      mp.worker_id = "w" + std::to_string(p);
      mp.size = 64ull << 30;
      mp.storage_class = StorageClass::RAM_GPU;
      mp.gpu_device_id = p;
      mp.ucx_endpoint = "127.0.0.1:1";
      ks->register_memory_pool(mp);
    }
    client::BlackbirdClientOptions o;
    o.keystone_host = "127.0.0.1";
    o.keystone_port = rpc.rpc_port();
    o.node_id = "gpu0";
    o.register_session = false;
    client::BlackbirdClient cl(o);
    if (cl.connect() != ErrorCode::OK) return 1;
    cl.set_device_transport(std::make_shared<NullTransport>());
    WorkerConfig cfg;
    cfg.replication_factor = 1;
    cfg.max_workers_per_copy = 1;
    cfg.ttl_ms = 0;
    cfg.preferred_node = "gpu1";
    cfg.preferred_classes = {StorageClass::RAM_GPU};
    std::vector<const void*> src(static_cast<size_t>(batch), reinterpret_cast<const void*>(0x10000));
    std::vector<void*> dst(static_cast<size_t>(batch), reinterpret_cast<void*>(0x10000));
    const std::vector<size_t> sizes(static_cast<size_t>(batch), size);
    double t_put = 0, t_get = 0, t_rm = 0;
    for (int it = 0; it < iters + 1; ++it) {
      std::vector<ObjectKey> keys;
      for (int i = 0; i < batch; ++i) keys.push_back("dc/" + std::to_string(it) + "/" + std::to_string(i));
      auto a = Clk::now();
      auto e1 = cl.batch_put_device(keys, src, sizes, cfg, nullptr);
      auto b = Clk::now();
      auto e2 = cl.batch_get_device(keys, dst, sizes, nullptr, nullptr);
      auto c = Clk::now();
      cl.batch_remove(keys);
      auto d = Clk::now();
      if (e1[0] != ErrorCode::OK || e2[0] != ErrorCode::OK) {
        std::fprintf(stderr, "devclient bench: %s / %s\n", std::string(to_string(e1[0])).c_str(), std::string(to_string(e2[0])).c_str());
        return 1;
      }
      if (it) t_put += ms(a, b), t_get += ms(b, c), t_rm += ms(c, d);  // first round warms the channel and the caches up
    }
    const double n = static_cast<double>(batch) * iters;
    std::printf("{\"mode\": \"devclient\", \"batch\": %d, \"size\": %zu, \"put_us_per_obj\": %.3f, \"get_us_per_obj\": %.3f, "
                "\"remove_us_per_obj\": %.3f, \"put_objects_per_s\": %.0f, \"get_objects_per_s\": %.0f}\n",
                batch, size, t_put * 1000 / n, t_get * 1000 / n, t_rm * 1000 / n, n / t_put * 1000, n / t_get * 1000);
    rpc.stop();
    ks->stop();
    return 0;
  }
  if (mode == "control") {
    // Control-plane throughput: T clients drive batch_put_start -> batch_put_complete -> batch_get_workers ->
    // batch_remove_object against an in-process keystone with synthetic pools (no data plane involved).
    const int threads = std::max(1, static_cast<int>(args.num("threads", 4)));
    const int batch = std::max(1, static_cast<int>(args.num("batch", 4096)));
    const int iters = std::max(1, static_cast<int>(args.num("iterations", 20)));
    const int npools = std::max(1, static_cast<int>(args.num("pools", 8)));
    const bool over_rpc = args.has("rpc");
    KeystoneConfig kc;
    kc.cluster_id = "bench";
    kc.listen_address = "127.0.0.1:0";
    kc.http_metrics_port = "off";
    kc.enable_gc = false;
    kc.rpc_threads = std::max(2, threads);
    auto ks = std::make_shared<keystone::KeystoneService>(kc, nullptr);
    if (ks->initialize() != ErrorCode::OK || ks->start() != ErrorCode::OK) return 1;
    rpc::RpcService rpc(ks, kc);
    if (over_rpc && rpc.start() != ErrorCode::OK) return 1;
    for (int p = 0; p < npools; ++p) {
      WorkerRecord w;
      w.worker_id = "w" + std::to_string(p);
      w.node_id = "n" + std::to_string(p);
      w.ucx_endpoint = "127.0.0.1:1";
      ks->register_worker(w);
      MemoryPool mp;
      mp.id = "p" + std::to_string(p);
      mp.node_id = w.node_id;
      mp.worker_id = w.worker_id;
      mp.size = 64ull << 30;
      mp.storage_class = StorageClass::RAM_GPU;
      mp.ucx_endpoint = w.ucx_endpoint;
      ks->register_memory_pool(mp);
    }
    std::vector<double> t_start(threads), t_done(threads), t_get(threads), t_rm(threads);
    std::vector<std::thread> ts;
    const auto t0 = Clk::now();
    for (int t = 0; t < threads; ++t) {
      ts.emplace_back([&, t] {
        std::shared_ptr<rpc::KeystoneApi> api;
        if (over_rpc) {
          auto c = std::make_shared<rpc::KeystoneRpcClient>();
          if (c->connect("127.0.0.1", rpc.rpc_port(), 5000) != ErrorCode::OK) return;
          api = c;
        } else {
          api = std::make_shared<rpc::LocalKeystoneApi>(ks);
        }
        WorkerConfig cfg;
        cfg.replication_factor = 1;
        cfg.max_workers_per_copy = 1;
        cfg.ttl_ms = 0;
        for (int it = 0; it < iters; ++it) {
          std::vector<keystone::PutStartItem> items;
          std::vector<ObjectKey> keys;
          for (int i = 0; i < batch; ++i) {
            keys.push_back("t" + std::to_string(t) + "/" + std::to_string(it) + "/" + std::to_string(i));
            items.push_back({keys.back(), 256, cfg});
          }
          const std::vector<keystone::ShardChecksums> sums(keys.size());
          auto a = Clk::now();
          auto placed = api->batch_put_start(items);
          auto b = Clk::now();
          api->batch_put_complete(keys, sums);
          auto c = Clk::now();
          auto got = api->batch_get_workers(keys);
          auto d = Clk::now();
          api->batch_remove_object(keys);
          auto e = Clk::now();
          t_start[t] += ms(a, b), t_done[t] += ms(b, c), t_get[t] += ms(c, d), t_rm[t] += ms(d, e);
          if (placed.empty() || !placed[0].ok() || got.empty() || !got[0].ok()) std::fprintf(stderr, "control bench: operation failed\n");
        }
      });
    }
    for (auto& th : ts) th.join();
    const double wall = ms(t0, Clk::now());
    const double objs = static_cast<double>(threads) * batch * iters;
    auto per = [&](const std::vector<double>& v) { return std::accumulate(v.begin(), v.end(), 0.0) * 1000.0 / objs; };
    std::printf("{\"mode\": \"control\", \"transport\": \"%s\", \"threads\": %d, \"batch\": %d, \"objects\": %.0f, \"wall_ms\": %.1f, "
                "\"object_lifecycles_per_s\": %.0f, \"put_start_us_per_obj\": %.3f, \"put_complete_us_per_obj\": %.3f, "
                "\"get_workers_us_per_obj\": %.3f, \"remove_us_per_obj\": %.3f}\n",
                over_rpc ? "tcp" : "in-process", threads, batch, objs, wall, objs * 1000.0 / wall, per(t_start), per(t_done), per(t_get), per(t_rm));
    rpc.stop();
    ks->stop();
    return 0;
  }
  auto hp = split_host_port(args.get("keystone", "127.0.0.1:9090"));
  if (!hp) return 2;
  client::BlackbirdClientOptions o;
  o.keystone_host = hp->first;
  o.keystone_port = static_cast<uint16_t>(hp->second);
  o.io_parallelism = static_cast<size_t>(args.num("parallelism", 4));
  client::BlackbirdClient cl(o);
  auto t_setup = Clk::now();
  if (cl.connect() != ErrorCode::OK) {
    std::fprintf(stderr, "cannot connect to keystone\n");
    return 1;
  }
  const double setup_ms = ms(t_setup, Clk::now());
  const size_t size = static_cast<size_t>(args.num("size", 1 << 20));
  const int iters = static_cast<int>(args.num("iterations", 10));
  const int batch = static_cast<int>(std::max<long long>(1, args.num("batch", 1)));
  WorkerConfig cfg;
  cfg.replication_factor = static_cast<size_t>(args.num("replicas", 1));
  cfg.max_workers_per_copy = static_cast<size_t>(args.num("max-workers", 1));
  if (args.get("checksum") == "crc32c") cfg.checksum = ChecksumAlgo::CRC32C;
  if (args.get("checksum") == "xxh3") cfg.checksum = ChecksumAlgo::XXH3;
  if (args.get("checksum") == "none") cfg.checksum = ChecksumAlgo::NONE;
  std::vector<uint8_t> data(size);
  std::mt19937_64 rng(1);
  for (size_t i = 0; i + 8 <= size; i += 8) {
    uint64_t v = rng();
    std::memcpy(&data[i], &v, 8);
  }
  const std::string prefix = args.get("key-prefix", "bench-" + std::to_string(Clk::now().time_since_epoch().count()));
  std::vector<double> wr, rd;
  int failures = 0;
  std::vector<uint8_t> read_buf(batch == 1 ? size : 0);
  auto t_total = Clk::now();
  for (int it = 0; it < iters; ++it) {
    std::vector<ObjectKey> keys;
    std::vector<const uint8_t*> ptrs;
    std::vector<size_t> sizes;
    for (int b = 0; b < batch; ++b) {
      keys.push_back(prefix + "-" + std::to_string(it) + "-" + std::to_string(b));
      ptrs.push_back(data.data());
      sizes.push_back(size);
    }
    auto a = Clk::now();
    auto ecs = batch == 1 ? std::vector<ErrorCode>{cl.put(keys[0], data.data(), size, cfg)} : cl.batch_put(keys, ptrs, sizes, cfg);
    auto b2 = Clk::now();
    bool ok = std::all_of(ecs.begin(), ecs.end(), [](ErrorCode e) { return e == ErrorCode::OK; });
    if (ok) {
      if (batch == 1) {  // like the reference's benchmark_client (:230-239): read back into a reused buffer
        size_t got = 0;
        ok = cl.get_into(keys[0], read_buf.data(), read_buf.size(), &got) == ErrorCode::OK && got == size;
      } else {
        auto got = cl.batch_get(keys);
        ok = std::all_of(got.begin(), got.end(), [](const auto& r) { return r.ok(); });
      }
    }
    auto c = Clk::now();
    if (!ok) {
      ++failures;
    } else {
      wr.push_back(ms(a, b2));
      rd.push_back(ms(b2, c));
    }
    cl.batch_remove(keys);
  }
  const double total_ms = ms(t_total, Clk::now());
  auto avg = [](const std::vector<double>& v) { return v.empty() ? 0.0 : std::accumulate(v.begin(), v.end(), 0.0) / static_cast<double>(v.size()); };
  const double bytes = static_cast<double>(size) * batch;
  std::printf("{\"size\": %zu, \"batch\": %d, \"iterations\": %zu, \"failures\": %d, \"setup_ms\": %.3f, \"total_ms\": %.3f, "
              "\"write_avg_ms\": %.4f, \"write_p50_ms\": %.4f, \"write_p99_ms\": %.4f, \"write_MiBps\": %.1f, "
              "\"read_avg_ms\": %.4f, \"read_p50_ms\": %.4f, \"read_p99_ms\": %.4f, \"read_MiBps\": %.1f}\n",
              size, batch, wr.size(), failures, setup_ms, total_ms, avg(wr), pct(wr, 0.5), pct(wr, 0.99),
              wr.empty() ? 0.0 : bytes * 1000.0 / (avg(wr) * 1048576.0), avg(rd), pct(rd, 0.5), pct(rd, 0.99),
              rd.empty() ? 0.0 : bytes * 1000.0 / (avg(rd) * 1048576.0));
  return failures ? 1 : 0;
}
