// bb-p2p-probe: what does this box's NVLink / NVSwitch actually deliver, per access method?
//
// Single process, all visible GPUs, peer access enabled all-pairs.  For every method the probe moves `--mib` MiB per
// active GPU per iteration and reports payload GB/s per GPU (device-timed with CUDA events on every GPU's stream,
// min / mean over the active GPUs).  The numbers are the roofline denominators the fused kernels are judged against
// (BASELINE.md section 4: "per-object cudaMemcpyPeerAsync" comparator + the measured peer peak).
//
//   methods : memcpy      cudaMemcpyPeerAsync (copy engines)
//             stg         SIMT kernel, local LDG.128 -> peer STG.128 (push)
//             ldg         SIMT kernel, peer LDG.128 -> local STG.128 (pull)
//             bulk_push   TMA ring: cp.async.bulk local -> smem -> cp.async.bulk peer   (what bb_xfer's put does)
//             bulk_pull   TMA ring: cp.async.bulk peer -> smem -> cp.async.bulk local   (what bb_xfer's get does)
//             mc_simt     multimem.st.v4 from registers: 1 writer -> all GPUs of the multicast group (NVLS broadcast)
//             mc_smem     TMA local -> smem, W warps multimem.st from smem (what bb_xfer's NVLS fan-out does)
//   patterns: uni (0 -> 1), bidir (0 <-> 1), ring (i -> i+1 for every GPU)
//
// JSON lines on stdout, one per measurement.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#define CK(x)                                                                                     \
  do {                                                                                            \
    cudaError_t e_ = (x);                                                                         \
    if (e_ != cudaSuccess) {                                                                      \
      std::fprintf(stderr, "%s:%d %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));   \
      std::exit(1);                                                                               \
    }                                                                                             \
  } while (0)
#define CKD(x)                                                                        \
  do {                                                                                \
    CUresult r_ = (x);                                                                \
    if (r_ != CUDA_SUCCESS) {                                                         \
      const char* s_ = nullptr;                                                       \
      cuGetErrorString(r_, &s_);                                                      \
      std::fprintf(stderr, "%s:%d %s -> %s\n", __FILE__, __LINE__, #x, s_ ? s_ : "?"); \
      return false;                                                                   \
    }                                                                                 \
  } while (0)

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t par) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(b)), "r"(par)
        : "memory");
  }
}
__device__ __forceinline__ void bulk_g2s(void* s, const void* g, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(s)),
               "l"(g), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* g, const void* s, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g), "r"(smem_u32(s)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_n(int n) {
  switch (n) {
    case 0: asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory"); break;
    case 3: asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory"); break;
    case 4: asm volatile("cp.async.bulk.wait_group.read 4;" ::: "memory"); break;
    default: asm volatile("cp.async.bulk.wait_group.read 6;" ::: "memory"); break;
  }
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void mc_st_v4(void* p, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}

// ---------------------------------------------------------------- SIMT copies
template <int UNROLL>
__global__ void __launch_bounds__(512) k_copy_v4(const uint4* __restrict__ src, uint4* __restrict__ dst, uint64_t n16) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + (UNROLL - 1) * stride < n16; i += UNROLL * stride) {
    uint4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) v[u] = __ldcs(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) __stcs(dst + i + u * stride, v[u]);
  }
  for (; i < n16; i += stride) dst[i] = src[i];
}

__global__ void __launch_bounds__(512) k_mc_simt(const uint4* __restrict__ src, uint4* mc, uint64_t n16) {
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = __ldcs(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u) mc_st_v4(mc + i + u * stride, v[u]);
  }
  for (; i < n16; i += stride) mc_st_v4(mc + i, src[i]);
}

// ---------------------------------------------------------------- TMA ring (bulk in, bulk out or multimem out)
// warp 0: producer.  warp 1: bulk store issuer.  warps 2..: multimem store warps (mc mode).
struct RingParams {
  const uint8_t* src;
  uint8_t* dst;
  uint64_t nbytes;
  uint32_t tile;
  uint32_t stages;
  uint32_t lag;
  uint32_t mc_warps;  // 0 = bulk store
  uint32_t interleave;
};

__global__ void __launch_bounds__(320, 1) k_ring(const RingParams p) {
  extern __shared__ __align__(1024) uint8_t sm[];
  uint64_t* full = reinterpret_cast<uint64_t*>(sm);
  uint64_t* empty = full + 32;
  uint8_t* tiles = sm + 1024;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t ntiles = p.nbytes / p.tile;
  uint64_t t0, cnt, step;
  if (p.interleave) {
    t0 = blockIdx.x;
    step = gridDim.x;
    cnt = blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  } else {
    const uint64_t per = (ntiles + gridDim.x - 1) / gridDim.x;
    t0 = per * blockIdx.x;
    step = 1;
    cnt = t0 < ntiles ? min(per, ntiles - t0) : 0;
  }
  if (threadIdx.x == 0) {
    for (uint32_t i = 0; i < p.stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], p.mc_warps ? p.mc_warps : 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      for (uint64_t it = 0; it < cnt; ++it) {
        const uint32_t s = it % p.stages, par = (it / p.stages) & 1;
        mbar_wait(&empty[s], par ^ 1);
        mbar_expect(&full[s], p.tile);
        bulk_g2s(tiles + static_cast<uint64_t>(s) * p.tile, p.src + (t0 + it * step) * p.tile, p.tile, &full[s]);
      }
    }
  } else if (p.mc_warps == 0) {
    if (warp == 1 && lane == 0) {
      for (uint64_t it = 0; it < cnt; ++it) {
        const uint32_t s = it % p.stages, par = (it / p.stages) & 1;
        mbar_wait(&full[s], par);
        bulk_s2g(p.dst + (t0 + it * step) * p.tile, tiles + static_cast<uint64_t>(s) * p.tile, p.tile);
        bulk_commit();
        if (it >= p.lag) {
          bulk_wait_read_n(static_cast<int>(p.lag));
          mbar_arrive(&empty[(it - p.lag) % p.stages]);
        }
      }
      bulk_wait_all();
    }
  } else if (warp - 1 < p.mc_warps) {
    const uint32_t w = warp - 1;
    const uint32_t slice = p.tile / p.mc_warps;  // bytes of a tile per store warp
    for (uint64_t it = 0; it < cnt; ++it) {
      const uint32_t s = it % p.stages, par = (it / p.stages) & 1;
      mbar_wait(&full[s], par);
      const uint8_t* st = tiles + static_cast<uint64_t>(s) * p.tile + w * slice;
      uint8_t* g = p.dst + (t0 + it * step) * p.tile + w * slice;
#pragma unroll 4
      for (uint32_t o = lane * 16; o < slice; o += 512) mc_st_v4(g + o, *reinterpret_cast<const uint4*>(st + o));
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
  }
}

// ---------------------------------------------------------------- launch -> completion-flag floor
__global__ void k_flag(volatile uint32_t* flag, uint32_t v) {
  __threadfence_system();
  *flag = v;
}
__global__ void k_flag_copy(const uint4* src, uint4* dst, uint32_t n16, volatile uint32_t* flag, uint32_t v) {
  for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) dst[i] = src[i];
  __threadfence_system();
  __syncwarp();
  if (threadIdx.x == 0) *flag = v;
}

struct Dev {
  int id;
  cudaStream_t st;
  cudaEvent_t e0, e1;
  uint8_t* src;
  uint8_t* dst;
};

struct Mc {
  bool ok = false;
  CUdeviceptr mc_va = 0;
  std::vector<CUdeviceptr> uc_va;
  std::vector<CUmemGenericAllocationHandle> mem;
  CUmemGenericAllocationHandle mch = 0;
  size_t size = 0;
};

bool mc_setup(int ndev, size_t bytes, Mc* m) {
  CKD(cuInit(0));
  int sup = 0;
  CKD(cuDeviceGetAttribute(&sup, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, 0));
  if (!sup) {
    std::fprintf(stderr, "multicast not supported\n");
    return false;
  }
  CUmulticastObjectProp mp{};
  mp.numDevices = ndev;
  mp.handleTypes = CU_MEM_HANDLE_TYPE_NONE;
  size_t gran = 0;
  mp.size = bytes;
  CKD(cuMulticastGetGranularity(&gran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED));
  bytes = (bytes + gran - 1) / gran * gran;
  mp.size = bytes;
  m->size = bytes;
  CKD(cuMulticastCreate(&m->mch, &mp));
  for (int d = 0; d < ndev; ++d) CKD(cuMulticastAddDevice(m->mch, d));
  m->mem.resize(ndev);
  m->uc_va.resize(ndev);
  for (int d = 0; d < ndev; ++d) {
    CK(cudaSetDevice(d));
    CUmemAllocationProp ap{};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = d;
    CKD(cuMemCreate(&m->mem[d], bytes, &ap, 0));
    CKD(cuMulticastBindMem(m->mch, 0, m->mem[d], 0, bytes, 0));
    CKD(cuMemAddressReserve(&m->uc_va[d], bytes, gran, 0, 0));
    CKD(cuMemMap(m->uc_va[d], bytes, 0, m->mem[d], 0));
    CUmemAccessDesc ad{};
    ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ad.location.id = d;
    ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CKD(cuMemSetAccess(m->uc_va[d], bytes, &ad, 1));
  }
  CKD(cuMemAddressReserve(&m->mc_va, bytes, gran, 0, 0));
  CKD(cuMemMap(m->mc_va, bytes, 0, m->mch, 0));
  std::vector<CUmemAccessDesc> ads(ndev);
  for (int d = 0; d < ndev; ++d) {
    ads[d].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ads[d].location.id = d;
    ads[d].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  }
  CKD(cuMemSetAccess(m->mc_va, bytes, ads.data(), ndev));
  m->ok = true;
  return true;
}

struct Opt {
  size_t mib = 1024;
  int iters = 5;
  int ndev = 0;
  bool quick = false;
  bool mc = true;
  bool only_mc = false;
  bool latency = false;
};

void report(const char* method, const char* pattern, const std::string& cfg, const std::vector<float>& ms, size_t bytes, int iters,
            int fanout = 1) {
  double mn = 1e30, sum = 0;
  for (float m : ms) {
    const double g = static_cast<double>(bytes) * iters / (m * 1e-3) / 1e9;
    mn = std::min(mn, g);
    sum += g;
  }
  std::printf("{\"method\": \"%s\", \"pattern\": \"%s\", \"cfg\": \"%s\", \"active_gpus\": %zu, \"GBps_per_gpu_min\": %.1f, "
              "\"GBps_per_gpu_mean\": %.1f, \"delivered_GBps_per_writer\": %.1f}\n",
              method, pattern, cfg.c_str(), ms.size(), mn, sum / ms.size(), sum / ms.size() * fanout);
  std::fflush(stdout);
}

}  // namespace

int main(int argc, char** argv) {
  Opt o;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    if (a == "--mib" && i + 1 < argc) o.mib = std::strtoull(argv[++i], nullptr, 10);
    else if (a == "--iters" && i + 1 < argc) o.iters = std::atoi(argv[++i]);
    else if (a == "--gpus" && i + 1 < argc) o.ndev = std::atoi(argv[++i]);
    else if (a == "--quick") o.quick = true;
    else if (a == "--no-mc") o.mc = false;
    else if (a == "--only-mc") o.only_mc = true;  // skip the unicast sweep (ncu application replay re-runs the whole program)
    else if (a == "--latency") o.latency = true;
  }
  int n = 0;
  CK(cudaGetDeviceCount(&n));
  if (o.ndev <= 0 || o.ndev > n) o.ndev = n;
  n = o.ndev;
  if (n < 2 && !o.latency) {
    std::printf("{\"error\": \"need >= 2 GPUs, have %d\"}\n", n);
    return 0;
  }
  const size_t bytes = o.mib << 20;
  if (o.latency) {
    // how long does it take, on this box, from cudaLaunchKernel to the host seeing a flag the kernel wrote to pinned
    // memory?  (the floor under any single-object put / get latency); vs the same with an event record + synchronize
    CK(cudaSetDevice(0));
    if (n > 1) {
      cudaError_t e = cudaDeviceEnablePeerAccess(1, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e);
      (void)cudaGetLastError();
    }
    volatile uint32_t* flag = nullptr;
    CK(cudaHostAlloc(const_cast<uint32_t**>(&flag), 64, cudaHostAllocDefault));
    *flag = 0;
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cudaEvent_t ev;
    CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    uint4 *a = nullptr, *b = nullptr, *peer = nullptr;
    CK(cudaMalloc(&a, 4096));
    CK(cudaMalloc(&b, 4096));
    if (n > 1) {
      CK(cudaSetDevice(1));
      CK(cudaMalloc(&peer, 4096));
      CK(cudaSetDevice(0));
    }
    auto pct = [](std::vector<double> v, double q) {
      std::sort(v.begin(), v.end());
      return v[std::min(v.size() - 1, static_cast<size_t>(q * v.size()))];
    };
    auto now_us = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    for (int mode = 0; mode < 5; ++mode) {
      if (mode == 3 && !peer) continue;
      std::vector<double> t;
      for (uint32_t it = 1; it <= 2200; ++it) {
        const double t0 = now_us();
        if (mode == 0) k_flag<<<1, 32, 0, st>>>(flag, it);
        else if (mode == 1) k_flag_copy<<<1, 32, 0, st>>>(a, b, 256, flag, it);
        else if (mode == 3) k_flag_copy<<<1, 32, 0, st>>>(a, peer, 256, flag, it);
        else k_flag<<<1, 32, 0, st>>>(flag, it);
        if (mode == 2) {
          CK(cudaEventRecord(ev, st));
          CK(cudaEventSynchronize(ev));
        } else if (mode == 4) {
          CK(cudaStreamSynchronize(st));
        } else {
          while (*flag != it) {
          }
        }
        const double t1 = now_us();
        if (it > 200) t.push_back(t1 - t0);
      }
      const char* names[] = {"launch+flag (empty kernel)", "launch+flag (4 KiB local copy, 1 warp)", "launch+event record+event sync (empty kernel)",
                             "launch+flag (4 KiB copy to peer, 1 warp)", "launch+stream sync (empty kernel)"};
      std::printf("{\"latency\": \"%s\", \"p50_us\": %.2f, \"p99_us\": %.2f}\n", names[mode], pct(t, 0.5), pct(t, 0.99));
    }
    return 0;
  }
  std::vector<Dev> dv(n);
  for (int d = 0; d < n; ++d) {
    CK(cudaSetDevice(d));
    for (int p = 0; p < n; ++p)
      if (p != d) {
        cudaError_t e = cudaDeviceEnablePeerAccess(p, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e);
        (void)cudaGetLastError();
      }
    dv[d].id = d;
    CK(cudaStreamCreateWithFlags(&dv[d].st, cudaStreamNonBlocking));
    CK(cudaEventCreate(&dv[d].e0));
    CK(cudaEventCreate(&dv[d].e1));
    CK(cudaMalloc(&dv[d].src, bytes));
    CK(cudaMalloc(&dv[d].dst, bytes));
    CK(cudaMemset(dv[d].src, 0x5A + d, bytes));
    CK(cudaMemset(dv[d].dst, 0, bytes));
    CK(cudaFuncSetAttribute(k_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  struct Pattern {
    const char* name;
    std::vector<int> active;
  };
  std::vector<Pattern> pats;
  pats.push_back({"uni", {0}});
  pats.push_back({"bidir", {0, 1}});
  if (n > 2) {
    std::vector<int> all(n);
    for (int d = 0; d < n; ++d) all[d] = d;
    pats.push_back({"ring", all});
  }
  auto sync_all = [&] {
    for (int d = 0; d < n; ++d) {
      CK(cudaSetDevice(d));
      CK(cudaDeviceSynchronize());
    }
  };
  // run `fn(dev, peer)` on every active device (dev -> (dev+1) % n), timed per device
  auto run = [&](const Pattern& pt, auto&& fn) {
    std::vector<float> ms;
    for (int rep = 0; rep < 2; ++rep) {  // rep 0 = warm-up
      sync_all();
      const int it = rep == 0 ? 1 : o.iters;
      for (int d : pt.active) {
        CK(cudaSetDevice(d));
        CK(cudaEventRecord(dv[d].e0, dv[d].st));
      }
      for (int i = 0; i < it; ++i)
        for (int d : pt.active) {
          CK(cudaSetDevice(d));
          fn(dv[d], dv[(d + 1) % n]);
        }
      for (int d : pt.active) {
        CK(cudaSetDevice(d));
        CK(cudaEventRecord(dv[d].e1, dv[d].st));
      }
      sync_all();
      if (rep == 1)
        for (int d : pt.active) {
          float m = 0;
          CK(cudaEventElapsedTime(&m, dv[d].e0, dv[d].e1));
          ms.push_back(m);
        }
    }
    CK(cudaGetLastError());
    return ms;
  };
  auto ring_launch = [&](const Dev& me, const uint8_t* src, uint8_t* dst, int ctas, uint32_t tile, uint32_t stages, uint32_t lag,
                         uint32_t mc_warps, uint32_t interleave) {
    RingParams p{src, dst, bytes, tile, stages, lag, mc_warps, interleave};
    const size_t smem = 1024 + static_cast<size_t>(tile) * stages;
    k_ring<<<ctas, 320, smem, me.st>>>(p);
  };

  if (o.only_mc) pats.clear();
  for (const Pattern& pt : pats) {
    report("memcpy", pt.name, "cudaMemcpyPeerAsync",
           run(pt, [&](const Dev& me, const Dev& peer) { CK(cudaMemcpyPeerAsync(peer.dst, peer.id, me.src, me.id, bytes, me.st)); }), bytes,
           o.iters);
    for (int ctas : {132, 264, 528}) {
      if (o.quick && ctas != 264) continue;
      char cfg[64];
      std::snprintf(cfg, sizeof cfg, "ctas=%d x512 unroll4", ctas);
      report("stg", pt.name, cfg, run(pt, [&](const Dev& me, const Dev& peer) {
               k_copy_v4<4><<<ctas, 512, 0, me.st>>>(reinterpret_cast<const uint4*>(me.src), reinterpret_cast<uint4*>(peer.dst), bytes / 16);
             }), bytes, o.iters);
      report("ldg", pt.name, cfg, run(pt, [&](const Dev& me, const Dev& peer) {
               k_copy_v4<4><<<ctas, 512, 0, me.st>>>(reinterpret_cast<const uint4*>(peer.src), reinterpret_cast<uint4*>(me.dst), bytes / 16);
             }), bytes, o.iters);
    }
    report("stg", pt.name, "ctas=264 x512 unroll8", run(pt, [&](const Dev& me, const Dev& peer) {
             k_copy_v4<8><<<264, 512, 0, me.st>>>(reinterpret_cast<const uint4*>(me.src), reinterpret_cast<uint4*>(peer.dst), bytes / 16);
           }), bytes, o.iters);
    report("ldg", pt.name, "ctas=264 x512 unroll8", run(pt, [&](const Dev& me, const Dev& peer) {
             k_copy_v4<8><<<264, 512, 0, me.st>>>(reinterpret_cast<const uint4*>(peer.src), reinterpret_cast<uint4*>(me.dst), bytes / 16);
           }), bytes, o.iters);
    struct RC {
      int ctas;
      uint32_t tile, stages, lag, inter;
    };
    std::vector<RC> rcs = {{128, 16384, 8, 2, 0},  {128, 16384, 12, 6, 0}, {132, 16384, 12, 6, 0}, {128, 32768, 6, 3, 0},
                           {132, 32768, 6, 3, 0},  {128, 65536, 3, 1, 0},  {64, 32768, 6, 3, 0},   {128, 16384, 12, 6, 1},
                           {128, 8192, 24, 6, 0},  {96, 32768, 6, 3, 0},   {132, 65536, 3, 1, 0},  {128, 32768, 6, 3, 1}};
    if (o.quick) rcs.resize(4);
    for (const RC& rc : rcs) {
      char cfg[96];
      std::snprintf(cfg, sizeof cfg, "ctas=%d tile=%u stages=%u lag=%u inter=%u inflight_MiB=%.1f", rc.ctas, rc.tile, rc.stages, rc.lag, rc.inter,
                    rc.ctas * static_cast<double>(rc.tile) * rc.stages / 1048576.0);
      report("bulk_push", pt.name, cfg, run(pt, [&](const Dev& me, const Dev& peer) {
               ring_launch(me, me.src, peer.dst, rc.ctas, rc.tile, rc.stages, rc.lag, 0, rc.inter);
             }), bytes, o.iters);
      report("bulk_pull", pt.name, cfg, run(pt, [&](const Dev& me, const Dev& peer) {
               ring_launch(me, peer.src, me.dst, rc.ctas, rc.tile, rc.stages, rc.lag, 0, rc.inter);
             }), bytes, o.iters);
    }
  }

  // correctness spot check of the ring kernel (bulk_push 0 -> 1)
  {
    CK(cudaSetDevice(0));
    CK(cudaMemset(dv[1].dst, 0, bytes));
    ring_launch(dv[0], dv[0].src, dv[1].dst, 128, 16384, 12, 6, 0, 0);
    CK(cudaStreamSynchronize(dv[0].st));
    std::vector<uint8_t> h(4096);
    CK(cudaMemcpy(h.data(), dv[1].dst + bytes - 4096, 4096, cudaMemcpyDeviceToHost));
    bool ok = true;
    for (uint8_t b : h) ok = ok && b == 0x5A;
    std::printf("{\"check\": \"bulk_push tail bytes\", \"ok\": %s}\n", ok ? "true" : "false");
  }

  if (o.mc) {
    for (int g : {2, 3, 4, 8}) {
      if (g > n) break;
      Mc m;
      if (!mc_setup(g, bytes, &m)) {
        std::printf("{\"method\": \"mc\", \"group\": %d, \"error\": \"multicast setup failed\"}\n", g);
        break;
      }
      Pattern one{"1-writer", {0}};
      Pattern all{"all-writers", {}};
      for (int d = 0; d < g; ++d) all.active.push_back(d);
      for (const Pattern* pt : {&one, &all}) {
        char cfg[96];
        for (int ctas : {132, 264}) {
          std::snprintf(cfg, sizeof cfg, "group=%d ctas=%d x512", g, ctas);
          report("mc_simt", pt->name, cfg, run(*pt, [&](const Dev& me, const Dev&) {
                   k_mc_simt<<<ctas, 512, 0, me.st>>>(reinterpret_cast<const uint4*>(me.src), reinterpret_cast<uint4*>(m.mc_va), bytes / 16);
                 }), bytes, o.iters, g);
        }
        for (uint32_t w : {1u, 2u, 4u, 8u}) {
          std::snprintf(cfg, sizeof cfg, "group=%d ctas=128 tile=16384 stages=8 store_warps=%u", g, w);
          report("mc_smem", pt->name, cfg, run(*pt, [&](const Dev& me, const Dev&) {
                   ring_launch(me, me.src, reinterpret_cast<uint8_t*>(m.mc_va), 128, 16384, 8, 0, w, 0);
                 }), bytes, o.iters, g);
        }
      }
      // verify: every member sees device 0's pattern after a 1-writer broadcast
      CK(cudaSetDevice(0));
      k_mc_simt<<<264, 512, 0, dv[0].st>>>(reinterpret_cast<const uint4*>(dv[0].src), reinterpret_cast<uint4*>(m.mc_va), bytes / 16);
      CK(cudaStreamSynchronize(dv[0].st));
      bool ok = true;
      for (int d = 0; d < g; ++d) {
        uint8_t h[256];
        CK(cudaSetDevice(d));
        CK(cudaMemcpy(h, reinterpret_cast<void*>(m.uc_va[d] + bytes / 2), 256, cudaMemcpyDeviceToHost));
        for (uint8_t b : h) ok = ok && b == 0x5A;
      }
      std::printf("{\"check\": \"multicast broadcast group=%d\", \"ok\": %s}\n", g, ok ? "true" : "false");
      // teardown
      cuMemUnmap(m.mc_va, m.size);
      cuMemAddressFree(m.mc_va, m.size);
      for (int d = 0; d < g; ++d) {
        cuMulticastUnbind(m.mch, d, 0, m.size);
        cuMemUnmap(m.uc_va[d], m.size);
        cuMemAddressFree(m.uc_va[d], m.size);
        cuMemRelease(m.mem[d]);
      }
      cuMemRelease(m.mch);
    }
  }
  return 0;
}
