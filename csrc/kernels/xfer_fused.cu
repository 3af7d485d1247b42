// bb_xfer: the fused batched put/get kernel (sm_90a).
//
// Replaces the reference's per-shard UCX RMA calls (blackbird_client.cpp:231-237 put,
// :315-327 get; SURVEY K1/K4/K6/K11/K13) with ONE launch per batch.  Every CTA owns a contiguous
// run of 16 KiB tiles of the batch (at most 8 tiles, two CTAs per SM, for NONE / XXH3 / BBH64; one
// persistent CTA per SM for CRC32C: see kStagesFor) and pipelines them through 6 (8) smem stages:
//
//   warp 0  producer : descriptor lookup (32 tiles looked up in parallel, xfer_common.cuh), zero-pads short
//                      tiles, `cp.async.bulk` global -> shared (TMA, mbarrier complete_tx).
//                      The source may be local HBM (put) or a peer GPU's slab over NVLink (get).  A gathering load
//                      (XFER_GATHER: a put of a strided source) fills the tile from its source row segments, one per
//                      lane, so the tile is byte for byte the tile of the dense object.  A paged one (XFER_PAGED)
//                      reads each row segment from its page, whose address it loads from the page table.
//   warp 2  store    : `cp.async.bulk` shared -> global to 1..3 destinations (local or
//                      peer-mapped: replica fan-out with a single HBM read), or `multimem.st`
//                      to an NVLS multicast address (one store, N replicas).  A store window (XFER_WINDOW) cuts
//                      each tile to its span; a strided one (XFER_STRIDED) to its row segments, one per lane.  A
//                      scattering store (XFER_SCATTER: a get into a strided destination) stores the whole tile as
//                      the row segments of the destination rows, one per lane; a paged one (XFER_PAGED) as the
//                      segments of its pages.
//   warp 3  finalizer: folds the per-tile partials into per-object digests in registers; an
//                      object that lives entirely inside this CTA's run is finalised with no
//                      global atomics; only the <=2 objects straddling a CTA boundary use them.
//                      Compares with the expected digest on get (CHECKSUM_MISMATCH source).
//   warps 4-7 epilogue: BBH64: the warpgroup issues 2x4 `wgmma.mma_async.m64n16k32.s32.u8.u8` that
//                      read the landed tile *in place* as the A operand against the BBH64 weight
//                      matrix (bbh_tile.cuh); the 128x16 s32 accumulators land in registers ->
//                      position-dependent 64-bit row hashes -> warp sum.  CRC32C: each warp streams its 4 KiB quarter of
//                      the tile as 8 Horner chains per lane through lane-private nibble shift tables
//                      (bank-conflict free); the chains run on across the tiles of an object and are
//                      combined (chain / lane / quarter, GF(2) shift algebra) once per object and CTA.
//
// Payload bytes never pass through registers on the BBH64 / copy-only unicast path: TMA in,
// tensor core reads shared memory, TMA out.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common/checksum.h"
#include "common/tchash_def.h"
#include "common/xxh3.h"
#include "kernels/bbh_tile.cuh"
#include "kernels/ptx.cuh"
#include "kernels/xfer.h"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {
namespace {

using namespace bb::ptx;

constexpr int kThreads = 256;
constexpr int kStoreLag = 2;         // stores may trail this many tiles before their stage is released
static_assert(kTileBytes == tchash::kTileBytes);

// Launch geometry.  The DRAM-bound digests (NONE, XXH3, BBH64) run short CTAs of at most kRunTiles tiles, two resident
// per SM with 6 stages each (12 tiles in flight per SM), and leave the balancing to the hardware block scheduler: a CTA
// that finishes frees its slot for the next run, so a launch no longer ends with the slowest SM's fixed share of the
// batch.  CRC32C is bound by shared-memory lookups, not by DRAM, and each CTA builds ~14 KB of shift tables before its
// first tile: it keeps one persistent CTA per SM with 8 stages.
template <int ALGO>
constexpr int kStagesFor = ALGO == ALGO_CRC32C ? 8 : 6;
// CTAs per SM that shared memory admits at STAGES stages of 16 KiB (checked against SmemT below).
constexpr int resident_ctas(int stages) { return stages <= 6 ? 2 : 1; }
// Tiles per CTA run of the short-CTA geometry (128 KiB).  bench/cta_balance.py at 64 x 64 MiB, XXH3, H100 SXM 80 GB at
// 700 W, kernel-only put ms for runs of 64 / 32 / 24 / 16 / 12 / 8 / 4 tiles: 3.00 / 2.98 / 2.97 / 2.94 / 2.93 / 2.88 /
// 2.86 (one persistent CTA per SM: 3.01).  Shorter runs raise the steady rate and cut the end-of-launch tail to ~10 µs
// at 8 tiles.  4-tile runs were another 1% faster on that local-HBM shape, but a run
// shorter than the 6-stage ring cannot fill it, and peer reads over NVLink need every tile in flight to hide latency.
constexpr uint32_t kRunTiles = 8;

__constant__ uint64_t c_col_mul[tchash::kN];
__constant__ uint32_t c_xpow_tiles[32];  // x^(8 * 16384 * 2^j) mod P  (CRC32C cross-CTA combine)
__constant__ uint8_t c_xxh_secret[xxh3::kSecretSize];  // XXH3 default secret

// CRC shift tables: index -> byte distance
enum CrcTab : int { T128 = 0, T4, T8, T16, T32, T64, T4096, T16384, TCHAIN, TJUMP, kNumCrcTabs };
constexpr int kCrcChains = 8;                     // independent Horner chains per lane
constexpr int kCrcChainRows = 32 / kCrcChains;   // rows (of 128 B) of a tile quarter per chain
constexpr uint64_t kCrcTabBytes[kNumCrcTabs] = {128, 4, 8, 16, 32, 64, 4096, 16384, kCrcChainRows * 128,
                                                16384 - (kCrcChainRows - 1) * 128};

struct StageMeta {  // 64 bytes
  uint64_t dst[kMaxDst];
  uint64_t nbytes;
  uint64_t expect;
  uint32_t desc;
  uint32_t tile_in_obj;
  uint32_t bytes;
  uint32_t ndst_flags;  // ndst | flags << 8
  uint32_t obj_ntiles;
  uint32_t crc_unpad;
};
static_assert(sizeof(StageMeta) == 64);

struct LookupEntry {  // producer-private staging of 32 parallel lookups
  StageMeta m;
  uint64_t src;
  uint64_t pad;
};

template <int ALGO, int kStages>
struct __align__(1024) SmemT {
  uint8_t tile[kStages][kTileBytes];
  uint8_t w[2048];
  uint64_t full[kStages];
  uint64_t epi_done[kStages];
  uint64_t empty[kStages];
  StageMeta meta[kStages];
  uint64_t part[kStages][4];
  LookupEntry lk[32];
  uint32_t dirty[kStages];
  uint32_t crc_t[ALGO == ALGO_CRC32C ? kNumCrcTabs : 1][4][256];
  // x^(8*128) shift as 8 nibble tables with one private copy per lane ([nibble][value][lane]: lane l only ever
  // touches bank l, so the 8 lookups of a step are bank-conflict free whatever the data is).
  // 2 KiB of slack: the kernel rounds the table's shared address up to 2048 so that the value index (bits 7-10)
  // can be OR-ed into the lane's base address with a single LOP3.
  uint32_t crc_nib[ALGO == ALGO_CRC32C ? 8 * 16 * 32 + 512 : 1];
  // XXH3: per-(block, lane) stripe sums of every tile in flight, written by the epilogue warps and consumed by the
  // finalizer's scramble chain; and the secret words in the order the epilogue indexes them
  // ([0..22] = accumulate keys (word s + lane), [24..31] = keys of the last stripe, [32..39] = scramble keys, [40..47] = merge keys).
  uint64_t xs[ALGO == ALGO_XXH3 ? kStages : 1][ALGO == ALGO_XXH3 ? 16 : 1][8];
  uint64_t xkey[ALGO == ALGO_XXH3 ? 48 : 1];
};

struct Params {
  const XferDesc* descs;
  const uint32_t* tile_start;
  uint32_t ndesc;
  uint32_t total_tiles;
  unsigned long long* sum_ws;
  uint32_t* done_ws;
  uint64_t* digest_out;
  uint32_t* status_out;
  const uint32_t* crc_tables;  // [kNumCrcTabs][4][256]
  uint32_t* debug_d;
  // Optional per-tile pipeline trace (diagnostics): [tile][4] globaltimer ns = load issued, tile landed in smem,
  // store issued, smem slot released.
  unsigned long long* trace_d;
  // Small batches carry their descriptor table in the kernel parameters (constant bank): no H2D
  // copy ahead of the launch, which is most of a single-object put/get's latency.
  uint32_t use_inline;
  uint32_t inl_tile_start[kInlineDescs + 1];
  XferDesc inl_descs[kInlineDescs];
  // Row patterns of XFER_STRIDED, XFER_GATHER and XFER_SCATTER descriptors (XferLaunch::strides), and their copy for
  // inline batches.
  const XferStride* strides;
  XferStride inl_strides[kInlineDescs];
};

// s * x^(8k) mod P through the 4x256 table of distance k.
__device__ __forceinline__ uint32_t crc_shift(const uint32_t (*t)[256], uint32_t s) {
  return t[0][s & 0xFFu] ^ t[1][(s >> 8) & 0xFFu] ^ t[2][(s >> 16) & 0xFFu] ^ t[3][s >> 24];
}

// One nibble of the lane-private x^(8*128) shift: table [nibble J][value][lane], 2 KiB per nibble, base 2 KiB aligned
// so the value index (bits 7-10) is OR-ed into the lane's base address by one LOP3.  The table is read-only after setup.
template <int J>
__device__ __forceinline__ uint32_t crc_nib_lookup(uint32_t v, uint32_t nib_lane) {
  const uint32_t x = (4 * J >= 7) ? (v >> (4 * J >= 7 ? 4 * J - 7 : 0)) : (v << (4 * J >= 7 ? 0 : 7 - 4 * J));
  uint32_t addr, t;
  asm("lop3.b32 %0, %1, 0x780, %2, 0xEA;" : "=r"(addr) : "r"(x), "r"(nib_lane));  // (x & 0x780) | base
  asm("ld.shared.u32 %0, [%1+%2];" : "=r"(t) : "r"(addr), "n"(J * 2048));
  return t;
}
__device__ __forceinline__ uint32_t crc_nib_shift(uint32_t v, uint32_t nib_lane) {
  return crc_nib_lookup<0>(v, nib_lane) ^ crc_nib_lookup<1>(v, nib_lane) ^ crc_nib_lookup<2>(v, nib_lane) ^
         crc_nib_lookup<3>(v, nib_lane) ^ crc_nib_lookup<4>(v, nib_lane) ^ crc_nib_lookup<5>(v, nib_lane) ^
         crc_nib_lookup<6>(v, nib_lane) ^ crc_nib_lookup<7>(v, nib_lane);
}

// x^(8*16384*k) mod P, computed cooperatively by a full warp (lane j owns bit j of k).
__device__ __forceinline__ uint32_t warp_xpow_tiles(uint32_t k, uint32_t lane) {
  uint32_t v = ((k >> lane) & 1u) ? c_xpow_tiles[lane] : 0x80000000u;  // 0x80000000 == 1
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t other = __shfl_xor_sync(0xffffffffu, v, o);
    v = gf2_mulmod_dev(v, other);
  }
  return v;
}

template <int ALGO, int kStages>
__global__ void __launch_bounds__(kThreads, resident_ctas(kStages)) bb_xfer_kernel(const __grid_constant__ Params p) {
  using Smem = SmemT<ALGO, kStages>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  constexpr bool kBbh = (ALGO == ALGO_BBH64);
  constexpr bool kCrc = (ALGO == ALGO_CRC32C);
  constexpr bool kXxh = (ALGO == ALGO_XXH3);
  constexpr bool kSum = kBbh || kXxh;  // digest = finalize(commutative sum of per-tile terms)
  constexpr bool kHash = kBbh || kCrc || kXxh;

  const auto [t0, my_tiles] = cta_tile_run(p.total_tiles);

  // ------------------------------------------------------------------ setup
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&s.full[i], 1);
      mbar_init(&s.epi_done[i], 4);
      mbar_init(&s.empty[i], kHash ? 2 : 1);  // store warp (+ finalizer)
      s.dirty[i] = kTileBytes;
    }
    fence_mbar_init();
  }
  if constexpr (kBbh) {
    bbh_load_weights(s.w, threadIdx.x, kThreads);
    fence_proxy_async_smem();
  }
  if constexpr (kCrc) {
    uint32_t* dstt = &s.crc_t[0][0][0];
    for (uint32_t i = threadIdx.x; i < kNumCrcTabs * 1024; i += kThreads) dstt[i] = __ldg(&p.crc_tables[i]);
    __syncthreads();
    uint32_t* nibt = s.crc_nib + ((2048u - (smem_u32(s.crc_nib) & 2047u)) & 2047u) / 4u;
    for (uint32_t i = threadIdx.x; i < 8 * 16 * 32; i += kThreads) {  // [nibble j][value v][lane]
      const uint32_t j = i >> 9, v = (i >> 5) & 15u;
      nibt[i] = crc_shift(s.crc_t[T128], v << (4 * j));
    }
  }
  if constexpr (kXxh) {
    if (threadIdx.x < 48) {
      const uint32_t i = threadIdx.x;
      uint64_t v = 0;
      const uint32_t off = i < 24 ? 8u * min(i, 22u) : i < 32 ? xxh3::kSecretSize - xxh3::kStripe - xxh3::kLastAccStart + 8u * (i - 24)
                           : i < 40 ? xxh3::kSecretSize - xxh3::kStripe + 8u * (i - 32) : xxh3::kMergeStart + 8u * (i - 40);
      for (int b = 7; b >= 0; --b) v = (v << 8) | c_xxh_secret[off + b];
      s.xkey[i] = v;
    }
  }
  __syncthreads();

  if (warp == 0) {
    // ================================================================ TMA producer
    uint32_t it = 0;
    uint32_t g_desc = 0xFFFFFFFFu;  // descriptor whose source rows are in `gst`
    XferStride gst{1, 1, 0};
    for (uint32_t base = 0; base < my_tiles; base += 32) {
      const uint32_t idx = base + lane;
      if (idx < my_tiles) {
        const uint32_t t = t0 + idx;
        const DescTable<true> inl{p.inl_descs, p.inl_tile_start, p.ndesc};
        const DescTable<false> tab{p.descs, p.tile_start, p.ndesc};
        uint32_t lo, first, next;
        uint4 w[4];
        if (p.use_inline) {
          lo = inl.desc_of_tile(t), first = inl.start(lo), next = inl.start(lo + 1);
          inl.load(lo, w);
        } else {
          lo = tab.desc_of_tile(t), first = tab.start(lo), next = tab.start(lo + 1);
          tab.load(lo, w);
        }
        const XferDesc d = desc_from_words(w);
        LookupEntry& e = s.lk[lane];
        e.src = reinterpret_cast<uint64_t>(d.src);
        for (uint32_t r = 0; r < kMaxDst; ++r) e.m.dst[r] = reinterpret_cast<uint64_t>(d.dst[r]);
        e.m.nbytes = d.nbytes;
        e.m.expect = d.expect;
        e.m.desc = lo;
        e.m.tile_in_obj = t - first;
        e.m.ndst_flags = (d.ndst & 0xFFu) | (d.flags << 8);
        e.m.obj_ntiles = next - first;
        e.m.crc_unpad = d.reserved;
      }
      __syncwarp();
      const uint32_t cnt = min(32u, my_tiles - base);
      for (uint32_t i = 0; i < cnt; ++i, ++it) {
        const uint32_t stage = it % kStages;
        const uint32_t par = (it / kStages) & 1u;
        const LookupEntry& e = s.lk[i];
        const uint64_t src_i = e.src;
        const uint64_t off = static_cast<uint64_t>(e.m.tile_in_obj) * kTileBytes;
        const uint32_t bytes = static_cast<uint32_t>(min(static_cast<uint64_t>(kTileBytes), e.m.nbytes - off));
        const uint32_t b16 = bytes & ~15u;
        const uint32_t tail = bytes & 15u;
        const bool gather = (e.m.ndst_flags >> 8) & XFER_GATHER;
        mbar_wait(&s.empty[stage], par ^ 1u);
        bool wrote = false;
        if constexpr (kHash) {
          const uint32_t dirty = s.dirty[stage];
          for (uint32_t o = b16 + lane * 16; o < dirty; o += 512) {
            *reinterpret_cast<uint4*>(&s.tile[stage][o]) = make_uint4(0, 0, 0, 0);
            wrote = true;
          }
        }
        uint32_t tx = b16;  // bytes the stage's bulk loads deliver
        if (gather) {
          // one row segment per lane; the pad above may have zeroed the 16-byte chunk that holds a gathered tail, so the
          // gathered bytes are written after it
          __syncwarp();
          if (e.m.desc != g_desc) {
            g_desc = e.m.desc;
            if (p.use_inline) gst = p.inl_strides[g_desc];
            else gst = load_stride(p.strides, g_desc);
          }
          const uint32_t seg_tx = (e.m.ndst_flags >> 8) & XFER_PAGED
                                      ? gather_row_segments<true>(s.tile[stage], &s.full[stage], src_i, off, bytes, gst, lane)
                                      : gather_row_segments(s.tile[stage], &s.full[stage], src_i, off, bytes, gst, lane);
          tx = __reduce_add_sync(0xffffffffu, seg_tx);
          wrote = true;
        } else if (lane < tail) {
          s.tile[stage][b16 + lane] = *reinterpret_cast<const uint8_t*>(src_i + off + b16 + lane);
          wrote = true;
        }
        if (wrote) fence_proxy_async_smem();
        if (lane < 4) {
          uint4 v = reinterpret_cast<const uint4*>(&e.m)[lane];
          if (lane == 3) v.x = bytes;  // StageMeta::bytes is the first word of uint4 #3
          reinterpret_cast<uint4*>(&s.meta[stage])[lane] = v;
        }
        __syncwarp();
        if (lane == 0) {
          s.dirty[stage] = (bytes + 15u) & ~15u;
          mbar_arrive_expect_tx(&s.full[stage], tx);
          if (b16 && !gather) bulk_g2s(s.tile[stage], reinterpret_cast<const void*>(src_i + off), b16, &s.full[stage]);
          if (p.trace_d) p.trace_d[static_cast<uint64_t>(t0 + base + i) * 4 + 0] = globaltimer_ns();
        }
        __syncwarp();
      }
      __syncwarp();
    }
  } else if (warp == 1) {
    // idle: the BBH64 tensor-core product is issued by the epilogue warpgroup that consumes it
  } else if (warp == 2) {
    // ================================================================ store warp
    // Bulk async-groups belong to the thread that commits them: every lane commits one group per tile (empty unless the
    // lane stored a strided segment) and waits on its own groups before lane 0 releases the stage.
    uint32_t st_desc = 0xFFFFFFFFu;  // descriptor whose row pattern is in `st`
    XferStride st{1, 1, 0};
    for (uint32_t it = 0; it < my_tiles; ++it) {
      const uint32_t stage = it % kStages;
      const uint32_t par = (it / kStages) & 1u;
      mbar_wait(&s.full[stage], par);
      if (p.trace_d && lane == 0) p.trace_d[static_cast<uint64_t>(t0 + it) * 4 + 1] = globaltimer_ns();
      const StageMeta& m = s.meta[stage];
      const uint64_t off = static_cast<uint64_t>(m.tile_in_obj) * kTileBytes;
      const uint32_t ndst = m.ndst_flags & 0xFFu;
      const uint32_t flags = m.ndst_flags >> 8;
      const bool strided = flags & (XFER_STRIDED | XFER_SCATTER);
      // the whole tile, or its part inside the window [dst[1], dst[2]) (object offsets)
      const auto [x0, x1, a0, a1, h1, tb] = tile_span(off, m.bytes, flags & XFER_WINDOW, m.dst[1], m.dst[2]);
      if (strided) {
        // one row segment per lane (a tile can hold thousands of short rows): TMA middle, head and tail byte-wise; a
        // strided window's rows, or the destination rows of a scattering store
        if (m.desc != st_desc) {
          st_desc = m.desc;
          if (p.use_inline) st = p.inl_strides[st_desc];
          else st = load_stride(p.strides, st_desc);
        }
        if (flags & XFER_PAGED) scatter_row_segments<true>(s.tile[stage], m.dst[0], off, m.bytes, st, lane);
        else if (flags & XFER_SCATTER) scatter_row_segments(s.tile[stage], m.dst[0], off, m.bytes, st, lane);
        else store_row_segments(s.tile[stage], m.dst[0], off, x0, x1, st, lane);
      } else if (flags & XFER_MULTIMEM) {
        uint8_t* mc = reinterpret_cast<uint8_t*>(m.dst[0] + off);
        for (uint32_t o = a0 + lane * 16; o < a1; o += 512)
          multimem_st_v4(mc + o, *reinterpret_cast<const uint4*>(&s.tile[stage][o]));
      } else if (lane == 0) {
        for (uint32_t r = 0; r < ndst; ++r)
          if (a1 > a0) bulk_s2g(reinterpret_cast<void*>(m.dst[r] + off + a0), &s.tile[stage][a0], a1 - a0);
      }
      bulk_commit();
      if (p.trace_d && lane == 0) p.trace_d[static_cast<uint64_t>(t0 + it) * 4 + 2] = globaltimer_ns();
      const uint32_t o = lane < 16 ? x0 + lane : tb + (lane - 16u);
      if (!strided && o < (lane < 16 ? h1 : x1)) {
        const uint8_t b = s.tile[stage][o];
        for (uint32_t r = 0; r < ndst; ++r) *reinterpret_cast<uint8_t*>(m.dst[r] + off + o) = b;
      }
      if (it >= kStoreLag) bulk_wait_read<kStoreLag>();
      __syncwarp();
      if (it >= kStoreLag && lane == 0) {
        mbar_arrive(&s.empty[(it - kStoreLag) % kStages]);
        if (p.trace_d) p.trace_d[static_cast<uint64_t>(t0 + it - kStoreLag) * 4 + 3] = globaltimer_ns();
      }
    }
    bulk_wait_read<0>();
    __syncwarp();
    if (lane == 0) {
      const uint32_t first = my_tiles > kStoreLag ? my_tiles - kStoreLag : 0;
      for (uint32_t it = first; it < my_tiles; ++it) {
        mbar_arrive(&s.empty[it % kStages]);
        if (p.trace_d) p.trace_d[static_cast<uint64_t>(t0 + it) * 4 + 3] = globaltimer_ns();
      }
    }
    bulk_wait<0>();  // writes performed before the kernel retires
  } else if (warp == 3) {
    // ================================================================ finalizer
    if constexpr (kHash) {
      uint32_t cur_d = 0xFFFFFFFFu, cnt = 0;
      uint64_t acc = 0;
      // Folds one finished tile (its StageMeta `m` and the epilogue's partials) into the running per-object state and,
      // when this CTA's share of the object is complete, publishes / combines it.
      auto account = [&](uint32_t it, const StageMeta& m, uint64_t p0, uint64_t p1, uint64_t p2, uint64_t p3) {
        if (m.desc != cur_d) {
          cur_d = m.desc;
          acc = 0;
          cnt = 0;
        }
        if constexpr (kSum) acc += p0 + p1 + p2 + p3;
        ++cnt;
        const bool obj_end = (m.tile_in_obj + 1 == m.obj_ntiles);
        if (obj_end || it + 1 == my_tiles) {
          if constexpr (kCrc) {
            // The epilogue warps carry their per-lane accumulators across the tiles of an object and publish the
            // four quarter values only here: together they are the CRC polynomial of this CTA's whole run of it.
            const auto* t4k = s.crc_t[T4096];
            uint32_t t = crc_shift(t4k, static_cast<uint32_t>(p0)) ^ static_cast<uint32_t>(p1);
            t = crc_shift(t4k, t) ^ static_cast<uint32_t>(p2);
            t = crc_shift(t4k, t) ^ static_cast<uint32_t>(p3);
            acc = t;
          }
          // ---- this CTA's contribution to object cur_d is complete
          uint64_t digest = 0;
          bool have = false;
          const bool raw = kSum && ((m.ndst_flags >> 8) & XFER_RAW_SUM);
          if (cnt == m.obj_ntiles) {  // object lives entirely in this CTA: no atomics
            if constexpr (kSum) digest = raw ? acc : tchash::finalize(acc, m.nbytes);
            else digest = gf2_mulmod_dev(static_cast<uint32_t>(acc), m.crc_unpad) ^ static_cast<uint32_t>(m.expect >> 32) ^ 0xFFFFFFFFu;
            have = true;
          } else {
            uint64_t contrib = acc;
            if constexpr (kCrc) {
              const uint32_t after = m.obj_ntiles - 1u - m.tile_in_obj;  // tiles of this object after my run
              contrib = gf2_mulmod_dev(static_cast<uint32_t>(acc), warp_xpow_tiles(after, lane));
            }
            uint32_t prev = 0;
            if (lane == 0) {
              if constexpr (kSum) atomicAdd(&p.sum_ws[cur_d], static_cast<unsigned long long>(contrib));
              else atomicXor(&p.sum_ws[cur_d], static_cast<unsigned long long>(contrib));
              __threadfence();
              prev = atomicAdd(&p.done_ws[cur_d], cnt);
            }
            prev = __shfl_sync(0xffffffffu, prev, 0);
            if (prev + cnt == m.obj_ntiles) {  // last contributor finalises and re-zeroes
              if (lane == 0) {
                __threadfence();
                const uint64_t sum = atomicExch(&p.sum_ws[cur_d], 0ull);
                p.done_ws[cur_d] = 0;
                if constexpr (kSum) digest = raw ? sum : tchash::finalize(sum, m.nbytes);
                else digest = gf2_mulmod_dev(static_cast<uint32_t>(sum), m.crc_unpad) ^ static_cast<uint32_t>(m.expect >> 32) ^ 0xFFFFFFFFu;
              }
              have = true;
            }
          }
          if (have && lane == 0) {
            const uint64_t want = kSum ? m.expect : (m.expect & 0xFFFFFFFFull);
            p.digest_out[cur_d] = digest;
            p.status_out[cur_d] = (((m.ndst_flags >> 8) & XFER_VERIFY) && digest != want) ? 1u : 0u;
          }
          cur_d = 0xFFFFFFFFu;
        }
      };
      if constexpr (kXxh) {
        // XXH3: the epilogue warps left the 16 x 8 (block, lane) stripe sums of each tile in s.xs; what remains is the
        // serial part of the algorithm -- 15 scrambles per accumulator lane, then the merge.  The chain is latency bound
        // (~40 dependent cycles per step), so four tiles are chained at once, one per group of 8 lanes.
        const uint32_t g = lane >> 3, l8 = lane & 7u;
        const uint64_t skey = s.xkey[32 + l8], mkey = s.xkey[40 + l8];
        for (uint32_t it0 = 0; it0 < my_tiles; it0 += 4) {
          const uint32_t n = min(4u, my_tiles - it0);
          for (uint32_t j = 0; j < n; ++j) mbar_wait(&s.epi_done[(it0 + j) % kStages], ((it0 + j) / kStages) & 1u);
          const uint32_t st = (it0 + min(g, n - 1u)) % kStages;  // idle groups redo the last tile (their result is ignored)
          uint64_t a = xxh3::init_acc(l8);
#pragma unroll
          for (int b = 0; b < 15; ++b) a = xxh3::scramble(a + s.xs[st][b][l8], skey);
          a += s.xs[st][15][l8];
          const uint64_t nb = shfl_u64(a, static_cast<int>((lane + 1u) & 31u));  // the odd lane's accumulator and key
          const uint64_t nk = shfl_u64(mkey, static_cast<int>((lane + 1u) & 31u));
          uint64_t mg = (l8 & 1u) ? 0ull : xxh3::mul128_fold64(a ^ mkey, nb ^ nk);
          mg += shfl_xor_u64(mg, 2);
          mg += shfl_xor_u64(mg, 4);
          const uint64_t h = xxh3::avalanche(mg + static_cast<uint64_t>(kTileBytes) * xxh3::P64_1);  // XXH3_64bits(tile), in lanes l8 == 0
          __syncwarp();
          for (uint32_t j = 0; j < n; ++j) {
            const uint32_t stage = (it0 + j) % kStages;
            const StageMeta m = s.meta[stage];
            const uint64_t hj = shfl_u64(h, static_cast<int>(j * 8u));
            __syncwarp();
            if (lane == 0) mbar_arrive(&s.empty[stage]);
            const uint32_t ti = m.tile_in_obj + (((m.ndst_flags >> 8) & XFER_RAW_SUM) ? m.crc_unpad : 0u);
            account(it0 + j, m, tchash::mix64(hj + (static_cast<uint64_t>(ti) + 1ull) * tchash::kGold), 0, 0, 0);
          }
        }
      } else {
        for (uint32_t it = 0; it < my_tiles; ++it) {
          const uint32_t stage = it % kStages;
          const uint32_t par = (it / kStages) & 1u;
          mbar_wait(&s.epi_done[stage], par);
          const StageMeta m = s.meta[stage];
          const uint64_t p0 = s.part[stage][0], p1 = s.part[stage][1], p2 = s.part[stage][2], p3 = s.part[stage][3];
          __syncwarp();
          if (lane == 0) mbar_arrive(&s.empty[stage]);
          account(it, m, p0, p1, p2, p3);
        }
      }
    }
  } else {
    // ================================================================ epilogue warps 4..7
    if constexpr (kBbh) {
      const uint32_t q = warp & 3u;
      const uint32_t w_addr = smem_u32(s.w);
      for (uint32_t it = 0; it < my_tiles; ++it) {
        const uint32_t stage = it % kStages;
        const uint32_t par = (it / kStages) & 1u;
        mbar_wait(&s.full[stage], par);  // tile landed (TMA + the producer's fenced zero padding) and its StageMeta
        uint32_t d[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) d[k] = 0;
        bbh_tile_mma(smem_u32(s.tile[stage]), w_addr, d);
        // position of this tile in the hashed object (a RAW_SUM slice starts at a non-zero tile index)
        const uint32_t ti = s.meta[stage].tile_in_obj + (((s.meta[stage].ndst_flags >> 8) & XFER_RAW_SUM) ? s.meta[stage].crc_unpad : 0u);
        const uint64_t tot = bbh_tile_rows(d, c_col_mul, ti, q, lane);
        if (lane == 0) {
          s.part[stage][q] = tot;
          mbar_arrive(&s.epi_done[stage]);
        }
        if (p.debug_d) {
          uint32_t* o = p.debug_d + static_cast<uint64_t>(t0 + it) * tchash::kRows * tchash::kN;
#pragma unroll
          for (uint32_t k = 0; k < 16; ++k) o[bbh_acc_row(k, q, lane) * tchash::kN + bbh_acc_col(k, lane)] = d[k];
        }
      }
    } else if constexpr (kXxh) {
      // XXH3 stripe sums.  A block's 16 stripe contributions do not depend on the accumulator, so all 16 x 8 (block,
      // lane) sums of the tile are computed at once: quarter-warp = one 1 KiB block, thread = (lane pair, half of the
      // stripes), one LDS.128 per stripe = the two 8-byte lanes of the pair (so the "swap" addend stays in the thread).
      // The odd half visits its stripes shifted by one: the 8 threads of a quarter then cover all 32 banks every time.
      const uint32_t e = threadIdx.x - 128u;
      const uint32_t blk = (e >> 5) * 4u + ((e & 31u) >> 3);
      const uint32_t pair = (e >> 1) & 3u, half = e & 1u;
      for (uint32_t it = 0; it < my_tiles; ++it) {
        const uint32_t stage = it % kStages;
        const uint32_t par = (it / kStages) & 1u;
        mbar_wait(&s.full[stage], par);
        const uint8_t* base = &s.tile[stage][blk * 1024u + pair * 16u];
        uint64_t s0 = 0, s1 = 0;
#pragma unroll
        for (uint32_t k = 0; k < 8; ++k) {
          const uint32_t stp = half * 8u + ((k + half) & 7u);
          const uint4 d = *reinterpret_cast<const uint4*>(base + stp * 64u);
          const uint64_t dv0 = (static_cast<uint64_t>(d.y) << 32) | d.x, dv1 = (static_cast<uint64_t>(d.w) << 32) | d.z;
          const uint32_t ki = (blk == 15u && stp == 15u) ? 24u + 2u * pair : stp + 2u * pair;  // the tile's very last stripe has its own key
          const uint64_t q0 = dv0 ^ s.xkey[ki], q1 = dv1 ^ s.xkey[ki + 1u];
          s0 += static_cast<uint64_t>(static_cast<uint32_t>(q0)) * (q0 >> 32) + dv1;
          s1 += static_cast<uint64_t>(static_cast<uint32_t>(q1)) * (q1 >> 32) + dv0;
        }
        s0 += shfl_xor_u64(s0, 1);
        s1 += shfl_xor_u64(s1, 1);
        if (half == 0u) {
          s.xs[stage][blk][2u * pair] = s0;
          s.xs[stage][blk][2u * pair + 1u] = s1;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&s.epi_done[stage]);
      }
    } else if constexpr (kCrc) {
      // Quarter q of every tile, lane l: words l, l+32, ... (bank-conflict free); consecutive words of a lane are
      // 128 B apart -> one x^(8*128) shift per step through the lane-private nibble tables.  Four independent Horner
      // chains per lane (kCrcChains x kCrcChainRows rows) hide the latency of the dependent lookups, and the chains
      // run on ACROSS the tiles of an object (a chain's next row in the following tile is 16384 - (kCrcChainRows-1)*128 bytes
      // further), so the lane / chain / quarter combine is paid once per object and CTA, not once per tile.
      const uint32_t q = warp & 3u;
      const uint32_t nib_lane = ((smem_u32(s.crc_nib) + 2047u) & ~2047u) + lane * 4u;  // bits 7-10 clear
      const auto* tj = s.crc_t[TJUMP];
      uint32_t a[kCrcChains];
#pragma unroll
      for (int c = 0; c < kCrcChains; ++c) a[c] = 0;
      for (uint32_t it = 0; it < my_tiles; ++it) {
        const uint32_t stage = it % kStages;
        const uint32_t par = (it / kStages) & 1u;
        mbar_wait(&s.full[stage], par);  // also acquires the producer's StageMeta writes
        const uint32_t tio = s.meta[stage].tile_in_obj;
        const bool fresh = (it == 0) || (tio == 0);
        const bool flush = (tio + 1 == s.meta[stage].obj_ntiles) || (it + 1 == my_tiles);
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(&s.tile[stage][q * 4096]) + lane;
        if (fresh) {
#pragma unroll
          for (int c = 0; c < kCrcChains; ++c) a[c] = wp[c * kCrcChainRows * 32];
        } else {
#pragma unroll
          for (int c = 0; c < kCrcChains; ++c) a[c] = crc_shift(tj, a[c]) ^ wp[c * kCrcChainRows * 32];
        }
#pragma unroll
        for (int i = 1; i < kCrcChainRows; ++i) {
#pragma unroll
          for (int c = 0; c < kCrcChains; ++c) a[c] = crc_nib_shift(a[c], nib_lane) ^ wp[(c * kCrcChainRows + i) * 32];
        }
        if (flush) {
          const auto* tc = s.crc_t[TCHAIN];  // chains are kCrcChainRows rows of 128 B apart
          uint32_t v = a[0];
#pragma unroll
          for (int c = 1; c < kCrcChains; ++c) v = crc_shift(tc, v) ^ a[c];
          // combine lanes: value(l) covers bytes [4l, 4l+4) of each 128-byte row group
          uint32_t o;
          o = __shfl_down_sync(0xffffffffu, v, 1);  v = crc_shift(s.crc_t[T4], v) ^ o;
          o = __shfl_down_sync(0xffffffffu, v, 2);  v = crc_shift(s.crc_t[T8], v) ^ o;
          o = __shfl_down_sync(0xffffffffu, v, 4);  v = crc_shift(s.crc_t[T16], v) ^ o;
          o = __shfl_down_sync(0xffffffffu, v, 8);  v = crc_shift(s.crc_t[T32], v) ^ o;
          o = __shfl_down_sync(0xffffffffu, v, 16); v = crc_shift(s.crc_t[T64], v) ^ o;
          if (lane == 0) s.part[stage][q] = crc_shift(s.crc_t[T4], v);  // the CRC's final x^32 factor
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&s.epi_done[stage]);
      }
    }
  }

}

PerDeviceOnce g_consts;      // __constant__ uploads
PerDeviceOnce g_crc_once;    // CRC32C shift tables, on the first CRC32C launch
uint32_t* g_crc_tables[kMaxDevices] = {};

template <int ALGO>
using SmemOf = SmemT<ALGO, kStagesFor<ALGO>>;
template <int ALGO>
constexpr auto kKernelOf = bb_xfer_kernel<ALGO, kStagesFor<ALGO>>;

// Two CTAs per SM: 227 KiB of shared memory per SM for blocks, each block also reserving 1 KiB for the system.
template <int ALGO>
constexpr bool fits_resident = resident_ctas(kStagesFor<ALGO>) * (sizeof(SmemOf<ALGO>) + 1024) <= 228 * 1024;
static_assert(fits_resident<ALGO_NONE> && fits_resident<ALGO_CRC32C> && fits_resident<ALGO_XXH3> && fits_resident<ALGO_BBH64>);

template <int ALGO>
cudaError_t launch_t(int dev, const Params& p, int grid, cudaStream_t st) {
  const cudaError_t e = set_max_dynamic_smem_once<kKernelOf<ALGO>>(dev, static_cast<int>(sizeof(SmemOf<ALGO>)));
  if (e != cudaSuccess) return e;
  kKernelOf<ALGO><<<grid, kThreads, sizeof(SmemOf<ALGO>), st>>>(p);
  return cudaGetLastError();
}

template <int ALGO>
int resident_t(int dev) {
  int n = 0;
  if (set_max_dynamic_smem_once<kKernelOf<ALGO>>(dev, static_cast<int>(sizeof(SmemOf<ALGO>))) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kKernelOf<ALGO>, kThreads, sizeof(SmemOf<ALGO>)) != cudaSuccess)
    return -1;
  return n;
}

}  // namespace

int xfer_smem_bytes(int algo) {
  switch (algo) {
    case ALGO_NONE: return static_cast<int>(sizeof(SmemOf<ALGO_NONE>));
    case ALGO_CRC32C: return static_cast<int>(sizeof(SmemOf<ALGO_CRC32C>));
    case ALGO_XXH3: return static_cast<int>(sizeof(SmemOf<ALGO_XXH3>));
    default: return static_cast<int>(sizeof(SmemOf<ALGO_BBH64>));
  }
}

XferGeometry xfer_geometry(int algo, uint32_t total_tiles, int max_ctas) {
  static const int env_ctas = [] { const char* e = std::getenv("BB_XFER_CTAS"); return e ? std::atoi(e) : 0; }();
  const bool crc = algo == ALGO_CRC32C;
  XferGeometry g;
  g.stages = crc ? kStagesFor<ALGO_CRC32C> : kStagesFor<ALGO_XXH3>;
  g.smem_bytes = xfer_smem_bytes(algo);
  if (total_tiles == 0) return g;
  const uint64_t sms = static_cast<uint64_t>(current_sm_count());
  uint64_t grid;
  if (max_ctas > 0 || env_ctas > 0) grid = static_cast<uint64_t>(max_ctas > 0 ? max_ctas : env_ctas);
  else if (crc) grid = sms;  // one persistent CTA per SM
  else grid = std::max(std::min(sms * resident_ctas(g.stages), uint64_t{total_tiles}), (uint64_t{total_tiles} + kRunTiles - 1) / kRunTiles);
  grid = std::min<uint64_t>(grid, total_tiles);
  // cta_tile_run gives every CTA ceil(total / grid) tiles: launch only the CTAs that get any
  const uint64_t tpc = (total_tiles + grid - 1) / grid;
  g.grid = static_cast<int>((total_tiles + tpc - 1) / tpc);
  return g;
}

int xfer_resident_ctas(int algo) {
  int dev = 0;
  if (current_device(&dev) != cudaSuccess) return -1;
  switch (algo) {
    case ALGO_NONE: return resident_t<ALGO_NONE>(dev);
    case ALGO_CRC32C: return resident_t<ALGO_CRC32C>(dev);
    case ALGO_XXH3: return resident_t<ALGO_XXH3>(dev);
    default: return resident_t<ALGO_BBH64>(dev);
  }
}

uint32_t crc_unpad_for(uint64_t nbytes) {
  // x^(-8*pad) mod P where pad = zero bytes appended to reach a whole number of tiles.
  // Memoised per pad value (pad < 16384): batches of equal-size objects pay one table hit.
  const uint32_t pad = static_cast<uint32_t>((kTileBytes - (nbytes % kTileBytes)) % kTileBytes);
  static std::mutex mu;
  static std::vector<uint32_t> cache(kTileBytes, 0);  // 0 is never a valid power of x
  {
    std::lock_guard<std::mutex> lk(mu);
    if (cache[pad]) return cache[pad];
  }
  // x^-1 in reflected form: reverse one LFSR bit-step.  Forward: v -> (v>>1) ^ (v&1 ? P : 0);
  // a set top bit means the step XORed P in, so v_prev = ((v ^ P) << 1) | 1.
  static const uint32_t xinv8 = [] {
    uint32_t v = 0x80000000u;  // 1
    for (int i = 0; i < 8; ++i) v = (v & 0x80000000u) ? (((v ^ 0x82F63B78u) << 1) | 1u) : (v << 1);
    return v;  // x^-8
  }();
  uint32_t result = 0x80000000u, base = xinv8;
  for (uint32_t e = pad; e; e >>= 1) {
    if (e & 1) result = gf2_mulmod(result, base);
    base = gf2_mulmod(base, base);
  }
  std::lock_guard<std::mutex> lk(mu);
  cache[pad] = result;
  return result;
}

uint32_t crc_init_term_for(uint64_t nbytes) {
  static std::mutex mu;
  static std::unordered_map<uint64_t, uint32_t> cache;
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(nbytes);
    if (it != cache.end()) return it->second;
  }
  const uint32_t v = gf2_mulmod(0xFFFFFFFFu, gf2_xpow_bytes(nbytes));
  std::lock_guard<std::mutex> lk(mu);
  if (cache.size() > 65536) cache.clear();
  cache.emplace(nbytes, v);
  return v;
}

int launch_xfer(const XferLaunch& l) {
  if (l.ndesc == 0 || l.total_tiles == 0) return 0;
  if (l.small_path && !l.debug_d && !l.trace_d) return launch_xfer_small(l);
  int dev = 0;
  cudaError_t e = current_device(&dev);
  if (e != cudaSuccess) return static_cast<int>(e);
  e = g_consts.run(dev, [] {
    uint64_t h[tchash::kN];
    for (uint32_t n = 0; n < tchash::kN; ++n) h[n] = tchash::col_mul(n);
    cudaError_t e = cudaMemcpyToSymbol(c_col_mul, h, sizeof h);
    if (e != cudaSuccess) return e;
    uint32_t xp[32];
    uint32_t b = gf2_xpow_bytes(kTileBytes);
    for (int j = 0; j < 32; ++j) {
      xp[j] = b;
      b = gf2_mulmod(b, b);
    }
    e = cudaMemcpyToSymbol(c_xpow_tiles, xp, sizeof xp);
    if (e != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_xxh_secret, xxh3::kSecret, sizeof xxh3::kSecret);
  });
  if (e != cudaSuccess) return static_cast<int>(e);
  if (l.algo == ALGO_CRC32C) {
    e = g_crc_once.run(dev, [dev] {
      static uint32_t host_t[kNumCrcTabs][4][256];  // under g_crc_once's lock
      for (int t = 0; t < kNumCrcTabs; ++t) crc32c_shift_table(kCrcTabBytes[t], host_t[t]);
      cudaError_t e = cudaSuccess;
      if (!g_crc_tables[dev] && (e = cudaMalloc(reinterpret_cast<void**>(&g_crc_tables[dev]), sizeof host_t)) != cudaSuccess) return e;
      return cudaMemcpy(g_crc_tables[dev], host_t, sizeof host_t, cudaMemcpyHostToDevice);
    });
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  Params p;
  p.descs = l.descs;
  p.tile_start = l.tile_start;
  p.use_inline = 0;
  if (l.host_descs && l.ndesc <= kInlineDescs) {
    p.use_inline = 1;
    std::memcpy(p.inl_descs, l.host_descs, l.ndesc * sizeof(XferDesc));
    std::memcpy(p.inl_tile_start, l.host_tile_start, (l.ndesc + 1) * sizeof(uint32_t));
    if (l.host_strides) std::memcpy(p.inl_strides, l.host_strides, l.ndesc * sizeof(XferStride));
  }
  p.strides = l.strides;
  p.ndesc = l.ndesc;
  p.total_tiles = l.total_tiles;
  p.sum_ws = reinterpret_cast<unsigned long long*>(l.sum_ws);
  p.done_ws = l.done_ws;
  p.digest_out = l.digest_out;
  p.status_out = l.status_out;
  p.crc_tables = g_crc_tables[dev];
  p.debug_d = l.debug_d;
  p.trace_d = reinterpret_cast<unsigned long long*>(l.trace_d);
  const int grid = xfer_geometry(l.algo, l.total_tiles, l.max_ctas).grid;
  cudaStream_t st = static_cast<cudaStream_t>(l.stream);
  switch (l.algo) {
    case ALGO_NONE: e = launch_t<ALGO_NONE>(dev, p, grid, st); break;
    case ALGO_CRC32C: e = launch_t<ALGO_CRC32C>(dev, p, grid, st); break;
    case ALGO_BBH64: e = launch_t<ALGO_BBH64>(dev, p, grid, st); break;
    case ALGO_XXH3: e = launch_t<ALGO_XXH3>(dev, p, grid, st); break;
    default: return static_cast<int>(cudaErrorNotSupported);
  }
  return static_cast<int>(e);
}

}  // namespace bb::gpu
