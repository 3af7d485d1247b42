// bb_xfer_small: the small-object latency tier of the fused transfer (SURVEY K2, §7.4 #1).
//
// The reference's only end-to-end client moves a 64-byte object with one `ucp_put_nbx` + flush and one `ucp_get_nbx`
// (clients/ucx_client.cpp:188-257).  For objects of <= 4 KiB the persistent TMA / wgmma pipeline of bb_xfer_kernel is
// all set-up cost (mbarriers, weight matrix, tile padding), so batches made
// of small objects only take this path instead: ONE WARP PER OBJECT, no shared-memory staging of the payload, no TMA.
//
//   lane l owns bytes [128 l, 128 l + 128) of the object: 8 x LDG.128 (local HBM, peer slab over NVLink, or pinned host)
//   -> registers -> 8 x STG.128 to 1..3 destinations (local / peer-mapped), or multimem.st to an NVLS multicast window.
//   The digest is computed on the registers and is bit-identical to the big kernel's (the Keystone cannot tell which
//   path wrote an object):
//     BBH64  : the tile product D = A.W is evaluated with dp4a against the same weight matrix (packed in shared memory);
//              lane l holds K-chunk (l & 7) of rows (l >> 3) * 8 + j, partial row hashes are combined by shuffles;
//     CRC32C : each lane runs the word-at-a-time table CRC over its 128 bytes, lanes are combined with per-lane
//              x^(8*distance) multipliers in GF(2)[x]/P (same "raw remainder, un-pad, init term" algebra and the same
//              GF(2) multiply, xfer_common.cuh, as the big kernel).
//   A put of 4096 objects is 512 CTAs x 8 warps in one launch; a single put/get is one warp.
#include <cuda_runtime.h>

#include <cstring>

#include "common/checksum.h"
#include "common/tchash_def.h"
#include "common/xxh3.h"
#include "kernels/ptx.cuh"
#include "kernels/xfer.h"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {
namespace {

using namespace bb::ptx;

constexpr int kWarpsPerCta = 8;

// XXH3: [0..23] accumulate keys (word = stripe + lane), [24..31] scramble keys, [32..39] merge keys, [40..47] the stripe sum of
// an all-zero block per lane (blocks 4..14 of a <= 4 KiB object), [48..55] the same for the tile's last block (its last
// stripe has its own key)
__constant__ uint64_t c_xxh[56];
__constant__ uint32_t c_lane_mul[32];  // x^(8 * (128 * (31 - l) + 12288)) mod P: lane l's segment -> position in a 16 KiB tile

struct SmallParams {
  const XferDesc* descs;
  uint32_t ndesc;
  uint32_t use_inline;
  uint64_t* digest_out;
  uint32_t* status_out;
  const uint32_t* crc_t4;  // [4][256] shift-by-4-bytes table
  uint64_t zero_rows;      // BBH64: sum of the contributions of the all-zero rows 32..127 of tile 0
  // Completion by flag (latency path): status_out lives in pinned host memory, was preset to kSmallPending by the host,
  // and is written LAST, after a system-scope fence that orders it behind the object's peer / local stores -- the host
  // spins on it instead of recording and waiting for a CUDA event (which costs more than this whole kernel).
  uint32_t flag_mode;
  XferDesc inl_descs[kInlineDescs];
};

// The per-object work of one warp: load (<= 4 KiB, lane l owns bytes [128 l, 128 l + 128)), store to the destinations, digest on
// the registers.  Shared by the batch kernel (one warp per descriptor) and the mailbox kernel (one resident warp).
// s_w / s_t4 / s_xk: shared-memory tables of the algorithm (BBH64 packed weights, CRC32C x^32 table, XXH3 accumulate keys).
// VOL: the caller is a resident kernel -- source loads must bypass L1 (`ld.volatile`): a line cached by an earlier request for
// the same address would otherwise be served stale (L1 is only invalidated at kernel boundaries).
template <int ALGO, bool VOL>
__device__ __forceinline__ void small_object(uint64_t src, const uint64_t (&dst)[kMaxDst], uint32_t ndst, uint64_t nbytes, uint64_t expect,
                                             uint32_t flags, uint32_t reserved, uint32_t lane, uint64_t zero_rows, const uint32_t* s_w,
                                             const uint32_t* s_t4, const uint64_t* s_xk, uint64_t* digest_out, uint32_t* status_out) {
  const uint32_t n = static_cast<uint32_t>(nbytes);  // <= kSmallBytes (host checked)
  // ---- load: lane's 128-byte segment, zero beyond the object
  // Zero first, then ONLY predicated loads: with an `else v[j] = 0` after each load, the zeroing of the lanes past the object
  // writes the register the other lanes' load is still filling, the scoreboard makes it wait, and the eight loads of a lane
  // go out one round trip after the other -- 256 B ... 2 KiB gets over NVLink took 10 us longer than 4 KiB ones.
  uint4 v[8];
  const uint32_t seg = lane * 128u;
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t o = seg + 16u * j;
    if (o + 16u <= n) {
      if constexpr (VOL) {
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[j].x), "=r"(v[j].y), "=r"(v[j].z), "=r"(v[j].w) : "l"(src + o) : "memory");
      } else {
        v[j] = ld_nc_v4(reinterpret_cast<const void*>(src + o));
      }
    }
  }
  if (n & 15u) {  // the one partial 16-byte chunk of the object (byte loads), owned by exactly one (lane, j)
    const uint32_t po = n & ~15u;
    if (po >= seg && po < seg + 128u) {
      uint32_t w[4] = {0, 0, 0, 0};
      for (uint32_t b = 0; b < n - po; ++b)
        w[b >> 2] |= static_cast<uint32_t>(*reinterpret_cast<const volatile uint8_t*>(src + po + b)) << (8u * (b & 3u));
      const uint32_t pj = (po - seg) >> 4;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (static_cast<uint32_t>(j) == pj) v[j] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  // ---- store
  if (flags & XFER_MULTIMEM) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t o = seg + 16u * j;
      if (o + 16u <= n) multimem_st_v4(reinterpret_cast<void*>(dst[0] + o), v[j]);
    }
  } else {
    for (uint32_t r = 0; r < ndst; ++r) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t o = seg + 16u * j;
        if (o + 16u <= n) {
          st_na_v4(reinterpret_cast<void*>(dst[r] + o), v[j]);
        } else if (o < n) {
          const uint32_t w[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
          for (uint32_t b = 0; b < n - o; ++b)
            *reinterpret_cast<uint8_t*>(dst[r] + o + b) = static_cast<uint8_t>(w[b >> 2] >> (8u * (b & 3u)));
        }
      }
    }
  }
  if constexpr (ALGO == ALGO_NONE) {
    *digest_out = 0;
    *status_out = 0;
    return;
  }

  // ---- digest on the registers
  uint64_t digest = 0;
  if constexpr (ALGO == ALGO_BBH64) {
    // tile offset o = 128 lane + 16 j  ->  row (lane >> 3) * 8 + j,  K chunk kc = lane & 7 (k = 16 kc + byte)
    const uint32_t kc = lane & 7u;
    uint64_t rr[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) rr[j] = 0;
#pragma unroll
    for (uint32_t nn = 0; nn < 16; ++nn) {
      const uint32_t w0 = s_w[nn * 32 + kc * 4 + 0], w1 = s_w[nn * 32 + kc * 4 + 1], w2 = s_w[nn * 32 + kc * 4 + 2],
                     w3 = s_w[nn * 32 + kc * 4 + 3];
      const uint64_t kn = tchash::col_mul(nn);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t dp = __dp4a(v[j].x, w0, 0u);
        dp = __dp4a(v[j].y, w1, dp);
        dp = __dp4a(v[j].z, w2, dp);
        dp = __dp4a(v[j].w, w3, dp);
        rr[j] += static_cast<uint64_t>(dp) * kn;
      }
    }
    // the 8 K chunks of a row sit in the 8 lanes of a group: add them up, then lane (group, j == lane & 7) owns row j
    uint64_t mine = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint64_t t = rr[j];
      t += shfl_xor_u64(t, 1);
      t += shfl_xor_u64(t, 2);
      t += shfl_xor_u64(t, 4);
      if (static_cast<uint32_t>(j) == kc) mine = t;
    }
    const uint32_t row = (lane >> 3) * 8u + kc;
    uint64_t c = tchash::row_contrib(mine, row);  // tile index 0
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += shfl_xor_u64(c, o);
    digest = tchash::finalize(c + zero_rows, nbytes);
  } else if constexpr (ALGO == ALGO_XXH3) {
    // Standard XXH3-64 of the object zero padded to one 16 KiB tile.  Lane l holds stripes 2 (l & 7) and 2 (l & 7) + 1 of
    // block l >> 3 (64 B each = the 8 accumulator lanes): it forms the 8 per-lane products of both stripes, the 8 lanes
    // of a block group are summed by a reduce-scatter (7 exchanges), after which lane l owns stripe-sum [block l >> 3]
    // [acc lane l & 7] -- exactly what the scramble chain of acc lane (l & 7) wants to pull in, block after block.
    uint64_t S[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) S[i] = 0;
    const uint32_t st0 = 2u * (lane & 7u);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {  // v[4h + q] = acc lanes 2q, 2q + 1 of stripe st0 + h
        const uint4 d = v[4 * h + q];
        const uint64_t dv0 = (static_cast<uint64_t>(d.y) << 32) | d.x, dv1 = (static_cast<uint64_t>(d.w) << 32) | d.z;
        const uint64_t q0 = dv0 ^ s_xk[st0 + h + 2 * q], q1 = dv1 ^ s_xk[st0 + h + 2 * q + 1];
        S[2 * q] += static_cast<uint64_t>(static_cast<uint32_t>(q0)) * (q0 >> 32) + dv1;
        S[2 * q + 1] += static_cast<uint64_t>(static_cast<uint32_t>(q1)) * (q1 >> 32) + dv0;
      }
    }
    uint64_t m4[4], m2[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint64_t keep = (lane & 4u) ? S[i + 4] : S[i], send = (lane & 4u) ? S[i] : S[i + 4];
      m4[i] = keep + shfl_xor_u64(send, 4);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint64_t keep = (lane & 2u) ? m4[i + 2] : m4[i], send = (lane & 2u) ? m4[i] : m4[i + 2];
      m2[i] = keep + shfl_xor_u64(send, 2);
    }
    const uint64_t tot = ((lane & 1u) ? m2[1] : m2[0]) + shfl_xor_u64((lane & 1u) ? m2[0] : m2[1], 1);  // [block lane >> 3][acc lane & 7]
    const uint32_t l8 = lane & 7u;
    uint64_t a = xxh3::init_acc(l8);
    const uint64_t skey = c_xxh[24 + l8], zero_blk = c_xxh[40 + l8];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      a = xxh3::scramble(a + shfl_u64(tot, static_cast<int>(l8 + 8u * b)), skey);
    }
#pragma unroll
    for (int b = 4; b < 15; ++b) a = xxh3::scramble(a + zero_blk, skey);
    a += c_xxh[48 + l8];
    const uint64_t mkey = c_xxh[32 + l8];
    const uint64_t nb = shfl_u64(a, static_cast<int>((lane + 1u) & 31u));
    uint64_t mg = (l8 & 1u) ? 0ull : xxh3::mul128_fold64(a ^ mkey, nb ^ c_xxh[32 + ((l8 + 1u) & 7u)]);
    mg += shfl_xor_u64(mg, 2);
    mg += shfl_xor_u64(mg, 4);
    const uint64_t h = xxh3::avalanche(mg + static_cast<uint64_t>(kTileBytes) * xxh3::P64_1);
    digest = tchash::finalize(tchash::mix64(h + tchash::kGold), nbytes);  // tile index 0
  } else {
    // CRC32C raw remainder of the lane's 128 bytes (x^32 factor included), word at a time through the x^32 shift table
    uint32_t s = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t w[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t t = s ^ w[q];
        s = s_t4[t & 0xFFu] ^ s_t4[256 + ((t >> 8) & 0xFFu)] ^ s_t4[512 + ((t >> 16) & 0xFFu)] ^ s_t4[768 + (t >> 24)];
      }
    }
    // place the segment inside a zero-padded 16 KiB tile and add the lanes up (XOR)
    uint32_t acc = gf2_mulmod_dev(s, c_lane_mul[lane]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc ^= __shfl_xor_sync(0xffffffffu, acc, o);
    digest = gf2_mulmod_dev(acc, reserved) ^ static_cast<uint32_t>(expect >> 32) ^ 0xFFFFFFFFu;
    expect &= 0xFFFFFFFFull;
  }
  *digest_out = digest;
  *status_out = ((flags & XFER_VERIFY) && digest != expect) ? 1u : 0u;
}

template <int ALGO>
__global__ void __launch_bounds__(kWarpsPerCta * 32) bb_xfer_small_kernel(const __grid_constant__ SmallParams p) {
  __shared__ uint32_t s_w[ALGO == ALGO_BBH64 ? 16 * 32 : 1];       // Wp[n][w]: W[4w + b][n] in byte b
  __shared__ uint32_t s_t4[ALGO == ALGO_CRC32C ? 4 * 256 : 1];
  __shared__ uint64_t s_xk[ALGO == ALGO_XXH3 ? 24 : 1];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  if constexpr (ALGO == ALGO_BBH64) {
    for (uint32_t i = threadIdx.x; i < 16 * 32; i += blockDim.x) {
      const uint32_t n = i >> 5, w = i & 31u;
      s_w[i] = tchash::weight(4 * w, n) | (tchash::weight(4 * w + 1, n) << 8) | (tchash::weight(4 * w + 2, n) << 16) |
               (tchash::weight(4 * w + 3, n) << 24);
    }
    __syncthreads();
  }
  if constexpr (ALGO == ALGO_CRC32C) {
    for (uint32_t i = threadIdx.x; i < 4 * 256; i += blockDim.x) s_t4[i] = __ldg(&p.crc_t4[i]);
    __syncthreads();
  }
  if constexpr (ALGO == ALGO_XXH3) {
    if (threadIdx.x < 24) s_xk[threadIdx.x] = c_xxh[threadIdx.x];
    __syncthreads();
  }
  const uint32_t d = blockIdx.x * kWarpsPerCta + warp;
  if (d >= p.ndesc) return;
  // ---- descriptor (every lane reads the same words: broadcast)
  const XferDesc q = p.use_inline ? DescTable<true>{p.inl_descs, nullptr, p.ndesc}[d] : DescTable<false>{p.descs, nullptr, p.ndesc}[d];
  const uint64_t dst[kMaxDst] = {reinterpret_cast<uint64_t>(q.dst[0]), reinterpret_cast<uint64_t>(q.dst[1]), reinterpret_cast<uint64_t>(q.dst[2])};
  uint64_t digest = 0;
  uint32_t status = 0;
  small_object<ALGO, false>(reinterpret_cast<uint64_t>(q.src), dst, q.ndst, q.nbytes, q.expect, q.flags, q.reserved, lane, p.zero_rows, s_w, s_t4, s_xk, &digest, &status);
  if (p.flag_mode) {
    __threadfence_system();  // every lane: its stores of the payload are performed system-wide ...
    __syncwarp();            // ... before lane 0 publishes the result
  }
  if (lane == 0) {
    if (ALGO != ALGO_NONE || p.flag_mode) p.digest_out[d] = digest;
    if (p.flag_mode) __threadfence_system();
    if (ALGO != ALGO_NONE || p.flag_mode) *reinterpret_cast<volatile uint32_t*>(&p.status_out[d]) = status;
  }
}

// ================================================================ the mailbox: a resident warp instead of a launch
// A single small put / get through the batch kernel costs a kernel launch: ~8.9 us on this box before anything else
// (profiles/r2_nvlink/README.md).  The mailbox kernel removes the launch from the steady state: ONE warp stays resident and
// polls a ring of 64-byte request slots in pinned host memory (one PCIe read per poll, ~1.4 us); the host posts a request by
// filling a slot and writing its sequence number last, the warp runs small_object() on it and writes digest + status +
// sequence number into the matching result slot (pinned), which the host spins on.  The kernel *lingers*: it exits by itself
// after `linger_ns` without a request (and unconditionally after `max_ns`), announcing it in MailCtl, so cudaDeviceSynchronize
// and friends never wait longer than that; the next request simply launches it again (and that launch carries the request).
__device__ __forceinline__ uint32_t ld_sys_u32(const volatile uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(32) bb_mailbox_kernel(const MailSlot* slots, MailResult* results, MailCtl* ctl, uint32_t first_seq,
                                                        uint32_t epoch, uint64_t linger_ns, uint64_t max_ns, const uint32_t* crc_t4,
                                                        uint64_t zero_rows) {
  __shared__ uint32_t s_w[16 * 32];
  __shared__ uint32_t s_t4[4 * 256];
  __shared__ uint64_t s_xk[24];
  const uint32_t lane = threadIdx.x;
  for (uint32_t i = lane; i < 16 * 32; i += 32) {
    const uint32_t n = i >> 5, w = i & 31u;
    s_w[i] = tchash::weight(4 * w, n) | (tchash::weight(4 * w + 1, n) << 8) | (tchash::weight(4 * w + 2, n) << 16) | (tchash::weight(4 * w + 3, n) << 24);
  }
  for (uint32_t i = lane; i < 4 * 256; i += 32) s_t4[i] = __ldg(&crc_t4[i]);
  if (lane < 24) s_xk[lane] = c_xxh[lane];
  __syncwarp();
  uint32_t seq = first_seq;
  const uint64_t t_start = globaltimer_ns();
  uint64_t t_last = t_start;
  while (true) {
    // one 64-byte read of the slot (16 lanes x 4 B, a single PCIe request = a consistent snapshot of the cache line);
    // word 15 is the sequence number the host writes last
    const volatile uint32_t* sp = reinterpret_cast<const volatile uint32_t*>(&slots[seq % kMailSlots]);
    const uint32_t word = lane < 16 ? ld_sys_u32(sp + lane) : 0u;
    if (__shfl_sync(0xffffffffu, word, 15) != seq) {
      const uint64_t now = globaltimer_ns();
      if (now - t_last > linger_ns || now - t_start > max_ns) break;
      continue;
    }
    auto w64 = [&](int i) {
      const uint32_t lo = __shfl_sync(0xffffffffu, word, i), hi = __shfl_sync(0xffffffffu, word, i + 1);
      return (static_cast<uint64_t>(hi) << 32) | lo;
    };
    const uint64_t src = w64(0);
    const uint64_t dst[kMaxDst] = {w64(2), 0, 0};
    const uint64_t expect = w64(4);
    const uint32_t nbytes = __shfl_sync(0xffffffffu, word, 6), flags = __shfl_sync(0xffffffffu, word, 7);
    const uint32_t algo = __shfl_sync(0xffffffffu, word, 8), reserved = __shfl_sync(0xffffffffu, word, 9);
    uint64_t digest = 0;
    uint32_t status = 0;
    switch (algo) {
      case ALGO_XXH3: small_object<ALGO_XXH3, true>(src, dst, 1, nbytes, expect, flags, reserved, lane, zero_rows, s_w, s_t4, s_xk, &digest, &status); break;
      case ALGO_BBH64: small_object<ALGO_BBH64, true>(src, dst, 1, nbytes, expect, flags, reserved, lane, zero_rows, s_w, s_t4, s_xk, &digest, &status); break;
      case ALGO_CRC32C: small_object<ALGO_CRC32C, true>(src, dst, 1, nbytes, expect, flags, reserved, lane, zero_rows, s_w, s_t4, s_xk, &digest, &status); break;
      default: small_object<ALGO_NONE, true>(src, dst, 1, nbytes, expect, flags, reserved, lane, zero_rows, s_w, s_t4, s_xk, &digest, &status); break;
    }
    __threadfence_system();  // the object's stores (peer slab / local / host) are performed before the result says so
    __syncwarp();
    if (lane == 0) {
      // digest, status and the sequence number leave as ONE 16-byte store = one PCIe write into one cache line of the pinned
      // result ring: the host that sees the new `seq` sees the digest of the same write (no second system fence, which costs
      // a PCIe round trip)
      MailResult* r = &results[seq % kMailSlots];
      asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(r), "r"(static_cast<uint32_t>(digest)),
                   "r"(static_cast<uint32_t>(digest >> 32)), "r"(status), "r"(seq)
                   : "memory");
    }
    ++seq;
    t_last = globaltimer_ns();
  }
  if (lane == 0) {  // tell the host this incarnation is gone (posted writes stay in order: results first, then this)
    __threadfence_system();
    *reinterpret_cast<volatile uint32_t*>(&ctl->next_seq) = seq;
    __threadfence_system();
    *reinterpret_cast<volatile uint32_t*>(&ctl->exit_epoch) = epoch;
  }
}

struct SmallTables {
  uint32_t* t4 = nullptr;
  uint64_t zero_rows = 0;
};
SmallTables g_small[kMaxDevices];
PerDeviceOnce g_small_once;

// The current device's tables, made (and the __constant__ tables uploaded) on first use.
int ensure_small_state(SmallTables** out) {
  int dev = 0;
  cudaError_t e = current_device(&dev);
  if (e != cudaSuccess) return static_cast<int>(e);
  SmallTables& st = g_small[dev];
  e = g_small_once.run(dev, [&st] {
    uint32_t mul[32];
    for (uint32_t ln = 0; ln < 32; ++ln) mul[ln] = gf2_xpow_bytes(128ull * (31 - ln) + (kTileBytes - kSmallBytes));
    cudaError_t e = cudaMemcpyToSymbol(c_lane_mul, mul, sizeof mul);
    if (e != cudaSuccess) return e;
    uint32_t t4[4][256];
    crc32c_shift_table(4, t4);
    if (!st.t4 && (e = cudaMalloc(reinterpret_cast<void**>(&st.t4), sizeof t4)) != cudaSuccess) return e;
    e = cudaMemcpy(st.t4, t4, sizeof t4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return e;
    uint64_t z = 0;
    for (uint32_t m = kSmallBytes / 128; m < tchash::kRows; ++m) z += tchash::row_contrib(0, m);
    st.zero_rows = z;
    uint64_t xk[56] = {};
    for (uint32_t i = 0; i < 23; ++i) xk[i] = xxh3::secret64(8 * i);
    for (uint32_t i = 0; i < 8; ++i) {
      xk[24 + i] = xxh3::scramble_key(i);
      xk[32 + i] = xxh3::merge_key(i);
      uint64_t zsum = 0, zlast = 0;
      for (uint32_t sidx = 0; sidx < 16; ++sidx) {
        const uint64_t k = xxh3::stripe_key(sidx, i);
        zsum += static_cast<uint64_t>(static_cast<uint32_t>(k)) * (k >> 32);
        if (sidx < 15) zlast += static_cast<uint64_t>(static_cast<uint32_t>(k)) * (k >> 32);
      }
      const uint64_t lk = xxh3::last_key(i);
      zlast += static_cast<uint64_t>(static_cast<uint32_t>(lk)) * (lk >> 32);
      xk[40 + i] = zsum;
      xk[48 + i] = zlast;
    }
    return cudaMemcpyToSymbol(c_xxh, xk, sizeof xk);
  });
  if (e != cudaSuccess) return static_cast<int>(e);
  *out = &st;
  return 0;
}
}  // namespace

int launch_mailbox(const MailSlot* slots, MailResult* results, MailCtl* ctl, uint32_t first_seq, uint32_t epoch, uint64_t linger_ns,
                   uint64_t max_ns, void* stream) {
  SmallTables* st = nullptr;
  if (const int rc = ensure_small_state(&st)) return rc;
  bb_mailbox_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(slots, results, ctl, first_seq, epoch, linger_ns, max_ns, st->t4, st->zero_rows);
  return static_cast<int>(cudaGetLastError());
}

int launch_xfer_small(const XferLaunch& l) {
  if (l.ndesc == 0) return 0;
  SmallTables* st = nullptr;
  if (const int rc = ensure_small_state(&st)) return rc;
  SmallParams p;
  p.descs = l.descs;
  p.ndesc = l.ndesc;
  p.use_inline = 0;
  if (l.host_descs && l.ndesc <= kInlineDescs) {
    p.use_inline = 1;
    std::memcpy(p.inl_descs, l.host_descs, l.ndesc * sizeof(XferDesc));
  }
  p.digest_out = l.digest_out;
  p.status_out = l.status_out;
  p.crc_t4 = st->t4;
  p.zero_rows = st->zero_rows;
  p.flag_mode = l.flag_completion ? 1u : 0u;
  const int grid = static_cast<int>((l.ndesc + kWarpsPerCta - 1) / kWarpsPerCta);
  const int threads = l.ndesc < static_cast<uint32_t>(kWarpsPerCta) ? static_cast<int>(l.ndesc) * 32 : kWarpsPerCta * 32;
  cudaStream_t s = static_cast<cudaStream_t>(l.stream);
  switch (l.algo) {
    case ALGO_NONE: bb_xfer_small_kernel<ALGO_NONE><<<grid, threads, 0, s>>>(p); break;
    case ALGO_CRC32C: bb_xfer_small_kernel<ALGO_CRC32C><<<grid, threads, 0, s>>>(p); break;
    case ALGO_BBH64: bb_xfer_small_kernel<ALGO_BBH64><<<grid, threads, 0, s>>>(p); break;
    case ALGO_XXH3: bb_xfer_small_kernel<ALGO_XXH3><<<grid, threads, 0, s>>>(p); break;
    default: return static_cast<int>(cudaErrorNotSupported);
  }
  return static_cast<int>(cudaGetLastError());
}

}  // namespace bb::gpu
