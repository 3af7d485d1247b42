// bb_xfer_fp8: fused MXFP8 transfer kernels (sm_90a; SURVEY K12 "fp8 pack fused into put / unpack into get").
//
//   put  (PACK)   : TMA loads a 32 KiB bf16 tile -> 8 pack warps compute the E8M0 block scales and the E4M3
//                   payload *in shared memory* (the chunk codec of mxfp8.cuh, which the stand-alone kernels use
//                   too) -> the 16 KiB payload tile is hashed in place by wgmma (BBH64, same tile hash as
//                   bb_xfer) -> TMA stores payload + 512 B of scales to the
//                   (peer) slab -- to up to 3 replicas of the object from the one converted tile.  The bf16 data
//                   is read from HBM once and only the 0.52x packed bytes cross NVLink (once per replica).
//                   With XFER_GATHER (puts of a sliced tensor) the producer fills the bf16 tile from the source rows,
//                   one row segment per lane, by the rule of SourceRows (common/store_window.h) in bf16 bytes, so the
//                   tile, the packed object and its digest are those of a put of the compacted rows.  With
//                   XFER_GATHER | XFER_PAGED (puts of the blocks of a paged cache) the row segments are the pages of
//                   SourcePages in wide bytes, each read from the address in the page table, so the tile is that
//                   of the concatenated pages; an MX block may straddle two pages, the codec never sees it.  With
//                   XFER_GATHER | XFER_SEGMENTS (puts of a list of tensors) the lanes take the segments of the
//                   SourceSegments table that overlap the tile, in wide bytes, so the tile is that of the concatenated
//                   segments and an MX block may straddle two segments the same way.
//   get  (UNPACK) : TMA loads payload tile + scales from the slab -> tensor-core hash of the payload tile ->
//                   8 unpack warps expand to bf16 in shared memory -> TMA stores the 32 KiB tile to the caller.
//                   With XFER_WINDOW (element-range gets) only the bf16 bytes [win.lo, win.hi) of the object are
//                   stored, object byte x at dst[0] + x; every tile is still loaded and hashed, so the digest is the
//                   whole object's, and tiles outside the window are not unpacked.  With XFER_STRIDED as well
//                   (slices along an inner dimension) the store warp stores only the window's row segments, densely,
//                   one per lane, by the same rule as bb_xfer; a tile wholly inside a gap between rows is still unpacked.
//                   With XFER_SCATTER instead (gets into a sliced tensor) the store warp stores every 32 KiB bf16 tile
//                   as the row segments of the destination rows, by the SourceRows rule in bf16 bytes, as bb_xfer does;
//                   with XFER_SCATTER | XFER_PAGED (gets into the blocks of a paged cache) as the segments of the
//                   destination pages, by the SourcePages rule in wide bytes; with XFER_SCATTER | XFER_SEGMENTS (gets
//                   into a list of tensors) as the tile's parts of the destination segments, a null segment not stored.
//
// The stored object keeps the layout of the unfused path ([E4M3 payload n][E8M0 scales n/32], common/mxfp8.h), and so
// does its digest: BBH64 is a sum of per-tile terms, this kernel accumulates the payload tiles (tile index 0..T-1)
// and returns the *unfinalised* sum per object; the scales region (tiles T..) is hashed as an XFER_RAW_SUM slice
// by bb_xfer and the host adds the two sums and finalises.  Objects hold any multiple of 32 elements: a tail tile is
// converted and stored like the others (its scale bytes past the last 16-byte multiple go byte-wise) but not hashed
// here -- in the packed object its hash tile also contains the first scale bytes, so the slice the host hashes simply
// starts at the last whole payload tile.
//
// Warp roles (24 warps): 0 producer, 1 idle, 2 store, 3 accumulator, 4-7 epilogue (the warpgroup issues the wgmma
// tile product, bbh_tile.cuh, and turns its register accumulators into row hashes), 8-23 convert (pack / unpack).  Two shared-memory rings: 3 x 32 KiB bf16 tiles and 6 x (16 KiB payload + 512 B scales).
#include <cuda_runtime.h>

#include <algorithm>

#include "common/tchash_def.h"
#include "kernels/bbh_tile.cuh"
#include "kernels/mxfp8.cuh"
#include "kernels/ptx.cuh"
#include "kernels/xfer.h"
#include "kernels/xfer_common.cuh"

namespace bb::gpu {
namespace {

using namespace bb::ptx;

constexpr int kConvertWarps = 16;           // warps 8..23 (the pack side is ALU bound: ncu issue-active 51 % with 8)
constexpr int kFpThreads = (8 + kConvertWarps) * 32;
constexpr uint32_t kScaleBytes = kTileBytes / 32;

// One instantiation per wide element size WB: 2 (bf16, and fp16 by XFER_WIDE_F16) or 4 (fp32).  A wide tile is the
// WB * 16 KiB of one 16 KiB payload tile, so the fp32 rings are shorter: 3 wide + 6 payload stages would not fit.
template <uint32_t WB>
struct FpCfg {
  static constexpr int kWideStages = WB == 2 ? 3 : 2;  // ring of WB * 16 KiB wide tiles
  static constexpr int kTileStages = WB == 2 ? 6 : 4;  // ring of 16 KiB payload tiles (+ 512 B scales)
  static constexpr uint32_t kWideBytes = WB * kTileBytes;  // wide side of one payload tile
};
constexpr int kFpStoreLag = 1;

__constant__ uint64_t c_fp_col_mul[tchash::kN];

struct FpMeta {            // 64 bytes
  uint64_t dst[kMaxDst];   // pack: this tile's payload address in every replica; unpack: dst[0] = the tile's bf16
                           // destination, dst[1..2] = the object's store window [lo, hi) in bf16 bytes
  int64_t scales_delta;    // pack: (tile's scales address) - (tile's payload address), the same in every replica
  uint32_t desc;
  uint32_t tile_in_obj;
  uint32_t obj_ntiles;
  uint32_t ndst;           // pack: replicas written by this pass (1..kMaxDst)
  uint32_t valid;          // payload bytes (= elements) of this tile: 16384, or the multiple-of-32 tail of the object
  uint32_t strided;        // unpack: XFER_STRIDED when the descriptor's window is strided, XFER_SCATTER when its
                           // destination is rows; pack: XFER_GATHER when its source is rows (the pattern in
                           // FpParams::strides either way); XFER_PAGED as well when those rows are pages,
                           // and XFER_PAGE_ROWS when the pages are in-page rows, or XFER_SEGMENTS when they are the
                           // segments of a table; unpack: XFER_WINDOW_ROWS when the window's result lands in rows
                           // (with XFER_STRIDED for a strided window)
  uint32_t f16;            // XFER_WIDE_F16: the wide side is fp16 (2-byte instantiation only)
  uint32_t pad;
};
static_assert(sizeof(FpMeta) == 64);

struct FpLookup {
  FpMeta m;
  uint64_t src;         // pack: bf16 source; unpack: payload source
  uint64_t src_scales;  // unpack: scales source
};

// Two rings: the wide ring only spans load -> convert (pack) or convert -> store (unpack), the payload
// ring spans convert/load -> tensor-core hash -> store/accumulate.  Decoupling them lets 3 + 6 slots cover a
// pipeline that would need 6 x 48.5 KiB as one ring (bf16 / fp16; fp32: 2 + 4).
template <uint32_t WB, int kWideStages = FpCfg<WB>::kWideStages, int kTileStages = FpCfg<WB>::kTileStages>
struct __align__(1024) SmemFp {
  static constexpr uint32_t kWideBytes = FpCfg<WB>::kWideBytes;
  uint8_t tile[kTileStages][kTileBytes];
  uint8_t wide[kWideStages][kWideBytes];
  uint8_t scales[kTileStages][kScaleBytes];
  uint8_t w[2048];
  uint64_t t_full[kTileStages];   // payload tile + scales ready (pack: convert warps; unpack: TMA)
  uint64_t t_empty[kTileStages];
  uint64_t w_full[kWideStages];   // wide tile ready (pack: TMA; unpack: convert warps)
  uint64_t w_empty[kWideStages];
  uint64_t epi_done[kTileStages];
  FpMeta t_meta[kTileStages];
  FpMeta w_meta[kWideStages];
  uint64_t part[kTileStages][4];
  FpLookup lk[32];
};
// 227 KiB: the opt-in dynamic shared memory of one sm_90 CTA
static_assert(sizeof(SmemFp<2>) <= 227 * 1024 && sizeof(SmemFp<4>) <= 227 * 1024, "SmemFp exceeds the shared memory of one CTA");

struct FpParams {
  const XferDesc* descs;
  const uint32_t* tile_start;
  uint32_t ndesc;
  uint32_t total_tiles;
  unsigned long long* sum_ws;  // [ndesc] raw BBH64 sums of the payload tiles (zero on entry)
  const XferStride* strides;   // row patterns of the XFER_STRIDED / XFER_SCATTER (unpack) or XFER_GATHER (pack) descriptors
                               // (XferLaunch::strides), else null
};

template <bool UNPACK, uint32_t WB>
__global__ void __launch_bounds__(kFpThreads, 1) bb_xfer_fp8_kernel(const __grid_constant__ FpParams p) {
  constexpr int kWideStages = FpCfg<WB>::kWideStages;
  constexpr int kTileStages = FpCfg<WB>::kTileStages;
  constexpr uint32_t kWideBytes = FpCfg<WB>::kWideBytes;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  SmemFp<WB>& s = *reinterpret_cast<SmemFp<WB>*>(smem_raw);
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t lane = threadIdx.x & 31u;

  const auto [t0, my_tiles] = cta_tile_run(p.total_tiles);

  if (threadIdx.x == 0) {
    for (int i = 0; i < kTileStages; ++i) {
      mbar_init(&s.t_full[i], UNPACK ? 1 : kConvertWarps);
      mbar_init(&s.t_empty[i], UNPACK ? kConvertWarps + 1 : 2);  // unpack: convert warps + accumulator; pack: store + accumulator
      mbar_init(&s.epi_done[i], 4);
    }
    for (int i = 0; i < kWideStages; ++i) {
      mbar_init(&s.w_full[i], UNPACK ? kConvertWarps : 1);
      mbar_init(&s.w_empty[i], UNPACK ? 1 : kConvertWarps);
    }
    fence_mbar_init();
  }
  bbh_load_weights(s.w, threadIdx.x, kFpThreads);
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 0) {
    // ================================================================ TMA producer
    uint32_t it = 0;
    uint32_t g_desc = 0xFFFFFFFFu;  // pack: descriptor whose source rows are in `gst`
    XferStride gst{1, 1, 0};
    for (uint32_t base = 0; base < my_tiles; base += 32) {
      const uint32_t idx = base + lane;
      if (idx < my_tiles) {
        const uint32_t t = t0 + idx;
        const DescTable<false> tab{p.descs, p.tile_start, p.ndesc};
        const uint32_t lo = tab.desc_of_tile(t);
        const uint32_t first = tab.start(lo);
        const uint32_t next = tab.start(lo + 1);
        const XferDesc d = tab[lo];
        const uint64_t src = reinterpret_cast<uint64_t>(d.src), d0 = reinterpret_cast<uint64_t>(d.dst[0]),
                       d1 = reinterpret_cast<uint64_t>(d.dst[1]), d2 = reinterpret_cast<uint64_t>(d.dst[2]);
        const uint64_t nbytes = d.nbytes;  // payload bytes == elements
        const uint32_t ti = t - first;
        FpLookup& e = s.lk[lane];
        e.m.desc = lo;
        e.m.tile_in_obj = ti;
        e.m.obj_ntiles = next - first;
        e.m.strided = d.flags & (UNPACK ? XFER_STRIDED | XFER_SCATTER | XFER_PAGED | XFER_PAGE_ROWS | XFER_WINDOW_ROWS | XFER_SEGMENTS
                                        : XFER_GATHER | XFER_PAGED | XFER_PAGE_ROWS | XFER_SEGMENTS);
        e.m.f16 = d.flags & XFER_WIDE_F16;
        e.m.pad = 0;
        e.m.valid = static_cast<uint32_t>(min(static_cast<uint64_t>(kTileBytes), nbytes - static_cast<uint64_t>(ti) * kTileBytes));
        // the packed object is [payload nbytes][scales nbytes/32]: a tile's scales sit (nbytes - ti*(16384-512)) past its payload
        e.m.scales_delta = static_cast<int64_t>(nbytes) - static_cast<int64_t>(ti) * static_cast<int64_t>(kTileBytes - kScaleBytes);
        if constexpr (UNPACK) {
          e.src = src + static_cast<uint64_t>(ti) * kTileBytes;  // payload tile in the slab
          e.src_scales = e.src + e.m.scales_delta;               // its scales
          e.m.dst[0] = d0 + static_cast<uint64_t>(ti) * kWideBytes;  // wide destination
          // store window in wide bytes of the object (XferDesc::win); a whole-object get stores [0, 2^64), i.e. every tile whole
          const bool win = d.flags & XFER_WINDOW;
          e.m.dst[1] = win ? d1 : 0;
          e.m.dst[2] = win ? d2 : ~0ull;
          e.m.ndst = 1;
        } else {
          // wide source tile; for a gathering load the pattern's row 0 (the tile's rows are found from its object offset)
          e.src = e.m.strided ? src : src + static_cast<uint64_t>(ti) * kWideBytes;
          e.src_scales = 0;
          e.m.dst[0] = d0 + static_cast<uint64_t>(ti) * kTileBytes;
          e.m.dst[1] = d1 + static_cast<uint64_t>(ti) * kTileBytes;
          e.m.dst[2] = d2 + static_cast<uint64_t>(ti) * kTileBytes;
          e.m.ndst = min(max(d.ndst, 1u), kMaxDst);
        }
      }
      __syncwarp();
      const uint32_t cnt = min(32u, my_tiles - base);
      for (uint32_t i = 0; i < cnt; ++i, ++it) {
        const FpLookup& e = s.lk[i];
        if constexpr (UNPACK) {
          const uint32_t ts = it % kTileStages, tp = (it / kTileStages) & 1u;
          mbar_wait(&s.t_empty[ts], tp ^ 1u);
          if (lane < 4) reinterpret_cast<uint4*>(&s.t_meta[ts])[lane] = reinterpret_cast<const uint4*>(&e.m)[lane];
          __syncwarp();
          // a tail tile carries valid/32 scale bytes: the 16-byte multiple by TMA, the rest byte-wise
          const uint32_t sb = e.m.valid / 32u, sb16 = sb & ~15u;
          if (lane < (sb & 15u)) s.scales[ts][sb16 + lane] = *reinterpret_cast<const uint8_t*>(e.src_scales + sb16 + lane);
          __syncwarp();
          if (lane == 0) {
            mbar_arrive_expect_tx(&s.t_full[ts], e.m.valid + sb16);
            bulk_g2s(s.tile[ts], reinterpret_cast<const void*>(e.src), e.m.valid, &s.t_full[ts]);
            if (sb16) bulk_g2s(s.scales[ts], reinterpret_cast<const void*>(e.src_scales), sb16, &s.t_full[ts]);
          }
        } else {
          const uint32_t ws = it % kWideStages, wp = (it / kWideStages) & 1u;
          mbar_wait(&s.w_empty[ws], wp ^ 1u);
          if (lane < 4) reinterpret_cast<uint4*>(&s.w_meta[ws])[lane] = reinterpret_cast<const uint4*>(&e.m)[lane];
          uint32_t tx = WB * e.m.valid;  // bytes the stage's bulk loads deliver
          if (e.m.strided) {
            // Gathering load (XFER_GATHER): one source row segment per lane, so the wide tile is byte for byte the tile of
            // the compacted rows.  A short last tile needs no zero pad: only its `valid` elements are stored, and it is
            // not hashed here.  The lanes' head and tail bytes are generic shared stores read only by the convert warps'
            // generic loads (no TMA store or wgmma reads the wide tile), so no async-proxy fence: the __syncwarp below
            // orders them before lane 0's arrive (release), and the convert warps' wait on w_full (acquire) orders that
            // before their loads.
            if (e.m.desc != g_desc) {
              g_desc = e.m.desc;
              gst = load_stride(p.strides, g_desc);
            }
            // XFER_PAGED: the rows are the pages of the table in gst, e.src is not read
            const uint64_t off = static_cast<uint64_t>(e.m.tile_in_obj) * kWideBytes;
            // XFER_PAGE_ROWS: their in-page rows, whose pattern is read here so that `gst` stays three words
            // XFER_SEGMENTS: the segments of the table in gst that overlap the tile
            const uint32_t seg_tx =
                e.m.strided & XFER_SEGMENTS    ? gather_row_segments<false, false, true>(s.wide[ws], &s.w_full[ws], e.src, off, WB * e.m.valid, gst, lane)
                : e.m.strided & XFER_PAGE_ROWS ? gather_row_segments<true, true>(s.wide[ws], &s.w_full[ws], e.src, off, WB * e.m.valid,
                                                                               load_stride(p.strides, g_desc, true), lane)
                : e.m.strided & XFER_PAGED   ? gather_row_segments<true>(s.wide[ws], &s.w_full[ws], e.src, off, WB * e.m.valid, gst, lane)
                                             : gather_row_segments(s.wide[ws], &s.w_full[ws], e.src, off, WB * e.m.valid, gst, lane);
            tx = __reduce_add_sync(0xffffffffu, seg_tx);
          }
          __syncwarp();
          if (lane == 0) {
            mbar_arrive_expect_tx(&s.w_full[ws], tx);
            if (!e.m.strided) bulk_g2s(s.wide[ws], reinterpret_cast<const void*>(e.src), WB * e.m.valid, &s.w_full[ws]);
          }
        }
        __syncwarp();
      }
      __syncwarp();
    }
  } else if (warp == 1) {
    // idle: the tensor-core hash of the payload tile is issued by the epilogue warpgroup that consumes it
  } else if (warp == 2) {
    // ================================================================ store warp
    // Bulk async-groups belong to the thread that commits them: every lane commits one group per tile (empty unless the
    // lane stored something by TMA) and waits on its own groups before lane 0 releases the slot.
    constexpr int kRing = UNPACK ? kWideStages : kTileStages;
    uint32_t pat_desc = 0xFFFFFFFFu;  // unpack: descriptor whose row pattern is in `pat`
    XferStride pat{1, 1, 0};
    for (uint32_t it = 0; it < my_tiles; ++it) {
      const uint32_t st = it % kRing, par = (it / kRing) & 1u;
      if constexpr (UNPACK) {
        mbar_wait(&s.w_full[st], par);
        const FpMeta& m = s.w_meta[st];
        // the tile's wide bytes inside the store window: the middle by TMA, head and tail byte-wise (as bb_xfer does); a
        // strided window (XFER_STRIDED) cuts them further to its row segments, one per lane
        const uint64_t off = static_cast<uint64_t>(m.tile_in_obj) * kWideBytes;
        const auto [x0, x1, a0, a1, h1, tb] = tile_span(off, WB * m.valid, true, m.dst[1], m.dst[2]);
        if (m.strided) {
          if (m.desc != pat_desc) {
            pat_desc = m.desc;
            pat = load_stride(p.strides, pat_desc);
          }
          // m.dst[0] = dst[0] + off; a scattering store has no window, so [x0, x1) is the whole tile.  A paged or segmented
          // one stores into the pages or segments of the table in `pat` and does not read dst[0].
          if (m.strided & XFER_WINDOW_ROWS)  // the window's segments cut at the destination rows of the dense result
            store_window_rows(s.wide[st], m.dst[0] - off, off, x0, x1, m.dst[1], m.strided & XFER_STRIDED,
                              load_stride(p.strides, m.desc, true), lane);
          else if (m.strided & XFER_SEGMENTS) scatter_row_segments<false, false, true>(s.wide[st], m.dst[0] - off, off, x1, pat, lane);
          else if (m.strided & XFER_PAGE_ROWS)
            scatter_row_segments<true, true>(s.wide[st], m.dst[0] - off, off, x1, load_stride(p.strides, pat_desc, true), lane);
          else if (m.strided & XFER_PAGED) scatter_row_segments<true>(s.wide[st], m.dst[0] - off, off, x1, pat, lane);
          else if (m.strided & XFER_SCATTER) scatter_row_segments(s.wide[st], m.dst[0] - off, off, x1, pat, lane);
          else store_row_segments(s.wide[st], m.dst[0] - off, off, x0, x1, pat, lane);
        } else {
          if (lane == 0 && a1 > a0) bulk_s2g(reinterpret_cast<void*>(m.dst[0] + a0), &s.wide[st][a0], a1 - a0);
          const uint32_t o = lane < 16 ? x0 + lane : tb + (lane - 16u);
          if (o < (lane < 16 ? h1 : x1)) *reinterpret_cast<uint8_t*>(m.dst[0] + o) = s.wide[st][o];
        }
      } else {
        mbar_wait(&s.t_full[st], par);
        const FpMeta& m = s.t_meta[st];
        const uint32_t sb = m.valid / 32u, sb16 = sb & ~15u;
        if (lane == 0) {
          for (uint32_t r = 0; r < m.ndst; ++r) {  // replica fan-out: converted once, stored to every copy
            bulk_s2g(reinterpret_cast<void*>(m.dst[r]), s.tile[st], m.valid);
            if (sb16) bulk_s2g(reinterpret_cast<void*>(m.dst[r] + m.scales_delta), s.scales[st], sb16);
          }
        }
        if (lane < (sb & 15u)) {  // tail tile: the scale bytes past the last 16-byte multiple
          const uint8_t v = s.scales[st][sb16 + lane];
          for (uint32_t r = 0; r < m.ndst; ++r) *reinterpret_cast<uint8_t*>(m.dst[r] + m.scales_delta + sb16 + lane) = v;
        }
      }
      bulk_commit();
      if (it >= kFpStoreLag) bulk_wait_read<kFpStoreLag>();
      __syncwarp();
      if (it >= kFpStoreLag && lane == 0) {
        if constexpr (UNPACK) mbar_arrive(&s.w_empty[(it - kFpStoreLag) % kRing]);
        else mbar_arrive(&s.t_empty[(it - kFpStoreLag) % kRing]);
      }
    }
    bulk_wait_read<0>();
    __syncwarp();
    if (lane == 0) {
      const uint32_t first = my_tiles > kFpStoreLag ? my_tiles - kFpStoreLag : 0;
      for (uint32_t it = first; it < my_tiles; ++it) {
        if constexpr (UNPACK) mbar_arrive(&s.w_empty[it % kRing]);
        else mbar_arrive(&s.t_empty[it % kRing]);
      }
    }
    bulk_wait<0>();  // writes performed before the kernel retires
  } else if (warp == 3) {
    // ================================================================ accumulator: per-object raw sums
    uint32_t cur_d = 0xFFFFFFFFu;
    uint64_t acc = 0;
    for (uint32_t it = 0; it < my_tiles; ++it) {
      const uint32_t ts = it % kTileStages, tp = (it / kTileStages) & 1u;
      mbar_wait(&s.epi_done[ts], tp);
      const uint32_t d = s.t_meta[ts].desc;
      // A tail tile holds payload AND the first scale bytes of the packed object's hash tile: it is hashed from the
      // stored bytes as part of the host's RAW_SUM slice, not here.
      const uint64_t sum = s.t_meta[ts].valid == kTileBytes ? s.part[ts][0] + s.part[ts][1] + s.part[ts][2] + s.part[ts][3] : 0;
      __syncwarp();
      if (lane == 0) mbar_arrive(&s.t_empty[ts]);
      if (d != cur_d) {
        if (cur_d != 0xFFFFFFFFu && lane == 0) atomicAdd(&p.sum_ws[cur_d], static_cast<unsigned long long>(acc));
        cur_d = d;
        acc = 0;
      }
      acc += sum;
    }
    if (cur_d != 0xFFFFFFFFu && lane == 0) atomicAdd(&p.sum_ws[cur_d], static_cast<unsigned long long>(acc));
  } else if (warp < 8) {
    // ================================================================ epilogue warpgroup 4..7: wgmma -> row hashes
    const uint32_t q = warp & 3u;
    const uint32_t w_addr = smem_u32(s.w);
    for (uint32_t it = 0; it < my_tiles; ++it) {
      const uint32_t ts = it % kTileStages, tp = (it / kTileStages) & 1u;
      mbar_wait(&s.t_full[ts], tp);  // pack: written by the convert warps (generic proxy, fenced); unpack: TMA
      uint32_t d[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) d[k] = 0;
      bbh_tile_mma(smem_u32(s.tile[ts]), w_addr, d);
      const uint64_t tot = bbh_tile_rows(d, c_fp_col_mul, s.t_meta[ts].tile_in_obj, q, lane);
      if (lane == 0) {
        s.part[ts][q] = tot;
        mbar_arrive(&s.epi_done[ts]);
      }
    }
  } else {
    // ================================================================ convert warps 8..15
    const uint32_t cw = warp - 8;  // convert warp: chunks [cw*kPer, (cw+1)*kPer) of the tile's 2048 chunks of 8 elements
    constexpr uint32_t kPer = 2048 / kConvertWarps;
    for (uint32_t it = 0; it < my_tiles; ++it) {
      const uint32_t ts = it % kTileStages, tp = (it / kTileStages) & 1u;
      const uint32_t ws = it % kWideStages, wp = (it / kWideStages) & 1u;
      if constexpr (UNPACK) {
        mbar_wait(&s.t_full[ts], tp);         // payload + scales landed
        mbar_wait(&s.w_empty[ws], wp ^ 1u);   // wide slot drained by the store warp
        const FpMeta& m = s.t_meta[ts];
        // a tile outside the store window is hashed (epilogue) but neither unpacked nor stored; one that overlaps it is
        // unpacked whole.  The barrier arrivals below are the same for every tile.
        const TileSpan sp = tile_span(static_cast<uint64_t>(m.tile_in_obj) * kWideBytes, WB * m.valid, true, m.dst[1], m.dst[2]);
        const uint2* pay = reinterpret_cast<const uint2*>(s.tile[ts]);
        uint4* out = reinterpret_cast<uint4*>(s.wide[ws]);
        const bool f16 = m.f16;
        if (sp.x1 > sp.x0) {
#pragma unroll 4
          for (uint32_t k = 0; k < kPer / 32; ++k) {
            const uint32_t c = cw * kPer + k * 32 + lane;
            unpack_wide_chunk<WB>(pay[c], s.scales[ts][c >> 2], f16, out, c);
          }
        }
        if (cw == 0 && lane < 4) reinterpret_cast<uint4*>(&s.w_meta[ws])[lane] = reinterpret_cast<const uint4*>(&s.t_meta[ts])[lane];
        fence_proxy_async_smem();  // generic-proxy writes -> TMA store
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&s.w_full[ws]);
          mbar_arrive(&s.t_empty[ts]);
        }
      } else {
        mbar_wait(&s.w_full[ws], wp);         // wide tile landed
        mbar_wait(&s.t_empty[ts], tp ^ 1u);   // payload slot released by store + accumulator
        const uint4* in = reinterpret_cast<const uint4*>(s.wide[ws]);
        uint2* pay = reinterpret_cast<uint2*>(s.tile[ts]);
        const bool f16 = s.w_meta[ws].f16;
#pragma unroll 4
        for (uint32_t k = 0; k < kPer / 32; ++k) {
          const uint32_t c = cw * kPer + k * 32 + lane;
          pack_wide_chunk<WB>(in, c, f16, &pay[c], &s.scales[ts][c >> 2], (c & 3u) == 0);
        }
        if (cw == 0 && lane < 4) reinterpret_cast<uint4*>(&s.t_meta[ts])[lane] = reinterpret_cast<const uint4*>(&s.w_meta[ws])[lane];
        fence_proxy_async_smem();  // generic-proxy writes -> tensor core / TMA store readers
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&s.t_full[ts]);
          mbar_arrive(&s.w_empty[ws]);
        }
      }
    }
  }

}

PerDeviceOnce g_fp_consts;  // __constant__ uploads

}  // namespace

int xfer_fp8_smem_bytes(uint32_t wide_bytes) {
  return static_cast<int>(wide_bytes == 4 ? sizeof(SmemFp<4>) : sizeof(SmemFp<2>));
}

template <bool UNPACK, uint32_t WB>
static cudaError_t launch_fp8_kernel(int dev, int grid, const FpParams& p, cudaStream_t st) {
  const cudaError_t e = set_max_dynamic_smem_once<bb_xfer_fp8_kernel<UNPACK, WB>>(dev, static_cast<int>(sizeof(SmemFp<WB>)));
  if (e != cudaSuccess) return e;
  bb_xfer_fp8_kernel<UNPACK, WB><<<grid, kFpThreads, sizeof(SmemFp<WB>), st>>>(p);
  return cudaGetLastError();
}

int launch_xfer_fp8(const XferLaunch& l, bool unpack, uint32_t wide_bytes) {
  if (wide_bytes != 2 && wide_bytes != 4) return static_cast<int>(cudaErrorInvalidValue);
  if (l.ndesc == 0 || l.total_tiles == 0) return 0;
  int dev = 0;
  cudaError_t e = current_device(&dev);
  if (e != cudaSuccess) return static_cast<int>(e);
  e = g_fp_consts.run(dev, [] {
    uint64_t h[tchash::kN];
    for (uint32_t n = 0; n < tchash::kN; ++n) h[n] = tchash::col_mul(n);
    return cudaMemcpyToSymbol(c_fp_col_mul, h, sizeof h);
  });
  if (e != cudaSuccess) return static_cast<int>(e);
  FpParams p;
  p.descs = l.descs;
  p.tile_start = l.tile_start;
  p.ndesc = l.ndesc;
  p.total_tiles = l.total_tiles;
  p.sum_ws = reinterpret_cast<unsigned long long*>(l.sum_ws);
  p.strides = l.strides;
  int grid = l.max_ctas > 0 ? l.max_ctas : std::min(current_sm_count(), 128);
  grid = static_cast<int>(std::min<uint32_t>(static_cast<uint32_t>(grid), l.total_tiles));
  cudaStream_t st = static_cast<cudaStream_t>(l.stream);
  if (wide_bytes == 4) e = unpack ? launch_fp8_kernel<true, 4>(dev, grid, p, st) : launch_fp8_kernel<false, 4>(dev, grid, p, st);
  else e = unpack ? launch_fp8_kernel<true, 2>(dev, grid, p, st) : launch_fp8_kernel<false, 2>(dev, grid, p, st);
  return static_cast<int>(e);
}

}  // namespace bb::gpu
