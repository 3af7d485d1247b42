// Host-visible API of the sm_90a data-plane kernels (plain C++; no CUDA types leak out).
//
// These kernels replace the reference's UCX call sites (SURVEY K1-K7): `ucp_put_nbx`
// (blackbird_client.cpp:231-237), `ucp_get_nbx` (:315-327) and the CPU byte compare
// (ucx_client.cpp:277).  One launch moves a whole *batch* of objects described by a device
// descriptor table, fusing the transfer with the checksum (and optional replica fan-out).
#pragma once
#include <cstddef>
#include <cstdint>

#include "common/mxfp8.h"

namespace bb::gpu {

constexpr uint32_t kTileBytes = 16384;   // one TMA tile == one BBH64 tile (tchash_def.h)
constexpr uint32_t kMaxDst = 3;          // replicas written by a single tile pass

enum XferFlags : uint32_t {
  XFER_VERIFY = 1u << 0,    // compare digest with `expect`; status[i] = 1 on mismatch
  XFER_MULTIMEM = 1u << 1,  // dst[0] is an NVLS multicast address: store with multimem.st
  // BBH64 / XXH3 (the tile-sum digests): digest_out receives the *unfinalised* 64-bit tile sum and `reserved` is added to every tile
  // index, so a byte range can be hashed as a slice of a larger object (its sums add up with the slices
  // hashed elsewhere; the host finalises).  With ndst == 0 the descriptor is hash-only (nothing is stored).
  XFER_RAW_SUM = 1u << 2,
  // Store window (range reads): every tile is still loaded and hashed, but only object bytes [win.lo, win.hi) are
  // stored.  Only with ndst == 1, never with XFER_MULTIMEM or XFER_RAW_SUM.  The fused MXFP8 get honours it too, with the
  // window in bf16 bytes of the unpacked object; an MXFP8 put never carries it.
  XFER_WINDOW = 1u << 3,
  // Strided store window (slices along an inner dimension), only together with XFER_WINDOW, in bb_xfer and the fused
  // MXFP8 get: the rule of common/store_window.h with row == 0, so dst[0] is where the pattern's row 0 lands and the rows
  // land densely from there.  The pattern is the descriptor's entry of the launch's XferStride table; the MXFP8 get
  // counts all of it in bf16 bytes of the unpacked object.
  XFER_STRIDED = 1u << 4,
  // Gathering load (puts of a strided source), in bb_xfer and the fused MXFP8 put: the rule of SourceRows
  // (common/store_window.h), so `src` is where the pattern's row 0 starts and object byte x is read from
  // src + ((x + phase) / width) * pitch + (x + phase) % width.  The pattern is the descriptor's entry of the launch's
  // XferStride table; the MXFP8 put counts all of it in bf16 bytes of the source.  Never with XFER_WINDOW, XFER_STRIDED or
  // XFER_RAW_SUM; with 1-3 destinations or XFER_MULTIMEM.  The tile in shared memory is byte for byte the tile of the
  // dense object, so the digest and the stored bytes are those of a put of the compacted rows.
  XFER_GATHER = 1u << 5,
  // Scattering store (gets into a strided destination), the mirror of XFER_GATHER, in bb_xfer and the fused MXFP8 get: the
  // same SourceRows rule applied to the destination, so dst[0] is where the pattern's row 0 starts and object byte x is
  // stored at dst[0] + ((x + phase) / width) * pitch + (x + phase) % width.  The pattern is the descriptor's entry of the
  // launch's XferStride table; the MXFP8 get counts all of it in bf16 bytes of the destination.  Only with ndst == 1; never
  // with XFER_WINDOW, XFER_STRIDED, XFER_GATHER, XFER_MULTIMEM or XFER_RAW_SUM.  The tile in shared memory is the object's
  // tile, so the digest and the verify are those of a plain get.
  XFER_SCATTER = 1u << 6,
  // Fused MXFP8 only: the descriptor's wide side is fp16, not bf16 (mxfp8::Wide::F16), in the 2-byte instantiation of
  // the kernel.  A batch of bf16 and fp16 items is one launch; fp32 items take the 4-byte instantiation, a launch of their
  // own.
  XFER_WIDE_F16 = 1u << 7,
  // Paged source or destination, in bb_xfer and the fused MXFP8 put and get, together with XFER_GATHER (a put reads its
  // pages) or XFER_SCATTER (a get stores into them): the rule of SourcePages (common/store_window.h), object byte x at
  // pages[(x + phase) / page] + (x + phase) % page.  The descriptor's XferStride entry is {device address of its first
  // page entry, page, phase}; `src` (put) or dst[0] (get) is not read.  The MXFP8 kernels count page and phase in bytes
  // of the wide side.  The destination forms are those of XFER_GATHER or XFER_SCATTER; never with XFER_WINDOW,
  // XFER_STRIDED or XFER_RAW_SUM.  The tile in shared memory is the dense object's tile, so the digest, the verify and
  // the stored bytes are those of a contiguous put or get.
  XFER_PAGED = 1u << 8,
  // With XFER_PAGED only: every page is rows inside its block, the in-page row pattern of SourcePages: with the entry's
  // row_width and row_pitch, c = (x + phase) % page and k = (x + phase) / page, object byte x is at
  // pages[k] + (c / row_width) * row_pitch + c % row_width.  The kernels then move the dense object's rows of row_width
  // bytes one per lane instead of whole pages; the tile is still the dense object's tile.
  XFER_PAGE_ROWS = 1u << 9,
  // With XFER_WINDOW (and XFER_STRIDED for a strided window) only, one destination: the window's dense result lands in
  // rows (WindowRows, common/store_window.h).  Stored unit x has the dense index p = x - lo (a range window) or
  // p = ((x + phase) / pitch) * width + (x + phase) % pitch (a strided window, the descriptor's pattern), and lands at
  // dst[0] + ((p + row_phase) / row_width) * row_pitch + (p + row_phase) % row_width.  The window pattern is the entry's
  // pitch / width / phase as for XFER_STRIDED; the destination rows are its row_width / row_pitch / row_phase words,
  // which XFER_PAGE_ROWS uses for in-page rows and which no other descriptor reads.  Only the engine sets it (from a
  // WINDOW_ROWS layout); never with XFER_SCATTER, XFER_GATHER, XFER_PAGED, XFER_MULTIMEM or XFER_RAW_SUM.  Every tile
  // is still loaded and hashed, so the digest and the verify are those of a plain get.
  XFER_WINDOW_ROWS = 1u << 10,
  // Segmented source or destination (SourceSegments, common/store_window.h), in bb_xfer and bb_xfer_fp8, together with
  // XFER_GATHER (a put or a pack reads its segments) or XFER_SCATTER (a get or an unpack stores into them), in bytes (of
  // the wide side for bb_xfer_fp8): the object is the concatenation of segments of any sizes, object byte x at
  // addr[k] + (x - start[k]) for the segment k with start[k] <= x < start[k + 1].  The descriptor's XferStride entry is {device address of its first segment entry, number of segments, object offset of the
  // descriptor's byte 0}; the entries are 16-byte SegmentEntry {start, addr} pairs followed by one whose start ends the
  // last segment.  `src` (put) or dst[0] (get) is not read.  Per tile the walking warp finds the tile's first segment by a
  // 32-way search and takes the segments that overlap the tile one per lane.  A get's segment whose address is 0 is not
  // stored (a null segment).  Only the engine sets it (from a SEGMENTS layout); never with XFER_PAGED, XFER_PAGE_ROWS,
  // XFER_WINDOW, XFER_STRIDED, XFER_WINDOW_ROWS or XFER_RAW_SUM.  The tile in shared memory is the dense object's tile,
  // so the digest, the verify and the stored bytes are those of a contiguous put or get of the concatenation (for
  // bb_xfer_fp8 the wide tile is the concatenation's, so an MX block may straddle two segments).
  XFER_SEGMENTS = 1u << 11,
};

// 64-byte transfer descriptor, one per (object shard, direction).
//
// dst[0] is where object byte 0 lands, so byte x is stored at dst[0] + x.  With XFER_WINDOW the caller's buffer holds only
// the window: dst[0] is then the virtual base `buffer - lo`, an address that is never dereferenced outside [lo, hi).  A
// windowed descriptor has one destination, so the words of dst[1] / dst[2] carry the window bounds (`win`).
struct XferDesc {
  const void* src;          // 16-byte aligned; local or peer-mapped
  union {
    void* dst[kMaxDst];     // 16-byte aligned; local, peer-mapped or multicast
    struct {
      void* base;           // = dst[0]
      uint64_t lo, hi;      // XFER_WINDOW: byte range of the object that is stored, lo <= hi <= nbytes
    } win;
  };
  uint64_t nbytes;
  uint32_t first_tile;      // exclusive prefix sum of ceil(nbytes / kTileBytes)
  uint32_t ndst;
  uint64_t expect;          // BBH64: expected digest.  CRC32C: (init_term << 32) | expected crc
  uint32_t flags;
  uint32_t reserved;        // CRC32C: x^(-8*pad) mod P (crc_unpad_for); BBH64 + XFER_RAW_SUM: tile index base
};
static_assert(sizeof(XferDesc) == 64, "XferDesc must be 64 bytes");
static_assert(offsetof(XferDesc, win.lo) == offsetof(XferDesc, dst) + 8 && offsetof(XferDesc, win.hi) == offsetof(XferDesc, dst) + 16,
              "the window bounds are the words of dst[1] / dst[2]");

// Row pattern of an XFER_STRIDED descriptor (see XferFlags): 0 < width <= pitch, phase < pitch.  With pitch == width and
// phase == 0 it stores exactly the plain window.  Every stored row must be co-aligned with the tile (the destination of
// object byte x congruent to x mod 16), so that the kernel only bulk-stores 16-byte congruent spans.  An XFER_GATHER
// descriptor's entry is its source rows instead: 0 < width <= pitch, phase < width, and the source of object byte x
// congruent to x mod 16 (SourceRows::coaligned).  An XFER_SCATTER descriptor's entry is its destination rows, under the
// same rules.  An XFER_PAGED descriptor's entry is {pages, page, phase}: `pages` the device address of the first of its
// page entries (uint64_t addresses, one per page the descriptor touches), `page` in `width`, phase < page, every page
// co-aligned: pages[k] + phase 16-byte aligned (SourcePages::coaligned).  row_width and row_pitch are read only for
// XFER_PAGE_ROWS descriptors: 0 < row_width < row_pitch, page % row_width == 0, (row_pitch - row_width) % 16 == 0.  An
// XFER_WINDOW_ROWS descriptor's entry holds its window pattern (XFER_STRIDED only) in the first three words and its
// destination rows in the last three: 0 < row_width < row_pitch, row_phase < row_width, and every stored byte's
// destination congruent to its object offset mod 16 (WindowRows::coaligned).  An XFER_SEGMENTS descriptor's entry is
// {segs, nseg, phase}: `segs` (in `pages`) the 16-byte aligned device address of its first segment entry, `nseg` (in
// `width`) the segments its bytes touch, `phase` the object offset of its byte 0, and every non-null segment co-aligned:
// addr[k] + phase - start[k] 16-byte aligned (SourceSegments::coaligned).
struct XferStride {
  union {
    uint64_t pitch;
    uint64_t pages;  // XFER_PAGED; XFER_SEGMENTS: the segment entries
  };
  uint64_t width, phase;
  uint64_t row_width = 0, row_pitch = 0;  // XFER_PAGE_ROWS, XFER_WINDOW_ROWS
  uint64_t row_phase = 0;                 // XFER_WINDOW_ROWS
};

constexpr uint32_t kSmallBytes = 4096;     // objects up to this size may take the warp-per-object path (xfer_small.cu)
constexpr uint32_t kSmallPending = 0xFFFFFFFFu;  // value of a status slot whose object has not completed yet (flag completion)
constexpr uint32_t kInlineDescs = 8;       // descriptors that fit in the kernel parameter block
constexpr uint32_t kDirectResults = 64;    // batches up to this size write digests straight to pinned host memory

enum XferAlgo : int { ALGO_NONE = 0, ALGO_CRC32C = 1, ALGO_BBH64 = 2, ALGO_XXH3 = 3 };

struct XferLaunch {
  const XferDesc* descs = nullptr;       // device pointer, ndesc entries
  const uint32_t* tile_start = nullptr;  // device pointer, ndesc+1 entries (prefix sums)
  uint32_t ndesc = 0;
  uint32_t total_tiles = 0;
  uint64_t* sum_ws = nullptr;            // device, ndesc entries, must be zero on entry (self-cleaning)
  uint32_t* done_ws = nullptr;           // device, ndesc entries, must be zero on entry (self-cleaning)
  uint64_t* digest_out = nullptr;        // device, ndesc entries
  uint32_t* status_out = nullptr;        // device, ndesc entries (0 ok / 1 checksum mismatch)
  const uint32_t* crc_tables = nullptr;  // device, CRC32C shift tables (only ALGO_CRC32C)
  uint32_t* debug_d = nullptr;           // optional: raw accumulators [tile][128][16] (tests)
  uint64_t* trace_d = nullptr;           // optional: per-tile pipeline timestamps [tile][4] (globaltimer ns)
  // Optional host copies of the two tables: batches of <= kInlineDescs descriptors travel in the
  // kernel parameters instead (descs / tile_start may then be null).
  const XferDesc* host_descs = nullptr;
  const uint32_t* host_tile_start = nullptr;
  // Row patterns of the XFER_STRIDED, XFER_GATHER and XFER_SCATTER descriptors, one entry per descriptor (the entries of unflagged
  // descriptors are never read, nor row_width / row_pitch / row_phase of descriptors without XFER_PAGE_ROWS or XFER_WINDOW_ROWS); null when the batch has none.  host_strides is their copy for the kernel parameters of an
  // inline batch; a batch with XFER_PAGED descriptors has no inline copy (their entries point into device memory).
  const XferStride* strides = nullptr;
  const XferStride* host_strides = nullptr;
  int algo = ALGO_BBH64;
  bool small_path = false;               // every descriptor is <= kSmallBytes, none is a RAW_SUM slice: warp-per-object kernel
  bool flag_completion = false;          // small path only: status_out (pinned, preset to kSmallPending) is the completion flag
  int max_ctas = 0;                      // 0 = the default geometry (xfer_geometry)
  void* stream = nullptr;                // cudaStream_t
};

// Returns 0 on success, else a cudaError_t value.
int launch_xfer(const XferLaunch& l);
// What launch_xfer's fused kernel launches for a batch of `total_tiles` tiles on the current device.  CRC32C: one
// persistent CTA per SM.  The other digests: CTAs of at most 8 tiles, at least two per SM, which the block scheduler
// hands to whichever SM frees a slot first.  max_ctas > 0 (or else BB_XFER_CTAS) sets the grid instead.  Every CTA gets
// ceil(total_tiles / grid) consecutive tiles and CTAs that would get none are not launched.
struct XferGeometry {
  int grid = 0;        // CTAs
  int stages = 0;      // 16 KiB shared-memory pipeline stages per CTA
  int smem_bytes = 0;  // dynamic shared memory per CTA
};
XferGeometry xfer_geometry(int algo, uint32_t total_tiles, int max_ctas);
// CTAs of the fused kernel for `algo` the current device keeps resident per SM (occupancy query); -1 on a CUDA error.
int xfer_resident_ctas(int algo);
// ---- mailbox (xfer_small.cu): a resident warp fed through pinned host memory, so that a single small put / get costs no
// kernel launch.  All three structures live in pinned host memory (the device reads / writes them over PCIe).
constexpr uint32_t kMailSlots = 16;
struct MailSlot {  // 64 bytes = one cache line = one PCIe read; the host writes `seq` LAST
  uint64_t src;
  uint64_t dst;
  uint64_t expect;     // as XferDesc::expect
  uint32_t nbytes;     // <= kSmallBytes
  uint32_t flags;      // XferFlags (no MULTIMEM, no RAW_SUM)
  uint32_t algo;       // XferAlgo
  uint32_t reserved;   // as XferDesc::reserved
  uint32_t pad[5];
  uint32_t seq;        // word 15
};
static_assert(sizeof(MailSlot) == 64, "MailSlot must be one cache line");
struct alignas(64) MailResult {  // 64 bytes; the device writes the first 16 bytes (digest, status, seq) with one store
  uint64_t digest;
  uint32_t status;
  uint32_t seq;
  uint32_t pad[12];
};
static_assert(sizeof(MailResult) == 64 && offsetof(MailResult, seq) == 12);
struct MailCtl {
  uint32_t exit_epoch;  // epoch of the last kernel incarnation that has exited (== the launched epoch: nobody is polling)
  uint32_t next_seq;    // first sequence number that incarnation did NOT consume
  uint32_t pad[14];
};
// Launches one incarnation of the mailbox kernel on `stream`: it serves requests from sequence number `first_seq` on and
// exits after `linger_ns` without a request or `max_ns` in total, then writes (next_seq, exit_epoch = epoch) into *ctl.
int launch_mailbox(const MailSlot* slots, MailResult* results, MailCtl* ctl, uint32_t first_seq, uint32_t epoch, uint64_t linger_ns,
                   uint64_t max_ns, void* stream);

// Small-object latency tier: one warp per descriptor, digest bit-identical to launch_xfer's (needs descs; not tile_start).
int launch_xfer_small(const XferLaunch& l);
int xfer_smem_bytes(int algo);
// Fused MXFP8 transfer (xfer_mxfp8.cu).  The packed object is one contiguous [payload n][scales n/32] extent.  The wide
// side holds `wide_bytes` (2 or 4) bytes per element: bf16, or fp16 for descriptors with XFER_WIDE_F16, when it is 2;
// fp32 when it is 4.  Below, "bf16 bytes" means bytes of that wide side.
// Descriptors: pack (put): src = bf16 source, dst[0..ndst-1] = base of the packed object in every replica (the scales
// follow the payload), nbytes = payload bytes (= elements, a multiple of kTileBytes); unpack (get): src = base of the
// packed object, dst[0] = bf16 destination (where element 0 lands); an unpack descriptor may carry XFER_WINDOW, whose
// `win` is then in bf16 bytes of the object ([2 * first element, 2 * end element)), and XFER_STRIDED, whose pattern in
// `strides` (a device table; no inline copy) is in bf16 bytes too; or instead XFER_SCATTER, with dst[0] where the
// destination pattern's row 0 starts and the pattern in bf16 bytes in `strides`.  `sum_ws` receives the unfinalised BBH64 sum of the
// payload tiles per descriptor (must be zero on entry); descs / tile_start are device tables.
int launch_xfer_fp8(const XferLaunch& l, bool unpack, uint32_t wide_bytes = 2);
// Dynamic shared memory of the instantiation for `wide_bytes`-byte elements (its ring stage counts differ).
int xfer_fp8_smem_bytes(uint32_t wide_bytes = 2);

// ---- page tables from device-resident block ids (resolve_blocks.cu; the rule is SourceBlocks in common/store_window.h)
// One job fills the page entries of one XFER_PAGED descriptor whose layout is a SourceBlocks: entries[t] is page first + t
// of the object, t < count.  Every id (and selection entry) of the object is checked first, so that every shard of it
// reaches the same verdict, which the job writes to *verdict: kBlocksOk, kBlocksOutOfRange or kBlocksDuplicate (a get's
// repeated id or selection entry).  A refused get's entries are all 0 (null pages: nothing is stored), a refused put's
// all outer[q] (block 0 of the page's slice, inside the caller's cache).  n_blocks and, with a selection, n_stored are
// at most kBlocksMaxDistinct for a get.
constexpr uint32_t kBlocksOk = 0, kBlocksOutOfRange = 1, kBlocksDuplicate = 2;
constexpr uint64_t kBlocksMaxDistinct = uint64_t{1} << 18;
struct BlocksJob {
  uint64_t* entries;
  const uint64_t* outer;  // device copy of the n_outer slice addresses
  const void* ids;
  const void* sel;  // null: no selection
  uint64_t n_outer, n_ids, n_stored, n_blocks, stride, first, count;
  uint32_t id_bytes;  // 4 or 8, for ids and sel alike
  uint32_t get;       // refuse duplicates; a refused table is all null
  uint32_t* verdict;  // pinned host memory
  uint32_t pad;
};
// Launches one CTA per job of the device table `jobs` on `stream`.  Returns 0 or a cudaError_t value.
int launch_resolve_blocks(const BlocksJob* jobs, uint32_t njobs, void* stream);

// CRC32C per-object constants (host): un-padding multiplier and the init-register term.
uint32_t crc_unpad_for(uint64_t nbytes);
uint32_t crc_init_term_for(uint64_t nbytes);

// Number of tiles of an object (0 for empty objects).
inline uint32_t tiles_of(uint64_t nbytes) { return static_cast<uint32_t>((nbytes + kTileBytes - 1) / kTileBytes); }

// ---- comparators / utilities (baseline.cu)
// Plain vectorised copy kernel (the "unfused copy kernel" comparator of BASELINE.md §4).
int launch_copy_simt(void* dst, const void* src, uint64_t nbytes, void* stream);
// Stand-alone CRC32C over device memory (comparator: "separate CRC32C kernel"); result is the
// standard CRC32C written to *out (device).  `tables` = device copy of crc tables (see crc_tables_host()).
int launch_crc32c_simt(const void* data, uint64_t nbytes, uint32_t* out, uint32_t* scratch, void* stream);
// L2 flush helper: writes `nbytes` of a scratch buffer.
int launch_fill(void* dst, uint64_t nbytes, uint32_t value, void* stream);
// Fills a buffer with deterministic pseudo-random bytes (synthetic objects).
int launch_random_fill(void* dst, uint64_t nbytes, uint64_t seed, void* stream);

// MXFP8 pack / unpack (mxfp8.cu): bf16 / fp16 / fp32 <-> [E4M3 payload | E8M0 scale per 32 elements].
// n_elems % 32 == 0; packed size = n_elems + n_elems / 32 bytes (common/mxfp8.h); the wide side 16-byte aligned.
int launch_mxfp8_pack(const void* src_wide, uint64_t n_elems, void* dst_packed, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);
int launch_mxfp8_unpack(const void* src_packed, uint64_t n_elems, void* dst_wide, void* stream, mxfp8::Wide wide = mxfp8::Wide::BF16);

}  // namespace bb::gpu
