"""Seeded random batches through XferEngine.run and run_fp8, mixing every descriptor kind in one batch, against host models.

A byte round draws an algorithm, a grid and a batch of whole objects (1-3 destinations), windowed and strided gets,
gathered puts (1-3 destinations), gets scattered into rows, paged puts (1-3 destinations) and paged gets, XFER_RAW_SUM
slices (stored and hash-only, with a random tile base), zero-length items and verified items with a right or a wrong
expected digest, at sizes around tile edges, warp-path sizes and sizes that straddle CTA runs.  Page tables have pages
of 16 bytes to a few MiB (and single pages of any size), phases 0, random and page - 1, repeated pages (puts) and
unused entries past the object's pages that point at bytes no item may touch.  Some rounds are all-small
(bb_xfer_small) or single small items on an idle stream (the mailbox), sometimes with one scattered or paged item,
which sends the whole batch to bb_xfer; some add one item that breaks a rule, which the engine must refuse before any
launch.  The source is written on the caller's stream (or on a second stream ordered by an event) right before the
call, without a host synchronize.
An fp8 round is of 2-byte types (bf16 and fp16 mixed per item in one launch) or of fp32.  It packs objects (plain,
gathered or paged, pages of one 16-byte granule up to more than a tile, so that MX blocks straddle pages; 1-3
replicas) and unpacks them whole, through an element window or a strided window, into rows or into pages, each in a
type drawn per item: in some rounds every object is read as a type of the other size.  Some rounds first offer a batch
that mixes 2- and 4-byte items, which must be refused before any launch.

The models this trusts, and where each is checked:
  - numpy slicing for every byte a descriptor stores, with the placement rules of stored() in test_strided_get.py and
    the SourceRows and SourcePages rules written out below (rows_at, pages_at);
  - bb.crc32c, bb.bbh64, bb.xxh3t64 and their _partial forms, checked in test_common.py against golden values,
    _bbh64_numpy and python-xxhash;
  - the exact float64 MXFP8 models of test_mxfp8_exhaustive.py (model_pack, model_unpack, same_bits) and
    test_mxfp8_wide.py (model_pack_w, model_unpack_w, same_wide), checked there against torch's float8_e4m3fn,
    bfloat16, float16 and float32 conversions.
Every failure names the seed, the round and the item with a one-line description, so that it can be replayed alone.
BB_RANDOM_ROUNDS=k runs k more rounds per seed."""
import collections
import os

import numpy as np
import pytest
import torch

from test_mxfp8 import special_blocks
from test_mxfp8_exhaustive import gathered_source, model_pack, model_unpack, same_bits
from test_mxfp8_wide import gathered, model_pack_w, model_unpack_w, same_wide
from test_strided_get import stored
from test_xfer_kernels import Layout

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
GUARD16 = 0x5A5A
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
EXTRA = int(os.environ.get("BB_RANDOM_ROUNDS", "0"))
BYTE_SEEDS = [11, 23, 37, 41, 59, 67]
BYTE_ROUNDS = 30 + EXTRA  # per seed
FP8_SEEDS = [5, 13, 29]
FP8_ROUNDS = 10 + EXTRA
HBM_BUDGET = 2 << 30

KINDS = ["whole", "window", "strided", "gather", "slice", "slice-hash", "zero", "verify-ok", "verify-bad", "scatter", "pput", "pget"]
FORCED = ["scatter", "pput", "pget"]  # kinds a small or mailbox round may hold one of, which then takes bb_xfer
# "forced": a small or mailbox round that takes bb_xfer for its scattered or paged item
PATHS = ["fused", "warp", "mailbox", "forced", "fp8-pack", "fp8-unpack", "rejected", "fp8-rejected"]
SEEN = collections.Counter()  # (kind, algo) and path -> occurrences, for the coverage test at the end
DONE = set()  # tests of this module that ran to the end


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    free, _ = torch.cuda.mem_get_info()
    if free < HBM_BUDGET + (512 << 20):
        pytest.skip(f"needs about 2 GiB of free device memory, {free >> 20} MiB free")


@pytest.fixture(scope="module")
def eng():
    from blackbird_b200 import _bb

    e = _bb.XferEngine(0, 4096, 2)
    yield e
    e.set_max_ctas(0)
    e.set_small_path(True)
    e.set_mailbox(True)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _model(bb, algo):
    return {"NONE": lambda b: 0, "CRC32C": bb.crc32c, "BBH64": bb.bbh64, "XXH3": bb.xxh3t64}[algo]


class Arena:
    """Regions of one buffer, each starting at a chosen residue mod `mod` (buffers are 512-byte aligned, so the residue of
    an offset is that of its address), 16 to 47 bytes after the previous one: every gap holds guard bytes."""

    def __init__(self, rng):
        self.rng, self.end = rng, 0

    def take(self, n, residue=0, mod=16):
        o = self.end + 16 + int(self.rng.integers(0, 32))
        o += (residue - o) % mod
        self.end = o + n
        return o

    def pages(self, count, n, residue=0, mod=16):
        """take(n, residue, mod) `count` times, vectorised (page tables reach tens of thousands of entries): regions in
        address order, 1 to 3 units of `mod` of guard after the previous one, as an int64 array."""
        step = (n + mod - 1) // mod * mod
        gaps = mod * self.rng.integers(1, 4, count)
        start = self.end + 16 + (residue - self.end - 16) % mod
        offs = start + np.arange(count, dtype=np.int64) * step + np.cumsum(gaps) - gaps[0]
        self.end = int(offs[-1]) + n
        return offs

    @property
    def total(self):
        return max(self.end + 64, 4 * T)  # the refused items of _bad_item address the first 4 tiles


# ---------------------------------------------------------------------------------------------------- byte items


def _draw_size(rng, big=True):
    """A mixture: warp-path sizes, tile multiples +- a few bytes, and (big=True) sizes up to 3 MiB that straddle CTA runs."""
    r = rng.random()
    if r < 0.45 or not big:
        return int(rng.integers(1, 4097))
    if r < 0.85:
        return max(1, int(rng.integers(0, 9)) * T + int(rng.choice([-17, -16, -15, -1, 0, 1, 15, 16, 17])))
    return int(rng.integers(1, 3 * MiB))


def _edge(rng, n):
    """An object offset on a tile edge +- 1, inside a tile, 0 or n."""
    r = rng.random()
    if r < 0.4:
        return int(min(n, max(0, int(rng.integers(0, n // T + 1)) * T + int(rng.integers(-1, 2)))))
    if r < 0.5:
        return int(rng.choice([0, n]))
    return int(rng.integers(0, n + 1))


def _window(rng, n):
    a, b = sorted((_edge(rng, n), _edge(rng, n)))
    return a, b


def _pattern(rng, n):
    """(lo, hi, pitch, width, phase) inside the engine's rules: (pitch - width) % 16 == 0 unless the window holds one row."""
    kind = rng.choice(["w1", "wp", "wp16", "any"])
    base = int(rng.choice([int(rng.integers(1, 16)), 16, int(rng.integers(17, 2000)), T - 3, T, T + 16, int(rng.integers(T, 3 * T))]))
    if kind == "w1":  # width 1
        width, pitch = 1, 1 + 16 * (base // 16)
    elif kind == "wp":  # width == pitch
        width = pitch = base
    elif kind == "wp16":  # width == pitch - 16k
        pitch = base + 16 * int(rng.integers(1, 4))
        width = pitch - 16 * int(rng.integers(1, (pitch - 1) // 16 + 1))
    else:  # any gap: the window stays inside one row
        pitch = base + int(rng.integers(1, 40))
        width = int(rng.integers(1, pitch + 1))
    phase = int(rng.choice([0, int(rng.integers(0, pitch)), pitch - 1]))
    if kind == "any" and width < pitch and (pitch - width) % 16:
        row = int(rng.integers(0, (n + phase) // pitch + 1))
        r0 = max(0, row * pitch - phase)
        r1 = min(n, (row + 1) * pitch - phase)
        if r1 <= r0:
            return 0, 0, pitch, width, phase
        lo = int(rng.integers(r0, r1 + 1))
        return lo, int(rng.integers(lo, r1 + 1)), pitch, width, phase
    lo, hi = _window(rng, n)
    return lo, hi, pitch, width, phase


def _gather_pattern(rng, n):
    """(pitch, width, phase) of a gathered put of n bytes: phase < width, (pitch - width) % 16 == 0, extent below 12 MiB."""
    width = int(rng.choice([1, 16, int(rng.integers(1, 300)), int(rng.integers(300, 3 * T)), n]))
    width = max(1, min(width, n))
    pitch = width + 16 * int(rng.choice([0, 1, int(rng.integers(1, 64)), int(rng.integers(64, 1200))]))
    while (n // width + 1) * pitch > 8 * MiB:
        pitch = width + 16 * ((pitch - width) // 32)
    phase = int(rng.choice([0, int(rng.integers(0, width)), width - 1]))
    return pitch, width, phase


MAX_PAGES = 40000  # entries a table of the random rounds needs at most (the 131,072-page table has its own test)


def _page_shape(rng, n):
    """(n, page, phase, pages, spare) of a page table for an object of about n bytes: pages of 16 bytes (1024 per tile),
    48, odd multiples of 16, a tile, a tile + 16 or a few MiB, or a single page of a size that is no multiple of 16;
    phase 0, random or page - 1; `spare` unused entries after the object's pages."""
    spare = int(rng.choice([0, 0, 1, 3]))
    if rng.random() < 0.1:
        page = int(rng.integers(1, 5000)) | 1
        phase = int(rng.choice([0, int(rng.integers(0, page)), page - 1]))
        return max(1, min(n, page - phase)), page, phase, 1, spare
    page = int(rng.choice([16, 48, 16 * (2 * int(rng.integers(0, 300)) + 1), T, T + 16, int(rng.integers(1, 4)) * MiB + 16 * int(rng.integers(0, 64))]))
    phase = int(rng.choice([0, int(rng.integers(0, page)), page - 1]))
    n = min(n, MAX_PAGES * page - phase)
    return n, page, phase, (n - 1 + phase) // page + 1, spare


def rows_at(n, pitch, width, phase):
    """Offsets from row 0 of object bytes [0, n): the SourceRows rule."""
    y = np.arange(n, dtype=np.int64) + phase
    return y // width * pitch + y % width


def pages_at(n, addrs, page, phase):
    """Offsets of object bytes [0, n) in a page table: the SourcePages rule."""
    y = np.arange(n, dtype=np.int64) + phase
    return np.asarray(addrs, dtype=np.int64)[y // page] + y % page


class Item:
    """One descriptor of a byte batch: its engine tuple, the object bytes it hashes, the bytes it stores and where."""

    def __init__(self, kind, desc):
        self.kind, self.desc = kind, desc
        self.src = None       # (offset, n) of the object in the source buffer, a gather (offset, n, pitch, width, phase)
                              # or source pages (offsets, n, page, phase)
        self.stores = []      # (destination offset, stored object offsets xs or None = all, result offsets ds or None)
        self.flags, self.wrong, self.tile_base, self.win, self.rows, self.ndst = 0, False, 0, None, None, 1
        self.dst_rows = self.dst_pages = None  # scatter (pitch, width, phase); destination pages (offsets, page, phase)
        self.dst_offs = []    # destination pointer offsets (a strided item's dst[0] may lie before its region)

    def obj(self, host):
        if self.src is None:
            return host[:0]
        if len(self.src) == 2:
            o, n = self.src
            return host[o:o + n]
        if len(self.src) == 4:
            offs, n, page, phase = self.src
            return host[pages_at(n, offs, page, phase)]
        o, n, pitch, width, phase = self.src
        return host[o + rows_at(n, pitch, width, phase)]

    @property
    def forced(self):
        """Whether the item has a gathering load or a scattering store, which only bb_xfer has."""
        return self.kind in ("gather", "scatter", "pput", "pget")

    def digest(self, bb, algo, host):
        b = self.obj(host)
        if self.kind in ("slice", "slice-hash"):
            if b.size == 0:
                return 0
            part = bb.bbh64_partial if algo == "BBH64" else bb.xxh3t64_partial
            return part(np.concatenate([np.zeros(self.tile_base * T, dtype=np.uint8), b]), self.tile_base, -(-b.size // T))
        return _model(bb, algo)(b)

    def tuple(self, src_ptr, dst_ptr, expect):
        """The engine tuple.  A paged side's pointer (not read) is its buffer's start, so that no address leaves a buffer."""
        dsts = [dst_ptr + o for o in self.dst_offs]
        src_pages = dst_pages = None
        if self.src and len(self.src) == 4:
            offs, n, page, phase = self.src
            s, src_pages = src_ptr, ([src_ptr + int(a) for a in offs], page, phase)
        else:
            s = src_ptr + (self.src[0] if self.src else 0)
        if self.dst_pages is not None:
            offs, page, phase = self.dst_pages
            dsts, dst_pages = [dst_ptr], ([dst_ptr + int(a) for a in offs], page, phase)
        return (s, dsts, self.src[1] if self.src else 0, expect, self.flags, self.tile_base, self.win, self.rows, self.dst_rows,
                src_pages, dst_pages)


ROUND_BYTES = 64 * MiB  # source bytes of a round past which its items take warp-path sizes


def make_item(bb, rng, kind, sa, da, small=False, one_dst=False):
    """A random valid item of `kind`; sa / da are the source and destination arenas.  small: warp-path sizes only."""
    it = Item(kind, "")
    ndst = 1 if one_dst else int(rng.integers(1, 4))
    small = small or sa.end > ROUND_BYTES or da.end > ROUND_BYTES

    def _size(rng):
        return _draw_size(rng, big=not small)

    if kind in ("whole", "verify-ok", "verify-bad", "zero"):
        n = 0 if kind == "zero" else _size(rng)
        o = sa.take(n)
        it.src = (o, n)
        it.dst_offs = [da.take(n) for _ in range(ndst)]
        it.stores = [(d, None, None) for d in it.dst_offs]
        it.desc = f"{kind} n={n} ndst={len(it.dst_offs)}"
    elif kind == "window":
        n = _size(rng)
        lo, hi = _window(rng, n)
        it.src, it.win = (sa.take(n), n), (lo, hi)
        r = da.take(hi - lo, residue=lo % 16)
        it.dst_offs = [r - lo]
        it.stores = [(r - lo, np.arange(lo, hi), np.arange(lo, hi))]
        it.desc = f"window n={n} [{lo}, {hi})"
    elif kind == "strided":
        n = _size(rng)
        w = _pattern(rng, n)
        lo, hi, pitch, width, phase = w
        xs, ds = stored(n, w)
        lo_d = int(ds.min()) if ds.size else 0
        res = lo_d - phase + (lo + phase) // pitch * (pitch - width)  # dst[0] + phase - r_lo * gap is 16-byte aligned
        r = da.take(int(ds.max()) + 1 - lo_d if ds.size else 0, residue=res % 16)
        it.src, it.win = (sa.take(n), n), w
        it.dst_offs = [r - lo_d]
        it.stores = [(r - lo_d, xs, ds)]
        it.desc = f"strided n={n} window [{lo}, {hi}) pitch={pitch} width={width} phase={phase}"
    elif kind == "gather":
        n = _size(rng)
        pitch, width, phase = _gather_pattern(rng, n)
        last = n - 1 + phase
        extent = last // width * pitch + last % width + 1
        o = sa.take(extent, residue=(-phase) % 16)
        it.src, it.rows = (o, n, pitch, width, phase), (pitch, width, phase)
        it.dst_offs = [da.take(n) for _ in range(ndst)]
        it.stores = [(d, None, None) for d in it.dst_offs]
        it.desc = f"gather n={n} pitch={pitch} width={width} phase={phase} ndst={ndst}"
    elif kind == "scatter":
        n = _size(rng)
        if rng.random() < 0.15:  # the object fits in one row: any gap
            phase = int(rng.integers(0, 64))
            width = n + phase + int(rng.integers(0, 40))
            pitch = width + int(rng.integers(1, 40))
        else:
            pitch, width, phase = _gather_pattern(rng, n)
        at = rows_at(n, pitch, width, phase)
        r = da.take(int(at[-1]) + 1, residue=(-phase) % 16)  # dst[0] + phase is 16-byte aligned: the rows are co-aligned
        it.src, it.dst_rows = (sa.take(n), n), (pitch, width, phase)
        it.dst_offs = [r]
        it.stores = [(r, np.arange(n), at)]
        it.desc = f"scatter n={n} pitch={pitch} width={width} phase={phase}"
    elif kind in ("pput", "pget"):
        n, page, phase, npages, spare = _page_shape(rng, _size(rng))
        arena = sa if kind == "pput" else da
        # every page holds the bytes it is read or stored at, addr + phase 16-byte aligned; the spare entries past the
        # object's pages are regions of their own (source bytes no other item reads, or destination guard bytes)
        offs = arena.pages(npages + spare, min(page, phase + n), residue=(-phase) % 16)
        offs = np.concatenate([offs[:npages][rng.permutation(npages)], offs[npages:]])
        repeats = 0
        if kind == "pput" and npages > 1 and rng.random() < 0.2:  # some pages repeat
            k = rng.integers(0, npages, max(1, npages // 4))
            offs[k] = offs[rng.integers(0, npages, k.size)]
            repeats = k.size
        if kind == "pput":
            it.src = (offs, n, page, phase)
            it.dst_offs = [da.take(n) for _ in range(ndst)]
            it.stores = [(d, None, None) for d in it.dst_offs]
        else:
            it.src, it.dst_pages = (sa.take(n), n), (offs, page, phase)
            it.stores = [(0, np.arange(n), pages_at(n, offs, page, phase))]
        it.desc = f"{kind} n={n} page={page} phase={phase} pages={npages} spare={spare} repeats={repeats} ndst={len(it.dst_offs) or 1}"
    else:  # slice, slice-hash
        n = int(rng.choice([0, _size(rng), _size(rng)]))
        it.tile_base = int(rng.choice([0, 1, 3, int(rng.integers(0, 64))]))
        it.flags = bb.XFER_RAW_SUM
        it.src = (sa.take(n), n)
        if kind == "slice":
            it.dst_offs = [da.take(n)]
            it.stores = [(it.dst_offs[0], None, None)]
        it.desc = f"{kind} n={n} tile_base={it.tile_base}"
    if kind in ("verify-ok", "verify-bad") or (kind in ("window", "strided", "gather", "scatter", "pput", "pget", "zero") and rng.random() < 0.5):
        it.flags |= bb.XFER_VERIFY
        it.wrong = kind == "verify-bad" or (kind != "verify-ok" and rng.random() < 0.5)
        it.desc += " verify=" + ("wrong" if it.wrong else "right")
    return it


def _round_plan(rng, algo):
    """(mode, kinds of the items): mode 'mixed', 'small' (every item may take bb_xfer_small) or 'mailbox'."""
    r = rng.random()
    if r < 0.35:
        if r < 0.15:
            mode, kinds = "mailbox", ["whole"] * int(rng.integers(1, 9))
        else:
            count = int(rng.choice([int(rng.integers(1, 9)), int(rng.integers(9, 65)), int(rng.integers(65, 300))]))
            mode, kinds = "small", [str(rng.choice(["whole", "whole", "zero", "verify-ok", "verify-bad"])) for _ in range(count)]
        if rng.random() < 0.3:  # one scattered or paged item of a warp-path size: the batch takes bb_xfer
            kinds[int(rng.integers(0, len(kinds)))] = str(rng.choice(FORCED))
        return mode, kinds
    count = int(rng.choice([int(rng.integers(1, 9)), int(rng.integers(9, 65)), int(rng.integers(65, 300))]))
    kinds = [k for k in KINDS if algo in ("BBH64", "XXH3") or not k.startswith("slice")]
    return "mixed", [str(rng.choice(kinds)) for _ in range(count)]


def _bad_item(rng, bb, src, dst, n):
    """(item, error) breaking one rule of the engine."""
    s, d = src.data_ptr() + 64, dst.data_ptr() + 64
    cases = [((s, d, n, 0, 0, 0, (0, n, 100, 0, 0)), "INVALID_ARGUMENT"),                       # width 0
             ((s, d, n, 0, 0, 0, (0, n + 1)), "INVALID_ARGUMENT"),                              # window past the object
             ((s + 8, d, n), "INVALID_ADDRESS"),                                                # misaligned source
             ((s, [d, d + 8], n), "INVALID_ADDRESS"),                                           # misaligned replica
             ((s, d, n, 0, bb.XFER_MULTIMEM, 0, (0, n)), "INVALID_ARGUMENT"),                   # window with MULTIMEM
             ((s, d, n, 0, bb.XFER_RAW_SUM, 0, (0, n)), "INVALID_ARGUMENT"),                    # window with RAW_SUM
             ((s, d, n, 0, 0, 0, None, (100, 50, 50)), "INVALID_ARGUMENT"),                     # gather phase >= width
             ((s, d, n, 0, 0, 0, None, (100, 60, 0)), "INVALID_ADDRESS"),                       # gather gap of 40 bytes
             ((s, [], n), "INVALID_ARGUMENT"),                                                  # no destination, no RAW_SUM
             ((s, d, 100, 0, 0, 0, None, None, None, ([s], 4096, 4096)), "INVALID_ARGUMENT"),   # phase >= page
             ((s, d, 3 * 4096 + 1, 0, 0, 0, None, None, None, ([s, s + 2 * T, s + T], 4096, 0)), "INVALID_ARGUMENT"),  # table too short
             ((s, d, 5000, 0, 0, 0, None, None, None, ([s, s + T + 4], 4096, 0)), "INVALID_ADDRESS"),    # later page misaligned
             ((s, d, 5000, 0, 0, 0, None, None, None, ([s, s + T], 4008, 0)), "INVALID_ADDRESS"),        # pages, page % 16
             ((s, d, 5000, 0, 0, 0, None, None, None, None, ([d, d + T + 8], 4096, 0)), "INVALID_ADDRESS"),  # a get's later page
             ((s, d, n, 0, 0, 0, (0, 500), None, None, ([s], 4096, 0)), "INVALID_ARGUMENT"),    # pages with a window
             ((s, [d, d + T], n, 0, 0, 0, None, None, (96, 80, 0)), "INVALID_ARGUMENT")]        # scatter, two destinations
    return cases[int(rng.integers(0, len(cases)))]


def _grid(rng):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return int(rng.choice([1, 2, 3, 7, 31, sms, sms + 1, 2 * sms, 0]))


def byte_round(bb, eng, seed, rnd):
    rng = np.random.default_rng([seed, rnd])
    algo = ALGOS[int(rng.integers(0, 4))]
    A = getattr(bb.ChecksumAlgo, algo)
    grid = _grid(rng)
    mode, kinds = _round_plan(rng, algo)
    sa, da = Arena(rng), Arena(rng)
    items = [make_item(bb, rng, k, sa, da, small=mode != "mixed", one_dst=mode == "mailbox") for k in kinds]
    where = f"seed {seed} round {rnd} ({algo}, grid {grid}, {mode}, {len(items)} items)"
    src = torch.empty(sa.total, dtype=torch.uint8, device="cuda")
    dst = torch.empty(da.total, dtype=torch.uint8, device="cuda")
    fill_seed = seed * 1000 + rnd
    bb.random_fill(src.data_ptr(), src.numel(), fill_seed, _stream())
    host = src.cpu().numpy()  # synchronizes: the model's source, before the one the engine reads is written again
    digests = [it.digest(bb, algo, host) for it in items]
    tuples = []
    for it, dg in zip(items, digests):
        expect = dg ^ 1 if it.wrong else dg
        tuples.append(it.tuple(src.data_ptr(), dst.data_ptr(), expect))
    # the source the engine reads is written on the caller's stream (or a second stream ordered by an event) just before
    # the call: if a completion mode ran ahead of the caller's work, the engine would read zeros or guard bytes
    side = mode != "mailbox" and rng.random() < 0.3
    src.zero_()
    dst.fill_(GUARD)
    if side:
        s2 = torch.cuda.Stream()
        s2.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s2):
            bb.random_fill(src.data_ptr(), src.numel(), fill_seed, s2.cuda_stream)
            ev = torch.cuda.Event()
            ev.record(s2)
        torch.cuda.current_stream().wait_event(ev)
    else:
        bb.random_fill(src.data_ptr(), src.numel(), fill_seed, _stream())
    eng.set_max_ctas(grid)
    eng.set_mailbox(mode == "mailbox")
    if mode == "mailbox":
        torch.cuda.synchronize()  # the mailbox serves only an idle caller stream
    # one item in five rounds breaks a rule: the whole batch is refused before any launch and nothing is written
    if mode == "mixed" and rng.random() < 0.2:
        bad, err = _bad_item(rng, bb, src, dst, 1000)
        pos = int(rng.integers(0, len(tuples) + 1))
        before = (eng.launches, eng.small_launches, eng.mailbox_requests)
        with pytest.raises(RuntimeError, match=err):
            eng.run(tuples[:pos] + [bad] + tuples[pos:], A, _stream())
        assert (eng.launches, eng.small_launches, eng.mailbox_requests) == before, f"{where}: a refused batch launched"
        torch.cuda.synchronize()
        assert bool((dst == GUARD).all()), f"{where}: a refused batch wrote bytes"
        SEEN["rejected"] += 1
    before = (eng.launches, eng.small_launches, eng.mailbox_requests, eng.mailbox_launches)
    dg, st, _ = eng.run(tuples, A, _stream())
    torch.cuda.synchronize()
    launches, small, mail, mail_launches = (a - b for a, b in zip((eng.launches, eng.small_launches, eng.mailbox_requests,
                                                                    eng.mailbox_launches), before))
    # the path the engine's rules choose, from the items alone
    busy = [it for it in items if it.src and it.src[1] > 0 and not (algo == "NONE" and it.win is not None and it.win[1] <= it.win[0])]
    all_small = all(it.kind in ("whole", "verify-ok", "verify-bad") and it.src[1] <= 4096 for it in busy)
    # a scattered or paged item takes bb_xfer for the whole batch, whatever its size and the number of items
    if not busy:
        path, want = "none", (0, 0, 0)
    elif mode != "mixed" and any(it.forced for it in busy):
        path, want = "forced", (1, 0, 0)
    elif mode == "mailbox":
        path, want = "mailbox", (0, 0, len(busy))
    elif all_small:
        path, want = "warp", (1, 1, 0)
    else:
        path, want = "fused", (1, 0, 0)
    assert (launches - mail_launches, small, mail) == want, f"{where}: ran (launches, small, mailbox) = {(launches - mail_launches, small, mail)}, want the {path} path"
    SEEN[path] += 1
    # digests and status
    for i, (it, d, s) in enumerate(zip(items, dg, st)):
        want_d = 0 if algo == "NONE" else digests[i]
        want_s = int(algo != "NONE" and bool(it.flags & bb.XFER_VERIFY) and it.wrong)
        assert d == want_d and s == want_s, f"{where}, item {i} [{it.desc}]: digest {d:#x} status {s}, want {want_d:#x} status {want_s}"
        SEEN[(it.kind, algo)] += 1
    # every destination byte, and the guard bytes around every result and between objects
    want = np.full(dst.numel(), GUARD, dtype=np.uint8)
    owner = np.full(dst.numel(), -1, dtype=np.int32)
    for i, it in enumerate(items):
        b = it.obj(host)
        for base, xs, ds in it.stores:
            if xs is None:
                want[base:base + b.size] = b
                owner[base:base + b.size] = i
            elif xs.size:
                want[base + ds] = b[xs]
                owner[base + ds] = i
    got = dst.cpu().numpy()
    bad = np.nonzero(got != want)[0]
    if bad.size:
        first = int(bad[0])
        near = owner[max(0, first - 64):first + 64]
        idx = sorted({int(v) for v in near if v >= 0})
        pytest.fail(f"{where}: {bad.size} destination bytes differ, first at {first} (got {got[first]:#x}, want {want[first]:#x}); "
                    f"items near it: {[(i, items[i].desc) for i in idx]}")


@pytest.mark.parametrize("seed", BYTE_SEEDS)
def test_random_byte_batches(bb, eng, seed):
    """Random mixed byte batches: every destination byte, every guard byte, digest, verify status and path."""
    for rnd in range(BYTE_ROUNDS):
        byte_round(bb, eng, seed, rnd)
    DONE.add(("bytes", seed))


# ---------------------------------------------------------------------------------------------------- MXFP8 items


def _bf16(rng, n):
    """n bf16 patterns across many binades: each 32-element block has its own top exponent and its elements reach 12
    binades below it, subnormals and zeros included."""
    blocks = n // 32
    top = rng.integers(1, 255, blocks)[:, None]
    e = np.clip(top - rng.integers(0, 13, (blocks, 32)), 0, 254)
    bits = (e << 7) | rng.integers(0, 128, (blocks, 32)) | (rng.integers(0, 2, (blocks, 32)) << 15)
    return bits.reshape(-1).astype(np.uint16)


def _fp8_size(rng):
    r = rng.random()
    if r < 0.3:
        return 32 * int(rng.integers(1, T // 32))
    if r < 0.55:
        return T + 32 * int(rng.choice([-1, 0, 1]))
    return int(rng.integers(2, 7)) * T + 32 * int(rng.integers(0, T // 32))


def _specials(rng, x):
    """special_blocks() at tile starts, tile ends and in the tail of x (bf16 patterns, in place)."""
    sp = special_blocks().cpu().view(torch.int16).numpy().view(np.uint16)
    n = x.size
    for t in range(0, n, T):
        k = 32 * int(rng.integers(1, 9))
        if rng.random() < 0.5 and t + k <= n:
            x[t:t + k] = sp[:k]
        end = min(n, t + T)
        if rng.random() < 0.5 and end - k >= t:
            x[end - k:end] = sp[-k:]
    if n % T and rng.random() < 0.7:
        k = min(n % T, 32 * int(rng.integers(1, 9)))
        x[n - k:] = sp[:k]


WIDES = ["bf16", "f16", "f32"]
WB = {"bf16": 2, "f16": 2, "f32": 4}  # bytes per element
SIDES = ["2-byte", "fp32"]  # an fp8 batch's element size: bf16 and fp16 mixed per item, or fp32
PACK_FORMS = ["plain", "gather", "paged"]
UNPACK_FORMS = ["whole", "window", "strided", "scatter", "paged"]
WGUARD = {2: 0x5A5A, 4: 0x5A5A5A5A}


def _sprinkle(rng, bits, specials):
    """bits with about one element in 200 replaced by one of `specials`."""
    at = rng.random(bits.size) < 0.005
    bits[at] = rng.choice(np.array(specials, dtype=np.int64), int(at.sum()))
    return bits


def _f16(rng, n):
    """n fp16 patterns across every binade: each 32-element block has its own top exponent field (0: a block of
    subnormals and zeros) and its elements reach 12 binades below it; a few are +-Inf, NaN, +-0, max or the smallest
    subnormal."""
    blocks = n // 32
    top = rng.integers(0, 31, blocks)[:, None]
    e = np.clip(top - rng.integers(0, 13, (blocks, 32)), 0, 30)
    bits = (e << 10) | rng.integers(0, 1 << 10, (blocks, 32)) | (rng.integers(0, 2, (blocks, 32)) << 15)
    return _sprinkle(rng, bits.reshape(-1), [0x7C00, 0xFC00, 0x7E00, 0xFE01, 0x0000, 0x8000, 0x7BFF, 0x0001]).astype(np.uint16)


def _f32(rng, n):
    """n fp32 patterns across every binade, as _f16: subnormal blocks, and a few +-Inf, NaN, +-0, max and 2^-149."""
    blocks = n // 32
    top = rng.integers(0, 255, blocks)[:, None]
    e = np.clip(top - rng.integers(0, 13, (blocks, 32)), 0, 254)
    bits = (e << 23) | rng.integers(0, 1 << 23, (blocks, 32)) | (rng.integers(0, 2, (blocks, 32)) << 31)
    return _sprinkle(rng, bits.reshape(-1), [0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0, 0x80000000, 0x7F7FFFFF, 1]).astype(np.uint32)


def _values(rng, w, n):
    if w == "bf16":
        x = _bf16(rng, n)
        _specials(rng, x)
        return x
    return _f16(rng, n) if w == "f16" else _f32(rng, n)


def _pack_model(x, w):
    return model_pack(x) if w == "bf16" else model_pack_w(x, w)


def _unpack_model(packed, n, w):
    """The values a get of type w stores: the unpack of the packed bytes in that type, whatever type packed them."""
    return model_unpack(packed, n) if w == "bf16" else model_unpack_w(packed, n, w)


def _same(got, want, w, what):
    if w == "bf16":
        same_bits(got, want, "bf16", what)
    else:
        same_wide(got, want, w, what)


def _fp8_gather(rng, per):
    """(pitch, width, phase) in elements of a gathered pack or a scattered unpack: (pitch - width) % per == 0 (16 bytes),
    phase < width."""
    width = int(rng.choice([per, 5 * per, int(rng.integers(1, 3000))]))
    return width + per * int(rng.choice([0, 1, int(rng.integers(1, 40))])), width, int(rng.choice([0, int(rng.integers(0, width)), width - 1]))


def _fp8_pages(rng, n, per):
    """(page, phase, pages, spare) in elements of a table for n elements: pages of one 16-byte granule (a payload tile
    spans 2048 or 4096 of them), an odd number of granules (MX blocks straddle pages), a tile, a tile + 40 granules or a
    multiple of 4 granules, or a single page of any size; `spare` unused entries after the object's pages."""
    spare = int(rng.choice([0, 0, 1, 2]))
    if rng.random() < 0.15:
        page = n + int(rng.integers(0, 100))
        return page, int(rng.integers(0, page - n + 1)), 1, spare
    page = per * int(rng.choice([1, 3, 2 * int(rng.integers(0, 200)) + 1, T // per, T // per + 40, 4 * int(rng.integers(1, 8))]))
    phase = int(rng.choice([0, int(rng.integers(0, page)), page - 1]))
    return page, phase, (n - 1 + phase) // page + 1, spare


def _page_offsets(rng, arena, n, page, phase, npages, spare, b, mod):
    """Offsets (in units of the arena) of a table's pages, in random order, each holding what it is read or stored at
    with addr + phase 16-byte aligned; the spare entries are regions of their own after them."""
    unit = 16 // mod  # bytes per arena unit
    offs = arena.pages(npages + spare, min(page, phase + n) * b // unit, residue=(-phase * b // unit) % mod, mod=mod)
    return np.concatenate([offs[:npages][rng.permutation(npages)], offs[npages:]])


def _unpack_window(rng, n, per, strided):
    """(lo, hi) or (lo, hi, pitch, width, phase) in elements, (pitch - width) % per == 0."""
    lo, hi = sorted(int(v) for v in rng.integers(0, n + 1, 2))
    if rng.random() < 0.3 and lo >= T:  # from a tile edge +- 1
        lo = min(hi, lo // T * T + int(rng.integers(-1, 2)))
    if not strided:
        return lo, hi
    width = int(rng.choice([1, per, int(rng.integers(1, 400)), int(rng.integers(400, T))]))
    pitch = width + per * int(rng.choice([0, 1, int(rng.integers(1, 200))]))
    phase = int(rng.choice([0, int(rng.integers(0, pitch)), pitch - 1]))
    return lo, hi, pitch, width, phase


def _gathered(x, w, pitch, width, phase):
    return gathered_source(x, pitch, width, phase) if w == "bf16" else gathered(x, w, pitch, width, phase)


def _other_side(rng, side):
    """Per-item types of the other element size than `side`."""
    return "f32" if side == "2-byte" else str(rng.choice(["bf16", "f16"]))


def fp8_round(bb, eng, seed, rnd):
    """One fp8 round on the current stream; it waits for that stream only, so test_device_threads.py runs rounds from
    several threads at once."""
    rng = np.random.default_rng([seed, rnd, 8])
    mx = {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}
    grid = _grid(rng)
    eng.set_max_ctas(grid)
    side = SIDES[int(rng.random() < 0.4)]
    count = int(rng.integers(1, 10))
    sizes = [_fp8_size(rng) for _ in range(count)]
    types = ["f32" if side == "fp32" else str(rng.choice(["bf16", "f16"])) for _ in sizes]
    b = WB[types[0]]
    per = 16 // b
    xs = [_values(rng, w, n) for w, n in zip(types, sizes)]
    forms = [str(rng.choice(PACK_FORMS)) for _ in sizes]
    nrep = [int(rng.integers(1, 4)) for _ in sizes]
    where = f"fp8 seed {seed} round {rnd} ({side}, grid {grid}, {count} objects)"
    packed = [_pack_model(x, w) for x, w in zip(xs, types)]
    lay = Layout([p.size for p in packed])
    reps = [lay.guarded() for _ in range(3)]
    # the paged sources: pages of one guard-filled byte buffer
    pg = Arena(rng)
    args, descs = [], []
    for i, (x, w, f) in enumerate(zip(xs, types, forms)):
        if f == "gather":
            args.append(_fp8_gather(rng, per))
        elif f == "paged":
            page, phase, npg, spare = _fp8_pages(rng, x.size, per)
            args.append((_page_offsets(rng, pg, x.size, page, phase, npg, spare, b, 16), page, phase))
            f += f" page={page} phase={phase} pages={npg} spare={spare}"
        else:
            args.append(None)
        descs.append(f"{w} n={x.size} {f if f != 'gather' else f'gather={args[-1]}'} replicas={nrep[i]}")
    host_pg = np.full(pg.total, GUARD, dtype=np.uint8)
    for x, f, a in zip(xs, forms, args):
        if f == "paged":
            host_pg[pages_at(x.size * b, a[0], a[1] * b, a[2] * b)] = x.view(np.uint8)
    pg_dev = torch.from_numpy(host_pg).cuda()
    srcs, items = [], []  # srcs keeps the sources alive until the kernel has read them
    for i, (x, w, f, a, o) in enumerate(zip(xs, types, forms, args, lay.offs)):
        gather = pages = None
        if f == "plain":
            s = torch.from_numpy(x.view(np.int16 if b == 2 else np.int32).copy()).cuda()
            ptr = s.data_ptr()
        elif f == "gather":
            s, off = _gathered(x, w, *a)  # the gaps hold NaN, Inf and max
            ptr, gather = s.data_ptr() + b * off, a
        else:
            s, ptr = pg_dev, pg_dev.data_ptr()
            pages = ([ptr + int(v) for v in a[0]], a[1], a[2])
        srcs.append(s)
        items.append((ptr, [reps[k].data_ptr() + o for k in range(nrep[i])], x.size, None, None, gather, None, mx[w], pages))
    # one round in four first offers a batch that mixes 2- and 4-byte items: refused before any launch, nothing written
    if rng.random() < 0.25:
        other = _other_side(rng, side)
        odd_src = torch.zeros(32 * WB[other], dtype=torch.uint8, device="cuda")
        odd_out = torch.full((64,), GUARD, dtype=torch.uint8, device="cuda")
        pos = int(rng.integers(0, count + 1))
        odd = (odd_src.data_ptr(), odd_out.data_ptr(), 32, None, None, None, None, mx[other])
        before = (eng.launches, eng.small_launches)
        with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
            eng.run_fp8(items[:pos] + [odd] + items[pos:], False, _stream(), wide=mx[types[0]])
        assert (eng.launches, eng.small_launches) == before, f"{where}: a batch of {other} at {pos} among {side} items launched"
        torch.cuda.current_stream().synchronize()
        assert all(bool((r == GUARD).all()) for r in reps) and bool((odd_out == GUARD).all()), f"{where}: a refused batch wrote bytes"
        SEEN["fp8-rejected"] += 1
    dg, st, _ = eng.run_fp8(items, False, _stream(), wide=mx[types[0]])
    torch.cuda.current_stream().synchronize()
    SEEN["fp8-pack"] += 1
    assert st == [0] * count, f"{where}: pack status {st}"
    for i, (p, d) in enumerate(zip(packed, dg)):
        assert d == bb.bbh64(p), f"{where}, item {i} [{descs[i]}]: digest"
        SEEN[("pack", types[i], forms[i])] += 1
    for k in range(3):
        got = reps[k].cpu().numpy()
        used = [i for i in range(count) if nrep[i] > k]
        want = np.full(lay.total, GUARD, dtype=np.uint8)
        for i in used:
            want[lay.offs[i]:lay.offs[i] + packed[i].size] = packed[i]
        outside = np.ones(lay.total, dtype=bool)
        for i in used:
            outside[lay.offs[i]:lay.offs[i] + packed[i].size] = False
        assert bool((got[outside] == want[outside]).all()), f"{where}: replica {k} written outside its objects"
        for i in used:
            same_bits(got[lay.offs[i]:lay.offs[i] + packed[i].size][sizes[i]:], packed[i][sizes[i]:], "e8m0",
                      f"{where}, item {i} [{descs[i]}], replica {k}: block scales")
            same_bits(got[lay.offs[i]:lay.offs[i] + sizes[i]], packed[i][:sizes[i]], "e4m3",
                      f"{where}, item {i} [{descs[i]}], replica {k}: payload")
    # unpack every object from replica 0, in a type of its own (the other element size in some rounds: every item is then
    # read as a type it was not packed from): whole, through an element window or a strided window, into rows or pages,
    # with a right or a wrong expected digest
    gside = side if rng.random() < 0.7 else SIDES[1 - SIDES.index(side)]
    gtypes = ["f32" if gside == "fp32" else str(rng.choice(["bf16", "f16"])) for _ in sizes]
    gb = WB[gtypes[0]]
    gper = 16 // gb
    uforms = [str(rng.choice(UNPACK_FORMS)) for _ in sizes]
    wrong = [bool(rng.random() < 0.25) for _ in sizes]
    ar = Arena(rng)  # in elements of the get's type
    plan = []  # (pointer offset in elements, window, scatter, pages (offsets, page, phase), object elements xs_, result elements ds)
    for n, f in zip(sizes, uforms):
        win = scat = pages = None
        if f == "whole":
            r = ar.take(n, 0, gper)
            xs_, ds, at = np.arange(n), r + np.arange(n), r
        elif f == "window":
            win = _unpack_window(rng, n, gper, False)
            r = ar.take(win[1] - win[0], win[0] % gper, gper)
            xs_ = np.arange(win[0], win[1])
            at, ds = r - win[0], r - win[0] + xs_
        elif f == "strided":
            win = _unpack_window(rng, n, gper, True)
            lo, hi, pitch, width, phase = win
            xs_, d_ = stored(n, win)
            lo_d = int(d_.min()) if d_.size else 0
            res = lo_d - phase + (lo + phase) // pitch * (pitch - width)  # the rows' first elements are co-aligned
            r = ar.take(int(d_.max()) + 1 - lo_d if d_.size else 0, res % gper, gper)
            at, ds = r - lo_d, r - lo_d + d_
        elif f == "scatter":
            scat = _fp8_gather(rng, gper)
            rows = rows_at(n, *scat)
            r = ar.take(int(rows[-1]) + 1, (-scat[2]) % gper, gper)  # row 0 + phase is 16-byte aligned
            xs_, ds, at = np.arange(n), r + rows, r
        else:
            page, phase, npg, spare = _fp8_pages(rng, n, gper)
            offs = _page_offsets(rng, ar, n, page, phase, npg, spare, gb, gper)
            pages = (offs, page, phase)
            xs_, ds, at = np.arange(n), pages_at(n, offs, page, phase), 0
            f += f" page={page} phase={phase} pages={npg} spare={spare}"
        plan.append((at, win, scat, pages, xs_, ds, f))
    out = torch.full((ar.total,), WGUARD[gb], dtype=torch.int16 if gb == 2 else torch.int32, device="cuda")
    optr = out.data_ptr()
    gets = []
    for i, (at, win, scat, pages, _, _, _) in enumerate(plan):
        pg_ = None if pages is None else ([optr + gb * int(v) for v in pages[0]], pages[1], pages[2])
        gets.append((optr + gb * at, reps[0].data_ptr() + lay.offs[i], sizes[i], dg[i] ^ int(wrong[i]), win, None, scat, mx[gtypes[i]], None, pg_))
    dg2, st2, _ = eng.run_fp8(gets, True, _stream(), wide=mx[gtypes[0]])
    torch.cuda.current_stream().synchronize()
    SEEN["fp8-unpack"] += 1
    udesc = [f"{descs[i]}; get as {gtypes[i]}: {plan[i][6]} window={plan[i][1]} scatter={plan[i][2]}" for i in range(count)]
    for i in range(count):
        assert dg2[i] == dg[i] and st2[i] == int(wrong[i]), f"{where}, item {i} [{udesc[i]}]: digest / status {st2[i]}"
        SEEN[("unpack", gtypes[i], uforms[i])] += 1
        SEEN[("cross", side)] += gtypes[i] != types[i]
    got = out.cpu().numpy().view(np.uint16 if gb == 2 else np.uint32)
    want = np.full(ar.total, WGUARD[gb], dtype=got.dtype)
    written = np.zeros(ar.total, dtype=bool)
    for i, (_, _, _, _, xs_, ds, _) in enumerate(plan):
        if xs_.size:
            want[ds] = _unpack_model(packed[i], sizes[i], gtypes[i])[xs_]
        written[ds] = True
    for i, (_, _, _, _, xs_, ds, _) in enumerate(plan):
        if ds.size:  # the results and the guard elements around and between their rows or pages
            lo, hi = int(ds.min()) - gper, int(ds.max()) + 1 + gper
            _same(got[lo:hi], want[lo:hi], gtypes[i], f"{where}, item {i} [{udesc[i]}]: unpacked")
    outside = np.nonzero(~written & (got != WGUARD[gb]))[0]
    assert outside.size == 0, f"{where}: unpack wrote {outside.size} elements outside its results, first at {outside[:4].tolist()}"


@pytest.mark.parametrize("seed", FP8_SEEDS)
def test_random_fp8_batches(bb, eng, seed):
    """Random MXFP8 pack and unpack batches against the exact model."""
    for rnd in range(FP8_ROUNDS):
        fp8_round(bb, eng, seed, rnd)
    DONE.add(("fp8", seed))


def test_every_kind_algorithm_and_path_occurred():
    """The generators above reached every (item kind x algorithm) and every path at least a few times."""
    if len(DONE) < len(BYTE_SEEDS) + len(FP8_SEEDS):
        pytest.skip("runs only after every random test of this module ran")
    missing = []
    for k in KINDS:
        for a in ALGOS:
            if k.startswith("slice") and a not in ("BBH64", "XXH3"):
                continue
            if SEEN[(k, a)] < 3:
                missing.append((k, a, SEEN[(k, a)]))
    missing += [(p, SEEN[p]) for p in PATHS if SEEN[p] < 3]
    for w in WIDES:
        missing += [(op, w, f, SEEN[(op, w, f)]) for op, forms in (("pack", PACK_FORMS), ("unpack", UNPACK_FORMS)) for f in forms
                    if SEEN[(op, w, f)] < 3]
    missing += [("cross-type read", side, SEEN[("cross", side)]) for side in SIDES if SEEN[("cross", side)] < 1]
    print("\ncoverage:", {str(k): v for k, v in sorted(SEEN.items(), key=str)})
    assert not missing, f"categories reached fewer than 3 times: {missing}"
