"""Seeded random batches through XferEngine.run and run_fp8, mixing every descriptor kind in one batch, against host models.

A byte round draws an algorithm, a grid and a batch of whole objects (1-3 destinations), windowed and strided gets,
gathered puts (1-3 destinations), XFER_RAW_SUM slices (stored and hash-only, with a random tile base), zero-length
items and verified items with a right or a wrong expected digest, at sizes around tile edges, warp-path sizes and sizes
that straddle CTA runs.  Some rounds are all-small (bb_xfer_small) or single small items on an idle stream (the
mailbox); some add one item that breaks a rule, which the engine must refuse before any launch.  The source is written
on the caller's stream (or on a second stream ordered by an event) right before the call, without a host synchronize.
An fp8 round packs bf16 objects (plain and gathered, 1-3 replicas) and unpacks them whole, through an element window or
through a strided window.

The models this trusts, and where each is checked:
  - numpy slicing for every byte a descriptor stores, with the placement rules of stored() in test_strided_get.py and
    the SourceRows rule written out below;
  - bb.crc32c, bb.bbh64, bb.xxh3t64 and their _partial forms, checked in test_common.py against golden values,
    _bbh64_numpy and python-xxhash;
  - the exact float64 MXFP8 model of test_mxfp8_exhaustive.py (model_pack, model_unpack, same_bits), checked there
    against torch's float8_e4m3fn and bfloat16 conversions.
Every failure names the seed, the round and the item with a one-line description, so that it can be replayed alone.
BB_RANDOM_ROUNDS=k runs k more rounds per seed."""
import collections
import os

import numpy as np
import pytest
import torch

from test_mxfp8 import special_blocks
from test_mxfp8_exhaustive import gathered_source, model_pack, model_unpack, same_bits
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

KINDS = ["whole", "window", "strided", "gather", "slice", "slice-hash", "zero", "verify-ok", "verify-bad"]
PATHS = ["fused", "warp", "mailbox", "fp8-pack", "fp8-unpack", "rejected"]
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

    @property
    def total(self):
        return self.end + 64


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


class Item:
    """One descriptor of a byte batch: its engine tuple, the object bytes it hashes, the bytes it stores and where."""

    def __init__(self, kind, desc):
        self.kind, self.desc = kind, desc
        self.src = None       # (offset, n) of the object in the source buffer, or a gather (offset, n, pitch, width, phase)
        self.stores = []      # (destination offset, stored object offsets xs or None = all, result offsets ds or None)
        self.flags, self.wrong, self.tile_base, self.win, self.rows, self.ndst = 0, False, 0, None, None, 1
        self.dst_offs = []    # destination pointer offsets (a strided item's dst[0] may lie before its region)

    def obj(self, host):
        if self.src is None:
            return host[:0]
        if len(self.src) == 2:
            o, n = self.src
            return host[o:o + n]
        o, n, pitch, width, phase = self.src
        y = np.arange(n, dtype=np.int64) + phase
        return host[o + y // width * pitch + y % width]  # the SourceRows rule

    def digest(self, bb, algo, host):
        b = self.obj(host)
        if self.kind in ("slice", "slice-hash"):
            if b.size == 0:
                return 0
            part = bb.bbh64_partial if algo == "BBH64" else bb.xxh3t64_partial
            return part(np.concatenate([np.zeros(self.tile_base * T, dtype=np.uint8), b]), self.tile_base, -(-b.size // T))
        return _model(bb, algo)(b)

    def tuple(self, src_ptr, dst_ptr, expect):
        dsts = [dst_ptr + o for o in self.dst_offs]
        s = src_ptr + (self.src[0] if self.src else 0)
        return (s, dsts, self.src[1] if self.src else 0, expect, self.flags, self.tile_base, self.win, self.rows)


ROUND_BYTES = 64 * MiB  # source bytes of a round past which its items take warp-path sizes


def make_item(bb, rng, kind, sa, da, small=False, one_dst=False):
    """A random valid item of `kind`; sa / da are the source and destination arenas.  small: warp-path sizes only."""
    it = Item(kind, "")
    ndst = 1 if one_dst else int(rng.integers(1, 4))
    small = small or sa.end > ROUND_BYTES

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
    else:  # slice, slice-hash
        n = int(rng.choice([0, _size(rng), _size(rng)]))
        it.tile_base = int(rng.choice([0, 1, 3, int(rng.integers(0, 64))]))
        it.flags = bb.XFER_RAW_SUM
        it.src = (sa.take(n), n)
        if kind == "slice":
            it.dst_offs = [da.take(n)]
            it.stores = [(it.dst_offs[0], None, None)]
        it.desc = f"{kind} n={n} tile_base={it.tile_base}"
    if kind in ("verify-ok", "verify-bad") or (kind in ("window", "strided", "gather", "zero") and rng.random() < 0.5):
        it.flags |= bb.XFER_VERIFY
        it.wrong = kind == "verify-bad" or (kind != "verify-ok" and rng.random() < 0.5)
        it.desc += " verify=" + ("wrong" if it.wrong else "right")
    return it


def _round_plan(rng, algo):
    """(mode, kinds of the items): mode 'mixed', 'small' (every item may take bb_xfer_small) or 'mailbox'."""
    r = rng.random()
    if r < 0.15:
        return "mailbox", ["whole"] * int(rng.integers(1, 9))
    if r < 0.35:
        count = int(rng.choice([int(rng.integers(1, 9)), int(rng.integers(9, 65)), int(rng.integers(65, 300))]))
        return "small", [str(rng.choice(["whole", "whole", "zero", "verify-ok", "verify-bad"])) for _ in range(count)]
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
             ((s, [], n), "INVALID_ARGUMENT")]                                                  # no destination, no RAW_SUM
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
    if not busy:
        path, want = "none", (0, 0, 0)
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


def _fp8_gather(rng):
    """(pitch, width, phase) in elements of a gathered pack: (pitch - width) % 8 == 0, phase < width."""
    width = int(rng.choice([8, 40, int(rng.integers(1, 3000))]))
    return width + 8 * int(rng.choice([0, 1, int(rng.integers(1, 40))])), width, int(rng.choice([0, int(rng.integers(0, width)), width - 1]))


def _unpack_window(rng, n):
    """None (whole), (lo, hi) or (lo, hi, pitch, width, phase) in elements, (pitch - width) % 8 == 0."""
    r = rng.random()
    if r < 0.3:
        return None
    lo, hi = sorted(int(v) for v in rng.integers(0, n + 1, 2))
    if rng.random() < 0.3 and lo >= T:  # from a tile edge +- 1
        lo = min(hi, lo // T * T + int(rng.integers(-1, 2)))
    if r < 0.6:
        return lo, hi
    width = int(rng.choice([1, 8, int(rng.integers(1, 400)), int(rng.integers(400, T))]))
    pitch = width + 8 * int(rng.choice([0, 1, int(rng.integers(1, 200))]))
    phase = int(rng.choice([0, int(rng.integers(0, pitch)), pitch - 1]))
    return lo, hi, pitch, width, phase


def fp8_round(bb, eng, seed, rnd):
    rng = np.random.default_rng([seed, rnd, 8])
    grid = _grid(rng)
    eng.set_max_ctas(grid)
    count = int(rng.integers(1, 10))
    sizes = [_fp8_size(rng) for _ in range(count)]
    xs = []
    for n in sizes:
        x = _bf16(rng, n)
        _specials(rng, x)
        xs.append(x)
    pats = [None if rng.random() < 0.5 else _fp8_gather(rng) for _ in sizes]
    nrep = [int(rng.integers(1, 4)) for _ in sizes]
    descs = [f"n={n} gather={p} replicas={r}" for n, p, r in zip(sizes, pats, nrep)]
    where = f"fp8 seed {seed} round {rnd} (grid {grid}, {count} objects)"
    packed = [model_pack(x) for x in xs]
    lay = Layout([p.size for p in packed])
    reps = [lay.guarded() for _ in range(3)]
    srcs, items = [], []  # srcs keeps the sources alive until the kernel has read them
    for x, p, r, o in zip(xs, pats, nrep, lay.offs):
        if p is None:
            s, off = torch.from_numpy(x.view(np.int16).copy()).cuda(), 0
        else:
            s, off = gathered_source(x, *p)  # the gaps hold NaN, Inf and bf16 max
        srcs.append(s)
        items.append((s.data_ptr() + 2 * off, [reps[k].data_ptr() + o for k in range(r)], x.size, None, None, p))
    dg, st, _ = eng.run_fp8(items, False, _stream())
    torch.cuda.synchronize()
    SEEN["fp8-pack"] += 1
    assert st == [0] * count, f"{where}: pack status {st}"
    for i, (p, d) in enumerate(zip(packed, dg)):
        assert d == bb.bbh64(p), f"{where}, item {i} [{descs[i]}]: digest"
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
    # unpack every object from replica 0: whole, element window or strided window, a right or a wrong expected digest
    wins = [_unpack_window(rng, n) for n in sizes]
    wrong = [bool(rng.random() < 0.25) for _ in sizes]
    ar = Arena(rng)
    bases, maps = [], []
    for n, w in zip(sizes, wins):
        if w is None:
            xs_, ds = np.arange(n), np.arange(n)
            r = ar.take(n, 0, 8)
            base = r
        elif len(w) == 2:
            xs_, ds = np.arange(w[0], w[1]), np.arange(w[0], w[1])
            r = ar.take(w[1] - w[0], w[0] % 8, 8)
            base = r - w[0]
        else:
            lo, hi, pitch, width, phase = w
            xs_, ds = stored(n, w)
            lo_d = int(ds.min()) if ds.size else 0
            res = lo_d - phase + (lo + phase) // pitch * (pitch - width)
            r = ar.take(int(ds.max()) + 1 - lo_d if ds.size else 0, res % 8, 8)
            base = r - lo_d
        bases.append(base)
        maps.append((xs_, ds))
    out = torch.full((ar.total,), GUARD16, dtype=torch.int16, device="cuda")
    gets = []
    for i, (n, w, b) in enumerate(zip(sizes, wins, bases)):
        it = (out.data_ptr() + 2 * b, reps[0].data_ptr() + lay.offs[i], n, dg[i] ^ int(wrong[i]))
        gets.append(it + ((w,) if w is not None else ()))
    dg2, st2, _ = eng.run_fp8(gets, True, _stream())
    torch.cuda.synchronize()
    SEEN["fp8-unpack"] += 1
    for i in range(count):
        assert dg2[i] == dg[i] and st2[i] == int(wrong[i]), f"{where}, item {i} [{descs[i]}, window {wins[i]}]: digest / status {st2[i]}"
    got = out.cpu().numpy().view(np.uint16)
    want = np.full(ar.total, GUARD16, dtype=np.uint16)
    for i, (b, (xs_, ds)) in enumerate(zip(bases, maps)):
        if xs_.size:
            want[b + ds] = model_unpack(packed[i], sizes[i])[xs_]
    written = np.zeros(ar.total, dtype=bool)
    for i, (b, (xs_, ds)) in enumerate(zip(bases, maps)):
        written[b + ds] = True
        lo = b + (int(ds.min()) if ds.size else 0)
        hi = b + (int(ds.max()) + 1 if ds.size else 0)
        same_bits(got[lo - 8:hi + 8], want[lo - 8:hi + 8], "bf16", f"{where}, item {i} [{descs[i]}, window {wins[i]}]: unpacked")
    outside = np.nonzero(~written & (got != GUARD16))[0]
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
    print("\ncoverage:", {str(k): v for k, v in sorted(SEEN.items(), key=str)})
    assert not missing, f"categories reached fewer than 3 times: {missing}"
