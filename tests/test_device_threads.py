"""The device data plane called from several host threads at once, against the same host models as the single-threaded
tests.

A client's device calls release the GIL, and every thread of one client shares its GpuFabric and so one XferEngine;
AsyncTensorStore(client, workers=N) runs N worker threads against one client.  Each test here starts its threads' rounds
together (threading.Barrier), each thread on its own CUDA stream with its own buffers and keys:
  - one XferEngine made with 2 slots, shared by 8 threads running random byte batches (every descriptor kind of
    test_xfer_random.py, 1-3 destinations, mailbox-sized, warp-path and CTA-run-spanning batches, every algorithm) and
    the random MXFP8 rounds of test_xfer_random.py (fp8_round): more threads than slots, so the slot table grows;
  - one GpuRankCluster client (HBM slab and pinned DRAM pool) shared by 6 threads running random sequences of every
    byte and fp8 device put and get, and removes, each result and each recorded digest checked against the host model;
  - AsyncTensorStore(client, workers=4) with dozens of futures in flight;
  - device gets racing the Keystone's tier moves, compactions and re-puts of the objects they read.
The last test checks that calls of each kind really overlapped calls of other threads.

Models trusted: numpy slicing with the SourceRows / SourcePages rules of test_xfer_random.py (rows_at, pages_at);
bb.crc32c / bb.bbh64 / bb.xxh3t64 and their _partial forms (checked in test_common.py); the exact MXFP8 models of
test_mxfp8_exhaustive.py and test_mxfp8_wide.py.  BB_RANDOM_ROUNDS=k runs k more rounds per thread."""
import collections
import os
import threading
import time

import numpy as np
import pytest
import torch

from test_device_path import _counter, _ref
from test_xfer_random import (ALGOS, GUARD, KINDS, WB, WGUARD, Arena, _pack_model, _same, _unpack_model, fp8_round, make_item,
                              pages_at)

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
EXTRA = int(os.environ.get("BB_RANDOM_ROUNDS", "0"))
ENGINE_THREADS, ENGINE_ROUNDS = 8, 14 + EXTRA
CLIENT_THREADS, CLIENT_ROUNDS = 6, 24 + EXTRA
STORE_FUTURES = 48 + 4 * EXTRA
RACE_SECONDS = 4.0 + EXTRA
LOG = []  # (test, thread, kind, start, end) of every timed call
DONE = set()  # tests of this module that ran to the end
OVERLAP_KINDS = ["put", "get", "fp8-put", "fp8-get", "mailbox"]


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    free, _ = torch.cuda.mem_get_info()
    if free < (8 << 30):
        pytest.skip(f"needs about 8 GiB of free device memory, {free >> 20} MiB free")


def _timed(test, tid, kind, fn, *args, **kw):
    t0 = time.perf_counter()
    out = fn(*args, **kw)
    LOG.append((test, tid, kind, t0, time.perf_counter()))
    return out


def _threads(n, rounds, body, barriers=()):
    """body(tid, rnd, stream) for every round on n threads, each with a stream of its own (current inside body); a barrier
    starts every round.  A failing thread also breaks `barriers`, the body's own, so that no thread waits for it.  Every
    thread is joined; the first failure is raised with its thread."""
    barrier = threading.Barrier(n)
    errors = []

    def run(tid):
        torch.cuda.set_device(0)
        s = torch.cuda.Stream()
        try:
            with torch.cuda.stream(s):
                for rnd in range(rounds):
                    barrier.wait(timeout=600)
                    body(tid, rnd, s)
            s.synchronize()
        except BaseException as e:  # pytest.fail raises a BaseException
            errors.append((tid, e))
            for b in (barrier, *barriers):  # the other threads stop at their next barrier
                b.abort()

    ts = [threading.Thread(target=run, args=(i,), name=f"bb-test-{i}") for i in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    real = [e for e in errors if not isinstance(e[1], threading.BrokenBarrierError)] or errors
    if real:
        tid, e = real[0]
        raise AssertionError(f"thread {tid}: {e}") from e


# ---------------------------------------------------------------------------------------------------- one shared engine


def _byte_mode(tid, rnd):
    """The generator of engine_byte_round and its mode: 'mailbox', 'small' or 'mixed'."""
    rng = np.random.default_rng([71, tid, rnd])
    algo = ALGOS[int(rng.integers(0, 4))]
    r = rng.random()
    return rng, algo, "mailbox" if r < 0.3 else "small" if r < 0.5 else "mixed"


def engine_byte_round(bb, eng, tid, rnd, s, held=None):
    """A random byte batch through the shared engine on stream s: digests, verify status, every destination and guard
    byte.  Mailbox rounds are 1-8 single-destination objects of at most 4 KiB on an idle stream.  With `held` (a pair of
    barriers) the batch is submitted, held in flight across both and only then waited for; otherwise it is run."""
    rng, algo, mode = _byte_mode(tid, rnd)
    if mode == "mailbox":
        mode, kinds = "mailbox", ["whole"] * int(rng.integers(1, 9))
    elif mode == "small":
        kinds = [str(rng.choice(["whole", "whole", "zero", "verify-ok", "verify-bad"])) for _ in range(int(rng.integers(1, 100)))]
    else:
        usable = [k for k in KINDS if algo in ("BBH64", "XXH3") or not k.startswith("slice")]
        count = int(rng.choice([int(rng.integers(1, 9)), int(rng.integers(9, 65)), int(rng.integers(65, 200))]))
        kinds = [str(rng.choice(usable)) for _ in range(count)]
    sa, da = Arena(rng), Arena(rng)
    items = [make_item(bb, rng, k, sa, da, small=mode != "mixed", one_dst=mode == "mailbox") for k in kinds]
    where = f"thread {tid} round {rnd} ({algo}, {mode}, {len(items)} items)"
    host = rng.integers(0, 256, sa.total, dtype=np.uint8)
    digests = [it.digest(bb, algo, host) for it in items]
    src = torch.from_numpy(host).cuda()
    dst = torch.full((da.total,), GUARD, dtype=torch.uint8, device="cuda")
    tuples = [it.tuple(src.data_ptr(), dst.data_ptr(), d ^ 1 if it.wrong else d) for it, d in zip(items, digests)]
    if mode == "mailbox":
        s.synchronize()  # the mailbox serves only an idle caller stream
    kind = "mailbox" if mode == "mailbox" else "bytes"
    t0 = time.perf_counter()
    if held is None:
        dg, st, _ = eng.run(tuples, getattr(bb.ChecksumAlgo, algo), s.cuda_stream)
    else:
        ticket = eng.submit(tuples, getattr(bb.ChecksumAlgo, algo), s.cuda_stream)
        for b in held:
            b.wait(timeout=600)
        dg, st, _ = eng.wait(ticket)
    LOG.append(("engine", tid, kind, t0, time.perf_counter()))
    for i, (it, d, v) in enumerate(zip(items, dg, st)):
        want_d = 0 if algo == "NONE" else digests[i]
        want_s = int(algo != "NONE" and bool(it.flags & bb.XFER_VERIFY) and it.wrong)
        assert d == want_d and v == want_s, f"{where}, item {i} [{it.desc}]: digest {d:#x} status {v}, want {want_d:#x} status {want_s}"
    want = np.full(dst.numel(), GUARD, dtype=np.uint8)
    for it in items:
        b = it.obj(host)
        for base, xs, ds in it.stores:
            if xs is None:
                want[base:base + b.size] = b
            elif xs.size:
                want[base + ds] = b[xs]
    got = dst.cpu().numpy()
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{where}: {bad.size} destination bytes differ, first at {bad[:4].tolist()}"


class _ThreadEngine:
    """The shared engine as fp8_round drives it from one thread: the grid stays the engine's (set_max_ctas is
    engine-wide), launches counts this thread's calls that returned, and every call is timed."""

    def __init__(self, eng, tid):
        self.eng, self.tid, self.launches, self.small_launches = eng, tid, 0, 0

    def set_max_ctas(self, n):
        pass

    def run_fp8(self, items, unpack, stream, wide):
        out = _timed("engine", self.tid, "fp8-get" if unpack else "fp8-put", self.eng.run_fp8, items, unpack, stream, wide=wide)
        self.launches += 1
        return out


def _is_byte_round(tid, rnd):
    return np.random.default_rng([72, tid, rnd]).random() < 0.7


def test_one_engine_shared_by_eight_threads(bb):
    """8 threads share one XferEngine created with 2 slots: byte rounds and fp8 rounds (pack then unpack) with results
    exact against the models.  In odd rounds every call runs as it comes.  In even rounds every byte thread submits its
    batch and holds it in flight while the fp8 threads run their packs and unpacks, and only then waits: as many slots
    are held at once as the round has byte threads, so the table must grow past 2, and every fp8 call overlaps every
    held batch.  The first mailbox-sized batch of such a round finds the mailbox idle and is served by it."""
    eng = bb.XferEngine(0, 4096, 2)
    m0 = eng.mailbox_requests
    submitted, fp8_done = threading.Barrier(ENGINE_THREADS), threading.Barrier(ENGINE_THREADS)

    def body(tid, rnd, s):
        held = rnd % 2 == 0
        if _is_byte_round(tid, rnd):
            engine_byte_round(bb, eng, tid, rnd, s, held=(submitted, fp8_done) if held else None)
            return
        if held:
            submitted.wait(timeout=600)
        fp8_round(bb, _ThreadEngine(eng, tid), 1000 + tid, rnd)
        if held:
            fp8_done.wait(timeout=600)

    _threads(ENGINE_THREADS, ENGINE_ROUNDS, body, barriers=(submitted, fp8_done))
    # the plan is fixed by the seeds: the most byte threads of one held round, and whether a held round mails a batch
    held_rounds = range(0, ENGINE_ROUNDS, 2)
    most = max(sum(_is_byte_round(t, r) for t in range(ENGINE_THREADS)) for r in held_rounds)
    mailed = any(_is_byte_round(t, r) and _byte_mode(t, r)[2] == "mailbox" for r in held_rounds for t in range(ENGINE_THREADS))
    print(f"\nengine: {eng.slots} slots (at most {most} batches held at once), {eng.launches} launches, "
          f"{eng.mailbox_requests - m0} mailbox requests")
    assert most > 2 and mailed, "the seeds no longer give a held round of 3 byte threads and a mailed batch"
    assert eng.slots >= most, f"{most} batches were in flight at once on {eng.slots} slots"
    assert eng.mailbox_requests > m0
    DONE.add("engine")


# ---------------------------------------------------------------------------------------------------- one shared client


def _cluster(cid, tmp_path=None):
    from blackbird_b200.parallel import GpuRankCluster

    kw = dict(nvme_bytes=512 << 20, nvme_path=str(tmp_path)) if tmp_path is not None else {}
    return GpuRankCluster(slab_bytes=4 << 30, cluster_id=cid, dram_bytes=512 << 20, high_watermark=1.0, **kw)


def _cfg(bb, algo, tier="RAM_GPU"):
    return bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[getattr(bb.StorageClass, tier)])


def _mx(bb, w):
    return {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}[w]


def _wide_bits(rng, n, w):
    """n finite patterns of type w, block by block across many binades."""
    field, lo, hi, mant, sign = {"bf16": (7, 60, 200, 7, 15), "f16": (10, 2, 31, 10, 15), "f32": (23, 60, 200, 23, 31)}[w]
    top = rng.integers(lo, hi, n // 32)[:, None]
    e = np.clip(top - rng.integers(0, 10, (n // 32, 32)), 0, hi - 1)
    bits = (e << field) | rng.integers(0, 1 << mant, (n // 32, 32)) | (rng.integers(0, 2, (n // 32, 32)) << sign)
    return bits.reshape(-1).astype(np.uint32 if w == "f32" else np.uint16)


def _dev(a):
    """A device copy of host array a (any dtype), as bytes, on the current stream."""
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def _aligned(rng, sizes, unit=16):
    """Offsets of regions of the given byte sizes in one buffer, 16-byte aligned, 16 to 64 guard bytes apart; the total."""
    offs, o = [], 64
    for n in sizes:
        offs.append(o)
        o = (o + n + 16 + int(rng.integers(0, 4)) * 16 + 15) // 16 * 16
    return offs, o + 64


class ClientThread:
    """One thread's share of a client: its own keys, stream and host model of what it stored."""

    def __init__(self, bb, cl, tid, s):
        self.bb, self.cl, self.c, self.tid, self.s = bb, cl, cl.client, tid, s
        self.rng = np.random.default_rng([73, tid])
        self.objs, self.fp8, self.gone, self.next, self.rnd = {}, {}, [], 0, 0
        self.ops = collections.Counter()

    def where(self, what):
        return f"thread {self.tid} round {self.rnd}: {what}"

    def key(self):
        self.next += 1
        return f"t{self.tid}/k{self.next}"

    def size(self, small):
        rng = self.rng
        if small:
            return int(rng.integers(1, 4097))
        return int(rng.choice([int(rng.integers(1, 4097)), int(rng.integers(4097, 3 * T)), int(rng.integers(3 * T, 2 * MiB))]))

    def check_digest(self, key, algo, blob):
        sh = self.c.get_workers(key)[0].shards
        assert len(sh) == 1 and sh[0].checksum == _ref(self.bb, algo)(blob), self.where(f"{key}: recorded digest")

    # -------------------------------------------------------------------------------------------- byte puts
    def put(self):
        bb, rng = self.bb, self.rng
        small = rng.random() < 0.3
        count = 1 if small else int(rng.integers(1, 6))
        form = "plain" if small else str(rng.choice(["plain", "strided", "paged"]))
        algo, tier = ALGOS[int(rng.integers(0, 4))], str(rng.choice(["RAM_GPU", "RAM_CPU"]))
        keys = [self.key() for _ in range(count)]
        blobs = [rng.integers(0, 256, self.size(small), dtype=np.uint8) for _ in keys]
        cfg = _cfg(bb, algo, tier)
        kind = "mailbox" if small else "put"
        if form == "plain":
            offs, total = _aligned(rng, [b.size for b in blobs])
            buf = rng.integers(0, 256, total, dtype=np.uint8)
            for o, b in zip(offs, blobs):
                buf[o:o + b.size] = b
            src = _dev(buf)
            ecs = _timed("client", self.tid, kind, self.c.batch_put_device, keys, [src.data_ptr() + o for o in offs],
                         [b.size for b in blobs], cfg, self.s.cuda_stream)
        elif form == "strided":
            shapes = []
            for i, b in enumerate(blobs):
                width = int(rng.integers(1, min(b.size, 3000) + 1))
                rows = b.size // width
                blobs[i] = b[:rows * width]
                shapes.append((width, width + 16 * int(rng.integers(0, 20)), rows))
            offs, total = _aligned(rng, [(r - 1) * p + w for w, p, r in shapes])
            buf = rng.integers(0, 256, total, dtype=np.uint8)
            for o, b, (w, p, r) in zip(offs, blobs, shapes):
                for j in range(r):
                    buf[o + j * p:o + j * p + w] = b[j * w:(j + 1) * w]
            src = _dev(buf)
            ecs = _timed("client", self.tid, kind, self.c.batch_put_device_strided, keys, [src.data_ptr() + o for o in offs],
                         *[[sh[k] for sh in shapes] for k in range(3)], cfg, self.s.cuda_stream)
        else:
            pages, page_bytes, bufs = [], [], []
            for i, b in enumerate(blobs):
                page = 16 * int(rng.choice([1, 7, 64, 256, int(rng.integers(1, 600))]))
                npg = max(1, b.size // page)
                blobs[i] = b = rng.integers(0, 256, npg * page, dtype=np.uint8)
                slots = rng.permutation(npg + 2)[:npg]  # pages in random order, with unused slots between them
                buf = rng.integers(0, 256, (npg + 2) * page, dtype=np.uint8)
                for j, sl in enumerate(slots):
                    buf[sl * page:(sl + 1) * page] = b[j * page:(j + 1) * page]
                bufs.append(_dev(buf))
                pages.append([bufs[-1].data_ptr() + int(sl) * page for sl in slots])
                page_bytes.append(page)
            ecs = _timed("client", self.tid, kind, self.c.batch_put_device_paged, keys, pages, page_bytes, cfg, self.s.cuda_stream)
        assert ecs == [bb.ErrorCode.OK] * count, self.where(f"{form} put of {[b.size for b in blobs]}: {ecs}")
        for k, b in zip(keys, blobs):
            self.check_digest(k, algo, b)
            self.objs[k] = b
        self.ops[f"put {form}"] += 1

    # -------------------------------------------------------------------------------------------- byte gets
    def get(self):
        bb, rng = self.bb, self.rng
        if not self.objs:
            return self.put()
        names = sorted(self.objs)
        small = rng.random() < 0.3
        keys = [str(rng.choice(names)) for _ in range(1 if small else int(rng.integers(1, 6)))]
        form = "whole" if small else str(rng.choice(["whole", "range", "strided", "scatter", "paged"]))
        if small and self.objs[keys[0]].size > 4096:
            small = False
        # (bytes of the result region, object bytes xs -> region offsets ds, call arguments); a range or strided get's
        # pointer is shifted so that its virtual base (pointer - offset) is 16-byte aligned (the fused kernel), or in some
        # gets not (the host-staged path)
        plans = []
        for k in keys:
            b = self.objs[k]
            n = b.size
            if form == "whole":
                plans.append((n + 16, np.arange(n), np.arange(n), (n + 16,)))
            elif form == "range":
                off = int(rng.integers(0, n))
                ln = int(rng.integers(1, n - off + 1))
                sh = off % 16 if rng.random() < 0.8 else 0
                plans.append((ln + 16, np.arange(off, off + ln), sh + np.arange(ln), (off, ln), sh))
            elif form == "strided":
                off = int(rng.integers(0, n))
                width = int(rng.integers(1, min(n - off, 2000) + 1))
                pitch = width + 16 * int(rng.integers(0, 30))
                rows = int(rng.integers(1, 2 + (n - off - width) // max(pitch, 1)))
                xs = np.concatenate([np.arange(off + r * pitch, off + r * pitch + width) for r in range(rows)])
                sh = off % 16 if rng.random() < 0.8 else 0
                plans.append((rows * width + 16, xs, sh + np.arange(xs.size), (off, width, pitch, rows), sh))
            elif form == "scatter":
                width = int(rng.integers(1, min(n, 3000) + 1))
                pitch = width + 16 * int(rng.integers(0, 20))
                rows = -(-n // width)
                ds = np.arange(n) // width * pitch + np.arange(n) % width
                plans.append(((rows - 1) * pitch + width, np.arange(n), ds, (width, pitch, rows)))
            else:
                page = 16 * int(rng.choice([1, 5, 64, 256, int(rng.integers(1, 600))]))
                npg = -(-n // page) + int(rng.integers(0, 2))
                slots = rng.permutation(npg + 1)[:npg]
                plans.append(((npg + 1) * page, np.arange(n), pages_at(n, slots * page, page, 0), (slots, page)))
        offs, total = _aligned(rng, [p[0] for p in plans])
        out = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
        p0, st = out.data_ptr(), self.s.cuda_stream
        ptrs = [p0 + o + (p[4] if len(p) > 4 else 0) for o, p in zip(offs, plans)]
        kind = "mailbox" if small else "get"
        col = lambda j: [p[3][j] for p in plans]  # noqa: E731
        if form == "whole":
            ecs, sizes = _timed("client", self.tid, kind, self.c.batch_get_device, keys, ptrs, col(0), st)
            assert sizes == [self.objs[k].size for k in keys], self.where(f"sizes {sizes}")
        elif form == "range":
            ecs = _timed("client", self.tid, kind, self.c.batch_get_device_range, keys, ptrs, col(0), col(1), st)
        elif form == "strided":
            ecs = _timed("client", self.tid, kind, self.c.batch_get_device_strided, keys, ptrs, col(0), col(1), col(2), col(3), st)
        elif form == "scatter":
            ecs, _ = _timed("client", self.tid, kind, self.c.batch_get_device_scatter, keys, ptrs, col(0), col(1), col(2), st)
        else:
            pages = [[p0 + o + int(sl) * p[3][1] for sl in p[3][0]] for o, p in zip(offs, plans)]
            ecs, _ = _timed("client", self.tid, kind, self.c.batch_get_device_paged, keys, pages, col(1), st)
        assert ecs == [bb.ErrorCode.OK] * len(keys), self.where(f"{form} get of {keys}: {ecs}")
        want = np.full(total, GUARD, dtype=np.uint8)
        for k, o, p in zip(keys, offs, plans):
            want[o + p[2]] = self.objs[k][p[1]]
        got = out.cpu().numpy()
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, self.where(f"{form} get of {keys}: {bad.size} bytes differ, first at {bad[:4].tolist()} (regions {offs})")
        self.ops[f"get {form}"] += 1

    # -------------------------------------------------------------------------------------------- fp8 puts and gets
    def put_fp8(self):
        bb, rng = self.bb, self.rng
        count, w = int(rng.integers(1, 4)), str(rng.choice(["bf16", "f16", "f32"]))
        form, tier = str(rng.choice(["plain", "strided", "paged"])), str(rng.choice(["RAM_GPU", "RAM_CPU"]))
        b = WB[w]
        keys = [self.key() for _ in range(count)]
        xs, keep = [], []
        cfg = _cfg(bb, "BBH64", tier)
        if form == "plain":
            for _ in keys:
                xs.append(_wide_bits(rng, 32 * int(rng.choice([int(rng.integers(1, 200)), int(rng.integers(T // 32 - 1, 3 * T // 32))])), w))
                keep.append(_dev(xs[-1]))
            args = ([t.data_ptr() for t in keep], [x.size for x in xs])
            call = self.c.batch_put_device_fp8
        elif form == "strided":
            shapes = []
            for _ in keys:
                width = 32 * int(rng.integers(1, 9))
                pitch, rows = width + (16 // b) * int(rng.integers(0, 20)), int(rng.integers(1, 60))
                x = _wide_bits(rng, width * rows, w)
                buf = np.zeros((rows - 1) * pitch + width, dtype=x.dtype)
                for r in range(rows):
                    buf[r * pitch:r * pitch + width] = x[r * width:(r + 1) * width]
                xs.append(x)
                keep.append(_dev(buf))
                shapes.append((width, pitch, rows))
            args = ([t.data_ptr() for t in keep], *[[sh[k] for sh in shapes] for k in range(3)])
            call = self.c.batch_put_device_fp8_strided
        else:
            pages, page_elems = [], []
            for _ in keys:
                page, npg = 32 * int(rng.choice([1, 3, 16, int(rng.integers(1, 40))])), int(rng.integers(1, 30))
                x = _wide_bits(rng, page * npg, w)
                slots = rng.permutation(npg + 1)[:npg]
                buf = np.zeros((npg + 1) * page, dtype=x.dtype)
                for j, sl in enumerate(slots):
                    buf[sl * page:(sl + 1) * page] = x[j * page:(j + 1) * page]
                xs.append(x)
                keep.append(_dev(buf))
                pages.append([keep[-1].data_ptr() + int(sl) * page * b for sl in slots])
                page_elems.append(page)
            args = (pages, page_elems)
            call = self.c.batch_put_device_fp8_paged
        ecs = _timed("client", self.tid, "fp8-put", call, keys, *args, cfg, self.s.cuda_stream, wide=_mx(bb, w))
        assert ecs == [bb.ErrorCode.OK] * count, self.where(f"{form} fp8 put of {w} {[x.size for x in xs]}: {ecs}")
        for k, x in zip(keys, xs):
            packed = _pack_model(x, w)
            self.check_digest(k, "BBH64", packed)
            self.fp8[k] = (x.size, packed, {})
        self.ops[f"fp8 put {form} {w}"] += 1

    def back(self, key, w):
        """What an fp8 get of type w stores: the unpack of the packed bytes in that type."""
        n, packed, cache = self.fp8[key]
        if w not in cache:
            cache[w] = _unpack_model(packed, n, w)
        return cache[w]

    def get_fp8(self):
        bb, rng = self.bb, self.rng
        if not self.fp8:
            return self.put_fp8()
        names = sorted(self.fp8)
        keys = [str(rng.choice(names)) for _ in range(int(rng.integers(1, 4)))]
        w = str(rng.choice(["bf16", "f16", "f32"]))  # the get's type, whatever type packed the object
        b = WB[w]
        per = 16 // b
        form = str(rng.choice(["whole", "range", "strided", "scatter", "paged"]))
        plans = []  # (elements of the result region, object elements xs -> region elements ds, call arguments)
        for k in keys:
            n = self.fp8[k][0]
            if form == "whole":
                plans.append((n, np.arange(n), np.arange(n), (n,)))
            elif form == "range":
                off = int(rng.integers(0, n))
                ln = int(rng.integers(1, n - off + 1))
                sh = off % per  # the virtual base (pointer - b * offset) 16-byte aligned, as the fused unpack needs
                plans.append((ln + per, np.arange(off, off + ln), sh + np.arange(ln), (n, off, ln), sh))
            elif form == "strided":
                off = int(rng.integers(0, n))
                width = int(rng.integers(1, min(n - off, 2000) + 1))
                pitch = width + per * int(rng.integers(0, 30))
                rows = int(rng.integers(1, 2 + (n - off - width) // max(pitch, 1)))
                xs = np.concatenate([np.arange(off + r * pitch, off + r * pitch + width) for r in range(rows)])
                sh = off % per
                plans.append((xs.size + per, xs, sh + np.arange(xs.size), (n, off, width, pitch, rows), sh))
            elif form == "scatter":
                divs = [d for d in (1, 2, 3, 4, 8, 16) if n % d == 0]
                rows = int(rng.choice(divs))
                width = n // rows
                pitch = width + per * int(rng.integers(0, 20))
                ds = np.arange(n) // width * pitch + np.arange(n) % width
                plans.append(((rows - 1) * pitch + width, np.arange(n), ds, (n, width, pitch, rows)))
            else:
                blocks = n // 32
                page = 32 * int(rng.choice([d for d in (1, 2, 3, 4, 8, 16, blocks) if blocks % d == 0]))
                npg = n // page
                slots = rng.permutation(npg + 1)[:npg]
                plans.append(((npg + 1) * page, np.arange(n), pages_at(n, slots * page, page, 0), (slots, page)))
        offs, total = _aligned(rng, [p[0] * b for p in plans])
        out = torch.full((total // b,), WGUARD[b], dtype=torch.int16 if b == 2 else torch.int32, device="cuda")
        p0, st = out.data_ptr(), self.s.cuda_stream
        ptrs = [p0 + o + b * (p[4] if len(p) > 4 else 0) for o, p in zip(offs, plans)]
        col = lambda j: [p[3][j] for p in plans]  # noqa: E731
        mx = _mx(bb, w)
        if form == "whole":
            ecs = _timed("client", self.tid, "fp8-get", self.c.batch_get_device_fp8, keys, ptrs, col(0), st, wide=mx)
        elif form == "range":
            ecs = _timed("client", self.tid, "fp8-get", self.c.batch_get_device_fp8_range, keys, ptrs, col(0), col(1), col(2), st, wide=mx)
        elif form == "strided":
            ecs = _timed("client", self.tid, "fp8-get", self.c.batch_get_device_fp8_strided, keys, ptrs, col(0), col(1), col(2), col(3),
                         col(4), st, wide=mx)
        elif form == "scatter":
            ecs = _timed("client", self.tid, "fp8-get", self.c.batch_get_device_fp8_scatter, keys, ptrs, col(0), col(1), col(2), col(3),
                         st, wide=mx)
        else:
            pages = [[p0 + o + int(sl) * p[3][1] * b for sl in p[3][0]] for o, p in zip(offs, plans)]
            ecs = _timed("client", self.tid, "fp8-get", self.c.batch_get_device_fp8_paged, keys, pages, col(1), st, wide=mx)
        assert ecs == [bb.ErrorCode.OK] * len(keys), self.where(f"{form} fp8 get as {w} of {keys}: {ecs}")
        got = out.cpu().numpy().view(np.uint16 if b == 2 else np.uint32)
        want = np.full(got.size, WGUARD[b], dtype=got.dtype)
        for k, o, p in zip(keys, offs, plans):
            want[o // b + p[2]] = self.back(k, w)[p[1]]
        _same(got, want, w, self.where(f"{form} fp8 get as {w} of {keys} (regions {offs})"))
        self.ops[f"fp8 get {form} {w}"] += 1

    def remove(self):
        bb, rng = self.bb, self.rng
        pool = sorted(self.objs) + sorted(self.fp8)
        if len(pool) < 4:
            return self.put()
        ks = [str(k) for k in rng.choice(pool, int(rng.integers(1, 3)), replace=False)]
        assert self.c.batch_remove(ks) == [bb.ErrorCode.OK] * len(ks), self.where(f"remove {ks}")
        for k in ks:
            self.objs.pop(k, None)
            self.fp8.pop(k, None)
        out = torch.zeros(64, dtype=torch.uint8, device="cuda")
        ecs, _ = self.c.batch_get_device(ks[:1], [out.data_ptr()], [64], self.s.cuda_stream)
        assert ecs == [bb.ErrorCode.OBJECT_NOT_FOUND], self.where(f"get of removed {ks[0]}: {ecs}")
        self.ops["remove"] += 1

    def step(self, rnd):
        self.rnd = rnd
        ops = [self.put, self.get, self.put_fp8, self.get_fp8, self.remove]
        op = ops[int(self.rng.choice(len(ops), p=[0.25, 0.3, 0.15, 0.2, 0.1]))] if rnd >= 2 else ops[rnd * 2]
        op()


def test_one_client_shared_by_six_threads(bb):
    """6 threads share one client: random byte and fp8 device puts and gets of every shape, and removes; every call OK,
    every result and guard byte exact, every recorded digest the model's.  One thread also moves a batch of two 260 MiB
    objects, which the client pipelines in two chunks."""
    cl = _cluster("t-threads-client")
    try:
        cl.client.set_device_pipeline_chunks(2)
        state = {}
        big = {}

        def body(tid, rnd, s):
            if tid not in state:
                state[tid] = ClientThread(bb, cl, tid, s)
            state[tid].step(rnd)
            if tid == 0 and rnd == CLIENT_ROUNDS // 2:  # a pipelined batch, amid the other threads' calls
                n = 260 * MiB
                src = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
                bb.random_fill(src.data_ptr(), src.numel(), 99, s.cuda_stream)
                keys = ["t0/big0", "t0/big1"]
                ecs = _timed("client", 0, "put", cl.client.batch_put_device, keys, [src.data_ptr(), src.data_ptr() + n], [n, n],
                             _cfg(bb, "CRC32C"), s.cuda_stream)
                assert ecs == [bb.ErrorCode.OK] * 2, ecs
                out = torch.zeros_like(src)
                ecs, sizes = _timed("client", 0, "get", cl.client.batch_get_device, keys, [out.data_ptr(), out.data_ptr() + n], [n, n],
                                    s.cuda_stream)
                assert ecs == [bb.ErrorCode.OK] * 2 and sizes == [n, n], ecs
                s.synchronize()
                assert torch.equal(out, src), "pipelined get"
                host = src.cpu().numpy()
                for i, k in enumerate(keys):
                    assert cl.client.get_workers(k)[0].shards[0].checksum == bb.crc32c(host[i * n:(i + 1) * n]), k
                big["done"] = True
                assert cl.client.batch_remove(keys) == [bb.ErrorCode.OK] * 2

        _threads(CLIENT_THREADS, CLIENT_ROUNDS, body)
        ops = collections.Counter()
        for t in state.values():
            ops.update(t.ops)
        print(f"\nclient operations: {dict(sorted(ops.items()))}")
        assert big.get("done")
        for op in ("put plain", "put strided", "put paged", "get whole", "get range", "get strided", "get scatter", "get paged"):
            assert ops[op] > 0, f"no {op} in {CLIENT_ROUNDS} rounds of {CLIENT_THREADS} threads"
        assert sum(v for k, v in ops.items() if k.startswith("fp8 put")) > 3 and sum(v for k, v in ops.items() if k.startswith("fp8 get")) > 3
    finally:
        cl.stop()
    DONE.add("client")


# ---------------------------------------------------------------------------------------------------- AsyncTensorStore


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy().view(np.uint16 if t.element_size() == 2 else np.uint32)


def _packed_back(t):
    """What a pack_fp8 put + get of tensor t returns, from the exact model (w = t's type)."""
    w = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}[t.dtype]
    x = _bits(t.contiguous()).reshape(-1)
    return _unpack_model(_pack_model(x, w), x.size, w), w


def test_async_tensor_store_with_four_workers(bb):
    """AsyncTensorStore(workers=4): dozens of put_async, get_async, get_into_async, put_blocks_async and
    get_blocks_into_async futures in flight at once; results equal torch exactly, and the exact model for pack_fp8."""
    from blackbird_b200.ops import AsyncTensorStore

    cl = _cluster("t-threads-async")
    ts = AsyncTensorStore(cl.client, workers=4)
    try:
        g = torch.Generator(device="cuda").manual_seed(5)
        dtypes = [torch.bfloat16, torch.float16, torch.float32]
        jobs = []  # (key, tensor, pack_fp8, ids, dim) of the puts
        futs = []
        for i in range(STORE_FUTURES):
            dt = dtypes[i % 3]
            if i % 4 == 3:  # the blocks of a paged cache
                cache = torch.randn(3, 24, 16, 64, device="cuda", generator=g).to(dt)
                ids = torch.randperm(24, device="cpu", generator=torch.Generator().manual_seed(i))[:5].tolist()
                jobs.append((f"a/{i}", cache, i % 8 == 7, ids, 1))
                futs.append(ts.put_blocks_async([f"a/{i}"], [cache], [ids], dim=1, pack_fp8=i % 8 == 7))
            else:
                shape = [(64,), (33, 96), (1024, 160)][i % 4]
                t = torch.randn(*shape, device="cuda", generator=g).to(dt) * (1 + i)
                pack = i % 5 == 0
                jobs.append((f"a/{i}", t, pack, None, None))
                futs.append(ts.put_async([f"a/{i}"], [t], pack_fp8=pack))
        assert [f.result(timeout=300) for f in futs] == [1] * len(futs)

        def want_of(key, t, pack, ids, dim):
            src = t if ids is None else t.index_select(dim, torch.tensor(ids, device=t.device))
            if not pack:
                return _bits(src).reshape(-1), None
            return _packed_back(src)

        gets, intos, blocks = [], [], []
        for key, t, pack, ids, dim in jobs:
            if ids is not None:
                cache = torch.zeros_like(t)
                blocks.append((key, t, pack, ids, dim, cache, ts.get_blocks_into_async([key], [cache], [ids], dim=dim)))
            elif int(key.split("/")[1]) % 2:
                out = torch.zeros_like(t)
                intos.append((key, t, pack, out, ts.get_into_async([key], [out])))
            else:
                gets.append((key, t, pack, ts.get_async([key])))
        for key, t, pack, fut in gets:
            (got,) = fut.result(timeout=300)
            want, w = want_of(key, t, pack, None, None)
            assert got.shape == t.shape and got.dtype == t.dtype, key
            if w is None:
                assert np.array_equal(_bits(got).reshape(-1), want), key
            else:
                _same(_bits(got).reshape(-1), want, w, key)
        for key, t, pack, out, fut in intos:
            assert fut.result(timeout=300)[0] is out
            want, w = want_of(key, t, pack, None, None)
            if w is None:
                assert np.array_equal(_bits(out).reshape(-1), want), key
            else:
                _same(_bits(out).reshape(-1), want, w, key)
        for key, t, pack, ids, dim, cache, fut in blocks:
            assert fut.result(timeout=300)[0] is cache
            want, w = want_of(key, t, pack, ids, dim)
            got = _bits(cache.index_select(dim, torch.tensor(ids, device=cache.device))).reshape(-1)
            if w is None:
                assert np.array_equal(got, want), key
            else:
                _same(got, want, w, key)
            rest = [j for j in range(cache.shape[dim]) if j not in ids]
            assert not bool(cache.index_select(dim, torch.tensor(rest, device=cache.device)).view(-1).ne(0).any()), f"{key}: wrote outside its blocks"
    finally:
        ts.close()
        cl.stop()
    DONE.add("async")


# ---------------------------------------------------------------------------------------------------- gets racing tier moves


def test_device_gets_race_tier_moves_on_the_gpu(bb, tmp_path):
    """Reader threads run byte, range and fp8 device gets on one shared client while the main thread removes and re-puts
    objects, compacts the HBM slab and moves objects between HBM, DRAM and (byte objects only) NVMe.  A get answers OK
    with exact bytes, OBJECT_NOT_FOUND or OBJECT_NOT_READY: never CHECKSUM_MISMATCH for an intact object, never wrong
    bytes."""
    E = bb.ErrorCode
    cl = _cluster("t-threads-race", tmp_path)
    try:
        rng = np.random.default_rng(81)
        algos = ["XXH3", "CRC32C", "BBH64"]
        names = [f"r/{i}" for i in range(12)]
        blobs = {k: rng.integers(0, 256, int(rng.integers(1000, 3 * MiB)), dtype=np.uint8) for k in names}
        algo_of = {k: algos[i % 3] for i, k in enumerate(names)}
        fnames = [f"f/{i}" for i in range(6)]
        fx = {k: _wide_bits(rng, 32 * int(rng.integers(1, 3 * T // 32)), "bf16") for k in fnames}
        fback = {k: _unpack_model(_pack_model(x, "bf16"), x.size, "bf16") for k, x in fx.items()}
        srcs = {k: _dev(v) for k, v in blobs.items()}
        fsrcs = {k: _dev(x) for k, x in fx.items()}
        st = torch.cuda.current_stream().cuda_stream
        for k in names:
            assert cl.client.batch_put_device([k], [srcs[k].data_ptr()], [blobs[k].size], _cfg(bb, algo_of[k]), st) == [E.OK]
        for k in fnames:
            assert cl.client.batch_put_device_fp8([k], [fsrcs[k].data_ptr()], [fx[k].size], _cfg(bb, "BBH64"), st) == [E.OK]
        torch.cuda.synchronize()
        refresh0 = _counter(cl.client, "get_placement_refresh_total")
        stop = threading.Event()
        errors, reads = [], collections.Counter()
        allowed = (E.OBJECT_NOT_FOUND, E.OBJECT_NOT_READY)

        def reader(tid):
            torch.cuda.set_device(0)
            s = torch.cuda.Stream()
            r = np.random.default_rng([82, tid])
            try:
                with torch.cuda.stream(s):
                    while not stop.is_set():
                        op = int(r.integers(0, 3))
                        if op < 2:
                            ks = [str(k) for k in r.choice(names, 3, replace=False)]
                            offs, total = _aligned(r, [blobs[k].size for k in ks])
                            out = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
                            ptrs = [out.data_ptr() + o for o in offs]
                            if op == 0:
                                ecs, _ = _timed("race", tid, "get", cl.client.batch_get_device, ks, ptrs, [blobs[k].size for k in ks], s.cuda_stream)
                                spans = [(0, blobs[k].size) for k in ks]
                            else:
                                spans = []
                                for k in ks:
                                    a = int(r.integers(0, blobs[k].size))
                                    spans.append((a, int(r.integers(1, blobs[k].size - a + 1))))
                                ptrs = [p + a % 16 for p, (a, _) in zip(ptrs, spans)]
                                ecs = _timed("race", tid, "get", cl.client.batch_get_device_range, ks, ptrs, [a for a, _ in spans],
                                             [n for _, n in spans], s.cuda_stream)
                            got = out.cpu().numpy()
                            for k, o, (a, n), ec in zip(ks, offs, spans, ecs):
                                o += a % 16 if op == 1 else 0
                                if ec == E.OK:
                                    if not np.array_equal(got[o:o + n], blobs[k][a:a + n]):
                                        errors.append((k, "wrong bytes"))
                                elif ec not in allowed:
                                    errors.append((k, str(ec)))
                        else:
                            ks = [str(k) for k in r.choice(fnames, 2, replace=False)]
                            offs, total = _aligned(r, [2 * fx[k].size for k in ks])
                            out = torch.full((total // 2,), WGUARD[2], dtype=torch.int16, device="cuda")
                            ecs = _timed("race", tid, "fp8-get", cl.client.batch_get_device_fp8, ks, [out.data_ptr() + o for o in offs],
                                         [fx[k].size for k in ks], s.cuda_stream)
                            got = out.cpu().numpy().view(np.uint16)
                            for k, o, ec in zip(ks, offs, ecs):
                                if ec == E.OK:
                                    if not np.array_equal(got[o // 2:o // 2 + fx[k].size], fback[k]):
                                        errors.append((k, "wrong values"))
                                elif ec not in allowed:
                                    errors.append((k, str(ec)))
                        reads[tid] += 1
            except BaseException as e:
                errors.append((f"reader {tid}", repr(e)))

        threads = [threading.Thread(target=reader, args=(i,), name=f"bb-reader-{i}") for i in range(3)]
        for t in threads:
            t.start()
        moves, compacted = collections.Counter(), 0
        try:
            api = cl.client.keystone()
            t_end = time.time() + RACE_SECONDS
            while time.time() < t_end and not errors:
                k = str(rng.choice(names))
                assert cl.client.remove(k) == E.OK
                compacted += api.compact_pool("hbm0", 8)
                assert cl.client.batch_put_device([k], [srcs[k].data_ptr()], [blobs[k].size], _cfg(bb, algo_of[k]), st) == [E.OK]
                k2 = str(rng.choice([x for x in names if x != k]))
                tier = str(rng.choice(["RAM_GPU", "RAM_CPU", "NVME"]))
                assert cl.client.migrate(k2, getattr(bb.StorageClass, tier)) == E.OK, (k2, tier)
                moves[tier] += 1
                f = str(rng.choice(fnames))
                ftier = str(rng.choice(["RAM_GPU", "RAM_CPU"]))
                assert cl.client.migrate(f, getattr(bb.StorageClass, ftier)) == E.OK, (f, ftier)
                moves["fp8 " + ftier] += 1
                time.sleep(0.005)
        finally:
            stop.set()
            for t in threads:
                t.join()
        refreshes = _counter(cl.client, "get_placement_refresh_total") - refresh0
        print(f"\nrace: reads {dict(reads)}, moves {dict(moves)}, compaction moves {compacted}, placement refreshes {refreshes}")
        assert not errors, errors[:5]
        assert sum(reads.values()) > 30 and sum(moves.values()) + compacted > 0
    finally:
        cl.stop()
    DONE.add("race")


# ---------------------------------------------------------------------------------------------------- coverage


def test_calls_of_every_kind_overlapped_other_threads():
    """Calls of each kind overlapped in time a call of another thread of the same test several times: byte puts and gets
    (engine byte batches count as both), fp8 puts and gets, and mailbox-sized batches."""
    if not {"engine", "client", "async", "race"} <= DONE:
        pytest.skip("runs only after every threaded test of this module ran")
    calls = list(LOG)
    overlaps = collections.Counter()
    by_test = collections.defaultdict(list)
    for c in calls:
        by_test[c[0]].append(c)
    for test, cs in by_test.items():
        cs.sort(key=lambda c: c[3])
        for i, (_, tid, kind, t0, t1) in enumerate(cs):
            if any(o[1] != tid and o[3] < t1 and t0 < o[4] for o in cs if o is not cs[i] and o[3] < t1):
                for k in (("put", "get") if kind == "bytes" else (kind,)):
                    overlaps[k] += 1
    print(f"\noverlapping calls by kind: {dict(overlaps)} of {len(calls)} calls")
    missing = {k: overlaps[k] for k in OVERLAP_KINDS if overlaps[k] < 5}
    assert not missing, f"kinds that overlapped another thread's call fewer than 5 times: {missing}"
