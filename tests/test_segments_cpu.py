"""Segment-list puts and gets (batch_put_device_segments, batch_get_device_segments) on CPU: the SourceSegments rule
against an independent numpy model, and both client calls through the HostLoopbackTransport, which stands in for the GPU
fabric, so the client's segment logic -- the table rebased to every shard, replica fan-out, fail-over, the host-staged
path with its per-run copies -- runs in the CPU suite.  Segment addresses here are host addresses: the loopback's
"device pointers" are host pointers."""
import os

import numpy as np
import pytest

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
T = 16384
GUARD = 0xA5


def make_client(bb, c, node="node-0"):
    cl = c.client(node_id=node)
    io = c.client(node_id=node)
    bb.attach_loopback_transport(cl, io, False)
    return cl


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, replicas, stripes, algo="XXH3"):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=stripes, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[bb.StorageClass.RAM_CPU])


# ---------------------------------------------------------------- the rule against an independent model
def model_bytes(segs):
    """Per object byte: (address, segment index), or address -1 inside a null segment; zero-length segments hold none."""
    addr, seg = [], []
    for k, (a, n) in enumerate(segs):
        addr += [a + i if a else -1 for i in range(n)]
        seg += [k] * n
    return np.array(addr, dtype=np.int64), np.array(seg, dtype=np.int64)


def model_runs(addr, lo, hi):
    """Maximal runs of bytes [lo, hi) (as offsets from lo) whose addresses follow one another, null bytes in none."""
    out, x = [], lo
    while x < hi:
        if addr[x] < 0:
            x += 1
            continue
        y = x + 1
        while y < hi and addr[y] >= 0 and addr[y] == addr[y - 1] + 1:
            y += 1
        out.append((x - lo, int(addr[x]), y - x))
        x = y
    return out


def model_coaligned(addr, lo, hi):
    """Every non-null byte x of [lo, hi) lives at an address congruent to x - lo mod 16."""
    x = np.arange(lo, hi)
    a = addr[lo:hi]
    return bool(np.all((a < 0) | ((a - (x - lo)) % 16 == 0)))


def random_segments(rng, aligned):
    """Segment lists with zero-length, sub-16-byte, null, tile-straddling and many-tile segments."""
    segs, base, off = [], int(rng.integers(1, 1 << 30)) * 16, 0
    for _ in range(int(rng.integers(1, 40))):
        r = rng.random()
        n = 0 if r < 0.1 else int(rng.integers(1, 16)) if r < 0.35 else int(rng.integers(16, 3 * T)) if r < 0.9 else int(rng.integers(3 * T, 9 * T))
        adjacent = rng.random() < 0.3
        if rng.random() < 0.1:
            a = 0
        elif adjacent and segs and segs[-1][0]:
            a = segs[-1][0] + segs[-1][1]
        else:
            base += int(rng.integers(1, 1 << 20)) * 16
            a = base + (off % 16 if aligned else int(rng.integers(0, 16)))
        segs.append((a, n))
        off += n
    return segs


def test_source_segments_match_the_numpy_model(bb):
    rng = np.random.default_rng(17)
    for trial in range(200):
        segs = random_segments(rng, aligned=trial % 2 == 0)
        ec, t, size = bb.SourceSegments.from_segments(segs)
        assert ec == bb.ErrorCode.OK
        kept = [(a, n) for a, n in segs if n]
        assert size == sum(n for _, n in kept) and t.nseg == len(kept) and t.phase == 0
        if not kept:  # only empty segments: a zero-byte object without a table
            assert size == 0 and not t.segmented() and t.entries == []
            continue
        starts = np.concatenate([[0], np.cumsum([n for _, n in kept])]).astype(int).tolist()
        assert t.entries == [(starts[k], kept[k][0]) for k in range(len(kept))] + [(size, 0)]
        addr, seg = model_bytes(kept)
        assert t.has_null(size) == any(a == 0 for a, _ in kept)
        # every shard cut: 16 KiB tiles, odd cuts, inside segments and at their edges
        cuts = sorted(set([0, size] + starts + [int(c) for c in rng.integers(0, size + 1, 6)] + list(range(0, size, 3 * T + 5))))
        for lo, hi in zip(cuts, cuts[1:] + [size]):
            r = t.rebase(lo)
            n = hi - lo
            assert r.phase == lo and r.valid(n) and not r.valid(size - lo + 1)
            if lo < size:  # entry 0 holds the shard's first byte
                assert r.entries[0] == (starts[seg[lo]], kept[seg[lo]][0])
                assert r.segments_for(n) == (len(set(seg[lo:hi].tolist())) if n else 0)
            assert r.runs(n) == model_runs(addr, lo, hi)
            assert r.coaligned(n) == model_coaligned(addr, lo, hi)
            assert t.fused_get_aligned(lo, n) == model_coaligned(addr, lo, hi)
            assert r.has_null(n) == bool(np.any(addr[lo:hi] < 0))


def test_from_segments_edges(bb):
    ec, t, size = bb.SourceSegments.from_segments([])
    assert ec == bb.ErrorCode.OK and size == 0 and not t.segmented()
    ec, t, size = bb.SourceSegments.from_segments([(64, 0), (128, 0)])  # only empty segments: a zero-byte object
    assert ec == bb.ErrorCode.OK and size == 0 and not t.segmented()
    ec, _, _ = bb.SourceSegments.from_segments([(64, 1 << 63), (128, 1 << 63)])
    assert ec == bb.ErrorCode.VALUE_OUT_OF_RANGE
    # adjacent segments merge into one run; a null one ends it
    ec, t, size = bb.SourceSegments.from_segments([(1024, 16), (1040, 5), (0, 7), (1045, 3), (1048, 8)])
    assert size == 39 and t.runs(39) == [(0, 1024, 21), (28, 1045, 11)]
    assert t.rebase(10).runs(29) == [(0, 1034, 11), (18, 1045, 11)]
    assert not t.coaligned(39) and t.rebase(28).coaligned(11) is False and t.rebase(0).coaligned(21)
    # numpy (n, 2) arrays are taken whole
    ec, t, size = bb.SourceSegments.from_segments(np.array([[32, 16], [96, 4]], dtype=np.uint64))
    assert size == 20 and t.entries == [(0, 32), (16, 96), (20, 0)]
    with pytest.raises(ValueError):
        bb.SourceSegments.from_segments(np.zeros((2, 3), dtype=np.uint64))


# ---------------------------------------------------------------- client calls through the loopback transport
class Arena:
    """One guard-filled host buffer that segments are carved from, each placed co-aligned with its object offset (or
    skewed off it), with guard bytes between them."""

    def __init__(self, nbytes):
        self.raw = np.full(nbytes, GUARD, dtype=np.uint8)
        self.base = self.raw.ctypes.data
        self.o = (-self.base) % 16 + 64

    def segments(self, lens, skew=0):
        """Offsets into raw of segments of lens, segment k at an address congruent to its object offset (+ skew)."""
        offs, start = [], 0
        for n in lens:
            self.o = (self.o + 15) // 16 * 16 + 32
            offs.append(self.o + (start + skew) % 16)
            self.o = offs[-1] + n
            start += n
        assert self.o + 64 < len(self.raw)
        return offs

    def pairs(self, offs, lens, null=()):
        return [(0 if k in null else self.base + o, n) for k, (o, n) in enumerate(zip(offs, lens))]

    def fill(self, offs, lens, blob):
        x = 0
        for o, n in zip(offs, lens):
            self.raw[o:o + n] = blob[x:x + n]
            x += n


def _lens(rng, k):
    return [int(rng.choice([0, 1, 7, 15, 16, 100, 4096, T - 3, T + 17, 3 * T + 5])) for _ in range(k)]


def _digests(cl, key):
    return [[s.checksum for s in cp.shards] for cp in cl.get_workers(key)]


def test_put_equals_a_put_of_the_concatenation_and_reads_back_both_ways(bb):
    rng = np.random.default_rng(1)
    with LocalCluster(cluster_id="sgp", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        n0 = _counter(cl, "device_put_segments_total")
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            for replicas, stripes in ((1, 1), (2, 1), (1, 3), (2, 2)):
                lens = _lens(rng, int(rng.integers(1, 20)))
                size = sum(lens)
                ar = Arena(size + 64 * len(lens) + 4096)
                offs = ar.segments(lens)
                blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
                ar.fill(offs, lens, blob)
                before = ar.raw.copy()
                cfg = _cfg(bb, replicas, stripes, algo)
                key, ref = f"s/{algo}/{replicas}/{stripes}", f"r/{algo}/{replicas}/{stripes}"
                assert cl.batch_put_device_segments([key], [ar.pairs(offs, lens)], cfg, 0) == [bb.ErrorCode.OK]
                assert np.array_equal(ar.raw, before)  # a put reads only
                assert cl.batch_put_device([ref], [blob.ctypes.data], [size], cfg, 0) == [bb.ErrorCode.OK]
                if stripes == 1:
                    assert _digests(cl, key) == _digests(cl, ref)
                out = np.zeros(max(size, 1), np.uint8)
                ecs, sizes = cl.batch_get_device([key], [out.ctypes.data], [size], 0)
                assert ecs == [bb.ErrorCode.OK] and sizes == [size] and np.array_equal(out[:size], blob)
                # a segment get of the plain object, into differently cut segments
                lens2 = list(rng.permutation(lens))
                ar2 = Arena(size + 64 * len(lens) + 4096)
                offs2 = ar2.segments(lens2)
                ecs, sizes = cl.batch_get_device_segments([ref], [ar2.pairs(offs2, lens2)], 0)
                assert ecs == [bb.ErrorCode.OK] and sizes == [size]
                want = np.full_like(ar2.raw, GUARD)
                ar2.raw, got = want, ar2.raw
                ar2.fill(offs2, lens2, blob)
                assert np.array_equal(got, want)
        assert _counter(cl, "device_put_segments_total") == n0 + 16
        assert _counter(cl, "device_get_segments_total") == 16


def test_staged_items_and_their_fused_neighbours(bb):
    """A segment whose address is not congruent to its object offset mod 16 stages its object through the host, one copy
    per run; co-aligned items of the same call keep the (loopback) fused path; guards stay untouched; null segments of a
    get are not stored."""
    with LocalCluster(cluster_id="sgs", n_workers=3, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1, 1)  # one shard per object: where a placement cuts is test_source_segments_match_the_numpy_model's
        shapes = [([100, 3, 4096, T + 1], 0), ([7, 9, 2 * T], 3), ([T], 0), ([1, 1, 1], 5)]
        ar = Arena(4 * MiB)
        offs = [ar.segments(lens, skew) for lens, skew in shapes]
        blobs = [np.frombuffer(os.urandom(sum(lens)), dtype=np.uint8).copy() for lens, _ in shapes]
        for o, (lens, _), b in zip(offs, shapes, blobs):
            ar.fill(o, lens, b)
        keys = [f"st{i}" for i in range(len(shapes))]
        staged = _counter(cl, "device_put_host_staged_total")
        assert cl.batch_put_device_segments(keys, [ar.pairs(o, lens) for o, (lens, _) in zip(offs, shapes)], cfg, 0) == [bb.ErrorCode.OK] * 4
        assert _counter(cl, "device_put_host_staged_total") == staged + 2
        for k, b in zip(keys, blobs):
            out = np.zeros(b.size, np.uint8)
            assert cl.batch_get_device([k], [out.ctypes.data], [out.size], 0)[0] == [bb.ErrorCode.OK] and np.array_equal(out, b)
        dst = Arena(4 * MiB)
        doffs = [dst.segments(lens, skew) for lens, skew in shapes]
        nulls = [{1}, {0}, set(), {2}]
        staged = _counter(cl, "device_get_host_staged_total")
        ecs, sizes = cl.batch_get_device_segments(keys, [dst.pairs(o, lens, nl) for o, (lens, _), nl in zip(doffs, shapes, nulls)], 0)
        assert ecs == [bb.ErrorCode.OK] * 4 and sizes == [b.size for b in blobs]
        assert _counter(cl, "device_get_host_staged_total") == staged + 2
        want = np.full_like(dst.raw, GUARD)
        for o, (lens, _), b, nl in zip(doffs, shapes, blobs, nulls):
            x = 0
            for k, (a, n) in enumerate(zip(o, lens)):
                if k not in nl:
                    want[a:a + n] = b[x:x + n]
                x += n
        assert np.array_equal(dst.raw, want)


def test_sizes_overflow_refusals_and_empty_lists(bb):
    with LocalCluster(cluster_id="sgz", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1, 1)
        ar = Arena(1 * MiB)
        lens = [4096, 100, 5000]
        offs = ar.segments(lens)
        blob = np.frombuffer(os.urandom(sum(lens)), dtype=np.uint8).copy()
        ar.fill(offs, lens, blob)
        ok = ar.pairs(offs, lens)
        ecs = cl.batch_put_device_segments(["z", "null", "ovf", "ok"], [[], ar.pairs(offs, lens, {1}), [(ar.base, 1 << 63)] * 2, ok], cfg, 0)
        assert ecs == [bb.ErrorCode.OK, bb.ErrorCode.INVALID_ARGUMENT, bb.ErrorCode.VALUE_OUT_OF_RANGE, bb.ErrorCode.OK]
        assert not cl.object_exists("null") and not cl.object_exists("ovf")
        dst = Arena(1 * MiB)
        small = dst.segments([4096, 100])
        big = dst.segments([3000, 3000, 3000, 3000])
        snapshot = dst.raw.copy()
        ecs, sizes = cl.batch_get_device_segments(["z", "ok", "ok"], [[], dst.pairs(small, [4096, 100]), dst.pairs(big, [3000] * 4)], 0)
        assert ecs == [bb.ErrorCode.OK, bb.ErrorCode.BUFFER_OVERFLOW, bb.ErrorCode.OK]
        assert sizes[0] == 0 and sizes[2] == blob.size
        want = snapshot  # the short object fills the segments in order; the last 2804 bytes of capacity stay untouched
        dst.raw, got = want, dst.raw
        dst.fill(big, [3000] * 4, np.concatenate([blob, snapshot[big[3] + 196:big[3] + 3000]]))
        assert np.array_equal(got, want)
        ecs, _ = cl.batch_get_device_segments(["ok"], [[(dst.base, 1 << 63), (dst.base, 1 << 63)]], 0)
        assert ecs == [bb.ErrorCode.VALUE_OUT_OF_RANGE]
        assert cl.batch_put_device_segments(["a", "b"], [[]], cfg, 0) == [bb.ErrorCode.INVALID_PARAMETERS] * 2
        ecs, _ = cl.batch_get_device_segments(["nope"], [[]], 0)
        assert ecs == [bb.ErrorCode.OBJECT_NOT_FOUND]


def test_fail_over_and_refresh(bb):
    with LocalCluster(cluster_id="sgf", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))

        lens = _lens(np.random.default_rng(5), 30)
        ar = Arena(sum(lens) + 4096 * 8)
        offs = ar.segments(lens)
        blob = np.frombuffer(os.urandom(sum(lens)), dtype=np.uint8).copy()
        ar.fill(offs, lens, blob)
        assert cl.batch_put_device_segments(["f"], [ar.pairs(offs, lens)], _cfg(bb, 3, 2), 0) == [bb.ErrorCode.OK]
        copies = cl.get_workers("f")
        mm = _counter(cl, "checksum_mismatch_total")
        for cp in copies:  # one corrupt copy at a time: the get fails over, segments right, guards untouched
            flip(cp.shards[-1], 77)
            dst = Arena(sum(lens) + 4096 * 8)
            doffs = dst.segments(lens)
            ecs, _ = cl.batch_get_device_segments(["f"], [dst.pairs(doffs, lens)], 0)
            assert ecs == [bb.ErrorCode.OK]
            want = np.full_like(dst.raw, GUARD)
            dst.raw, got = want, dst.raw
            dst.fill(doffs, lens, blob)
            assert np.array_equal(got, want)
            flip(cp.shards[-1], 77)
        assert _counter(cl, "checksum_mismatch_total") > mm
        for cp in copies:
            flip(cp.shards[0], 5)
        ref = _counter(cl, "get_placement_refresh_total")
        dst = Arena(sum(lens) + 4096 * 8)
        ecs, _ = cl.batch_get_device_segments(["f"], [dst.pairs(dst.segments(lens), lens)], 0)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1


# ---------------------------------------------------------------- TensorStore checks that need no GPU
def test_tensor_store_bundle_checks_before_any_transfer():
    torch = pytest.importorskip("torch")
    from blackbird_b200.ops import TensorStore

    class NoCalls:
        def __getattr__(self, name):
            raise AssertionError(f"client.{name} called")

    ts = TensorStore.__new__(TensorStore)
    ts.client, ts.config = NoCalls(), None
    with pytest.raises(ValueError, match="CUDA"):
        ts.batch_put_bundles(["k"], [{"w": torch.zeros(4)}])  # a CPU tensor
    with pytest.raises(TypeError, match="not a tensor"):
        ts.batch_put_bundles(["k"], [{"w": 3}])
    with pytest.raises(TypeError, match="bundle is a mapping"):
        ts.batch_put_bundles(["k"], [torch.zeros(4)])
    with pytest.raises(TypeError, match="complex"):
        ts.batch_put_bundles(["k"], [[torch.zeros(4, dtype=torch.complex64)]])
    with pytest.raises(ValueError, match="differ in length"):
        ts.batch_put_bundles(["k", "l"], [{}])
