"""Paged puts and gets (batch_put_device_paged, batch_get_device_paged) on CPU: the HostLoopbackTransport stands in for
the GPU fabric, so the client's paged logic -- the page table rebased to every shard, replica fan-out, fail-over, the
placement refresh, the host-staged path with its per-run copies -- runs in the CPU suite, under the same SourcePages rule
the kernel follows.  Page addresses here are host addresses: the loopback's "device pointers" are host pointers."""
import os

import numpy as np
import pytest

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
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
def model_addr(addrs, page, phase, x):
    """Where object byte x lives: addrs[(x + phase) // page] + (x + phase) % page."""
    y = np.asarray(x, dtype=np.int64) + phase
    return np.asarray(addrs, dtype=np.int64)[y // page] + y % page


def model_runs(addrs, page, phase, n):
    """Maximal runs of object bytes whose addresses follow one another."""
    if n == 0:
        return []
    a = model_addr(addrs, page, phase, np.arange(n))
    cut = np.nonzero(np.diff(a) != 1)[0] + 1
    starts = np.concatenate([[0], cut])
    ends = np.concatenate([cut, [n]])
    return [(int(s), int(a[s]), int(e - s)) for s, e in zip(starts, ends)]


def model_coaligned(addrs, page, phase, n):
    if n == 0:
        return True
    k = (n - 1 + phase) // page + 1
    if k > 1 and page % 16:
        return False
    return all((a + phase) % 16 == 0 for a in addrs[:k])


def test_source_pages_match_the_numpy_model(bb):
    rng = np.random.default_rng(7)
    for _ in range(300):
        npages = int(rng.integers(1, 40))
        page = int(rng.choice([1, 3, 16, 48, 100, 4096]))
        # addresses: sometimes adjacent runs, sometimes shuffled, sometimes misaligned
        base = int(rng.integers(0, 1 << 40)) * 16
        order = rng.permutation(npages) if rng.random() < 0.5 else np.arange(npages)
        addrs = [base + int(o) * page + (int(rng.integers(0, 16)) if rng.random() < 0.2 else 0) for o in order]
        ec, t, size = bb.SourcePages.from_pages(addrs, page)
        assert ec == bb.ErrorCode.OK and size == npages * page and t.npages == npages and t.phase == 0
        assert t.addrs == addrs
        off = int(rng.integers(0, size + 1))
        r = t.rebase(off)
        k = min(off // page, npages)
        assert (r.phase, r.addrs, r.npages) == (off % page, addrs[k:], npages - k)
        n = size - off
        assert r.runs(n) == model_runs(addrs[k:], page, off % page, n)
        assert r.coaligned(n) == model_coaligned(addrs[k:], page, off % page, n)
        # runs cover object bytes [0, n) in order at the rule's addresses
        xs = [x for x, _, m in r.runs(n) for x in range(x, x + m)]
        assert xs == list(range(n))
        # the client's get rule: also page % 16 == 0 whenever the table has more than one page
        want = (npages <= 1 or page % 16 == 0) and model_coaligned(addrs[k:], page, off % page, n)
        assert t.fused_get_aligned(off, n) == want


def test_from_pages_errors(bb):
    ec, t, size = bb.SourcePages.from_pages([], 0)
    assert ec == bb.ErrorCode.OK and size == 0 and not t.paged()
    ec, _, _ = bb.SourcePages.from_pages([16, 32], 0)
    assert ec == bb.ErrorCode.INVALID_ARGUMENT
    ec, _, _ = bb.SourcePages.from_pages([16, 32], 1 << 63)
    assert ec == bb.ErrorCode.VALUE_OUT_OF_RANGE
    # numpy arrays and CPU tensors are taken whole; lists element by element
    torch = pytest.importorskip("torch")
    assert bb.SourcePages.from_pages(np.array([32, 64], dtype=np.uint64), 16)[1].addrs == [32, 64]
    assert bb.SourcePages.from_pages(torch.tensor([48, 16]), 16)[1].addrs == [48, 16]
    with pytest.raises(ValueError):
        bb.SourcePages.from_pages(np.zeros((2, 2), dtype=np.int64), 16)


# ---------------------------------------------------------------- client calls through the loopback transport
class Arena:
    """One guard-filled host buffer that pages are carved from, 16-byte aligned plus a chosen skew, with guard bytes
    between and around them."""

    def __init__(self, nbytes):
        self.raw = np.full(nbytes, GUARD, dtype=np.uint8)
        self.base = self.raw.ctypes.data
        self.o = (-self.base) % 16 + 64

    def pages(self, n, page, skew=0, shuffle=None):
        offs = []
        for _ in range(n):
            offs.append(self.o + skew)
            self.o = (self.o + skew + page + 15) // 16 * 16 + 32  # a guard gap after every page
        assert self.o < len(self.raw)
        if shuffle is not None:
            offs = [offs[i] for i in shuffle.permutation(n)]
        return offs

    def addrs(self, offs):
        return [self.base + o for o in offs]

    def fill(self, offs, page, blob):
        for k, o in enumerate(offs):
            self.raw[o:o + page] = blob[k * page:(k + 1) * page]

    def gather(self, offs, page):
        return np.concatenate([self.raw[o:o + page] for o in offs]) if offs else np.zeros(0, np.uint8)


def _digests(cl, key):
    return [[s.checksum for s in cp.shards] for cp in cl.get_workers(key)]


def test_put_equals_a_put_of_the_concatenation_and_reads_back_both_ways(bb):
    rng = np.random.default_rng(1)
    with LocalCluster(cluster_id="pgp", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        n0 = _counter(cl, "device_put_paged_total")
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            for replicas, stripes in ((1, 1), (2, 1), (1, 3), (2, 2)):
                for page in (16, 4096, 48 * 1024 + 16):
                    ar = Arena(40 * page + 1 * MiB)
                    npg = int(rng.integers(1, 24))
                    offs = ar.pages(npg, page, shuffle=rng)
                    blob = np.frombuffer(os.urandom(npg * page), dtype=np.uint8).copy()
                    ar.fill(offs, page, blob)
                    before = ar.raw.copy()
                    cfg = _cfg(bb, replicas, stripes, algo)
                    key, ref = f"p/{algo}/{replicas}/{stripes}/{page}", f"r/{algo}/{replicas}/{stripes}/{page}"
                    assert cl.batch_put_device_paged([key], [np.array(ar.addrs(offs), dtype=np.uint64)], [page], cfg, 0) == [bb.ErrorCode.OK]
                    assert np.array_equal(ar.raw, before)  # a put reads only
                    assert cl.batch_put_device([ref], [blob.ctypes.data], [blob.size], cfg, 0) == [bb.ErrorCode.OK]
                    if stripes == 1:  # same layout: the same digests shard for shard
                        assert _digests(cl, key) == _digests(cl, ref)
                    # plain device get of the paged object, paged get of the plain object
                    out = np.zeros(blob.size, np.uint8)
                    ecs, sizes = cl.batch_get_device([key], [out.ctypes.data], [out.size], 0)
                    assert ecs == [bb.ErrorCode.OK] and sizes == [blob.size] and np.array_equal(out, blob)
                    ar2 = Arena(40 * page + 1 * MiB)
                    offs2 = ar2.pages(npg, page, shuffle=rng)
                    ecs, sizes = cl.batch_get_device_paged([ref], [ar2.addrs(offs2)], [page], 0)
                    assert ecs == [bb.ErrorCode.OK] and sizes == [blob.size]
                    want = np.full_like(ar2.raw, GUARD)
                    ar2.raw, got = want, ar2.raw
                    ar2.fill(offs2, page, blob)
                    assert np.array_equal(got, want)
        assert _counter(cl, "device_put_paged_total") == n0 + 4 * 4 * 3
        assert _counter(cl, "device_get_paged_total") > 0 and _counter(cl, "device_get_paged_bytes_total") > 0


def test_repeated_pages_on_put_and_mid_page_shard_edges(bb):
    """A put may list a page twice; striped copies cut pages in the middle, so shards start with a nonzero phase."""
    with LocalCluster(cluster_id="pgr", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        page = 4096 + 48
        ar = Arena(64 * page)
        offs = ar.pages(7, page)
        blob = np.frombuffer(os.urandom(7 * page), dtype=np.uint8).copy()
        ar.fill(offs, page, blob)
        order = [3, 3, 0, 6, 1, 3, 5, 2, 2, 4, 6]
        want = np.concatenate([blob[k * page:(k + 1) * page] for k in order])
        cfg = _cfg(bb, 2, 3)
        assert cl.batch_put_device_paged(["rep"], [[ar.base + offs[k] for k in order]], [page], cfg, 0) == [bb.ErrorCode.OK]
        lens = [s.length for s in cl.get_workers("rep")[0].shards]
        assert len(lens) >= 2 and any(np.cumsum(lens)[:-1] % page != 0)
        out = np.zeros(want.size, np.uint8)
        ecs, _ = cl.batch_get_device(["rep"], [out.ctypes.data], [out.size], 0)
        assert ecs == [bb.ErrorCode.OK] and np.array_equal(out, want)
        # back into fresh pages through a striped get
        dst = Arena(64 * page)
        doffs = dst.pages(len(order), page, shuffle=np.random.default_rng(3))
        ecs, sizes = cl.batch_get_device_paged(["rep"], [dst.addrs(doffs)], [page], 0)
        assert ecs == [bb.ErrorCode.OK] and sizes == [want.size]
        assert np.array_equal(dst.gather(doffs, page), want)


def test_staged_items_and_their_fused_neighbours(bb):
    """Misaligned pages and page % 16 != 0 are staged through the host, one copy per run; aligned items in the same call
    keep the (loopback) fused path.  Guard bytes stay untouched either way."""
    with LocalCluster(cluster_id="pgs", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1, 1)
        shapes = [(4096, 0, 5), (4096, 3, 5), (100, 0, 9), (100, 0, 1), (33, 5, 1)]  # (page, skew, pages)
        ar = Arena(4 * MiB)
        offs = [ar.pages(n, p, skew=s) for p, s, n in shapes]
        blobs = [np.frombuffer(os.urandom(n * p), dtype=np.uint8).copy() for p, _, n in shapes]
        for o, (p, _, _), b in zip(offs, shapes, blobs):
            ar.fill(o, p, b)
        keys = [f"s{i}" for i in range(len(shapes))]
        staged = _counter(cl, "device_put_host_staged_total")
        assert cl.batch_put_device_paged(keys, [ar.addrs(o) for o in offs], [p for p, _, _ in shapes], cfg, 0) == [bb.ErrorCode.OK] * 5
        # 1: misaligned, 2: 100-byte pages over several pages; 3 and 4 are single pages (3 aligned: fused)
        assert _counter(cl, "device_put_host_staged_total") == staged + 3
        for k, b in zip(keys, blobs):
            out = np.zeros(b.size, np.uint8)
            assert cl.batch_get_device([k], [out.ctypes.data], [out.size], 0)[0] == [bb.ErrorCode.OK] and np.array_equal(out, b)
        dst = Arena(4 * MiB)
        doffs = [dst.pages(n, p, skew=s) for p, s, n in shapes]
        staged = _counter(cl, "device_get_host_staged_total")
        ecs, sizes = cl.batch_get_device_paged(keys, [dst.addrs(o) for o in doffs], [p for p, _, _ in shapes], 0)
        assert ecs == [bb.ErrorCode.OK] * 5 and sizes == [b.size for b in blobs]
        # 1, 2 and 4 miss the get rule (4: one misaligned page); 3 is a single aligned page
        assert _counter(cl, "device_get_host_staged_total") == staged + 3
        want = np.full_like(dst.raw, GUARD)
        for o, (p, _, _), b in zip(doffs, shapes, blobs):
            for k, a in enumerate(o):
                want[a:a + p] = b[k * p:(k + 1) * p]
        assert np.array_equal(dst.raw, want)


def test_sizes_overflow_and_zero_pages(bb):
    with LocalCluster(cluster_id="pgz", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1, 1)
        ar = Arena(1 * MiB)
        offs = ar.pages(4, 4096)
        blob = np.frombuffer(os.urandom(4 * 4096), dtype=np.uint8).copy()
        ar.fill(offs, 4096, blob)
        # zero pages: a zero-byte object; page 0 with pages and an overflowing size are refused before any allocation
        ecs = cl.batch_put_device_paged(["z", "bad0", "ovf", "ok"], [[], ar.addrs(offs), [ar.base] * 3, ar.addrs(offs)],
                                        [4096, 0, 1 << 63, 4096], cfg, 0)
        assert ecs == [bb.ErrorCode.OK, bb.ErrorCode.INVALID_ARGUMENT, bb.ErrorCode.VALUE_OUT_OF_RANGE, bb.ErrorCode.OK]
        assert not cl.object_exists("bad0") and not cl.object_exists("ovf")
        before = _counter(cl, "device_put_paged_total")
        dst = Arena(1 * MiB)
        d3 = dst.pages(3, 4096)
        d6 = dst.pages(6, 4096)
        snapshot = dst.raw.copy()
        ecs, sizes = cl.batch_get_device_paged(["z", "ok", "ok", "ok"], [[], dst.addrs(d3), [], dst.addrs(d6)], [4096, 4096, 0, 4096], 0)
        assert ecs == [bb.ErrorCode.OK, bb.ErrorCode.BUFFER_OVERFLOW, bb.ErrorCode.BUFFER_OVERFLOW, bb.ErrorCode.OK]
        assert sizes[0] == 0 and sizes[3] == blob.size
        # the short object fills its first four pages; the other two, and everything else, are untouched
        want = snapshot
        for k in range(4):
            want[d6[k]:d6[k] + 4096] = blob[k * 4096:(k + 1) * 4096]
        assert np.array_equal(dst.raw, want)
        assert _counter(cl, "device_put_paged_total") == before
        ecs, _ = cl.batch_get_device_paged(["ok"], [[dst.base] * 4], [1 << 62], 0)
        assert ecs == [bb.ErrorCode.VALUE_OUT_OF_RANGE]


def test_fail_over_and_refresh(bb):
    with LocalCluster(cluster_id="pgf", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))

        page = 16 * 1024 + 16
        ar = Arena(80 * page)
        offs = ar.pages(64, page, shuffle=np.random.default_rng(5))
        blob = np.frombuffer(os.urandom(64 * page), dtype=np.uint8).copy()
        ar.fill(offs, page, blob)
        assert cl.batch_put_device_paged(["f"], [ar.addrs(offs)], [page], _cfg(bb, 3, 2), 0) == [bb.ErrorCode.OK]
        copies = cl.get_workers("f")
        mm = _counter(cl, "checksum_mismatch_total")
        for cp in copies:  # one corrupt copy at a time: the get fails over, pages right, guards untouched
            flip(cp.shards[-1], 777)
            dst = Arena(80 * page)
            doffs = dst.pages(64, page, shuffle=np.random.default_rng(6))
            ecs, _ = cl.batch_get_device_paged(["f"], [dst.addrs(doffs)], [page], 0)
            assert ecs == [bb.ErrorCode.OK]
            want = np.full_like(dst.raw, GUARD)
            for k, o in enumerate(doffs):
                want[o:o + page] = blob[k * page:(k + 1) * page]
            assert np.array_equal(dst.raw, want)
            flip(cp.shards[-1], 777)
        assert _counter(cl, "checksum_mismatch_total") > mm
        for cp in copies:
            flip(cp.shards[0], 5)
        ref = _counter(cl, "get_placement_refresh_total")
        dst = Arena(80 * page)
        doffs = dst.pages(64, page)
        ecs, _ = cl.batch_get_device_paged(["f"], [dst.addrs(doffs)], [page], 0)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1


def test_arity_and_missing_keys(bb):
    with LocalCluster(cluster_id="pga", n_workers=1, pool_bytes=16 * MiB) as c:
        cl = make_client(bb, c)
        assert cl.batch_put_device_paged(["a", "b"], [[]], [16], _cfg(bb, 1, 1), 0) == [bb.ErrorCode.INVALID_PARAMETERS] * 2
        ecs, _ = cl.batch_get_device_paged(["nope"], [[]], [16], 0)
        assert ecs == [bb.ErrorCode.OBJECT_NOT_FOUND]
