"""Sparse page tables (partial restores of paged objects) on CPU: a page address of 0 is a page a get does not store.  The
SourcePages rule against a numpy model that skips null pages, and batch_get_device_paged / batch_get_device_fp8_paged
with such tables through the HostLoopbackTransport -- striped and replicated objects, fail-over, the placement refresh and
the host-staged path -- with every guard byte checked; puts refuse null pages.  Page addresses here are host addresses:
the loopback's "device pointers" are host pointers."""
import os

import numpy as np

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
GUARD = 0xA5
NP = {"bf16": np.uint16, "f16": np.float16, "f32": np.float32}
SIZE = {"bf16": 2, "f16": 2, "f32": 4}


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


def mxw(bb, w):
    return {"bf16": bb.MxWide.BF16, "f16": bb.MxWide.F16, "f32": bb.MxWide.F32}[w]


# ---------------------------------------------------------------- the rule against an independent model
def model_runs(addrs, page, phase, n):
    """Maximal runs of stored object bytes whose addresses follow one another; bytes in null pages are not stored."""
    if n == 0:
        return []
    x = np.arange(n)
    y = x + phase
    pg = np.asarray(addrs, dtype=np.int64)[y // page]
    keep = pg != 0
    x, a = x[keep], (pg + y % page)[keep]
    if x.size == 0:
        return []
    cut = np.nonzero((np.diff(a) != 1) | (np.diff(x) != 1))[0] + 1
    starts = np.concatenate([[0], cut])
    ends = np.concatenate([cut, [x.size]])
    return [(int(x[s]), int(a[s]), int(e - s)) for s, e in zip(starts, ends)]


def model_coaligned(addrs, page, phase, n):
    if n == 0:
        return True
    k = (n - 1 + phase) // page + 1
    if k > 1 and page % 16:
        return False
    return all(a == 0 or (a + phase) % 16 == 0 for a in addrs[:k])


def test_null_pages_match_the_numpy_model(bb):
    rng = np.random.default_rng(21)
    for trial in range(400):
        npages = int(rng.integers(1, 40))
        page = int(rng.choice([1, 3, 16, 48, 100, 4096]))
        base = int(rng.integers(1, 1 << 40)) * 16
        order = rng.permutation(npages) if rng.random() < 0.5 else np.arange(npages)
        addrs = [base + int(o) * page + (int(rng.integers(0, 16)) if rng.random() < 0.2 else 0) for o in order]
        dense = list(addrs)
        if trial % 4:  # a quarter of the tables have no null page and must behave as before
            p = rng.choice([0.1, 0.5, 0.9, 1.0])
            addrs = [0 if rng.random() < p else a for a in addrs]
        ec, t, size = bb.SourcePages.from_pages(addrs, page)
        assert ec == bb.ErrorCode.OK and size == npages * page
        off = int(rng.integers(0, size + 1))
        r = t.rebase(off)
        k = min(off // page, npages)
        n = size - off
        assert r.runs(n) == model_runs(addrs[k:], page, off % page, n)
        assert r.coaligned(n) == model_coaligned(addrs[k:], page, off % page, n)
        want = (npages <= 1 or page % 16 == 0) and model_coaligned(addrs[k:], page, off % page, n)
        assert t.fused_get_aligned(off, n) == want
        touched = (n - 1 + off % page) // page + 1 if n else 0
        assert r.has_null(n) == any(a == 0 for a in addrs[k:k + touched])
        if addrs == dense:  # no null page: exactly the dense rule (adjacent pages merge into one run)
            _, td, _ = bb.SourcePages.from_pages(dense, page)
            assert td.rebase(off).runs(n) == r.runs(n)


# ---------------------------------------------------------------- client calls through the loopback transport
class Arena:
    """One guard-filled host buffer that pages are carved from: 16-byte aligned plus a chosen skew, with a guard gap
    after every page."""

    def __init__(self, nbytes):
        self.raw = np.full(nbytes, GUARD, dtype=np.uint8)
        self.base = self.raw.ctypes.data
        self.o = (-self.base) % 16 + 64

    def pages(self, n, page, skew=0, shuffle=None):
        offs = []
        for _ in range(n):
            offs.append(self.o + skew)
            self.o = (self.o + skew + page + 15) // 16 * 16 + 32
        assert self.o < len(self.raw)
        if shuffle is not None:
            offs = [offs[i] for i in shuffle.permutation(n)]
        return offs

    def table(self, offs, stored):
        """The page table with the pages not in `stored` (a boolean mask) null."""
        return np.array([self.base + o if s else 0 for o, s in zip(offs, stored)], dtype=np.uint64)

    def expect(self, offs, stored, page, blob):
        want = np.full_like(self.raw, GUARD)
        for k, (o, s) in enumerate(zip(offs, stored)):
            if s:
                want[o:o + page] = blob[k * page:(k + 1) * page]
        return want


def _masks(rng, n):
    """Selections: a prefix, a random subset, one page, none, all."""
    k = int(rng.integers(1, n + 1))
    return [np.arange(n) < k, rng.random(n) < 0.5, np.arange(n) == int(rng.integers(0, n)), np.zeros(n, bool), np.ones(n, bool)]


def test_sparse_gets_store_only_the_selected_pages(bb):
    rng = np.random.default_rng(22)
    with LocalCluster(cluster_id="spg", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        for algo in ("XXH3", "NONE"):
            for replicas, stripes in ((1, 1), (2, 1), (1, 3), (2, 2)):
                for page, skew in ((4096, 0), (48 * 1024 + 16, 0), (100, 0), (4096, 3)):  # the last two are host-staged
                    npg = int(rng.integers(2, 20))
                    blob = np.frombuffer(os.urandom(npg * page), dtype=np.uint8).copy()
                    key = f"s/{algo}/{replicas}/{stripes}/{page}/{skew}"
                    assert cl.batch_put_device([key], [blob.ctypes.data], [blob.size], _cfg(bb, replicas, stripes, algo), 0) == [bb.ErrorCode.OK]
                    for mask in _masks(rng, npg):
                        ar = Arena(npg * (page + 64) + MiB)
                        offs = ar.pages(npg, page, skew=skew, shuffle=rng)
                        ecs, sizes = cl.batch_get_device_paged([key], [ar.table(offs, mask)], [page], 0)
                        assert ecs == [bb.ErrorCode.OK] and sizes == [blob.size], (key, mask)
                        assert np.array_equal(ar.raw, ar.expect(offs, mask, page, blob)), (key, mask)


def test_sparse_gets_fail_over_refresh_and_verify_with_no_page_stored(bb):
    with LocalCluster(cluster_id="spf", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))

        page, npg = 16 * 1024 + 16, 48
        blob = np.frombuffer(os.urandom(npg * page), dtype=np.uint8).copy()
        assert cl.batch_put_device(["f"], [blob.ctypes.data], [blob.size], _cfg(bb, 3, 2), 0) == [bb.ErrorCode.OK]
        mask = np.arange(npg) < 5  # a prefix: the corrupt byte lies in a shard whose pages are not stored
        fo = _counter(cl, "replica_failover_total")
        for cp in cl.get_workers("f"):
            flip(cp.shards[-1], 777)
            ar = Arena(npg * (page + 64) + MiB)
            offs = ar.pages(npg, page, shuffle=np.random.default_rng(5))
            ecs, _ = cl.batch_get_device_paged(["f"], [ar.table(offs, mask)], [page], 0)
            assert ecs == [bb.ErrorCode.OK]
            assert np.array_equal(ar.raw, ar.expect(offs, mask, page, blob))
            flip(cp.shards[-1], 777)
        assert _counter(cl, "replica_failover_total") > fo
        # an all-null table stores nothing and reads OK ...
        ar = Arena(npg * (page + 64) + MiB)
        offs = ar.pages(npg, page)
        ecs, sizes = cl.batch_get_device_paged(["f"], [ar.table(offs, np.zeros(npg, bool))], [page], 0)
        assert ecs == [bb.ErrorCode.OK] and sizes == [blob.size]
        assert (ar.raw == GUARD).all()
        # ... but still verifies: with every copy corrupt the get refreshes once and reports the mismatch
        for cp in cl.get_workers("f"):
            flip(cp.shards[0], 5)
        ref = _counter(cl, "get_placement_refresh_total")
        ecs, _ = cl.batch_get_device_paged(["f"], [ar.table(offs, np.zeros(npg, bool))], [page], 0)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1
        assert (ar.raw == GUARD).all()
        # a single corrupt copy with no page stored is a mismatch too
        one = np.frombuffer(os.urandom(4 * 4096), dtype=np.uint8).copy()
        assert cl.batch_put_device(["one"], [one.ctypes.data], [one.size], _cfg(bb, 1, 1), 0) == [bb.ErrorCode.OK]
        flip(cl.get_workers("one")[0].shards[0], 100)
        ecs, _ = cl.batch_get_device_paged(["one"], [np.zeros(4, np.uint64)], [4096], 0)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]


def _values(rng, n, w):
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-12, 12, n))).astype(np.float32)
    v[::97] = np.nan
    v[7::331] = 0.0
    x = v.astype(NP[w]) if w != "bf16" else (v.view(np.uint32) >> 16).astype(np.uint16)
    return x.view(np.uint8)


def test_sparse_fp8_gets_in_every_wide_type(bb):
    rng = np.random.default_rng(23)
    with LocalCluster(cluster_id="spx", n_workers=3, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}
        for w in ("bf16", "f16", "f32"):
            b, wd = SIZE[w], mxw(bb, w)
            for pe, npg in ((2048 + 24, 16), (64, 40), (8192, 3)):  # MX blocks straddle pages in the first
                blob = _values(rng, pe * npg, w)
                key = f"x/{w}/{pe}"
                assert cl.batch_put_device_fp8([key], [blob.ctypes.data], [pe * npg], bb.WorkerConfig(
                    replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU]), 0, wide=wd) == [bb.ErrorCode.OK]
                want = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(blob.view(NP[w]), wd), pe * npg, wd), dtype=np.uint8)
                for mask in _masks(rng, npg):
                    ar = Arena(npg * (pe * b + 64) + MiB)
                    offs = ar.pages(npg, pe * b, shuffle=rng)
                    assert cl.batch_get_device_fp8_paged([key], [ar.table(offs, mask)], [pe], 0, wide=wd) == [bb.ErrorCode.OK]
                    assert np.array_equal(ar.raw, ar.expect(offs, mask, pe * b, want)), (w, pe, mask)
            # fail-over past a corrupt copy, then every copy corrupt with nothing stored: CHECKSUM_MISMATCH
            copies = cl.get_workers(key)

            def flip(sh, pos):
                wk = [wk for wk in c.workers if wk.backend(sh.pool_id) is not None][0]
                off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
                be = wk.backend(sh.pool_id)
                be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))

            mask = np.arange(npg) == 1
            flip(copies[0].shards[0], 11)
            ar = Arena(npg * (pe * b + 64) + MiB)
            offs = ar.pages(npg, pe * b)
            assert cl.batch_get_device_fp8_paged([key], [ar.table(offs, mask)], [pe], 0, wide=wd) == [bb.ErrorCode.OK]
            assert np.array_equal(ar.raw, ar.expect(offs, mask, pe * b, want))
            flip(copies[1].shards[0], 11)
            ar = Arena(npg * (pe * b + 64) + MiB)
            offs = ar.pages(npg, pe * b)
            assert cl.batch_get_device_fp8_paged([key], [ar.table(offs, np.zeros(npg, bool))], [pe], 0, wide=wd) == [bb.ErrorCode.CHECKSUM_MISMATCH]
            assert (ar.raw == GUARD).all()


def test_puts_refuse_null_pages_alone(bb):
    E = bb.ErrorCode
    with LocalCluster(cluster_id="spp", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        ar = Arena(4 * MiB)
        offs = ar.pages(8, 4096)
        ar.raw[:] = np.frombuffer(os.urandom(ar.raw.size), dtype=np.uint8)
        full = ar.table(offs, np.ones(8, bool))
        holed = ar.table(offs, np.arange(8) != 3)
        before = _counter(cl, "device_put_paged_total")
        ecs = cl.batch_put_device_paged(["a", "hole", "b"], [full, holed, full], [4096] * 3, _cfg(bb, 1, 1), 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.OK]
        assert not cl.object_exists("hole") and cl.object_exists("a") and cl.object_exists("b")
        assert _counter(cl, "device_put_paged_total") == before + 2
        ecs = cl.batch_put_device_fp8_paged(["fa", "fhole", "fb"], [full, holed, full], [2048] * 3, _cfg(bb, 1, 1), 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.OK]
        assert not cl.object_exists("fhole") and cl.object_exists("fa") and cl.object_exists("fb")
