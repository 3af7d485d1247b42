"""Paged puts and gets whose pages are rows inside their blocks (a head slice of a KV cache) on CPU: the in-page row
pattern of SourcePages / SourceBlocks against an independent numpy model, and the eight paged and blocks client calls
through the HostLoopbackTransport, which follows the same rule the kernels do.  Addresses here are host addresses."""
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
def model_addr(addrs, page, phase, rw, rp, x):
    """Where object byte x lives: page k = (x + phase) // page, c = (x + phase) % page, then c's row and column."""
    y = np.asarray(x, dtype=np.int64) + phase
    k, c = y // page, y % page
    inner = c if rw == 0 else c // rw * rp + c % rw
    return np.asarray(addrs, dtype=np.int64)[k] + inner


def model_runs(addrs, page, phase, rw, rp, n):
    """Maximal runs of object bytes whose addresses follow one another, skipping null pages."""
    if n == 0:
        return []
    x = np.arange(n)
    a = model_addr(addrs, page, phase, rw, rp, x)
    live = np.asarray(addrs, dtype=np.int64)[(x + phase) // page] != 0
    runs, s = [], None
    for i in range(n):
        if not live[i]:
            if s is not None:
                runs.append((s, int(a[s]), i - s))
            s = None
        elif s is None or a[i] != a[i - 1] + 1:
            if s is not None:
                runs.append((s, int(a[s]), i - s))
            s = i
    if s is not None:
        runs.append((s, int(a[s]), n - s))
    return runs


def model_coaligned(addrs, page, phase, rw, rp, n):
    if n == 0:
        return True
    k = (n - 1 + phase) // page + 1
    if (k > 1 and page % 16) or (rw and (rp - rw) % 16):
        return False
    return all(a == 0 or (a + phase) % 16 == 0 for a in addrs[:k])


def test_rows_match_the_numpy_model(bb):
    rng = np.random.default_rng(17)
    for _ in range(300):
        npages = int(rng.integers(1, 12))
        rw = int(rng.choice([1, 3, 16, 32, 48]))
        n = int(rng.choice([2, 3, 4, 8]))
        rp = rw + int(rng.choice([1, 5, 16, 32, 80]))
        page = rw * n
        extent = (n - 1) * rp + rw
        base = int(rng.integers(1, 1 << 40)) * 16
        order = rng.permutation(npages)
        addrs = [base + int(o) * (extent + 64) + (int(rng.integers(0, 16)) if rng.random() < 0.2 else 0) for o in order]
        if rng.random() < 0.3:
            addrs[int(rng.integers(0, npages))] = 0  # a null page (partial restore)
        ec, t, size = bb.SourcePages.from_pages(addrs, page, rw, rp)
        assert ec == bb.ErrorCode.OK and size == npages * page and (t.row_width, t.row_pitch) == (rw, rp)
        # every object byte at the model's address
        x = np.arange(size)
        live = np.asarray(addrs, dtype=np.int64)[x // page] != 0
        got = {}
        for xs, at, m in t.runs(size):
            for j in range(m):
                got[xs + j] = at + j
        want = model_addr(addrs, page, 0, rw, rp, x)
        assert sorted(got) == list(x[live]) and all(got[i] == want[i] for i in got)
        for off in sorted({0, size, *[int(v) for v in rng.integers(0, size + 1, 6)]}):
            r = t.rebase(off)
            k = min(off // page, npages)
            assert (r.phase, r.addrs, r.row_width, r.row_pitch) == (off % page, addrs[k:], rw, rp)
            assert r.runs(size - off) == model_runs(addrs[k:], page, off % page, rw, rp, size - off)
            assert r.coaligned(size - off) == model_coaligned(addrs[k:], page, off % page, rw, rp, size - off)
            # the get rule: also page % 16 whenever the table has several pages, and the row gap from the call's shape
            fused = (npages <= 1 or page % 16 == 0) and model_coaligned(addrs[k:], page, off % page, rw, rp, size - off)
            assert t.fused_get_aligned(off, size - off) == fused
        ok, w = t.to_wide_bytes(2)
        assert ok and (w.page, w.row_width, w.row_pitch, w.addrs) == (2 * page, 2 * rw, 2 * rp, addrs)


def test_row_gap_decides_fusing_even_for_one_row(bb):
    """A shard that holds a single in-page row still needs a gap that is a multiple of 16: the call's shape decides."""
    ec, t, size = bb.SourcePages.from_pages([4096, 8192], 64, 32, 40)
    assert ec == bb.ErrorCode.OK and size == 128
    assert not t.coaligned(16)
    assert not t.fused_get_aligned(0, 16) and not t.fused_get_aligned(0, size)
    ec, t, _ = bb.SourcePages.from_pages([4096, 8192], 64, 32, 48)
    assert t.fused_get_aligned(0, 16) and t.fused_get_aligned(0, 128)


def test_pattern_admission_codes(bb):
    E = bb.ErrorCode
    sp = bb.SourcePages.from_pages
    assert sp([16, 4096], 64, 32, 16)[0] == E.INVALID_ARGUMENT   # row_width > row_pitch
    assert sp([16, 4096], 64, 24, 48)[0] == E.INVALID_ARGUMENT   # page % row_width != 0
    assert sp([16, 4096], 64, 32, 0)[0] == E.INVALID_ARGUMENT    # exactly one of them 0
    assert sp([16, 4096], 64, 0, 48)[0] == E.INVALID_ARGUMENT
    assert sp([16, 4096], 1 << 62, 1, 1 << 62)[0] == E.VALUE_OUT_OF_RANGE  # the page's extent overflows
    assert sp([], 64, 32, 16)[0] == E.OK  # no pages: a zero-byte object
    # rows that touch, and one row per page, are plain pages
    for rw, rp in ((32, 32), (64, 96)):
        ec, t, size = sp([16, 4096], 64, rw, rp)
        assert ec == E.OK and size == 128 and (t.row_width, t.row_pitch) == (0, 0)
    ids = np.array([1, 0], dtype=np.int32)
    db = bb.DeviceBlocks
    assert db([16], ids.ctypes.data, 2, 4, 4096, 64, row_width=32, row_pitch=16).size()[0] == E.INVALID_ARGUMENT
    assert db([16], ids.ctypes.data, 2, 4, 4096, 64, row_width=24, row_pitch=48).size()[0] == E.INVALID_ARGUMENT
    assert db([16], ids.ctypes.data, 2, 4, 4096, 64, row_width=0, row_pitch=48).size()[0] == E.INVALID_ARGUMENT
    assert db([16], ids.ctypes.data, 2, 4, 4096, 64, row_width=32, row_pitch=48).size() == (E.OK, 128)
    b = db([16], ids.ctypes.data, 2, 4, 4096, 64, row_width=32, row_pitch=48)
    ok, w = b.to_wide_bytes(4)
    assert ok and (w.page, w.row_width, w.row_pitch) == (256, 128, 192)
    # closed-form co-alignment: the row gap counts like the stride
    assert b.coaligned(128)
    assert not db([16], ids.ctypes.data, 2, 4, 4096, 64, row_width=32, row_pitch=40).coaligned(128)


# ---------------------------------------------------------------- client calls through the loopback transport
class HeadCache:
    """A guard-filled host cache of `nb` blocks, each `nrows` rows of `pitch` bytes; the slice is `width` bytes at `col`
    of every row (a head slice).  Page k of a table is block ids[k]'s slice."""

    def __init__(self, nb, nrows, pitch, width, col, skew=0):
        self.nb, self.nrows, self.pitch, self.width, self.col = nb, nrows, pitch, width, col
        self.block = nrows * pitch + 32
        self.raw = np.full(nb * self.block + 64, GUARD, dtype=np.uint8)
        self.o = (-self.raw.ctypes.data) % 16 + skew

    def addrs(self, ids):
        return [self.raw.ctypes.data + self.o + int(b) * self.block + self.col for b in ids]

    def rows(self, b):
        s = self.o + b * self.block + self.col
        return [slice(s + r * self.pitch, s + r * self.pitch + self.width) for r in range(self.nrows)]

    def fill(self, rng):
        for b in range(self.nb):
            for sl in self.rows(b):
                self.raw[sl] = rng.integers(0, 256, self.width, dtype=np.uint8)

    def selected(self, ids):
        return np.concatenate([self.raw[sl] for b in ids for sl in self.rows(int(b))])

    def expect(self, ids, blob):
        want = np.full_like(self.raw, GUARD)
        x = 0
        for b in ids:
            for sl in self.rows(int(b)):
                want[sl] = blob[x:x + self.width]
                x += self.width
        return want

    @property
    def page(self):
        return self.nrows * self.width


def test_paged_rows_put_and_get_match_the_dense_object(bb):
    """A paged put of head slices stores the dense index_select bytes (same digests as a plain put of them), and a paged
    get stores exactly the rows, every guard byte untouched: striped, replicated, every digest."""
    rng = np.random.default_rng(3)
    with LocalCluster(cluster_id="prw", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            for replicas, stripes in ((1, 1), (2, 1), (1, 3), (2, 2)):
                src = HeadCache(12, 16, 512, 128, 256)
                src.fill(rng)
                ids = rng.permutation(12)[:7]
                blob = src.selected(ids)
                before = src.raw.copy()
                cfg = _cfg(bb, replicas, stripes, algo)
                key, ref = f"h/{algo}/{replicas}/{stripes}", f"r/{algo}/{replicas}/{stripes}"
                assert cl.batch_put_device_paged([key], [src.addrs(ids)], [src.page], cfg, 0, rows=[(128, 512)]) == [bb.ErrorCode.OK]
                assert np.array_equal(src.raw, before)
                assert cl.batch_put_device([ref], [blob.ctypes.data], [blob.size], cfg, 0) == [bb.ErrorCode.OK]
                if stripes == 1:
                    assert [[s.checksum for s in cp.shards] for cp in cl.get_workers(key)] == \
                        [[s.checksum for s in cp.shards] for cp in cl.get_workers(ref)]
                out = np.zeros(blob.size, np.uint8)
                ecs, _ = cl.batch_get_device([key], [out.ctypes.data], [out.size], 0)
                assert ecs == [bb.ErrorCode.OK] and np.array_equal(out, blob)
                dst = HeadCache(12, 16, 512, 128, 256)
                into = rng.permutation(12)[:7]
                ecs, sizes = cl.batch_get_device_paged([ref], [dst.addrs(into)], [dst.page], 0, rows=[(128, 512)])
                assert ecs == [bb.ErrorCode.OK] and sizes == [blob.size]
                assert np.array_equal(dst.raw, dst.expect(into, blob))


def test_staged_rows_and_null_pages(bb):
    """Items that are not co-aligned (a skewed cache, a gap that is not a multiple of 16) are staged through the host
    row by row, next to fused ones; a null page stores nothing; rows=None entries are plain pages."""
    rng = np.random.default_rng(4)
    with LocalCluster(cluster_id="prs", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1, 2)
        caches = [HeadCache(6, 8, 256, 64, 64), HeadCache(6, 8, 256, 64, 64, skew=4), HeadCache(6, 8, 200, 64, 16)]
        for h in caches:
            h.fill(rng)
        ids = [3, 0, 5]
        keys = ["fused", "skew", "gap"]
        staged = _counter(cl, "device_put_host_staged_total")
        assert cl.batch_put_device_paged(keys, [h.addrs(ids) for h in caches], [h.page for h in caches], cfg, 0,
                                         rows=[(64, h.pitch) for h in caches]) == [bb.ErrorCode.OK] * 3
        assert _counter(cl, "device_put_host_staged_total") == staged + 2
        for k, h in zip(keys, caches):
            assert np.array_equal(np.frombuffer(cl.get(k), dtype=np.uint8), h.selected(ids))
        dsts = [HeadCache(6, 8, h.pitch, 64, h.col, skew=4 if k == "skew" else 0) for k, h in zip(keys, caches)]
        into = [1, 4, 2]
        staged = _counter(cl, "device_get_host_staged_total")
        ecs, _ = cl.batch_get_device_paged(keys, [d.addrs(into) for d in dsts], [d.page for d in dsts], 0,
                                           rows=[(64, d.pitch) for d in dsts])
        assert ecs == [bb.ErrorCode.OK] * 3 and _counter(cl, "device_get_host_staged_total") > staged
        for k, h, d in zip(keys, caches, dsts):
            assert np.array_equal(d.raw, d.expect(into, h.selected(ids))), k
        # a null page: its rows are not stored, the others are
        d = HeadCache(6, 8, 256, 64, 64)
        table = d.addrs(into)
        table[1] = 0
        ecs, _ = cl.batch_get_device_paged(["fused"], [table], [d.page], 0, rows=[(64, 256)])
        assert ecs == [bb.ErrorCode.OK]
        want = d.expect(into, caches[0].selected(ids))
        for sl in d.rows(4):
            want[sl] = GUARD
        assert np.array_equal(d.raw, want)
        # rows=[None] is a plain paged get of whole pages
        plain = np.full(3 * 512 + 64, GUARD, dtype=np.uint8)
        p0 = (-plain.ctypes.data) % 16
        addrs = [plain.ctypes.data + p0 + 512 * k for k in range(3)]
        ecs, _ = cl.batch_get_device_paged(["fused"], [addrs], [512], 0, rows=[None])
        assert ecs == [bb.ErrorCode.OK] and np.array_equal(plain[p0:p0 + 1536], caches[0].selected(ids))
        # the pattern's admission errors, per item, before anything is stored
        ecs = cl.batch_put_device_paged(["e1", "e2"], [caches[0].addrs(ids)] * 2, [512, 512], cfg, 0, rows=[(64, 32), (48, 256)])
        assert ecs == [bb.ErrorCode.INVALID_ARGUMENT] * 2 and not cl.object_exists("e1")
        assert cl.batch_put_device_paged(["e3"], [caches[0].addrs(ids)], [512], cfg, 0, rows=[(64, 256), (64, 256)]) == \
            [bb.ErrorCode.INVALID_PARAMETERS]


def test_fail_over_and_refresh_with_rows(bb):
    with LocalCluster(cluster_id="prf", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))

        src = HeadCache(20, 16, 1024, 256, 512)
        src.fill(np.random.default_rng(8))
        ids = list(range(19, -1, -1))
        assert cl.batch_put_device_paged(["f"], [src.addrs(ids)], [src.page], _cfg(bb, 3, 2), 0, rows=[(256, 1024)]) == [bb.ErrorCode.OK]
        blob = src.selected(ids)
        copies = cl.get_workers("f")
        for cp in copies:
            flip(cp.shards[-1], 77)
            dst = HeadCache(20, 16, 1024, 256, 512)
            ecs, _ = cl.batch_get_device_paged(["f"], [dst.addrs(ids)], [dst.page], 0, rows=[(256, 1024)])
            assert ecs == [bb.ErrorCode.OK] and np.array_equal(dst.raw, dst.expect(ids, blob))
            flip(cp.shards[-1], 77)
        for cp in copies:
            flip(cp.shards[0], 5)
        ref = _counter(cl, "get_placement_refresh_total")
        dst = HeadCache(20, 16, 1024, 256, 512)
        ecs, _ = cl.batch_get_device_paged(["f"], [dst.addrs(ids)], [dst.page], 0, rows=[(256, 1024)])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH] and _counter(cl, "get_placement_refresh_total") == ref + 1


def _bf16_values(rng, n):
    return (rng.standard_normal(n).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)


def test_packed_and_blocks_calls_with_rows(bb):
    """The MXFP8 paged calls and the byte and MXFP8 blocks calls take the pattern too: the stored objects are those of
    the dense slices (packed: packing them), gets store exactly the rows, refused ids store nothing, and an item that is
    not co-aligned is NOT_IMPLEMENTED."""
    E, W = bb.ErrorCode, bb.MxWide.BF16
    rng = np.random.default_rng(9)
    with LocalCluster(cluster_id="prp", n_workers=2, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        # bf16 cache: rows of 64 elements (128 bytes) every 256 elements, 8 rows per block
        src = HeadCache(10, 8, 512, 128, 128)
        for b in range(10):
            for sl in src.rows(b):
                src.raw[sl] = _bf16_values(rng, 64).view(np.uint8)
        ids = np.array([4, 9, 0, 2], dtype=np.int32)
        dense = src.selected(ids)
        n = dense.size // 2
        packed_want = np.frombuffer(bb.mxfp8_pack_ref(dense.view(np.uint16), W), dtype=np.uint8)
        unpacked = np.frombuffer(bb.mxfp8_unpack_ref(packed_want, n, W), dtype=np.uint8)
        pe, rows = src.page // 2, (64, 256)
        skew = HeadCache(10, 8, 512, 128, 128, skew=2)
        assert cl.batch_put_device_fp8_paged(["p8", "p8s"], [src.addrs(ids), skew.addrs(ids)], [pe, pe], cfg, 0, wide=W,
                                             rows=[rows, rows]) == [E.OK, E.NOT_IMPLEMENTED]
        assert np.array_equal(np.frombuffer(cl.get("p8"), dtype=np.uint8), packed_want)
        dst = HeadCache(10, 8, 512, 128, 128)
        into = np.array([1, 3, 8, 6], dtype=np.int32)
        assert cl.batch_get_device_fp8_paged(["p8"], [dst.addrs(into)], [pe], 0, wide=W, rows=[rows]) == [E.OK]
        assert np.array_equal(dst.raw, dst.expect(into, unpacked))

        def blocks(cache, i, unit, sel=None, n_stored=0):
            return bb.DeviceBlocks([cache.raw.ctypes.data + cache.o + cache.col], i.ctypes.data, i.size, cache.nb, cache.block,
                                   cache.page // unit, id_bytes=i.itemsize, sel=0 if sel is None else sel.ctypes.data,
                                   n_stored=n_stored, row_width=cache.width // unit, row_pitch=cache.pitch // unit)

        high = np.array([4, 10, 0, 2], dtype=np.int32)
        assert cl.batch_put_device_blocks(["b", "bhigh"], [blocks(src, ids, 1), blocks(src, high, 1)], cfg, 0) == [E.OK, E.VALUE_OUT_OF_RANGE]
        assert np.array_equal(np.frombuffer(cl.get("b"), dtype=np.uint8), dense) and not cl.object_exists("bhigh")
        dst = HeadCache(10, 8, 512, 128, 128)
        ecs, sizes = cl.batch_get_device_blocks(["b"], [blocks(dst, into, 1)], 0)
        assert ecs == [E.OK] and sizes == [dense.size] and np.array_equal(dst.raw, dst.expect(into, dense))
        dup = np.array([1, 1, 8, 6], dtype=np.int32)
        dst = HeadCache(10, 8, 512, 128, 128)
        assert cl.batch_get_device_blocks(["b"], [blocks(dst, dup, 1)], 0)[0] == [E.INVALID_ARGUMENT]
        assert (dst.raw == GUARD).all()
        # a partial restore: stored blocks 3 and 0 into cache blocks 7 and 5
        sel, part = np.array([3, 0], dtype=np.int32), np.array([7, 5], dtype=np.int32)
        dst = HeadCache(10, 8, 512, 128, 128)
        assert cl.batch_get_device_blocks(["b"], [blocks(dst, part, 1, sel, 4)], 0)[0] == [E.OK]
        per = src.page
        assert np.array_equal(dst.raw, dst.expect(part, np.concatenate([dense[3 * per:4 * per], dense[:per]])))
        # packed blocks
        assert cl.batch_put_device_fp8_blocks(["b8", "b8s"], [blocks(src, ids, 2), blocks(skew, ids, 2)], cfg, 0, wide=W) == \
            [E.OK, E.NOT_IMPLEMENTED]
        assert np.array_equal(np.frombuffer(cl.get("b8"), dtype=np.uint8), packed_want)
        dst = HeadCache(10, 8, 512, 128, 128)
        assert cl.batch_get_device_fp8_blocks(["b8"], [blocks(dst, into, 2)], 0, wide=W) == [E.OK]
        assert np.array_equal(dst.raw, dst.expect(into, unpacked))
        # blocks that are not co-aligned have no host-staged path
        ecs, _ = cl.batch_get_device_blocks(["b"], [blocks(skew, into, 1)], 0)
        assert ecs == [E.NOT_IMPLEMENTED]
