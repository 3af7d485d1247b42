"""Paged puts and gets from block ids that stay on the device, on CPU: the SourceBlocks rule (its host resolve, verdicts,
rebase at shard cuts and closed-form co-alignment) against an independent numpy model, and batch_put_device_blocks /
batch_get_device_blocks through the HostLoopbackTransport -- striped and replicated objects, fail-over, the placement
refresh, placements that would need host staging, and refused ids -- with every guard byte checked.  The loopback's
"device" pointers are host pointers, so the ids here are numpy arrays that its host resolve reads."""
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
def model_verdict(ids, n_blocks, sel, n_stored, get):
    """0 OK, 1 out of range, 2 duplicate (a get's)."""
    if ((ids < 0) | (ids >= n_blocks)).any() or (sel is not None and ((sel < 0) | (sel >= n_stored)).any()):
        return 1
    if get and (np.unique(ids).size != ids.size or (sel is not None and np.unique(sel).size != sel.size)):
        return 2
    return 0


def model_table(outer, ids, stride, sel, n_stored, verdict, get):
    """Every page address of the object, page r = q * per + k; refused: 0 for a get, outer[q] for a put."""
    outer = np.asarray(outer, dtype=np.int64)
    per = ids.size if sel is None else n_stored
    if verdict:
        return np.zeros(outer.size * per, np.int64) if get else np.repeat(outer, per)
    if sel is None:
        return (outer[:, None] + ids[None, :].astype(np.int64) * stride).reshape(-1)
    t = np.zeros((outer.size, n_stored), np.int64)
    t[:, sel] = outer[:, None] + ids[None, :].astype(np.int64) * stride
    return t.reshape(-1)


def test_source_blocks_match_the_numpy_model(bb):
    E = bb.ErrorCode
    codes = {0: E.OK, 1: E.VALUE_OUT_OF_RANGE, 2: E.INVALID_ARGUMENT}
    rng = np.random.default_rng(31)
    for trial in range(500):
        dt = np.int32 if trial % 2 else np.int64
        n_outer = int(rng.integers(1, 6))
        n_blocks = int(rng.integers(1, 40))
        n_ids = int(rng.integers(1, 12))
        stride = int(rng.choice([16, 48, 4096, 100]))
        page = int(rng.choice([16, 48, 4096, 3]))
        outer = [int(rng.integers(1, 1 << 36)) * 16 + (int(rng.integers(0, 16)) if rng.random() < 0.2 else 0) for _ in range(n_outer)]
        ids = rng.integers(-1 if rng.random() < 0.1 else 0, n_blocks + (1 if rng.random() < 0.1 else 0), n_ids).astype(dt)
        if rng.random() < 0.5:  # most tables without repeats
            ids = rng.permutation(max(n_blocks, n_ids))[:n_ids].astype(dt)
        sel, n_stored = None, 0
        if rng.random() < 0.4:
            n_stored = n_ids + int(rng.integers(0, 5))
            sel = rng.permutation(n_stored)[:n_ids].astype(dt)
            if rng.random() < 0.2:
                sel[0] = sel[-1] if rng.random() < 0.5 else n_stored
        b = bb.DeviceBlocks(outer, ids.ctypes.data, n_ids, n_blocks, stride, page, id_bytes=ids.itemsize,
                            sel=0 if sel is None else sel.ctypes.data, n_stored=n_stored)
        ec, size = b.size()
        per = n_ids if sel is None else n_stored
        assert ec == E.OK and size == n_outer * per * page and b.npages == n_outer * per
        for get in (False, True):
            v = model_verdict(ids.astype(np.int64), n_blocks, None if sel is None else sel.astype(np.int64), n_stored, get)
            want = model_table(outer, ids, stride, None if sel is None else sel.astype(np.int64), n_stored, v, get)
            off = int(rng.integers(0, size))
            r = b.rebase(off)
            assert r.first == off // page and r.phase == off % page
            count = r.npages - r.first
            got_v, table = r.resolve(count, get)
            assert got_v == codes[v], (trial, get)
            assert np.array_equal(np.asarray(table, dtype=np.uint64), want[r.first:].astype(np.uint64)), (trial, get)
        # closed-form co-alignment: every table the ids could make is co-aligned, without reading them
        n = size - off
        touched = (n - 1 + off % page) // page + 1
        assert r.coaligned(n) == ((touched <= 1 or page % 16 == 0) and stride % 16 == 0 and all((o + off % page) % 16 == 0 for o in outer))
        assert b.fused_get_aligned(off, n) == ((b.npages <= 1 or page % 16 == 0) and r.coaligned(n))
        assert b.has_null() == (sel is not None)


def test_source_blocks_shape_errors(bb):
    E = bb.ErrorCode
    ids = np.arange(4, dtype=np.int32)
    assert bb.DeviceBlocks([16], ids.ctypes.data, 4, 8, 16, 0).size()[0] == E.INVALID_ARGUMENT  # page 0 with pages
    assert bb.DeviceBlocks([16], ids.ctypes.data, 4, 8, 16, 16, id_bytes=2).size()[0] == E.INVALID_ARGUMENT
    assert bb.DeviceBlocks([16], ids.ctypes.data, 4, 8, 16, 16, sel=ids.ctypes.data, n_stored=0).size()[0] == E.INVALID_ARGUMENT
    assert bb.DeviceBlocks([16] * 4, ids.ctypes.data, 4, 8, 16, 1 << 62).size()[0] == E.VALUE_OUT_OF_RANGE
    assert bb.DeviceBlocks([], ids.ctypes.data, 4, 8, 16, 16).size() == (E.OK, 0)
    assert not bb.DeviceBlocks([16], ids.ctypes.data, 4, 1 << 19, 16, 16).distinct_checkable()


# ---------------------------------------------------------------- client calls through the loopback transport
class Cache:
    """Per-layer caches [n_outer, n_blocks, page] in guard-filled host memory: block b of slice o of layer l at
    outer[l * n_outer + o] + b * stride, with a guard gap after every page when stride > page."""

    def __init__(self, layers, n_outer, n_blocks, page, stride, skew=0, fill=False):
        self.shape = (layers, n_outer, n_blocks)
        self.page, self.stride = page, stride
        self.raw = np.full(layers * n_outer * n_blocks * stride + 4096, GUARD, dtype=np.uint8)
        self.o0 = (-self.raw.ctypes.data) % 16 + 64 + skew
        self.outer = [self.raw.ctypes.data + self.o0 + q * n_blocks * stride for q in range(layers * n_outer)]
        if fill:
            for q in range(layers * n_outer):
                for b in range(n_blocks):
                    at = self.o0 + (q * n_blocks + b) * stride
                    self.raw[at:at + page] = np.frombuffer(os.urandom(page), dtype=np.uint8)

    def block(self, q, b):
        at = self.o0 + (q * self.shape[2] + b) * self.stride
        return self.raw[at:at + self.page]

    def blocks(self, ids, sel=None, n_stored=0):
        return bb_blocks(self, ids, sel, n_stored)

    def selected(self, ids):
        """The stored object of a put of `ids`: every slice's blocks, layer-major."""
        return np.concatenate([self.block(q, int(b)) for q in range(len(self.outer)) for b in ids])

    def expect(self, ids, blob, sel=None, n_stored=0):
        """The raw memory after a get of `blob` into blocks `ids` (with a selection, stored block sel[m] into ids[m])."""
        want = np.full_like(self.raw, GUARD)
        per = len(ids) if sel is None else n_stored
        for q in range(len(self.outer)):
            for m, b in enumerate(ids):
                r = q * per + (m if sel is None else int(sel[m]))
                at = self.o0 + (q * self.shape[2] + int(b)) * self.stride
                want[at:at + self.page] = blob[r * self.page:(r + 1) * self.page]
        return want


_BB = None


def bb_blocks(cache, ids, sel, n_stored):
    return _BB.DeviceBlocks(cache.outer, ids.ctypes.data, ids.size, cache.shape[2], cache.stride, cache.page, id_bytes=ids.itemsize,
                            sel=0 if sel is None else sel.ctypes.data, n_stored=n_stored)


@pytest.fixture(autouse=True)
def _bind(bb):
    global _BB
    _BB = bb


def test_blocks_round_trip_striped_and_replicated(bb):
    E = bb.ErrorCode
    rng = np.random.default_rng(32)
    with LocalCluster(cluster_id="lbk", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        for algo in ("XXH3", "NONE"):
            for replicas, stripes in ((1, 1), (2, 1), (1, 3), (2, 2)):
                for dt in (np.int32, np.int64):
                    src = Cache(3, 2, 24, 4096, 4096 + 48, fill=True)
                    ids = rng.permutation(24)[:int(rng.integers(2, 9))].astype(dt)
                    key = f"b/{algo}/{replicas}/{stripes}/{dt.__name__}"
                    assert cl.batch_put_device_blocks([key], [src.blocks(ids)], _cfg(bb, replicas, stripes, algo), 0) == [E.OK]
                    blob = src.selected(ids)
                    back = np.zeros_like(blob)
                    ecs, sizes = cl.batch_get_device([key], [back.ctypes.data], [back.size], 0)
                    assert ecs == [E.OK] and sizes == [blob.size] and np.array_equal(back, blob), key
                    # whole, into other blocks of another cache
                    dst = Cache(3, 2, 24, 4096, 4096 + 48)
                    into = rng.permutation(24)[:ids.size].astype(dt)
                    ecs, sizes = cl.batch_get_device_blocks([key], [dst.blocks(into)], 0)
                    assert ecs == [E.OK] and sizes == [blob.size]
                    assert np.array_equal(dst.raw, dst.expect(into, blob)), key
                    # partial: k of the stored blocks
                    k = int(rng.integers(1, ids.size + 1))
                    sel = rng.permutation(ids.size)[:k].astype(dt)
                    dst = Cache(3, 2, 24, 4096, 4096 + 48)
                    into = rng.permutation(24)[:k].astype(dt)
                    ecs, sizes = cl.batch_get_device_blocks([key], [dst.blocks(into, sel, ids.size)], 0)
                    assert ecs == [E.OK] and sizes == [blob.size]
                    assert np.array_equal(dst.raw, dst.expect(into, blob, sel, ids.size)), key


def test_blocks_gets_fail_over_and_refresh(bb):
    E = bb.ErrorCode
    with LocalCluster(cluster_id="lbf", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))

        src = Cache(2, 1, 16, 4096, 4096, fill=True)
        ids = np.array([5, 1, 9, 12], dtype=np.int32)
        assert cl.batch_put_device_blocks(["f"], [src.blocks(ids)], _cfg(bb, 3, 2), 0) == [E.OK]
        blob = src.selected(ids)
        fo = _counter(cl, "replica_failover_total")
        for cp in cl.get_workers("f"):
            flip(cp.shards[-1], 77)
            dst = Cache(2, 1, 16, 4096, 4096)
            ecs, _ = cl.batch_get_device_blocks(["f"], [dst.blocks(ids)], 0)
            assert ecs == [E.OK] and np.array_equal(dst.raw, dst.expect(ids, blob))
            flip(cp.shards[-1], 77)
        assert _counter(cl, "replica_failover_total") > fo
        for cp in cl.get_workers("f"):
            flip(cp.shards[0], 5)
        ref = _counter(cl, "get_placement_refresh_total")
        dst = Cache(2, 1, 16, 4096, 4096)
        ecs, _ = cl.batch_get_device_blocks(["f"], [dst.blocks(ids)], 0)
        assert ecs == [E.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1


def test_unaligned_blocks_are_not_staged(bb):
    """A table that is not co-aligned would need the host to read the ids: NOT_IMPLEMENTED, the put cancelled, the get
    storing nothing, while the rest of the batch completes."""
    E = bb.ErrorCode
    with LocalCluster(cluster_id="lbs", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        good = Cache(2, 1, 8, 4096, 4096, fill=True)
        skewed = Cache(2, 1, 8, 4096, 4096, skew=4, fill=True)
        odd = Cache(2, 1, 8, 4096, 4096 + 8, fill=True)
        ids = np.array([3, 0, 6], dtype=np.int64)
        ecs = cl.batch_put_device_blocks(["a", "skew", "odd", "b"], [good.blocks(ids), skewed.blocks(ids), odd.blocks(ids), good.blocks(ids)],
                                         _cfg(bb, 1, 1), 0)
        assert ecs == [E.OK, E.NOT_IMPLEMENTED, E.NOT_IMPLEMENTED, E.OK]
        assert cl.object_exists("a") and cl.object_exists("b") and not cl.object_exists("skew") and not cl.object_exists("odd")
        dst = Cache(2, 1, 8, 4096, 4096, skew=4)
        ok = Cache(2, 1, 8, 4096, 4096)
        ecs, _ = cl.batch_get_device_blocks(["a", "b"], [dst.blocks(ids), ok.blocks(ids)], 0)
        assert ecs == [E.NOT_IMPLEMENTED, E.OK]
        assert (dst.raw == GUARD).all() and np.array_equal(ok.raw, ok.expect(ids, good.selected(ids)))


def test_refused_ids_store_nothing_and_the_batch_carries_on(bb):
    E = bb.ErrorCode
    with LocalCluster(cluster_id="lbr", n_workers=3, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        src = Cache(2, 2, 8, 4096, 4096 + 16, fill=True)
        good = np.array([2, 7, 1], dtype=np.int32)
        high = np.array([2, 8, 1], dtype=np.int32)
        neg = np.array([2, -1, 1], dtype=np.int64)
        dup = np.array([2, 2, 1], dtype=np.int32)
        before = _counter(cl, "device_put_blocks_total")
        ecs = cl.batch_put_device_blocks(["p", "high", "neg", "dup", "sel", "q"],
                                         [src.blocks(good), src.blocks(high), src.blocks(neg), src.blocks(dup),
                                          src.blocks(good, good, 8), src.blocks(good)], _cfg(bb, 2, 2), 0)
        # a put may repeat ids, as batch_put_device_paged may repeat pages; it may not take a selection
        assert ecs == [E.OK, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.OK, E.INVALID_ARGUMENT, E.OK]
        for k, there in (("p", True), ("high", False), ("neg", False), ("dup", True), ("sel", False), ("q", True)):
            assert cl.object_exists(k) == there, k
        assert _counter(cl, "device_put_blocks_total") == before + 3
        back = np.zeros(src.selected(dup).size, np.uint8)
        assert cl.batch_get_device(["dup"], [back.ctypes.data], [back.size], 0)[0] == [E.OK]
        assert np.array_equal(back, src.selected(dup))
        blob = src.selected(good)
        caches = [Cache(2, 2, 8, 4096, 4096 + 16) for _ in range(6)]
        sel_high, sel_dup, sel_two, two = (np.array(v, np.int32) for v in ([0, 3, 1], [0, 1, 1], [2, 0], good[:2]))  # alive for the call
        tables = [caches[0].blocks(good), caches[1].blocks(high), caches[2].blocks(dup), caches[3].blocks(good, sel_high, 3),
                  caches[4].blocks(good, sel_dup, 3), caches[5].blocks(two, sel_two, 3)]
        ecs, sizes = cl.batch_get_device_blocks(["p"] * 6, tables, 0)
        assert ecs == [E.OK, E.VALUE_OUT_OF_RANGE, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.INVALID_ARGUMENT, E.OK]
        assert np.array_equal(caches[0].raw, caches[0].expect(good, blob))
        for k in (1, 2, 3, 4):
            assert (caches[k].raw == GUARD).all(), k
        assert np.array_equal(caches[5].raw, caches[5].expect(two, blob, sel_two, 3))
        # the refusal is the answer, not a copy's fault: no fail-over, no refresh
        fo, ref = _counter(cl, "replica_failover_total"), _counter(cl, "get_placement_refresh_total")
        assert cl.batch_get_device_blocks(["p"], [caches[1].blocks(high)], 0)[0] == [E.VALUE_OUT_OF_RANGE]
        assert (_counter(cl, "replica_failover_total"), _counter(cl, "get_placement_refresh_total")) == (fo, ref)
        # a bound too large for the duplicate check is NOT_IMPLEMENTED for a get, not for a put
        big = bb.DeviceBlocks(src.outer, good.ctypes.data, 3, 1 << 19, 4096 + 16, 4096)
        assert cl.batch_get_device_blocks(["p"], [big], 0)[0] == [E.NOT_IMPLEMENTED]
        assert cl.batch_put_device_blocks(["big"], [big], _cfg(bb, 1, 1), 0) == [E.OK]


def _values(rng, n):
    """n bf16 values (as uint16) of many binades, some NaN and zero."""
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-12, 12, n))).astype(np.float32)
    v[::97] = np.nan
    v[7::331] = 0.0
    return (v.view(np.uint32) >> 16).astype(np.uint16)


def test_packed_blocks_through_the_loopback(bb):
    """batch_put_device_fp8_blocks / batch_get_device_fp8_blocks: the stored packed object is that of packing the gathered
    blocks (an MX block may straddle two pages), gets unpack into the named blocks whole and partial, refused ids cancel
    the put or store nothing, and an unaligned table is NOT_IMPLEMENTED."""
    E, W = bb.ErrorCode, bb.MxWide.BF16
    rng = np.random.default_rng(34)
    pe = 2048 + 16  # elements per page
    with LocalCluster(cluster_id="lbx", n_workers=2, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        src = Cache(2, 2, 12, pe * 2, pe * 2 + 32)
        for q in range(4):
            for b in range(12):
                src.block(q, b)[:] = _values(rng, pe).view(np.uint8)
        ids = np.array([7, 0, 11, 4], dtype=np.int32)
        high = np.array([7, 12, 1, 4], dtype=np.int32)

        def blocks(cache, i, sel=None, n_stored=0):
            return bb.DeviceBlocks(cache.outer, i.ctypes.data, i.size, 12, cache.stride, pe, id_bytes=i.itemsize,
                                   sel=0 if sel is None else sel.ctypes.data, n_stored=n_stored)

        skew = Cache(2, 2, 12, pe * 2, pe * 2 + 32, skew=2)
        assert cl.batch_put_device_fp8_blocks(["x", "high", "skew"], [blocks(src, ids), blocks(src, high), blocks(skew, ids)], cfg, 0, wide=W) == \
            [E.OK, E.VALUE_OUT_OF_RANGE, E.NOT_IMPLEMENTED]
        assert cl.object_exists("x") and not cl.object_exists("high") and not cl.object_exists("skew")
        n = 4 * ids.size * pe
        packed_want = np.frombuffer(bb.mxfp8_pack_ref(src.selected(ids).view(np.uint16), W), dtype=np.uint8)
        assert np.array_equal(np.frombuffer(cl.get("x"), dtype=np.uint8), packed_want)
        want = np.frombuffer(bb.mxfp8_unpack_ref(packed_want, n, W), dtype=np.uint8)
        for sel in (None, np.array([3, 0], dtype=np.int32)):
            into = np.array([9, 2, 5, 1], dtype=np.int64) if sel is None else np.array([10, 6], dtype=np.int32)
            if sel is not None:
                into = into.astype(np.int32)
            dst = Cache(2, 2, 12, pe * 2, pe * 2 + 32)
            assert cl.batch_get_device_fp8_blocks(["x"], [blocks(dst, into, sel, 0 if sel is None else ids.size)], 0, wide=W) == [E.OK]
            assert np.array_equal(dst.raw, dst.expect(into, want, sel, 0 if sel is None else ids.size))
        dup = np.array([9, 9, 5, 1], dtype=np.int32)
        dst = Cache(2, 2, 12, pe * 2, pe * 2 + 32)
        assert cl.batch_get_device_fp8_blocks(["x"], [blocks(dst, dup)], 0, wide=W) == [E.INVALID_ARGUMENT]
        assert (dst.raw == GUARD).all()
        short = np.array([9, 2, 5], dtype=np.int32)  # the pages must hold exactly the stored object
        assert cl.batch_get_device_fp8_blocks(["x"], [blocks(dst, short)], 0, wide=W) == [E.INVALID_ARGUMENT]
        assert (dst.raw == GUARD).all()
