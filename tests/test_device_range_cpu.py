"""Byte-range device gets (batch_get_device_range) on CPU: the HostLoopbackTransport stands in for the GPU fabric, so the
client's range logic -- ops for the overlapping shards only, windows in shard coordinates, replica choice and fail-over,
the host-staged path, the placement refresh -- runs in the CPU suite.  The loopback transport keeps the fabric's contract:
an overlapping shard is read whole and verified, only the window is stored."""
import os
import random
import threading
import time

import numpy as np

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


class Shards:
    """Shard offsets of an object's copies and byte flips in the worker that holds a shard."""

    def __init__(self, c, cl):
        self.c, self.cl = c, cl
        self.pools = {p.id: p for p in cl.keystone().get_memory_pools()}

    def layout(self, key):
        out = []
        for cp in self.cl.get_workers(key):
            offs, o = [], 0
            for sh in cp.shards:
                offs.append((o, sh))
                o += sh.length
            out.append(offs)
        return out

    def flip(self, sh, pos):
        w = [w for w in self.c.workers if w.backend(sh.pool_id) is not None][0]
        off = sh.location["remote_addr"] - self.pools[sh.pool_id].ucx_remote_addr + pos
        b = w.backend(sh.pool_id)
        b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))


def _aligned(n):
    """A guard-filled host buffer and the first 64-byte aligned offset in it past 64 guard bytes."""
    raw = np.full(n + 256, GUARD, dtype=np.uint8)
    a = (-raw.ctypes.data) % 64 + 64
    return raw, a


def _get_ranges(cl, keys, ranges, align_skew=None):
    """Range gets into one guard-filled buffer; returns (error codes, buffer, offsets of the ranges in it)."""
    total = sum(n + 128 for _, n in ranges)
    raw, base = _aligned(total)
    dsts, o = [], base
    for i, (_, n) in enumerate(ranges):
        dsts.append(o + (align_skew or {}).get(i, 0))
        o += (n + 127) // 64 * 64 + 64
    ecs = cl.batch_get_device_range(keys, [raw.ctypes.data + d for d in dsts], [a for a, _ in ranges], [n for _, n in ranges], 0)
    return ecs, raw, dsts


def _check(raw, dsts, blobs, ranges, ok):
    want = np.full_like(raw, GUARD)
    for d, b, (a, n), good in zip(dsts, blobs, ranges, ok):
        if good:
            want[d:d + n] = b[a:a + n]
    assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]


def test_ranges_inside_one_stripe_across_stripe_edges_and_over_all_stripes(bb):
    with LocalCluster(cluster_id="rngcpu", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        sh = Shards(c, cl)
        size = 3 * MiB + 12345
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
            key = f"r/{algo}"
            assert cl.batch_put_device([key], [blob.ctypes.data], [size], _cfg(bb, 1, 4, algo), 0) == [bb.ErrorCode.OK]
            (lay,) = sh.layout(key)
            assert len(lay) == 4, [s.length for _, s in lay]
            e1, e2 = lay[1][0], lay[2][0]  # stripe edges
            ranges = [(5, 1000),                       # inside the first stripe
                      (e1 + 17, lay[1][1].length - 40),  # inside the second stripe
                      (e1 - 3, 7),                     # across a stripe edge
                      (e1 - 100, e2 - e1 + 200),      # over two edges
                      (0, size),                       # the whole object
                      (1, size - 2),                   # every stripe, trimmed at both ends
                      (size - 1, 1),                   # the last byte
                      (e2, 0)]                         # empty
            keys = [key] * len(ranges)
            ecs, raw, dsts = _get_ranges(cl, keys, ranges)
            assert ecs == [bb.ErrorCode.OK] * len(ranges), (algo, ecs)
            _check(raw, dsts, [blob] * len(ranges), ranges, [True] * len(ranges))
        assert _counter(cl, "device_get_range_total") == 4 * 8
        assert _counter(cl, "device_get_range_bytes_total") > 0


def test_range_errors_fail_alone(bb):
    with LocalCluster(cluster_id="rngerr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 100000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["e"], [blob.ctypes.data], [size], _cfg(bb, 1, 2), 0) == [bb.ErrorCode.OK]
        ranges = [(10, 50), (size - 10, 11), (size + 1, 0), (2**64 - 8, 16), (40, 60), (0, 0), (size, 0)]
        keys = ["e", "e", "e", "e", "missing", "e", "e"]
        ecs, raw, dsts = _get_ranges(cl, keys, ranges)
        E = bb.ErrorCode
        assert ecs == [E.OK, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.OBJECT_NOT_FOUND, E.OK, E.OK], ecs
        _check(raw, dsts, [blob] * len(ranges), ranges, [e == E.OK for e in ecs])


def test_a_corrupt_shard_outside_the_range_is_not_read(bb):
    with LocalCluster(cluster_id="rngnon", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        sh = Shards(c, cl)
        size = 4 * MiB  # four 1 MiB stripes: every stripe start is 16-byte aligned, so the transport path is taken
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["n"], [blob.ctypes.data], [size], _cfg(bb, 2, 4), 0) == [bb.ErrorCode.OK]
        lay = sh.layout("n")
        for copy in lay:  # stripe 3 is corrupt in every copy
            sh.flip(copy[3][1], 9)
        mm, fo = _counter(cl, "checksum_mismatch_total"), _counter(cl, "replica_failover_total")
        # stripe 1 and the head of stripe 2, at a 16-byte aligned offset (the transport's path) and at an odd one, whose
        # virtual base is misaligned (the host-staged path): neither reads stripe 3
        for skew in (16 - lay[0][1][0] % 16, 3):
            r = (lay[0][1][0] + skew, lay[0][2][0] - lay[0][1][0])
            ecs, raw, dsts = _get_ranges(cl, ["n"], [r])
            assert ecs == [bb.ErrorCode.OK], skew
            _check(raw, dsts, [blob], [r], [True])
        assert _counter(cl, "checksum_mismatch_total") == mm and _counter(cl, "replica_failover_total") == fo
        # a range that reaches into stripe 3 fails on every copy
        ecs, _, _ = _get_ranges(cl, ["n"], [(lay[0][3][0] - 5, 10)])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]


def test_a_corrupt_byte_outside_the_window_of_an_overlapping_shard_fails_over(bb):
    with LocalCluster(cluster_id="rngfo", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        sh = Shards(c, cl)
        size = 2 * MiB + 5
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["f"], [blob.ctypes.data], [size], _cfg(bb, 2, 2), 0) == [bb.ErrorCode.OK]
        lay = sh.layout("f")
        r = (100, 1000)  # inside stripe 0; the flips below are far outside it
        mm = _counter(cl, "checksum_mismatch_total")
        for c_ in range(2):  # one copy at a time is corrupt: exactly one of the two gets starts on the corrupt one
            pos = lay[c_][0][1].length - 3
            sh.flip(lay[c_][0][1], pos)
            ecs, raw, dsts = _get_ranges(cl, ["f"], [r])
            assert ecs == [bb.ErrorCode.OK]
            _check(raw, dsts, [blob], [r], [True])
            sh.flip(lay[c_][0][1], pos)  # restore
        assert _counter(cl, "checksum_mismatch_total") == mm + 1
        # both copies corrupt outside the window: the range fails, after one placement refresh that re-reads the same range
        for copy in lay:
            sh.flip(copy[0][1], 7)
        ref = _counter(cl, "get_placement_refresh_total")
        ecs, raw, _ = _get_ranges(cl, ["f"], [r])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1


def test_unaligned_virtual_bases_are_staged_and_their_neighbours_are_not(bb):
    with LocalCluster(cluster_id="rngal", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 300000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["a"], [blob.ctypes.data], [size], _cfg(bb, 1, 1), 0) == [bb.ErrorCode.OK]
        # a striped object whose second stripe starts at an address that is not a multiple of 16
        striped = np.frombuffer(os.urandom(size + 3), dtype=np.uint8).copy()
        assert cl.batch_put_device(["b"], [striped.ctypes.data], [striped.size], _cfg(bb, 1, 2), 0) == [bb.ErrorCode.OK]
        (lay,) = Shards(c, cl).layout("b")
        e1 = lay[1][0]
        assert len(lay) == 2 and e1 % 16, [o for o, _ in lay]
        # (ptr - offset) % 16: 0, 0, 3, 0 -- only the third is staged.  The fifth, inside the second stripe, is aligned at
        # that stripe's start but not at the first stripe's: a range checks every shard of every copy, so it is staged too.
        ranges = [(16, 5000), (7, 100), (20, 4000), (1, 33), (e1 + 17, 1000)]
        skew = {0: 0, 1: 7, 2: 7, 3: 1, 4: 1}
        staged = _counter(cl, "device_get_host_staged_total")
        ecs, raw, dsts = _get_ranges(cl, ["a"] * 4 + ["b"], ranges, skew)
        assert ecs == [bb.ErrorCode.OK] * 5
        _check(raw, dsts, [blob] * 4 + [striped], ranges, [True] * 5)
        assert _counter(cl, "device_get_host_staged_total") == staged + 2


def test_range_gets_survive_concurrent_migration(bb):
    """Readers of byte ranges racing with compaction, tier moves and re-puts get the right bytes or a clean not-found:
    the placement refresh re-reads the same ranges."""
    with LocalCluster(cluster_id="rngmig", n_workers=1, pool_bytes=24 * MiB) as c:
        c.keystone.install_data_server_mover()
        c.add_worker("worker-cxl", "node-0", [("cxl-0", bb.StorageClass.CXL_MEMORY, 64 * MiB, "")])
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1, 1)
        names = [f"o{i}" for i in range(12)]
        blobs = {k: np.frombuffer(os.urandom(MiB // 2 + 4096 * i), dtype=np.uint8).copy() for i, k in enumerate(names)}
        for k, v in blobs.items():
            assert cl.batch_put_device([k], [v.ctypes.data], [v.size], cfg, 0) == [bb.ErrorCode.OK]
        stop = threading.Event()
        errors, reads = [], [0]

        def reader(seed):
            rc = make_client(bb, c)
            rng = random.Random(seed)
            while not stop.is_set():
                ks = rng.sample(names, 3)
                rs = []
                for k in ks:
                    a = rng.randrange(blobs[k].size)
                    rs.append((a, rng.randrange(blobs[k].size - a + 1)))
                outs = [np.zeros(n, dtype=np.uint8) for _, n in rs]
                ecs = rc.batch_get_device_range(ks, [o.ctypes.data for o in outs], [a for a, _ in rs], [n for _, n in rs], 0)
                for k, (a, n), o, ec in zip(ks, rs, outs, ecs):
                    if ec == bb.ErrorCode.OK:
                        if not np.array_equal(o, blobs[k][a:a + n]):
                            errors.append((k, "wrong bytes"))
                    elif ec not in (bb.ErrorCode.OBJECT_NOT_FOUND, bb.ErrorCode.OBJECT_NOT_READY):
                        errors.append((k, str(ec)))
                reads[0] += 1

        ts = [threading.Thread(target=reader, args=(s,)) for s in range(3)]
        [t.start() for t in ts]
        api = cl.keystone()
        rng = random.Random(11)
        moves, t_end = 0, time.time() + 2.0
        while time.time() < t_end:
            k = rng.choice(names)
            assert cl.remove(k) == bb.ErrorCode.OK
            moves += api.compact_pool("pool-0", 4)
            assert cl.batch_put_device([k], [blobs[k].ctypes.data], [blobs[k].size], cfg, 0) == [bb.ErrorCode.OK]
            k2 = rng.choice([x for x in names if x != k])
            tier = cl.get_workers(k2)[0].shards[0].storage_class
            assert cl.migrate(k2, bb.StorageClass.CXL_MEMORY if tier == bb.StorageClass.RAM_CPU else bb.StorageClass.RAM_CPU) == bb.ErrorCode.OK
        stop.set()
        [t.join() for t in ts]
        assert not errors, errors[:5]
        assert reads[0] > 30 and moves > 0
