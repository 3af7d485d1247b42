"""Element-range gets of MXFP8-packed tensors (batch_get_device_fp8_range) on CPU: the HostLoopbackTransport stands in for
the GPU fabric, so the client's range logic -- per-item errors, the per-item alignment rule of the virtual base, replica
fail-over, the placement refresh -- runs in the CPU suite.  The loopback transport keeps the fused kernel's contract: the
whole packed object is read and verified, only the window is unpacked and stored."""
import random
import threading
import time

import numpy as np

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
T = 16384
GUARD = 0xA5A5


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


def _cfg(bb, replicas):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])


def _bf16(rng, n):
    """Truncated bf16 bit patterns of normal samples (uint16)."""
    return ((rng.standard_normal(n) * 3).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)


def _unpacked(bb, b):
    return np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(b), b.size), dtype=np.uint16)


def _flip(c, cl, sh, pos):
    pools = {p.id: p for p in cl.keystone().get_memory_pools()}
    w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
    off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
    b = w.backend(sh.pool_id)
    b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))


def _get(cl, keys, ns, ranges, skew=None):
    """Element-range gets into one guard-filled uint16 host buffer.  Range i lands at a region whose virtual base
    (region - 2 * lo bytes) is 16-byte aligned, moved by skew[i] elements; returns (error codes, buffer, regions)."""
    total = sum(c + 32 for _, c in ranges) + 64
    raw = np.full(total, GUARD, dtype=np.uint16)
    o = ((-raw.ctypes.data) % 16) // 2 + 16  # a 16-byte aligned element with guards before it
    regions = []
    for i, (lo, c) in enumerate(ranges):
        r = o + lo % 8 + (skew or {}).get(i, 0)
        regions.append(r)
        o = (r + c + 7) // 8 * 8 + 16
    ecs = cl.batch_get_device_fp8_range(keys, [raw.ctypes.data + 2 * r for r in regions], ns, [lo for lo, _ in ranges],
                                        [c for _, c in ranges], 0)
    return ecs, raw, regions


def _check(raw, regions, refs, ranges, ok):
    """Every region holds its slice of the reference (when ok) and every other element is still a guard."""
    want = np.full_like(raw, GUARD)
    for r, ref, (lo, c), good in zip(regions, refs, ranges, ok):
        if good:
            want[r:r + c] = ref[lo:lo + c]
    assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]


def _ranges(n):
    """Whole, one element, inside a tile, across a tile edge, in the tail, lo % 8 in {0, 1, 7}, empty."""
    cand = [(0, n), (5, 1), (100, 300), (T - 3, 10), (n - 40, 40), (n - 1, 1), (8, n - 16), (1, n - 9), (7, 33), (n // 2, 0)]
    return [(lo, c) for lo, c in cand if 0 <= lo and lo + c <= n]


def test_fp8_ranges_with_one_and_two_copies(bb):
    with LocalCluster(cluster_id="fp8rng", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(1)
        ns = [32, T + 96, 3 * T + 96]
        bfs = [_bf16(rng, n) for n in ns]
        refs = [_unpacked(bb, b) for b in bfs]
        n0, b0 = _counter(cl, "device_get_fp8_range_total"), _counter(cl, "device_get_fp8_range_bytes_total")
        want_n = want_b = 0
        for rep in (1, 2):
            keys = [f"r{rep}/{n}" for n in ns]
            assert cl.batch_put_device_fp8(keys, [b.ctypes.data for b in bfs], ns, _cfg(bb, rep), 0) == [bb.ErrorCode.OK] * 3
            assert all(len(cl.get_workers(k)) == rep for k in keys)
            ks, nn, rr, rf = [], [], [], []
            for k, n, ref in zip(keys, ns, refs):
                for r in _ranges(n):
                    ks.append(k), nn.append(n), rr.append(r), rf.append(ref)
            ecs, raw, regions = _get(cl, ks, nn, rr)
            assert ecs == [bb.ErrorCode.OK] * len(ks), ecs
            _check(raw, regions, rf, rr, [True] * len(ks))
            want_n += len(ks)
            want_b += 2 * sum(c for _, c in rr)
        assert _counter(cl, "device_get_fp8_range_total") == n0 + want_n
        assert _counter(cl, "device_get_fp8_range_bytes_total") == b0 + want_b


def test_fp8_range_errors_and_misaligned_bases_fail_alone(bb):
    with LocalCluster(cluster_id="fp8rngerr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(2)
        n = 2 * T + 64
        b = _bf16(rng, n)
        ref = _unpacked(bb, b)
        assert cl.batch_put_device_fp8(["e"], [b.ctypes.data], [n], _cfg(bb, 1), 0) == [bb.ErrorCode.OK]
        # a packed object striped over two workers cannot take the fused kernel
        packed = np.frombuffer(bb.mxfp8_pack_ref(b), dtype=np.uint8).copy()
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        assert cl.batch_put_device(["s"], [packed.ctypes.data], [packed.size], striped, 0) == [bb.ErrorCode.OK]
        assert len(cl.get_workers("s")[0].shards) == 2
        E = bb.ErrorCode
        cases = [("e", (10, 50), 0, E.OK),
                 ("e", (n - 10, 11), 0, E.VALUE_OUT_OF_RANGE),
                 ("e", (n + 1, 0), 0, E.VALUE_OUT_OF_RANGE),
                 ("e", (2**64 - 8, 16), 0, E.VALUE_OUT_OF_RANGE),
                 ("missing", (0, 32), 0, E.OBJECT_NOT_FOUND),
                 ("e", (40, 0), 0, E.OK),
                 ("e", (T - 5, 9), 1, E.NOT_IMPLEMENTED),   # virtual base 2 bytes off
                 ("e", (3, 100), 4, E.NOT_IMPLEMENTED),     # 8 bytes off
                 ("s", (0, 64), 0, E.NOT_IMPLEMENTED),      # striped
                 ("e", (n - 33, 33), 0, E.OK)]
        skew = {i: s for i, (_, _, s, _) in enumerate(cases)}
        ranges = [r for _, r, _, _ in cases]
        ecs, raw, regions = _get(cl, [k for k, _, _, _ in cases], [n] * len(cases), ranges, skew)
        assert ecs == [e for _, _, _, e in cases], ecs
        _check(raw, regions, [ref] * len(cases), ranges, [e == E.OK for e in ecs])
        # the whole-object call keeps its own rules
        out = np.zeros(n, dtype=np.uint16)
        assert cl.batch_get_device_fp8(["e"], [out.ctypes.data], [n], 0) == [E.OK] and np.array_equal(out, ref)


def test_fp8_range_fails_over_from_a_copy_corrupt_outside_the_window(bb):
    with LocalCluster(cluster_id="fp8rngfo", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(3)
        n = 3 * T + 96
        b = _bf16(rng, n)
        ref = _unpacked(bb, b)
        assert cl.batch_put_device_fp8(["f"], [b.ctypes.data], [n], _cfg(bb, 2), 0) == [bb.ErrorCode.OK]
        copies = [cp.shards[0] for cp in cl.get_workers("f")]
        r = (T + 100, 200)  # the flips below are far outside it: payload byte n - 5, the last scale byte
        for pos in (n - 5, n + n // 32 - 1):
            fo = _counter(cl, "replica_failover_total")
            for sh in copies:  # one copy at a time is corrupt: exactly one of the two gets starts on it
                _flip(c, cl, sh, pos)
                ecs, raw, regions = _get(cl, ["f"], [n], [r])
                assert ecs == [bb.ErrorCode.OK]
                _check(raw, regions, [ref], [r], [True])
                _flip(c, cl, sh, pos)  # restore
            assert _counter(cl, "replica_failover_total") == fo + 1, pos
        # every copy corrupt outside the window: the range fails after one placement refresh that re-reads the same range,
        # and no byte outside the window is written on any attempt
        for sh in copies:
            _flip(c, cl, sh, 7)
        ref_n = _counter(cl, "get_placement_refresh_total")
        ecs, raw, regions = _get(cl, ["f", "f"], [n, n], [r, (0, 0)])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH, bb.ErrorCode.OK]
        assert _counter(cl, "get_placement_refresh_total") == ref_n + 1
        outside = np.ones(raw.size, dtype=bool)
        outside[regions[0]:regions[0] + r[1]] = False
        assert bool((raw[outside] == GUARD).all())


def test_fp8_range_gets_survive_concurrent_compaction_and_migration(bb):
    """Readers of element ranges racing with compaction, tier moves and re-puts get the right values or a clean
    not-found: the placement refresh re-reads the same ranges."""
    with LocalCluster(cluster_id="fp8rngmig", n_workers=1, pool_bytes=24 * MiB) as c:
        c.keystone.install_data_server_mover()
        c.add_worker("worker-cxl", "node-0", [("cxl-0", bb.StorageClass.CXL_MEMORY, 64 * MiB, "")])
        cl = make_client(bb, c)
        cfg = _cfg(bb, 1)
        rng = np.random.default_rng(5)
        names = [f"t{i}" for i in range(10)]
        ns = {k: T * (8 + i) + 32 * i for i, k in enumerate(names)}
        bf = {k: _bf16(rng, ns[k]) for k in names}
        want = {k: _unpacked(bb, bf[k]) for k in names}
        for k in names:
            assert cl.batch_put_device_fp8([k], [bf[k].ctypes.data], [ns[k]], cfg, 0) == [bb.ErrorCode.OK]
        stop = threading.Event()
        errors, reads = [], [0]

        def reader(seed):
            rc = make_client(bb, c)
            r = random.Random(seed)
            while not stop.is_set():
                ks = r.sample(names, 3)
                rs = []
                for k in ks:
                    lo = r.randrange(ns[k])
                    rs.append((lo, r.randrange(ns[k] - lo + 1)))
                outs = [np.zeros(cnt + 8, dtype=np.uint16) for _, cnt in rs]
                # element lo % 8 of a 16-byte aligned buffer: the virtual base is aligned
                ptrs = [o.ctypes.data + ((-o.ctypes.data) % 16) + 2 * (lo % 8) for o, (lo, _) in zip(outs, rs)]
                ecs = rc.batch_get_device_fp8_range(ks, ptrs, [ns[k] for k in ks], [lo for lo, _ in rs], [cnt for _, cnt in rs], 0)
                for k, (lo, cnt), o, p, ec in zip(ks, rs, outs, ptrs, ecs):
                    if ec == bb.ErrorCode.OK:
                        s = (p - o.ctypes.data) // 2
                        if not np.array_equal(o[s:s + cnt], want[k][lo:lo + cnt]):
                            errors.append((k, "wrong values"))
                    elif ec not in (bb.ErrorCode.OBJECT_NOT_FOUND, bb.ErrorCode.OBJECT_NOT_READY):
                        errors.append((k, str(ec)))
                reads[0] += 1

        ts = [threading.Thread(target=reader, args=(s,)) for s in range(3)]
        [t.start() for t in ts]
        api = cl.keystone()
        r = random.Random(17)
        moves, t_end = 0, time.time() + 2.0
        while time.time() < t_end:
            k = r.choice(names)
            assert cl.remove(k) == bb.ErrorCode.OK
            moves += api.compact_pool("pool-0", 4)
            assert cl.batch_put_device_fp8([k], [bf[k].ctypes.data], [ns[k]], cfg, 0) == [bb.ErrorCode.OK]
            k2 = r.choice([x for x in names if x != k])
            tier = cl.get_workers(k2)[0].shards[0].storage_class
            assert cl.migrate(k2, bb.StorageClass.CXL_MEMORY if tier == bb.StorageClass.RAM_CPU else bb.StorageClass.RAM_CPU) == bb.ErrorCode.OK
        stop.set()
        [t.join() for t in ts]
        assert not errors, errors[:5]
        assert reads[0] > 30 and moves > 0
