"""Strided gets of MXFP8-packed tensors (batch_get_device_fp8_strided) on CPU: the HostLoopbackTransport stands in for the
GPU fabric, so the client's strided logic -- the row pattern of the fused unpack, per-item errors, the per-item alignment
rule, replica fail-over, the placement refresh -- runs in the CPU suite.  The loopback transport keeps the fused kernel's
contract: the whole packed object is read and verified, only the rows are unpacked and stored, densely."""
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


def rows_of(ref, offset, width, pitch, rows):
    """The dense result of a strided get: row r = ref[offset + r * pitch, + width)."""
    if rows == 0 or width == 0:
        return ref[:0]
    return np.concatenate([ref[offset + r * pitch:offset + r * pitch + width] for r in range(rows)])


def _get(cl, keys, ns, pats, skew=None):
    """Strided gets into one guard-filled uint16 host buffer.  Pattern i = (offset, width, pitch, rows) lands at a region
    whose virtual base (region - 2 * offset bytes) is 16-byte aligned, moved by skew[i] elements; returns (error codes,
    buffer, regions)."""
    total = sum(w * r + 32 for _, w, _, r in pats) + 64
    raw = np.full(total, GUARD, dtype=np.uint16)
    o = ((-raw.ctypes.data) % 16) // 2 + 16  # a 16-byte aligned element with guards before it
    regions = []
    for i, (off, w, _, r) in enumerate(pats):
        reg = o + off % 8 + (skew or {}).get(i, 0)
        regions.append(reg)
        o = (reg + w * r + 7) // 8 * 8 + 16
    ecs = cl.batch_get_device_fp8_strided(keys, [raw.ctypes.data + 2 * r for r in regions], ns, [p[0] for p in pats],
                                          [p[1] for p in pats], [p[2] for p in pats], [p[3] for p in pats], 0)
    return ecs, raw, regions


def _check(raw, regions, refs, pats, ok):
    """Every region holds its rows of the reference (when ok) and every other element is still a guard."""
    want = np.full_like(raw, GUARD)
    for reg, ref, p, good in zip(regions, refs, pats, ok):
        if good:
            dense = rows_of(ref, *p)
            want[reg:reg + dense.size] = dense
    assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]


def _patterns(n):
    """(offset, width, pitch, rows): KV-head slices, 8 elements every 64, rows longer than a tile, offsets that are not a
    multiple of the pitch or of 8, width == pitch, one row, rows that end at the last element, no rows, zero width.
    Every gap is a multiple of 8 elements, so that every pattern takes the fused path."""
    cand = [(128, 128, 1024, n // 1024 - 1), (0, 8, 64, n // 64), (3, 16, 24, 100), (T - 8, T + 8, 3 * T, 1),
            (5, T + 40, T + 48, (n - 5) // (T + 48)), (7, 100, 100, (n - 7) // 100), (n - 96, 96, 1, 1),
            (n - 2 * 72 - 24, 24, 72, 3), (40, 0, 64, 9), (40, 16, 64, 0)]
    return [p for p in cand if p[3] == 0 or p[0] + (p[3] - 1) * p[2] + p[1] <= n]


def test_fp8_strided_with_one_and_two_copies(bb):
    with LocalCluster(cluster_id="fp8str", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(1)
        ns = [T + 96, 3 * T + 96, 4 * T]
        bfs = [_bf16(rng, n) for n in ns]
        refs = [_unpacked(bb, b) for b in bfs]
        n0, b0 = _counter(cl, "device_get_fp8_strided_total"), _counter(cl, "device_get_fp8_strided_bytes_total")
        want_n = want_b = 0
        for rep in (1, 2):
            keys = [f"r{rep}/{n}" for n in ns]
            assert cl.batch_put_device_fp8(keys, [b.ctypes.data for b in bfs], ns, _cfg(bb, rep), 0) == [bb.ErrorCode.OK] * 3
            assert all(len(cl.get_workers(k)) == rep for k in keys)
            ks, nn, pp, rf = [], [], [], []
            for k, n, ref in zip(keys, ns, refs):
                for p in _patterns(n):
                    ks.append(k), nn.append(n), pp.append(p), rf.append(ref)
            ecs, raw, regions = _get(cl, ks, nn, pp)
            assert ecs == [bb.ErrorCode.OK] * len(ks), ecs
            _check(raw, regions, rf, pp, [True] * len(ks))
            want_n += len(ks)
            want_b += 2 * sum(w * r for _, w, _, r in pp)
        assert _counter(cl, "device_get_fp8_strided_total") == n0 + want_n
        assert _counter(cl, "device_get_fp8_strided_bytes_total") == b0 + want_b


def test_fp8_strided_errors_and_misaligned_items_fail_alone(bb):
    with LocalCluster(cluster_id="fp8strerr", n_workers=2, pool_bytes=32 * MiB) as c:
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
        cases = [("e", (10, 52, 100, 20), 0, E.OK),
                 ("e", (10, 101, 100, 2), 0, E.INVALID_ARGUMENT),        # width > pitch
                 ("e", (10, 50, 100, n // 100 + 1), 0, E.VALUE_OUT_OF_RANGE),  # the last row passes the end
                 ("e", (n - 50, 50, 100, 2), 0, E.VALUE_OUT_OF_RANGE),   # the second row passes the end
                 ("e", (0, 8, 2**63, 3), 0, E.VALUE_OUT_OF_RANGE),        # (rows - 1) * pitch overflows
                 ("missing", (40, 60, 200, 4), 0, E.OBJECT_NOT_FOUND),
                 ("e", (0, 0, 100, 5), 0, E.OK),                          # width 0
                 ("e", (5, 10, 100, 0), 0, E.OK),                         # no rows
                 ("e", (10, 101, 100, 1), 0, E.OK),                       # one row may be wider than the pitch: a range
                 ("e", (3, 40, 72, 30), 1, E.NOT_IMPLEMENTED),            # virtual base 2 bytes off
                 ("e", (3, 40, 75, 30), 0, E.NOT_IMPLEMENTED),            # gap of 35 elements
                 ("e", (3, 40, 44, 30), 0, E.NOT_IMPLEMENTED),            # gap of 4 elements
                 ("s", (0, 64, 128, 4), 0, E.NOT_IMPLEMENTED),            # striped
                 ("e", (3, 40, 48, 30), 0, E.OK),                         # gap of 8 elements
                 ("e", (n - 40, 8, 16, 3), 0, E.OK)]                      # the last row ends the object
        skew = {i: s for i, (_, _, s, _) in enumerate(cases)}
        pats = [p for _, p, _, _ in cases]
        ecs, raw, regions = _get(cl, [k for k, _, _, _ in cases], [n] * len(cases), pats, skew)
        assert ecs == [e for _, _, _, e in cases], ecs
        _check(raw, regions, [ref] * len(cases), pats, [e == E.OK for e in ecs])
        # one row is the range get of the same elements
        ecs, raw, regions = _get(cl, ["e"], [n], [(T - 3, 300, 7, 1)])
        assert ecs == [E.OK]
        _check(raw, regions, [ref], [(T - 3, 300, 7, 1)], [True])
        assert cl.batch_get_device_fp8_strided(["e"], [0], [n], [0], [1], [1], [1, 2], 0) == [E.INVALID_PARAMETERS]


def test_fp8_strided_fails_over_from_a_copy_corrupt_in_a_gap(bb):
    with LocalCluster(cluster_id="fp8strfo", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(3)
        n = 3 * T + 96
        b = _bf16(rng, n)
        ref = _unpacked(bb, b)
        assert cl.batch_put_device_fp8(["f"], [b.ctypes.data], [n], _cfg(bb, 2), 0) == [bb.ErrorCode.OK]
        copies = [cp.shards[0] for cp in cl.get_workers("f")]
        p = (128, 128, 1024, 40)  # payload byte 300 lies in the gap after row 0; scale byte 20 covers elements 640..671
        for pos in (300, n + 20):
            fo = _counter(cl, "replica_failover_total")
            for sh in copies:  # one copy at a time is corrupt: exactly one of the two gets starts on it
                _flip(c, cl, sh, pos)
                ecs, raw, regions = _get(cl, ["f"], [n], [p])
                assert ecs == [bb.ErrorCode.OK]
                _check(raw, regions, [ref], [p], [True])
                _flip(c, cl, sh, pos)  # restore
            assert _counter(cl, "replica_failover_total") == fo + 1, pos
        # every copy corrupt in a gap: the get fails after one placement refresh that re-reads the same rows, and no
        # element outside the rows is written on any attempt
        for sh in copies:
            _flip(c, cl, sh, 300)
        ref_n = _counter(cl, "get_placement_refresh_total")
        ecs, raw, regions = _get(cl, ["f", "f"], [n, n], [p, (0, 16, 64, 0)])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH, bb.ErrorCode.OK]
        assert _counter(cl, "get_placement_refresh_total") == ref_n + 1
        outside = np.ones(raw.size, dtype=bool)
        outside[regions[0]:regions[0] + p[1] * p[3]] = False
        assert bool((raw[outside] == GUARD).all())
