"""Strided device gets (batch_get_device_strided) on CPU: the HostLoopbackTransport stands in for the GPU fabric, so the
client's strided logic -- the shards that hold a stored byte and no others, the row pattern in shard coordinates, replica
choice and fail-over, the host-staged path with its row compaction -- runs in the CPU suite.  The loopback transport keeps
the fabric's contract: a shard that is read is read whole and verified, only its bytes of the rows are stored."""
import os

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


def rows_of(blob, offset, width, pitch, rows):
    """The dense result of a strided get: rows[r] = blob[offset + r * pitch, + width)."""
    return b"".join(bytes(blob[offset + r * pitch:offset + r * pitch + width]) for r in range(rows))


def _get_strided(cl, keys, pats, skew=None):
    """Strided gets into one guard-filled host buffer, every result at its own region congruent to offset mod 16 (so the
    virtual base is aligned) plus skew[i]; returns (error codes, buffer, region offsets)."""
    total = sum(w * r + 256 for _, w, _, r in pats)
    raw = np.full(total + 256, GUARD, dtype=np.uint8)
    base = (-raw.ctypes.data) % 64 + 64
    dsts, o = [], base
    for i, (off, w, _, r) in enumerate(pats):
        dsts.append(o + off % 16 + (skew or {}).get(i, 0))
        o += (w * r + 127) // 64 * 64 + 64
    ecs = cl.batch_get_device_strided(keys, [raw.ctypes.data + d for d in dsts], [p[0] for p in pats], [p[1] for p in pats],
                                      [p[2] for p in pats], [p[3] for p in pats], 0)
    return ecs, raw, dsts


def _check(raw, dsts, blobs, pats, ok):
    want = np.full_like(raw, GUARD)
    for d, b, p, good in zip(dsts, blobs, pats, ok):
        if good:
            dense = np.frombuffer(rows_of(b, *p), dtype=np.uint8)
            want[d:d + dense.size] = dense
    assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]


def test_strided_rows_over_stripes_match_numpy(bb):
    """Patterns inside one stripe, rows that cross stripe edges, a pitch above the stripe size (shards in the column gaps
    are skipped), widths of 1, 15, 16, 17 bytes and width == pitch, for every algorithm."""
    with LocalCluster(cluster_id="strcpu", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        sh = Shards(c, cl)
        size = 3 * MiB + 12345
        n0 = _counter(cl, "device_get_strided_total")
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
            key = f"s/{algo}"
            assert cl.batch_put_device([key], [blob.ctypes.data], [size], _cfg(bb, 1, 4, algo), 0) == [bb.ErrorCode.OK]
            (lay,) = sh.layout(key)
            assert len(lay) == 4
            e1 = lay[1][0]
            pats = [(5, 1, 17, 1000),                 # (offset, width, pitch, rows)
                    (100, 15, 31, 3000),
                    (e1 - 4000, 16, 48, 200),         # rows across a stripe edge
                    (e1 - 3, 17, 33, 500),            # a row split by the stripe edge
                    (1, 100, 100, 50),                # width == pitch: one range
                    (7, 300, 1100 * 1024, 3),         # pitch above the stripe size
                    (0, 4096, 8192, size // 8192),    # every stripe
                    (size - 20, 20, 64, 1)]           # one row: a range
            keys = [key] * len(pats)
            ecs, raw, dsts = _get_strided(cl, keys, pats)
            assert ecs == [bb.ErrorCode.OK] * len(pats), (algo, ecs)
            _check(raw, dsts, [blob] * len(pats), pats, [True] * len(pats))
        assert _counter(cl, "device_get_strided_total") == n0 + 4 * 8
        assert _counter(cl, "device_get_strided_bytes_total") > 0


def test_strided_errors_fail_alone(bb):
    with LocalCluster(cluster_id="strerr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 100000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["e"], [blob.ctypes.data], [size], _cfg(bb, 1, 2), 0) == [bb.ErrorCode.OK]
        pats = [(10, 50, 100, 20),          # ok
                (10, 101, 100, 2),          # width > pitch
                (10, 50, 100, 1001),        # the last row passes the end
                (size - 50, 50, 100, 2),    # the second row passes the end
                (0, 8, 2**63, 3),           # (rows - 1) * pitch overflows
                (40, 60, 200, 4),           # missing key
                (0, 0, 100, 5),             # width 0
                (5, 10, 100, 0),            # no rows
                (10, 101, 100, 1),          # one row may be wider than the pitch: a range
                (size - 7, 7, 16, 1)]       # the last bytes
        keys = ["e"] * 5 + ["missing"] + ["e"] * 4
        ecs, raw, dsts = _get_strided(cl, keys, pats)
        E = bb.ErrorCode
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.OBJECT_NOT_FOUND,
                       E.OK, E.OK, E.OK, E.OK], ecs
        _check(raw, dsts, [blob] * len(pats), pats, [e == E.OK for e in ecs])


def test_a_shard_in_a_column_gap_is_not_read(bb):
    """Rows 2 MiB apart over four 1 MiB stripes: stripe 1 lies wholly between rows 0 and 1, stripe 3 past the last row.
    Both are corrupt in every copy and the get still verifies without a mismatch."""
    with LocalCluster(cluster_id="strgap", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        sh = Shards(c, cl)
        size = 4 * MiB
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["g"], [blob.ctypes.data], [size], _cfg(bb, 2, 4), 0) == [bb.ErrorCode.OK]
        lay = sh.layout("g")
        assert [o for o, _ in lay[0]] == [0, MiB, 2 * MiB, 3 * MiB]
        for copy in lay:
            sh.flip(copy[1][1], 9)
            sh.flip(copy[3][1], 9)
        mm = _counter(cl, "checksum_mismatch_total")
        pat = (MiB - 32, 32, 2 * MiB, 2)  # row 0 ends stripe 0, row 1 ends stripe 2
        for skew in (0, 3):  # the fused path and the host-staged one
            ecs, raw, dsts = _get_strided(cl, ["g"], [pat], {0: skew})
            assert ecs == [bb.ErrorCode.OK], skew
            _check(raw, dsts, [blob], [pat], [True])
        assert _counter(cl, "checksum_mismatch_total") == mm
        # a pattern whose rows reach into stripe 1 fails on every copy
        ecs, _, _ = _get_strided(cl, ["g"], [(MiB - 32, 48, 2 * MiB, 2)])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]


def test_a_corrupt_byte_in_a_gap_of_a_read_shard_fails_over(bb):
    with LocalCluster(cluster_id="strfo", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        sh = Shards(c, cl)
        size = 2 * MiB + 5
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["f"], [blob.ctypes.data], [size], _cfg(bb, 2, 2), 0) == [bb.ErrorCode.OK]
        lay = sh.layout("f")
        pat = (100, 64, 1024, 900)  # stripe 0 only; byte 100 + 64 + 8 lies in the gap after row 0
        mm = _counter(cl, "checksum_mismatch_total")
        for c_ in range(2):  # one copy at a time is corrupt: exactly one of the two gets starts on it
            sh.flip(lay[c_][0][1], 172)
            ecs, raw, dsts = _get_strided(cl, ["f"], [pat])
            assert ecs == [bb.ErrorCode.OK]
            _check(raw, dsts, [blob], [pat], [True])
            sh.flip(lay[c_][0][1], 172)
        assert _counter(cl, "checksum_mismatch_total") == mm + 1
        for copy in lay:
            sh.flip(copy[0][1], 172)
        ref = _counter(cl, "get_placement_refresh_total")
        ecs, _, _ = _get_strided(cl, ["f"], [pat])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        assert _counter(cl, "get_placement_refresh_total") == ref + 1


def test_misaligned_items_are_staged_and_their_neighbours_are_not(bb):
    """(ptr - offset) % 16 != 0 or a row gap that is not a multiple of 16, even where every shard read holds one row:
    staged through the host (rows compacted there); the other items of the batch take the transport."""
    with LocalCluster(cluster_id="stral", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 300000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["a"], [blob.ctypes.data], [size], _cfg(bb, 1, 1), 0) == [bb.ErrorCode.OK]
        big = np.frombuffer(os.urandom(2 * MiB), dtype=np.uint8).copy()
        assert cl.batch_put_device(["b"], [big.ctypes.data], [big.size], _cfg(bb, 1, 2), 0) == [bb.ErrorCode.OK]
        (lay,) = Shards(c, cl).layout("b")
        assert [o for o, _ in lay] == [0, MiB]
        # item 2: misaligned base; item 3: gap 35; item 4: gap MiB - 24 with one row in each stripe it reads
        pats = [(16, 100, 132, 50), (7, 33, 49, 80), (20, 40, 72, 30), (3, 40, 75, 30), (16, 32, MiB + 8, 2)]
        skew = {2: 5}
        staged = _counter(cl, "device_get_host_staged_total")
        ecs, raw, dsts = _get_strided(cl, ["a"] * 4 + ["b"], pats, skew)
        assert ecs == [bb.ErrorCode.OK] * 5
        _check(raw, dsts, [blob] * 4 + [big], pats, [True] * 5)
        assert _counter(cl, "device_get_host_staged_total") == staged + 3


def test_one_row_counts_as_a_range(bb):
    with LocalCluster(cluster_id="strone", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 200000
        blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
        assert cl.batch_put_device(["o"], [blob.ctypes.data], [size], _cfg(bb, 1, 2), 0) == [bb.ErrorCode.OK]
        ecs, raw, dsts = _get_strided(cl, ["o"], [(99000, 3000, 7, 1)])
        assert ecs == [bb.ErrorCode.OK]
        _check(raw, dsts, [blob], [(99000, 3000, 7, 1)], [True])
        assert _counter(cl, "device_get_strided_bytes_total") == 3000
