"""Strided device puts (batch_put_device_strided) on CPU: the HostLoopbackTransport stands in for the GPU fabric, so the
client's strided put logic -- validation before any allocation, the source rows in shard coordinates, replica fan-out,
the host-staged path with its row compaction -- runs in the CPU suite.  The loopback transport keeps the fabric's
contract: each shard is written as the compaction of its rows, so the stored object and its recorded digests are those
of a contiguous put of the compacted bytes.  The rule itself (SourceRows, common/store_window.h) is checked against a
numpy model."""
import os
import random

import numpy as np
import pytest

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
KiB = 1 << 10


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


def compact(src, width, pitch, rows):
    """The object a strided put stores: rows[r] = src[r * pitch, + width), back to back."""
    return b"".join(bytes(src[r * pitch:r * pitch + width]) for r in range(rows))


class Sources:
    """Random source buffers at a chosen skew from a 64-byte boundary; kept alive for the test."""

    def __init__(self):
        self.keep = []

    def __call__(self, extent, skew=0):
        raw = np.frombuffer(os.urandom(extent + 128), dtype=np.uint8).copy()
        self.keep.append(raw)
        o = (-raw.ctypes.data) % 64 + skew
        return raw[o:o + extent], raw.ctypes.data + o


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.get_workers(key)]


def _put_and_check(bb, cl, cfg, pats, src_of, tag, staged=None):
    """Strided puts of pats = [(width, pitch, rows, skew)], each checked against the numpy compaction (read back with
    batch_get) and against a contiguous put of the compacted bytes (every copy's shard checksums).  `staged`: how many
    of the strided puts must have been staged through the host."""
    keys, ptrs, srcs = [], [], []
    for j, (w, p, r, skew) in enumerate(pats):
        src, ptr = src_of((r - 1) * p + w if r else 0, skew)
        keys.append(f"{tag}/{j}"), ptrs.append(ptr), srcs.append(src)
    n_staged = _counter(cl, "device_put_host_staged_total")
    ecs = cl.batch_put_device_strided(keys, ptrs, [p[0] for p in pats], [p[1] for p in pats], [p[2] for p in pats], cfg, 0)
    assert ecs == [bb.ErrorCode.OK] * len(pats), (tag, ecs)
    if staged is not None:
        assert _counter(cl, "device_put_host_staged_total") == n_staged + staged
    want = [compact(s, w, p, r) for s, (w, p, r, _) in zip(srcs, pats)]
    for (ec, blob), wb, key in zip(cl.batch_get(keys), want, keys):
        assert ec == bb.ErrorCode.OK, key
        assert bytes(blob) == wb, key
    dense = [np.frombuffer(wb, dtype=np.uint8).copy() for wb in want]
    ckeys = [k + "/c" for k in keys]
    assert cl.batch_put_device(ckeys, [d.ctypes.data for d in dense], [d.size for d in dense], cfg, 0) == [bb.ErrorCode.OK] * len(pats)
    for k, ck in zip(keys, ckeys):
        got, ref = _sums(cl, k), _sums(cl, ck)
        assert len(got) == len(ref) == cfg.replication_factor
        assert all(g == ref[0] for g in got) and all(r == ref[0] for r in ref), (k, got, ref)
    return srcs


def test_source_rows_rule_matches_numpy(bb):
    S = bb.SourceRows
    E = bb.ErrorCode
    assert S.from_rows(17, 16, 2)[0] == E.INVALID_ARGUMENT
    assert S.from_rows(17, 16, 1)[0] == E.OK and not S.from_rows(17, 16, 1)[1].strided()
    assert S.from_rows(2**63, 2**63, 2)[0] == E.VALUE_OUT_OF_RANGE      # rows * width
    assert S.from_rows(8, 2**63, 3)[0] == E.VALUE_OUT_OF_RANGE          # (rows - 1) * pitch
    for w, p, r in ((0, 16, 5), (5, 16, 0), (16, 16, 9)):
        ec, rows, size, extent = S.from_rows(w, p, r)
        assert ec == E.OK and not rows.strided() and size == w * r
    ec, rows, size, extent = S.from_rows(10, 48, 7)
    assert ec == E.OK and (rows.pitch, rows.width, rows.phase) == (48, 10, 0) and size == 70 and extent == 6 * 48 + 10
    rng = random.Random(5)
    for _ in range(300):
        w = rng.randint(1, 70)
        p = w + rng.choice([0, 1, 16, 32, rng.randint(0, 90)])
        r = rng.randint(2, 12)
        ec, rows, size, extent = S.from_rows(w, p, r)
        assert ec == E.OK
        src = np.arange(extent, dtype=np.int64)
        idx = np.frombuffer(b"".join(src[k * p:k * p + w].tobytes() for k in range(r)), dtype=np.int64)  # source index of object byte
        assert idx.size == size
        off = rng.randint(0, size)
        sub, shift = rows.rebase(off)
        n = rng.randint(0, size - off)
        # the walk from the rebased origin reads exactly the model's source bytes
        got = np.full(n, -1, dtype=np.int64)
        for x, at, k in sub.runs(n):
            got[x:x + k] = shift + at + np.arange(k)
        assert np.array_equal(got, idx[off:off + n])
        assert sub.extent(n) == (got[-1] + 1 - shift if n else 0)
        # co-alignment: the source of every byte of the span congruent to its index mod 16
        for base in (0, 16 * rng.randint(0, 9) + rng.randint(0, 15)):
            if n:
                want = bool(np.all((base + idx[off:off + n] - np.arange(n)) % 16 == 0))
                assert sub.coaligned(base + shift, n) == want, (w, p, r, off, n, base)
    c = S()
    assert not c.strided() and c.rebase(77)[1] == 77
    assert c.runs(5) == [(0, 0, 5)] and c.coaligned(32, 5) and not c.coaligned(33, 5)


def test_strided_puts_match_compaction_and_contiguous_digests(bb):
    """Heads and tails, widths of 1 to 15 bytes, pitches below, at and above 16 KiB, one and four stripes (shard
    boundaries mid-row, so the shards' patterns start at phase != 0), for every algorithm."""
    with LocalCluster(cluster_id="sputcpu", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        src_of = Sources()
        n0 = _counter(cl, "device_put_strided_total")
        pats = [(w, 16 + w, 997, 0) for w in (1, 7, 15)]              # narrow rows, gap 16
        pats += [(100, 132, 3000, 0), (4000, 16 * KiB, 40, 0), (16 * KiB, 16 * KiB + 48, 9, 0),
                 (20000, 40000, 13, 0), (333, 333, 77, 0), (5000, 7, 1, 0)]  # width == pitch and one row: contiguous
        # over four stripes these two keep aligned shard starts that fall mid-row: their shards' patterns have phase != 0
        pats += [(64, 96, 1001, 0), (1088, 16 * KiB + 64, 41, 0)]
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            for stripes in (1, 4):
                _put_and_check(bb, cl, _cfg(bb, 1, stripes, algo), pats, src_of, f"{algo}/{stripes}",
                               staged=None if stripes == 4 else 0)
        assert _counter(cl, "device_put_strided_total") == n0 + 8 * len(pats)
        assert _counter(cl, "device_put_strided_bytes_total") > 0


@pytest.mark.parametrize("replicas", [2, 3])
def test_strided_puts_with_replicas(bb, replicas):
    with LocalCluster(cluster_id=f"sputrep{replicas}", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pats = [(48, 80, 5000, 0), (1000, 3000, 300, 0), (3, 19, 100, 0)]
        _put_and_check(bb, cl, _cfg(bb, replicas, 2), pats, Sources(), "r")


def test_misaligned_sources_are_staged(bb):
    """A source start that is not 16-byte aligned, or a row gap that is not a multiple of 16, is staged through the host
    (one copy of the extent, rows compacted there); the other items keep the transport."""
    with LocalCluster(cluster_id="sputal", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        pats = [(100, 132, 512, 0), (100, 132, 500, 5), (40, 75, 800, 0), (64, 96, 700, 0)]
        _put_and_check(bb, cl, _cfg(bb, 1, 2), pats, Sources(), "m", staged=2)


def test_strided_put_errors(bb):
    with LocalCluster(cluster_id="sputerr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        E = bb.ErrorCode
        src, ptr = Sources()(100000)
        cfg = _cfg(bb, 1, 1)
        pats = [(10, 50, 20),        # ok
                (101, 100, 2),       # width > pitch
                (2**62, 2**62, 8),   # rows * width overflows
                (8, 2**63, 3),       # (rows - 1) * pitch overflows
                (0, 100, 5),         # width 0: a zero-byte object
                (10, 100, 0)]        # no rows: a zero-byte object
        keys = [f"e{j}" for j in range(len(pats))]
        ecs = cl.batch_put_device_strided(keys, [ptr] * len(pats), [p[0] for p in pats], [p[1] for p in pats], [p[2] for p in pats], cfg, 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.OK, E.OK], ecs
        # nothing was allocated for the refused items
        assert [e for e, _ in cl.batch_get(keys[1:4])] == [E.OBJECT_NOT_FOUND] * 3
        got = cl.batch_get([keys[0], keys[4], keys[5]])
        assert bytes(got[0][1]) == compact(src, 10, 50, 20)
        assert [bytes(b) for _, b in got[1:]] == [b"", b""]
        ref = cl.batch_put_device(["z"], [ptr], [0], cfg, 0)
        assert ref == [E.OK]
        # lengths that differ fail the whole batch
        assert cl.batch_put_device_strided(["x", "y"], [ptr], [1, 1], [1, 1], [1, 1], cfg, 0) == [E.INVALID_PARAMETERS] * 2
        assert cl.batch_put_device_strided(["x"], [ptr], [1], [1, 2], [1], cfg, 0) == [E.INVALID_PARAMETERS]
