"""Packed puts of sliced bf16 tensors (batch_put_device_fp8_strided) on CPU: the HostLoopbackTransport stands in for the GPU
fabric, so the client's logic -- validation before any allocation, the source rows of each item, replica fan-out, the
metrics -- runs in the CPU suite.  The loopback transport keeps the fused kernel's contract: the elements are compacted
from their rows (SourceRows, common/store_window.h) and packed, so the stored object and its digest are those of
batch_put_device_fp8 of the compacted rows."""
import numpy as np

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
T = 16384


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


class Sources:
    """Random bf16 bit patterns (uint16) in host buffers starting `skew` elements past a 64-byte boundary; kept alive."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.keep = []

    def __call__(self, extent, skew=0):
        raw = ((self.rng.standard_normal(extent + 64) * 3).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        self.keep.append(raw)
        o = ((-raw.ctypes.data) % 64) // 2 + skew
        return raw[o:o + extent], raw.ctypes.data + 2 * o


def compact(src, width, pitch, rows):
    """The tensor a strided put stores: row r = src[r * pitch, + width), back to back."""
    return np.concatenate([src[r * pitch:r * pitch + width] for r in range(rows)]) if rows and width else src[:0]


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.get_workers(key)]


# (elem_width, elem_pitch, rows, skew): one KV head of eight, 8-element rows (16 bytes, 2048 per tile), a 16-byte gap, rows
# of 1000 elements, rows longer than a tile, an object with a partial last tile, width == pitch, one row wider than the
# pitch, and a start 8 elements (16 bytes) past a 64-byte boundary.  Every element count is a multiple of 32.
PATTERNS = [(128, 1024, 64, 0), (8, 64, 2048, 0), (40, 48, 800, 0), (1000, 1008, 32, 0), (T + 48, T + 56, 2, 0),
            (96, 160, 3 * T // 96 + 1, 8), (64, 64, 10, 0), (96, 1, 1, 0), (256, 512, 16, 8)]


def _put_and_check(bb, cl, src_of, pats, tag, replicas):
    keys, ptrs, srcs = [], [], []
    for j, (w, p, r, skew) in enumerate(pats):
        src, ptr = src_of((r - 1) * p + w, skew)
        keys.append(f"{tag}/{j}"), ptrs.append(ptr), srcs.append(src)
    ecs = cl.batch_put_device_fp8_strided(keys, ptrs, [p[0] for p in pats], [p[1] for p in pats], [p[2] for p in pats],
                                          _cfg(bb, replicas), 0)
    assert ecs == [bb.ErrorCode.OK] * len(pats), (tag, ecs)
    dense = [compact(s, w, p, r) for s, (w, p, r, _) in zip(srcs, pats)]
    # the stored bytes are the reference packing of the compacted rows, in every copy
    for (ec, blob), d, key in zip(cl.batch_get(keys), dense, keys):
        assert ec == bb.ErrorCode.OK, key
        assert bytes(blob) == bb.mxfp8_pack_ref(d), key
        assert len(cl.get_workers(key)) == replicas
    # the recorded digests are those of a packed put of the compacted rows
    ckeys = [k + "/c" for k in keys]
    assert cl.batch_put_device_fp8(ckeys, [d.ctypes.data for d in dense], [d.size for d in dense], _cfg(bb, replicas), 0) == \
        [bb.ErrorCode.OK] * len(pats)
    for k, ck in zip(keys, ckeys):
        assert _sums(cl, k) == _sums(cl, ck), k
    # every fp8 get reads it: whole, and a strided slice of it
    outs = [np.zeros(d.size, dtype=np.uint16) for d in dense]
    assert cl.batch_get_device_fp8(keys, [o.ctypes.data for o in outs], [d.size for d in dense], 0) == [bb.ErrorCode.OK] * len(pats)
    for o, d in zip(outs, dense):
        assert np.array_equal(o, np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(d), d.size), dtype=np.uint16))
    for k, d in zip(keys, dense):
        ref = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(d), d.size), dtype=np.uint16)
        n_rows = d.size // 64
        out = np.zeros(16 * n_rows + 64, dtype=np.uint16)
        at = ((-out.ctypes.data) % 16) // 2
        assert cl.batch_get_device_fp8_strided([k], [out.ctypes.data + 2 * at], [d.size], [0], [16], [64], [n_rows], 0) == [bb.ErrorCode.OK]
        assert np.array_equal(out[at:at + 16 * n_rows], compact(ref, 16, 64, n_rows)), k
    return sum(2 * w * r for w, _, r, _ in pats)


def test_fp8_strided_put_stores_the_compacted_rows_with_one_to_three_copies(bb):
    with LocalCluster(cluster_id="fp8sp", n_workers=3, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        src_of = Sources(1)
        n0, b0 = _counter(cl, "device_put_fp8_strided_total"), _counter(cl, "device_put_fp8_strided_bytes_total")
        want_b = 0
        for rep in (1, 2, 3):
            want_b += _put_and_check(bb, cl, src_of, PATTERNS, f"r{rep}", rep)
        assert _counter(cl, "device_put_fp8_strided_total") == n0 + 3 * len(PATTERNS)
        assert _counter(cl, "device_put_fp8_strided_bytes_total") == b0 + want_b


def test_fp8_strided_put_errors_fail_alone_before_any_allocation(bb):
    with LocalCluster(cluster_id="fp8sperr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        src_of = Sources(2)
        E = bb.ErrorCode
        # (elem_width, elem_pitch, rows, skew, expected)
        cases = [(128, 1024, 8, 0, E.OK),
                 (101, 100, 2, 0, E.INVALID_ARGUMENT),               # width > pitch with several rows
                 (8, 2**63, 3, 0, E.VALUE_OUT_OF_RANGE),             # (rows - 1) * pitch overflows
                 (2**62, 2**62 + 8, 2, 0, E.VALUE_OUT_OF_RANGE),     # the source extent in bytes overflows
                 (128, 1024, 8, 1, E.NOT_IMPLEMENTED),               # start 2 bytes off 16
                 (40, 44, 32, 0, E.NOT_IMPLEMENTED),                 # gap of 4 elements
                 (40, 75, 32, 0, E.NOT_IMPLEMENTED),                 # gap of 35 elements
                 (32, 32, 1, 4, E.NOT_IMPLEMENTED),                  # one row, 8 bytes off 16
                 (40, 48, 32, 0, E.OK)]                              # gap of 8 elements
        keys, ptrs, srcs = [], [], []
        for j, (w, p, r, skew, _) in enumerate(cases):
            extent = (r - 1) * p + w if (r - 1) * p + w < 1 << 20 else 64  # the overflowing cases are refused unread
            src, ptr = src_of(extent, skew)
            keys.append(f"e/{j}"), ptrs.append(ptr), srcs.append(src)
        n0 = _counter(cl, "device_put_fp8_strided_total")
        ecs = cl.batch_put_device_fp8_strided(keys, ptrs, [c_[0] for c_ in cases], [c_[1] for c_ in cases], [c_[2] for c_ in cases],
                                              _cfg(bb, 1), 0)
        assert ecs == [c_[4] for c_ in cases], ecs
        assert _counter(cl, "device_put_fp8_strided_total") == n0 + 2
        for k, s, (w, p, r, _, e) in zip(keys, srcs, cases):
            assert cl.object_exists(k) == (e == E.OK), k
            if e == E.OK:
                ec, blob = cl.batch_get([k])[0]
                assert ec == E.OK and bytes(blob) == bb.mxfp8_pack_ref(compact(s, w, p, r))
        # an element count that is not a whole number of MX blocks fails the batch, as batch_put_device_fp8 does
        a, pa = src_of(1024 * 7 + 128)
        b, pb = src_of(64 * 4 + 20)
        ecs = cl.batch_put_device_fp8_strided(["n/0", "n/1"], [pa, pb], [128, 24], [1024, 64], [8, 5], _cfg(bb, 1), 0)
        assert ecs == [E.INVALID_PARAMETERS] * 2
        assert ecs == cl.batch_put_device_fp8(["n/0", "n/1"], [pa, pb], [1024, 120], _cfg(bb, 1), 0)
        assert not cl.object_exists("n/0") and not cl.object_exists("n/1")
        assert cl.batch_put_device_fp8_strided(["x"], [pa], [128], [1024], [1, 2], _cfg(bb, 1), 0) == [E.INVALID_PARAMETERS]
