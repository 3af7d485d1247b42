"""Gets into strided destinations (batch_get_device_scatter, batch_get_device_fp8_scatter) on CPU: the HostLoopbackTransport
stands in for the GPU fabric, so the client's scatter logic -- the destination rows rebased to every shard, replica choice
and fail-over, the placement refresh, the host-staged path with its 2-D copy -- runs in the CPU suite.  The loopback keeps
the fabric's contract: every shard is read whole and verified, and only the object's bytes of the rows are written."""
import os

import numpy as np

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20
GUARD = 0xA5


def make_client(bb, c, node="node-0", reach_disk=False):
    cl = c.client(node_id=node)
    io = c.client(node_id=node)
    bb.attach_loopback_transport(cl, io, reach_disk)
    return cl


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, replicas, stripes, algo="XXH3", cls="RAM_CPU"):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=stripes, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[getattr(bb.StorageClass, cls)])


def scatter_model(blob, width, pitch, phase=0):
    """Where each object byte lands: byte x at ((x + phase) // width) * pitch + (x + phase) % width."""
    x = np.arange(len(blob), dtype=np.int64) + phase
    return (x // width) * pitch + x % width


def _scatter(cl, keys, pats, skew=None):
    """Scattered gets into one guard-filled buffer: pattern i = (width, pitch, rows) lands at a 16-byte aligned region, moved
    by skew[i] bytes, with guard bytes before and after it; returns (error codes, sizes, buffer, regions)."""
    total = sum((r - 1) * p + w + 256 if r else 256 for w, p, r in pats) + 256
    raw = np.full(total, GUARD, dtype=np.uint8)
    o = (-raw.ctypes.data) % 16 + 64
    regions = []
    for i, (w, p, r) in enumerate(pats):
        reg = o + (skew or {}).get(i, 0)
        regions.append(reg)
        o = (reg + ((r - 1) * p + w if r else 0) + 15) // 16 * 16 + 64
    ecs, sizes = cl.batch_get_device_scatter(keys, [raw.ctypes.data + g for g in regions], [p[0] for p in pats], [p[1] for p in pats],
                                             [p[2] for p in pats], 0)
    return ecs, sizes, raw, regions


def _check(raw, regions, blobs, pats, ok):
    """Every region holds its object at the rule's places (when ok); every other byte, gaps included, is still a guard."""
    want = np.full_like(raw, GUARD)
    for reg, b, (w, p, _), good in zip(regions, blobs, pats, ok):
        if good and len(b):
            want[reg + scatter_model(b, w, p)] = b
    assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]


def _put(bb, cl, key, size, cfg):
    blob = np.frombuffer(os.urandom(size), dtype=np.uint8).copy()
    assert cl.batch_put_device([key], [blob.ctypes.data], [size], cfg, 0) == [bb.ErrorCode.OK]
    return blob


def test_rule_matches_the_numpy_model(bb):
    """SourceRows.runs (the rule the transports store by) agrees with the model, phases included."""
    for width, pitch, phase, n in [(1, 3, 0, 40), (16, 32, 5, 1000), (100, 100, 0, 250), (17, 48, 16, 333)]:
        blob = np.arange(n, dtype=np.int64)
        dst = np.full(n // width * pitch + 2 * pitch, -1, dtype=np.int64)
        for x, at, k in bb.SourceRows(pitch, width, phase).runs(n):
            dst[at:at + k] = blob[x:x + k]
        want = np.full_like(dst, -1)
        want[scatter_model(blob, width, pitch, phase)] = blob
        assert np.array_equal(dst, want)


def test_round_trips_over_stripes_for_every_algorithm(bb):
    """Striped objects whose shard boundaries fall mid-row and inside gaps; rows of 1, 15, 16, 17 bytes and more."""
    with LocalCluster(cluster_id="scpu", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        n0 = _counter(cl, "device_get_scatter_total")
        for algo in ("XXH3", "CRC32C", "BBH64", "NONE"):
            for stripes in (2, 3, 4):
                size = 3 * MiB + 4321
                key = f"s/{algo}/{stripes}"
                blob = _put(bb, cl, key, size, _cfg(bb, 1, stripes, algo))
                pats = [(1, 3, size), (17, 33, -(-size // 17)), (4096, 8192, size // 4096 + 1), (size, size + 16, 1),
                        (1000, 1000, size // 1000 + 1), (48, 64, size // 48 + 1)]
                ecs, sizes, raw, regions = _scatter(cl, [key] * len(pats), pats)
                assert ecs == [bb.ErrorCode.OK] * len(pats), (algo, stripes, ecs)
                assert sizes == [size] * len(pats)
                _check(raw, regions, [blob] * len(pats), pats, [True] * len(pats))
        assert _counter(cl, "device_get_scatter_total") == n0 + 4 * 3 * 6


def test_fail_over_keeps_the_gaps_and_all_corrupt_refreshes_once(bb):
    with LocalCluster(cluster_id="scfo", n_workers=6, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def flip(sh, pos):
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + pos
            b = w.backend(sh.pool_id)
            b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))

        for replicas in (2, 3):
            size = 2 * MiB + 77
            key = f"f{replicas}"
            blob = _put(bb, cl, key, size, _cfg(bb, replicas, 2))
            copies = cl.get_workers(key)
            pat = (64, 1024, -(-size // 64))
            mm = _counter(cl, "checksum_mismatch_total")
            for cp in copies:  # one corrupt copy at a time: the get fails over, rows right, gaps untouched
                flip(cp.shards[-1], 12345)
                ecs, _, raw, regions = _scatter(cl, [key], [pat])
                assert ecs == [bb.ErrorCode.OK]
                _check(raw, regions, [blob], [pat], [True])
                flip(cp.shards[-1], 12345)
            assert _counter(cl, "checksum_mismatch_total") > mm
            for cp in copies:
                flip(cp.shards[0], 99)
            ref = _counter(cl, "get_placement_refresh_total")
            ecs, _, raw, regions = _scatter(cl, [key], [pat])
            assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
            assert _counter(cl, "get_placement_refresh_total") == ref + 1
            # the loopback stores nothing from a copy that fails: every byte outside the rows is still a guard
            _check(raw, regions, [blob], [pat], [False])


def test_misaligned_items_are_staged_and_their_neighbours_are_not(bb):
    with LocalCluster(cluster_id="scal", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 300001
        blob = _put(bb, cl, "a", size, _cfg(bb, 1, 1))
        big = _put(bb, cl, "b", 2 * MiB, _cfg(bb, 1, 2))
        # 0: fused; 1: misaligned pointer; 2: gap 35; 3: gap 24 whose shards hold one row each; 4: fused over two stripes;
        # 5: one row at an odd address
        pats = [(100, 132, 3001), (100, 116, 3001), (33, 68, -(-size // 33)), (MiB, MiB + 24, 2), (32, 48, 2 * MiB // 32), (size, size, 1)]
        skew = {1: 3, 5: 1}
        staged = _counter(cl, "device_get_host_staged_total")
        ecs, sizes, raw, regions = _scatter(cl, ["a", "a", "a", "b", "b", "a"], pats, skew)
        assert ecs == [bb.ErrorCode.OK] * 6, ecs
        _check(raw, regions, [blob, blob, blob, big, big, blob], pats, [True] * 6)
        assert _counter(cl, "device_get_host_staged_total") == staged + 4  # items 0 and 4 went to the transport
        assert sizes == [size, size, size, 2 * MiB, 2 * MiB, size]


def test_disk_placements_are_staged(bb, tmp_path):
    with LocalCluster(cluster_id="scnv", n_workers=1, pool_bytes=32 * MiB) as c:
        c.add_worker("worker-disk", "node-9", [("disk-0", bb.StorageClass.NVME, 64 * MiB, str(tmp_path))])
        cl = make_client(bb, c)
        size = 100000
        blob = _put(bb, cl, "n", size, _cfg(bb, 1, 1, cls="NVME"))
        assert cl.get_workers("n")[0].shards[0].storage_class == bb.StorageClass.NVME
        ram = _put(bb, cl, "r", size, _cfg(bb, 1, 1))
        staged = _counter(cl, "device_get_host_staged_total")
        pats = [(64, 96, -(-size // 64)), (64, 96, -(-size // 64))]
        ecs, _, raw, regions = _scatter(cl, ["n", "r"], pats)
        assert ecs == [bb.ErrorCode.OK] * 2
        _check(raw, regions, [blob, ram], pats, [True, True])
        assert _counter(cl, "device_get_host_staged_total") == staged + 1


def test_errors_short_objects_and_empty_rows(bb):
    with LocalCluster(cluster_id="scerr", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 10000
        blob = _put(bb, cl, "e", size, _cfg(bb, 1, 2))
        pats = [(100, 128, 100),          # exactly the object
                (101, 100, 2),            # width > pitch
                (8, 2**63, 3),            # the extent overflows
                (2**32, 2**33, 2**33),    # the size overflows
                (100, 128, 99),           # the object is larger than the rows
                (64, 80, 200),            # a shorter object fills its bytes in row order
                (100, 128, 0),            # no rows: capacity 0
                (100, 128, 100)]          # missing key
        keys = ["e"] * 7 + ["missing"]
        E = bb.ErrorCode
        total = sum(p[2] * p[1] for p in pats if p[1] < 2**20 and p[2] < 2**20) + 4096
        raw = np.full(total, GUARD, dtype=np.uint8)
        o = (-raw.ctypes.data) % 16 + 64
        regions = []
        for w, p, r in pats:
            regions.append(o)
            if p < 2**20 and r < 2**20:
                o += r * p + 64
        ecs, sizes = cl.batch_get_device_scatter(keys, [raw.ctypes.data + g for g in regions], [p[0] for p in pats],
                                                 [p[1] for p in pats], [p[2] for p in pats], 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.VALUE_OUT_OF_RANGE, E.VALUE_OUT_OF_RANGE, E.BUFFER_OVERFLOW, E.OK,
                       E.BUFFER_OVERFLOW, E.OBJECT_NOT_FOUND], ecs
        assert sizes[0] == size and sizes[5] == size and sizes[1] == 0
        want = np.full_like(raw, GUARD)
        for k in (0, 5):
            want[regions[k] + scatter_model(blob, pats[k][0], pats[k][1])] = blob
        assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]


def test_one_row_and_width_equal_to_pitch_are_plain_gets(bb):
    with LocalCluster(cluster_id="scone", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = 200003
        blob = _put(bb, cl, "o", size, _cfg(bb, 1, 2))
        plain = np.full(size + 64, GUARD, dtype=np.uint8)
        p0 = (-plain.ctypes.data) % 16
        ecs, sizes = cl.batch_get_device(["o"], [plain.ctypes.data + p0], [size], 0)
        assert ecs == [bb.ErrorCode.OK] and sizes == [size]
        for pat in [(size, size, 1), (1000, 1000, 201), (size + 5, 7, 1)]:
            got = np.full(size + 64, GUARD, dtype=np.uint8)
            ecs, sizes = cl.batch_get_device_scatter(["o"], [got.ctypes.data + p0], [pat[0]], [pat[1]], [pat[2]], 0)
            assert ecs == [bb.ErrorCode.OK] and sizes == [size]
            assert np.array_equal(got, plain)


# ---------------------------------------------------------------- MXFP8
def _bf16(rng, n):
    return ((rng.standard_normal(n) * 3).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)


def test_fp8_scatter_matches_the_cpu_codec(bb):
    with LocalCluster(cluster_id="scfp8", n_workers=2, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(7)
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        shapes = [(64, 64 + 8, 32), (16384, 16384 + 24, 3), (8, 16, 4096), (96, 96, 7), (32 * 1000, 32 * 1000, 1)]
        keys, refs = [], []
        for k, (w, p, r) in enumerate(shapes):
            src = _bf16(rng, w * r)
            keys.append(f"p{k}")
            assert cl.batch_put_device_fp8([keys[-1]], [src.ctypes.data], [src.size], cfg, 0) == [bb.ErrorCode.OK]
            refs.append(np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(src), src.size), dtype=np.uint16))
        total = sum(p * r + 64 for _, p, r in shapes) + 64
        raw = np.full(total, 0xA5A5, dtype=np.uint16)
        o = ((-raw.ctypes.data) % 16) // 2 + 16
        regions = []
        for w, p, r in shapes:
            regions.append(o)
            o += (p * r + 7) // 8 * 8 + 16
        # every copy is read by the fused path's rule; one corrupt copy fails over to the other
        (cp0, _) = cl.get_workers(keys[1])
        pools = {q.id: q for q in cl.keystone().get_memory_pools()}
        sh = cp0.shards[0]
        w_ = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
        off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + 5
        b = w_.backend(sh.pool_id)
        b.write(off, bytes([b.read(off, 1)[0] ^ 0xFF]))
        n0 = _counter(cl, "device_get_fp8_scatter_total")
        ecs = cl.batch_get_device_fp8_scatter(keys, [raw.ctypes.data + 2 * g for g in regions], [w * r for w, _, r in shapes],
                                              [s[0] for s in shapes], [s[1] for s in shapes], [s[2] for s in shapes], 0)
        assert ecs == [bb.ErrorCode.OK] * len(shapes), ecs
        want = np.full_like(raw, 0xA5A5)
        for reg, ref, (w, p, _) in zip(regions, refs, shapes):
            want[reg + scatter_model(ref, w, p)] = ref
        assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]
        assert _counter(cl, "device_get_fp8_scatter_total") == n0 + len(shapes)


def test_fp8_scatter_errors_fail_alone(bb):
    with LocalCluster(cluster_id="scfp8e", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(3)
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        src = _bf16(rng, 1024)
        assert cl.batch_put_device_fp8(["q"], [src.ctypes.data], [1024], cfg, 0) == [bb.ErrorCode.OK]
        ref = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(src), 1024), dtype=np.uint16)
        raw = np.full(8 * 4096, 0xA5A5, dtype=np.uint16)
        base = ((-raw.ctypes.data) % 16) // 2 + 16
        E = bb.ErrorCode
        # (ptr offset in elements, width, pitch, rows)
        items = [(0, 32, 40, 32),        # ok
                 (4096, 32, 40, 31),     # rows * width != n_elems
                 (8192, 32, 36, 32),     # gap of 4 elements
                 (12289, 32, 40, 32),    # misaligned pointer
                 (16384, 40, 32, 2),     # width > pitch
                 (20480, 1024, 1024, 1)]  # one row: a plain fp8 get
        ecs = cl.batch_get_device_fp8_scatter(["q"] * len(items), [raw.ctypes.data + 2 * (base + it[0]) for it in items], [1024] * len(items),
                                              [it[1] for it in items], [it[2] for it in items], [it[3] for it in items], 0)
        assert ecs == [E.OK, E.INVALID_ARGUMENT, E.NOT_IMPLEMENTED, E.NOT_IMPLEMENTED, E.INVALID_ARGUMENT, E.OK], ecs
        want = np.full_like(raw, 0xA5A5)
        want[base + scatter_model(ref, 32, 40)] = ref
        want[base + 20480:base + 20480 + 1024] = ref
        assert np.array_equal(raw, want), np.nonzero(raw != want)[0][:8]
