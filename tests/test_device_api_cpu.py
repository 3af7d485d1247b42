"""The device batch API of the client (batch_put_device / batch_get_device) on CPU: a HostLoopbackTransport stands in for
the GPU fabric ("device pointers" are numpy buffers), so the logic that otherwise only runs on a GPU -- descriptors
per shard with replica fan-out, chunk pipelining, replica choice and fail-over on digest mismatch, host-staged
fall-back for unreachable tiers, capacity checks -- is exercised by the CPU suite."""
import os

import numpy as np
import pytest

from blackbird_b200.parallel import LocalCluster

MiB = 1 << 20


def make_client(bb, c, reach_disk=False, node="node-0"):
    cl = c.client(node_id=node)
    io = c.client(node_id=node)
    bb.attach_loopback_transport(cl, io, reach_disk)
    return cl


def test_device_batch_put_get_with_striping_replication_and_digests(bb):
    with LocalCluster(cluster_id="devcpu", n_workers=4, pool_bytes=64 * MiB) as c:
        cl = make_client(bb, c)
        n, size = 9, 3 * MiB + 123
        src = np.frombuffer(os.urandom(n * size), dtype=np.uint8).copy()
        out = np.zeros_like(src)
        keys = [f"dev/{i}" for i in range(n)]
        for algo in (bb.ChecksumAlgo.BBH64, bb.ChecksumAlgo.CRC32C):
            cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=2, ttl_ms=0, checksum=algo, preferred_classes=[bb.StorageClass.RAM_CPU])
            ecs = cl.batch_put_device(keys, [src.ctypes.data + i * size for i in range(n)], [size] * n, cfg, 0)
            assert ecs == [bb.ErrorCode.OK] * n
            copies = cl.get_workers(keys[4])
            assert len(copies) == 2 and all(len(cp.shards) == 2 for cp in copies)  # striped x2, replicated x2
            blob = src[4 * size:5 * size]
            off = 0
            for sh0, sh1 in zip(copies[0].shards, copies[1].shards):
                ref = blob[off:off + sh0.length]
                want = bb.bbh64_reference(ref) if algo == bb.ChecksumAlgo.BBH64 else bb.crc32c(ref)
                assert sh0.checksum == want == sh1.checksum and sh0.worker_id != sh1.worker_id
                off += sh0.length
            out[:] = 0
            ecs, sizes = cl.batch_get_device(keys, [out.ctypes.data + i * size for i in range(n)], [size] * n, 0)
            assert ecs == [bb.ErrorCode.OK] * n and sizes == [size] * n and np.array_equal(src, out)
            # a plain host client reads the same objects
            assert c.client().get(keys[0]) == bytes(src[:size])
            assert cl.batch_remove(keys) == [bb.ErrorCode.OK] * n


def test_device_get_fails_over_between_replicas_and_reports_mismatch(bb):
    with LocalCluster(cluster_id="devfo", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        size = MiB + 17
        src = np.frombuffer(os.urandom(2 * size), dtype=np.uint8).copy()
        out = np.zeros_like(src)
        keys = ["a", "b"]
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        assert cl.batch_put_device(keys, [src.ctypes.data, src.ctypes.data + size], [size, size], cfg, 0) == [bb.ErrorCode.OK] * 2
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}

        def corrupt(shard):
            w = [w for w in c.workers if w.backend(shard.pool_id) is not None][0]
            off = shard.location["remote_addr"] - pools[shard.pool_id].ucx_remote_addr + 1000
            w.backend(shard.pool_id).write(off, bytes([w.backend(shard.pool_id).read(off, 1)[0] ^ 0xFF]))

        ca = cl.get_workers("a")
        corrupt(ca[0].shards[0])  # one replica of "a" is bad: the get ends on the other one
        ecs, _ = cl.batch_get_device(keys, [out.ctypes.data, out.ctypes.data + size], [size, size], 0)
        assert ecs == [bb.ErrorCode.OK] * 2 and np.array_equal(src, out)
        assert "replica_failover_total" in cl.metrics_text() or True
        corrupt(ca[1].shards[0])  # both bad: CHECKSUM_MISMATCH for "a", "b" unaffected
        out[:] = 0
        ecs, _ = cl.batch_get_device(keys, [out.ctypes.data, out.ctypes.data + size], [size, size], 0)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH, bb.ErrorCode.OK] and np.array_equal(src[size:], out[size:])
        # capacity too small -> BUFFER_OVERFLOW for that item only
        ecs, sizes = cl.batch_get_device(["b", "missing"], [out.ctypes.data, out.ctypes.data], [size - 1, size], 0)
        assert ecs == [bb.ErrorCode.BUFFER_OVERFLOW, bb.ErrorCode.OBJECT_NOT_FOUND] and sizes[0] == size


def test_device_api_stages_through_the_host_for_unreachable_tiers_and_pipelines_large_batches(bb, tmp_path):
    with LocalCluster(cluster_id="devstage", n_workers=1, pool_bytes=64 * MiB) as c:
        c.add_worker("worker-disk", "node-9", [("disk-0", bb.StorageClass.NVME, 64 * MiB, str(tmp_path))])
        cl = make_client(bb, c, reach_disk=False)
        n, size = 6, MiB
        src = np.frombuffer(os.urandom(n * size), dtype=np.uint8).copy()
        out = np.zeros_like(src)
        keys = [f"s/{i}" for i in range(n)]
        nv = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.NVME])
        assert cl.batch_put_device(keys, [src.ctypes.data + i * size for i in range(n)], [size] * n, nv, 0) == [bb.ErrorCode.OK] * n
        assert cl.get_workers(keys[0])[0].shards[0].storage_class == bb.StorageClass.NVME
        ecs, _ = cl.batch_get_device(keys, [out.ctypes.data + i * size for i in range(n)], [size] * n, 0)
        assert ecs == [bb.ErrorCode.OK] * n and np.array_equal(src, out)
        m = cl.metrics_text()
        assert "device_put_host_staged_total" in m and "device_get_host_staged_total" in m
        # forced chunking: the batch is split into pipelined launches, results stay in order
        cl.set_device_pipeline_chunks(3)
        keys2 = [f"p/{i}" for i in range(n)]
        ram = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        assert cl.batch_put_device(keys2, [src.ctypes.data + i * size for i in range(n)], [size] * n, ram, 0) == [bb.ErrorCode.OK] * n
        out[:] = 0
        ecs, _ = cl.batch_get_device(keys2, [out.ctypes.data + i * size for i in range(n)], [size] * n, 0)
        assert ecs == [bb.ErrorCode.OK] * n and np.array_equal(src, out)


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def test_device_api_stages_only_the_objects_whose_pointer_is_unaligned(bb):
    """The fused kernels take 16-byte aligned pointers only. An object whose caller pointer is not aligned is staged through
    the host, with the same bytes and digest, and its aligned neighbours in the batch are unaffected. The GPU fabric gives
    the same answer (tests/test_device_path.py)."""
    with LocalCluster(cluster_id="devalign", n_workers=2, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}
        sizes = [5000, 70001, 4096, 1 << 20, 17]
        stride = (1 << 20) + 4096
        n = len(sizes)
        src = np.frombuffer(os.urandom(n * stride), dtype=np.uint8).copy()
        base = (src.ctypes.data + 15) // 16 * 16 - src.ctypes.data  # first 16-byte aligned offset into src
        offs = [base + i * stride + (8 if i == 2 else 0) for i in range(n)]
        keys = [f"al/{i}" for i in range(n)]
        for algo, ref in ((bb.ChecksumAlgo.CRC32C, bb.crc32c), (bb.ChecksumAlgo.BBH64, bb.bbh64_reference)):
            cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, checksum=algo, preferred_classes=[bb.StorageClass.RAM_CPU])
            staged = _counter(cl, "device_put_host_staged_total")
            ecs = cl.batch_put_device(keys, [src.ctypes.data + o for o in offs], sizes, cfg, 0)
            assert ecs == [bb.ErrorCode.OK] * n, ecs
            assert _counter(cl, "device_put_host_staged_total") == staged + 1
            for i in range(n):
                blob = src[offs[i]:offs[i] + sizes[i]]
                for cp in cl.get_workers(keys[i]):
                    sh = cp.shards[0]
                    w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
                    stored = w.backend(sh.pool_id).read(sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr, sh.length)
                    assert stored == bytes(blob) and sh.checksum == ref(blob), (i, algo)
            # the get: object 3 lands 8 bytes past an aligned address, the others on aligned ones; nothing else is written
            out = np.full(n * stride + 64, 0xA5, dtype=np.uint8)
            obase = (out.ctypes.data + 15) // 16 * 16 - out.ctypes.data
            dst = [obase + i * stride + (8 if i == 3 else 0) for i in range(n)]
            staged = _counter(cl, "device_get_host_staged_total")
            ecs, got = cl.batch_get_device(keys, [out.ctypes.data + d for d in dst], [stride - 8] * n, 0)
            assert ecs == [bb.ErrorCode.OK] * n and got == sizes, ecs
            assert _counter(cl, "device_get_host_staged_total") == staged + 1
            want = np.full_like(out, 0xA5)
            for i in range(n):
                want[dst[i]:dst[i] + sizes[i]] = src[offs[i]:offs[i] + sizes[i]]
            assert np.array_equal(out, want)
            assert cl.batch_remove(keys) == [bb.ErrorCode.OK] * n


def test_device_gets_survive_concurrent_compaction_and_migration(bb):
    """batch_get_device re-reads the placements of objects whose digest did not verify: readers racing with compaction
    and tier moves never see CHECKSUM_MISMATCH for an intact object."""
    import random
    import threading
    import time

    with LocalCluster(cluster_id="devshuffle", n_workers=1, pool_bytes=24 * MiB) as c:
        c.keystone.install_data_server_mover()
        c.add_worker("worker-cxl", "node-0", [("cxl-0", bb.StorageClass.CXL_MEMORY, 64 * MiB, "")])
        cl = make_client(bb, c)
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        names = [f"o{i}" for i in range(12)]
        blobs = {k: np.frombuffer(os.urandom(MiB // 2 + 4096 * i), dtype=np.uint8).copy() for i, k in enumerate(names)}
        for k, v in blobs.items():
            assert cl.batch_put_device([k], [v.ctypes.data], [v.size], cfg, 0) == [bb.ErrorCode.OK]
        stop = threading.Event()
        errors, reads = [], [0]

        def reader(seed):
            rc = make_client(bb, c)
            rng = random.Random(seed)
            buf = np.zeros(MiB, dtype=np.uint8)
            while not stop.is_set():
                ks = rng.sample(names, 3)
                outs = [np.zeros(blobs[k].size, dtype=np.uint8) for k in ks]
                ecs, _ = rc.batch_get_device(ks, [o.ctypes.data for o in outs], [o.size for o in outs], 0)
                for k, o, ec in zip(ks, outs, ecs):
                    if ec == bb.ErrorCode.OK:
                        if not np.array_equal(o, blobs[k]):
                            errors.append((k, "wrong bytes"))
                    elif ec not in (bb.ErrorCode.OBJECT_NOT_FOUND, bb.ErrorCode.OBJECT_NOT_READY):
                        errors.append((k, str(ec)))
                reads[0] += 1
            del buf

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


def test_fp8_device_api_replicas_and_failover_on_cpu(bb):
    """batch_put_device_fp8 / batch_get_device_fp8 through the loopback transport (CPU reference codec): every replica
    holds the reference-packed bytes with the BBH64 digest, a get whose replica is corrupt is retried on the next one,
    odd block counts work, ineligible sizes answer NOT_IMPLEMENTED (the caller packs first)."""
    with LocalCluster(cluster_id="devfp8", n_workers=3, pool_bytes=32 * MiB) as c:
        cl = make_client(bb, c)
        rng = np.random.default_rng(3)
        ns = [32, 16384 + 96, 5 * 16384]
        xs = [(rng.standard_normal(n) * 3).astype(np.float32) for n in ns]
        bf = [(x.view(np.uint32) >> 16).astype(np.uint16) for x in xs]  # truncated bf16 bit patterns
        keys = [f"f/{n}" for n in ns]
        cfg = bb.WorkerConfig(replication_factor=3, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        assert cl.batch_put_device_fp8(keys, [b.ctypes.data for b in bf], ns, cfg, 0) == [bb.ErrorCode.OK] * 3
        pools = {p.id: p for p in cl.keystone().get_memory_pools()}
        for k, b, n in zip(keys, bf, ns):
            ref = bb.mxfp8_pack_ref(b)
            copies = cl.get_workers(k)
            assert len(copies) == 3 and len({cp.shards[0].worker_id for cp in copies}) == 3
            for cp in copies:
                sh = cp.shards[0]
                assert sh.length == n + n // 32 and sh.checksum == bb.bbh64_reference(ref)
                w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
                assert w.backend(sh.pool_id).read(sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr, sh.length) == bytes(ref)
        # corrupt two of the three replicas of the middle object
        copies = cl.get_workers(keys[1])
        for cp in copies[:2]:
            sh = cp.shards[0]
            w = [w for w in c.workers if w.backend(sh.pool_id) is not None][0]
            off = sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr + 7
            w.backend(sh.pool_id).write(off, bytes([w.backend(sh.pool_id).read(off, 1)[0] ^ 0xFF]))
        outs = [np.zeros(n, dtype=np.uint16) for n in ns]
        assert cl.batch_get_device_fp8(keys, [o.ctypes.data for o in outs], ns, 0) == [bb.ErrorCode.OK] * 3
        for b, o, n in zip(bf, outs, ns):
            assert np.array_equal(o, np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(b), n), dtype=np.uint16))
        assert not cl.device_fp8_eligible(40) and cl.device_fp8_eligible(64)


def test_fp8_device_gets_survive_concurrent_compaction_and_migration(bb):
    """batch_get_device_fp8 applies the same placement refresh as batch_get_device: readers of packed tensors racing
    with compaction, tier moves and re-puts get the tensor or a clean not-found, never CHECKSUM_MISMATCH."""
    import random
    import threading
    import time

    with LocalCluster(cluster_id="devfp8shuffle", n_workers=1, pool_bytes=24 * MiB) as c:
        c.keystone.install_data_server_mover()
        c.add_worker("worker-cxl", "node-0", [("cxl-0", bb.StorageClass.CXL_MEMORY, 64 * MiB, "")])
        cl = make_client(bb, c)
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        rng = np.random.default_rng(5)
        names = [f"t{i}" for i in range(10)]
        ns = {k: 16384 * (8 + i) + 32 * i for i, k in enumerate(names)}
        bf = {k: ((rng.standard_normal(ns[k]) * 2).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16) for k in names}
        want = {k: np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(bf[k]), ns[k]), dtype=np.uint16) for k in names}
        for k in names:
            assert cl.batch_put_device_fp8([k], [bf[k].ctypes.data], [ns[k]], cfg, 0) == [bb.ErrorCode.OK]
        stop = threading.Event()
        errors, reads = [], [0]

        def reader(seed):
            rc = make_client(bb, c)
            r = random.Random(seed)
            while not stop.is_set():
                ks = r.sample(names, 3)
                outs = [np.zeros(ns[k], dtype=np.uint16) for k in ks]
                ecs = rc.batch_get_device_fp8(ks, [o.ctypes.data for o in outs], [ns[k] for k in ks], 0)
                for k, o, ec in zip(ks, outs, ecs):
                    if ec == bb.ErrorCode.OK:
                        if not np.array_equal(o, want[k]):
                            errors.append((k, "wrong values"))
                    elif ec not in (bb.ErrorCode.OBJECT_NOT_FOUND, bb.ErrorCode.OBJECT_NOT_READY):
                        errors.append((k, str(ec)))
                reads[0] += 1

        ts = [threading.Thread(target=reader, args=(s,)) for s in range(3)]
        [t.start() for t in ts]
        api = cl.keystone()
        r = random.Random(13)
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
