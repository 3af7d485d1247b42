"""GPU tests of the device put / get path as callers reach it: batch_put_device / batch_get_device on a GpuRankCluster, through
the client's chunk planning and the fabric's descriptor building, against a host model of the store.

For every copy of every object the model reads the stored bytes back through the worker's backend and checks them against
the source slice, checks the digest the Keystone recorded against the CPU model of those bytes, and checks every get
destination byte for byte, including guard bytes past each object up to its capacity."""
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MiB = 1 << 20
GUARD = 0xA5
ALGOS = ["XXH3", "CRC32C", "BBH64", "NONE"]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")
    return torch


def _stream(torch):
    return torch.cuda.current_stream().cuda_stream


def _ref(bb, algo):
    return {"XXH3": bb.xxh3t64, "CRC32C": bb.crc32c, "BBH64": bb.bbh64, "NONE": lambda b: 0}[algo]


def _cfg(bb, algo, replicas=1, tier="RAM_GPU"):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, checksum=getattr(bb.ChecksumAlgo, algo),
                           preferred_classes=[getattr(bb.StorageClass, tier)])


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _random(torch, n, seed, pinned=False):
    """n random bytes at a 256-byte aligned address (device memory, or pinned host memory filled from the device)."""
    import blackbird_b200._bb as bb

    dev = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    bb.random_fill(dev.data_ptr(), dev.numel(), seed, _stream(torch))
    if not pinned:
        return dev
    host = torch.empty(dev.numel(), dtype=torch.uint8, pin_memory=True)
    host.copy_(dev)
    torch.cuda.synchronize()
    return host


class Store:
    """Host model of the store: what every copy of an object must hold, read back through the worker that owns it."""

    def __init__(self, bb, cl):
        self.bb, self.cl = bb, cl
        self.pools = {p.id: p for p in cl.client.keystone().get_memory_pools()}

    def _where(self, sh):
        be = self.cl.worker.backend(sh.pool_id)
        if sh.location["kind"] == "gpu":
            return be, sh.offset
        return be, sh.location["remote_addr"] - self.pools[sh.pool_id].ucx_remote_addr  # pinned DRAM pool

    def stored(self, sh, pos=0, n=None):
        n = sh.length - pos if n is None else n
        if n == 0:
            return b""
        be, off = self._where(sh)
        return be.read(off + pos, n)

    def flip(self, sh, pos):
        be, off = self._where(sh)
        be.write(off + pos, bytes([be.read(off + pos, 1)[0] ^ 0xFF]))

    def check(self, key, blob, algo, copies):
        """Every copy holds `blob` (a numpy uint8 array) and carries the CPU model's digest of what it holds."""
        placed = self.cl.client.get_workers(key)
        assert len(placed) == copies, (key, len(placed))
        ref = _ref(self.bb, algo)
        for c, cp in enumerate(placed):
            off = 0
            for s, sh in enumerate(cp.shards):
                assert sh.checksum_algo == getattr(self.bb.ChecksumAlgo, algo)
                got = self.stored(sh)
                assert got == blob[off:off + sh.length].tobytes(), (key, c, s)
                assert sh.checksum == ref(np.frombuffer(got, dtype=np.uint8)), (key, c, s)
                off += sh.length
            assert off == blob.size, (key, c)
        return placed


def _host(t):
    return t.cpu().numpy() if t.is_cuda else t.numpy()


def _check_get(torch, out, dsts, src, offs, sizes):
    """`out` holds object i at dsts[i] and the guard byte everywhere else."""
    want = torch.full_like(out, GUARD)
    for d, o, n in zip(dsts, offs, sizes):
        want[d:d + n] = src[o:o + n].to(want.device)
    torch.cuda.synchronize()
    if not torch.equal(out, want):
        bad = (out != want).nonzero()
        raise AssertionError(f"get wrote {bad.numel()} wrong bytes, first at {int(bad[0])}: objects at {dsts}")


def _layout(sizes, align=256, skew=None):
    """Offsets of objects packed back to back at `align`-byte boundaries; skew = {index: extra bytes}."""
    offs, off = [], 0
    for i, n in enumerate(sizes):
        offs.append(off + (skew or {}).get(i, 0))
        off += (n + 16 + align - 1) // align * align + align
    return offs, off


@pytest.mark.parametrize("algo", ALGOS)
def test_replicas_past_the_fan_out_of_one_tile_pass(bb, torch_cuda, algo):
    """Replication 1 to 5 on one slab. One tile pass writes at most kMaxDst (3) copies, so the fabric gives replicas 4 and 5
    an extra pass over the same source: every copy must hold the source and carry its digest. A get whose first-pass
    copies are all corrupt must end on a copy written by the extra pass; with every copy corrupt it reports
    CHECKSUM_MISMATCH for that object only."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-rep-{algo}", max_replicas=5)
    try:
        s = _stream(torch)
        store = Store(bb, cl)
        sizes = [3 * bb.TILE_BYTES + 5, 100000, 4097, 2 * MiB + 48]
        offs, total = _layout(sizes)
        src = _random(torch, total, 11)
        host = _host(src)
        for rep in range(1, 6):
            keys = [f"rep{rep}/{i}" for i in range(len(sizes))]
            l0 = cl.fabric.launches
            ecs = cl.client.batch_put_device(keys, [src.data_ptr() + o for o in offs], sizes, _cfg(bb, algo, rep), s)
            assert ecs == [bb.ErrorCode.OK] * len(sizes), (rep, ecs)
            assert cl.fabric.launches == l0 + 1  # the extra pass is more descriptors in the same launch
            placed = [store.check(k, host[o:o + n], algo, rep) for k, o, n in zip(keys, offs, sizes)]
            out = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
            ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [n + 16 for n in sizes], s)
            assert ecs == [bb.ErrorCode.OK] * len(sizes) and got == sizes, (rep, ecs)
            _check_get(torch, out, offs, src, offs, sizes)
            if algo == "NONE":
                continue
            # corrupt the copies of object 1 that the first tile pass wrote (all but the last when there is no extra pass)
            first_pass = min(rep - 1, 3)
            for c in placed[1][:first_pass]:
                store.flip(c.shards[0], 777 + rep)
            fo = _counter(cl.client, "replica_failover_total")
            out.fill_(GUARD)
            ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [n + 16 for n in sizes], s)
            assert ecs == [bb.ErrorCode.OK] * len(sizes) and got == sizes, (rep, ecs)
            _check_get(torch, out, offs, src, offs, sizes)
            assert _counter(cl.client, "replica_failover_total") == fo + first_pass  # one re-read per corrupt copy
            # every copy corrupt: that object fails, its neighbours do not
            for c in placed[1][first_pass:]:
                store.flip(c.shards[0], 5)
            out.fill_(GUARD)
            ecs, _ = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [n + 16 for n in sizes], s)
            assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH if i == 1 else bb.ErrorCode.OK for i in range(len(sizes))], (rep, ecs)
            rest = [i for i in range(len(sizes)) if i != 1]
            torch.cuda.synchronize()
            for i in rest:
                assert torch.equal(out[offs[i]:offs[i] + sizes[i]], src[offs[i]:offs[i] + sizes[i]]), (rep, i)
            assert cl.client.batch_remove(keys) == [bb.ErrorCode.OK] * len(sizes)
    finally:
        cl.stop()


def _plan(sizes, want, depth=3):
    """The chunk plan of BlackbirdClient::plan_chunks for a forced chunk count (chunks of at least 256 MiB)."""
    total, min_chunk = sum(sizes), 256 * MiB
    if depth < 2 or len(sizes) < 2 or total < 2 * min_chunk:
        return [(0, len(sizes))]
    want = min(want, total // min_chunk, len(sizes))
    if want <= 1:
        return [(0, len(sizes))]
    target, chunks, begin, acc = total // want, [], 0, 0
    for i, n in enumerate(sizes):
        acc += n
        if acc >= target and i + 1 < len(sizes) and len(chunks) + 1 < want:
            chunks.append((begin, i + 1))
            begin, acc = i + 1, 0
    chunks.append((begin, len(sizes)))
    return chunks


def test_chunk_plans_of_uneven_batches(bb, torch_cuda):
    """Forced 2, 3 and 4 chunks on a batch of uneven sizes whose chunk edges fall before, on and after a 420 MiB object:
    one launch per chunk, every object in exactly one chunk with its own digest. A get is planned from its capacities, not
    from the sizes: a batch of small objects read into large buffers is split although its put was not."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=(1 << 30) + (256 << 20), cluster_id="t-chunks")
    try:
        s = _stream(torch)
        store = Store(bb, cl)
        sizes = [150 * MiB + 5, 120 * MiB + 4097, 12 * MiB + 17, 420 * MiB + 3, 150 * MiB, 4097, 200 * MiB + 1, 64 * MiB - 3, 3 * MiB]
        big = 3
        plans = {c: _plan(sizes, c) for c in (2, 3, 4)}
        edges = {e for p in plans.values() for _, e in p[:-1]}
        assert {big, big + 1, big + 4} <= edges and plans[4] == [(0, 3), (3, 4), (4, 7), (7, 9)], plans
        offs, total = _layout(sizes)
        src = _random(torch, total, 23)
        host = _host(src)
        out = torch.empty(total, dtype=torch.uint8, device="cuda")
        for (chunks, plan), algo in zip(plans.items(), ["XXH3", "CRC32C", "BBH64"]):
            keys = [f"ch{chunks}/{i}" for i in range(len(sizes))]
            cl.client.set_device_pipeline_chunks(chunks)
            l0 = cl.fabric.launches
            ecs = cl.client.batch_put_device(keys, [src.data_ptr() + o for o in offs], sizes, _cfg(bb, algo), s)
            assert ecs == [bb.ErrorCode.OK] * len(sizes), (chunks, ecs)
            assert cl.fabric.launches - l0 == len(plan), (chunks, plan)
            for k, o, n in zip(keys, offs, sizes):
                store.check(k, host[o:o + n], algo, 1)
            out.fill_(GUARD)
            l0 = cl.fabric.launches
            ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [n + 16 for n in sizes], s)
            assert ecs == [bb.ErrorCode.OK] * len(sizes) and got == sizes, (chunks, ecs)
            assert cl.fabric.launches - l0 == len(_plan([n + 16 for n in sizes], chunks))
            _check_get(torch, out, offs, src, offs, sizes)
            assert cl.client.batch_remove(keys) == [bb.ErrorCode.OK] * len(sizes)
        del out
        # small objects, large capacities: the put is one launch, the get four
        small = [MiB + 7 * i for i in range(8)]
        caps = [160 * MiB] * 8
        assert _plan(small, 4) == [(0, 8)] and len(_plan(caps, 4)) == 4
        keys = [f"cap/{i}" for i in range(8)]
        cl.client.set_device_pipeline_chunks(4)
        l0 = cl.fabric.launches
        ecs = cl.client.batch_put_device(keys, [src.data_ptr() + i * 2 * MiB for i in range(8)], small, _cfg(bb, "NONE"), s)
        assert ecs == [bb.ErrorCode.OK] * 8 and cl.fabric.launches == l0 + 1, ecs
        for i, k in enumerate(keys):
            store.check(k, host[i * 2 * MiB:i * 2 * MiB + small[i]], "NONE", 1)
        out = torch.full((sum(caps),), GUARD, dtype=torch.uint8, device="cuda")
        dsts = [i * caps[0] for i in range(8)]
        ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + d for d in dsts], caps, s)
        assert ecs == [bb.ErrorCode.OK] * 8 and got == small, ecs
        assert cl.fabric.launches == l0 + 5
        _check_get(torch, out, dsts, src, [i * 2 * MiB for i in range(8)], small)
        cl.client.set_device_pipeline_chunks(0)
    finally:
        cl.stop()


@pytest.mark.parametrize("algo", ALGOS)
def test_engine_thresholds_reached_through_the_client(bb, torch_cuda, algo):
    """Batches of 1, 8, 9, 64 and 65 small objects and objects of 4096 / 4097 bytes: up to 8 objects of <= 4096 bytes go
    to the resident mailbox warp (no launch), more take the warp-per-object kernel, anything larger the TMA kernel. Every
    path stores the same bytes and digests. Zero-length objects are accepted, round-trip, and record the empty digest."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-thr-{algo}")
    try:
        s = _stream(torch)
        store = Store(bb, cl)
        f = cl.fabric
        src = _random(torch, 80 * 8192, 31)
        host = _host(src)
        cases = [  # (sizes, path)
            ([4096], "mailbox"),
            ([1, 17, 4096, 4095, 16, 2000, 3000, 4096], "mailbox"),
            ([4096 - i * 100 for i in range(9)], "small"),
            ([(i * 67) % 4096 + 1 for i in range(63)] + [4096], "small"),
            ([(i * 61) % 4096 + 1 for i in range(64)] + [4096], "small"),
            ([4097], "tma"),
            ([4096] * 4 + [4097] + [4096] * 4, "tma"),
            ([0], "none"),
            ([0, 4096, 0, 17, 0], "mailbox"),
            ([0] + [100] * 8 + [0, 4097], "tma"),
        ]
        for case, (sizes, path) in enumerate(cases):
            n = len(sizes)
            offs = [i * 8192 for i in range(n)]
            keys = [f"thr{case}/{i}" for i in range(n)]
            for direction in ("put", "get"):
                torch.cuda.synchronize()  # the mailbox serves only a caller stream with nothing pending
                l0, sl0, mb0, ml0 = f.launches, f.small_launches, f.mailbox_requests, f.mailbox_launches
                if direction == "put":
                    ecs = cl.client.batch_put_device(keys, [src.data_ptr() + o for o in offs], sizes, _cfg(bb, algo), s)
                    assert ecs == [bb.ErrorCode.OK] * n, (case, ecs)
                else:
                    out = torch.full((n * 8192,), GUARD, dtype=torch.uint8, device="cuda")
                    torch.cuda.synchronize()
                    ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [8192 - 16] * n, s)
                    assert ecs == [bb.ErrorCode.OK] * n and got == sizes, (case, ecs)
                    _check_get(torch, out, offs, src, offs, sizes)
                busy = sum(1 for x in sizes if x)
                # (transfer launches, warp-per-object launches, mailbox requests); the mailbox warp's own (re)launches
                # are not transfer launches
                want = {"mailbox": (0, 0, busy), "small": (1, 1, 0), "tma": (1, 0, 0), "none": (0, 0, 0)}[path]
                ran = (f.launches - l0 - (f.mailbox_launches - ml0), f.small_launches - sl0, f.mailbox_requests - mb0)
                assert ran == want, (case, direction, path)
            for k, o, sz in zip(keys, offs, sizes):
                store.check(k, host[o:o + sz], algo, 1)
            if algo != "NONE" and n > 1:
                # one corrupt object in the batch is reported on its own
                bad = max(range(n), key=lambda i: sizes[i])
                store.flip(cl.client.get_workers(keys[bad])[0].shards[0], sizes[bad] - 1)
                out = torch.full((n * 8192,), GUARD, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                ecs, _ = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [8192 - 16] * n, s)
                assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH if i == bad else bb.ErrorCode.OK for i in range(n)], (case, ecs)
            assert cl.client.batch_remove(keys) == [bb.ErrorCode.OK] * n
    finally:
        cl.stop()


@pytest.mark.parametrize("pinned", [False, True], ids=["device-buffers", "pinned-host-buffers"])
@pytest.mark.parametrize("algo", ALGOS)
def test_hbm_and_dram_tiers_in_one_batch(bb, torch_cuda, algo, pinned):
    """Objects put to this GPU's HBM slab and to a pinned DRAM pool, read back in one batch_get_device by one launch, from
    and into device memory or pinned host memory (as bench.py's zero_copy mode passes them). A corrupt object in each tier
    is reported for that object only."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-tiers-{algo}-{int(pinned)}", dram_bytes=64 << 20)
    try:
        s = _stream(torch)
        sizes = [5000, 3 * bb.TILE_BYTES + 7, 1 * MiB + 48, 4096, 200001, 17, 2 * MiB, 70000]
        tiers = ["RAM_GPU", "RAM_CPU"] * 4
        n = len(sizes)
        offs, total = _layout(sizes)
        src = _random(torch, total, 41, pinned=pinned)
        host = _host(src)
        keys = [f"tier/{i}" for i in range(n)]
        for tier in ("RAM_GPU", "RAM_CPU"):
            idx = [i for i in range(n) if tiers[i] == tier]
            l0 = cl.fabric.launches
            ecs = cl.client.batch_put_device([keys[i] for i in idx], [src.data_ptr() + offs[i] for i in idx], [sizes[i] for i in idx],
                                             _cfg(bb, algo, 1, tier), s)
            assert ecs == [bb.ErrorCode.OK] * len(idx), (tier, ecs)
            assert cl.fabric.launches == l0 + 1
        assert cl.fabric.mapped_host_pools() == 1
        store = Store(bb, cl)
        for i in range(n):
            sh = store.check(keys[i], host[offs[i]:offs[i] + sizes[i]], algo, 1)[0].shards[0]
            assert sh.storage_class == getattr(bb.StorageClass, tiers[i]), i
        out = torch.full((total,), GUARD, dtype=torch.uint8, pin_memory=True) if pinned else torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
        l0 = cl.fabric.launches
        ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [n_ + 16 for n_ in sizes], s)
        assert ecs == [bb.ErrorCode.OK] * n and got == sizes, ecs
        assert cl.fabric.launches == l0 + 1  # both tiers in one launch
        assert _counter(cl.client, "device_get_host_staged_total") == 0
        _check_get(torch, out, offs, src, offs, sizes)
        if algo == "NONE":
            return
        for i in (2, 5):  # one object in HBM, one in DRAM
            store.flip(cl.client.get_workers(keys[i])[0].shards[0], sizes[i] // 2)
        out.fill_(GUARD)
        ecs, _ = cl.client.batch_get_device(keys, [out.data_ptr() + o for o in offs], [n_ + 16 for n_ in sizes], s)
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH if i in (2, 5) else bb.ErrorCode.OK for i in range(n)], ecs
    finally:
        cl.stop()


@pytest.mark.parametrize("algo", ALGOS)
def test_misaligned_caller_pointers_are_staged_without_failing_the_batch(bb, torch_cuda, algo):
    """A put whose object 2 starts 8 bytes past an aligned address, then a get whose object 4 lands 8 bytes past one. The
    fused kernels take 16-byte aligned pointers only: the client stages that object through the host before any launch,
    and its aligned neighbours still take the fused kernel, in one launch. Every object ends with the right bytes and
    digest, as on the CPU transport (tests/test_device_api_cpu.py)."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id=f"t-align-{algo}")
    try:
        s = _stream(torch)
        store = Store(bb, cl)
        sizes = [100000, 5000, 70001, 2 * MiB + 3, 4096, 300]
        n = len(sizes)
        offs, total = _layout(sizes, skew={2: 8})
        src = _random(torch, total, 53)
        host = _host(src)
        keys = [f"al/{i}" for i in range(n)]
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_put_host_staged_total")
        ecs = cl.client.batch_put_device(keys, [src.data_ptr() + o for o in offs], sizes, _cfg(bb, algo, 2), s)
        assert ecs == [bb.ErrorCode.OK] * n, ecs
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_put_host_staged_total") == st0 + 1
        for k, o, sz in zip(keys, offs, sizes):
            store.check(k, host[o:o + sz], algo, 2)
        dsts, dtotal = _layout(sizes, skew={4: 8})
        out = torch.full((dtotal,), GUARD, dtype=torch.uint8, device="cuda")
        l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
        ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + d for d in dsts], [sz + 8 for sz in sizes], s)
        assert ecs == [bb.ErrorCode.OK] * n and got == sizes, ecs
        assert cl.fabric.launches == l0 + 1 and _counter(cl.client, "device_get_host_staged_total") == st0 + 1
        _check_get(torch, out, dsts, src, offs, sizes)
        if algo == "NONE":
            return
        # the staged get verifies on the CPU and fails over between replicas like the fused one
        store.flip(cl.client.get_workers(keys[4])[0].shards[0], 100)
        store.flip(cl.client.get_workers(keys[0])[0].shards[0], 100)
        out.fill_(GUARD)
        ecs, got = cl.client.batch_get_device(keys, [out.data_ptr() + d for d in dsts], [sz + 8 for sz in sizes], s)
        assert ecs == [bb.ErrorCode.OK] * n and got == sizes, ecs
        _check_get(torch, out, dsts, src, offs, sizes)
    finally:
        cl.stop()


BIG = (1 << 32) + 16385  # more than 2^18 tiles: byte offsets and tile counts past 32 bits


def _timed(fn, blob):
    t0 = time.perf_counter()
    v = fn(blob)
    return v, time.perf_counter() - t0


def test_engine_object_past_4_gib(bb, torch_cuda):
    """One object of 2^32 + 16385 bytes through XferEngine.run for every algorithm: the digest equals the CPU model, every
    byte lands, nothing is written past the object, and verification passes and fails as it should."""
    torch = torch_cuda
    eng = bb.XferEngine(0, 64, 2)
    s = _stream(torch)
    src = _random(torch, BIG, 61)
    dst = torch.full((BIG + 4096,), GUARD, dtype=torch.uint8, device="cuda")
    host = _host(src)
    try:
        for algo in ALGOS:
            dg, st, _ = eng.run([(src.data_ptr(), dst.data_ptr(), BIG)], getattr(bb.ChecksumAlgo, algo), s)
            torch.cuda.synchronize()
            want, secs = _timed(_ref(bb, algo), host)
            print(f"\n{algo}: CPU model of {BIG} bytes took {secs:.2f} s")
            assert st == [0] and (algo == "NONE" or dg[0] == want), algo
            assert torch.equal(dst[:BIG], src) and bool((dst[BIG:] == GUARD).all()), algo
            if algo != "NONE":
                for expect, status in ((want, 0), (want ^ (1 << 20), 1)):
                    _, st, _ = eng.run([(src.data_ptr(), dst.data_ptr(), BIG, expect, bb.XFER_VERIFY)], getattr(bb.ChecksumAlgo, algo), s)
                    assert st == [status], algo
            dst[:BIG].fill_(0)
    finally:
        del src, dst, host
        torch.cuda.empty_cache()


def test_client_object_past_4_gib(bb, torch_cuda):
    """One object of 2^32 + 16385 bytes put and got through the client at replication 1, for every algorithm: stored bytes,
    recorded digest, get result and guard bytes; a flipped byte past the first 4 GiB is caught by the get."""
    torch = torch_cuda
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=(1 << 32) + (64 << 20), cluster_id="t-4g")
    src = out = host = None
    try:
        s = _stream(torch)
        store = Store(bb, cl)
        src = _random(torch, BIG, 67)
        host = _host(src)
        out = torch.empty(BIG + 4096, dtype=torch.uint8, device="cuda")
        step = 256 * MiB
        for algo in ALGOS:
            key = f"big/{algo}"
            assert cl.client.batch_put_device([key], [src.data_ptr()], [BIG], _cfg(bb, algo), s) == [bb.ErrorCode.OK]
            sh = cl.client.get_workers(key)[0].shards
            assert [x.length for x in sh] == [BIG]
            sh = sh[0]
            for pos in range(0, BIG, step):
                assert store.stored(sh, pos, min(step, BIG - pos)) == host[pos:pos + step].tobytes(), (algo, pos)
            want, secs = _timed(_ref(bb, algo), host)
            print(f"\n{algo}: CPU model of {BIG} bytes took {secs:.2f} s")
            assert sh.checksum == want, algo
            out.fill_(GUARD)
            ecs, got = cl.client.batch_get_device([key], [out.data_ptr()], [BIG + 4096], s)
            assert ecs == [bb.ErrorCode.OK] and got == [BIG], (algo, ecs)
            torch.cuda.synchronize()
            assert torch.equal(out[:BIG], src) and bool((out[BIG:] == GUARD).all()), algo
            if algo != "NONE":
                store.flip(sh, BIG - 3)
                ecs, _ = cl.client.batch_get_device([key], [out.data_ptr()], [BIG + 4096], s)
                assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH], algo
            assert cl.client.batch_remove([key]) == [bb.ErrorCode.OK]
    finally:
        del src, out, host
        cl.stop()
        torch.cuda.empty_cache()
