"""Paged puts and gets on the GPU: the paged gathering load and scattering store of bb_xfer (XFER_PAGED) through
XferEngine, the client's batch_put_device_paged / batch_get_device_paged on a GpuRankCluster, and TensorStore's block
puts and gets.  A paged descriptor reads or stores its object's bytes in pages at arbitrary addresses; the tile in shared
memory is the dense object's, so every check covers the pages, the guard bytes around and between them, and the digest,
which must equal that of a plain transfer of the concatenated pages."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
ALGOS = ["NONE", "CRC32C", "BBH64", "XXH3"]
GRIDS = [1, 7, "sms", "2sms"]


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")


@pytest.fixture(scope="module")
def _engine():
    from blackbird_b200 import _bb

    return _bb.XferEngine(0, 4096, 2)


@pytest.fixture
def eng(_engine):
    yield _engine
    _engine.set_max_ctas(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _grid(g):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"sms": sms, "2sms": 2 * sms}.get(g, g)


def _model(bb, algo):
    return {"NONE": lambda b: 0, "CRC32C": bb.crc32c, "BBH64": bb.bbh64, "XXH3": bb.xxh3t64}[algo]


def _random(bb, n, seed):
    t = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    bb.random_fill(t.data_ptr(), t.numel(), seed, _stream())
    return t


def rows_index(n, pitch, width, phase):
    y = np.arange(n, dtype=np.int64) + phase
    return y // width * pitch + y % width


def pages_index(n, addrs, page, phase):
    """Where each object byte lives: the rule of SourcePages."""
    y = np.arange(n, dtype=np.int64) + phase
    return np.asarray(addrs, dtype=np.int64)[y // page] + y % page


class Carver:
    """Hands out regions of one buffer, each after a guard gap: pages in random order, each placed so that addr + phase
    is 16-byte aligned (SourcePages::coaligned)."""

    def __init__(self, rng):
        self.o, self.rng = 64, rng

    def region(self, n, align_at=0):
        self.o = (self.o + 15) // 16 * 16 + (16 - align_at % 16) % 16
        at = self.o
        self.o += n + 48
        return at

    def pages(self, npages, page, phase):
        slots = [self.region(page + 16) for _ in range(npages)]
        return [slots[i] + (16 - phase % 16) % 16 for i in self.rng.permutation(npages)]


class Batch:
    """One launch mixing paged puts and gets with plain, windowed, gathered and scattered items.  A spec is (kind, nbytes,
    arg): pput / pget (page, phase) | plain None | window (lo, hi) | gather (pitch, width, phase) | scatter (pitch, width,
    phase).  Sources are regions of one random buffer, destinations regions of one guard-filled buffer."""

    def __init__(self, bb, specs, algo, seed=11):
        rng = np.random.default_rng(seed)
        src_c, dst_c = Carver(rng), Carver(rng)
        self.specs, src_ix, dst_at, extra = specs, [], [], []
        for kind, n, arg in specs:
            if kind == "pput":
                page, phase = arg
                addrs = src_c.pages(max(1, (n - 1 + phase) // page + 1), page, phase)
                src_ix.append(pages_index(n, addrs, page, phase))
                dst_at.append(dst_c.region(n) + np.arange(n))
                extra.append(addrs)
            elif kind == "pget":
                page, phase = arg
                src_ix.append(src_c.region(n) + np.arange(n))
                addrs = dst_c.pages(max(1, (n - 1 + phase) // page + 1), page, phase)
                dst_at.append(pages_index(n, addrs, page, phase))
                extra.append(addrs)
            elif kind == "gather":
                src_ix.append(src_c.region(int(rows_index(n, *arg).max()) + 1, arg[2]) + rows_index(n, *arg))
                dst_at.append(dst_c.region(n) + np.arange(n))
                extra.append(None)
            elif kind == "scatter":
                src_ix.append(src_c.region(n) + np.arange(n))
                r = dst_c.region(int(rows_index(n, *arg).max()) + 1, arg[2])
                dst_at.append(r + rows_index(n, *arg))
                extra.append(r)
            elif kind == "window":
                lo, hi = arg
                src_ix.append(src_c.region(n) + np.arange(n))
                r = dst_c.region(hi - lo, -lo)  # the virtual base r - lo is 16-byte aligned
                dst_at.append(r + np.arange(hi - lo))
                extra.append(r)
            else:
                src_ix.append(src_c.region(n) + np.arange(n))
                dst_at.append(dst_c.region(n) + np.arange(n))
                extra.append(None)
        self.src = _random(bb, src_c.o + 64, seed)
        host = self.src.cpu().numpy()
        self.objs = [host[ix] for ix in src_ix]
        self.digests = [_model(bb, algo)(o.tobytes()) for o in self.objs]
        self.dst = torch.full((dst_c.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        self.stored = [np.arange(n) if kind != "window" else np.arange(*arg) for kind, n, arg in specs]
        self.dst_at = dst_at
        verify = 0 if algo == "NONE" else bb.XFER_VERIFY
        S, D = self.src.data_ptr(), self.dst.data_ptr()
        self.items = []
        for (kind, n, arg), six, dat, ex, dg in zip(specs, src_ix, dst_at, extra, self.digests):
            if kind == "pput":
                it = (0, D + int(dat[0]) if n else D, n, dg, 0, 0, None, None, None, ([S + a for a in ex], arg[0], arg[1]))
            elif kind == "pget":
                it = (S + int(six[0]) if n else S, 0, n, dg, verify, 0, None, None, None, None, ([D + a for a in ex], arg[0], arg[1]))
            elif kind == "gather":
                it = (S + int(six[0]) - arg[2], D + int(dat[0]), n, dg, 0, 0, None, arg)
            elif kind == "scatter":
                it = (S + int(six[0]), D + ex, n, dg, verify, 0, None, None, arg)
            elif kind == "window":
                it = (S + int(six[0]), D + ex - arg[0], n, dg, verify, 0, arg)
            else:
                it = (S + int(six[0]), D + int(dat[0]), n, dg, verify)
            self.items.append(it)

    def check(self, what):
        torch.cuda.synchronize()
        want = np.full(self.dst.numel(), GUARD, dtype=np.uint8)
        for obj, at, st in zip(self.objs, self.dst_at, self.stored):
            want[at] = obj[st]
        got = self.dst.cpu().numpy()
        if not np.array_equal(got, want):
            pytest.fail(f"{what}: bytes differ at {np.nonzero(got != want)[0][:8].tolist()}")


def paged_specs():
    """Pages of 16, 48, 4 KiB, 16 KiB + 16 and 3 MiB; one-page items; nonzero phases; tiles of more than 32 pages (a 16 KiB
    tile holds 1024 pages of 16 bytes, 341 of 48); objects that end mid-page."""
    out = []
    for kind in ("pput", "pget"):
        out += [(kind, 3 * T + 16, (16, 0)), (kind, 2 * T + 5, (48, 0)), (kind, 5 * 4096, (4096, 0)), (kind, 4 * (T + 16) - 9, (T + 16, 0)),
                (kind, 7 * MiB + 100, (3 * MiB, 0)), (kind, 4096, (4096, 0)), (kind, 77, (4096, 0)), (kind, 3 * T, (4096, 1000)),
                (kind, 200 * 48 - 40, (48, 32)), (kind, 1, (16, 3))]
    return out


@pytest.mark.parametrize("algo", ALGOS)
def test_paged_items_at_every_grid(bb, eng, algo):
    """Every paged shape in one device-table batch with plain, windowed, gathered and scattered items mixed in, at grids of
    1, 7, the SM count and twice the SM count: the pages and destinations equal the objects, every guard byte is intact,
    the digests equal the CPU model of the dense object (a plain put of the concatenation), and a wrong expected digest
    on a paged get gives status 1."""
    A = getattr(bb.ChecksumAlgo, algo)
    specs = paged_specs() + [("plain", 3 * T + 7, None), ("window", 2 * T + 9, (100, T + 333)), ("gather", 2 * T + 1, (48, 32, 5)),
                             ("scatter", 3 * T + 5, (4016, 4000, 123))]
    b = Batch(bb, specs, algo)
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        b.dst.fill_(GUARD)
        dg, st, _ = eng.run(b.items, A, _stream())
        assert st == [0] * len(specs), (g, st)
        if algo != "NONE":
            assert dg == b.digests, g
        b.check(f"{algo} grid={g}")
    eng.set_max_ctas(0)
    if algo != "NONE":
        bad = [it[:3] + (it[3] ^ 1,) + it[4:] if k == "pget" else it for it, (k, _, _) in zip(b.items, specs)]
        _, st, _ = eng.run(bad, A, _stream())
        assert st == [1 if k == "pget" else 0 for k, _, _ in specs]


def test_paged_puts_fan_out_and_small_items_take_the_fused_kernel(bb, eng):
    """A paged put writes 1-3 destinations in one tile pass; batches of <= 8 descriptors and objects of <= 4 KiB that are
    paged never take the inline parameters' path, the warp-per-object kernel or the mailbox, and occupancy is unchanged."""
    rng = np.random.default_rng(2)
    src = _random(bb, 64 * 4096, 9)
    host = src.cpu().numpy()
    slots = [int(s) * 4096 for s in rng.permutation(64)[:3]]
    obj = np.concatenate([host[s:s + 4096] for s in slots])[:3 * 4096 - 100]
    n = obj.size
    dst = torch.full((3, (n + 64 + 15) // 16 * 16), GUARD, dtype=torch.uint8, device="cuda")  # 16-byte aligned rows
    pages = ([src.data_ptr() + s for s in slots], 4096, 0)
    sl, mb, la = eng.small_launches, eng.mailbox_requests, eng.launches
    dg, st, _ = eng.run([(0, [dst[r].data_ptr() for r in range(3)], n, 0, 0, 0, None, None, None, pages)], bb.ChecksumAlgo.XXH3, _stream())
    assert dg == [bb.xxh3t64(obj.tobytes())] and st == [0]
    torch.cuda.synchronize()
    for r in range(3):
        got = dst[r].cpu().numpy()
        assert np.array_equal(got[:n], obj) and bool((got[n:] == GUARD).all())
    b = Batch(bb, [("pput", 4096, (48, 16)), ("pget", 100, (16, 0)), ("pget", 1, (4096, 5)), ("plain", 64, None)], "XXH3", seed=4)
    dg, st, _ = eng.run(b.items, bb.ChecksumAlgo.XXH3, _stream())
    assert st == [0] * 4 and dg == b.digests
    b.check("small")
    assert eng.small_launches == sl and eng.mailbox_requests == mb and eng.launches == la + 2
    for algo in ALGOS:
        assert bb.xfer_geometry(getattr(bb.ChecksumAlgo, algo), 10000)["resident_ctas_per_sm"] == (1 if algo == "CRC32C" else 2), algo


def test_rejected_paged_items(bb, eng):
    """Forbidden combinations and misaligned pages are refused before any launch, and nothing is written."""
    src = _random(bb, 8 * T, 1)
    dst = torch.full((8 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    sp = ([s, s + 2 * T, s + T], 4096, 0)
    dp = ([d + 4 * T, d, d + 2 * T], 4096, 0)
    pat = (96, 80, 0)
    E = "INVALID_ARGUMENT"
    bad = [((s, d, 1000, 0, bb.XFER_PAGED), E),                                                  # flag without pages
           ((0, d, 1000, 0, 0, 0, (0, 500), None, None, sp), E),                                 # with a window
           ((0, d, 1000, 0, 0, 0, (0, 1000, 96, 80, 0), None, None, sp), E),                     # with a strided window
           ((s, [], 1000, 0, bb.XFER_RAW_SUM, 0, None, None, None, sp), E),                      # with RAW_SUM
           ((s, d, 1000, 0, 0, 0, None, pat, None, sp), E),                                      # with source rows
           ((0, 0, 1000, 0, 0, 0, None, None, None, sp, dp), E),                                 # both sides paged
           ((0, d, 3 * 4096 + 1, 0, 0, 0, None, None, None, sp), E),                             # table too short
           ((0, d, 3 * 4096 - 100, 0, 0, 0, None, None, None, (sp[0], 4096, 200)), E),           # too short with the phase
           ((0, d, 100, 0, 0, 0, None, None, None, (sp[0], 4096, 4096)), E),                     # phase >= page
           ((0, d, 1000, 0, 0, 0, None, None, None, (sp[0], 0, 0)), E),                          # page 0
           ((s, 0, 1000, 0, 0, 0, None, None, pat, None, dp), E),                                # with destination rows
           ((s, [d, d + T], 1000, 0, 0, 0, None, None, None, None, dp), E),                      # get: two destinations
           ((s, d, 1008, 0, bb.XFER_MULTIMEM, 0, None, None, None, None, dp), E),                # get: multicast
           ((0, d, 5000, 0, 0, 0, None, None, None, ([s + 8, s + T], 4096, 0)), "INVALID_ADDRESS"),     # first page
           ((0, d, 5000, 0, 0, 0, None, None, None, ([s, s + T + 4], 4096, 0)), "INVALID_ADDRESS"),     # later page
           ((0, d, 5000, 0, 0, 0, None, None, None, ([s, s + T], 4008, 0)), "INVALID_ADDRESS"),         # page % 16
           ((0, d, 3000, 0, 0, 0, None, None, None, ([s], 4096, 7)), "INVALID_ADDRESS"),                # first page + phase
           ((0, d, 5000, 0, 0, 0, None, None, None, ([s - 8, s + T], 4096, 8)), "INVALID_ADDRESS"),     # later page + phase
           ((s, 0, 5000, 0, 0, 0, None, None, None, None, ([d, d + T + 8], 4096, 0)), "INVALID_ADDRESS")]
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([(s, d + 6 * T, 64, 0, 0), it], A, _stream())  # the valid neighbour is not written either
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all())
    # one page of any size is fine, and a single page only needs addrs[0] + phase aligned
    eng.run([(0, d, 3000, 0, 0, 0, None, None, None, ([s - 7], 4001, 7))], A, _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst[:3000], src[:3000]) and bool((dst[3000:] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- client
def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


@pytest.mark.parametrize("algo", ["XXH3", "CRC32C"])
def test_client_paged_puts_and_gets(bb, algo):
    """Objects replicated in HBM, in a pinned DRAM pool and striped over both (shard edges mid-page): the fused items of
    one call go in one launch, a misaligned item is staged alone; the stored object is the concatenation; paged gets
    fill the pages and nothing else; a corrupt replica fails over; a re-read after compact_pool still lands right."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id=f"t-paged-{algo}", dram_bytes=64 << 20, max_replicas=3)
    try:
        A = getattr(bb.ChecksumAlgo, algo)
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096, checksum=A,
                                  preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        hbm = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_GPU])
        dram = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_CPU])
        rng = np.random.default_rng(8)
        hole = _random(bb, 4 * MiB, 20)  # removed before compact_pool, which then moves the paged objects into its space
        assert cl.client.batch_put_device(["hole"], [hole.data_ptr()], [hole.numel()], hbm, _stream()) == [bb.ErrorCode.OK]
        cache = _random(bb, 32 << 20, 21)
        host = cache.cpu().numpy()
        # (cfg, page, pages, skew)
        shapes = [(striped, 32768 + 48, 40, 0), (hbm, 4096, 100, 0), (dram, T + 16, 17, 0), (hbm, 4096, 9, 8)]
        free = list(rng.permutation((32 << 20) // (64 * 1024)))
        keys, lists, objs = [], [], []
        for k, (cfg, page, npg, skew) in enumerate(shapes):
            offs = [int(free.pop()) * 64 * 1024 + skew for _ in range(npg)]
            keys.append(f"pg{k}")
            lists.append([cache.data_ptr() + o for o in offs])
            objs.append(np.concatenate([host[o:o + page] for o in offs]))
            stp0 = _counter(cl.client, "device_put_host_staged_total")
            assert cl.client.batch_put_device_paged([keys[-1]], [lists[-1]], [page], cfg, _stream()) == [bb.ErrorCode.OK]
            assert _counter(cl.client, "device_put_host_staged_total") == stp0 + (1 if skew else 0)
            out = torch.empty(objs[-1].size, dtype=torch.uint8, device="cuda")
            ecs, sizes = cl.client.batch_get_device([keys[-1]], [out.data_ptr()], [out.numel()], _stream())
            assert ecs == [bb.ErrorCode.OK] and sizes == [objs[-1].size]
            assert np.array_equal(out.cpu().numpy(), objs[-1]), k
        # gets into fresh pages of a guard-filled cache, all in one call
        dstc = torch.full((32 << 20,), GUARD, dtype=torch.uint8, device="cuda")
        free = list(rng.permutation((32 << 20) // (64 * 1024)))
        doffs = [[int(free.pop()) * 64 * 1024 + sk for _ in range(npg)] for _, _, npg, sk in shapes]
        want = np.full(dstc.numel(), GUARD, dtype=np.uint8)
        for o, (_, page, _, _), obj in zip(doffs, shapes, objs):
            want[pages_index(obj.size, o, page, 0)] = obj

        def get_all():
            dstc.fill_(GUARD)
            l0, st0 = cl.fabric.launches, _counter(cl.client, "device_get_host_staged_total")
            ecs, sizes = cl.client.batch_get_device_paged(keys, [[dstc.data_ptr() + a for a in o] for o in doffs], [s[1] for s in shapes],
                                                          _stream())
            assert ecs == [bb.ErrorCode.OK] * len(keys), ecs
            assert sizes == [o.size for o in objs]
            assert _counter(cl.client, "device_get_host_staged_total") == st0 + 1  # the skewed pages only
            assert cl.fabric.launches > l0
            torch.cuda.synchronize()
            got = dstc.cpu().numpy()
            assert np.array_equal(got, want), np.nonzero(got != want)[0][:8]

        get_all()
        # a corrupt HBM replica of pg1: the get fails over to the other copy
        store_pools = {p.id: p for p in cl.client.keystone().get_memory_pools()}
        sh = cl.client.get_workers("pg1")[0].shards[0]
        be = cl.worker.backend(sh.pool_id)
        off = sh.offset if sh.location["kind"] == "gpu" else sh.location["remote_addr"] - store_pools[sh.pool_id].ucx_remote_addr
        be.write(off + 1234, bytes([be.read(off + 1234, 1)[0] ^ 0xFF]))
        fo = _counter(cl.client, "replica_failover_total") + _counter(cl.client, "checksum_mismatch_total")
        get_all()
        assert _counter(cl.client, "replica_failover_total") + _counter(cl.client, "checksum_mismatch_total") > fo
        be.write(off + 1234, bytes([be.read(off + 1234, 1)[0] ^ 0xFF]))
        # compaction moves objects into the hole a removal leaves; the paged get reads their new placements
        before = cl.client.get_workers("pg1")[0].shards[0].offset
        assert cl.client.batch_remove(["hole"]) == [bb.ErrorCode.OK]
        assert cl.client.keystone().compact_pool(sh.pool_id) > 0
        assert cl.client.get_workers("pg1")[0].shards[0].offset != before
        get_all()
        E = bb.ErrorCode
        ecs, _ = cl.client.batch_get_device_paged(["pg1", "pg1", "pg1"], [[dstc.data_ptr()] * 99, [dstc.data_ptr()], []], [4096, 0, 4096],
                                                  _stream())
        assert ecs == [E.BUFFER_OVERFLOW, E.INVALID_ARGUMENT, E.BUFFER_OVERFLOW], ecs
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore
def _cache(dtype, shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dtype.is_floating_point:
        return torch.randn(shape, generator=g, device="cuda").to(dtype)
    return torch.randint(-128, 127, shape, generator=g, device="cuda").to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32, torch.int8])
def test_tensor_store_blocks(bb, dtype, monkeypatch):
    """put_blocks equals index_select and get_blocks_into equals index_copy_ over the whole sentinel-filled cache, for
    caches shaped [L, 2, NB, 16, 8, 128] along dims 0, 1 and 2, through the paged calls; the stored tensors interoperate
    with get, get_rows and get_slice."""
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    from blackbird_b200.ops import tensor_store

    monkeypatch.setattr(tensor_store, "PAGED_MIN_PAGE_BYTES", 0)  # the paged calls at every page size of these shapes
    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-paged-ts-{str(dtype)[6:]}")
    try:
        store = TensorStore(cl.client)
        cache = _cache(dtype, (4, 2, 32, 16, 8, 128), 3)
        rng = np.random.default_rng(4)
        put0 = _counter(cl.client, "device_put_paged_total")
        get0 = _counter(cl.client, "device_get_paged_total")
        st0 = [_counter(cl.client, f"device_{op}_host_staged_total") for op in ("put", "get")]
        for dim, ids in ((0, [3, 1]), (1, [1, 0]), (2, list(rng.permutation(32)[:7])), (2, torch.tensor([5, 30, 2], device="cuda"))):
            key = f"b{dim}-{len(ids)}"
            store.put_blocks(key, cache, ids, dim=dim)
            idx = torch.as_tensor(ids if not isinstance(ids, torch.Tensor) else ids.cpu(), dtype=torch.int64, device="cuda")
            sel = cache.index_select(dim, idx)
            assert torch.equal(store.get(key), sel)
            assert torch.equal(store.get_rows(key, 0, 1), sel[0:1])
            assert torch.equal(store.get_slice(key, 3, 2, 9), sel.narrow(3, 2, 7).contiguous())
            # back into other blocks of a sentinel-filled cache
            dst = torch.full_like(cache, 7)
            perm = rng.permutation(cache.shape[dim])[:len(ids)]
            store.get_blocks_into(key, dst, list(perm), dim=dim)
            want = torch.full_like(cache, 7).index_copy_(dim, torch.as_tensor(perm, dtype=torch.int64, device="cuda"), sel)
            assert torch.equal(dst, want), (dim, ids)
        assert _counter(cl.client, "device_put_paged_total") == put0 + 4
        assert _counter(cl.client, "device_get_paged_total") == get0 + 4
        # and every one of them took the fused kernel: nothing was staged through the host
        assert [_counter(cl.client, f"device_{op}_host_staged_total") for op in ("put", "get")] == st0
    finally:
        cl.stop()


def test_tensor_store_block_fallbacks_and_errors(bb):
    """Non-contiguous pages, odd page sizes and pack_fp8 take index_select / index_copy_ with the same results; every error
    is raised before any transfer; the async forms order themselves after the caller's stream."""
    from blackbird_b200.ops.tensor_store import AsyncTensorStore, TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-paged-ts-fb")
    try:
        store = TensorStore(cl.client)
        put0 = _counter(cl.client, "device_put_paged_total")
        base = _cache(torch.bfloat16, (4, 2, 32, 16, 8, 128), 5)
        cases = [("nc", base[:, :, :, :, :4], 2),               # pages are not one contiguous block
                 ("odd", _cache(torch.int8, (3, 20, 7, 5), 6), 1),  # 35-byte pages
                 ("tr", base.transpose(0, 2), 0)]                # a transposed cache
        for key, cache, dim in cases:
            ids = [2, 0, 1]
            store.put_blocks(key, cache, ids, dim=dim)
            sel = cache.index_select(dim, torch.tensor(ids, device="cuda"))
            assert torch.equal(store.get(key), sel)
            dst = torch.full_like(cache, 3)
            store.get_blocks_into(key, dst, [1, 2, 0], dim=dim)
            assert torch.equal(dst, torch.full_like(cache, 3).index_copy_(dim, torch.tensor([1, 2, 0], device="cuda"), sel))
        store.put_blocks("fp8", base, [4, 9], dim=2, pack_fp8=True)
        got = store.get("fp8")
        assert got.shape == base.index_select(2, torch.tensor([4, 9], device="cuda")).shape and got.dtype == torch.bfloat16
        dst = torch.zeros_like(base)
        store.get_blocks_into("fp8", dst, [0, 1], dim=2)
        assert torch.equal(dst.index_select(2, torch.tensor([0, 1], device="cuda")), got)
        assert bool((dst[:, :, 2:] == 0).all())
        assert _counter(cl.client, "device_put_paged_total") == put0  # none of these took the paged call
        # errors, before any transfer
        store.put_blocks("e", base, [1, 2], dim=2)
        dst = torch.full_like(base, 9)
        for args, exc in [(("missing", dst, [0, 1], 2), KeyError), (("e", dst.float(), [0, 1], 2), TypeError),
                          (("e", dst, [0, 1, 2], 2), ValueError), (("e", dst.cpu(), [0, 1], 2), ValueError),
                          (("e", dst, [1, 1], 2), ValueError), (("e", dst, [0, 32], 2), IndexError), (("e", dst, [0, 1], 1), ValueError)]:
            with pytest.raises(exc):
                store.get_blocks_into(*args[:3], dim=args[3])
        assert bool((dst == 9).all())
        for bad_dim in (6, -7):  # out of range, as index_select would say: never wrapped
            with pytest.raises(IndexError):
                store.put_blocks("never", base, [0, 1], dim=bad_dim)
            with pytest.raises(IndexError):
                store.get_blocks_into("e", dst, [0, 1], dim=bad_dim)
        # an expanded cache (stride-0 outer dim) is never paged: a get into it would write overlapping pages
        exp = base[:1].expand(4, *base.shape[1:])
        assert TensorStore._block_pages(exp, 2, np.array([0, 1])) is None
        assert TensorStore._block_pages(base, 2, np.array([0, 1])) is not None
        store.put_blocks("exp", exp, [5, 6], dim=2)
        assert torch.equal(store.get("exp"), exp.index_select(2, torch.tensor([5, 6], device="cuda")))
        # pages below PAGED_MIN_PAGE_BYTES (16 KiB here) take index_select, with the same result
        small = _cache(torch.int8, (4, 2, 32, 16, 8, 128), 7)
        store.put_blocks("small", small, [3, 9], dim=2)
        assert torch.equal(store.get("small"), small.index_select(2, torch.tensor([3, 9], device="cuda")))
        assert _counter(cl.client, "device_put_paged_total") == put0 + 1  # only "e" above
        with pytest.raises(IndexError):
            store.put_blocks("never", base, [0, 40], dim=2)
        assert not cl.client.object_exists("never") and not cl.client.object_exists("never#meta")
        # async: the side stream waits for the caller's writes to the cache, and the caller's later reads see the get
        astore = AsyncTensorStore(cl.client)
        try:
            src = torch.zeros_like(base)
            torch.cuda._sleep(20_000_000)
            src.copy_(base)
            astore.put_blocks_async(["a"], [src], [[3, 7]], dim=2).result()
            out = torch.full_like(base, 1)
            res = astore.get_blocks_into_async(["a"], [out], [[0, 5]], dim=2).result()
            assert res[0] is out
            sel = base.index_select(2, torch.tensor([3, 7], device="cuda"))
            assert torch.equal(out, torch.full_like(base, 1).index_copy_(2, torch.tensor([0, 5], device="cuda"), sel))
        finally:
            astore.close()
    finally:
        cl.stop()
