"""Partial restores of paged objects on the GPU: a page-table entry of 0 is a page the paged scattering store of bb_xfer
and of the fused unpack does not store (SourcePages' null page).  Every check snapshots the whole destination buffer:
bytes change only in the stored pages, and the digest and verify status are those of the dense get, because the whole
object is still read and hashed.  Then the client on a GpuRankCluster (HBM and DRAM tiers), and
TensorStore.get_blocks_into(..., blocks=...) against index_copy_ of index_select, on both routes."""
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


def _carve(rng, npages, page, phase, at):
    """Offsets of npages pages after `at`, each after a guard gap and with offset + phase 16-byte aligned, shuffled; and
    the next free offset."""
    slots = []
    for _ in range(npages):
        at = (at + 15) // 16 * 16 + 48
        slots.append(at + (16 - phase % 16) % 16)
        at = slots[-1] + page
    return [slots[i] for i in rng.permutation(npages)], at + 64


def _masks(rng, n):
    """Which pages are stored: a prefix, a random subset, one page, none, every page."""
    return [np.arange(n) < int(rng.integers(1, n + 1)), rng.random(n) < 0.5, np.arange(n) == int(rng.integers(0, n)), np.zeros(n, bool),
            np.ones(n, bool)]


# (n bytes, page, phase): short last tiles, pages that straddle tiles, tiles of hundreds of pages, a nonzero phase, one page
SHAPES = [(3 * T + 16, 16, 0), (2 * T + 5, 48, 0), (5 * 4096, 4096, 0), (4 * (T + 16) - 9, T + 16, 0), (3 * T, 4096, 1000),
          (7 * MiB + 100, 3 * MiB, 0), (77, 4096, 0)]


@pytest.mark.parametrize("algo", ALGOS)
def test_sparse_scattering_gets_at_every_grid(bb, eng, algo):
    """A batch of paged gets with random null pages at every grid: the stored pages hold the object, every other byte of
    the buffer is untouched, and digest and status equal those of the same batch with dense tables; a wrong expected
    digest gives status 1 even when no page is stored."""
    A = getattr(bb.ChecksumAlgo, algo)
    rng = np.random.default_rng(31)
    verify = 0 if algo == "NONE" else bb.XFER_VERIFY
    src_off, o = [], 64
    for n, _, _ in SHAPES:
        src_off.append(o)
        o = (o + n + 64 + 15) // 16 * 16
    src = _random(bb, o, 7)
    host = src.cpu().numpy()
    objs = [host[s:s + n] for s, (n, _, _) in zip(src_off, SHAPES)]
    digests = [_model(bb, algo)(x.tobytes()) for x in objs]
    at, offs = 64, []
    for n, page, phase in SHAPES:
        p, at = _carve(rng, (n - 1 + phase) // page + 1, page, phase, at)
        offs.append(p)
    dst = torch.full((at,), GUARD, dtype=torch.uint8, device="cuda")
    D = dst.data_ptr()

    def items(masks, expect=None):
        return [(src.data_ptr() + s, 0, n, dg if expect is None else expect, verify, 0, None, None, None, None,
                 ([D + a if keep else 0 for a, keep in zip(p, m)], page, phase))
                for s, (n, page, phase), dg, p, m in zip(src_off, SHAPES, digests, offs, masks)]

    def want(masks):
        w = np.full(dst.numel(), GUARD, dtype=np.uint8)
        for obj, (n, page, phase), p, m in zip(objs, SHAPES, offs, masks):
            y = np.arange(n) + phase
            k = y // page
            keep = m[k]
            w[(np.asarray(p, dtype=np.int64)[k] + y % page)[keep]] = obj[keep]
        return w

    dense = [np.ones(len(p), bool) for p in offs]
    dg0, st0, _ = eng.run(items(dense), A, _stream())
    assert st0 == [0] * len(SHAPES)
    if algo != "NONE":
        assert dg0 == digests
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        for j in range(5):
            masks = [_masks(rng, len(p))[j] for p in offs]
            dst.fill_(GUARD)
            dg, st, _ = eng.run(items(masks), A, _stream())
            assert (dg, st) == (dg0, st0), (g, j)
            torch.cuda.synchronize()
            got = dst.cpu().numpy()
            bad = np.nonzero(got != want(masks))[0]
            assert bad.size == 0, (algo, g, j, bad[:8].tolist())
    eng.set_max_ctas(0)
    if algo != "NONE":
        none = [np.zeros(len(p), bool) for p in offs]
        dst.fill_(GUARD)
        _, st, _ = eng.run([it[:3] + (it[3] ^ 1,) + it[4:] for it in items(none)], A, _stream())
        assert st == [1] * len(SHAPES)
        torch.cuda.synchronize()
        assert bool((dst == GUARD).all())


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
def test_sparse_fp8_unpack(bb, eng, dt):
    """The fused unpack into pages with null entries stores exactly the dense unpack's values in the stored pages, nothing
    elsewhere, with the dense get's digest and status; MX blocks straddle pages."""
    wide = {torch.bfloat16: bb.MxWide.BF16, torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[dt]
    b = torch.empty((), dtype=dt).element_size()
    per = 16 // b
    rng = np.random.default_rng(32)
    for pe, npg, ph in ((3 * per, 64, 0), (T, 2, 0), (T + 40 * per, 3, 0), (512 * per, 5, 100 * per + 3), (per, 2048 // per, 0)):
        n = max(32, (pe * npg - ph) // 32 * 32)
        g = torch.Generator(device="cuda").manual_seed(pe)
        obj = (torch.randn(n, generator=g, device="cuda") * 64).to(dt)
        packed = torch.zeros(n + n // 32 + 16, dtype=torch.uint8, device="cuda")
        dg, st, _ = eng.run_fp8([(obj.data_ptr(), packed.data_ptr(), n)], False, _stream(), wide=wide)
        ref = torch.empty_like(obj)
        eng.run_fp8([(ref.data_ptr(), packed.data_ptr(), n, dg[0])], True, _stream(), wide=wide)
        offs, at = _carve(rng, npg, pe * b, ph * b, 64)
        buf = torch.full((at,), GUARD, dtype=torch.uint8, device="cuda")
        refb = ref.view(torch.uint8).cpu().numpy()
        for m in _masks(rng, npg):
            buf.fill_(GUARD)
            table = [buf.data_ptr() + a if keep else 0 for a, keep in zip(offs, m)]
            dg2, st2, _ = eng.run_fp8([(0, packed.data_ptr(), n, dg[0], None, None, None, None, None, (table, pe, ph))], True, _stream(),
                                      wide=wide)
            assert st2 == [0] and dg2 == dg
            want = np.full(buf.numel(), GUARD, dtype=np.uint8)
            y = np.arange(n * b) + ph * b
            k = y // (pe * b)
            keep = m[k]
            want[(np.asarray(offs, dtype=np.int64)[k] + y % (pe * b))[keep]] = refb[keep]
            torch.cuda.synchronize()
            assert np.array_equal(buf.cpu().numpy(), want), (dt, pe, m.sum())


def test_paged_puts_with_a_null_page_are_refused_without_a_launch(bb, eng):
    src = _random(bb, 8 * T, 3)
    out = torch.full((8 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), out.data_ptr()
    launches = eng.launches
    with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
        eng.run([(s, d + 6 * T, 64, 0, 0), (0, d, 3 * 4096, 0, 0, 0, None, None, None, ([s, 0, s + T], 4096, 0))], bb.ChecksumAlgo.XXH3,
                _stream())
    with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
        eng.run_fp8([(0, d, 2 * 2048, None, None, None, None, None, ([0, s + T], 2048, 0))], False, _stream())
    assert eng.launches == launches
    torch.cuda.synchronize()
    assert bool((out == GUARD).all())


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def test_client_sparse_gets_on_every_tier(bb):
    """batch_get_device_paged and batch_get_device_fp8_paged with null pages on a GpuRankCluster, fused from HBM and
    through the host from an object moved to DRAM: stored pages right, everything else untouched; puts with a null page
    are refused alone."""
    from blackbird_b200.parallel import GpuRankCluster

    E = bb.ErrorCode
    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-sparse-client", dram_bytes=64 << 20)
    try:
        c = cl.client
        rng = np.random.default_rng(33)
        page, npg = 32 * 1024, 40
        cache = _random(bb, 64 * page, 34)
        host = cache.cpu().numpy()
        slots = [int(x) * page for x in rng.permutation(64)[:npg]]
        table = [cache.data_ptr() + o for o in slots]
        obj = np.concatenate([host[o:o + page] for o in slots])
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=bb.ChecksumAlgo.XXH3,
                              preferred_classes=[bb.StorageClass.RAM_GPU])
        holed = list(table)
        holed[5] = 0
        assert c.batch_put_device_paged(["a", "hole", "b"], [table, holed, table], [page] * 3, cfg, _stream()) == [E.OK, E.INVALID_ARGUMENT, E.OK]
        assert not c.object_exists("hole")
        pcache = torch.randn(npg * page // 2, device="cuda").to(torch.bfloat16)
        ptable = [pcache.data_ptr() + k * page for k in range(npg)]
        assert c.batch_put_device_fp8_paged(["f", "fh"], [ptable, [0] + ptable[1:]], [page // 2] * 2, cfg, _stream()) == [E.OK, E.INVALID_ARGUMENT]
        assert not c.object_exists("fh")
        fref = torch.empty_like(pcache)
        assert c.batch_get_device_fp8(["f"], [fref.data_ptr()], [fref.numel()], _stream()) == [E.OK]
        fref_b = fref.view(torch.uint8).cpu().numpy()
        assert c.migrate("b", bb.StorageClass.RAM_CPU) == E.OK
        assert c.get_workers("b")[0].shards[0].storage_class == bb.StorageClass.RAM_CPU
        dst = torch.full((80 * page,), GUARD, dtype=torch.uint8, device="cuda")
        for m in _masks(rng, npg):
            doffs = [int(x) * page for x in rng.permutation(80)[:npg]]
            t = [dst.data_ptr() + o if keep else 0 for o, keep in zip(doffs, m)]
            want = np.full(dst.numel(), GUARD, dtype=np.uint8)
            for k, (o, keep) in enumerate(zip(doffs, m)):
                if keep:
                    want[o:o + page] = obj[k * page:(k + 1) * page]
            for key in ("a", "b"):  # HBM (fused), DRAM
                dst.fill_(GUARD)
                ecs, sizes = c.batch_get_device_paged([key], [t], [page], _stream())
                assert ecs == [E.OK] and sizes == [obj.size], key
                torch.cuda.synchronize()
                assert np.array_equal(dst.cpu().numpy(), want), (key, m.sum())
            dst.fill_(GUARD)
            assert c.batch_get_device_fp8_paged(["f"], [t], [page // 2], _stream(), wide=bb.MxWide.BF16) == [E.OK]
            fwant = np.full(dst.numel(), GUARD, dtype=np.uint8)
            for k, (o, keep) in enumerate(zip(doffs, m)):
                if keep:
                    fwant[o:o + page] = fref_b[k * page:(k + 1) * page]
            torch.cuda.synchronize()
            assert np.array_equal(dst.cpu().numpy(), fwant), m.sum()
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore
class Recorder:
    """The real client, with the block-get calls logged as (name, page tables as null / non-null patterns, page sizes)
    and forwarded unchanged; other calls by name only."""

    def __init__(self, client):
        self.client, self.log = client, []

    def __getattr__(self, name):
        fn = getattr(self.client, name)
        if not name.startswith("batch_"):
            return fn

        def call(*args, **kw):
            if "paged" in name:
                self.log.append((name, [[int(x != 0) for x in p] for p in args[1]], list(args[2])))
            elif not name.endswith(("batch_get", "batch_put")) or not any(k.endswith("#meta") for k in args[0]):
                self.log.append((name,))
            return fn(*args, **kw)

        return call


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _cache(dtype, shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda").to(dtype)


@pytest.fixture(scope="module")
def env():
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=512 << 20, cluster_id="t-sparse-ts")
    rec = Recorder(cl.client)
    yield cl, rec, TensorStore(rec)
    cl.stop()


def _selections(rng, n, k):
    """(ids into a cache of k blocks..., blocks of a stored tensor of n blocks): a prefix, a permutation, one block, none,
    every block."""
    return [list(range(min(3, n))), list(rng.permutation(n)), [int(rng.integers(0, n))], [], list(range(n))]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("packed", [False, True])
def test_partial_restores_equal_index_copy_of_index_select(bb, env, dtype, packed, monkeypatch):
    """Both routes (pages above and below the thresholds), dims 0, 2 and -1, contiguous and non-contiguous caches: the
    cache is bit-identical to index_copy_ of index_select of the stored tensor, blocks=range(n) equals blocks=None, and the
    paged route sends a table over the whole stored object with only the selected blocks' pages set."""
    from blackbird_b200.ops import tensor_store

    cl, rec, store = env
    rng = np.random.default_rng(35)
    es = torch.empty((), dtype=dtype).element_size()
    bshape, wshape = (3, 2, 12, 4, 1024 // es), (4, 12, 8, 8192 // es)  # 4 KiB pages along dim 2, 64 KiB along dim 1
    # (parent shape, the view of it that is the cache, dim): narrowed and strided caches are not contiguous
    cases = [(bshape, lambda t: t, 2), (bshape, lambda t: t[:, :, :, :2], 2), (wshape, lambda t: t, 1), (bshape, lambda t: t, 0),
             (bshape, lambda t: t, -1), (wshape, lambda t: t[::2], 1)]
    for lo in (0, 1 << 40):  # every page paged; none
        monkeypatch.setattr(tensor_store, "PAGED_MIN_PAGE_BYTES", lo)
        monkeypatch.setattr(tensor_store, "FP8_PAGED_MIN_PAGE_BYTES", lo)
        monkeypatch.setattr(tensor_store, "FP8_PARTIAL_MIN_PAGE_BYTES", lo)
        for j, (shape, view, dim) in enumerate(cases):
            cache = view(_cache(dtype, shape, 36 + j))
            d = dim % cache.dim()
            n = min(5, cache.shape[d])
            stored_ids = list(rng.permutation(cache.shape[d])[:n])
            key = f"p{int(packed)}/{dtype}/{lo}/{j}"
            store.put_blocks(key, cache, stored_ids, dim=dim, pack_fp8=packed)
            stored = store.get(key)
            for blocks in _selections(rng, n, cache.shape[d]):
                ids = list(rng.permutation(cache.shape[d])[:len(blocks)])
                dst = view(_cache(dtype, shape, 50 + j))
                want = dst.clone().index_copy_(d, torch.tensor(ids, dtype=torch.int64, device="cuda"),
                                               stored.index_select(d, torch.tensor(blocks, dtype=torch.int64, device="cuda")))
                rec.log.clear()
                store.get_blocks_into(key, dst, ids, dim=dim, blocks=blocks)
                assert torch.equal(_bits(dst), _bits(want)), (key, blocks)
                paged = [e for e in rec.log if "paged" in e[0]]
                if not blocks:
                    assert rec.log == []  # validated, then nothing moved
                elif paged:
                    (name, tables, _), = paged
                    pattern = np.asarray(tables[0]).reshape(-1, n)
                    assert (pattern[:, blocks] == 1).all() and pattern.sum() == pattern.shape[0] * len(blocks)
                    assert name == ("batch_get_device_fp8_paged" if packed else "batch_get_device_paged")
                else:
                    assert any(e[0] in ("batch_get_device", "batch_get_device_fp8") for e in rec.log), rec.log
                if lo == 0 and blocks and d != cache.dim() - 1:
                    assert paged, (key, rec.log)
            # blocks=range(n) is blocks=None
            a, b2 = view(_cache(dtype, shape, 40)), view(_cache(dtype, shape, 40))
            ids = list(rng.permutation(cache.shape[d])[:n])
            store.get_blocks_into(key, a, ids, dim=dim, blocks=range(n))
            store.get_blocks_into(key, b2, ids, dim=dim)
            assert torch.equal(_bits(a), _bits(b2))
            store.remove([key])


def test_route_choice_follows_the_page_size(bb, env):
    """As shipped: 64 KiB pages take the paged calls, 4 KiB pages the whole get, packed 16 KiB pages too (below
    FP8_PARTIAL_MIN_PAGE_BYTES, though a whole restore of them is paged); a padded packed tensor the whole get."""
    cl, rec, store = env
    wide = _cache(torch.bfloat16, (2, 12, 8, 4096), 41)
    small = _cache(torch.bfloat16, (2, 12, 4, 512), 42)
    mid = _cache(torch.bfloat16, (2, 12, 8, 1024), 45)  # 16 KiB pages: below FP8_PARTIAL_MIN_PAGE_BYTES
    odd = _cache(torch.bfloat16, (2, 12, 3, 5), 43)
    for key, cache, packed, want in (("w", wide, False, "batch_get_device_paged"), ("wp", wide, True, "batch_get_device_fp8_paged"),
                                     ("s", small, False, "batch_get_device"), ("mp", mid, True, "batch_get_device_fp8"),
                                     ("o", odd, True, "batch_get_device")):
        store.put_blocks(key, cache, [0, 3, 7, 1], dim=1, pack_fp8=packed)
        rec.log.clear()
        dst = torch.zeros_like(cache)
        store.get_blocks_into(key, dst, [4, 9], dim=1, blocks=[2, 0])
        assert rec.log[-1][0] == want, (key, rec.log)
        if "paged" in want:  # the whole stored object's table, 2 outer rows of 4 stored blocks, blocks 2 and 0 set
            assert rec.log[-1][1] == [[1, 0, 1, 0] * 2]
        ref = torch.zeros_like(cache).index_copy_(1, torch.tensor([4, 9], device="cuda"), store.get(key).index_select(1, torch.tensor([2, 0], device="cuda")))
        assert torch.equal(dst, ref), key
        store.remove([key])


def test_errors_leave_the_cache_untouched_and_async(bb, env):
    from blackbird_b200.ops.tensor_store import AsyncTensorStore

    cl, rec, store = env
    base = _cache(torch.bfloat16, (2, 2, 16, 8, 1024), 44)
    store.put_blocks("e", base, [1, 2, 3, 4], dim=2)
    dst = torch.full_like(base, 9)
    cases = [(("missing", dst, [0], 2, [0]), KeyError), (("e", dst.float(), [0], 2, [0]), TypeError),
             (("e", dst, [0.5], 2, [0]), TypeError), (("e", dst, [0], 2, [1.0]), TypeError),
             (("e", dst[:, :1], [0], 2, [0]), ValueError), (("e", dst, [0, 1], 2, [0]), ValueError),
             (("e", dst, [1, 1], 2, [0, 2]), ValueError), (("e", dst, [0, 1], 2, [2, 2]), ValueError),
             (("e", dst.cpu(), [0], 2, [0]), ValueError), (("e", dst, [0], 2, [4]), IndexError), (("e", dst, [16], 2, [0]), IndexError),
             (("e", dst, [0], 2, [-1]), IndexError)]
    for (key, c, ids, dim, blocks), exc in cases:
        rec.log.clear()
        with pytest.raises(exc):
            store.get_blocks_into(key, c, ids, dim=dim, blocks=blocks)
        assert not [e for e in rec.log if "device" in e[0]], (key, ids, blocks)
    assert bool((dst == 9).all())
    stored = store.get("e")
    astore = AsyncTensorStore(cl.client)
    try:
        out = torch.zeros_like(base)
        torch.cuda._sleep(20_000_000)
        out.fill_(1)  # the side stream waits for this write
        res = astore.get_blocks_into_async(["e"], [out], [[7, 0]], dim=2, blocks=[[3, 1]]).result()
        assert res[0] is out
        want = torch.ones_like(base).index_copy_(2, torch.tensor([7, 0], device="cuda"), stored.index_select(2, torch.tensor([3, 1], device="cuda")))
        assert torch.equal(out, want)
    finally:
        astore.close()
