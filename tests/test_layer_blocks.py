"""Paged puts and gets from block ids that stay on the device, on the GPU: the transfer engine's resolve kernel builds the
page table from a SourceBlocks description, and a BLOCKS item must move the same bytes, with the same digests and verify
status, as the same item with the equivalent host page table, at every grid and algorithm, for bb_xfer and the fused
MXFP8 pack and unpack.  Refused ids report their verdict and store nothing.  Then the client on HBM and DRAM tiers, and
TensorStore.put_layer_blocks / get_layer_blocks_into against torch.stack(index_select) and per-layer index_copy_."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

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


class Cache:
    """A byte cache [n_slices, n_blocks, stride] on the device: slice q's block b at outer[q] + b * stride, the page its
    first `page` bytes, the rest of the stride a guard gap."""

    def __init__(self, bb, n_slices, n_blocks, page, stride, seed=None):
        self.page, self.stride, self.n_blocks = page, stride, n_blocks
        self.t = _random(bb, n_slices * n_blocks * stride, seed) if seed is not None else \
            torch.full((n_slices * n_blocks * stride,), GUARD, dtype=torch.uint8, device="cuda")
        self.outer = [self.t.data_ptr() + q * n_blocks * stride for q in range(n_slices)]

    def blocks(self, bb, ids, sel=None, n_stored=0):
        return bb.DeviceBlocks(self.outer, ids.data_ptr(), ids.numel(), self.n_blocks, self.stride, self.page, id_bytes=ids.element_size(),
                               sel=0 if sel is None else sel.data_ptr(), n_stored=n_stored)

    def table(self, ids, sel=None, n_stored=0):
        """The equivalent host page table (0 for pages a partial restore does not store)."""
        ids = ids.cpu().numpy().astype(np.int64)
        per = ids.size if sel is None else n_stored
        t = np.zeros((len(self.outer), per), np.int64)
        cols = np.arange(ids.size) if sel is None else sel.cpu().numpy().astype(np.int64)
        t[:, cols] = np.asarray(self.outer, np.int64)[:, None] + ids[None, :] * self.stride
        return [int(x) for x in t.reshape(-1)]


def _ids(rng, n, k, dtype):
    return torch.tensor(rng.permutation(n)[:k], dtype=dtype, device="cuda")


@pytest.mark.parametrize("algo", ALGOS)
def test_blocks_items_equal_host_tables_at_every_grid(bb, eng, algo):
    """Puts gathering from blocks and gets scattering into them (whole and partial), int32 and int64 ids: bytes, digests
    and status equal those of the host-table items, every guard byte stays."""
    A = getattr(bb.ChecksumAlgo, algo)
    rng = np.random.default_rng(41)
    verify = 0 if algo == "NONE" else bb.XFER_VERIFY
    # (slices, blocks, page, stride, ids): small pages, tile-straddling pages, big pages
    shapes = [(4, 40, 48, 64, 9), (2, 12, 16384 + 16, 16384 + 64, 5), (3, 6, 64 * 1024, 64 * 1024, 4), (1, 3, 4096, 4096, 1)]
    for dt in (torch.int32, torch.int64):
        caches = [Cache(bb, s, n, p, st, seed=50 + i) for i, (s, n, p, st, _) in enumerate(shapes)]
        ids = [_ids(rng, n, k, dt) for (_, n, _, _, k) in shapes]
        sizes = [s * k * p for (s, _, p, _, k) in shapes]
        slab = [torch.full((n + 64,), GUARD, dtype=torch.uint8, device="cuda") for n in sizes]
        ref = [torch.full_like(x, GUARD) for x in slab]
        for g in GRIDS:
            eng.set_max_ctas(_grid(g))
            for x, y in zip(slab, ref):
                x.fill_(GUARD), y.fill_(GUARD)
            res = eng.run([(0, s.data_ptr(), n, 0, 0, 0, None, None, None, None, None, c.blocks(bb, i)) for c, i, s, n in zip(caches, ids, slab, sizes)],
                          A, _stream())
            dg, st, _, verdicts = res
            dg0, st0, _ = eng.run([(0, r.data_ptr(), n, 0, 0, 0, None, None, None, (c.table(i), c.page, 0))
                                   for c, i, r, n in zip(caches, ids, ref, sizes)], A, _stream())
            assert verdicts == [bb.ErrorCode.OK] * len(shapes)
            torch.cuda.synchronize()
            assert (dg, st) == (dg0, st0)
            for x, y, n in zip(slab, ref, sizes):
                assert torch.equal(x, y)
                if algo != "NONE":
                    assert dg[sizes.index(n)] == _model(bb, algo)(x[:n].cpu().numpy().tobytes())
            # gets: whole, and partial into some of the stored blocks
            for partial in (False, True):
                dst = [Cache(bb, s, n, p, st) for (s, n, p, st, _) in shapes]
                dst0 = [Cache(bb, s, n, p, st) for (s, n, p, st, _) in shapes]
                into, sel, n_stored = [], [], []
                for (_, n, _, _, k) in shapes:
                    m = int(rng.integers(1, k + 1)) if partial else k
                    into.append(_ids(rng, n, m, dt))
                    sel.append(_ids(rng, k, m, dt) if partial else None)
                    n_stored.append(k if partial else 0)
                items = [(s.data_ptr(), 0, n, d, verify, 0, None, None, None, None, None, None, c.blocks(bb, i, q, ns))
                         for s, n, d, c, i, q, ns in zip(slab, sizes, dg, dst, into, sel, n_stored)]
                items0 = [(s.data_ptr(), 0, n, d, verify, 0, None, None, None, None, (c.table(i, q, ns), c.page, 0))
                          for s, n, d, c, i, q, ns in zip(slab, sizes, dg, dst0, into, sel, n_stored)]
                dg1, st1, _, v1 = eng.run(items, A, _stream())
                dg2, st2, _ = eng.run(items0, A, _stream())
                torch.cuda.synchronize()
                assert v1 == [bb.ErrorCode.OK] * len(shapes) and (dg1, st1) == (dg2, st2) and st1 == [0] * len(shapes)
                for c, c0 in zip(dst, dst0):
                    assert torch.equal(c.t, c0.t), (g, partial)


def test_refused_ids_store_nothing_and_raise_no_fault(bb, eng):
    """Out-of-range ids (put and get), a repeated get id and bad selections: each item reports its verdict, a refused get
    stores nothing, a refused put reads only block 0 of each slice, and the other items of the batch complete."""
    E = bb.ErrorCode
    A = bb.ChecksumAlgo.XXH3
    src = Cache(bb, 2, 16, 4096, 4096, seed=61)
    good = torch.tensor([3, 9, 1], dtype=torch.int32, device="cuda")
    bad = {"high": torch.tensor([3, 16, 1], dtype=torch.int32, device="cuda"), "neg": torch.tensor([3, -5, 1], dtype=torch.int64, device="cuda"),
           "huge": torch.tensor([3, 1 << 40, 1], dtype=torch.int64, device="cuda")}
    n = 2 * 3 * 4096
    slabs = [torch.full((n,), GUARD, dtype=torch.uint8, device="cuda") for _ in range(4)]
    dg, st, _, v = eng.run([(0, slabs[0].data_ptr(), n, 0, 0, 0, None, None, None, None, None, src.blocks(bb, good))] +
                           [(0, s.data_ptr(), n, 0, 0, 0, None, None, None, None, None, src.blocks(bb, b)) for s, b in zip(slabs[1:], bad.values())],
                           A, _stream())
    assert v == [E.OK] + [E.VALUE_OUT_OF_RANGE] * 3
    torch.cuda.synchronize()
    block0 = torch.cat([src.t[q * 16 * 4096:q * 16 * 4096 + 4096] for q in range(2) for _ in range(3)])
    for s in slabs[1:]:
        assert torch.equal(s, block0)
    dup = torch.tensor([4, 4, 0], dtype=torch.int32, device="cuda")
    sel_high = torch.tensor([0, 3, 1], dtype=torch.int32, device="cuda")
    sel_dup = torch.tensor([2, 2, 1], dtype=torch.int32, device="cuda")
    cases = [(good, None, 0, E.OK), (bad["high"], None, 0, E.VALUE_OUT_OF_RANGE), (dup, None, 0, E.INVALID_ARGUMENT),
             (good, sel_high, 3, E.VALUE_OUT_OF_RANGE), (good, sel_dup, 3, E.INVALID_ARGUMENT), (bad["huge"], None, 0, E.VALUE_OUT_OF_RANGE)]
    dsts = [Cache(bb, 2, 16, 4096, 4096) for _ in cases]
    _, st, _, v = eng.run([(slabs[0].data_ptr(), 0, n, dg[0], bb.XFER_VERIFY, 0, None, None, None, None, None, None, d.blocks(bb, i, s, ns))
                           for d, (i, s, ns, _) in zip(dsts, cases)], A, _stream())
    assert v == [c[3] for c in cases] and st == [0] * len(cases)
    torch.cuda.synchronize()
    want = Cache(bb, 2, 16, 4096, 4096)
    for q in range(2):
        for k, b in enumerate([3, 9, 1]):
            want.t[(q * 16 + b) * 4096:(q * 16 + b + 1) * 4096] = src.t[(q * 16 + [3, 9, 1][k]) * 4096:(q * 16 + [3, 9, 1][k] + 1) * 4096]
    assert torch.equal(dsts[0].t, want.t)
    for d in dsts[1:]:
        assert (d.t == GUARD).all()
    # a bound too large for the duplicate check: NOT_IMPLEMENTED for a get, before any launch
    big = bb.DeviceBlocks(src.outer, good.data_ptr(), 3, 1 << 19, 4096, 4096)
    with pytest.raises(RuntimeError, match="NOT_IMPLEMENTED"):
        eng.run([(slabs[0].data_ptr(), 0, n, 0, 0, 0, None, None, None, None, None, None, big)], A, _stream())


@pytest.mark.parametrize("wide", ["BF16", "F16", "F32"])
def test_fp8_pack_and_unpack_from_blocks(bb, eng, wide):
    """The fused MXFP8 pack reading blocks and unpack storing into them (whole and partial) equal the same items with host
    page tables, which the exact MXFP8 model checks: packed bytes, digests and stored elements."""
    W = getattr(bb.MxWide, wide)
    b = 4 if wide == "F32" else 2
    dt = {"BF16": torch.bfloat16, "F16": torch.float16, "F32": torch.float32}[wide]
    rng = np.random.default_rng(42)
    pe, n_blocks, k, slices = 2048 + 32, 20, 6, 3  # MX blocks straddle pages
    vals = (torch.randn(slices * n_blocks * pe, device="cuda") * 8).to(dt)
    src = Cache(bb, slices, n_blocks, pe * b, pe * b)
    src.t.copy_(vals.view(torch.uint8))
    ids = _ids(rng, n_blocks, k, torch.int32)
    n = slices * k * pe
    packed = [torch.full((n + n // 32,), GUARD, dtype=torch.uint8, device="cuda") for _ in range(2)]
    blk = bb.DeviceBlocks(src.outer, ids.data_ptr(), k, n_blocks, pe * b, pe, id_bytes=4)
    dg, _, _, v = eng.run_fp8([(0, packed[0].data_ptr(), n, None, None, None, None, None, None, None, blk)], False, _stream(), wide=W)
    dg0, _, _ = eng.run_fp8([(0, packed[1].data_ptr(), n, None, None, None, None, None, ([a for a in src.table(ids)], pe, 0))], False, _stream(), wide=W)
    torch.cuda.synchronize()
    assert v == [bb.ErrorCode.OK] and dg == dg0 and torch.equal(packed[0], packed[1])
    gathered = torch.cat([vals.view(slices, n_blocks, pe)[q, ids.long()] for q in range(slices)]).reshape(-1)
    model = np.frombuffer(bb.mxfp8_pack_ref(gathered.view({2: torch.int16, 4: torch.int32}[b]).cpu().numpy(), W), dtype=np.uint8)
    assert np.array_equal(packed[0].cpu().numpy(), model)
    for partial in (False, True):
        m = 4 if partial else k
        into = _ids(rng, n_blocks, m, torch.int64)
        sel = _ids(rng, k, m, torch.int64) if partial else None
        d1, d0 = Cache(bb, slices, n_blocks, pe * b, pe * b), Cache(bb, slices, n_blocks, pe * b, pe * b)
        db = bb.DeviceBlocks(d1.outer, into.data_ptr(), m, n_blocks, pe * b, pe, id_bytes=8, sel=0 if sel is None else sel.data_ptr(),
                             n_stored=k if partial else 0)
        _, st, _, v = eng.run_fp8([(0, packed[0].data_ptr(), n, dg[0], None, None, None, None, None, None, None, db)], True, _stream(), wide=W)
        _, st0, _ = eng.run_fp8([(0, packed[0].data_ptr(), n, dg[0], None, None, None, None, None, ([a for a in d0.table(into, sel, k if partial else 0)], pe, 0))],
                                True, _stream(), wide=W)
        torch.cuda.synchronize()
        assert v == [bb.ErrorCode.OK] and st == st0 == [0] and torch.equal(d1.t, d0.t)


def test_client_on_hbm_and_dram(bb):
    """batch_put_device_blocks / batch_get_device_blocks on a GpuRankCluster: fused from HBM, whole and partial; an object
    moved to the cluster's DRAM pool, which the fabric maps, reads over it, and puts land there too; refused ids cancel
    the put alone."""
    from blackbird_b200.parallel import GpuRankCluster

    E = bb.ErrorCode
    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-blocks-client", dram_bytes=64 << 20)
    try:
        c = cl.client
        rng = np.random.default_rng(43)
        src = Cache(bb, 4, 32, 32 * 1024, 32 * 1024, seed=70)
        ids = _ids(rng, 32, 10, torch.int32)
        high = torch.tensor([1, 2, 32], dtype=torch.int32, device="cuda")
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=bb.ChecksumAlgo.XXH3,
                              preferred_classes=[bb.StorageClass.RAM_GPU])
        assert c.batch_put_device_blocks(["a", "bad", "b"], [src.blocks(bb, ids), src.blocks(bb, high), src.blocks(bb, ids)], cfg, _stream()) == \
            [E.OK, E.VALUE_OUT_OF_RANGE, E.OK]
        assert not c.object_exists("bad")
        obj = torch.cat([src.t.view(4, 32, -1)[q, ids.long()].reshape(-1) for q in range(4)])
        back = torch.empty_like(obj)
        ecs, sizes = c.batch_get_device(["a"], [back.data_ptr()], [back.numel()], _stream())
        assert ecs == [E.OK] and torch.equal(back, obj)
        assert c.migrate("b", bb.StorageClass.RAM_CPU) == E.OK
        for key in ("a", "b"):
            for partial in (False, True):
                m = 3 if partial else 10
                into = _ids(rng, 32, m, torch.int64)
                sel = _ids(rng, 10, m, torch.int64) if partial else None
                dst = Cache(bb, 4, 32, 32 * 1024, 32 * 1024)
                ecs, sizes = c.batch_get_device_blocks([key], [dst.blocks(bb, into, sel, 10 if partial else 0)], _stream())
                assert ecs == [E.OK] and sizes == [obj.numel()], (key, partial)
                want = torch.full_like(dst.t, GUARD).view(4, 32, -1)
                o = obj.view(4, 10, -1)
                want[:, into.long()] = o[:, sel.long()] if partial else o
                torch.cuda.synchronize()
                assert torch.equal(dst.t, want.reshape(-1)), (key, partial)
        dram = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU])
        assert c.batch_put_device_blocks(["d"], [src.blocks(bb, ids)], dram, _stream()) == [E.OK]
        assert c.get_workers("d")[0].shards[0].storage_class == bb.StorageClass.RAM_CPU
        back.zero_()
        assert c.batch_get_device(["d"], [back.data_ptr()], [back.numel()], _stream())[0] == [E.OK] and torch.equal(back, obj)
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore
@pytest.fixture(scope="module")
def env():
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=1 << 30, cluster_id="t-layer-blocks")
    yield cl, TensorStore(cl.client)
    cl.stop()


def _layers(n, shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(shape, generator=g, device="cuda").to(dtype) for _ in range(n)]


class _Proxy:
    """The real client, with the names of its data calls logged (metadata puts and gets left out)."""

    def __init__(self, client):
        self.client, self.log = client, []

    def __getattr__(self, name):
        fn = getattr(self.client, name)
        if not name.startswith("batch_"):
            return fn

        def call(*a, **kw):
            if not any(str(k).endswith("#meta") for k in a[0]):
                self.log.append(name)
            return fn(*a, **kw)

        return call


@pytest.mark.parametrize("nl", [1, 4, 32])
def test_layer_blocks_equal_stack_of_index_select(bb, env, nl):
    """put_layer_blocks with CUDA ids stores torch.stack(index_select) through the device route; get, get_rows, get_slice
    and get_blocks_into on a stacked cache read it; get_layer_blocks_into restores index_copy_ per layer, whole and
    partial, also into a single tensor."""
    from blackbird_b200.ops.tensor_store import TensorStore

    cl, _ = env
    proxy = _Proxy(cl.client)
    store = TensorStore(proxy)
    rng = np.random.default_rng(44)
    for h, dt in ((16, torch.bfloat16), (16, torch.float32)):  # 32 and 64 KiB pages along dim 1
        shp = (2, 64, h, 8, 128)
        caches = _layers(nl, shp, dt, nl * 10 + h)
        for idt in (torch.int32, torch.int64):
            ids = _ids(rng, 64, 24, idt)
            key = f"lb/{nl}/{h}/{idt}"
            proxy.log.clear()
            store.put_layer_blocks(key, caches, ids, dim=1)
            assert proxy.log == ["batch_put_device_blocks"]
            want = torch.stack([c.index_select(1, ids.long()) for c in caches])
            got = store.get(key)
            assert got.dtype == dt and torch.equal(got, want)
            assert torch.equal(store.get_rows(key, nl // 2, nl), want[nl // 2:])
            assert torch.equal(store.get_slice(key, 2, 5, 20), want[:, :, 5:20])
            stacked = torch.zeros((nl, 2, 64, h, 8, 128), dtype=dt, device="cuda")
            into = list(rng.permutation(64)[:24])
            store.get_blocks_into(key, stacked, into, dim=2)
            assert torch.equal(stacked[:, :, into], want)
            for partial in (False, True):
                outs = [torch.zeros(shp, dtype=dt, device="cuda") for _ in range(nl)]
                m = 7 if partial else 24
                dst = _ids(rng, 64, m, idt)
                sel = _ids(rng, 24, m, idt) if partial else None
                proxy.log.clear()
                store.get_layer_blocks_into(key, outs, dst, dim=1, blocks=sel)
                assert proxy.log == ["batch_get_device_blocks"]
                for l, o in enumerate(outs):
                    ref = torch.zeros_like(o).index_copy_(1, dst.long(), want[l] if sel is None else want[l].index_select(1, sel.long()))
                    assert torch.equal(o, ref), (l, partial)
        one = caches[0]
        ids = _ids(rng, 64, 5, torch.int64)
        store.put_layer_blocks("lb/one", one, ids, dim=1)
        assert torch.equal(store.get("lb/one"), one.index_select(1, ids))
        out = torch.zeros_like(one)
        store.get_layer_blocks_into("lb/one", out, ids, dim=1)
        assert torch.equal(out, torch.zeros_like(one).index_copy_(1, ids, one.index_select(1, ids)))
        store.remove([f"lb/{nl}/{h}/{t}" for t in (torch.int32, torch.int64)] + ["lb/one"])


def _mx(bb, t):
    """`t` through the exact MXFP8 model: what a packed put of it reads back as."""
    es = t.element_size()
    w = {torch.bfloat16: bb.MxWide.BF16, torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[t.dtype]
    raw = t.reshape(-1).view({2: torch.int16, 4: torch.int32}[es]).cpu().numpy()
    back = np.frombuffer(bb.mxfp8_unpack_ref(bb.mxfp8_pack_ref(raw, w), t.numel(), w), dtype={2: np.int16, 4: np.int32}[es]).copy()
    return torch.from_numpy(back).view(t.dtype).reshape(t.shape).cuda()


def _bits(t):
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
def test_packed_layer_blocks_use_the_fp8_calls(bb, env, dt):
    """put_layer_blocks(..., pack_fp8=True) packs through batch_put_device_fp8_blocks and get_layer_blocks_into of the
    packed object unpacks through batch_get_device_fp8_blocks, whole and partial, equal to the exact MXFP8 model; a
    refused id stores nothing."""
    from blackbird_b200.ops.tensor_store import TensorStore

    cl, _ = env
    proxy = _Proxy(cl.client)
    store = TensorStore(proxy)
    rng = np.random.default_rng(47)
    caches = [(c * 16).to(dt) for c in _layers(4, (2, 64, 16, 8, 128), torch.float32, 11)]
    ids = _ids(rng, 64, 12, torch.int32)
    key = f"pk/{dt}"
    proxy.log.clear()
    store.put_layer_blocks(key, caches, ids, dim=1, pack_fp8=True)
    assert proxy.log == ["batch_put_device_fp8_blocks"]
    want = _mx(bb, torch.stack([c.index_select(1, ids.long()) for c in caches]))
    assert torch.equal(_bits(store.get(key)), _bits(want))
    for partial in (False, True):
        outs = [torch.zeros_like(c) for c in caches]
        m = 5 if partial else 12
        dst = _ids(rng, 64, m, torch.int64)
        sel = _ids(rng, 12, m, torch.int64) if partial else None
        proxy.log.clear()
        store.get_layer_blocks_into(key, outs, dst, dim=1, blocks=sel)
        assert proxy.log == ["batch_get_device_fp8_blocks"]
        for l, o in enumerate(outs):
            ref = torch.zeros_like(o).index_copy_(1, dst.long(), want[l] if sel is None else want[l].index_select(1, sel.long()))
            assert torch.equal(_bits(o), _bits(ref)), (l, partial)
    with pytest.raises(IndexError):
        store.put_layer_blocks(f"{key}/bad", caches, torch.tensor([3, 64], dtype=torch.int32, device="cuda"), dim=1, pack_fp8=True)
    assert not cl.client.object_exists(f"{key}/bad") and not cl.client.object_exists(f"{key}/bad#meta")
    outs = [torch.zeros_like(c) for c in caches]
    with pytest.raises(ValueError):
        store.get_layer_blocks_into(key, outs, torch.tensor([1] * 12, dtype=torch.int32, device="cuda"), dim=1)
    assert all((o == 0).all() for o in outs)
    store.remove([key])


def test_fallback_routes(bb, env):
    """Host ids, small pages, a layout the device route cannot read in place and layers that alias one another take
    index_select + stack + put and get + index_copy_, with the same results; so does a get the device route answers
    NOT_IMPLEMENTED (a cache of more blocks than the resolve kernel checks for repeats)."""
    from blackbird_b200.ops.tensor_store import TensorStore

    cl, _ = env
    proxy = _Proxy(cl.client)
    store = TensorStore(proxy)
    rng = np.random.default_rng(45)
    caches = _layers(3, (2, 32, 16, 8, 128), torch.bfloat16, 5)
    small = _layers(3, (2, 32, 1, 8, 128), torch.bfloat16, 6)  # 2 KiB pages, below LAYER_BLOCKS_MIN_PAGE_BYTES
    strided = [c[:, :, :, :, :64] for c in _layers(3, (2, 32, 16, 8, 128), torch.bfloat16, 7)]
    ids = _ids(rng, 32, 9, torch.int32)
    for name, cs, i, pack in (("host", caches, ids.tolist(), False), ("small", small, ids, False), ("strided", strided, ids, False),
                              ("host fp8", caches, ids.tolist(), True), ("aliased", [caches[0], caches[0]], ids, False)):
        proxy.log.clear()
        store.put_layer_blocks(f"fb/{name}", cs, i, dim=1, pack_fp8=pack)
        assert proxy.log and not any("blocks" in n for n in proxy.log), name
        want = torch.stack([c.index_select(1, ids.long()) for c in cs])
        got = store.get(f"fb/{name}")
        if pack:
            assert torch.equal(_bits(got), _bits(_mx(bb, want)))
            want = got
        else:
            assert torch.equal(got, want)
        # zeros_like of a sliced cache is dense: the strided case restores into slices of the same layout
        outs = [torch.zeros(c.shape[:-1] + (128,), dtype=c.dtype, device="cuda")[..., :64] if name == "strided" else torch.zeros_like(c)
                for c in cs]
        if name == "aliased":
            outs = [outs[0], outs[0]]
        proxy.log.clear()
        store.get_layer_blocks_into(f"fb/{name}", outs, i, dim=1)
        assert proxy.log and not any("blocks" in n for n in proxy.log), name
        for l, o in enumerate(outs):
            assert torch.equal(o.index_select(1, ids.long()), want[l]), name
    # more blocks than the duplicate bitmap covers: the put takes the device route, the get falls back after it
    big = torch.randn((1 << 18) + 8, 2048, device="cuda").to(torch.bfloat16)  # 4 KiB pages along dim 0
    bids = torch.tensor([5, (1 << 18) + 3, 7], dtype=torch.int64, device="cuda")
    proxy.log.clear()
    store.put_layer_blocks("fb/big", big, bids, dim=0)
    assert proxy.log == ["batch_put_device_blocks"]
    out = torch.zeros_like(big)
    proxy.log.clear()
    store.get_layer_blocks_into("fb/big", out, bids.flip(0), dim=0)
    assert proxy.log[0] == "batch_get_device_blocks" and len(proxy.log) > 1 and not any("blocks" in n for n in proxy.log[1:])
    assert torch.equal(out.index_select(0, bids.flip(0)), big.index_select(0, bids))
    with pytest.raises(IndexError):  # the fallback checks the ids on the host
        store.get_layer_blocks_into("fb/big", out, torch.tensor([1, 2, 1 << 20], dtype=torch.int64, device="cuda"), dim=0)
    del big, out
    store.remove(["fb/big"] + [f"fb/{n}" for n in ("host", "small", "strided", "host fp8", "aliased")])


def test_errors_after_the_call_store_nothing(bb, env):
    """Ids the device refuses raise after the call (IndexError out of range, ValueError for a repeated get id), store no
    object and no #meta, write no cache byte, and let the other keys complete; no CUDA indexing op sees them."""
    cl, store = env
    caches = _layers(2, (2, 32, 16, 8, 128), torch.bfloat16, 8)
    good = torch.tensor([4, 1, 30], dtype=torch.int32, device="cuda")
    high = torch.tensor([4, 32, 1], dtype=torch.int32, device="cuda")
    with pytest.raises(IndexError):
        store.batch_put_layer_blocks(["e/ok", "e/high", "e/ok2"], [caches, caches, caches], [good, high, good], dim=1)
    assert cl.client.object_exists("e/ok") and cl.client.object_exists("e/ok2")
    assert not cl.client.object_exists("e/high") and not cl.client.object_exists("e/high#meta")
    want = torch.stack([c.index_select(1, good.long()) for c in caches])
    for dst_ids, err in ((torch.tensor([0, 0, 2], dtype=torch.int64, device="cuda"), ValueError),
                         (torch.tensor([0, 99, 2], dtype=torch.int64, device="cuda"), IndexError)):
        outs = [torch.zeros_like(c) for c in caches]
        other = [torch.zeros_like(c) for c in caches]
        with pytest.raises(err):
            store.batch_get_layer_blocks_into(["e/ok", "e/ok2"], [outs, other], [dst_ids, good], dim=1)
        assert all((o == 0).all() for o in outs)
        for l, o in enumerate(other):
            assert torch.equal(o.index_select(1, good.long()), want[l])
    with pytest.raises(IndexError):  # a bad selection
        store.get_layer_blocks_into("e/ok", [torch.zeros_like(c) for c in caches], good[:2], dim=1,
                                    blocks=torch.tensor([0, 3], dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):  # shapes are checked before any transfer
        store.put_layer_blocks("e/mixed", [caches[0], caches[1][:, :16]], good, dim=1)


def test_ids_written_on_the_stream_are_used_and_nothing_syncs(bb, env):
    """Ids written on the caller's stream behind a long kernel are the ids the transfer uses, and the device route never
    copies them to the host (sync debug mode 'error' raises on any synchronising copy)."""
    cl, store = env
    caches = _layers(4, (2, 64, 16, 8, 128), torch.bfloat16, 9)
    ids = torch.zeros(16, dtype=torch.int64, device="cuda")
    real = torch.arange(40, 56, dtype=torch.int64, device="cuda").flip(0)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)
    ids.copy_(real)
    torch.cuda.set_sync_debug_mode("error")
    try:
        store.put_layer_blocks("s/put", caches, ids, dim=1)
        outs = [torch.zeros_like(c) for c in caches]
        torch.cuda._sleep(200_000_000)
        dst = torch.zeros(16, dtype=torch.int32, device="cuda")
        dst.copy_(torch.arange(16, dtype=torch.int32, device="cuda") * 3)
        store.get_layer_blocks_into("s/put", outs, dst, dim=1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = torch.stack([c.index_select(1, real) for c in caches])
    assert torch.equal(store.get("s/put"), want)
    for l, o in enumerate(outs):
        assert torch.equal(o.index_select(1, dst.long()), want[l])
        assert (o.sum(dim=(0, 2, 3, 4)) != 0).sum() == 16


def test_async_forms(bb, env):
    from blackbird_b200.ops.tensor_store import AsyncTensorStore

    cl, _ = env
    astore = AsyncTensorStore(cl.client, workers=2)
    try:
        caches = _layers(8, (2, 32, 16, 8, 128), torch.float16, 10)
        ids = torch.tensor([5, 2, 31, 0], dtype=torch.int32, device="cuda")
        assert astore.put_layer_blocks_async(["a/0", "a/1"], [caches, caches[:2]], [ids, ids], dim=1).result() == 2
        outs = [torch.zeros_like(c) for c in caches]
        sel = torch.tensor([3, 1], dtype=torch.int64, device="cuda")
        into = torch.tensor([7, 9], dtype=torch.int64, device="cuda")
        got = astore.get_layer_blocks_into_async(["a/0"], [outs], [into], dim=1, blocks=[sel]).result()
        assert got[0] is outs
        for c, o in zip(caches, outs):
            assert torch.equal(o, torch.zeros_like(c).index_copy_(1, into, c.index_select(1, ids.long()).index_select(1, sel)))
        with pytest.raises(IndexError):
            astore.put_layer_blocks_async(["a/bad"], [caches], [torch.tensor([40], dtype=torch.int32, device="cuda")], dim=1).result()
    finally:
        astore.close()
