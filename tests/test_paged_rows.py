"""Paged puts and gets of head-sliced KV blocks on the GPU: the in-page row pattern (XFER_PAGE_ROWS) of the paged
gathering load and scattering store in bb_xfer and bb_xfer_fp8 through XferEngine, the paged and blocks client calls on
HBM and DRAM tiers, and TensorStore's block methods on head slices of NHD and HND caches.  The tile in shared memory is
the dense object's, so digests must equal those of a plain transfer of the gathered rows, and gets must store exactly
the rows: every byte around them is checked."""
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
def eng():
    from blackbird_b200 import _bb

    e = _bb.XferEngine(0, 4096, 2)
    yield e
    e.set_max_ctas(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _grid(g):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"sms": sms, "2sms": 2 * sms}.get(g, g)


class Blocks:
    """A guard-filled device buffer of `nb` blocks, each `nrows` rows of `pitch` bytes; the slice is `width` bytes at
    `col` of every row.  Page k of a table over ids is block ids[k]'s slice."""

    def __init__(self, nb, nrows, pitch, width, col):
        self.nb, self.nrows, self.pitch, self.width, self.col = nb, nrows, pitch, width, col
        self.block = nrows * pitch + 48
        self.buf = torch.full((nb * self.block,), GUARD, dtype=torch.uint8, device="cuda")

    @property
    def page(self):
        return self.nrows * self.width

    def addrs(self, ids):
        return [self.buf.data_ptr() + int(b) * self.block + self.col for b in ids]

    def index(self, ids):
        """Byte offsets in buf of the dense object's bytes, in order."""
        r = np.arange(self.nrows)[:, None] * self.pitch + np.arange(self.width)[None, :]
        return (np.asarray(ids, dtype=np.int64)[:, None] * self.block + self.col + r.reshape(-1)[None, :]).reshape(-1)

    def fill(self, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.buf[torch.from_numpy(self.index(range(self.nb))).cuda()] = torch.randint(0, 256, (self.nb * self.page,), generator=g,
                                                                                       device="cuda", dtype=torch.uint8)

    def gather(self, ids):
        return self.buf[torch.from_numpy(self.index(ids)).cuda()]

    def expect(self, ids, blob, base=None):
        want = torch.full_like(self.buf, GUARD) if base is None else base.clone()
        want[torch.from_numpy(self.index(ids)).cuda()] = blob
        return want


@pytest.mark.parametrize("algo", ALGOS)
def test_engine_rows_at_every_grid(bb, eng, algo):
    """A paged put of in-page rows hashes like a contiguous put of the gathered rows; a paged get stores exactly the
    rows, with null pages stored nowhere; both at every grid."""
    A = getattr(bb.ChecksumAlgo, algo)
    src = Blocks(40, 16, 1024, 256, 512)
    src.fill(1)
    ids = list(np.random.default_rng(2).permutation(40)[:23])
    dense = src.gather(ids).contiguous()
    n = dense.numel()
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        pages = (src.addrs(ids), src.page, 0, 256, 1024)
        dg, st, _ = eng.run([(0, out.data_ptr(), n, 0, 0, 0, None, None, None, pages)], A, _stream())
        ref = torch.zeros_like(out)
        rg, _, _ = eng.run([(dense.data_ptr(), ref.data_ptr(), n, 0, 0)], A, _stream())
        torch.cuda.synchronize()
        assert dg == rg and st == [0] and torch.equal(out, dense), g
        dst = Blocks(40, 16, 1024, 256, 512)
        into = list(np.random.default_rng(3).permutation(40)[:23])
        table = dst.addrs(into)
        table[5] = 0  # a null page: a partial restore
        dg2, st2, _ = eng.run([(dense.data_ptr(), 0, n, 0, 0, 0, None, None, None, None, (table, dst.page, 0, 256, 1024))], A, _stream())
        torch.cuda.synchronize()
        assert st2 == [0] and dg2 == rg
        keep = [b for k, b in enumerate(into) if k != 5]
        blob = torch.cat([dense[k * dst.page:(k + 1) * dst.page] for k in range(len(into)) if k != 5])
        assert torch.equal(dst.buf, dst.expect(keep, blob)), g


def test_engine_rejects_bad_patterns(bb, eng):
    src = Blocks(4, 4, 256, 64, 0)
    out = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    A = bb.ChecksumAlgo.XXH3
    for pat, code in [((64, 72), "INVALID_ADDRESS"), ((48, 256), "INVALID_ARGUMENT"), ((64, 32), "INVALID_ARGUMENT")]:
        with pytest.raises(RuntimeError, match=code):
            eng.run([(0, out.data_ptr(), 1024, 0, 0, 0, None, None, None, (src.addrs(range(4)), 256, 0) + pat)], A, _stream())
    # XFER_PAGE_ROWS is the engine's to set: a caller's flag on pages without a pattern, on scatter rows or on a plain
    # item is refused before anything is launched
    F = bb.XFER_PAGE_ROWS
    for it in [(0, out.data_ptr(), 1024, 0, F, 0, None, None, None, (src.addrs(range(4)), 256, 0)),
               (src.buf.data_ptr(), out.data_ptr(), 256, 0, F, 0, None, None, (64, 64, 0)),
               (src.buf.data_ptr(), out.data_ptr(), 256, 0, F)]:
        with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
            eng.run([it], A, _stream())
    assert bool((out == 0).all())


@pytest.mark.parametrize("algo", ["NONE", "XXH3"])
def test_engine_rows_with_byte_wise_heads_and_tails(bb, eng, algo):
    """Rows of 24 bytes every 40: every row but the 16-byte aligned ones starts and ends inside a 16-byte chunk, so the
    walk moves heads and tails byte-wise (a gap of 16 keeps them co-aligned).  The put reads exactly the rows, the get
    stores exactly them and no guard byte around them."""
    A = getattr(bb.ChecksumAlgo, algo)
    src = Blocks(300, 4, 40, 24, 16)  # pages of 96 dense bytes, 160-byte extents
    src.fill(6)
    rng = np.random.default_rng(7)
    ids = list(rng.permutation(300)[:257])  # a 24672-byte object: two tiles, rows straddling the tile edge
    dense = src.gather(ids).contiguous()
    n = dense.numel()
    for g in (1, "sms"):
        eng.set_max_ctas(_grid(g))
        out = torch.zeros(n, dtype=torch.uint8, device="cuda")
        dg, st, _ = eng.run([(0, out.data_ptr(), n, 0, 0, 0, None, None, None, (src.addrs(ids), src.page, 0, 24, 40))], A, _stream())
        ref = torch.zeros_like(out)
        rg, _, _ = eng.run([(dense.data_ptr(), ref.data_ptr(), n, 0, 0)], A, _stream())
        torch.cuda.synchronize()
        assert dg == rg and st == [0] and torch.equal(out, dense), g
        dst = Blocks(300, 4, 40, 24, 16)
        into = list(rng.permutation(300)[:257])
        dg2, st2, _ = eng.run([(dense.data_ptr(), 0, n, 0, 0, 0, None, None, None, None, (dst.addrs(into), dst.page, 0, 24, 40))], A,
                              _stream())
        torch.cuda.synchronize()
        assert st2 == [0] and dg2 == rg and torch.equal(dst.buf, dst.expect(into, dense)), g


def test_engine_blocks_with_rows_and_refused_ids(bb, eng):
    A = bb.ChecksumAlgo.XXH3
    src = Blocks(30, 8, 512, 128, 256)
    src.fill(4)
    ids = torch.tensor([29, 3, 17, 0, 8], dtype=torch.int32, device="cuda")
    dense = src.gather(ids.tolist()).contiguous()
    n = dense.numel()
    base = src.buf.data_ptr() + 256

    def blocks(i, buf_base, nb=30):
        return bb.DeviceBlocks([buf_base], i.data_ptr(), i.numel(), nb, src.block, src.page, row_width=128, row_pitch=512)

    out = torch.zeros(n, dtype=torch.uint8, device="cuda")
    res = eng.run([(0, out.data_ptr(), n, 0, 0, 0, None, None, None, None, None, blocks(ids, base))], A, _stream())
    torch.cuda.synchronize()
    assert res[1] == [0] and res[3] == [bb.ErrorCode.OK] and torch.equal(out, dense)
    dst = Blocks(30, 8, 512, 128, 256)
    into = torch.tensor([1, 2, 28, 14, 7], dtype=torch.int32, device="cuda")
    res = eng.run([(dense.data_ptr(), 0, n, 0, 0, 0, None, None, None, None, None, None, blocks(into, dst.buf.data_ptr() + 256))], A, _stream())
    torch.cuda.synchronize()
    assert res[3] == [bb.ErrorCode.OK] and torch.equal(dst.buf, dst.expect(into.tolist(), dense))
    # refused ids store nothing
    for bad, code in [([1, 2, 30, 14, 7], bb.ErrorCode.VALUE_OUT_OF_RANGE), ([1, 2, 2, 14, 7], bb.ErrorCode.INVALID_ARGUMENT)]:
        d2 = Blocks(30, 8, 512, 128, 256)
        b = torch.tensor(bad, dtype=torch.int32, device="cuda")
        res = eng.run([(dense.data_ptr(), 0, n, 0, 0, 0, None, None, None, None, None, None, blocks(b, d2.buf.data_ptr() + 256))], A, _stream())
        torch.cuda.synchronize()
        assert res[3] == [code] and bool((d2.buf == GUARD).all())


def _bits(t):
    t = t.contiguous()
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _mx_model(bb, t):
    """unpack(pack(t)) by the exact MXFP8 model, in t's dtype and shape."""
    w = {torch.bfloat16: bb.MxWide.BF16, torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[t.dtype]
    x = _bits(t).cpu().numpy().reshape(-1)
    y = np.frombuffer(bb.mxfp8_unpack_ref(np.frombuffer(bb.mxfp8_pack_ref(x, w), dtype=np.uint8), x.size, w), dtype=x.dtype)
    return torch.from_numpy(y.copy()).cuda().view(t.dtype).view(t.shape)


@pytest.fixture(scope="module")
def env():
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-paged-rows", dram_bytes=64 << 20, max_replicas=3)
    yield cl
    cl.stop()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_client_packed_rows_match_the_model(bb, env, dtype):
    """batch_put_device_fp8_paged / batch_get_device_fp8_paged with rows: the stored object is that of packing the
    dense slices, and the get unpacks exactly into the rows (the rest of the cache untouched)."""
    W = {torch.bfloat16: bb.MxWide.BF16, torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[dtype]
    es = torch.empty((), dtype=dtype).element_size()
    g = torch.Generator(device="cuda").manual_seed(7)
    cache = torch.randn((2, 64, 16, 8, 64), device="cuda", generator=g).to(dtype)  # NHD, 8 heads of 64
    view = cache[:, :, :, 2:6, :]
    ids = [40, 3, 17, 62, 9, 0]
    from blackbird_b200.ops.tensor_store import TensorStore

    addrs, page, rows = TensorStore._block_pages(view, 1, np.array(ids), 0)
    ue = (rows[0] // es, rows[1] // es)
    cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])
    key = f"pk/{str(dtype)[6:]}"
    assert env.client.batch_put_device_fp8_paged([key], [addrs], [page // es], cfg, _stream(), wide=W, rows=[ue]) == [bb.ErrorCode.OK]
    dense = view.index_select(1, torch.tensor(ids, device="cuda"))
    packed_want = bb.mxfp8_pack_ref(_bits(dense).cpu().numpy().reshape(-1), W)
    assert env.client.get(key) == packed_want
    out = torch.full_like(cache, 3)
    into = [5, 6, 7, 1, 2, 60]
    oa, _, _ = TensorStore._block_pages(out[:, :, :, 2:6, :], 1, np.array(into), 0)
    assert env.client.batch_get_device_fp8_paged([key], [oa], [page // es], _stream(), wide=W, rows=[ue]) == [bb.ErrorCode.OK]
    ref = torch.full_like(cache, 3)
    ref[:, :, :, 2:6, :].index_copy_(1, torch.tensor(into, device="cuda"), _mx_model(bb, dense))
    assert torch.equal(_bits(out), _bits(ref))


@pytest.mark.parametrize("tier", ["hbm", "dram", "striped"])
def test_client_rows_on_tiers(bb, env, tier):
    """The byte paged and blocks calls with rows, on HBM, on the DRAM tier and striped over both: the object is the
    dense slices, gets store exactly the rows."""
    cls = {"hbm": [bb.StorageClass.RAM_GPU], "dram": [bb.StorageClass.RAM_CPU], "striped": [bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU]}[tier]
    cfg = bb.WorkerConfig(replication_factor=2 if tier == "hbm" else 1, max_workers_per_copy=2 if tier == "striped" else 1, ttl_ms=0,
                          checksum=bb.ChecksumAlgo.XXH3, preferred_classes=cls)
    src = Blocks(64, 16, 2048, 512, 1024)
    src.fill(11)
    ids = list(range(63, 0, -3))
    dense = src.gather(ids)
    key = f"tier/{tier}"
    assert env.client.batch_put_device_paged([key], [src.addrs(ids)], [src.page], cfg, _stream(), rows=[(512, 2048)]) == [bb.ErrorCode.OK]
    assert env.client.get(key) == dense.cpu().numpy().tobytes()
    dst = Blocks(64, 16, 2048, 512, 1024)
    into = list(range(1, 64, 3))
    ecs, sizes = env.client.batch_get_device_paged([key], [dst.addrs(into)], [dst.page], _stream(), rows=[(512, 2048)])
    torch.cuda.synchronize()
    assert ecs == [bb.ErrorCode.OK] and sizes == [dense.numel()] and torch.equal(dst.buf, dst.expect(into, dense))
    d_ids = torch.tensor(into, dtype=torch.int64, device="cuda")
    dst = Blocks(64, 16, 2048, 512, 1024)
    b = bb.DeviceBlocks([dst.buf.data_ptr() + 1024], d_ids.data_ptr(), d_ids.numel(), 64, dst.block, dst.page, id_bytes=8,
                        row_width=512, row_pitch=2048)
    ecs, _ = env.client.batch_get_device_blocks([key], [b], _stream())
    torch.cuda.synchronize()
    assert ecs == [bb.ErrorCode.OK] and torch.equal(dst.buf, dst.expect(into, dense))


# ---------------------------------------------------------------- TensorStore on head slices
class _Recorder:
    """The client, recording the names of the calls made through it."""

    def __init__(self, client):
        self._c, self.log, self.kw = client, [], []

    def clear(self):
        self.log.clear()
        self.kw.clear()

    def __getattr__(self, name):
        fn = getattr(self._c, name)
        if not callable(fn):
            return fn

        def call(*a, **kw):
            self.log.append(name)
            self.kw.append(kw)
            return fn(*a, **kw)

        return call


def _whole_calls(log):
    """The calls of the index_select / index_copy_ routes: a whole put or get of a tensor."""
    return [n for n in log if n in ("batch_put_device", "batch_put_device_fp8", "batch_get_device", "batch_get_device_fp8")]


def _layouts():
    # (name, cache shape, block dim, head dim): NHD [2, blocks, block_size, H, D] and HND [blocks, 2, H, block_size, D]
    # 32 KiB pages of 4-head slices (PAGED_MIN_PAGE_BYTES)
    return [("NHD", (2, 96, 32, 8, 128), 1, 3), ("HND", (96, 2, 8, 32, 128), 0, 2)]


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("layout", ["NHD", "HND"])
def test_tensor_store_head_slices(bb, env, layout, packed):
    """put_blocks / get_blocks_into (with blocks=) and put_layer_blocks / get_layer_blocks_into (CUDA ids) of a head
    slice take the fused paged calls, store what index_select of the view stores, and restore exactly the slice's rows:
    the other heads keep their canary values."""
    from blackbird_b200.ops.tensor_store import AsyncTensorStore, TensorStore

    name, shape, dim, hdim = [l for l in _layouts() if l[0] == layout][0]
    rec = _Recorder(env.client)
    store, plain = TensorStore(rec), TensorStore(env.client)
    g = torch.Generator(device="cuda").manual_seed(21)
    cache = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    view = cache.narrow(hdim, 2, 4)
    ids = [70, 3, 41, 12, 88, 5, 60, 33]
    sel = view.index_select(dim, torch.tensor(ids, device="cuda"))
    want = _mx_model(bb, sel) if packed else sel
    key, ref = f"hs/{layout}/{packed}", f"hs/{layout}/{packed}/ref"
    store.put_blocks(key, view, ids, dim=dim, pack_fp8=packed)
    assert [n for n in rec.log if n != "device_fp8_eligible"] == ["batch_put_device_fp8_paged" if packed else "batch_put_device_paged", "batch_put"], rec.log
    plain.put(ref, sel, pack_fp8=packed)  # the fallback's object: the same bytes and #meta
    assert env.client.get(key) == env.client.get(ref) and env.client.get(key + "#meta") == env.client.get(ref + "#meta")
    assert torch.equal(_bits(store.get(key)), _bits(want))
    # restore into another cache's slice: the other heads keep their canaries
    into = [1, 2, 95, 50, 7, 8, 77, 30]
    for obj in (key, ref):
        out = torch.full_like(cache, 7.0)
        rec.clear()
        store.get_blocks_into(obj, out.narrow(hdim, 2, 4), into, dim=dim)
        assert ("batch_get_device_fp8_paged" if packed else "batch_get_device_paged") in rec.log and not _whole_calls(rec.log), rec.log
        expect = torch.full_like(cache, 7.0)
        expect.narrow(hdim, 2, 4).index_copy_(dim, torch.tensor(into, device="cuda"), want)
        assert torch.equal(_bits(out), _bits(expect)), obj
    # partial restore: stored blocks 6 and 1 into cache blocks 90 and 91
    out = torch.full_like(cache, 7.0)
    store.get_blocks_into(key, out.narrow(hdim, 2, 4), [90, 91], dim=dim, blocks=[6, 1])
    expect = torch.full_like(cache, 7.0)
    expect.narrow(hdim, 2, 4).index_copy_(dim, torch.tensor([90, 91], device="cuda"), want.index_select(dim, torch.tensor([6, 1], device="cuda")))
    assert torch.equal(_bits(out), _bits(expect))
    # per-layer caches with CUDA ids, and the async form
    layers = [torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3)]
    lviews = [c.narrow(hdim, 2, 4) for c in layers]
    d_ids = torch.tensor(ids, dtype=torch.int32, device="cuda")
    rec.clear()
    store.put_layer_blocks(key + "/l", lviews, d_ids, dim=dim, pack_fp8=packed)
    assert ("batch_put_device_fp8_blocks" if packed else "batch_put_device_blocks") in rec.log and not _whole_calls(rec.log), rec.log
    lsel = torch.stack([v.index_select(dim, d_ids.long()) for v in lviews])
    lwant = _mx_model(bb, lsel) if packed else lsel
    assert torch.equal(_bits(store.get(key + "/l")), _bits(lwant))
    outs = [torch.full_like(c, 5.0) for c in layers]
    d_into = torch.tensor(into, dtype=torch.int64, device="cuda")
    rec.clear()
    astore = AsyncTensorStore(rec)
    try:
        astore.get_layer_blocks_into_async([key + "/l"], [[o.narrow(hdim, 2, 4) for o in outs]], [d_into], dim=dim).result()
    finally:
        astore.close()
    assert ("batch_get_device_fp8_blocks" if packed else "batch_get_device_blocks") in rec.log and not _whole_calls(rec.log), rec.log
    for l, o in enumerate(outs):
        expect = torch.full_like(o, 5.0)
        expect.narrow(hdim, 2, 4).index_copy_(dim, d_into, lwant[l])
        assert torch.equal(_bits(o), _bits(expect)), l
    plain.remove([key, ref, key + "/l"])


@pytest.mark.parametrize("packed", [False, True])
def test_tp_resharding_round_trip(bb, env, packed):
    """One NHD cache of 8 heads stored as two head-shard objects (what a TP-2 side reads), restored into two narrow
    caches of 4 heads and back from them into one wide cache: bit-exact, or exact to the MXFP8 model when packed.  Every
    put and get of a head slice takes the paged calls with the row pattern (32 KiB pages), none index_select."""
    from blackbird_b200.ops.tensor_store import TensorStore

    rec = _Recorder(env.client)
    store = TensorStore(rec)
    g = torch.Generator(device="cuda").manual_seed(31)
    wide = torch.randn((2, 64, 32, 8, 128), device="cuda", generator=g).to(torch.bfloat16)
    ids = [9, 40, 2, 33, 61]
    put_call = "batch_put_device_fp8_paged" if packed else "batch_put_device_paged"
    get_call = "batch_get_device_fp8_paged" if packed else "batch_get_device_paged"

    def rows_of(name):
        """The rows argument of the last call `name`, one pattern per object."""
        return [kw.get("rows") for n, kw in zip(rec.log, rec.kw) if n == name][-1]

    for s in range(2):
        rec.clear()
        store.put_blocks(f"tp/{packed}/h{s}", wide[:, :, :, 4 * s:4 * s + 4, :], ids, dim=1, pack_fp8=packed)
        assert put_call in rec.log and not _whole_calls(rec.log), rec.log
        assert rows_of(put_call) == [(1024 // (2 if packed else 1), 2048 // (2 if packed else 1))]
    narrow = [torch.zeros((2, 64, 32, 4, 128), dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    n_ids = [0, 1, 2, 3, 4]
    for s in range(2):
        rec.clear()
        store.get_blocks_into(f"tp/{packed}/h{s}", narrow[s], n_ids, dim=1)
        assert get_call in rec.log and not _whole_calls(rec.log), rec.log
    back = torch.zeros_like(wide)
    for s in range(2):
        store.put_blocks(f"tp/{packed}/n{s}", narrow[s], n_ids, dim=1)
        rec.clear()
        store.get_blocks_into(f"tp/{packed}/n{s}", back[:, :, :, 4 * s:4 * s + 4, :], ids, dim=1)
        assert "batch_get_device_paged" in rec.log and not _whole_calls(rec.log), rec.log
        assert rows_of("batch_get_device_paged") == [(1024, 2048)]
    sel = wide.index_select(1, torch.tensor(ids, device="cuda"))
    want = torch.cat([_mx_model(bb, sel[:, :, :, 4 * s:4 * s + 4, :]) for s in range(2)], dim=3) if packed else sel
    assert torch.equal(_bits(back.index_select(1, torch.tensor(ids, device="cuda"))), _bits(want))
    others = [b for b in range(64) if b not in ids]
    assert bool((back.index_select(1, torch.tensor(others, device="cuda")) == 0).all())
    store.remove([f"tp/{packed}/{p}{s}" for p in "hn" for s in range(2)])
