"""Paged puts and gets of MXFP8-packed tensors on the GPU: the paged gathering load of the fused pack kernel and the
paged scattering store of the fused unpack kernel (XFER_PAGED) through XferEngine.run_fp8, the client's
batch_put_device_fp8_paged / batch_get_device_fp8_paged on a GpuRankCluster, and TensorStore's packed block puts and
gets.  The wide tile in shared memory is the dense tile, so every packed object and digest must equal those of run_fp8 on
the concatenated pages, and every unpack into pages must store what an unpack into a contiguous buffer stores, with the
guard bytes around and between the pages untouched."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
GRIDS = [1, 7, "sms", "2sms"]
DTYPES = [torch.bfloat16, torch.float16, torch.float32]


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


def _wide(bb, dt):
    return {torch.bfloat16: bb.MxWide.BF16, torch.float16: bb.MxWide.F16, torch.float32: bb.MxWide.F32}[dt]


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _values(n, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(n, generator=g, device="cuda") * torch.exp2(torch.randint(-10, 10, (n,), generator=g, device="cuda").float())
    v[::101] = float("nan")
    return v.to(dt)


def _packed(n):
    return torch.full((n + n // 32 + 16,), GUARD, dtype=torch.uint8, device="cuda")


def pages_index(nb, addrs, page, phase):
    """Byte offsets of object bytes [0, nb): the rule of SourcePages, in bytes."""
    y = np.arange(nb, dtype=np.int64) + phase
    return np.asarray(addrs, dtype=np.int64)[y // page] + y % page


class Arena:
    """One guard-filled byte buffer that pages are carved from, in random order, each after a guard gap and placed so
    that its address + the phase is 16-byte aligned (SourcePages::coaligned)."""

    def __init__(self, nbytes, rng):
        self.buf = torch.full((nbytes,), GUARD, dtype=torch.uint8, device="cuda")
        self.o, self.rng = 64, rng

    def pages(self, npages, page, phase):
        slots = []
        for _ in range(npages):
            self.o = (self.o + 15) // 16 * 16
            slots.append(self.o + (16 - phase % 16) % 16)
            self.o += page + 64
        assert self.o <= self.buf.numel()
        return [slots[i] for i in self.rng.permutation(npages)]

    def addr(self, offs):
        return [self.buf.data_ptr() + o for o in offs]


# (page elements in units of 16 / b, i.e. of one 16-byte granule, pages, phase elements): pages smaller than a tile and not a
# multiple of 32 elements (MX blocks straddle pages), exactly a tile, larger than a tile with a tail tile, a nonzero phase,
# one-granule pages (a tile spans 1024 or 2048 pages), a single page
def _specs(b):
    per = 16 // b
    tile = T  # elements per payload tile
    return [(3 * per, 64, 0), (tile, 2, 0), (tile + 40 * per, 3, 0), (512 * per, 5, 100 * per + 3), (per, 4096 // per * 2, 0), (tile * 2, 1, 0)]


def _n_elems(page, npages, phase):
    """The largest whole number of MX blocks the table holds from its phase, at least one block."""
    return max(32, (page * npages - phase) // 32 * 32)


class Fp8Batch:
    """A pack and an unpack batch of one wide type: paged items of every spec, plus a contiguous and a gathered (pack) or
    scattered (unpack) item, with the reference packed objects and unpacked values from run_fp8 on contiguous tensors."""

    def __init__(self, bb, eng, dt, seed=3):
        rng = np.random.default_rng(seed)
        self.bb, self.dt, self.b = bb, dt, torch.empty((), dtype=dt).element_size()
        self.wide = _wide(bb, dt)
        b = self.b
        specs = _specs(b)
        self.specs = specs
        ns = [_n_elems(p, k, ph) for p, k, ph in specs]
        self.src = Arena(sum((p * b + 128) * k for p, k, _ in specs) + MiB, rng)
        self.objs, self.src_pages = [], []
        for j, ((p, k, ph), n) in enumerate(zip(specs, ns)):
            offs = self.src.pages(k, p * b, ph * b)
            obj = _values(n, dt, seed + j)
            ix = torch.from_numpy(pages_index(n * b, offs, p * b, ph * b)).cuda()
            self.src.buf[ix] = obj.view(torch.uint8)
            self.objs.append(obj)
            self.src_pages.append((offs, p, ph))
        # a contiguous and a gathered source: rows of 5 granules every 7
        per = 16 // b
        self.plain = _values(3 * T + 64, dt, seed + 50)
        rows_src = _values(7 * per * 200, dt, seed + 51).view(200, 7 * per)
        self.rows_src = rows_src
        self.gathered = rows_src[:, :5 * per].contiguous().view(-1)
        dense = self.objs + [self.plain, self.gathered]
        # reference: run_fp8 on the contiguous tensors
        self.ref_packed = [_packed(o.numel()) for o in dense]
        self.ref_digest, st, _ = eng.run_fp8([(o.data_ptr(), p.data_ptr(), o.numel()) for o, p in zip(dense, self.ref_packed)], False,
                                             _stream(), wide=self.wide)
        self.ref_wide = [torch.empty_like(o) for o in dense]
        _, st, _ = eng.run_fp8([(w.data_ptr(), p.data_ptr(), o.numel()) for o, p, w in zip(dense, self.ref_packed, self.ref_wide)], True,
                               _stream(), wide=self.wide)
        torch.cuda.synchronize()

    def pack_items(self):
        """(items, outputs): the paged, contiguous and gathered puts into fresh guard-filled packed buffers."""
        per = 16 // self.b
        outs = [_packed(o.numel()) for o in self.objs] + [_packed(self.plain.numel()), _packed(self.gathered.numel())]
        items = [(0, out.data_ptr(), o.numel(), None, None, None, None, None, (self.src.addr(offs), p, ph))
                 for o, out, (offs, p, ph) in zip(self.objs, outs, self.src_pages)]
        items.append((self.plain.data_ptr(), outs[-2].data_ptr(), self.plain.numel()))
        items.append((self.rows_src.data_ptr(), outs[-1].data_ptr(), self.gathered.numel(), None, None, (7 * per, 5 * per, 0)))
        return items, outs

    def unpack_items(self, rng, digests=None):
        """(items, destination arena, scatter buffer, contiguous buffer): the paged, contiguous and scattered gets of the
        reference packed objects, verified against `digests` (the reference ones by default)."""
        b, per = self.b, 16 // self.b
        dg = digests or self.ref_digest
        dst = Arena(sum((p * b + 128) * k for p, k, _ in self.specs) + MiB, rng)
        dpages = [dst.pages(k, p * b, ph * b) for p, k, ph in self.specs]
        items = [(0, pk.data_ptr(), o.numel(), d, None, None, None, None, None, (dst.addr(offs), p, ph))
                 for o, pk, d, offs, (p, _, ph) in zip(self.objs, self.ref_packed, dg, dpages, self.specs)]
        contig = torch.full((self.plain.numel() * b,), GUARD, dtype=torch.uint8, device="cuda")
        items.append((contig.data_ptr(), self.ref_packed[-2].data_ptr(), self.plain.numel(), dg[-2]))
        scat = torch.full((200 * 7 * per * b,), GUARD, dtype=torch.uint8, device="cuda")
        items.append((scat.data_ptr(), self.ref_packed[-1].data_ptr(), self.gathered.numel(), dg[-1], None, None, (7 * per, 5 * per, 0)))
        return items, dst, dpages, contig, scat

    def check_unpack(self, dst, dpages, contig, scat, what):
        torch.cuda.synchronize()
        b, per = self.b, 16 // self.b
        want = torch.full_like(dst.buf, GUARD)
        for w, offs, (p, _, ph) in zip(self.ref_wide, dpages, self.specs):
            want[torch.from_numpy(pages_index(w.numel() * b, offs, p * b, ph * b)).cuda()] = w.view(torch.uint8)
        bad = (dst.buf != want).nonzero()
        assert bad.numel() == 0, (what, bad[:8].flatten().tolist())
        assert torch.equal(contig, self.ref_wide[-2].view(torch.uint8)), what
        s = scat.view(200, 7 * per * b)
        assert torch.equal(s[:, :5 * per * b].reshape(-1), self.ref_wide[-1].view(torch.uint8)), what
        assert bool((s[:, 5 * per * b:] == GUARD).all()), what


@pytest.mark.parametrize("dt", DTYPES)
def test_paged_pack_and_unpack_at_every_grid(bb, eng, dt):
    """Paged items of every shape mixed with a contiguous and a gathered (pack) or scattered (unpack) item in one launch,
    at grids of 1, 7, the SM count and twice the SM count: packed bytes and digests equal run_fp8 on torch.cat of the
    pages, unpacks into pages store the reference values and leave every guard byte, and a corrupt byte gives status 1."""
    fb = Fp8Batch(bb, eng, dt)
    rng = np.random.default_rng(9)
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        items, outs = fb.pack_items()
        dg, st, _ = eng.run_fp8(items, False, _stream(), wide=fb.wide)
        torch.cuda.synchronize()
        assert st == [0] * len(items) and dg == fb.ref_digest, g
        for out, ref in zip(outs, fb.ref_packed):
            assert torch.equal(out, ref), (g, dt)
        items, dst, dpages, contig, scat = fb.unpack_items(rng)
        dg, st, _ = eng.run_fp8(items, True, _stream(), wide=fb.wide)
        assert st == [0] * len(items) and dg == fb.ref_digest, g
        fb.check_unpack(dst, dpages, contig, scat, f"{dt} grid={g}")
    eng.set_max_ctas(0)
    # a corrupt payload byte of one paged object: its status is 1, the others verify
    k = 2
    fb.ref_packed[k][777] ^= 0xFF
    try:
        items, *_ = fb.unpack_items(rng)
        _, st, _ = eng.run_fp8(items, True, _stream(), wide=fb.wide)
        assert st == [1 if j == k else 0 for j in range(len(items))]
    finally:
        fb.ref_packed[k][777] ^= 0xFF


def test_paged_fp8_after_paged_bb_xfer_and_a_growing_table(bb, eng):
    """A paged fp8 batch on the slot that last ran a paged bb_xfer batch, a non-paged fp8 batch after it, and a table of
    131,072 pages of 16 bytes that makes the slot's descriptor table grow: each equals its contiguous reference."""
    rng = np.random.default_rng(5)
    src = torch.randint(0, 256, (8 * MiB,), dtype=torch.uint8, device="cuda")
    dst = torch.zeros(MiB, dtype=torch.uint8, device="cuda")
    offs = [int(o) * 4096 for o in rng.permutation(64)[:40]]
    eng.run([(0, dst.data_ptr(), 40 * 4096, 0, 0, 0, None, None, None, ([src.data_ptr() + o for o in offs], 4096, 0))], bb.ChecksumAlgo.XXH3,
            _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst[:40 * 4096], torch.cat([src[o:o + 4096] for o in offs]))
    for npages, per_page in ((300, 64), (131072, 8)):  # bf16 pages of 128 and 16 bytes
        n = npages * per_page
        ar = Arena(npages * (per_page * 2 + 64) + MiB, rng)
        poffs = ar.pages(npages, per_page * 2, 0)
        obj = _values(n, torch.bfloat16, npages)
        ar.buf[torch.from_numpy(pages_index(n * 2, poffs, per_page * 2, 0)).cuda()] = obj.view(torch.uint8)
        ref, out = _packed(n), _packed(n)
        rdg, _, _ = eng.run_fp8([(obj.data_ptr(), ref.data_ptr(), n)], False, _stream())
        dg, st, _ = eng.run_fp8([(0, out.data_ptr(), n, None, None, None, None, None, (ar.addr(poffs), per_page, 0))], False, _stream())
        torch.cuda.synchronize()
        assert dg == rdg and st == [0] and torch.equal(out, ref), npages
        # a plain gathered fp8 batch right after, on the same slot: no page entry of the batch before carries over
        rows = obj.view(-1, 64)[:, :32].contiguous().view(-1)
        gref, gout = _packed(rows.numel()), _packed(rows.numel())
        rdg, _, _ = eng.run_fp8([(rows.data_ptr(), gref.data_ptr(), rows.numel())], False, _stream())
        dg, st, _ = eng.run_fp8([(obj.data_ptr(), gout.data_ptr(), rows.numel(), None, None, (64, 32, 0))], False, _stream())
        torch.cuda.synchronize()
        assert dg == rdg and torch.equal(gout, gref)
        # and the paged unpack of the same object back into fresh pages
        back = Arena(npages * (per_page * 2 + 64) + MiB, rng)
        boffs = back.pages(npages, per_page * 2, 0)
        want = torch.empty_like(obj)
        eng.run_fp8([(want.data_ptr(), ref.data_ptr(), n)], True, _stream())
        _, st, _ = eng.run_fp8([(0, ref.data_ptr(), n, None, None, None, None, None, None, (back.addr(boffs), per_page, 0))],
                               True, _stream())
        torch.cuda.synchronize()
        expect = torch.full_like(back.buf, GUARD)
        expect[torch.from_numpy(pages_index(n * 2, boffs, per_page * 2, 0)).cuda()] = want.view(torch.uint8)
        assert torch.equal(back.buf, expect), npages


def test_rejected_paged_fp8_items(bb, eng):
    """Pages on the wrong side, with rows or a window, short tables, phase >= page, wide-byte overflow and misaligned pages
    are refused before any launch, and nothing is written."""
    src = _values(8 * T, torch.bfloat16, 1)
    s = src.data_ptr()
    packed = _packed(8 * T)
    wide = torch.full((8 * T * 2,), GUARD, dtype=torch.uint8, device="cuda")
    p, w = packed.data_ptr(), wide.data_ptr()
    sp = ([s, s + 4 * T, s + 2 * T], 1024, 0)  # 1024 elements = 2 KiB pages
    dp = ([w + 4 * T, w, w + 2 * T], 1024, 0)
    IA, IAD = "INVALID_ARGUMENT", "INVALID_ADDRESS"
    ok_pack = (s, p + 2 * T, 64)
    ok_unpack = (w + 8 * T, p, 64)
    # refused packs
    for it, err in [((0, p, 1024, None, None, None, None, None, None, dp), IA),              # destination pages on a pack
                    ((s, p, 1024, None, None, (96, 64, 0), None, None, sp), IA),            # with source rows
                    ((0, p, 1024, None, (0, 512), None, None, None, sp), IA),               # with a window
                    ((0, p, 3 * 1024 + 32, None, None, None, None, None, sp), IA),          # table too short
                    ((0, p, 3 * 1024 - 32, None, None, None, None, None, (sp[0], 1024, 64)), IA),  # too short with the phase
                    ((0, p, 32, None, None, None, None, None, (sp[0], 1024, 1024)), IA),    # phase >= page
                    ((0, p, 32, None, None, None, None, None, ([s], 1 << 63, 0)), IA),      # page overflows in wide bytes
                    ((0, p, 1024, None, None, None, None, None, ([s + 2, s + 4 * T], 1024, 0)), IAD),  # first page
                    ((0, p, 2048, None, None, None, None, None, ([s, s + 4 * T + 8], 1024, 0)), IAD),  # later page
                    ((0, p, 2048, None, None, None, None, None, ([s, s + 4 * T, s + T], 1020, 0)), IAD),  # 2 * page % 16
                    ((0, p, 512, None, None, None, None, None, ([s], 1024, 3)), IAD)]:      # first page + phase
        with pytest.raises(RuntimeError, match=err):
            eng.run_fp8([ok_pack, it], False, _stream())
    torch.cuda.synchronize()
    assert bool((packed == GUARD).all())
    # refused unpacks (the packed buffer is read only)
    for it, err in [((0, p, 1024, None, None, None, None, None, sp), IA),                   # source pages on an unpack
                    ((w, p, 1024, None, None, None, (96, 64, 0), None, None, dp), IA),      # with destination rows
                    ((0, p, 1024, None, (0, 512), None, None, None, None, dp), IA),         # with a window
                    ((0, p, 3 * 1024 + 32, None, None, None, None, None, None, dp), IA),    # table too short
                    ((0, p, 1024, None, None, None, None, None, None, ([w + 8, w + 4 * T], 1024, 0)), IAD)]:
        with pytest.raises(RuntimeError, match=err):
            eng.run_fp8([ok_unpack, it], True, _stream())
    torch.cuda.synchronize()
    assert bool((wide == GUARD).all())
    # fp32 needs page % 4 elements, not % 8: pages of 1012 elements (4048 bytes) are co-aligned; 2016 elements end in the
    # second page
    src32 = _values(4 * 1024, torch.float32, 2)
    t = src32.data_ptr()
    ref, out = _packed(2016), _packed(2016)
    dense = torch.cat([src32[:1012], src32[1024:1024 + 1004]])
    rdg, _, _ = eng.run_fp8([(dense.data_ptr(), ref.data_ptr(), 2016)], False, _stream(), wide=bb.MxWide.F32)
    dg, st, _ = eng.run_fp8([(0, out.data_ptr(), 2016, None, None, None, None, None, ([t, t + 4096], 1012, 0))], False, _stream(),
                            wide=bb.MxWide.F32)
    torch.cuda.synchronize()
    assert dg == rdg and st == [0] and torch.equal(out, ref)


# ---------------------------------------------------------------------------------------------------- client
def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, replicas=1):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.client.get_workers(key)]


def _flip(cl, sh, pos):
    be = cl.worker.backend(sh.pool_id)
    be.write(sh.offset + pos, bytes([be.read(sh.offset + pos, 1)[0] ^ 0xFF]))


@pytest.mark.parametrize("dt", DTYPES)
def test_client_paged_puts_and_gets(bb, dt):
    """Paged puts with 2 and 3 copies read back by a plain batch_get_device_fp8, plain puts read back by paged gets into a
    guard-filled cache, digests equal to those of a plain put of the concatenation, and a corrupt copy failed over."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-fp8pg-{str(dt)[6:]}", max_replicas=3)
    try:
        E, wd, b = bb.ErrorCode, _wide(bb, dt), torch.empty((), dtype=dt).element_size()
        per_block = 8192 // b * 2  # 16 KiB blocks
        cache = _values(64 * per_block, dt, 4).view(64, per_block)
        rng = np.random.default_rng(6)
        sel = [list(rng.permutation(64)[:k]) for k in (40, 9)]
        keys = ["p2", "p3"]
        for key, ids, rep in zip(keys, sel, (2, 3)):
            n0 = _counter(cl.client, "device_put_fp8_paged_total")
            ecs = cl.client.batch_put_device_fp8_paged([key], [[cache[i].data_ptr() for i in ids]], [per_block], _cfg(bb, rep), _stream(), wide=wd)
            assert ecs == [E.OK] and _counter(cl.client, "device_put_fp8_paged_total") == n0 + 1
            assert len(cl.client.get_workers(key)) == rep
            dense = cache[torch.tensor(ids, device="cuda")].contiguous().view(-1)
            assert cl.client.batch_put_device_fp8([key + "/c"], [dense.data_ptr()], [dense.numel()], _cfg(bb, rep), _stream(), wide=wd) == [E.OK]
            assert _sums(cl, key) == _sums(cl, key + "/c")
            # the paged object through a plain get, and the plain object through a paged get
            whole = torch.empty_like(dense)
            assert cl.client.batch_get_device_fp8([key], [whole.data_ptr()], [dense.numel()], _stream(), wide=wd) == [E.OK]
            ref = torch.empty_like(dense)
            assert cl.client.batch_get_device_fp8([key + "/c"], [ref.data_ptr()], [dense.numel()], _stream(), wide=wd) == [E.OK]
            torch.cuda.synchronize()
            assert torch.equal(_bits(whole), _bits(ref))
            dst = torch.full((64 * per_block * b,), GUARD, dtype=torch.uint8, device="cuda").view(64, -1)
            new = list(rng.permutation(64)[:len(ids)])
            g0 = _counter(cl.client, "device_get_fp8_paged_total")
            for copy in [None] + [c.shards[0] for c in cl.client.get_workers(key + "/c")]:
                if copy is not None:  # one corrupt copy at a time: the get fails over
                    _flip(cl, copy, 999)
                dst.fill_(GUARD)
                ecs = cl.client.batch_get_device_fp8_paged([key + "/c"], [[dst[i].data_ptr() for i in new]], [per_block], _stream(), wide=wd)
                assert ecs == [E.OK]
                torch.cuda.synchronize()
                want = torch.full_like(dst, GUARD)
                want[torch.tensor(new, device="cuda")] = ref.view(torch.uint8).view(len(ids), -1)
                assert torch.equal(dst, want), (key, copy)
                if copy is not None:
                    _flip(cl, copy, 999)
            assert _counter(cl.client, "device_get_fp8_paged_total") == g0 + rep + 1
        # refusals fail alone: a size mismatch, a misaligned page; the third item is read
        dst = torch.full((64 * per_block * b,), GUARD, dtype=torch.uint8, device="cuda").view(64, -1)
        ecs = cl.client.batch_get_device_fp8_paged(["p3", "p3", "p3"], [[dst[i].data_ptr() for i in range(10)],
                                                                         [dst[i].data_ptr() + 2 for i in range(9)],
                                                                         [dst[i].data_ptr() for i in range(9)]], [per_block] * 3, _stream(), wide=wd)
        assert ecs == [E.INVALID_ARGUMENT, E.NOT_IMPLEMENTED, E.OK]
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore
@pytest.mark.parametrize("dt", DTYPES)
def test_tensor_store_packed_blocks(bb, dt):
    """put_blocks(pack_fp8=True) + get is bit for bit put(index_select, pack_fp8=True) + get, with the same digests;
    get_blocks_into equals index_copy_ of the unpacked blocks and leaves the other blocks; the paged route takes the paged
    calls and allocates no full-size temporary."""
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-fp8pg-ts-{str(dt)[6:]}")
    try:
        store = TensorStore(cl.client)
        cache = _values(4 * 2 * 48 * 16 * 8 * 128, dt, 7).view(4, 2, 48, 16, 8, 128)
        rng = np.random.default_rng(8)
        for dim, ids in ((0, [3, 1]), (2, list(rng.permutation(48)[:24])), (2, torch.tensor([5, 30, 2], device="cuda"))):
            key = f"b{dim}-{len(ids)}"
            idx = torch.as_tensor(ids if not isinstance(ids, torch.Tensor) else ids.cpu(), dtype=torch.int64, device="cuda")
            sel = cache.index_select(dim, idx)
            store.put(key + "/ref", sel, pack_fp8=True)
            torch.cuda.synchronize()
            p0, g0 = _counter(cl.client, "device_put_fp8_paged_total"), _counter(cl.client, "device_get_fp8_paged_total")
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            store.put_blocks(key, cache, ids, dim=dim, pack_fp8=True)
            torch.cuda.synchronize()
            put_extra = torch.cuda.max_memory_allocated() - base
            assert _counter(cl.client, "device_put_fp8_paged_total") == p0 + 1
            assert _sums(cl, key) == _sums(cl, key + "/ref")
            ref = store.get(key + "/ref")
            got = store.get(key)
            assert got.dtype == dt and got.shape == sel.shape and torch.equal(_bits(got), _bits(ref))
            dst = torch.full_like(cache, 7)
            perm = list(rng.permutation(cache.shape[dim])[:sel.shape[dim]])
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            store.get_blocks_into(key, dst, perm, dim=dim)
            torch.cuda.synchronize()
            get_extra = torch.cuda.max_memory_allocated() - base
            assert _counter(cl.client, "device_get_fp8_paged_total") == g0 + 1
            want = torch.full_like(cache, 7).index_copy_(dim, torch.as_tensor(perm, dtype=torch.int64, device="cuda"), ref)
            assert torch.equal(_bits(dst), _bits(want)), (dim, ids)
            full = sel.numel() * sel.element_size()
            assert put_extra < full // 8 and get_extra < full // 8, (put_extra, get_extra, full)
    finally:
        cl.stop()


def test_tensor_store_packed_block_fallbacks(bb):
    """Pages below FP8_PAGED_MIN_PAGE_BYTES, misaligned pages and an unfusable config take index_select + put / get +
    index_copy_ with the same results; a dtype MXFP8 does not take raises TypeError before anything is stored; the async
    forms route through the paged calls."""
    from blackbird_b200.ops.tensor_store import AsyncTensorStore, TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-fp8pg-ts-fb", dram_bytes=64 << 20)
    try:
        store = TensorStore(cl.client)
        unfusable = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096,
                                    preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        flat = _values(4 * 2 * 32 * 16 * 8 * 128 + 8, torch.bfloat16, 9)
        cases = [("small", _values(4 * 2 * 32 * 4 * 8 * 128, torch.bfloat16, 10).view(4, 2, 32, 4, 8, 128), None),  # 8 KiB pages
                 ("skew", flat[1:1 + 4 * 2 * 32 * 16 * 8 * 128].view(4, 2, 32, 16, 8, 128), None),             # 2 bytes off
                 ("unfus", flat[:4 * 2 * 32 * 16 * 8 * 128].view(4, 2, 32, 16, 8, 128), unfusable)]
        p0, g0 = _counter(cl.client, "device_put_fp8_paged_total"), _counter(cl.client, "device_get_fp8_paged_total")
        for key, cache, cfg in cases:
            ids = [7, 0, 20]
            sel = cache.index_select(2, torch.tensor(ids, device="cuda"))
            store.put(key + "/ref", sel, pack_fp8=True, config=cfg)
            store.put_blocks(key, cache, ids, dim=2, pack_fp8=True, config=cfg)
            ref = store.get(key + "/ref")
            assert torch.equal(_bits(store.get(key)), _bits(ref)), key
            dst = torch.full_like(cache, 3)
            store.get_blocks_into(key, dst, [1, 2, 0], dim=2)
            want = torch.full_like(cache, 3).index_copy_(2, torch.tensor([1, 2, 0], device="cuda"), ref)
            assert torch.equal(_bits(dst), _bits(want)), key
        assert _counter(cl.client, "device_put_fp8_paged_total") == p0
        # the unfusable object: its fused paged get (if it was striped) answered NOT_IMPLEMENTED and fell back; the others
        # never reached the paged get
        assert _counter(cl.client, "device_get_fp8_paged_total") <= g0 + 1
        with pytest.raises(TypeError):
            store.put_blocks("never", torch.zeros(4, 2, 32, 16, 8, 128, dtype=torch.int8, device="cuda"), [0], dim=2, pack_fp8=True)
        assert not cl.client.object_exists("never") and not cl.client.object_exists("never#meta")
        # async: the side stream waits for the caller's writes, and the paged calls serve both directions
        base = cases[2][1]
        astore = AsyncTensorStore(cl.client)
        try:
            src = torch.zeros_like(base)
            torch.cuda._sleep(20_000_000)
            src.copy_(base)
            p1, g1 = _counter(cl.client, "device_put_fp8_paged_total"), _counter(cl.client, "device_get_fp8_paged_total")
            astore.put_blocks_async(["a"], [src], [[3, 7]], dim=2, pack_fp8=True).result()
            out = torch.full_like(base, 1)
            res = astore.get_blocks_into_async(["a"], [out], [[0, 5]], dim=2).result()
            assert res[0] is out
            assert _counter(cl.client, "device_put_fp8_paged_total") == p1 + 1
            assert _counter(cl.client, "device_get_fp8_paged_total") == g1 + 1
            store.put("a/ref", base.index_select(2, torch.tensor([3, 7], device="cuda")), pack_fp8=True)
            want = torch.full_like(base, 1).index_copy_(2, torch.tensor([0, 5], device="cuda"), store.get("a/ref"))
            assert torch.equal(_bits(out), _bits(want))
        finally:
            astore.close()
    finally:
        cl.stop()
