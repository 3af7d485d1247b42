"""Segment-list puts and gets of MXFP8-packed tensors on the GPU: the segment-table gathering load of the fused pack
kernel and the segmented scattering store of the fused unpack kernel (XFER_SEGMENTS in bb_xfer_fp8) through
XferEngine.run_fp8, the client's batch_put_device_fp8_segments / batch_get_device_fp8_segments on a GpuRankCluster, and
TensorStore's packed bundles.  The wide tile in shared memory is the dense tile of the concatenation, so every packed
object and digest must equal those of run_fp8 on the concatenated segments, and every unpack into segments must store
what an unpack into a contiguous buffer stores, with the guard bytes around and between the segments untouched."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384
MiB = 1 << 20
GUARD = 0xA5
GRIDS = [1, 7, "sms", "2sms"]
DTYPES = [torch.bfloat16, torch.float16, torch.float32]
N10 = [None] * 10


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need CUDA (marked gpu)")


@pytest.fixture(scope="module")
def _engine():
    from blackbird_b200 import _bb

    return _bb.XferEngine(0, 8192, 2)


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
    v = torch.randn(max(n, 1), generator=g, device="cuda") * torch.exp2(torch.randint(-10, 10, (max(n, 1),), generator=g, device="cuda").float())
    v[::101] = float("nan")
    return v[:n].to(dt)


def _packed(n):
    return torch.full((n + n // 32 + 16,), GUARD, dtype=torch.uint8, device="cuda")


class Carver:
    """Byte regions of one buffer, each after a guard gap, placed so that region + align_at is 16-byte aligned."""

    def __init__(self):
        self.o = 64

    def region(self, n, align_at=0):
        self.o = (self.o + 15) // 16 * 16 + (16 - align_at % 16) % 16
        at = self.o
        self.o += n + 48
        return at

    def segments(self, lens, b, off, rng, null=0.0):
        """Byte offsets of segments of lens elements of b bytes (None: a null segment), segment k co-aligned for a
        descriptor that starts at element off (address = b * (start - off) mod 16), carved in random order."""
        starts = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        at = [0] * len(lens)
        for k in rng.permutation(len(lens)):
            at[k] = self.region(b * int(lens[k]) + 16, b * int(off - starts[k]))
        return [None if rng.random() < null else a for a in at]


def seg_index(lens, at, b):
    """Per wide byte of the object, the buffer offset it lives at (-1 in a null segment)."""
    return np.concatenate([np.arange(b * n) + a if a is not None else np.full(b * n, -1) for n, a in zip(lens, at)] or [np.zeros(0, np.int64)])


def seg_lens(rng, kind):
    if kind == "many-short":  # thousands of 1-23 element segments per tile
        lens = [int(x) for x in rng.integers(1, 24, 4000)]
    elif kind == "long":  # one segment over many tiles, zero-length and short ones around it
        lens = [5, 0, 40 * T + 3, 17, 0, 2 * T]
    else:
        lens = [int(rng.choice([0, 1, 15, 31, 33, 100, 4096, T - 1, T + 33])) for _ in range(40)]
    lens.append(-sum(lens) % 32 + 32)  # a whole number of MX blocks, rarely a whole number of tiles: a tail tile
    return lens


class SegBatch:
    """A pack and an unpack batch of one wide type: segment items of every kind, descriptors starting inside the table, a
    contiguous, a paged and a gathered (pack) or scattered (unpack) item, with the reference packed objects and
    unpacked values from run_fp8 on contiguous tensors."""

    def __init__(self, bb, eng, dt, seed=3):
        rng = np.random.default_rng(seed)
        self.dt, self.wide, b = dt, _wide(bb, dt), torch.empty((), dtype=dt).element_size()
        self.b, per = b, 16 // b
        src_c, self.dst_c = Carver(), Carver()
        self.specs = []  # (lens, off, source byte offsets, destination byte offsets)
        for kind in ("many-short", "long", "mixed"):
            for off in (0, 4096 + 32):
                lens = seg_lens(rng, kind)
                self.specs.append((lens, off, src_c.segments(lens, b, off, rng), self.dst_c.segments(lens, b, off, rng, null=0.15)))
        self.page_offs = [src_c.region(1024 * b) for _ in range(3)][::-1]
        self.dpage_offs = [self.dst_c.region(1024 * b) for _ in range(3)][::-1]
        self.src = torch.full((src_c.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        self.objs = []
        for j, (lens, off, at, _) in enumerate(self.specs):
            ix = torch.from_numpy(seg_index(lens, at, b)[b * off:]).cuda()
            obj = _values(ix.numel() // b, dt, seed + j)
            self.src[ix] = obj.view(torch.uint8)
            self.objs.append(obj)
        self.paged = _values(3 * 1024, dt, seed + 40)
        for k, o in enumerate(self.page_offs):
            self.src[o:o + 1024 * b] = self.paged[k * 1024:(k + 1) * 1024].view(torch.uint8)
        self.plain = _values(3 * T + 64, dt, seed + 50)
        self.rows_src = _values(7 * per * 200, dt, seed + 51).view(200, 7 * per)
        self.gathered = self.rows_src[:, :5 * per].contiguous().view(-1)
        dense = self.objs + [self.plain, self.paged, self.gathered]
        self.ref_packed = [_packed(o.numel()) for o in dense]
        self.ref_digest, _, _ = eng.run_fp8([(o.data_ptr(), p.data_ptr(), o.numel()) for o, p in zip(dense, self.ref_packed)], False, _stream(),
                                            wide=self.wide)
        self.ref_wide = [torch.empty_like(o) for o in dense]
        eng.run_fp8([(w.data_ptr(), p.data_ptr(), o.numel()) for o, p, w in zip(dense, self.ref_packed, self.ref_wide)], True, _stream(),
                    wide=self.wide)
        torch.cuda.synchronize()

    def _pairs(self, base, lens, at):
        return [(0 if a is None else base + a, n) for a, n in zip(at, lens)]

    def pack_items(self):
        per, S = 16 // self.b, self.src.data_ptr()
        outs = [_packed(o.numel()) for o in self.objs + [self.plain, self.paged, self.gathered]]
        items = [(0, out.data_ptr(), o.numel(), *N10, (self._pairs(S, lens, at), off, self.b))
                 for o, out, (lens, off, at, _) in zip(self.objs, outs, self.specs)]
        items.append((self.plain.data_ptr(), outs[-3].data_ptr(), self.plain.numel()))
        items.append((0, outs[-2].data_ptr(), self.paged.numel(), None, None, None, None, None, ([S + o for o in self.page_offs], 1024, 0)))
        items.append((self.rows_src.data_ptr(), outs[-1].data_ptr(), self.gathered.numel(), None, None, (7 * per, 5 * per, 0)))
        return items, outs

    def unpack_items(self):
        per, b = 16 // self.b, self.b
        dst = torch.full((self.dst_c.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        D = dst.data_ptr()
        items = [(0, pk.data_ptr(), o.numel(), d, *N10, (self._pairs(D, lens, dat), off, b))
                 for o, pk, d, (lens, off, _, dat) in zip(self.objs, self.ref_packed, self.ref_digest, self.specs)]
        contig = torch.full((self.plain.numel() * b,), GUARD, dtype=torch.uint8, device="cuda")
        items.append((contig.data_ptr(), self.ref_packed[-3].data_ptr(), self.plain.numel(), self.ref_digest[-3]))
        items.append((0, self.ref_packed[-2].data_ptr(), self.paged.numel(), self.ref_digest[-2], None, None, None, None, None,
                      ([D + o for o in self.dpage_offs], 1024, 0)))
        scat = torch.full((200 * 7 * per * b,), GUARD, dtype=torch.uint8, device="cuda")
        items.append((scat.data_ptr(), self.ref_packed[-1].data_ptr(), self.gathered.numel(), self.ref_digest[-1], None, None, (7 * per, 5 * per, 0)))
        return items, dst, contig, scat

    def check_unpack(self, dst, contig, scat, what):
        torch.cuda.synchronize()
        b, per = self.b, 16 // self.b
        want = torch.full_like(dst, GUARD)
        for w, (lens, off, _, dat) in zip(self.ref_wide, self.specs):
            ix = torch.from_numpy(seg_index(lens, dat, b)[b * off:]).cuda()
            keep = ix >= 0
            want[ix[keep]] = w.view(torch.uint8)[keep]
        for k, o in enumerate(self.dpage_offs):
            want[o:o + 1024 * b] = self.ref_wide[-2][k * 1024:(k + 1) * 1024].view(torch.uint8)
        bad = (dst != want).nonzero()
        assert bad.numel() == 0, (what, bad[:8].flatten().tolist())
        assert torch.equal(contig, self.ref_wide[-3].view(torch.uint8)), what
        s = scat.view(200, 7 * per * b)
        assert torch.equal(s[:, :5 * per * b].reshape(-1), self.ref_wide[-1].view(torch.uint8)), what
        assert bool((s[:, 5 * per * b:] == GUARD).all()), what


@pytest.mark.parametrize("dt", DTYPES)
def test_segment_pack_and_unpack_at_every_grid(bb, eng, dt):
    """Segment items -- thousands of 1-23 element segments per tile, one segment over forty tiles, zero-length segments,
    MX blocks straddling segments, tail tiles, descriptors that start inside the table, null destination segments --
    mixed with contiguous, paged and gathered / scattered items in one launch, at grids of 1, 7, the SM count and twice
    the SM count: packed bytes and digests equal run_fp8 of the concatenation, unpacks store the reference values and
    leave every guard byte, and a corrupt byte gives status 1."""
    sb = SegBatch(bb, eng, dt)
    for g in GRIDS:
        eng.set_max_ctas(_grid(g))
        items, outs = sb.pack_items()
        dg, st, _ = eng.run_fp8(items, False, _stream(), wide=sb.wide)
        torch.cuda.synchronize()
        assert st == [0] * len(items) and dg == sb.ref_digest, g
        for j, (out, ref) in enumerate(zip(outs, sb.ref_packed)):
            assert torch.equal(out, ref), (g, dt, j)
        items, dst, contig, scat = sb.unpack_items()
        dg, st, _ = eng.run_fp8(items, True, _stream(), wide=sb.wide)
        assert st == [0] * len(items) and dg == sb.ref_digest, g
        sb.check_unpack(dst, contig, scat, f"{dt} grid={g}")
    eng.set_max_ctas(0)
    k = 0
    sb.ref_packed[k][777] ^= 0xFF
    try:
        items, *_ = sb.unpack_items()
        _, st, _ = eng.run_fp8(items, True, _stream(), wide=sb.wide)
        assert st == [1 if j == k else 0 for j in range(len(items))]
    finally:
        sb.ref_packed[k][777] ^= 0xFF


def test_rejected_segment_fp8_items(bb, eng):
    """Segments on the wrong side, with a window, null in a pack, in another unit, too short, not co-aligned in wide bytes,
    or not a whole number of MX blocks, are refused before any launch, and nothing is written."""
    src = _values(8 * T, torch.bfloat16, 1)
    s = src.data_ptr()
    packed = _packed(8 * T)
    wide = torch.full((8 * T * 2,), GUARD, dtype=torch.uint8, device="cuda")
    p, w = packed.data_ptr(), wide.data_ptr()
    sg = [(s, 100), (s + 4 * T + 200, 1948)]  # 2048 elements; the second at element 100 = byte 200
    dg = [(w + 4 * T + 200, 100), (w, 1948)]
    IA, IAD = "INVALID_ARGUMENT", "INVALID_ADDRESS"
    ok_pack, ok_unpack = (s, p + 2 * T, 64), (w + 8 * T, p, 64)
    N9 = [None] * 9
    for it, err in [((0, p, 2048, *N10, None, (sg, 0, 2)), IA),                       # destination segments on a pack
                    ((0, p, 2048, None, (0, 512), *N9[:8], (sg, 0, 2)), IA),          # with a window
                    ((0, p, 2048, *N10, ([(s, 100), (0, 1948)], 0, 2)), IA),          # a null segment
                    ((0, p, 2048, *N10, ([(s, 200), (s + 4 * T + 200, 3896)], 0)), IA),  # a table of bytes
                    ((0, p, 2048, *N10, (sg, 0, 4)), IA),                             # fp32 elements on a bf16 item
                    ((0, p, 2080, *N10, (sg, 0, 2)), IA),                             # table too short
                    ((0, p, 2040, *N10, (sg, 0, 2)), IA),                             # not whole MX blocks
                    ((0, p, 2048, *N10, ([(s, 100), (s + 4 * T + 202, 1948)], 0, 2)), IAD),  # second segment off by one element
                    ((0, p, 1024, *N10, (sg, 97, 2)), IAD)]:                          # from element 97: 194 bytes into entry 0
        with pytest.raises(RuntimeError, match=err):
            eng.run_fp8([ok_pack, it], False, _stream())
    torch.cuda.synchronize()
    assert bool((packed == GUARD).all())
    for it, err in [((0, p, 2048, *N10, (dg, 0, 2)), IA),                             # source segments on an unpack
                    ((0, p, 2048, None, (0, 512), *N9, (dg, 0, 2)), IA),              # with a window
                    ((0, p, 2080, None, *N10, (dg, 0, 2)), IA),                       # table too short
                    ((0, p, 2048, None, *N10, ([(w + 4 * T + 202, 100), (w, 1948)], 0, 2)), IAD)]:
        with pytest.raises(RuntimeError, match=err):
            eng.run_fp8([ok_unpack, it], True, _stream())
    torch.cuda.synchronize()
    assert bool((wide == GUARD).all())


# ---------------------------------------------------------------------------------------------------- client
def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _sums(cl, key):
    return [[sh.checksum for sh in cp.shards] for cp in cl.client.get_workers(key)]


@pytest.mark.parametrize("dt", DTYPES)
def test_client_segment_puts_and_gets(bb, dt):
    """Segment puts with 1-3 copies in HBM and one in DRAM: digests equal those of a plain packed put of the
    concatenation, a plain fp8 get reads them, segment gets of the plain object fill the segments (nulls not stored) and
    nothing else, and a corrupt copy is failed over."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-fp8sg-{str(dt)[6:]}", dram_bytes=128 << 20, max_replicas=3)
    try:
        E, wd, b = bb.ErrorCode, _wide(bb, dt), torch.empty((), dtype=dt).element_size()
        pools = {p.id: p for p in cl.client.keystone().get_memory_pools()}
        rng = np.random.default_rng(6)
        cfgs = [bb.WorkerConfig(replication_factor=r, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU]) for r in (1, 2, 3)]
        cfgs.append(bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_CPU]))
        for j, (cfg, kind) in enumerate(zip(cfgs, ("mixed", "many-short", "long", "mixed"))):
            key = f"s{j}"
            lens = seg_lens(rng, kind)
            n = sum(lens)
            c_src, c_dst = Carver(), Carver()
            at = c_src.segments(lens, b, 0, rng)
            dat = c_dst.segments(lens, b, 0, rng, null=0.2)
            src = torch.full((c_src.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
            obj = _values(n, dt, 10 + j)
            src[torch.from_numpy(seg_index(lens, at, b)).cuda()] = obj.view(torch.uint8)
            pairs = [(src.data_ptr() + a, m) for a, m in zip(at, lens)]
            p0 = _counter(cl.client, "device_put_fp8_segments_total")
            assert cl.client.batch_put_device_fp8_segments([key], [pairs], cfg, _stream(), wide=wd) == [E.OK]
            assert _counter(cl.client, "device_put_fp8_segments_total") == p0 + 1
            assert cl.client.batch_put_device_fp8([key + "/c"], [obj.data_ptr()], [n], cfg, _stream(), wide=wd) == [E.OK]
            assert _sums(cl, key) == _sums(cl, key + "/c") and len(cl.client.get_workers(key)) == cfg.replication_factor
            whole, ref = torch.empty_like(obj), torch.empty_like(obj)
            assert cl.client.batch_get_device_fp8([key, key + "/c"], [whole.data_ptr(), ref.data_ptr()], [n, n], _stream(), wide=wd) == [E.OK] * 2
            torch.cuda.synchronize()
            assert torch.equal(_bits(whole), _bits(ref)), key
            dst = torch.full((c_dst.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
            dix = torch.from_numpy(seg_index(lens, dat, b)).cuda()
            want = torch.full_like(dst, GUARD)
            want[dix[dix >= 0]] = ref.view(torch.uint8)[dix >= 0]
            dpairs = [(0 if a is None else dst.data_ptr() + a, m) for a, m in zip(dat, lens)]
            copies = [c.shards[0] for c in cl.client.get_workers(key)] if cfg.replication_factor > 1 else []
            for copy in [None] + copies:
                if copy is not None:  # one corrupt copy at a time: the get fails over to another
                    be = cl.worker.backend(copy.pool_id)
                    off = (copy.offset if copy.location["kind"] == "gpu" else copy.location["remote_addr"] - pools[copy.pool_id].ucx_remote_addr) + 999
                    be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))
                dst.fill_(GUARD)
                ecs, sizes = cl.client.batch_get_device_fp8_segments([key], [dpairs], _stream(), wide=wd)
                assert ecs == [E.OK] and sizes == [n], (key, copy)
                torch.cuda.synchronize()
                assert torch.equal(dst, want), (key, copy)
                if copy is not None:
                    be.write(off, bytes([be.read(off, 1)[0] ^ 0xFF]))
        # refusals fail alone: one MX block short, a segment off its co-aligned address; the all-null third item is read
        # and verified and stores nothing
        dst.fill_(GUARD)
        ecs, _ = cl.client.batch_get_device_fp8_segments(["s3"] * 3, [[(0, n - 32)], [(dst.data_ptr() + b, 32), (0, n - 32)], [(0, n)]],
                                                         _stream(), wide=wd)
        assert ecs == [E.INVALID_ARGUMENT, E.NOT_IMPLEMENTED, E.OK]
        torch.cuda.synchronize()
        assert bool((dst == GUARD).all())
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore
class Recorder:
    """Wraps a client and counts its calls by name."""

    def __init__(self, client):
        self._c, self.calls = client, {}

    def __getattr__(self, name):
        f = getattr(self._c, name)

        def wrap(*a, **kw):
            self.calls[name] = self.calls.get(name, 0) + 1
            return f(*a, **kw)

        return wrap if callable(f) else f


def _bundle(dt, seed):
    b = {"zero_d": _values(1, dt, seed).view(()), "empty": _values(0, dt, seed + 1).view(0, 3), "odd": _values(33, dt, seed + 2),
         "mat": _values(7 * 13, dt, seed + 3).view(7, 13), "big": _values(T + 5, dt, seed + 4), "one": _values(32, dt, seed + 5)}
    b["nc"] = _values(6 * 10, dt, seed + 6).view(6, 10).t()         # not contiguous: copied first
    b["skew"] = _values(40, dt, seed + 7)[1:20]                      # 2 or 4 bytes off alignment: copied first
    return b


@pytest.mark.parametrize("dt", DTYPES)
def test_tensor_store_packed_bundles(bb, dt):
    """put_bundle(pack_fp8=True) of 0-d, zero-element, odd-sized, non-contiguous and misaligned entries: one fused segment
    call and one object; every entry of get_bundle is bit for bit put(t, pack_fp8=True) + get(t) (NaNs as bits); a subset
    get_bundle_into with non-contiguous outs and canaries takes one segment get; an unfusable config stores the same
    bytes; a batch mixing packed and plain bundles; the async forms."""
    from blackbird_b200.ops import AsyncTensorStore, TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id=f"t-fp8-bundles-{str(dt)[6:]}", dram_bytes=64 << 20)
    try:
        rec = Recorder(cl.client)
        store = TensorStore(rec)
        b = _bundle(dt, 1)
        store.put_bundle("pb", b, pack_fp8=True)
        assert rec.calls.get("batch_put_device_fp8_segments") == 1 and rec.calls.get("batch_put") == 1
        assert "batch_put_device" not in rec.calls
        refs = {}
        for name, t in b.items():
            if t.numel():
                store.put(f"ref/{name}", t, pack_fp8=True)
                refs[name] = store.get(f"ref/{name}")
        got = store.get_bundle("pb")
        assert list(got) == list(b)
        for name, t in b.items():
            assert got[name].dtype == dt and got[name].shape == t.shape, name
            if t.numel():
                assert torch.equal(_bits(got[name]), _bits(refs[name])), name
        # a subset restore into canary-framed outs, one of them non-contiguous; one fused segment get
        frames = {k: torch.full((b[k].numel() + 64,), 7.0, dtype=dt, device="cuda") for k in ("odd", "big", "zero_d")}
        outs = {k: f[32:32 + b[k].numel()].view(b[k].shape) for k, f in frames.items()}
        outs["nc"] = torch.zeros(6, 10, dtype=dt, device="cuda").t()
        g0 = rec.calls.get("batch_get_device_fp8_segments", 0)
        store.get_bundle_into("pb", outs)
        assert rec.calls["batch_get_device_fp8_segments"] == g0 + 1
        for k, f in frames.items():
            assert torch.equal(_bits(outs[k]), _bits(refs[k])), k
            assert bool((f[:32] == 7).all()) and bool((f[-32:] == 7).all()), k
        assert torch.equal(_bits(outs["nc"]), _bits(refs["nc"]))
        # an unfusable config (two shards a copy): packed first and put as bytes, the same stored object
        unfusable = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096,
                                    preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        store.put_bundle("pu", b, config=unfusable, pack_fp8=True)
        m = store._metas(["pu"], bundle=True)[0]
        assert m["packed"] == "mxfp8" and m["numel"] % 32 == 0
        raw = [torch.empty(bb.mxfp8_packed_bytes(m["numel"]), dtype=torch.uint8, device="cuda") for _ in range(2)]
        ecs, _ = cl.client.batch_get_device(["pb", "pu"], [r.data_ptr() for r in raw], [raw[0].numel()] * 2, _stream())
        assert ecs == [bb.ErrorCode.OK] * 2 and torch.equal(raw[0], raw[1])
        gu = store.get_bundle("pu")
        assert all(torch.equal(_bits(gu[k]), _bits(refs[k])) for k in refs)
        o = {"mat": torch.zeros(7, 13, dtype=dt, device="cuda")}
        store.get_bundle_into("pu", o)
        assert torch.equal(_bits(o["mat"]), _bits(refs["mat"]))
        # a batch mixing packed and plain bundles
        plain = {"i": torch.arange(10, device="cuda"), "x": torch.arange(9, dtype=torch.float32, device="cuda") / 3}
        store.put_bundle("plain", plain)
        both = store.batch_get_bundles(["pb", "plain"])
        assert torch.equal(_bits(both[0]["odd"]), _bits(refs["odd"])) and all(torch.equal(both[1][k], v) for k, v in plain.items())
        o1, o2 = {"one": torch.zeros(32, dtype=dt, device="cuda")}, {"i": torch.zeros(10, dtype=torch.int64, device="cuda")}
        store.batch_get_bundles_into(["pb", "plain"], [o1, o2])
        assert torch.equal(_bits(o1["one"]), _bits(refs["one"])) and torch.equal(o2["i"], plain["i"])
        # the async forms
        a = AsyncTensorStore(cl.client)
        try:
            assert a.put_bundles_async(["ab"], [b], pack_fp8=True).result() == 1
            o = {"big": torch.zeros(T + 5, dtype=dt, device="cuda")}
            a.get_bundles_into_async(["ab"], [o]).result()
            assert torch.equal(_bits(o["big"]), _bits(refs["big"]))
        finally:
            a.close()
    finally:
        cl.stop()
