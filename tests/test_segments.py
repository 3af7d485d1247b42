"""Segment-list puts and gets on the GPU: the segment-table gathering load and scattering store of bb_xfer
(XFER_SEGMENTS) through XferEngine, the client's batch_put_device_segments / batch_get_device_segments on a
GpuRankCluster, and TensorStore's bundles.  A segmented descriptor reads or stores its object's bytes in segments of any
sizes at arbitrary addresses; the tile in shared memory is the dense object's, so every check covers the segments, the
guard bytes around and between them, and the digest, which must equal that of a plain transfer of the concatenation."""
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


class Carver:
    """Regions of one buffer, each after a guard gap, placed so that region + align_at is 16-byte aligned."""

    def __init__(self):
        self.o = 64

    def region(self, n, align_at=0):
        self.o = (self.o + 15) // 16 * 16 + (16 - align_at % 16) % 16
        at = self.o
        self.o += n + 48
        return at

    def segments(self, lens, off, rng, null=0.0):
        """Offsets of segments of lens (None: a null segment), segment k co-aligned for a descriptor that starts at
        object byte off (address = object offset - off mod 16), carved in random order."""
        starts = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        order = rng.permutation(len(lens))
        at = [0] * len(lens)
        for k in order:
            at[k] = self.region(int(lens[k]) + 16, int(off - starts[k]))
        return [None if rng.random() < null else a for a in at]


def seg_index(lens, at):
    """Per object byte, the buffer offset it lives at (-1 in a null segment)."""
    return np.concatenate([np.arange(n) + a if a is not None else np.full(n, -1) for n, a in zip(lens, at)] or [np.zeros(0, np.int64)])


def seg_lens(rng, kind):
    if kind == "many-short":  # thousands of segments in a tile
        return [int(x) for x in rng.integers(1, 24, 3000)]
    if kind == "long":  # one segment over many tiles, with short ones around it
        return [5, 40 * T + 3, 17, 2 * T]
    if kind == "mixed":
        return [int(rng.choice([0, 1, 15, 16, 100, 4096, T - 1, T + 33, 3 * T])) for _ in range(40)]
    return [int(x) for x in rng.integers(1, 3 * T, 6)]


def test_segment_items_at_every_grid(bb, eng):
    """Segment puts and gets -- thousands of short segments per tile, one segment over forty tiles, zero-length and null
    segments, descriptors that start inside a segment (a shard's rebase) -- in one device-table batch with plain,
    windowed, gathered and paged items, at grids of 1, 7, the SM count and twice the SM count, for every digest: the
    stored bytes equal the concatenation, the digests the CPU model of a plain transfer of it, every guard byte is intact
    (nulls included), and a wrong expected digest on a segment get gives status 1."""
    rng = np.random.default_rng(3)
    src_c, dst_c = Carver(), Carver()
    specs = []  # (kind, lens, off, src offsets, dst offsets)
    for kind in ("many-short", "long", "mixed", "few"):
        for side in ("sput", "sget"):
            for off in (0, 4096 + 48):
                lens = seg_lens(rng, kind)
                total = sum(lens)
                off = min(off, total - 1)
                n = total - off
                if side == "sput":
                    at = src_c.segments(lens, off, rng)
                    specs.append((side, lens, off, seg_index(lens, at)[off:], dst_c.region(n) + np.arange(n)))
                else:
                    at = dst_c.segments(lens, off, rng, null=0.15)
                    specs.append((side, lens, off, src_c.region(n) + np.arange(n), seg_index(lens, at)[off:]))
                specs[-1] += (at,)
    others = [("plain", 3 * T + 7), ("window", 2 * T + 9), ("gather", 2 * T + 1), ("pput", 3 * 4096 - 5)]
    other_ix = []  # (source index, destination index, source pages)
    for kind, n in others:
        y = np.arange(n)
        if kind == "gather":  # rows of 32 bytes every 48, phase 5
            s = src_c.region(int(((y + 5) // 32 * 48 + (y + 5) % 32).max()) + 1, 5)
            other_ix.append((s + (y + 5) // 32 * 48 + (y + 5) % 32, dst_c.region(n) + y, None))
        elif kind == "pput":
            pages = [src_c.region(4096) for _ in range(3)][::-1]
            other_ix.append((np.asarray(pages)[y // 4096] + y % 4096, dst_c.region(n) + y, pages))
        elif kind == "window":  # the virtual base, region - 100, 16-byte aligned
            other_ix.append((src_c.region(n) + y, dst_c.region(n, -100) + y, None))
        else:
            other_ix.append((src_c.region(n) + y, dst_c.region(n) + y, None))
    src = _random(bb, src_c.o + 64, 5)
    host = src.cpu().numpy()
    dst = torch.full((dst_c.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
    S, D = src.data_ptr(), dst.data_ptr()
    for algo in ALGOS:
        A, model = getattr(bb.ChecksumAlgo, algo), _model(bb, algo)
        verify = 0 if algo == "NONE" else bb.XFER_VERIFY
        items, objs, want_at = [], [], []
        for side, lens, off, six, dix, at in specs:
            obj = host[six]
            objs.append(obj)
            n = obj.size
            pairs = [(0 if a is None else (S if side == "sput" else D) + a, m) for a, m in zip(at, lens)]
            if side == "sput":
                items.append((0, D + int(dix[0]), n, 0, 0, 0, None, None, None, None, None, None, None, None, (pairs, off)))
            else:
                items.append((S + int(six[0]), 0, n, model(obj.tobytes()), verify, 0, None, None, None, None, None, None, None, None, None,
                              (pairs, off)))
            want_at.append(dix)
        for (kind, n), (six, dix, pages) in zip(others, other_ix):
            obj = host[six]
            if kind == "window":
                items.append((S + int(six[0]), D + int(dix[0]) - 100, n, model(obj.tobytes()), verify, 0, (100, T + 333)))
                objs.append(obj[100:T + 333])
                want_at.append(dix[:T + 233])
                continue
            if kind == "gather":
                items.append((S + int(six[0]) - 5, D + int(dix[0]), n, 0, 0, 0, None, (48, 32, 5)))
            elif kind == "pput":
                items.append((0, D + int(dix[0]), n, 0, 0, 0, None, None, None, ([S + p for p in pages], 4096, 0)))
            else:
                items.append((S + int(six[0]), D + int(dix[0]), n, model(obj.tobytes()), verify))
            objs.append(obj)
            want_at.append(dix)
        want = np.full(dst.numel(), GUARD, dtype=np.uint8)
        for obj, at in zip(objs, want_at):
            keep = at >= 0
            want[at[keep]] = obj[keep]
        seg_digests = [model(o.tobytes()) for o in objs[:len(specs)]]
        for g in GRIDS:
            eng.set_max_ctas(_grid(g))
            dst.fill_(GUARD)
            dg, st, _ = eng.run(items, A, _stream())
            assert st == [0] * len(items), (algo, g, st)
            if algo != "NONE":
                assert dg[:len(specs)] == seg_digests, (algo, g)
            torch.cuda.synchronize()
            got = dst.cpu().numpy()
            assert np.array_equal(got, want), (algo, g, np.nonzero(got != want)[0][:8].tolist())
        eng.set_max_ctas(0)
        if algo != "NONE":
            bad = [it[:3] + (it[3] ^ 1,) + it[4:] if sp[0] == "sget" else it for it, sp in zip(items, specs + [("x",)] * len(others))]
            _, st, _ = eng.run(bad, A, _stream())
            assert st == [1 if sp[0] == "sget" else 0 for sp in specs] + [0] * len(others)


def test_segment_refusals_and_small_batches(bb, eng):
    """XFER_SEGMENTS among a caller's flags, forbidden combinations, null segments in a put and misaligned segments are
    refused before any launch (the valid neighbour is not written either); a small batch with a segmented item runs in
    bb_xfer, never the warp-per-object kernel or the mailbox; run_fp8 refuses segments."""
    src = _random(bb, 8 * T, 1)
    dst = torch.full((8 * T,), GUARD, dtype=torch.uint8, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    A = bb.ChecksumAlgo.XXH3
    sg = ([(s, 1000), (s + 2 * T + 1000, 3000)], 0)
    dg = ([(d, 1000), (d + 2 * T + 1000, 3000)], 0)
    N = [None] * 8
    E = "INVALID_ARGUMENT"
    bad = [((s, d, 1000, 0, bb.XFER_SEGMENTS), E),                                         # the caller's flag
           ((0, d, 4000, 0, bb.XFER_SEGMENTS, 0, *N, sg), E),                              # ... with segments
           ((0, d, 4000, 0, bb.XFER_PAGED, 0, *N, sg), E),                                 # with XFER_PAGED
           ((0, d, 4000, 0, 0, 0, (0, 500), *N[1:], sg), E),                               # with a window
           ((s, [], 4000, 0, bb.XFER_RAW_SUM, 0, *N, sg), E),                              # with RAW_SUM
           ((0, 0, 4000, 0, 0, 0, *N, sg, dg), E),                                         # both sides
           ((0, d, 4001, 0, 0, 0, *N, sg), E),                                             # table too short
           ((0, d, 4000, 0, 0, 0, *N, ([(s, 1000), (0, 3000)], 0)), E),                    # a null segment in a put
           ((s, [d, d + T], 4000, 0, 0, 0, *N, None, dg), E),                              # get: two destinations
           ((0, d, 4000, 0, 0, 0, *N, ([(s, 1000), (s + 2 * T, 3000)], 0)), "INVALID_ADDRESS"),   # 1000 != 0 mod 16
           ((s, 0, 4000, 0, 0, 0, *N, None, ([(d + 4, 1000), (d + 2 * T + 1000, 3000)], 0)), "INVALID_ADDRESS")]
    for it, err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run([(s, d + 6 * T, 64, 0, 0), it], A, _stream())
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all())
    with pytest.raises(RuntimeError, match=E):
        eng.run_fp8([(0, d, 4096, None, None, None, None, None, None, None, None, None, None, ([(s, 8192)], 0))], False, _stream())
    sl, mb, la = eng.small_launches, eng.mailbox_requests, eng.launches
    dg_, st, _ = eng.run([(0, d, 100, 0, 0, 0, *N, ([(s + 16, 60), (s + 4096 + 60 % 16, 40)], 0)), (s, d + T, 64, 0, 0)], A, _stream())
    torch.cuda.synchronize()
    host = src.cpu().numpy()
    obj = np.concatenate([host[16:76], host[4096 + 12:4096 + 52]])
    assert dg_[0] == bb.xxh3t64(obj.tobytes()) and st == [0, 0]
    assert np.array_equal(dst[:100].cpu().numpy(), obj) and bool((dst[100:T] == GUARD).all())
    assert eng.small_launches == sl and eng.mailbox_requests == mb and eng.launches == la + 1


# ---------------------------------------------------------------------------------------------------- client
def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def test_client_segment_puts_and_gets(bb):
    """Objects striped over HBM and DRAM, replicated in HBM and in DRAM: the segment put stores the concatenation (a plain
    get reads it, and a segment get reads a plain put); segment gets fill the segments and nothing else, nulls
    included; a corrupt replica fails over."""
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-segs", dram_bytes=64 << 20, max_replicas=3)
    try:
        A = bb.ChecksumAlgo.XXH3
        striped = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, min_shard_size=4096, checksum=A,
                                  preferred_classes=[bb.StorageClass.RAM_GPU, bb.StorageClass.RAM_CPU])
        hbm = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_GPU])
        dram = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=1, ttl_ms=0, checksum=A, preferred_classes=[bb.StorageClass.RAM_CPU])
        rng = np.random.default_rng(8)
        c_src, c_dst = Carver(), Carver()
        shapes = [(striped, seg_lens(rng, "mixed")), (hbm, seg_lens(rng, "many-short")), (dram, seg_lens(rng, "few")), (hbm, seg_lens(rng, "long"))]
        ats = [c_src.segments(lens, 0, rng) for _, lens in shapes]
        dats = [c_dst.segments(lens, 0, rng, null=0.2) for _, lens in shapes]
        src = _random(bb, c_src.o + 64, 21)
        host = src.cpu().numpy()
        keys = [f"sg{k}" for k in range(len(shapes))]
        objs = [host[seg_index(lens, at)] for (_, lens), at in zip(shapes, ats)]
        for k, ((cfg, lens), at) in enumerate(zip(shapes, ats)):
            pairs = [(src.data_ptr() + a, n) for a, n in zip(at, lens)]
            assert cl.client.batch_put_device_segments([keys[k]], [pairs], cfg, _stream()) == [bb.ErrorCode.OK]
            out = torch.empty(objs[k].size, dtype=torch.uint8, device="cuda")
            ecs, sizes = cl.client.batch_get_device([keys[k]], [out.data_ptr()], [out.numel()], _stream())
            assert ecs == [bb.ErrorCode.OK] and sizes == [objs[k].size] and np.array_equal(out.cpu().numpy(), objs[k]), k
        ref = torch.from_numpy(objs[0]).cuda()
        assert cl.client.batch_put_device(["plain"], [ref.data_ptr()], [ref.numel()], hbm, _stream()) == [bb.ErrorCode.OK]
        dst = torch.full((c_dst.o + 64,), GUARD, dtype=torch.uint8, device="cuda")
        want = np.full(dst.numel(), GUARD, dtype=np.uint8)
        for (_, lens), at, obj in zip(shapes, dats, objs):
            ix = seg_index(lens, at)
            want[ix[ix >= 0]] = obj[ix >= 0]

        def staged(name, pairs):
            """Whether the client's rule stages the get: a shard of a copy whose segments are not co-aligned from its start."""
            t = bb.SourceSegments.from_segments(pairs)[1]
            for cp in cl.client.get_workers(name):
                off = 0
                for sh in cp.shards:
                    if not t.fused_get_aligned(off, sh.length):
                        return True
                    off += sh.length
            return False

        def get_all(names):
            dst.fill_(GUARD)
            st0 = _counter(cl.client, "device_get_host_staged_total")
            lists = [[(0 if a is None else dst.data_ptr() + a, n) for a, n in zip(at, lens)] for (_, lens), at in zip(shapes, dats)]
            ecs, sizes = cl.client.batch_get_device_segments(names, lists, _stream())
            assert ecs == [bb.ErrorCode.OK] * len(names), ecs
            assert sizes == [o.size for o in objs]
            # only objects striped at cuts that are not 16-byte multiples are staged
            assert _counter(cl.client, "device_get_host_staged_total") == st0 + sum(staged(k, p) for k, p in zip(names, lists))
            torch.cuda.synchronize()
            got = dst.cpu().numpy()
            assert np.array_equal(got, want), np.nonzero(got != want)[0][:8]

        get_all(keys)
        get_all(["plain"] + keys[1:])  # a plain object through a segment get
        # a corrupt HBM replica of sg1: the get fails over to the other copy
        pools = {p.id: p for p in cl.client.keystone().get_memory_pools()}
        sh = cl.client.get_workers("sg1")[0].shards[0]
        be = cl.worker.backend(sh.pool_id)
        off = sh.offset if sh.location["kind"] == "gpu" else sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr
        be.write(off + 1234, bytes([be.read(off + 1234, 1)[0] ^ 0xFF]))
        mm = _counter(cl.client, "checksum_mismatch_total")
        get_all(keys)
        assert _counter(cl.client, "checksum_mismatch_total") > mm
        E = bb.ErrorCode
        ecs, _ = cl.client.batch_get_device_segments(["sg2", "sg2"], [[(dst.data_ptr(), 16)], [(0, 1)]], _stream())
        assert ecs == [E.BUFFER_OVERFLOW, E.BUFFER_OVERFLOW]
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore
def _t(dtype, shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dtype == torch.bool:
        return torch.randint(0, 2, shape, generator=g, device="cuda").bool()
    if dtype.is_floating_point:
        return torch.randn(shape, generator=g, device="cuda").to(dtype)
    return torch.randint(-100, 100, shape, generator=g, device="cuda").to(dtype)


def _bundle(seed):
    dts = [torch.bfloat16, torch.float32, torch.int8, torch.float16, torch.int64, torch.bool, torch.uint8, torch.float64, torch.int16, torch.int32]
    shapes = [(3, 5), (7,), (), (0,), (13, 3), (2, 0, 4), (33,), (1, 1, 9), (1000,), (2, 17)]
    return {f"p{k}.{str(dt)[6:]}": _t(dt, sh, seed + k) for k, (dt, sh) in enumerate(zip(dts, shapes))}


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


def test_tensor_store_bundles(bb):
    """put_bundle / get_bundle / get_bundle_into round trips of a mixed-dtype dict with odd sizes, 0-d and empty tensors;
    a subset restore with canaries around every out; non-contiguous outs; a module's state_dict loaded in place; one
    segment call and one object plus one `#meta` per bundle; TypeError for the wrong kind of key; the async forms."""
    from blackbird_b200.ops import AsyncTensorStore, TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-bundles")
    try:
        rec = Recorder(cl.client)
        store = TensorStore(rec)
        b = _bundle(1)
        b["odd"] = torch.arange(40, dtype=torch.int8, device="cuda")[3:20]  # misaligned: copied first
        b["nc"] = _t(torch.float32, (8, 6), 9).t()                          # not contiguous: copied first
        store.put_bundle("bd", b)
        assert rec.calls.get("batch_put_device_segments") == 1 and rec.calls.get("batch_put") == 1
        assert sorted(store.keys("bd")) == ["bd"]
        got = store.get_bundle("bd")
        assert isinstance(got, dict) and list(got) == list(b)
        for k in b:
            assert got[k].dtype == b[k].dtype and torch.equal(got[k], b[k]), k
        lst = [b["p0.bfloat16"], b["p2.int8"], b["p3.float16"]]
        store.put_bundle("bl", lst)
        gl = store.get_bundle("bl")
        assert isinstance(gl, list) and all(torch.equal(x, y) for x, y in zip(gl, lst))
        # subset restore into canary-framed outs; one non-contiguous out
        frames = {k: torch.full((b[k].numel() + 64,), 7, dtype=b[k].dtype, device="cuda") if b[k].dtype != torch.bool else
                  torch.ones(b[k].numel() + 64, dtype=torch.bool, device="cuda") for k in ("p1.float32", "p4.int64", "p8.int16")}
        outs = {k: f[32:32 + b[k].numel()].view(b[k].shape) for k, f in frames.items()}
        outs["nc"] = torch.zeros(8, 6, dtype=torch.float32, device="cuda").t()
        before = rec.calls.get("batch_get_device_segments", 0)
        store.get_bundle_into("bd", outs)
        assert rec.calls["batch_get_device_segments"] == before + 1
        for k, f in frames.items():
            assert torch.equal(outs[k], b[k]) and bool((f[:32] == f[0]).all()) and bool((f[-32:] == f[0]).all()), k
        assert torch.equal(outs["nc"], b["nc"])
        # a module's state_dict in place
        torch.manual_seed(0)
        m1, m2 = torch.nn.Sequential(torch.nn.Linear(33, 17), torch.nn.LayerNorm(17)).cuda(), torch.nn.Sequential(torch.nn.Linear(33, 17), torch.nn.LayerNorm(17)).cuda()
        store.put_bundle("mod", m1.state_dict())
        store.get_bundle_into("mod", m2.state_dict())
        assert all(torch.equal(x, y) for x, y in zip(m1.state_dict().values(), m2.state_dict().values()))
        # wrong kinds, missing names, dtype and shape checks, all before any transfer
        store.put("tensor", b["p0.bfloat16"])
        calls = dict(rec.calls)
        with pytest.raises(TypeError, match="bundle"):
            store.get("bd")
        with pytest.raises(TypeError, match="bundle"):
            store.get_into("bd", torch.empty(1, device="cuda"))
        with pytest.raises(TypeError, match="bundle"):
            store.get_slice("bd", 0, 0, 1)
        with pytest.raises(TypeError, match="tensor"):
            store.get_bundle("tensor")
        with pytest.raises(TypeError, match="tensor"):
            store.get_bundle_into("tensor", {})
        with pytest.raises(KeyError):
            store.get_bundle_into("bd", {"nope": b["p0.bfloat16"]})
        with pytest.raises(KeyError):
            store.get_bundle("missing")
        with pytest.raises(TypeError):
            store.get_bundle_into("bd", {"p0.bfloat16": b["p0.bfloat16"].float()})
        with pytest.raises(ValueError):
            store.get_bundle_into("bd", {"p1.float32": torch.zeros(8, device="cuda")})
        with pytest.raises(ValueError):
            store.get_bundle_into("bd", {"p1.float32": torch.zeros(7)})
        assert {k: v for k, v in rec.calls.items() if k != "batch_get"} == {k: v for k, v in calls.items() if k != "batch_get"}
        store.remove(["bd"])
        assert "bd" not in store.keys("bd")
        a = AsyncTensorStore(cl.client)
        try:
            assert a.put_bundles_async(["ab"], [b]).result() == 1
            o = {"p9.int32": torch.zeros(2, 17, dtype=torch.int32, device="cuda")}
            a.get_bundles_into_async(["ab"], [o]).result()
            assert torch.equal(o["p9.int32"], b["p9.int32"])
        finally:
            a.close()
    finally:
        cl.stop()


def test_random_bundles_partial_restores_and_corruption(bb):
    """Seeded random bundles, partial restores into canary-framed outs and corrupted copies, against a host model: a
    restore is the stored tensors for the names it gives and leaves everything else alone, and a corrupt copy is failed
    over."""
    from blackbird_b200.ops import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=256 << 20, cluster_id="t-bundles-rand")
    try:
        cfg = bb.WorkerConfig(replication_factor=2, max_workers_per_copy=1, ttl_ms=0, checksum=bb.ChecksumAlgo.XXH3,
                              preferred_classes=[bb.StorageClass.RAM_GPU])
        store = TensorStore(cl.client, cfg)
        rng = np.random.default_rng(99)
        model, corrupted = {}, 0
        pools = {p.id: p for p in cl.client.keystone().get_memory_pools()}
        dts = [torch.bfloat16, torch.float32, torch.int8, torch.uint8, torch.int64]
        for step in range(12):
            key = f"r{step % 5}"
            n = int(rng.integers(1, 60))
            bnd = {f"t{i}": _t(dts[int(rng.integers(0, 5))], tuple(int(x) for x in rng.integers(0, 40, int(rng.integers(0, 3)))), step * 100 + i)
                   for i in range(n)}
            if key in model:  # a key is written once: replace it
                store.remove([key])
            store.put_bundle(key, bnd)
            model[key] = {k: v.cpu() for k, v in bnd.items()}
            k2 = sorted(model)[int(rng.integers(0, len(model)))]
            names = [nm for nm in model[k2] if rng.random() < 0.4]
            frames = {nm: torch.zeros(model[k2][nm].numel() + 32, dtype=model[k2][nm].dtype, device="cuda") for nm in names}
            outs = {nm: f[16:16 + model[k2][nm].numel()].view(model[k2][nm].shape) for nm, f in frames.items()}
            copies = cl.client.get_workers(k2)
            if step % 3 == 1 and len(copies) == 2 and copies[0].shards and copies[0].shards[0].length:
                # corrupt one byte of copy 0, the copy a get on this one-GPU cluster reads first (both are local): the
                # restore fails its digest and fails over to the other copy
                sh = copies[0].shards[0]
                be = cl.worker.backend(sh.pool_id)
                base = sh.offset if sh.location["kind"] == "gpu" else sh.location["remote_addr"] - pools[sh.pool_id].ucx_remote_addr
                at = base + int(rng.integers(0, sh.length))
                be.write(at, bytes([be.read(at, 1)[0] ^ 0x5A]))
                mm = _counter(cl.client, "checksum_mismatch_total")
                store.get_bundle_into(k2, outs)
                assert _counter(cl.client, "checksum_mismatch_total") > mm, (step, k2)
                be.write(at, bytes([be.read(at, 1)[0] ^ 0x5A]))
                corrupted += 1
            else:
                store.get_bundle_into(k2, outs)
            for nm, f in frames.items():
                assert torch.equal(outs[nm].cpu(), model[k2][nm]), (step, k2, nm)
                assert not f[:16].any() and not f[16 + model[k2][nm].numel():].any()
            whole = store.get_bundle(k2)
            assert all(torch.equal(whole[nm].cpu(), v) for nm, v in model[k2].items())
        assert corrupted > 0
    finally:
        cl.stop()
