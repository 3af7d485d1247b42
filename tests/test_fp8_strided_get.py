"""Strided gets of MXFP8-packed tensors on the GPU: the strided store window of the fused unpack kernel (bb_xfer_fp8 with
XFER_STRIDED) through XferEngine.run_fp8, the client's batch_get_device_fp8_strided on a GpuRankCluster, and the fused
TensorStore.get_slice of packed tensors.  Every result is compared bit for bit with rows of
mxfp8_unpack_ref(mxfp8_pack_ref(x)), and every destination is guard-filled and checked element for element.  A strided get
still reads and hashes the whole packed object, so digests and verify status are those of a whole get."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384  # elements per payload tile (32 KiB of bf16)
MiB = 1 << 20
GUARD = 0x5A5A  # as int16 bit pattern
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


class Packed:
    """An n-element bf16 tensor packed by the CPU reference: `slab` holds [payload][scales] on the device, `ref` is the
    reference unpack (int16 bit patterns, on the device), `digest` the BBH64 of the packed bytes."""

    def __init__(self, bb, n, seed):
        g = np.random.default_rng(seed)
        x = ((g.standard_normal(n) * 4).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        x[:32] = 0  # an all-zero block (scale 0)
        packed = np.frombuffer(bb.mxfp8_pack_ref(x), dtype=np.uint8)
        self.n = n
        self.digest = bb.bbh64(packed)
        self.slab = torch.from_numpy(packed.copy()).cuda()
        ref = np.frombuffer(bb.mxfp8_unpack_ref(packed, n), dtype=np.int16)
        self.ref = torch.from_numpy(ref.copy()).cuda()


def stored(n, w):
    """(object elements, result elements relative to the item's bf16 pointer) that a window stores: w = None (whole),
    (lo, hi) or (lo, hi, pitch, width, phase)."""
    if w is None:
        x = np.arange(n, dtype=np.int64)
        return x, x
    x = np.arange(w[0], w[1], dtype=np.int64)
    if len(w) == 2:
        return x, x
    pitch, width, phase = w[2:]
    y = x + phase
    keep = y % pitch < width
    return x[keep], (y // pitch * width + y % pitch)[keep]


class Gets:
    """Unpack items reading `objs` into one guard-filled int16 buffer, each at its own region with guards on both sides.
    The bf16 pointer of an item is placed so that its rows are co-aligned (unless `skew` moves it by elements)."""

    def __init__(self, objs, wins, skew=0):
        self.objs, self.wins = objs, wins
        self.maps, self.bases, o = [], [], 64
        for obj, w in zip(objs, wins):
            xs, ds = stored(obj.n, w)
            lo_d = int(ds.min()) if ds.size else 0
            hi_d = int(ds.max()) + 1 if ds.size else 0
            # region start o holds result element lo_d, so the bf16 pointer is o - lo_d elements; the engine wants
            # 2 * (pointer + phase - r_lo * (pitch - width)) 16-byte aligned for the window's first row r_lo
            res = lo_d
            if w is not None and len(w) == 5:
                pitch, width, phase = w[2:]
                res = lo_d - phase + (w[0] + phase) // pitch * (pitch - width)
            o = (o + 7) // 8 * 8 + res % 8 + skew
            self.bases.append(o - lo_d)
            self.maps.append((xs, ds))
            o += hi_d - lo_d + 64
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.int16, device="cuda")
        self.items = []
        for obj, w, b in zip(objs, wins, self.bases):
            it = (self.dst.data_ptr() + 2 * b, obj.slab.data_ptr(), obj.n, obj.digest)
            self.items.append(it if w is None else it + (w,))

    def want(self):
        want = torch.full_like(self.dst, GUARD)
        for obj, b, (xs, ds) in zip(self.objs, self.bases, self.maps):
            if xs.size:
                want[torch.from_numpy(b + ds).cuda()] = obj.ref[torch.from_numpy(xs).cuda()]
        return want

    def check(self, what):
        torch.cuda.synchronize()
        want = self.want()
        if not torch.equal(self.dst, want):
            bad = (self.dst != want).nonzero().flatten()[:8].tolist()
            pytest.fail(f"{what}: elements differ at {bad}; bases {self.bases[:8]}")


def patterns(n):
    """Strided windows (lo, hi, pitch, width, phase) of an n-element object: pitch 64 (256 rows per tile, so that lanes
    loop) with widths 8 and 16; rows longer than a tile; pitches of 4 tiles (tiles wholly inside a gap); phases 0, 5 and
    pitch - 1; width == pitch; windows that start and end inside a row and reach into the tail tile; one row across a
    tile edge whose gap is no multiple of 8; an empty window."""
    out = [(0, n, 64, 8, 0), (0, n, 64, 16, 5), (0, n, 64, 8, 63), (T - 3, n - 7, 64, 8, 11),
           (0, n, 3 * T, T + 8, 0), (5, n, 3 * T + 8, T + 16, 3 * T), (0, n, 4 * T, 64, 0), (T + 1, n, 4 * T, 4 * T - 8, 7),
           (0, n, 1000, 40, 999), (0, n, 1000, 1000, 0), (T - 3, n - 7, 1000, 1000, 11), (0, n, 40, 32, 0),
           (T - 8, T + 8, 100, 16, 24), (5 * T + 100, 5 * T + 100, 64, 8, 0)]
    return [(lo, min(hi, n), p, wd, ph) for lo, hi, p, wd, ph in out if lo <= min(hi, n)]


# ---------------------------------------------------------------------------------------------------- engine


def test_fp8_strided_windows_at_every_grid(bb, eng):
    """Every pattern of an object with a tail tile, in batches of more than 8 items with whole and windowed items mixed
    in, at grids of 1, 7, the SM count and twice the SM count, so that rows straddle tiles and CTA runs."""
    n = 8 * T + 96
    obj = Packed(bb, n, 11)
    ps = patterns(n)
    for chunk in range(0, len(ps), 8):
        ws = ps[chunk:chunk + 8] + [None, (T + 1, 3 * T - 1), None]
        g = Gets([obj] * len(ws), ws)
        assert len(ws) > 8
        for grid in GRIDS:
            eng.set_max_ctas(_grid(grid))
            g.dst.fill_(GUARD)
            dg, st, _ = eng.run_fp8(g.items, True, _stream())
            assert st == [0] * len(ws) and dg == [obj.digest] * len(ws), (chunk, grid, st)
            g.check(f"chunk={chunk} grid={grid}")


def test_fp8_strided_batches_mix_objects(bb, eng):
    """Objects of one tail tile only, of whole tiles and of 4 Mi elements (a KV layer's heads) in one batch."""
    objs = [Packed(bb, n, 40 + i) for i, n in enumerate([32, 3 * T + 96, 4 * T, 4 * MiB])]
    wins = [(0, 32, 16, 8, 0), (0, 3 * T + 96, 128, 24, 100), None, (0, 4 * T, 2048, 512, 0), (0, 4 * MiB, 1024, 128, 1024 - 128),
            (1024, 4 * MiB, 1024, 256, 0), (8, 24), (T - 1, 3 * T + 96, 2 * T, 8, 1), (0, 4 * MiB, 1024, 1024, 0), None]
    pick = [0, 1, 2, 2, 3, 3, 0, 1, 3, 1]
    g = Gets([objs[i] for i in pick], wins)
    dg, st, _ = eng.run_fp8(g.items, True, _stream())
    assert st == [0] * len(wins) and dg == [objs[i].digest for i in pick]
    g.check("mixed")


def test_fp8_a_flipped_byte_in_a_gap_fails_verification(bb, eng):
    """Payload and scale bytes are hashed whole: a flip in a gap between rows gives status 1, and still only the rows are
    written, with the values they have."""
    n = 3 * T + 96
    obj = Packed(bb, n, 3)
    w = (0, n, 1024, 128, 0)  # rows [1024 r, 1024 r + 128)
    for pos in (300, 2 * T + 500, n + 20, n + (T + 512) // 32):  # payload of tiles 0 and 2, scale bytes of tiles 0 and 1
        obj.slab[pos] ^= 0x41
        g = Gets([obj, obj], [w, (T + 5, 2 * T - 3, 1024, 128, 0)])
        _, st, _ = eng.run_fp8(g.items, True, _stream())
        assert st == [1, 1], (pos, st)
        g.check(f"flip at {pos}")
        obj.slab[pos] ^= 0x41
    g = Gets([obj], [w])
    dg, st, _ = eng.run_fp8(g.items, True, _stream())
    assert st == [0] and dg == [obj.digest]
    g.check("restored")


def test_fp8_rejected_patterns(bb, eng):
    obj = Packed(bb, 2 * T, 1)
    n = obj.n
    dst = torch.full((4 * T,), GUARD, dtype=torch.int16, device="cuda")
    d, s = dst.data_ptr(), obj.slab.data_ptr()
    x = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    slab2 = torch.zeros_like(obj.slab)
    bad = [(([(d, s, n, obj.digest, (0, n, 100, 0, 0))], True), "INVALID_ARGUMENT"),      # width 0
           (([(d, s, n, obj.digest, (0, n, 100, 101, 0))], True), "INVALID_ARGUMENT"),    # width > pitch
           (([(d, s, n, obj.digest, (0, n, 100, 50, 100))], True), "INVALID_ARGUMENT"),   # phase >= pitch
           (([(d, s, n, obj.digest, (0, n + 1, 100, 50, 0))], True), "INVALID_ARGUMENT"), # past the object
           (([(d, s, n, obj.digest, (0, n, 2**63, 8, 0))], True), "INVALID_ARGUMENT"),    # pitch overflows its bytes
           (([(x.data_ptr(), slab2.data_ptr(), n, 0, (0, n, 64, 8, 0))], False), "INVALID_ARGUMENT"),  # a stride on a put
           (([(d, s, n, obj.digest, (0, n, 100, 54, 0))], True), "INVALID_ADDRESS"),      # gap of 46 elements
           (([(d, s, n, obj.digest, (0, n, 100, 52, 4))], True), "INVALID_ADDRESS"),      # row 0 starts 8 bytes off
           (([(d + 2, s, n, obj.digest, (0, n, 96, 80, 0))], True), "INVALID_ADDRESS")]   # pointer 2 bytes off
    for (items, unpack), err in bad:
        with pytest.raises(RuntimeError, match=err):
            eng.run_fp8(items, unpack, _stream())
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all()) and bool((slab2 == 0).all())
    # a window inside one row may leave any gap: that row's base is what has to be co-aligned.  Elements [130, 160) of row
    # 1 land at bf16 byte 2 * (60 + 30) past the pointer, d + 4 (congruent to 2 * 130 mod 16) for the pointer d - 176.
    _, st, _ = eng.run_fp8([(d - 176, s, n, obj.digest, (130, 180, 100, 60, 0))], True, _stream())
    torch.cuda.synchronize()
    assert st == [0]
    assert torch.equal(dst[2:32], obj.ref[130:160]) and bool((dst[:2] == GUARD).all()) and bool((dst[32:] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- client


def _counter(client, name):
    for line in client.metrics_text().splitlines():
        if line.startswith(f"bb_client_{name} "):
            return int(float(line.split()[1]))
    return 0


def _cfg(bb, replicas=1):
    return bb.WorkerConfig(replication_factor=replicas, max_workers_per_copy=1, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU])


def _flip(cl, sh, pos):
    be = cl.worker.backend(sh.pool_id)
    be.write(sh.offset + pos, bytes([be.read(sh.offset + pos, 1)[0] ^ 0xFF]))


def _put(bb, cl, key, obj, replicas):
    """Stores obj's packed bytes as one BBH64 shard per copy (the layout of a fused put) and checks the recorded digest."""
    assert cl.client.batch_put_device([key], [obj.slab.data_ptr()], [obj.slab.numel()], _cfg(bb, replicas), _stream()) == [bb.ErrorCode.OK]
    copies = cl.client.get_workers(key)
    assert len(copies) == replicas and all(len(c.shards) == 1 and c.shards[0].checksum == obj.digest for c in copies)
    return [c.shards[0] for c in copies]


def _strided_get(cl, keys, objs, pats, skew=None):
    """Strided gets (offset, width, pitch, rows) into one guard-filled buffer, each result at element offset % 8 of a
    16-byte aligned region (+ skew); returns (error codes, buffer, regions)."""
    regions, o = [], 64
    for i, (off, w, _, r) in enumerate(pats):
        reg = (o + 7) // 8 * 8 + off % 8 + (skew or {}).get(i, 0)
        regions.append(reg)
        o = reg + w * r + 64
    out = torch.full((o + 64,), GUARD, dtype=torch.int16, device="cuda")
    ecs = cl.client.batch_get_device_fp8_strided(keys, [out.data_ptr() + 2 * r for r in regions], [ob.n for ob in objs],
                                                 [p[0] for p in pats], [p[1] for p in pats], [p[2] for p in pats],
                                                 [p[3] for p in pats], _stream())
    return ecs, out, regions


def _check_strided(out, regions, objs, pats, ok):
    want = torch.full_like(out, GUARD)
    for reg, obj, (off, w, p, n), good in zip(regions, objs, pats, ok):
        if good and w and n:
            rows = obj.ref[off:off + (n - 1) * p + w].unfold(0, w, p).reshape(-1) if n > 1 else obj.ref[off:off + w]
            want[reg:reg + w * n] = rows
    torch.cuda.synchronize()
    if not torch.equal(out, want):
        pytest.fail(f"strided get wrote wrong elements at {(out != want).nonzero().flatten()[:8].tolist()}")


def test_client_fp8_strided_with_one_and_two_copies(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8str-rep")
    try:
        objs = [Packed(bb, n, 60 + i) for i, n in enumerate([3 * T + 96, 64, 32 * 8 * 128])]
        n0, b0 = _counter(cl.client, "device_get_fp8_strided_total"), _counter(cl.client, "device_get_fp8_strided_bytes_total")
        asked = asked_b = 0
        for rep in (1, 2):
            keys = [f"r{rep}/{i}" for i in range(len(objs))]
            for k, obj in zip(keys, objs):
                _put(bb, cl, k, obj, rep)
            ks, os_, ps = [], [], []
            for k, obj in zip(keys, objs):
                n = obj.n
                for p in [(0, 8, 64, n // 64), (128, 128, 1024, max(n // 1024 - 1, 0)), (3, 16, 24, (n - 19) // 24), (T - 3, 300, 7, 1),
                          (0, 32, 32, n // 32), (5, 8, 16, 0), (40, 0, 64, 3)]:
                    if p[3] == 0 or p[0] + (p[3] - 1) * p[2] + p[1] <= n:
                        ks.append(k), os_.append(obj), ps.append(p)
            l0 = cl.fabric.launches
            ecs, out, regions = _strided_get(cl, ks, os_, ps)
            assert ecs == [bb.ErrorCode.OK] * len(ks), ecs
            assert cl.fabric.launches == l0 + 2  # the fused kernel and the scales batch
            _check_strided(out, regions, os_, ps, [True] * len(ks))
            asked += len(ks)
            asked_b += 2 * sum(w * r for _, w, _, r in ps)
        assert _counter(cl.client, "device_get_fp8_strided_total") == n0 + asked
        assert _counter(cl.client, "device_get_fp8_strided_bytes_total") == b0 + asked_b
    finally:
        cl.stop()


def test_client_fp8_strided_errors_and_misaligned_items_fail_alone(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8str-err")
    try:
        a, b = Packed(bb, 3 * T + 96, 70), Packed(bb, 2 * T, 71)
        _put(bb, cl, "a", a, 1)
        _put(bb, cl, "b", b, 1)
        E = bb.ErrorCode
        cases = [("a", a, (T - 3, 104, 1000, 20), 0, E.OK),
                 ("a", a, (10, 101, 100, 2), 0, E.INVALID_ARGUMENT),
                 ("a", a, (a.n - 100, 50, 64, 3), 0, E.VALUE_OUT_OF_RANGE),
                 ("b", b, (0, 8, 2**63, 3), 0, E.VALUE_OUT_OF_RANGE),
                 ("missing", b, (0, 32, 64, 2), 0, E.OBJECT_NOT_FOUND),
                 ("b", b, (40, 0, 64, 5), 0, E.OK),
                 ("b", b, (40, 16, 64, 0), 0, E.OK),
                 ("a", a, (5, 64, 128, 40), 3, E.NOT_IMPLEMENTED),   # virtual base 6 bytes off
                 ("a", a, (5, 64, 100, 40), 0, E.NOT_IMPLEMENTED),   # gap of 36 elements
                 ("b", b, (0, b.n, 7, 1), 0, E.OK),
                 ("a", a, (a.n - 72 - 24, 24, 72, 2), 0, E.OK)]
        skew = {i: c[3] for i, c in enumerate(cases)}
        objs, pats = [c[1] for c in cases], [c[2] for c in cases]
        l0 = cl.fabric.launches
        ecs, out, regions = _strided_get(cl, [c[0] for c in cases], objs, pats, skew)
        strided_launches = cl.fabric.launches - l0
        assert ecs == [c[4] for c in cases], ecs
        _check_strided(out, regions, objs, pats, [e == E.OK for e in ecs])
        # the same objects read whole: one attempt costs the same launches
        outs = [torch.empty(o.n, dtype=torch.int16, device="cuda") for o in (a, b)]
        l0 = cl.fabric.launches
        assert cl.client.batch_get_device_fp8(["a", "b"], [o.data_ptr() for o in outs], [a.n, b.n], _stream()) == [E.OK, E.OK]
        assert strided_launches == cl.fabric.launches - l0 == 2
        torch.cuda.synchronize()
        assert torch.equal(outs[0], a.ref) and torch.equal(outs[1], b.ref)
    finally:
        cl.stop()


def test_client_fp8_strided_fails_over_from_a_copy_corrupt_in_a_gap(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8str-fo")
    try:
        obj = Packed(bb, 3 * T + 96, 80)
        shards = _put(bb, cl, "f", obj, 2)
        p = (128, 128, 1024, 40)  # payload byte 300 lies in the gap after row 0; scale byte 20 covers elements 640..671
        for pos in (300, obj.n + 20):
            fo = _counter(cl.client, "replica_failover_total")
            for sh in shards:  # one copy at a time is corrupt: exactly one of the two gets starts on it
                _flip(cl, sh, pos)
                ecs, out, regions = _strided_get(cl, ["f"], [obj], [p])
                assert ecs == [bb.ErrorCode.OK]
                _check_strided(out, regions, [obj], [p], [True])
                _flip(cl, sh, pos)
            assert _counter(cl.client, "replica_failover_total") == fo + 1, pos
        for sh in shards:
            _flip(cl, sh, 300)
        ecs, out, regions = _strided_get(cl, ["f"], [obj], [p])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        torch.cuda.synchronize()
        outside = torch.ones_like(out, dtype=torch.bool)
        outside[regions[0]:regions[0] + p[1] * p[3]] = False
        assert bool((out[outside] == GUARD).all())
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_get_slice_of_packed_tensors(bb):
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-fp8str-slice")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(9)
        ts = {"kv": torch.randn(64, 8, 128, device="cuda", generator=g).to(torch.bfloat16),   # a KV layer: heads along dim 1
              "w": torch.randn(96, 64, device="cuda", generator=g).to(torch.bfloat16),        # columns of a weight
              "pad": torch.randn(7, 9, device="cuda", generator=g).to(torch.bfloat16),        # 63 elements, padded to 64
              "big": torch.randn(3, 40, 4099, device="cuda", generator=g).to(torch.bfloat16)}  # rows across tile edges
        for k, t in ts.items():
            store.put(k, t, pack_fp8=True)
        whole = {k: store.get(k) for k in ts}
        # (key, dim, start, stop, fused): a slice misses the fused kernel only when its row gap is no multiple of 8 elements
        cases = [("kv", 1, 0, 1, True), ("kv", 1, 2, 4, True), ("kv", 1, 4, 8, True), ("kv", -1, 5, 37, True), ("kv", 2, 0, 128, True),
                 ("kv", 1, 3, 3, True), ("w", 1, 10, 50, True), ("w", 1, 3, 60, False), ("w", -1, 0, 64, True),
                 ("pad", 1, 1, 5, False), ("pad", 1, 0, 9, True), ("pad", 1, 4, 5, True), ("big", 1, 3, 11, True),
                 ("big", 2, 0, 4091, True), ("big", 2, 1, 4098, False), ("big", 1, 39, 40, False), ("kv", 0, 17, 40, False)]
        f0 = _counter(cl.client, "device_get_fp8_strided_total")
        for k, d, a, b, _ in cases:
            got = store.get_slice(k, d, a, b)
            want = whole[k].narrow(d, a, b - a).contiguous()
            assert got.dtype == torch.bfloat16 and got.shape == want.shape and got.is_contiguous(), (k, d, a, b)
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (k, d, a, b)
        fused = sum(f for *_, f in cases)
        assert _counter(cl.client, "device_get_fp8_strided_total") == f0 + fused
        outs = store.batch_get_slices([c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
        assert _counter(cl.client, "device_get_fp8_strided_total") == f0 + 2 * fused
        spans = []
        for o, (k, d, a, b, _) in zip(outs, cases):
            assert torch.equal(o.view(torch.int16), whole[k].narrow(d, a, b - a).contiguous().view(torch.int16)), (k, d, a, b)
            if o.numel():
                spans.append((o.data_ptr(), o.data_ptr() + 2 * o.numel()))
        spans.sort()
        assert all(e <= s for (_, e), (s, _) in zip(spans, spans[1:])), "results alias each other"
        # a packed tensor striped over the workers of a copy (unfused put) reads back through the whole-get fallback
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU],
                              checksum=bb.ChecksumAlgo.XXH3)
        x = torch.randn(50, 64, device="cuda", generator=g).to(torch.bfloat16)
        store.put("striped", x, pack_fp8=True, config=cfg)
        f1 = _counter(cl.client, "device_get_fp8_strided_total")
        got = store.get_slice("striped", 1, 8, 24)
        assert torch.equal(got.view(torch.int16), store.get("striped")[:, 8:24].contiguous().view(torch.int16))
        assert _counter(cl.client, "device_get_fp8_strided_total") == f1
    finally:
        cl.stop()
