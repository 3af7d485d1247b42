"""Element-range gets of MXFP8-packed tensors on the GPU: the store window of the fused unpack kernel (bb_xfer_fp8 with
XFER_WINDOW) through XferEngine.run_fp8, the client's batch_get_device_fp8_range on a GpuRankCluster, and the fused
TensorStore.get_rows.  Every result is compared bit for bit with mxfp8_unpack_ref(mxfp8_pack_ref(x))[lo:hi], and every
destination is guard-filled and checked element for element around each window.  A windowed get still reads and
hashes the whole packed object, so digests and verify status are those of the whole object."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

T = 16384  # elements per payload tile (32 KiB of bf16)
MiB = 1 << 20
GUARD = 0x5A5A  # as int16 bit pattern
GRIDS = [1, 7, "sms", "2sms"]
SIZES = [32, 64, 8192, T, T + 32, 3 * T + 96, 32 * MiB + 32]


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
        self.n, self.packed_host = n, packed
        self.digest = bb.bbh64(packed)
        self.slab = torch.from_numpy(packed.copy()).cuda()
        ref = np.frombuffer(bb.mxfp8_unpack_ref(packed, n), dtype=np.int16)
        self.ref = torch.from_numpy(ref.copy()).cuda()


def windows(n):
    """Element windows of an n-element object: empty, whole, inside one tile, across a tile edge, lo / hi on a tile edge and
    one element either side of it, inside the tail tile, and lo % 8 in {0, 1, 7}."""
    last = (n - 1) // T * T
    cand = [(0, 0), (n // 2, n // 2), (0, n), (min(5, n), min(n, 100)), (T - 7, T + 9), (T - 1, n), (T, n), (T + 1, n),
            (0, T - 1), (0, T), (0, T + 1), (2 * T - 1, 2 * T + 1), (last + 1, n - 1), (last, n), (8, n), (1, n), (7, n - 3),
            (17, 17 + 4096), (n - 1, n), (last + 7, last + 9)]
    out = []
    for w in cand:
        if 0 <= w[0] <= w[1] <= n and w not in out:
            out.append(w)
    return out


class Gets:
    """Unpack items reading `obj` into one guard-filled int16 buffer: item k stores window wins[k] (None: the whole tensor)
    at its own region, whose virtual base (region - lo elements) is 16-byte aligned, with guards around it."""

    def __init__(self, objs, wins):
        self.objs, self.wins = objs, wins
        self.regions, o = [], 64
        for obj, w in zip(objs, wins):
            lo, hi = w if w is not None else (0, obj.n)
            r = (o + 7) // 8 * 8 + lo % 8
            self.regions.append(r)
            o = r + hi - lo + 64
        self.dst = torch.full((o + 64,), GUARD, dtype=torch.int16, device="cuda")
        self.items = []
        for obj, w, r in zip(objs, wins, self.regions):
            lo = w[0] if w is not None else 0
            it = (self.dst.data_ptr() + 2 * (r - lo), obj.slab.data_ptr(), obj.n, obj.digest)
            self.items.append(it if w is None else it + (w,))

    def want(self, stored=None):
        want = torch.full_like(self.dst, GUARD)
        for k, (obj, w, r) in enumerate(zip(self.objs, self.wins, self.regions)):
            lo, hi = w if w is not None else (0, obj.n)
            if stored is None or stored[k]:
                want[r:r + hi - lo] = obj.ref[lo:hi]
        return want

    def check(self, what):
        torch.cuda.synchronize()
        want = self.want()
        if not torch.equal(self.dst, want):
            bad = (self.dst != want).nonzero().flatten()[:8].tolist()
            pytest.fail(f"{what}: elements differ at {bad}; regions {self.regions[:8]}")

    def guards_intact(self):
        torch.cuda.synchronize()
        inside = torch.zeros_like(self.dst, dtype=torch.bool)
        for obj, w, r in zip(self.objs, self.wins, self.regions):
            lo, hi = w if w is not None else (0, obj.n)
            inside[r:r + hi - lo] = True
        return bool((self.dst[~inside] == GUARD).all())


# ---------------------------------------------------------------------------------------------------- engine


def test_fp8_windows_at_every_object_size_and_grid(bb, eng):
    """Every window shape of every object size, one batch per size of more than 8 items with whole tensors mixed in, at
    grids of 1, 7, the SM count and twice the SM count, so that windows straddle CTA runs."""
    for n in SIZES:
        obj = Packed(bb, n, n)
        ws = windows(n)
        ws = ws[:3] + [None] + ws[3:] + [None]
        ws += [None] * (9 - len(ws))
        g = Gets([obj] * len(ws), ws)
        assert len(ws) > 8
        for grid in GRIDS:
            eng.set_max_ctas(_grid(grid))
            g.dst.fill_(GUARD)
            dg, st, _ = eng.run_fp8(g.items, True, _stream())
            assert st == [0] * len(ws) and dg == [obj.digest] * len(ws), (n, grid, st)
            g.check(f"n={n} grid={grid}")


def test_fp8_batches_mix_objects_windows_and_whole_tensors(bb, eng):
    objs = [Packed(bb, n, 40 + i) for i, n in enumerate([3 * T + 96, 64, T + 32, 5 * T, 8192])]
    wins = [(T - 1, 2 * T + 3), None, (1, T + 31), None, (8, 8), (T, T + 1), None, (4 * T - 3, 5 * T), (7, 8191), None]
    pick = [0, 1, 2, 3, 4, 0, 2, 3, 4, 0]
    g = Gets([objs[i] for i in pick], wins)
    dg, st, _ = eng.run_fp8(g.items, True, _stream())
    assert st == [0] * len(wins) and dg == [objs[i].digest for i in pick]
    g.check("mixed")


def test_fp8_a_flipped_byte_outside_the_window_fails_verification(bb, eng):
    """Payload and scale bytes are hashed whole: a flip outside the window gives status 1, and still nothing outside the
    window is written."""
    n = 3 * T + 96
    obj = Packed(bb, n, 3)
    w = (T + 5, 2 * T - 3)
    for pos in (100, 3 * T + 50, n + 2, n + n // 32 - 1):  # payload of tile 0, payload of the tail, two scale bytes
        obj.slab[pos] ^= 0x41
        g = Gets([obj, obj], [w, (0, 0)])
        _, st, _ = eng.run_fp8(g.items, True, _stream())
        assert st == [1, 1], (pos, st)
        assert g.guards_intact(), pos
        obj.slab[pos] ^= 0x41
    g = Gets([obj], [w])
    _, st, _ = eng.run_fp8(g.items, True, _stream())
    assert st == [0]
    g.check("restored")


def test_fp8_rejected_windows(bb, eng):
    obj = Packed(bb, 2 * T, 1)
    dst = torch.full((4 * T,), GUARD, dtype=torch.int16, device="cuda")
    d, s = dst.data_ptr(), obj.slab.data_ptr()
    x = torch.zeros(2 * T, dtype=torch.bfloat16, device="cuda")
    slab2 = torch.zeros_like(obj.slab)
    for items, unpack in [([(d, s, 2 * T, obj.digest, (10, 5))], True),        # lo > hi
                          ([(d, s, 2 * T, obj.digest, (0, 2 * T + 1))], True),  # past the object
                          ([(x.data_ptr(), slab2.data_ptr(), 2 * T, 0, (0, 32))], False)]:  # a window on a put
        with pytest.raises(RuntimeError, match="INVALID_ARGUMENT"):
            eng.run_fp8(items, unpack, _stream())
    torch.cuda.synchronize()
    assert bool((dst == GUARD).all()) and bool((slab2 == 0).all())


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


def _range_get(cl, keys, objs, ranges, skew=None):
    """Element-range gets into one guard-filled buffer; returns (error codes, buffer, regions)."""
    regions, o = [], 64
    for i, (lo, c) in enumerate(ranges):
        r = (o + 7) // 8 * 8 + lo % 8 + (skew or {}).get(i, 0)
        regions.append(r)
        o = r + c + 64
    out = torch.full((o + 64,), GUARD, dtype=torch.int16, device="cuda")
    ecs = cl.client.batch_get_device_fp8_range(keys, [out.data_ptr() + 2 * r for r in regions], [ob.n for ob in objs],
                                               [lo for lo, _ in ranges], [c for _, c in ranges], _stream())
    return ecs, out, regions


def _check_ranges(out, regions, objs, ranges, ok):
    want = torch.full_like(out, GUARD)
    for r, obj, (lo, c), good in zip(regions, objs, ranges, ok):
        if good:
            want[r:r + c] = obj.ref[lo:lo + c]
    torch.cuda.synchronize()
    if not torch.equal(out, want):
        pytest.fail(f"range get wrote wrong elements at {(out != want).nonzero().flatten()[:8].tolist()}")


def test_client_fp8_ranges_with_one_and_two_copies(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8rng-rep")
    try:
        objs = [Packed(bb, n, 60 + i) for i, n in enumerate([3 * T + 96, 64, 2 * T])]
        n0, b0 = _counter(cl.client, "device_get_fp8_range_total"), _counter(cl.client, "device_get_fp8_range_bytes_total")
        asked = asked_b = 0
        for rep in (1, 2):
            keys = [f"r{rep}/{i}" for i in range(len(objs))]
            for k, obj in zip(keys, objs):
                _put(bb, cl, k, obj, rep)
            ks, os_, rs = [], [], []
            for k, obj in zip(keys, objs):
                n = obj.n
                for r in [(0, n), (5, 1), (T - 3, 10), (n - 40, 40), (1, n - 9), (7, 33), (n // 2, 0)]:
                    if r[0] + r[1] <= n:
                        ks.append(k), os_.append(obj), rs.append(r)
            l0 = cl.fabric.launches
            ecs, out, regions = _range_get(cl, ks, os_, rs)
            assert ecs == [bb.ErrorCode.OK] * len(ks), ecs
            assert cl.fabric.launches == l0 + 2  # the fused kernel and the scales batch
            _check_ranges(out, regions, os_, rs, [True] * len(ks))
            asked += len(ks)
            asked_b += 2 * sum(c for _, c in rs)
        assert _counter(cl.client, "device_get_fp8_range_total") == n0 + asked
        assert _counter(cl.client, "device_get_fp8_range_bytes_total") == b0 + asked_b
    finally:
        cl.stop()


def test_client_fp8_range_errors_and_a_misaligned_base_fail_alone(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8rng-err")
    try:
        a, b = Packed(bb, 3 * T + 96, 70), Packed(bb, 2 * T, 71)
        _put(bb, cl, "a", a, 1)
        _put(bb, cl, "b", b, 1)
        E = bb.ErrorCode
        cases = [("a", a, (T - 3, 100), 0, E.OK),
                 ("a", a, (a.n - 10, 11), 0, E.VALUE_OUT_OF_RANGE),
                 ("b", b, (2**64 - 8, 16), 0, E.VALUE_OUT_OF_RANGE),
                 ("missing", b, (0, 32), 0, E.OBJECT_NOT_FOUND),
                 ("b", b, (40, 0), 0, E.OK),
                 ("a", a, (5, 2 * T), 3, E.NOT_IMPLEMENTED),  # virtual base 6 bytes off
                 ("b", b, (0, b.n), 0, E.OK),
                 ("a", a, (a.n - 33, 33), 0, E.OK)]
        skew = {i: c[3] for i, c in enumerate(cases)}
        objs, ranges = [c[1] for c in cases], [c[2] for c in cases]
        l0 = cl.fabric.launches
        ecs, out, regions = _range_get(cl, [c[0] for c in cases], objs, ranges, skew)
        range_launches = cl.fabric.launches - l0
        assert ecs == [c[4] for c in cases], ecs
        _check_ranges(out, regions, objs, ranges, [e == E.OK for e in ecs])
        # the same objects read whole: one attempt costs the same launches
        outs = [torch.empty(o.n, dtype=torch.int16, device="cuda") for o in (a, b)]
        l0 = cl.fabric.launches
        assert cl.client.batch_get_device_fp8(["a", "b"], [o.data_ptr() for o in outs], [a.n, b.n], _stream()) == [E.OK, E.OK]
        assert range_launches == cl.fabric.launches - l0 == 2
        torch.cuda.synchronize()
        assert torch.equal(outs[0], a.ref) and torch.equal(outs[1], b.ref)
    finally:
        cl.stop()


def test_client_fp8_range_fails_over_from_a_copy_corrupt_outside_the_window(bb):
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=64 << 20, cluster_id="t-fp8rng-fo")
    try:
        obj = Packed(bb, 3 * T + 96, 80)
        shards = _put(bb, cl, "f", obj, 2)
        r = (T + 100, 300)
        for pos in (obj.n - 5, obj.n + obj.n // 32 - 1):  # a payload byte and the last scale byte, outside the window
            fo = _counter(cl.client, "replica_failover_total")
            for sh in shards:  # one copy at a time is corrupt: exactly one of the two gets starts on it
                _flip(cl, sh, pos)
                ecs, out, regions = _range_get(cl, ["f"], [obj], [r])
                assert ecs == [bb.ErrorCode.OK]
                _check_ranges(out, regions, [obj], [r], [True])
                _flip(cl, sh, pos)
            assert _counter(cl.client, "replica_failover_total") == fo + 1, pos
        for sh in shards:
            _flip(cl, sh, 9)
        ecs, out, regions = _range_get(cl, ["f"], [obj], [r])
        assert ecs == [bb.ErrorCode.CHECKSUM_MISMATCH]
        torch.cuda.synchronize()
        outside = torch.ones_like(out, dtype=torch.bool)
        outside[regions[0]:regions[0] + r[1]] = False
        assert bool((out[outside] == GUARD).all())
    finally:
        cl.stop()


# ---------------------------------------------------------------------------------------------------- TensorStore


def test_tensor_store_get_rows_of_packed_tensors(bb):
    from blackbird_b200.ops.tensor_store import TensorStore
    from blackbird_b200.parallel import GpuRankCluster

    cl = GpuRankCluster(slab_bytes=128 << 20, cluster_id="t-fp8rng-rows")
    try:
        store = TensorStore(cl.client)
        g = torch.Generator(device="cuda").manual_seed(9)
        ts = {"kv": torch.randn(64, 2, 512, device="cuda", generator=g).to(torch.bfloat16),   # rows of 1024 elements
              "odd": torch.randn(96, 37, device="cuda", generator=g).to(torch.bfloat16),      # rows of 37: lo % 8 varies
              "pad": torch.randn(7, 9, device="cuda", generator=g).to(torch.bfloat16),        # 63 elements, padded to 64
              "big": torch.randn(40, 4099, device="cuda", generator=g).to(torch.bfloat16)}    # rows across tile edges
        for k, t in ts.items():
            store.put(k, t, pack_fp8=True)
        whole = {k: store.get(k) for k in ts}
        cases = [("kv", 0, 64), ("kv", 3, 4), ("kv", 17, 40), ("odd", 1, 2), ("odd", 5, 96), ("odd", 95, 96), ("odd", 8, 8),
                 ("pad", 0, 7), ("pad", 6, 7), ("pad", 2, 5), ("big", 3, 9), ("big", 39, 40)]
        f0 = _counter(cl.client, "device_get_fp8_range_total")
        for k, a, b in cases:
            got = store.get_rows(k, a, b)
            assert got.dtype == torch.bfloat16 and got.shape == whole[k][a:b].shape, (k, a, b)
            assert torch.equal(got.view(torch.int16), whole[k][a:b].view(torch.int16)), (k, a, b)
        assert _counter(cl.client, "device_get_fp8_range_total") == f0 + len(cases)
        outs = store.batch_get_rows([k for k, _, _ in cases], [a for _, a, _ in cases], [b for _, _, b in cases])
        assert _counter(cl.client, "device_get_fp8_range_total") == f0 + 2 * len(cases)
        spans = []
        for o, (k, a, b) in zip(outs, cases):
            assert torch.equal(o.view(torch.int16), whole[k][a:b].view(torch.int16)), (k, a, b)
            if o.numel():
                spans.append((o.data_ptr(), o.data_ptr() + 2 * o.numel()))
        spans.sort()
        assert all(e <= s for (_, e), (s, _) in zip(spans, spans[1:])), "results alias each other"
        # a packed tensor striped over the workers of a copy (unfused put) reads back through the whole-get fallback
        cfg = bb.WorkerConfig(replication_factor=1, max_workers_per_copy=2, ttl_ms=0, preferred_classes=[bb.StorageClass.RAM_GPU],
                              checksum=bb.ChecksumAlgo.XXH3)
        x = torch.randn(50, 64, device="cuda", generator=g).to(torch.bfloat16)
        store.put("striped", x, pack_fp8=True, config=cfg)
        f1 = _counter(cl.client, "device_get_fp8_range_total")
        assert torch.equal(store.get_rows("striped", 10, 31).view(torch.int16), store.get("striped")[10:31].view(torch.int16))
        assert _counter(cl.client, "device_get_fp8_range_total") == f1
    finally:
        cl.stop()
